// C entry points of oracle/_ref/libplstvo_ref_stereo.so: the reference's stereo step (matchGrid for points and lines,
// GridStructure, LineIterator, matchStereoPoints / matchStereoLines and the helpers they call) compiled from its own text,
// which oracle/make_ref_stereo.py cuts into oracle/_ref/extracted_stereo.inc.  Bound by oracle/stereo_ref.py.
#include "stereo_standin.h"
#include "include/plstvo.h"

int g_grid_rows = 48, g_grid_cols = 64;

#include "extracted_stereo_cam.inc"
namespace StVO {
#include "extracted_stereo.inc"
}  // namespace StVO

using namespace StVO;

namespace {

Mat rows_of(int n, const uint8_t* d) { return n > 0 ? Mat(n, d) : Mat(); }

void set_match_config(const PlStereoMatchConfig* mc) {
    g_grid_rows = mc->grid_rows;
    g_grid_cols = mc->grid_cols;
    Config::matchingSWs() = mc->matching_s_ws;
    Config::bestLRMatches() = mc->best_lr_matches != 0;
    Config::minRatio12P() = mc->min_ratio_12_p;
    Config::lineSimTh() = mc->line_sim_th;
}

void set_stereo_config(const PlStereoConfig* sc) {
    Config::maxDistEpip() = sc->max_dist_epip;
    Config::minDisp() = sc->min_disp;
    Config::lsMinDispRatio() = sc->ls_min_disp_ratio;
    Config::lineHorizTh() = sc->line_horiz_th;
    Config::stereoOverlapTh() = sc->stereo_overlap_th;
    Config::orbScaleFactor() = sc->orb_scale_factor;
    Config::lsdScale() = sc->lsd_scale;
}

GridWindow window(PlGridWindow w) {
    GridWindow g;
    g.width = std::make_pair(w.left, w.right);
    g.height = std::make_pair(w.up, w.down);
    return g;
}

// a StereoFrame with the grid scale of its constructor (src/stereoFrame.cpp:47-48) for a camera's image size
struct Frame {
    PinholeStereoCamera cam;
    StereoFrame f;
    explicit Frame(const PlCamera* c) {
        cam.width = c->width;
        cam.height = c->height;
        cam.fx = c->fx;
        cam.fy = c->fy;
        cam.cx = c->cx;
        cam.cy = c->cy;
        cam.b = c->b;
        f.cam = &cam;
        f.inv_width = GRID_COLS / static_cast<double>(c->width);
        f.inv_height = GRID_ROWS / static_cast<double>(c->height);
    }
    ~Frame() {
        for (auto p : f.stereo_pt) delete p;
        for (auto l : f.stereo_ls) delete l;
    }
};

void put2(double* o, const Vector2d& v) { o[0] = v(0); o[1] = v(1); }
void put3(double* o, const Vector3d& v) { o[0] = v(0); o[1] = v(1); o[2] = v(2); }

}  // namespace

extern "C" {

// matchGrid, points: the train grid filled as matchStereoPoints fills it (:135-139), from integer cells
int stereo_ref_match_grid_points(int rows, int cols, PlGridWindow w, int best_lr, double ratio, int n1, const int32_t* q_cell,
                                 const uint8_t* d1, int n2, const int32_t* t_cell, const uint8_t* d2, int32_t* m12) {
    Config::bestLRMatches() = best_lr != 0;
    Config::minRatio12P() = ratio;
    std::vector<point_2d> coords;
    for (int i = 0; i < n1; ++i) coords.push_back(std::make_pair(q_cell[2 * i], q_cell[2 * i + 1]));
    GridStructure grid(rows, cols);
    for (int idx = 0; idx < n2; ++idx) grid.at(t_cell[2 * idx], t_cell[2 * idx + 1]).push_back(idx);
    std::vector<int> matches_12;
    const int n = matchGrid(coords, rows_of(n1, d1), grid, rows_of(n2, d2), window(w), matches_12);
    for (int i = 0; i < n1; ++i) m12[i] = matches_12[(size_t)i];
    return n;
}

// matchGrid, lines: the train grid filled through getLineCoords as matchStereoLines fills it (:326-339); t_dir as given
int stereo_ref_match_grid_lines(int rows, int cols, PlGridWindow w, int best_lr, double ratio, double line_sim_th, int n1,
                                const int32_t* q_line, const uint8_t* d1, int n2, const double* t_line, const double* t_dir,
                                const uint8_t* d2, int32_t* m12) {
    Config::bestLRMatches() = best_lr != 0;
    Config::minRatio12P() = ratio;
    Config::lineSimTh() = line_sim_th;
    std::vector<line_2d> coords;
    for (int i = 0; i < n1; ++i) {
        const int32_t* q = q_line + 4 * (size_t)i;
        coords.push_back(std::make_pair(std::make_pair(q[0], q[1]), std::make_pair(q[2], q[3])));
    }
    GridStructure grid(rows, cols);
    std::vector<std::pair<double, double>> directions((size_t)n2);
    std::list<std::pair<int, int>> line_coords;
    for (int idx = 0; idx < n2; ++idx) {
        const double* L = t_line + 4 * (size_t)idx;
        directions[(size_t)idx] = std::make_pair(t_dir[2 * idx], t_dir[2 * idx + 1]);
        getLineCoords(L[0], L[1], L[2], L[3], line_coords);
        for (const std::pair<int, int>& p : line_coords) grid.at(p.first, p.second).push_back(idx);
    }
    std::vector<int> matches_12;
    const int n = matchGrid(coords, rows_of(n1, d1), grid, rows_of(n2, d2), directions, window(w), matches_12);
    for (int i = 0; i < n1; ++i) m12[i] = matches_12[(size_t)i];
    return n;
}

// getLineCoords: the cells LineIterator visits, up to cap of them; returns how many it visits
int stereo_ref_line_cells(double x1, double y1, double x2, double y2, int32_t* cells, int cap) {
    std::list<std::pair<int, int>> line_coords;
    getLineCoords(x1, y1, x2, y2, line_coords);
    int n = 0;
    for (const std::pair<int, int>& p : line_coords) {
        if (n < cap) { cells[2 * n] = p.first; cells[2 * n + 1] = p.second; }
        ++n;
    }
    return n;
}

double stereo_ref_line_segment_overlap_stereo(const PlStereoConfig* sc, double spl_obs, double epl_obs, double spl_proj,
                                              double epl_proj) {
    set_stereo_config(sc);
    StereoFrame f;
    return f.lineSegmentOverlapStereo(spl_obs, epl_obs, spl_proj, epl_proj);
}

// matchStereoPoints on one frame's raw key points: the PointFeature records in order and the rewritten pdesc_l rows
int stereo_ref_match_stereo_points(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l,
                                   const float* kp_l, const int32_t* octave_l, const uint8_t* desc_l, int n_r, const float* kp_r,
                                   const uint8_t* desc_r, double* pl, double* disp, double* P, double* sigma2, int32_t* level,
                                   uint8_t* desc_out) {
    set_match_config(mc);
    set_stereo_config(sc);
    Frame fr(cam);
    std::vector<KeyPoint> points_l((size_t)n_l), points_r((size_t)n_r);
    for (int i = 0; i < n_l; ++i) {
        points_l[(size_t)i].pt.x = kp_l[2 * i];
        points_l[(size_t)i].pt.y = kp_l[2 * i + 1];
        points_l[(size_t)i].octave = octave_l[i];
    }
    for (int i = 0; i < n_r; ++i) {
        points_r[(size_t)i].pt.x = kp_r[2 * i];
        points_r[(size_t)i].pt.y = kp_r[2 * i + 1];
    }
    fr.f.pdesc_l = rows_of(n_l, desc_l);
    fr.f.pdesc_r = rows_of(n_r, desc_r);
    fr.f.matchStereoPoints(points_l, points_r, fr.f.pdesc_l, fr.f.pdesc_r, true);
    const int k = (int)fr.f.stereo_pt.size();
    for (int i = 0; i < k; ++i) {
        const PointFeature* p = fr.f.stereo_pt[(size_t)i];
        put2(pl + 2 * i, p->pl);
        disp[i] = p->disp;
        put3(P + 3 * i, p->P);
        sigma2[i] = p->sigma2;
        level[i] = p->level;
    }
    if (k) std::memcpy(desc_out, fr.f.pdesc_l.ptr<uint8_t>(), (size_t)k * 32);
    return k;
}

// matchStereoLines on one frame's raw key lines (seg rows: startPointX, startPointY, endPointX, endPointY)
int stereo_ref_match_stereo_lines(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l,
                                  const float* seg_l, const float* angle_l, const int32_t* octave_l, const uint8_t* desc_l,
                                  int n_r, const float* seg_r, const uint8_t* desc_r, double* spl, double* epl, double* sdisp,
                                  double* edisp, double* sP, double* eP, double* le, double* angle, double* sigma2,
                                  int32_t* level, uint8_t* desc_out) {
    set_match_config(mc);
    set_stereo_config(sc);
    Frame fr(cam);
    std::vector<KeyLine> lines_l((size_t)n_l), lines_r((size_t)n_r);
    for (int i = 0; i < n_l; ++i) {
        KeyLine& k = lines_l[(size_t)i];
        k.startPointX = seg_l[4 * i];
        k.startPointY = seg_l[4 * i + 1];
        k.endPointX = seg_l[4 * i + 2];
        k.endPointY = seg_l[4 * i + 3];
        k.angle = angle_l[i];
        k.octave = octave_l[i];
    }
    for (int i = 0; i < n_r; ++i) {
        KeyLine& k = lines_r[(size_t)i];
        k.startPointX = seg_r[4 * i];
        k.startPointY = seg_r[4 * i + 1];
        k.endPointX = seg_r[4 * i + 2];
        k.endPointY = seg_r[4 * i + 3];
    }
    fr.f.ldesc_l = rows_of(n_l, desc_l);
    fr.f.ldesc_r = rows_of(n_r, desc_r);
    fr.f.matchStereoLines(lines_l, lines_r, fr.f.ldesc_l, fr.f.ldesc_r, true);
    const int k = (int)fr.f.stereo_ls.size();
    for (int i = 0; i < k; ++i) {
        const LineFeature* l = fr.f.stereo_ls[(size_t)i];
        put2(spl + 2 * i, l->spl);
        put2(epl + 2 * i, l->epl);
        sdisp[i] = l->sdisp;
        edisp[i] = l->edisp;
        put3(sP + 3 * i, l->sP);
        put3(eP + 3 * i, l->eP);
        put3(le + 3 * i, l->le);
        angle[i] = l->angle;
        sigma2[i] = l->sigma2;
        level[i] = l->level;
    }
    if (k) std::memcpy(desc_out, fr.f.ldesc_l.ptr<uint8_t>(), (size_t)k * 32);
    return k;
}

}  // extern "C"
