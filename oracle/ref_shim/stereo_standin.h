// stereo_standin.h — declarations the reference's stereo step (matchGrid, GridStructure, LineIterator, matchStereoPoints,
// matchStereoLines and their helpers) needs, so that oracle/make_ref_stereo.py can compile those definitions from the
// reference's own text.
//
// TEST INFRASTRUCTURE (oracle/_ref).  Everything in this file is OURS: a minimal cv::Mat of 32-byte descriptor rows,
// cv::KeyPoint and KeyLine with the fields the step reads, the Config accessors with the reference's names, and the
// class declarations with the reference's member names.  No definition here is the reference's.
#pragma once
#include <cstdint>
#include <cstring>
#include <limits>
#include <list>
#include <stdexcept>
#include <unordered_set>
#include <utility>
#include <vector>

#include "eigen_standin.h"

// ---- cv: descriptors are CV_8U rows of 32 bytes; the step only reads rows, pushes rows and copies ----
namespace cv {

class Mat {
public:
    int rows = 0, cols = 32;
    std::vector<uint8_t> data;
    Mat() {}
    Mat(int r, const uint8_t* src) : rows(r), data(src, src + (size_t)r * 32) {}
    Mat row(int i) const { return Mat(1, data.data() + (size_t)i * 32); }
    template <typename T> T* ptr() { return reinterpret_cast<T*>(data.data()); }
    template <typename T> const T* ptr() const { return reinterpret_cast<const T*>(data.data()); }
    void push_back(const Mat& m) {
        data.insert(data.end(), m.data.begin(), m.data.end());
        rows += m.rows;
    }
    void copyTo(Mat& dst) const { dst = *this; }
    bool empty() const { return rows == 0; }
};

struct Point2f {
    float x = 0.f, y = 0.f;
};

struct KeyPoint {
    Point2f pt;
    int octave = 0;
};

}  // namespace cv

struct KeyLine {   // cv::line_descriptor::KeyLine: the fields matchStereoLines reads
    float angle = 0.f;
    int octave = 0;
    float startPointX = 0.f, startPointY = 0.f, endPointX = 0.f, endPointY = 0.f;
};

using namespace cv;
using namespace std;
using namespace Eigen;

// the Config values the stereo step reads; same accessor signatures as include/config.h (static, by reference)
class Config {
public:
    static Config& getInstance() { static Config c; return c; }
    static bool& hasPoints() { return getInstance().has_points; }
    static bool& hasLines() { return getInstance().has_lines; }
    static bool& bestLRMatches() { return getInstance().best_lr_matches; }
    static int& matchingSWs() { return getInstance().matching_s_ws; }
    static double& orbScaleFactor() { return getInstance().orb_scale_factor; }
    static double& maxDistEpip() { return getInstance().max_dist_epip; }
    static double& minDisp() { return getInstance().min_disp; }
    static double& minRatio12P() { return getInstance().min_ratio_12_p; }
    static double& lsdScale() { return getInstance().lsd_scale; }
    static double& lineHorizTh() { return getInstance().line_horiz_th; }
    static double& stereoOverlapTh() { return getInstance().stereo_overlap_th; }
    static double& lineSimTh() { return getInstance().line_sim_th; }
    static double& lsMinDispRatio() { return getInstance().ls_min_disp_ratio; }
    bool has_points = true, has_lines = true, best_lr_matches = true;
    int matching_s_ws = 10;
    double orb_scale_factor = 1.2, max_dist_epip = 1.0, min_disp = 1.0, min_ratio_12_p = 0.9, lsd_scale = 1.2,
           line_horiz_th = 0.1, stereo_overlap_th = 0.75, line_sim_th = 0.75, ls_min_disp_ratio = 0.7;
};

// include/stereoFrame.h:51-52 fixes the grid at 48 x 64; here both are settable so every configured grid can be compared
extern int g_grid_rows, g_grid_cols;
#define GRID_ROWS g_grid_rows
#define GRID_COLS g_grid_cols

class PinholeStereoCamera {
public:
    int width, height;
    double fx, fy, cx, cy, b;
    Vector3d backProjection(const double& u, const double& v, const double& disp);
};

namespace StVO {

typedef std::pair<int, int> point_2d;          // include/matching.h:36-37
typedef std::pair<point_2d, point_2d> line_2d;

struct GridWindow {
    std::pair<int, int> width, height;
};

class GridStructure {
public:
    int rows, cols;
    GridStructure(int rows, int cols);
    ~GridStructure();
    std::list<int>& at(int x, int y);
    void get(int x, int y, const GridWindow& w, std::unordered_set<int>& indices) const;
    void clear();

private:
    std::vector<std::vector<std::list<int>>> grid;
    std::list<int> out_of_bounds;
};

void getLineCoords(double x1, double y1, double x2, double y2, std::list<std::pair<int, int>>& line_coords);

class LineIterator {
public:
    LineIterator(const double x1_, const double y1_, const double x2_, const double y2_);
    bool getNext(std::pair<int, int>& pixel);

private:
    const bool steep;
    double x1, y1, x2, y2;
    double dx, dy, error;
    int maxX, ystep;
    int y, x;
};

class PointFeature {
public:
    PointFeature(Vector2d pl_, double disp_, Vector3d P_, int idx_, int level_);
    Vector2d pl;
    double disp;
    Vector3d P;
    bool inlier;
    int idx;
    int level;
    double sigma2 = 1.0;
};

class LineFeature {
public:
    LineFeature(Vector2d spl_, double sdisp_, Vector3d sP_, Vector2d epl_, double edisp_, Vector3d eP_, Vector3d le_,
                double angle_, int idx_, int level_);
    Vector2d spl;
    double sdisp;
    Vector3d sP;
    Vector2d epl;
    double edisp;
    Vector3d eP;
    Vector3d le;
    bool inlier;
    int idx;
    double angle;
    int level;
    double sigma2 = 1.0;
};

class StereoFrame {
public:
    void matchStereoPoints(vector<KeyPoint> points_l, vector<KeyPoint> points_r, Mat& pdesc_l_, Mat pdesc_r, bool initial = false);
    void matchStereoLines(vector<KeyLine> lines_l, vector<KeyLine> lines_r, Mat& ldesc_l_, Mat ldesc_r, bool initial = false);
    void filterLineSegmentDisparity(Vector2d spl, Vector2d epl, Vector2d spr, Vector2d epr, double& disp_s, double& disp_e);
    double lineSegmentOverlapStereo(double spl_obs, double epl_obs, double spl_proj, double epl_proj);

    vector<PointFeature*> stereo_pt;
    vector<LineFeature*> stereo_ls;
    Mat pdesc_l, pdesc_r, ldesc_l, ldesc_r;
    PinholeStereoCamera* cam;
    double inv_width, inv_height;
};

}  // namespace StVO
