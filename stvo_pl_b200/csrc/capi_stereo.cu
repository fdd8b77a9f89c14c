// capi_stereo.cu — the C-ABI's stereo step: matchGrid, 3-D lifting, matchStereo in one device pass, and pose tracking from
// raw stereo features (the stereo step feeding the tracker without leaving HBM).
#include "host.cuh"

using namespace plstvo;

namespace {

int check_stereo_offsets(PlContext* ctx, int B, const int32_t* l_off, const int32_t* r_off) {
    return check_offsets(ctx, B, {l_off, r_off}, "bad offsets", "offsets are not non-decreasing", "more than 65535 features");
}

}  // namespace

namespace plstvo {

int StereoSet::check(PlContext* ctx) {
    if (const int rc = check_stereo_offsets(ctx, nf, l_off, r_off)) return rc;
    N1 = l_off[nf];
    N2 = r_off[nf];
    if ((N1 && (!xy_l || (!oct && !on_device) || !d1 || (lines && !ang) || (lift_only && !m12))) ||
        (N2 && (!xy_r || (!d2 && !lift_only))))
        return fail(ctx, PLSTVO_E_INVALID, "null input array");
    return 0;
}

void StereoSet::take(Arena& a) {
    const size_t cw = lines ? 4 : 2;   // floats per key point / segment
    auto host = [&](const void* p, size_t bytes) { return a.take(p && !on_device ? bytes : 0); };
    o_loff = a.take((size_t)(nf + 1) * 4);
    o_roff = a.take((size_t)(nf + 1) * 4);
    o_xyl = host(xy_l, N1 * cw * 4);
    o_xyr = host(xy_r, N2 * cw * 4);
    o_ang = a.take(lines ? N1 * 4 : 0);
    o_oct = a.take(on_device && oct ? 0 : N1 * 4);
    o_d1 = host(d1, N1 * 32);
    o_d2 = host(d2, N2 * 32);
    o_m12 = a.take(N1 * 4);
    o_cnt = a.take((size_t)nf * 4);
    o_gcnt = a.take(lift_only ? 0 : (size_t)nf * 4);
    o_prob = a.take(lift_only ? 0 : (size_t)nf * sizeof(GridProblem));
}

cudaError_t StereoSet::upload(const Arena& a, cudaStream_t s, const GridScratch* g, GridProblem* probs) const {
    const size_t cw = lines ? 4 : 2;
    if (g) g->fill(probs, nf, lines, l_off, r_off, in(a, d1, o_d1), in(a, d2, o_d2), a.i32(o_m12), a.i32(o_gcnt));
    cudaError_t e = cudaSuccess;
    auto up = [&](size_t o, const void* src, size_t bytes) { if (!e) e = a.up(o, src, bytes, s); };
    up(o_loff, l_off, (size_t)(nf + 1) * 4);
    up(o_roff, r_off, (size_t)(nf + 1) * 4);
    if (lines) up(o_ang, ang, N1 * 4);
    if (!on_device) {
        up(o_xyl, xy_l, N1 * cw * 4);
        up(o_xyr, xy_r, N2 * cw * 4);
        up(o_oct, oct, N1 * 4);
        up(o_d1, d1, N1 * 32);
        up(o_d2, d2, N2 * 32);
    } else if (!oct && N1 && !e) {
        e = cudaMemsetAsync(a.u8(o_oct), 0, N1 * 4, s);   // key lines of octave 0
    }
    up(o_m12, m12, N1 * 4);
    if (g) up(o_prob, probs, (size_t)nf * sizeof(GridProblem));
    return e;
}

cudaError_t StereoSet::match(const Arena& a, const GridScratch& g, const PlCamera& cam, const PlStereoMatchConfig& mc,
                             cudaStream_t s) const {
    // grid coordinates (src/stereoFrame.cpp:47-48: inv_width = GRID_COLS / image width, inv_height = GRID_ROWS / image height)
    const int rows = mc.grid_rows, cols = mc.grid_cols;
    const double inv_w = cols / static_cast<double>(cam.width), inv_h = rows / static_cast<double>(cam.height);
    const float *kl = in(a, xy_l, o_xyl), *kr = in(a, xy_r, o_xyr);
    const int n1 = (int)N1, n2 = (int)N2;
    const cudaError_t e =
        lines ? launch_stereo_cells_lines(n1, n2, inv_w, inv_h, kl, kr, a.i32(g.qcell), a.f64(g.tline), a.f64(g.tdir), s)
              : launch_stereo_cells_points(n1, n2, inv_w, inv_h, kl, kr, a.i32(g.qcell), a.i32(g.tcell), s);
    if (e) return e;
    // matchGrid with the stereo window (:141-143, :340-342: matching_s_ws cells to the left, same row)
    const GridParams prm{rows, cols, GRID_CAP, mc.best_lr_matches ? 1 : 0, PlGridWindow{mc.matching_s_ws, 0, 0, 0},
                         mc.min_ratio_12_p, mc.line_sim_th};
    return launch_match_grid(a.at<GridProblem>(o_prob), nf, prm, lines, s);
}

cudaError_t StereoSet::lift(const Arena& a, const PlCamera& cam, const PlStereoConfig& sc, int n, int first,
                            const RecPtrs& out, cudaStream_t s, const int32_t* out_off, const PlCamera* cams) const {
    const int32_t *lo = a.i32(o_loff) + first, *ro = a.i32(o_roff) + first, *o = in(a, oct, o_oct);
    const float *kl = in(a, xy_l, o_xyl), *kr = in(a, xy_r, o_xyr);
    const uint8_t* dl = in(a, d1, o_d1);
    int32_t* cnt = a.i32(o_cnt) + first;
    if (lines)
        return launch_lift_lines(cam, sc, n, lo, kl, a.f32(o_ang), o, dl, ro, kr, a.i32(o_m12), out, cnt, s, out_off, cams);
    return launch_lift_points(cam, sc, n, lo, kl, o, dl, ro, kr, a.i32(o_m12), out, cnt, s, out_off, cams);
}

}  // namespace plstvo

namespace {

// stand-alone lifting of st (lift_only) into out (host)
int stereo_lift(PlContext* ctx, const PlCamera* cam, const PlStereoConfig* scfg, StereoSet st, const RecPtrs& out,
                int32_t* counts) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (!cam || !scfg || st.nf < 0) return fail(ctx, PLSTVO_E_INVALID, "null camera / config or negative batch size");
    if (st.nf == 0) return 0;
    if (const int rc = st.check(ctx)) return rc;
    CK(ctx, cudaSetDevice(ctx->device));
    Arena a;
    st.take(a);
    const int first = st.lines ? LS_SPL : PT_PL, last = st.lines ? N_LIFT : LS_SPL;
    size_t o_rec[N_REC];
    take_records(a, st.N1, first, last, o_rec);
    CK(ctx, a.alloc(st.lines ? ctx->arena_lift_ls : ctx->arena_lift_pt));
    cudaStream_t s = ctx->s_main;
    CK(ctx, st.upload(a, s));
    CK(ctx, st.lift(a, *cam, *scfg, st.nf, 0, arena_records(a, o_rec, first, last), s));
    ctx->launches++;
    CK(ctx, down_records(a, out, o_rec, st.N1, first, last, s));
    return counts_total(ctx, s, st.nf, a.i32(st.o_cnt), counts);
}

}  // namespace

extern "C" {

// ---- matchGrid (stereo step) -------------------------------------------------------------------------------------
static int match_grid_common(PlContext* ctx, bool lines, int B, int rows, int cols, PlGridWindow w, int best_lr,
                             double ratio, double line_sim_th, const int32_t* q_off, const int32_t* q_cell,
                             const uint8_t* d1, const int32_t* t_off, const int32_t* t_cell, const double* t_line,
                             const double* t_dir, const uint8_t* d2, int32_t* m12, int32_t* counts) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (B < 0 || !grid_ok(rows, cols)) return fail(ctx, PLSTVO_E_INVALID, "bad grid");
    if (B == 0) return 0;
    if (!m12) return fail(ctx, PLSTVO_E_INVALID, "bad offsets");
    if (const int rc = check_stereo_offsets(ctx, B, q_off, t_off)) return rc;
    CK(ctx, cudaSetDevice(ctx->device));
    const int qw = lines ? 4 : 2;
    const size_t N1 = q_off[B], N2 = t_off[B];
    if ((N1 && (!q_cell || !d1)) || (N2 && (!d2 || (lines ? (!t_line || !t_dir) : !t_cell))))
        return fail(ctx, PLSTVO_E_INVALID, "null input array");
    // one arena for inputs, outputs and scratch
    Arena a;
    const size_t o_d1 = a.take(N1 * 32), o_d2 = a.take(N2 * 32), o_m12 = a.take(N1 * 4), o_cnt = a.take((size_t)B * 4);
    const GridScratch g(a, rows, cols, B, N1, N2, N2 * grid_cells_per_train(lines, rows, cols), !lines, lines);
    const size_t o_prob = a.take((size_t)B * sizeof(GridProblem));
    CK(ctx, a.alloc(ctx->arena_grid));
    std::vector<GridProblem> probs((size_t)B);
    g.fill(probs.data(), B, lines, q_off, t_off, a.u8(o_d1), a.u8(o_d2), a.i32(o_m12), a.i32(o_cnt));
    cudaStream_t s = ctx->s_main;
    CK(ctx, a.up(g.qcell, q_cell, N1 * qw * 4, s));
    CK(ctx, a.up(o_d1, d1, N1 * 32, s));
    CK(ctx, a.up(o_d2, d2, N2 * 32, s));
    if (lines) {
        CK(ctx, a.up(g.tline, t_line, N2 * 32, s));
        CK(ctx, a.up(g.tdir, t_dir, N2 * 16, s));
    } else {
        CK(ctx, a.up(g.tcell, t_cell, N2 * 8, s));
    }
    CK(ctx, a.up(o_prob, probs.data(), (size_t)B * sizeof(GridProblem), s));
    GridParams prm{rows, cols, GRID_CAP, best_lr ? 1 : 0, w, ratio, line_sim_th};
    CK(ctx, launch_match_grid(a.at<GridProblem>(o_prob), B, prm, lines, s));
    ctx->launches++;
    CK(ctx, a.down(m12, o_m12, N1 * 4, s));
    return counts_total(ctx, s, B, a.i32(o_cnt), counts, a.i32(o_cnt));
}

int plstvo_match_grid_points(PlContext* ctx, int B, int grid_rows, int grid_cols, PlGridWindow w, int best_lr_matches,
                             double min_ratio_12_p, const int32_t* q_off, const int32_t* q_cell, const uint8_t* d1,
                             const int32_t* t_off, const int32_t* t_cell, const uint8_t* d2, int32_t* m12,
                             int32_t* counts) {
    return match_grid_common(ctx, false, B, grid_rows, grid_cols, w, best_lr_matches, min_ratio_12_p, 0.0, q_off, q_cell, d1,
                             t_off, t_cell, nullptr, nullptr, d2, m12, counts);
}

int plstvo_match_grid_lines(PlContext* ctx, int B, int grid_rows, int grid_cols, PlGridWindow w, int best_lr_matches,
                            double min_ratio_12_p, double line_sim_th, const int32_t* q_off, const int32_t* q_line,
                            const uint8_t* d1, const int32_t* t_off, const double* t_line, const double* t_dir,
                            const uint8_t* d2, int32_t* m12, int32_t* counts) {
    return match_grid_common(ctx, true, B, grid_rows, grid_cols, w, best_lr_matches, min_ratio_12_p, line_sim_th, q_off,
                             q_line, d1, t_off, nullptr, t_line, t_dir, d2, m12, counts);
}

// ---- 3-D lifting of the stereo matches (src/stereoFrame.cpp:149-172, :348-397) ------------------------------
void plstvo_default_stereo_config(PlStereoConfig* c) {   // src/config.cpp:58-69, :96, :106
    if (!c) return;
    c->max_dist_epip = 1.0; c->min_disp = 1.0; c->ls_min_disp_ratio = 0.7; c->line_horiz_th = 0.1;
    c->stereo_overlap_th = 0.75; c->orb_scale_factor = 1.2; c->lsd_scale = 1.2;
}

int plstvo_stereo_lift_points(PlContext* ctx, const PlCamera* cam, const PlStereoConfig* scfg, int B, const int32_t* l_off,
                              const float* kp_l, const int32_t* octave_l, const uint8_t* desc_l, const int32_t* r_off,
                              const float* kp_r, const int32_t* m12, double* pt_pl, double* pt_disp, double* pt_P,
                              double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out, int32_t* src_idx, int32_t* counts) {
    const StereoSet st{false, B, l_off, r_off, nullptr, false, kp_l, kp_r, octave_l, desc_l, nullptr, true, m12};
    const RecPtrs out = RecPtrs::from(PT_PL, {pt_pl, pt_disp, pt_P, pt_sigma2, pt_level, pdesc_out, src_idx});
    return stereo_lift(ctx, cam, scfg, st, out, counts);
}

int plstvo_stereo_lift_lines(PlContext* ctx, const PlCamera* cam, const PlStereoConfig* scfg, int B, const int32_t* l_off,
                             const float* seg_l, const float* angle_l, const int32_t* octave_l, const uint8_t* desc_l,
                             const int32_t* r_off, const float* seg_r, const int32_t* m12, double* ls_spl, double* ls_epl,
                             double* ls_sdisp, double* ls_edisp, double* ls_sP, double* ls_eP, double* ls_le,
                             double* ls_angle, double* ls_sigma2, int32_t* ls_level, uint8_t* ldesc_out, int32_t* src_idx,
                             int32_t* counts) {
    const StereoSet st{true, B, l_off, r_off, angle_l, false, seg_l, seg_r, octave_l, desc_l, nullptr, true, m12};
    const RecPtrs out = RecPtrs::from(LS_SPL, {ls_spl, ls_epl, ls_sdisp, ls_edisp, ls_sP, ls_eP, ls_le, ls_angle, ls_sigma2,
                                               ls_level, ldesc_out, src_idx});
    return stereo_lift(ctx, cam, scfg, st, out, counts);
}

// ---- matchStereoPoints / matchStereoLines in one device pass (src/stereoFrame.cpp:120-173, :309-398) ----------------
void plstvo_default_stereo_match_config(PlStereoMatchConfig* c) {   // include/stereoFrame.h:51-52, src/config.cpp:51, :60, :63, :91
    if (!c) return;
    c->grid_rows = 48; c->grid_cols = 64; c->matching_s_ws = 10; c->best_lr_matches = 1;
    c->min_ratio_12_p = 0.9; c->line_sim_th = 0.75;
}

namespace {
// out: the host destinations of the set's lifted records
int match_stereo_common(PlContext* ctx, const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc,
                        StereoSet st, int32_t* m12, const RecPtrs& out, int32_t* counts) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    const int B = st.nf;
    if (!cam || !mc || !sc || B < 0) return fail(ctx, PLSTVO_E_INVALID, "null camera / config or negative batch size");
    const int rows = mc->grid_rows, cols = mc->grid_cols;
    if (!grid_ok(rows, cols) || cam->width <= 0 || cam->height <= 0)
        return fail(ctx, PLSTVO_E_INVALID, "bad grid or image size");
    if (B == 0) return 0;
    if (const int rc = st.check(ctx)) return rc;
    CK(ctx, cudaSetDevice(ctx->device));
    Arena a;
    st.take(a);
    const GridScratch g(a, rows, cols, B, st.N1, st.N2, st.N2 * grid_cells_per_train(st.lines, rows, cols), !st.lines, st.lines);
    const int first = st.lines ? LS_SPL : PT_PL, last = st.lines ? N_LIFT : LS_SPL;
    size_t o_rec[N_REC];
    take_records(a, st.N1, first, last, o_rec);
    CK(ctx, a.alloc(ctx->arena_stereo));
    std::vector<GridProblem> probs((size_t)B);
    cudaStream_t s = ctx->s_main;
    CK(ctx, st.upload(a, s, &g, probs.data()));
    CK(ctx, st.match(a, g, *cam, *mc, s));
    // lifting, reading the match list where matchGrid left it
    CK(ctx, st.lift(a, *cam, *sc, B, 0, arena_records(a, o_rec, first, last), s));
    ctx->launches += 3;
    CK(ctx, a.down(m12, st.o_m12, st.N1 * 4, s));
    CK(ctx, down_records(a, out, o_rec, st.N1, first, last, s));
    return counts_total(ctx, s, B, a.i32(st.o_cnt), counts, a.i32(st.o_gcnt));
}
}  // namespace

int plstvo_match_stereo_points(PlContext* ctx, const PlCamera* cam, const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                               int B, const int32_t* l_off, const float* kp_l, const int32_t* octave_l, const uint8_t* desc_l,
                               const int32_t* r_off, const float* kp_r, const uint8_t* desc_r, int32_t* m12, double* pt_pl,
                               double* pt_disp, double* pt_P, double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out,
                               int32_t* src_idx, int32_t* counts) {
    const RecPtrs out = RecPtrs::from(PT_PL, {pt_pl, pt_disp, pt_P, pt_sigma2, pt_level, pdesc_out, src_idx});
    const StereoSet st{false, B, l_off, r_off, nullptr, false, kp_l, kp_r, octave_l, desc_l, desc_r};
    return match_stereo_common(ctx, cam, mcfg, scfg, st, m12, out, counts);
}

int plstvo_match_stereo_lines(PlContext* ctx, const PlCamera* cam, const PlStereoMatchConfig* mcfg, const PlStereoConfig* scfg,
                              int B, const int32_t* l_off, const float* seg_l, const float* angle_l, const int32_t* octave_l,
                              const uint8_t* desc_l, const int32_t* r_off, const float* seg_r, const uint8_t* desc_r,
                              int32_t* m12, double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp, double* ls_sP,
                              double* ls_eP, double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level,
                              uint8_t* ldesc_out, int32_t* src_idx, int32_t* counts) {
    const RecPtrs out = RecPtrs::from(LS_SPL, {ls_spl, ls_epl, ls_sdisp, ls_edisp, ls_sP, ls_eP, ls_le, ls_angle, ls_sigma2,
                                               ls_level, ldesc_out, src_idx});
    const StereoSet st{true, B, l_off, r_off, angle_l, false, seg_l, seg_r, octave_l, desc_l, desc_r};
    return match_stereo_common(ctx, cam, mcfg, scfg, st, m12, out, counts);
}

}  // extern "C"

// ---- raw stereo features -> pose, records resident in HBM ---------------------------------------------------------
// sequence == false: B independent (prev, curr) pairs, four feature sets of B frames.
// sequence == true : prev holds NF = B + 1 consecutive frames, pair p = (frame p, frame p + 1); two feature sets of NF frames,
//                    every frame goes through the stereo step once and is lifted twice (as a previous and as a current frame).
// call != null     : prev holds the NF = B new frames of a session call's streams ids[0 .. B) (curr is unused).  Each new frame
//                    goes through the stereo step once and is lifted twice: as the current frame of pair p into the workspace,
//                    and in the previous-frame role into the session's next pool.  The streams' kept frames are gathered into
//                    the workspace's previous-frame arrays (insert; initialize tracks nothing and takes no results).
int plstvo::track_stereo_common(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                                const PlStereoConfig* sc, const StereoSet* prev, const StereoSet* curr, const PlPrior* priors,
                                PlPoseResult* results, int32_t* n_stereo, bool sequence, int slot, const StereoDevInputs* dev,
                                SessionCall* call) {
    // slot < 0: blocking (returns with the results in host memory); slot 0 / 1: enqueue only, results valid after plstvo_wait
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    const bool one_set = sequence || call;          // two feature sets (points, lines of one frame set)
    const bool track = !call || call->track;
    if (!cam || !cfg || !mc || !sc || !prev || (!one_set && !curr) || (track && !results))
        return fail(ctx, PLSTVO_E_INVALID, "null argument");
    const int NF = prev[0].nf;                      // frames per feature set
    const int B = sequence ? NF - 1 : NF;           // pairs
    if (NF < 0 || (!one_set && curr[0].nf != NF)) return fail(ctx, PLSTVO_E_SIZE, "prev and curr hold different numbers of frames");
    if (sequence && NF == 1) return 0;              // one frame: nothing to track
    const int rows = mc->grid_rows, cols = mc->grid_cols;
    if (!grid_ok(rows, cols) || cam->width <= 0 || cam->height <= 0)
        return fail(ctx, PLSTVO_E_INVALID, "bad grid or image size");
    if (NF == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    const int NSETS = one_set ? 2 : 4;
    if (one_set) curr = prev;                       // sets 2, 3 below are unused
    StereoSet sets[4] = {prev[0], prev[1], curr[0], curr[1]};   // {prev, curr} x {points, lines}
    Arena a;
    size_t maxN1 = 0, maxN2 = 0, max_items = 0, o_ooff[4], o_ooff2[4];
    for (int k = 0; k < NSETS; ++k) {
        StereoSet& st = sets[k];
        if (const int rc = st.check(ctx)) return rc;
        st.take(a);
        o_ooff[k] = a.take((size_t)(NF + 1) * 4);
        o_ooff2[k] = a.take((size_t)(NF + 1) * 4);
        maxN1 = std::max(maxN1, st.N1);
        maxN2 = std::max(maxN2, st.N2);
        max_items = std::max(max_items, st.N2 * grid_cells_per_train(st.lines, rows, cols));
    }
    // matchGrid scratch, shared by the four sets (they run one after the other on one stream)
    const GridScratch g(a, rows, cols, NF, maxN1, maxN2, max_items, true, true);
    CK(ctx, a.alloc(ctx->arena_track_stereo[slot + 1]));
    cudaStream_t s = ctx->s_main, sh = ctx->s_h2d;   // uploads of set k + 1 run under the kernels of set k
    // (this slot's arena is free: a blocking call ends synchronised, an async slot is reused only after its event completed)
    // pinned staging: 4 problem tables + 2 x 4 x B counters (pageable copies would block this thread on the stream)
    const size_t prob_bytes = ((size_t)NF * sizeof(GridProblem) + 255) / 256 * 256;
    PinnedBuf& staging = ctx->h_staging[slot + 1];
    CK(ctx, staging.ensure(4 * prob_bytes + (size_t)8 * NF * 4));
    uint8_t* hst = static_cast<uint8_t*>(staging.p);
    int32_t* cnt = reinterpret_cast<int32_t*>(hst + 4 * prob_bytes);
    int32_t* gcnt = cnt + (size_t)4 * NF;
    if (dev && dev->marks) CK(ctx, cudaEventRecord(dev->marks[0], s));
    bool joined = false;
    // ---- pass 1: cells -> matchGrid -> lifting filters (count only) per set ----
    for (int k = 0; k < NSETS; ++k) {
        const StereoSet& st = sets[k];
        CK(ctx, st.upload(a, sh, &g, reinterpret_cast<GridProblem*>(hst + (size_t)k * prob_bytes)));
        cudaEvent_t uploaded = next_event(ctx);
        CK(ctx, cudaEventRecord(uploaded, sh));
        CK(ctx, cudaStreamWaitEvent(s, uploaded, 0));
        if (st.lines && dev && dev->lines_ready && !joined) {   // the line descriptors come from another stream
            CK(ctx, cudaStreamWaitEvent(s, dev->lines_ready, 0));
            joined = true;
        }
        CK(ctx, st.match(a, g, *cam, *mc, s));
        CK(ctx, st.lift(a, *cam, *sc, NF, 0, RecPtrs{}, s));
        ctx->launches += 3;
        CK(ctx, cudaMemcpyAsync(cnt + (size_t)k * NF, a.u8(st.o_cnt), (size_t)NF * 4, cudaMemcpyDeviceToHost, s));
        CK(ctx, cudaMemcpyAsync(gcnt + (size_t)k * NF, a.u8(st.o_gcnt), (size_t)NF * 4, cudaMemcpyDeviceToHost, s));
    }
    CK(ctx, cudaStreamSynchronize(s));     // the one host hop: survivor counts -> compact offsets and the matcher's tile plan
    // compact offsets per set; in sequence mode the current-frame role of a set starts at its second frame
    std::vector<int32_t> ooff[4], ooff2[2];
    for (int k = 0; k < NSETS; ++k) {
        if (const int rc = check_grid_counts(ctx, NF, gcnt + (size_t)k * NF)) return rc;
        ooff[k].assign((size_t)NF + 1, 0);
        for (int p = 0; p < NF; ++p) {
            ooff[k][p + 1] = ooff[k][p] + cnt[(size_t)k * NF + p];
            if (n_stereo) {
                if (sequence || !track) n_stereo[(size_t)p * 2 + k] = cnt[(size_t)k * NF + p];
                else if (!call) n_stereo[(size_t)p * 4 + k] = cnt[(size_t)k * NF + p];
                else {   // an insert: the kept frame's counts, then the new frame's
                    const std::vector<int32_t>& kept = k ? call->kept_off_ls : call->kept_off_pt;
                    n_stereo[(size_t)p * 4 + k] = kept[(size_t)p + 1] - kept[(size_t)p];
                    n_stereo[(size_t)p * 4 + 2 + k] = cnt[(size_t)k * NF + p];
                }
            }
        }
        CK(ctx, a.up(o_ooff[k], ooff[k].data(), (size_t)(NF + 1) * 4, sh));
        if (sequence) {
            ooff2[k].assign((size_t)NF, 0);          // frames 1 .. NF - 1 as current frames: offsets relative to frame 1
            for (int p = 0; p < NF; ++p) ooff2[k][p] = ooff[k][p + 1] - ooff[k][1];
            CK(ctx, a.up(o_ooff2[k], ooff2[k].data(), (size_t)NF * 4, sh));
        }
    }
    // a cams session: the camera of each new frame (its stream's), for pass 2's lifts and for the solver (pair p = frame p)
    PlStereoSession* const ss = call ? call->ss : nullptr;
    const PlCamera* d_cams = nullptr;
    if (ss && !ss->cams.empty()) {
        std::vector<PlCamera> fc((size_t)NF);
        for (int k = 0; k < NF; ++k) fc[(size_t)k] = ss->cams[(size_t)call->ids[k]];
        CK(ctx, ss->d_cams.ensure((size_t)NF * sizeof(PlCamera)));
        CK(ctx, cudaMemcpyAsync(ss->d_cams.p, fc.data(), (size_t)NF * sizeof(PlCamera), cudaMemcpyHostToDevice, s));
        d_cams = ss->d_cams.as<PlCamera>();
    }
    // pass 2: the same lifting kernels, now writing at the compact offsets: the previous-frame role (a pool's or the
    // workspace's PREV_ROLE entries), the current-frame role (curr_rows below) and retention (every array)
    // session: the new frames' previous-frame role goes into the next pool, the untouched streams' kept frames follow it there
    if (call) {
        if (const int rc = session_plan(ctx, *call, cnt, cnt + NF, s)) return rc;
        for (int k = 0; k < 2; ++k)
            CK(ctx, sets[k].lift(a, *cam, *sc, B, 0, ss->pool[ss->cur ^ 1].rows, s, session_out_off(*call, k == 1), d_cams));
        ctx->launches += 2;
        if (const int rc = session_gather_others(ctx, *call, s)) return rc;
        if (call->retain) {   // plstvo_stereo_session_read: every record of the new frames, compact in call order
            SessionRetained& kr = ss->kept;
            CK(ctx, kr.lay_out((size_t)ooff[0][NF], (size_t)ooff[1][NF], track ? (size_t)call->kept_off_pt[NF] : 0,
                               track ? (size_t)call->kept_off_ls[NF] : 0));
            cudaEvent_t offsets_up = next_event(ctx);   // o_ooff, uploaded on sh above
            CK(ctx, cudaEventRecord(offsets_up, sh));
            CK(ctx, cudaStreamWaitEvent(s, offsets_up, 0));
            for (int k = 0; k < 2; ++k) CK(ctx, sets[k].lift(a, *cam, *sc, NF, 0, kr.rec, s, a.i32(o_ooff[k]), d_cams));
            ctx->launches += 2;
            if (call->plot)   // plotStereoFrame: drawn from the rows just retained, before the call's images can be reused
                if (const int rc = session_plot(ctx, *call, cam->width, cam->height, kr.rec, ooff[0], ooff[1], a.i32(o_ooff[0]),
                                                a.i32(o_ooff[1]), s))
                    return rc;
        }
        if (!track) {
            if (dev && dev->marks) {
                CK(ctx, cudaEventRecord(dev->marks[1], s));
                CK(ctx, cudaEventRecord(dev->marks[2], s));
            }
            if (slot < 0) CK(ctx, cudaStreamSynchronize(s));
            return 0;
        }
    }
    // ---- the tracker's plan on the compact lists; the records are written straight into its buffers ----
    PlFrameBatch fp{}, fc{};
    fp.B = fc.B = B;
    fp.pt_off = call ? call->kept_off_pt.data() : ooff[0].data();
    fp.ls_off = call ? call->kept_off_ls.data() : ooff[1].data();
    fc.pt_off = sequence ? ooff2[0].data() : call ? ooff[0].data() : ooff[2].data();
    fc.ls_off = sequence ? ooff2[1].data() : call ? ooff[1].data() : ooff[3].data();
    Workspace& ws = slot < 0 ? ctx->ws : ctx->ws_async[slot];
    const bool resident = dev && dev->priors_resident;   // ws_prepare keeps d_priors: B is the run's n at every step
    int rc = ws_prepare(ctx, ws, cam, cfg, &fp, &fc, true, priors != nullptr || resident, d_cams);
    if (rc) return rc;
    if (priors && !resident)
        CK(ctx, cudaMemcpyAsync(ws.d_priors.p, priors, (size_t)B * sizeof(PlPrior), cudaMemcpyHostToDevice, ctx->s_h2d));
    cudaEvent_t planned = next_event(ctx);
    CK(ctx, cudaEventRecord(planned, ctx->s_h2d));
    CK(ctx, cudaStreamWaitEvent(s, planned, 0));
    if (call) {
        if (const int rc2 = session_gather_named(ctx, *call, ws.prev.rows(PREV_ROLE), s)) return rc2;
    } else {
        for (int k = 0; k < 2; ++k)
            CK(ctx, sets[k].lift(a, *cam, *sc, B, 0, ws.prev.rows(PREV_ROLE), s, a.i32(o_ooff[k]), d_cams));
    }
    // the current-frame role: the set's frames from `first` on (sequence mode: the second frame)
    const int first = sequence ? 1 : 0;
    for (int k = 0; k < 2; ++k) {
        const int j = one_set ? k : 2 + k;
        CK(ctx, sets[j].lift(a, *cam, *sc, B, first, ws.curr.rows(CURR_ROLE), s, a.i32(sequence ? o_ooff2[j] : o_ooff[j]), d_cams));
    }
    ctx->launches += call ? 2 : 4;
    if (dev && dev->marks) CK(ctx, cudaEventRecord(dev->marks[1], s));
    rc = ws_launch_match(ctx, ws, 0, B, s);
    if (rc) return rc;
    rc = ws_launch_solve(ctx, ws, 0, B, true, s);
    if (rc) return rc;
    if (dev && dev->marks) CK(ctx, cudaEventRecord(dev->marks[2], s));
    if (call && call->retain) {   // the tracker's rows, indexed by the kept frames' features (fp's offsets)
        const SessionRetained& kr = ss->kept;
        for (int r = M12_PT; r < N_REC; ++r) {
            const size_t bytes = kr.rows[r] * (size_t)REC_BYTES[r];
            if (bytes) CK(ctx, cudaMemcpyAsync(kr.rec.p[r], ws.prev.rec[r].p, bytes, cudaMemcpyDeviceToDevice, s));
        }
    }
    if (dev && dev->tracked) return dev->tracked(ws);
    CK(ctx, cudaMemcpyAsync(results, ws.d_results.p, (size_t)B * sizeof(PlPoseResult), cudaMemcpyDeviceToHost, s));
    if (slot < 0) CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

namespace {
// the point set and the line set of f's frames into fs[0], fs[1] (null for a null f)
const StereoSet* feature_sets(const PlStereoFeatures* f, StereoSet* fs) {
    if (!f) return nullptr;
    fs[0] = StereoSet{false, f->B, f->pl_off, f->pr_off, nullptr, false, f->kp_l, f->kp_r, f->poct_l, f->pdesc_l, f->pdesc_r};
    fs[1] = StereoSet{true, f->B, f->ll_off, f->lr_off, f->angle_l, false, f->seg_l, f->seg_r, f->loct_l, f->ldesc_l, f->ldesc_r};
    return fs;
}
}  // namespace

extern "C" {

// ticket bookkeeping shared with plstvo_track_batch_async: two slots, plstvo_wait(ticket) blocks until the slot's results are home
static int stereo_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                        const PlStereoConfig* sc, const PlStereoFeatures* a, const PlStereoFeatures* b, const PlPrior* priors,
                        PlPoseResult* results, int32_t* n_stereo, bool sequence) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    const int slot = acquire_slot(ctx);
    if (slot < 0) return slot;
    StereoSet sa[2], sb[2];
    const int rc = track_stereo_common(ctx, cam, cfg, mc, sc, feature_sets(a, sa), feature_sets(b, sb), priors, results, n_stereo,
                                       sequence, slot);
    if (rc) return rc;
    CK(ctx, cudaEventRecord(ctx->slot_done[slot], ctx->s_main));
    ctx->slot_busy[slot] = true;
    return slot;
}

int plstvo_track_stereo_batch_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                                    const PlStereoConfig* sc, const PlStereoFeatures* prev, const PlStereoFeatures* curr,
                                    const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    return stereo_async(ctx, cam, cfg, mc, sc, prev, curr, priors, results, n_stereo, false);
}

int plstvo_track_stereo_sequence_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                                       const PlStereoConfig* sc, const PlStereoFeatures* frames, const PlPrior* priors,
                                       PlPoseResult* results, int32_t* n_stereo) {
    return stereo_async(ctx, cam, cfg, mc, sc, frames, nullptr, priors, results, n_stereo, true);
}

int plstvo_track_stereo_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                              const PlStereoConfig* sc, const PlStereoFeatures* prev, const PlStereoFeatures* curr,
                              const PlPrior* priors, PlPoseResult* results, int32_t* n_stereo) {
    StereoSet p[2], c[2];
    return track_stereo_common(ctx, cam, cfg, mc, sc, feature_sets(prev, p), feature_sets(curr, c), priors, results, n_stereo,
                               false, -1);
}

int plstvo_track_stereo_sequence(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                                 const PlStereoConfig* sc, const PlStereoFeatures* frames, const PlPrior* priors,
                                 PlPoseResult* results, int32_t* n_stereo) {
    StereoSet f[2];
    return track_stereo_common(ctx, cam, cfg, mc, sc, feature_sets(frames, f), nullptr, priors, results, n_stereo, true, -1);
}

}  // extern "C"
