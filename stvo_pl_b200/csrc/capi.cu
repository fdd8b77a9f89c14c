// capi.cu — host side of the C-ABI (include/plstvo.h): context, work planning, chunked H2D / compute / D2H pipelining of
// matching and tracking, throughput mode, instrumentation.  The stereo step is in capi_stereo.cu, feature extraction in
// capi_features.cu, what they share in host.cuh.  No CPU compute path exists in this library: without a CUDA
// device plstvo_create() fails with PLSTVO_E_NO_DEVICE and every other entry point needs a context.
#include <array>
#include <cstdlib>
#include <cstring>

#include "host.cuh"

using namespace plstvo;

struct PlDeviceBatch {
    Workspace ws;
};

namespace {

int pow2_ceil_host(int n) {
    int m = 1;
    while (m < n) m <<= 1;
    return m;
}


// Which solver a batch takes.  K2 (one fp64 CTA per pair, lists in shared memory) has the lower latency and follows the
// reference to rounding; the streamed solver (fp32 per-feature arithmetic, fp64 sums / algebra / outlier statistics, close stop
// tests re-decided in fp64) has the higher throughput once a batch is more than one wave of K2 CTAs, and is the only form for
// lists that do not fit K2's shared memory.  Default: streamed when the lists do not fit, or when the batch has more pairs than
// the device has SMs.  PLSTVO_STREAM_SOLVE=1: always streamed (tests on small frames); =0: never (K2, lists in global scratch
// if need be).
int stream_mode() {
    static const int m = [] {
        const char* v = getenv("PLSTVO_STREAM_SOLVE");
        return v ? atoi(v) : -1;
    }();
    return m;
}

// The solver plan of B pairs with at most cap_pt / cap_ls matched features and max_n2 current-frame rows per pair
SolvePlan plan_solve(const PlContext* ctx, int cap_pt, int cap_ls, int max_n2, int B, int solver_mode) {
    SolvePlan pl;
    pl.cap_pt = cap_pt;
    pl.cap_ls = cap_ls;
    // at least 32: the outlier statistics sort max(n, 32) padded entries (solve.cu: remove_outliers)
    pl.sort_cap = pow2_ceil_host(std::max(32, std::max(std::max(cap_pt, cap_ls), (max_n2 + 1) / 2)));
    // matched lists live in shared memory when they fit (C2: 152 KB), else in a global scratch slice (C5)
    static const bool no_smem = getenv("PLSTVO_K2_FEAT_GLOBAL") != nullptr;
    pl.feat_in_smem = !no_smem && k2_smem_bytes(cap_pt, cap_ls, pl.sort_cap, true) <= ctx->smem_optin;
    pl.fits = pl.feat_in_smem || k2_smem_bytes(cap_pt, cap_ls, pl.sort_cap, false) <= ctx->smem_optin;
    // (the robust main solver, solver_mode != 0, is K2-only: the streamed form would hand every problem back)
    pl.use_stream = stream_mode() == 1 ||
                    (stream_mode() != 0 && (!pl.feat_in_smem || (B > ctx->sm_count && solver_mode == 0)));
    if (!pl.feat_in_smem || pl.use_stream) pl.feat_stride = k2_feat_stride(cap_pt, cap_ls);
    return pl;
}

// carves the streamed solver's buffers for B problems out of one arena; slots = record slots (prev-frame features in track
// mode, list entries in explicit mode)
int stream_bufs_prepare(PlContext* ctx, DevBuf& arena, int B, size_t slots_pt, size_t slots_ls, StreamBufs* sb) {
    Arena a;
    const size_t o_rp = a.take((slots_pt + 512) * 2 * sizeof(float4)), o_rl = a.take((slots_ls + 256) * 4 * sizeof(float4));
    const size_t o_cp = a.take((size_t)B * 4), o_cl = a.take((size_t)B * 4), o_dt = a.take((size_t)B * 16 * 8);
    const size_t o_ac = a.take((size_t)B * 4), o_ctl = a.take((size_t)B * sizeof(StreamCtl));
    const size_t o_fp = a.take(slots_pt + 16), o_fl = a.take(slots_ls + 16), o_mp = a.take((slots_pt + 16) * 2);
    const size_t o_ml = a.take((slots_ls + 16) * 2), o_q = a.take((size_t)B * 2 * 4 + 16);
    CK(ctx, a.alloc(arena));
    sb->rec_pt = a.at<float4>(o_rp);
    sb->rec_ls = a.at<float4>(o_rl);
    sb->cnt_pt = a.i32(o_cp);
    sb->cnt_ls = a.i32(o_cl);
    sb->DT = a.f64(o_dt);
    sb->active = a.i32(o_ac);
    sb->ctl = a.at<StreamCtl>(o_ctl);
    sb->queue = a.i32(o_q);
    sb->flag_pt = a.u8(o_fp);
    sb->flag_ls = a.u8(o_fl);
    sb->midx_pt = a.at<uint16_t>(o_mp);
    sb->midx_ls = a.at<uint16_t>(o_ml);
    sb->sm_count = ctx->sm_count;
    return 0;
}

// the per-problem arrays of a chunk of pairs starting at p0 (record / flag arrays are indexed by absolute slots)
StreamBufs stream_bufs_at(const StreamBufs& sb, int p0) {
    StreamBufs r = sb;
    r.cnt_pt += p0; r.cnt_ls += p0; r.DT += (size_t)p0 * 16; r.active += p0; r.ctl += p0;
    r.queue += 2 * (size_t)p0;   // a chunk starts at a distinct pair: its two queue words are its own
    return r;
}

// Launches the planned solver on pairs [p0, p1) of a batch of B: prm filled but for the solver's fields, feat the batch's
// global list scratch (pl.feat_stride doubles per pair), slots_pt / slots_ls the record slots of the streamed solver's arena.
// marks: 4 events recorded between the solver's stages (instrumentation only).
// cams (optional, device, [B]): the camera of each pair instead of prm.cam.
int launch_solver(PlContext* ctx, SolveParams prm, const SolvePlan& pl, double* feat, DevBuf& stream_arena, int B,
                  size_t slots_pt, size_t slots_ls, int p0, int p1, cudaStream_t s, cudaEvent_t* marks = nullptr,
                  const PlCamera* cams = nullptr) {
    prm.first_pair = p0;
    prm.feat_scratch = pl.feat_in_smem ? nullptr : feat + (size_t)p0 * pl.feat_stride;
    prm.feat_scratch_stride = pl.feat_stride;
    prm.cap_pt = pl.cap_pt;
    prm.cap_ls = pl.cap_ls;
    prm.sort_cap = pl.sort_cap;
    prm.feat_in_smem = pl.feat_in_smem ? 1 : 0;
    if (pl.use_stream) {
        StreamBufs sb;
        int rc = stream_bufs_prepare(ctx, stream_arena, B, slots_pt, slots_ls, &sb);
        if (rc) return rc;
        prm.feat_scratch = feat + (size_t)p0 * pl.feat_stride;
        prm.feat_in_smem = 0;
        int nl = 0;
        CK(ctx, launch_stream_solve(prm, p1 - p0, stream_bufs_at(sb, p0), s, &nl, marks, cams));
        ctx->launches += nl;
        return 0;
    }
    if (marks)   // fused kernel: list building, both GN stages and the outlier pass are inside K2
        for (int k = 0; k < 4; ++k) CK(ctx, cudaEventRecord(marks[k], s));
    CK(ctx, launch_track_solve(prm, p1 - p0, s, cams));
    ctx->launches++;
    return 0;
}

// ---- planning -------------------------------------------------------------------------------------
int validate_frames(PlContext* ctx, const PlFrameBatch* prev, const PlFrameBatch* curr, bool need_features) {
    if (!prev || !curr) return fail(ctx, PLSTVO_E_INVALID, "null frame batch");
    if (prev->B != curr->B) return fail(ctx, PLSTVO_E_SIZE, "prev and curr hold a different number of frames");
    if (prev->B < 0) return fail(ctx, PLSTVO_E_INVALID, "negative batch size");
    if (prev->B == 0) return 0;
    if (!prev->pt_off || !prev->ls_off || !curr->pt_off || !curr->ls_off)
        return fail(ctx, PLSTVO_E_INVALID, "null offsets");
    if (const int rc = check_offsets(ctx, prev->B, {prev->pt_off, curr->pt_off, prev->ls_off, curr->ls_off},
                                     "offsets must start at 0", "offsets are not non-decreasing",
                                     "more than 65535 features in a frame"))
        return rc;
    const int np1 = prev->pt_off[prev->B], np2 = curr->pt_off[curr->B];
    const int nl1 = prev->ls_off[prev->B], nl2 = curr->ls_off[curr->B];
    if ((np1 && !prev->pdesc) || (np2 && !curr->pdesc) || (nl1 && !prev->ldesc) || (nl2 && !curr->ldesc))
        return fail(ctx, PLSTVO_E_INVALID, "null descriptor matrix");
    if (need_features) {
        if (np1 && (!prev->pt_P || !prev->pt_sigma2)) return fail(ctx, PLSTVO_E_INVALID, "prev point arrays missing");
        if (np2 && !curr->pt_pl) return fail(ctx, PLSTVO_E_INVALID, "curr pt_pl missing");
        if (nl1 && (!prev->ls_sP || !prev->ls_eP || !prev->ls_spl || !prev->ls_epl || !prev->ls_sigma2))
            return fail(ctx, PLSTVO_E_INVALID, "prev line arrays missing");
        if (nl2 && !curr->ls_le) return fail(ctx, PLSTVO_E_INVALID, "curr ls_le missing");
    }
    return 0;
}

// ---- the callers' arrays by records.h array ----
struct HostRec {
    int k;
    const void* src;
};
// a PlFrameBatch in the previous-frame role (PREV_ROLE) and in the current-frame role (CURR_ROLE)
std::array<HostRec, N_PREV> prev_fields(const PlFrameBatch* f) {
    return {{{PT_P, f->pt_P}, {PT_S2, f->pt_sigma2}, {PT_DESC, f->pdesc}, {LS_SPL, f->ls_spl}, {LS_EPL, f->ls_epl},
             {LS_SP, f->ls_sP}, {LS_EP, f->ls_eP}, {LS_S2, f->ls_sigma2}, {LS_LEVEL, f->ls_level}, {LS_DESC, f->ldesc}}};
}
std::array<HostRec, 4> curr_fields(const PlFrameBatch* f) {
    return {{{PT_PL, f->pt_pl}, {PT_DESC, f->pdesc}, {LS_LE, f->ls_le}, {LS_DESC, f->ldesc}}};
}
// explicit matched lists: the observations pl_obs and le_obs are current-frame rows, PT_PL and LS_LE
std::array<HostRec, 11> matched_fields(const PlMatchedBatch* m) {
    return {{{PT_P, m->pt_P}, {PT_PL, m->pt_pl_obs}, {PT_S2, m->pt_sigma2}, {INL_PT, m->pt_inlier}, {LS_SP, m->ls_sP},
             {LS_EP, m->ls_eP}, {LS_LE, m->ls_le_obs}, {LS_SPL, m->ls_spl}, {LS_EPL, m->ls_epl}, {LS_S2, m->ls_sigma2},
             {INL_LS, m->ls_inlier}}};
}

// the arrays matching-only calls (plstvo_match_batch, plstvo_f2f_tracking) size and move: the descriptors and m12
constexpr bool matching_rec(int k) { return k == PT_DESC || k == LS_DESC || k == M12_PT || k == M12_LS; }

// rows [first, first + count) of w bytes each, from an array of such rows to another; nothing for a null end or no rows
cudaError_t copy_rows(void* dst, const void* src, size_t w, size_t first, size_t count, cudaMemcpyKind kind, cudaStream_t s) {
    if (!dst || !src || !count) return cudaSuccess;
    return cudaMemcpyAsync(static_cast<uint8_t*>(dst) + first * w, static_cast<const uint8_t*>(src) + first * w, count * w,
                           kind, s);
}

// Uploads explicit lists m on s into dst: the offsets and every array of the PlMatchedBatch table, each buffer at least 16
// bytes (an empty list's too).  *rows: those arrays, a null entry for inlier flags the caller did not give (all true).
int upload_matched(PlContext* ctx, const PlMatchedBatch* m, FrameBufs& dst, cudaStream_t s, RecPtrs* rows) {
    const int B = m->B;
    const size_t n_pt = m->pt_off[B], n_ls = m->ls_off[B], off_bytes = (size_t)(B + 1) * 4;
    CK(ctx, dst.pt_off.ensure(std::max<size_t>(off_bytes, 16)));
    CK(ctx, cudaMemcpyAsync(dst.pt_off.p, m->pt_off, off_bytes, cudaMemcpyHostToDevice, s));
    CK(ctx, dst.ls_off.ensure(std::max<size_t>(off_bytes, 16)));
    CK(ctx, cudaMemcpyAsync(dst.ls_off.p, m->ls_off, off_bytes, cudaMemcpyHostToDevice, s));
    *rows = RecPtrs{};
    for (const HostRec& e : matched_fields(m)) {
        DevBuf& buf = dst.rec[e.k];
        const size_t bytes = (rec_is_point(e.k) ? n_pt : n_ls) * REC_BYTES[e.k];
        CK(ctx, buf.ensure(std::max<size_t>(bytes, 16)));
        if (e.src && bytes) CK(ctx, cudaMemcpyAsync(buf.p, e.src, bytes, cudaMemcpyHostToDevice, s));
        if (e.src || (e.k != INL_PT && e.k != INL_LS)) rows->p[e.k] = buf.p;
    }
    return 0;
}

}  // namespace

namespace plstvo {

// Builds the plan of a batch of pairs and sizes every device buffer.  `with_features` = track mode.
// d_cams (optional): the device camera of each pair, which the solver then reads instead of cam.
int ws_prepare(PlContext* ctx, Workspace& ws, const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
               const PlFrameBatch* curr, bool with_features, bool has_priors, const PlCamera* d_cams) {
    const int B = prev->B;
    ws.d_cams = d_cams;
    // Same shapes and matching parameters as the previous call on this workspace (a video stream, a benchmark loop):
    // the plan, the partial buffers and their device copies are still valid — skip the rebuild and its uploads.
    if (ws.planned && ws.B == B && ws.planned_features == with_features && ws.sm_planned == ctx->sm_count &&
        ws.cfg.has_points == cfg->has_points && ws.cfg.has_lines == cfg->has_lines &&
        ws.cfg.best_lr_matches == cfg->best_lr_matches && ws.cfg.min_ratio_12_p == cfg->min_ratio_12_p &&
        (ws.cfg.solver_mode != 0) == (cfg->solver_mode != 0) &&
        ws.cfg.min_ratio_12_l == cfg->min_ratio_12_l && (int)ws.p_off1.size() == B + 1 &&
        !memcmp(ws.p_off1.data(), prev->pt_off, (size_t)(B + 1) * 4) &&
        !memcmp(ws.p_off2.data(), curr->pt_off, (size_t)(B + 1) * 4) &&
        !memcmp(ws.l_off1.data(), prev->ls_off, (size_t)(B + 1) * 4) &&
        !memcmp(ws.l_off2.data(), curr->ls_off, (size_t)(B + 1) * 4)) {
        if (cam) ws.cam = *cam;
        ws.cfg = *cfg;
        ws.has_priors = has_priors;
        return 0;
    }
    ws.planned = false;
    ws.B = B;
    if (cam) ws.cam = *cam;
    ws.cfg = *cfg;
    ws.has_priors = has_priors;
    ws.p_off1.assign(prev->pt_off, prev->pt_off + B + 1);
    ws.p_off2.assign(curr->pt_off, curr->pt_off + B + 1);
    ws.l_off1.assign(prev->ls_off, prev->ls_off + B + 1);
    ws.l_off2.assign(curr->ls_off, curr->ls_off + B + 1);
    const size_t np1 = ws.p_off1[B], np2 = ws.p_off2[B], nl1 = ws.l_off1[B], nl2 = ws.l_off2[B];

    ws.problems.assign((size_t)2 * B, MatchProblem{});
    ws.tc_problems.assign((size_t)2 * B, TcProblem{});
    int cap_pt = 0, cap_ls = 0;
    ws.max_n2 = 0;
    size_t row_elems = 0, col_elems = 0, rowp_elems = 0, colp_elems = 0;
    for (int k = 0; k < 2; ++k) {
        ws.tc_items[k].clear();
        ws.item_start[k].assign((size_t)B + 1, 0);
    }
    const float nnr_p = (float)cfg->min_ratio_12_p, nnr_l = (float)cfg->min_ratio_12_l;   // double -> float at the call
    for (int p = 0; p < B; ++p) {
        ws.item_start[0][p] = (int32_t)ws.tc_items[0].size();
        ws.item_start[1][p] = (int32_t)ws.tc_items[1].size();
        for (int type = 0; type < 2; ++type) {
            MatchProblem& pr = ws.problems[(size_t)2 * p + type];
            TcProblem& tp = ws.tc_problems[(size_t)2 * p + type];
            const int n1 = type ? ws.l_off1[p + 1] - ws.l_off1[p] : ws.p_off1[p + 1] - ws.p_off1[p];
            const int n2 = type ? ws.l_off2[p + 1] - ws.l_off2[p] : ws.p_off2[p + 1] - ws.p_off2[p];
            const bool wanted = type ? cfg->has_lines != 0 : cfg->has_points != 0;
            pr.n1 = tp.n1 = n1;
            pr.n2 = tp.n2 = n2;
            pr.nnr = type ? nnr_l : nnr_p;
            pr.best_lr = cfg->best_lr_matches != 0;
            pr.enabled = (wanted && n1 > 0 && n2 > 0) ? 1 : 0;   // src/stereoFrameHandler.cpp:137-138, :160-161
            // offsets into the partial buffers are stored as element indices first, fixed up after allocation
            pr.rowpart = reinterpret_cast<uint2*>(row_elems);
            pr.colpart = reinterpret_cast<uint2*>(col_elems);
            tp.rowp = reinterpret_cast<uint32_t*>(rowp_elems);
            tp.colp = reinterpret_cast<uint32_t*>(colp_elems);
            if (pr.enabled) {
                row_elems += (size_t)n1;
                col_elems += (size_t)n2;
                rowp_elems += (size_t)((n2 + TC_CW - 1) / TC_CW) * n1;
                colp_elems += (size_t)n2;
                const int t2 = (n2 + TC_ROWS - 1) / TC_ROWS;
                for (int yb = 0; yb < (t2 + 1) / 2; ++yb) ws.tc_items[type].push_back(TcItem{2 * p + type, yb});
            }
            ws.max_n2 = std::max(ws.max_n2, n2);
            if (type == 0) cap_pt = std::max(cap_pt, n1);
            else cap_ls = std::max(cap_ls, n1);
        }
    }
    ws.item_start[0][B] = (int32_t)ws.tc_items[0].size();
    ws.item_start[1][B] = (int32_t)ws.tc_items[1].size();
    ws.solver = plan_solve(ctx, std::max(cap_pt, 1), std::max(cap_ls, 1), ws.max_n2, B, cfg->solver_mode);
    // the per-pair solver's limits only apply when it runs (track mode): matching-only calls take any frame up to
    // PLSTVO_MAX_FEATURES rows
    if (with_features && !ws.solver.fits)
        return fail(ctx, PLSTVO_E_TOO_LARGE, "frame too large for the per-pair solver's shared memory");

    // --- device storage: matching-only calls size the descriptors and m12, tracking every array of both roles ---
    auto grow = [&](FrameBufs& side, int k, size_t n_pt, size_t n_ls) {
        return with_features || matching_rec(k) ? side.rec[k].ensure((rec_is_point(k) ? n_pt : n_ls) * REC_BYTES[k])
                                                : cudaSuccess;
    };
    for (int k : PREV_ROLE) CK(ctx, grow(ws.prev, k, np1, nl1));
    for (int k = M12_PT; k < N_REC; ++k) CK(ctx, grow(ws.prev, k, np1, nl1));   // the tracker's rows
    for (int k : CURR_ROLE) CK(ctx, grow(ws.curr, k, np2, nl2));
    CK(ctx, ws.d_rowpart.ensure(row_elems * sizeof(uint2)));
    CK(ctx, ws.d_colpart.ensure(col_elems * sizeof(uint2)));
    CK(ctx, ws.d_problems.ensure(ws.problems.size() * sizeof(MatchProblem)));
    CK(ctx, ws.d_rowp.ensure(rowp_elems * sizeof(uint32_t)));
    CK(ctx, ws.d_colp.ensure(colp_elems * sizeof(uint32_t)));
    CK(ctx, ws.d_tcprob.ensure(ws.tc_problems.size() * sizeof(TcProblem)));
    for (int k = 0; k < 2; ++k) CK(ctx, ws.d_tcitems[k].ensure(ws.tc_items[k].size() * sizeof(TcItem)));
    if (!ws.d_sched.p) {   // scheduler words of the persistent matcher: one pair per compute stream, self re-arming
        CK(ctx, ws.d_sched.ensure(64));
        CK(ctx, cudaMemsetAsync(ws.d_sched.p, 0, 64, ctx->s_h2d));
    }
    if (with_features) {
        for (DevBuf* off : {&ws.prev.pt_off, &ws.curr.pt_off, &ws.prev.ls_off, &ws.curr.ls_off})
            CK(ctx, off->ensure((B + 1) * 4));
        CK(ctx, ws.d_priors.ensure((size_t)B * sizeof(PlPrior)));
        CK(ctx, ws.d_results.ensure((size_t)B * sizeof(PlPoseResult)));
        if (ws.solver.feat_stride) CK(ctx, ws.d_feat.ensure((size_t)B * ws.solver.feat_stride * sizeof(double)));
    }
    // --- fix up pointers, upload the plan ---
    for (int p = 0; p < B; ++p)
        for (int type = 0; type < 2; ++type) {
            MatchProblem& pr = ws.problems[(size_t)2 * p + type];
            pr.rowpart = ws.d_rowpart.as<uint2>() + reinterpret_cast<size_t>(pr.rowpart);
            pr.colpart = ws.d_colpart.as<uint2>() + reinterpret_cast<size_t>(pr.colpart);
            const int kd = type ? LS_DESC : PT_DESC, km = type ? M12_LS : M12_PT;
            const size_t r1 = type ? ws.l_off1[p] : ws.p_off1[p], r2 = type ? ws.l_off2[p] : ws.p_off2[p];
            pr.d1 = ws.prev.rec[kd].as<uint8_t>() + r1 * REC_BYTES[kd];
            pr.d2 = ws.curr.rec[kd].as<uint8_t>() + r2 * REC_BYTES[kd];
            pr.m12 = ws.prev.rec[km].as<int32_t>() + r1;
            // the matcher expands the rows of the workspace's own 32-byte-row arenas (16-byte aligned loads)
            TcProblem& tp = ws.tc_problems[(size_t)2 * p + type];
            tp.d1 = pr.d1;
            tp.d2 = pr.d2;
            tp.rowp = ws.d_rowp.as<uint32_t>() + reinterpret_cast<size_t>(tp.rowp);
            tp.colp = ws.d_colp.as<uint32_t>() + reinterpret_cast<size_t>(tp.colp);
        }
    cudaStream_t s = ctx->s_h2d;
    if (!ws.tc_problems.empty()) {
        CK(ctx, cudaMemcpyAsync(ws.d_tcprob.p, ws.tc_problems.data(), ws.tc_problems.size() * sizeof(TcProblem),
                                cudaMemcpyHostToDevice, s));
        for (int k = 0; k < 2; ++k)
            if (!ws.tc_items[k].empty())
                CK(ctx, cudaMemcpyAsync(ws.d_tcitems[k].p, ws.tc_items[k].data(), ws.tc_items[k].size() * sizeof(TcItem),
                                        cudaMemcpyHostToDevice, s));
    }
    if (!ws.problems.empty())
        CK(ctx, cudaMemcpyAsync(ws.d_problems.p, ws.problems.data(), ws.problems.size() * sizeof(MatchProblem),
                                cudaMemcpyHostToDevice, s));
    if (with_features) {
        CK(ctx, cudaMemcpyAsync(ws.prev.pt_off.p, ws.p_off1.data(), (B + 1) * 4, cudaMemcpyHostToDevice, s));
        CK(ctx, cudaMemcpyAsync(ws.curr.pt_off.p, ws.p_off2.data(), (B + 1) * 4, cudaMemcpyHostToDevice, s));
        CK(ctx, cudaMemcpyAsync(ws.prev.ls_off.p, ws.l_off1.data(), (B + 1) * 4, cudaMemcpyHostToDevice, s));
        CK(ctx, cudaMemcpyAsync(ws.curr.ls_off.p, ws.l_off2.data(), (B + 1) * 4, cudaMemcpyHostToDevice, s));
    }
    ws.planned = true;
    ws.planned_features = with_features;
    ws.sm_planned = ctx->sm_count;
    return 0;
}

// descriptors (+ features when with_features) of pairs [p0, p1) host -> device
int ws_upload_range(PlContext* ctx, Workspace& ws, const PlFrameBatch* prev, const PlFrameBatch* curr,
                    const PlPrior* priors, int p0, int p1, bool with_features, cudaStream_t s) {
    auto up = [&](FrameBufs& side, const auto& fields, const std::vector<int32_t>& pt_off, const std::vector<int32_t>& ls_off) {
        for (const HostRec& e : fields) {
            const std::vector<int32_t>& off = rec_is_point(e.k) ? pt_off : ls_off;
            if (with_features || matching_rec(e.k))
                if (const cudaError_t err = copy_rows(side.rec[e.k].p, e.src, REC_BYTES[e.k], off[p0], off[p1] - off[p0],
                                                      cudaMemcpyHostToDevice, s))
                    return err;
        }
        return cudaSuccess;
    };
    CK(ctx, up(ws.prev, prev_fields(prev), ws.p_off1, ws.l_off1));
    CK(ctx, up(ws.curr, curr_fields(curr), ws.p_off2, ws.l_off2));
    if (with_features)
        CK(ctx, copy_rows(ws.d_priors.p, priors, sizeof(PlPrior), p0, p1 - p0, cudaMemcpyHostToDevice, s));
    return 0;
}

int ws_launch_match(PlContext* ctx, Workspace& ws, int p0, int p1, cudaStream_t s, cudaEvent_t* marks) {
    const int a0 = ws.item_start[0][p0], a1 = ws.item_start[0][p1], b0 = ws.item_start[1][p0], b1 = ws.item_start[1][p1];
    if (a1 > a0 || b1 > b0) {
        if (marks) CK(ctx, cudaEventRecord(marks[0], s));   // operands are expanded inside the matcher: empty stage
        // launches on the two compute streams may overlap: each has its own pair of scheduler words
        int* sched = ws.d_sched.as<int>() + (s == ctx->s_alt ? 8 : 0);
        CK(ctx, launch_tc_hamming(ws.d_tcprob.as<TcProblem>(), ws.d_tcitems[0].as<TcItem>() + a0, a1 - a0,
                                  ws.d_tcitems[1].as<TcItem>() + b0, b1 - b0, sched, ctx->sm_count, s));
        if (marks) CK(ctx, cudaEventRecord(marks[1], s));
        CK(ctx, launch_tc_resolve(ws.d_problems.as<MatchProblem>() + (size_t)2 * p0, ws.d_tcprob.as<TcProblem>() + (size_t)2 * p0,
                                  2 * (p1 - p0), 4, s));
        ctx->launches += 2;
    }
    return 0;
}

int ws_launch_solve(PlContext* ctx, Workspace& ws, int p0, int p1, bool have_level, cudaStream_t s, cudaEvent_t* marks) {
    if (p1 <= p0) return 0;
    SolveParams prm{};
    prm.cam = ws.cam;
    prm.cfg = ws.cfg;
    prm.mode = 0;
    RecPtrs prev = ws.prev.rows(PREV_ROLE);
    if (!have_level) prev.p[LS_LEVEL] = nullptr;
    prm.prev = rows_dev(ws.prev.pt_off, ws.prev.ls_off, prev);
    prm.curr = rows_dev(ws.curr.pt_off, ws.curr.ls_off, ws.curr.rows(CURR_ROLE));
    prm.problems = ws.d_problems.as<MatchProblem>();
    prm.priors = ws.has_priors ? ws.d_priors.as<PlPrior>() : nullptr;
    prm.results = ws.d_results.as<PlPoseResult>();
    prm.inlier_pt = ws.prev.rec[INL_PT].as<uint8_t>();
    prm.inlier_ls = ws.prev.rec[INL_LS].as<uint8_t>();
    prm.phase_cycles = ws.d_phase.as<long long>();
    return launch_solver(ctx, prm, ws.solver, ws.d_feat.as<double>(), ws.d_stream, ws.B, (size_t)ws.p_off1[ws.B],
                         (size_t)ws.l_off1[ws.B], p0, p1, s, marks, ws.d_cams);
}

int ws_download_range(PlContext* ctx, Workspace& ws, int p0, int p1, PlPoseResult* results, int32_t* m12_pt,
                      int32_t* m12_ls, uint8_t* inl_pt, uint8_t* inl_ls, cudaStream_t s) {
    CK(ctx, copy_rows(results, ws.d_results.p, sizeof(PlPoseResult), p0, p1 - p0, cudaMemcpyDeviceToHost, s));
    const RecPtrs dst = RecPtrs::from(M12_PT, {m12_pt, inl_pt, m12_ls, inl_ls});
    for (int k = M12_PT; k < N_REC; ++k) {   // the tracker's rows, per previous-frame feature
        const std::vector<int32_t>& off = rec_is_point(k) ? ws.p_off1 : ws.l_off1;
        CK(ctx, copy_rows(dst.p[k], ws.prev.rec[k].p, REC_BYTES[k], off[p0], off[p1] - off[p0], cudaMemcpyDeviceToHost, s));
    }
    return 0;
}

// Pairs per chunk of the resident pass and of a pipelined end-to-end step: the whole batch up to one pair per SM, beyond that
// two halves (two launches per pass: measured best).
int pass_chunk(int B, int sm_count) { return std::max(1, std::max(std::min(B, sm_count), (B + 1) / 2)); }

// Pipeline chunking of the host-buffer entry point: small first chunks (the GPU starts working after a few MB have
// crossed PCIe), then chunks of about two thirds of the SM count in pairs (K2 runs one pair per SM; the rest of the
// chip keeps running the next chunk's distance tiles on the other compute stream).
// With batches in flight behind one another (plstvo_track_batch_async) the previous batch's kernels already hide the copy:
// no ramp, the resident pass's chunking (two launches per pass) is used instead.
std::vector<int> chunk_schedule(int B, int sm_count, bool pipelined) {
    std::vector<int> bounds{0};
    if (pipelined) {
        const int step = pass_chunk(B, sm_count);
        for (int p = step; p < B; p += step) bounds.push_back(p);
        bounds.push_back(B);
        return bounds;
    }
    // ramp 1/6, 1/3, 2/3 of the SM count, then equal chunks of at most one pair per SM
    int p = 0;
    for (int c = std::max(8, sm_count / 6); c < sm_count && p + c < B; c *= 2) {
        p += c;
        bounds.push_back(p);
    }
    const int rest = B - p;
    if (rest > 0) {
        const int n = (rest + sm_count - 1) / sm_count;
        for (int k = 1; k <= n; ++k) bounds.push_back(p + (int)((long)rest * k / n));
    }
    return bounds;
}

// resident pass: K1 / K2 over the whole batch, chunked over two streams so that the (latency-bound) per-pair
// solver of chunk i overlaps the (throughput-bound) distance tiles of chunk i+1
int ws_run(PlContext* ctx, Workspace& ws, bool have_level) {
    if (ws.B == 0) return 0;
    const int chunk = pass_chunk(ws.B, ctx->sm_count);
    cudaEvent_t start = next_event(ctx);
    CK(ctx, cudaEventRecord(start, ctx->s_main));
    CK(ctx, cudaStreamWaitEvent(ctx->s_alt, start, 0));
    int k = 0;
    for (int p0 = 0; p0 < ws.B; p0 += chunk, ++k) {
        const int p1 = std::min(ws.B, p0 + chunk);
        cudaStream_t s = (k & 1) ? ctx->s_alt : ctx->s_main;
        int rc = ws_launch_match(ctx, ws, p0, p1, s);
        if (rc) return rc;
        rc = ws_launch_solve(ctx, ws, p0, p1, have_level, s);
        if (rc) return rc;
    }
    cudaEvent_t done = next_event(ctx);
    CK(ctx, cudaEventRecord(done, ctx->s_alt));
    CK(ctx, cudaStreamWaitEvent(ctx->s_main, done, 0));
    return 0;
}

}  // namespace plstvo

// =====================================================================================================
extern "C" {

int plstvo_version(void) { return PLSTVO_VERSION; }

int plstvo_create(int device, PlContext** out) {
    if (!out) return PLSTVO_E_INVALID;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return PLSTVO_E_NO_DEVICE;
    if (device < 0) {
        if (cudaGetDevice(&device) != cudaSuccess) return PLSTVO_E_NO_DEVICE;
    }
    if (device >= n) return PLSTVO_E_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return PLSTVO_E_NO_DEVICE;
    if (prop.major != 9) return PLSTVO_E_NO_DEVICE;   // the kernels are built for sm_90a only
    if (cudaSetDevice(device) != cudaSuccess) return PLSTVO_E_NO_DEVICE;
    PlContext* ctx = new PlContext();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    cudaStreamCreateWithFlags(&ctx->s_main, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_alt, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking);
    *out = ctx;
    return 0;
}

void plstvo_destroy(PlContext* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    delete ctx;
}

const char* plstvo_last_error(const PlContext* ctx) { return ctx ? ctx->err.c_str() : "no context"; }

void plstvo_default_config(PlConfig* c) {   // src/config.cpp:36-113
    c->has_points = 1; c->has_lines = 1; c->best_lr_matches = 1; c->use_motion_model = 0;
    c->min_features = 10; c->max_iters = 5; c->max_iters_ref = 10; c->solver_mode = 0;
    c->min_ratio_12_p = 0.9; c->min_ratio_12_l = 0.9; c->homog_th = 1e-7; c->min_error = 1e-7;
    c->min_error_change = 1e-7; c->inlier_k = 4.0; c->lsd_scale = 1.2;
}

void plstvo_kitti_config(PlConfig* c) {   // config/config/config_kitti.yaml:19,27,45
    plstvo_default_config(c);
    c->min_ratio_12_p = 0.75;
    c->min_ratio_12_l = 0.75;
    c->inlier_k = 1.2;
}

int plstvo_synchronize(PlContext* ctx) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaStreamSynchronize(ctx->s_h2d));
    CK(ctx, cudaStreamSynchronize(ctx->s_main));
    CK(ctx, cudaStreamSynchronize(ctx->s_alt));
    CK(ctx, cudaStreamSynchronize(ctx->s_d2h));
    return 0;
}

void* plstvo_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
    return p;
}
void plstvo_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

int64_t plstvo_launch_count(const PlContext* ctx) { return ctx ? ctx->launches : 0; }

// ---- matching.h surface -------------------------------------------------------------------------------
// Plans the B problems of a plstvo_match_batch call as a points-only frame batch on ctx->ws, uploads them and enqueues K1
// (distance + top-2, resolve) on ctx->s_main.  The caller holds the lock, has validated B > 0
// and selected the device; on success ws.problems[2 p] is problem p, its partial keys pending on ctx->s_main.
static int match_batch_launch(PlContext* ctx, int B, const uint8_t* d1, const int32_t* off1, const uint8_t* d2,
                              const int32_t* off2, float nnr, int best_lr_matches) {
    std::vector<int32_t> zeros((size_t)B + 1, 0);
    PlFrameBatch a{}, b{};
    a.B = b.B = B;
    a.pt_off = off1; b.pt_off = off2;
    a.ls_off = b.ls_off = zeros.data();
    a.pdesc = d1; b.pdesc = d2;
    int rc = validate_frames(ctx, &a, &b, false);
    if (rc) return rc;
    PlConfig cfg;
    plstvo_default_config(&cfg);
    cfg.has_lines = 0;
    cfg.best_lr_matches = best_lr_matches;
    Workspace& ws = ctx->ws;
    rc = ws_prepare(ctx, ws, nullptr, &cfg, &a, &b, false, false);
    if (rc) return rc;
    ws.planned = false;                          // the plan is patched below: never reuse it
    for (auto& pr : ws.problems) pr.nnr = nnr;   // the caller's float, not the config's double
    CK(ctx, cudaMemcpyAsync(ws.d_problems.p, ws.problems.data(), ws.problems.size() * sizeof(MatchProblem),
                            cudaMemcpyHostToDevice, ctx->s_h2d));
    rc = ws_upload_range(ctx, ws, &a, &b, nullptr, 0, B, false, ctx->s_h2d);
    if (rc) return rc;
    cudaEvent_t up = next_event(ctx);
    CK(ctx, cudaEventRecord(up, ctx->s_h2d));
    CK(ctx, cudaStreamWaitEvent(ctx->s_main, up, 0));
    return ws_launch_match(ctx, ws, 0, B, ctx->s_main);
}

int plstvo_match_batch(PlContext* ctx, int B, const uint8_t* d1, const int32_t* off1, const uint8_t* d2,
                       const int32_t* off2, float nnr, int best_lr_matches, int32_t* m12, int32_t* counts) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (B < 0 || (B > 0 && (!off1 || !off2 || !m12))) return fail(ctx, PLSTVO_E_INVALID, "bad arguments");
    if (B == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = match_batch_launch(ctx, B, d1, off1, d2, off2, nnr, best_lr_matches);
    if (rc) return rc;
    Workspace& ws = ctx->ws;
    // finalize only the point problems (even indices): compact view
    CK(ctx, ctx->scratch.ensure((size_t)B * (sizeof(MatchProblem) + 4)));
    std::vector<MatchProblem> pts((size_t)B);
    for (int p = 0; p < B; ++p) pts[p] = ws.problems[(size_t)2 * p];
    MatchProblem* d_pts = ctx->scratch.as<MatchProblem>();
    int32_t* d_counts = reinterpret_cast<int32_t*>(d_pts + B);
    CK(ctx, cudaMemcpyAsync(d_pts, pts.data(), (size_t)B * sizeof(MatchProblem), cudaMemcpyHostToDevice, ctx->s_main));
    CK(ctx, launch_match_finalize(d_pts, B, ws.max_n2, d_counts, ctx->s_main));
    ctx->launches++;
    if ((rc = ws_download_range(ctx, ws, 0, B, nullptr, m12, nullptr, nullptr, nullptr, ctx->s_main))) return rc;
    return counts_total(ctx, ctx->s_main, B, d_counts, counts);
}

int plstvo_match(PlContext* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2, int stride_bytes,
                 float nnr, int best_lr_matches, int32_t* m12) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (stride_bytes != PLSTVO_DESC_BYTES) return fail(ctx, PLSTVO_E_INVALID, "descriptor rows must be 32 contiguous bytes");
    if (n1 < 0 || n2 < 0) return fail(ctx, PLSTVO_E_INVALID, "negative row count");
    if (n1 == 0) return 0;
    if (!m12) return fail(ctx, PLSTVO_E_INVALID, "null output");
    const int32_t o1[2] = {0, n1}, o2[2] = {0, n2};
    return plstvo_match_batch(ctx, 1, d1, o1, d2, o2, nnr, best_lr_matches, m12, nullptr);
}

int plstvo_match_nnr(PlContext* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2, int stride_bytes,
                     float nnr, int32_t* m12) {
    return plstvo_match(ctx, d1, n1, d2, n2, stride_bytes, nnr, 0, m12);
}

int plstvo_debug_tc_partials(PlContext* ctx, int B, const uint8_t* d1, const int32_t* off1, const uint8_t* d2,
                             const int32_t* off2, float nnr, uint32_t* rowp, uint32_t* colp, uint32_t* rowkey,
                             uint32_t* colkey) {
    if (!ctx) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (B < 0 || (B > 0 && (!off1 || !off2 || !rowp || !colp || !rowkey || !colkey)))
        return fail(ctx, PLSTVO_E_INVALID, "bad arguments");
    if (B == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = match_batch_launch(ctx, B, d1, off1, d2, off2, nnr, 1);
    if (rc) return rc;
    const Workspace& ws = ctx->ws;
    cudaStream_t s = ctx->s_main;
    size_t row0 = 0;   // first row word of problem p in the caller's rowp
    for (int p = 0; p < B; ++p) {
        const MatchProblem& pr = ws.problems[(size_t)2 * p];
        const TcProblem& tp = ws.tc_problems[(size_t)2 * p];
        const size_t nrow = (size_t)((pr.n2 + TC_CW - 1) / TC_CW) * pr.n1;
        if (pr.enabled) {   // a problem with an empty side has no words: its slots are left as they are
            CK(ctx, cudaMemcpyAsync(rowp + row0, tp.rowp, nrow * 4, cudaMemcpyDeviceToHost, s));
            CK(ctx, cudaMemcpyAsync(colp + off2[p], tp.colp, (size_t)pr.n2 * 4, cudaMemcpyDeviceToHost, s));
            CK(ctx, cudaMemcpyAsync(rowkey + 2 * (size_t)off1[p], pr.rowpart, (size_t)pr.n1 * sizeof(uint2),
                                    cudaMemcpyDeviceToHost, s));
            CK(ctx, cudaMemcpyAsync(colkey + 2 * (size_t)off2[p], pr.colpart, (size_t)pr.n2 * sizeof(uint2),
                                    cudaMemcpyDeviceToHost, s));
        }
        row0 += nrow;
    }
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

// ---- stereoFrameHandler.h surface ------------------------------------------------------------------------
int plstvo_f2f_tracking(PlContext* ctx, const PlConfig* cfg, const PlFrameBatch* prev, const PlFrameBatch* curr,
                        int32_t* m12_pt, int32_t* m12_ls, int32_t* n_matched) {
    if (!ctx || !cfg) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = validate_frames(ctx, prev, curr, false);
    if (rc) return rc;
    const int B = prev->B;
    if (B == 0) return 0;
    Workspace& ws = ctx->ws;
    rc = ws_prepare(ctx, ws, nullptr, cfg, prev, curr, false, false);
    if (rc) return rc;
    rc = ws_upload_range(ctx, ws, prev, curr, nullptr, 0, B, false, ctx->s_h2d);
    if (rc) return rc;
    cudaEvent_t up = next_event(ctx);
    CK(ctx, cudaEventRecord(up, ctx->s_h2d));
    CK(ctx, cudaStreamWaitEvent(ctx->s_main, up, 0));
    rc = ws_launch_match(ctx, ws, 0, B, ctx->s_main);
    if (rc) return rc;
    CK(ctx, ctx->scratch.ensure((size_t)2 * B * 4));
    CK(ctx, launch_match_finalize(ws.d_problems.as<MatchProblem>(), 2 * B, ws.max_n2, ctx->scratch.as<int32_t>(),
                                  ctx->s_main));
    ctx->launches++;
    if ((rc = ws_download_range(ctx, ws, 0, B, nullptr, m12_pt, m12_ls, nullptr, nullptr, ctx->s_main))) return rc;
    if (n_matched)
        CK(ctx, cudaMemcpyAsync(n_matched, ctx->scratch.p, (size_t)2 * B * 4, cudaMemcpyDeviceToHost, ctx->s_main));
    CK(ctx, cudaStreamSynchronize(ctx->s_main));
    return 0;
}

int plstvo_optimize_pose(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m,
                         const PlPrior* priors, PlPoseResult* results, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    if (!ctx || !cam || !cfg || !m || !results) return PLSTVO_E_INVALID;
    LOCK(ctx);
    const int B = m->B;
    if (B < 0) return fail(ctx, PLSTVO_E_INVALID, "negative batch size");
    if (B == 0) return 0;
    // (explicit lists may start past row 0 of their arrays)
    if (const int rc = check_offsets(ctx, B, {m->pt_off, m->ls_off}, "null offsets", "offsets are not non-decreasing",
                                     "list too long", false))
        return rc;
    CK(ctx, cudaSetDevice(ctx->device));
    int cap_pt = 1, cap_ls = 1;
    for (int p = 0; p < B; ++p) {
        cap_pt = std::max(cap_pt, m->pt_off[p + 1] - m->pt_off[p]);
        cap_ls = std::max(cap_ls, m->ls_off[p + 1] - m->ls_off[p]);
    }
    const size_t n = m->pt_off[B], l = m->ls_off[B];
    if (n && (!m->pt_P || !m->pt_pl_obs || !m->pt_sigma2)) return fail(ctx, PLSTVO_E_INVALID, "point arrays missing");
    if (l && (!m->ls_sP || !m->ls_eP || !m->ls_le_obs || !m->ls_spl || !m->ls_epl || !m->ls_sigma2))
        return fail(ctx, PLSTVO_E_INVALID, "line arrays missing");
    const SolvePlan plan = plan_solve(ctx, cap_pt, cap_ls, 0, B, cfg->solver_mode);
    if (!plan.fits) return fail(ctx, PLSTVO_E_TOO_LARGE, "lists too long for the per-pair solver's shared memory");

    Workspace& ws = ctx->ws;
    ws.planned = false;   // the explicit-list path reuses the workspace's buffers with its own layout
    cudaStream_t s = ctx->s_main;
    RecPtrs lists;
    if (const int rc = upload_matched(ctx, m, ws.prev, s, &lists)) return rc;
    CK(ctx, ws.d_results.ensure((size_t)B * sizeof(PlPoseResult)));
    CK(ctx, ws.d_priors.ensure((size_t)B * sizeof(PlPrior)));
    if (priors) CK(ctx, cudaMemcpyAsync(ws.d_priors.p, priors, (size_t)B * sizeof(PlPrior), cudaMemcpyHostToDevice, s));
    // output flags live in separate buffers (the input flags are read while the outputs are written)
    CK(ctx, ctx->gn_out[0].ensure(std::max<size_t>(n, 16)));
    CK(ctx, ctx->gn_out[1].ensure(std::max<size_t>(l, 16)));
    if (plan.feat_stride) CK(ctx, ws.d_feat.ensure((size_t)B * plan.feat_stride * sizeof(double)));
    SolveParams prm{};
    prm.cam = *cam;
    prm.cfg = *cfg;
    prm.mode = 1;
    prm.prev = prm.curr = rows_dev(ws.prev.pt_off, ws.prev.ls_off, lists);
    prm.priors = priors ? ws.d_priors.as<PlPrior>() : nullptr;
    prm.results = ws.d_results.as<PlPoseResult>();
    prm.inlier_pt = ctx->gn_out[0].as<uint8_t>();
    prm.inlier_ls = ctx->gn_out[1].as<uint8_t>();
    if (const int rc = launch_solver(ctx, prm, plan, ws.d_feat.as<double>(), ws.d_stream, B, n, l, 0, B, s)) return rc;
    CK(ctx, cudaMemcpyAsync(results, ws.d_results.p, (size_t)B * sizeof(PlPoseResult), cudaMemcpyDeviceToHost, s));
    if (inlier_pt && n) CK(ctx, cudaMemcpyAsync(inlier_pt, ctx->gn_out[0].p, n, cudaMemcpyDeviceToHost, s));
    if (inlier_ls && l) CK(ctx, cudaMemcpyAsync(inlier_ls, ctx->gn_out[1].p, l, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

// enqueue one batch on the context's streams: chunked H2D -> K1 -> K2 -> D2H, nothing is waited for.  cams (optional, host,
// [B]): pair p is solved under cams[p] instead of cam.
static int track_enqueue(PlContext* ctx, Workspace& ws, const PlCamera* cam, const PlConfig* cfg,
                         const PlFrameBatch* prev, const PlFrameBatch* curr, const PlPrior* priors,
                         PlPoseResult* results, int32_t* m12_pt, int32_t* m12_ls, uint8_t* inlier_pt,
                         uint8_t* inlier_ls, bool pipelined, const PlCamera* cams = nullptr) {
    const int B = prev->B;
    if (cams) {   // ahead of the first chunk's uploads on the same stream, so every chunk's solver sees it
        CK(ctx, ws.d_pair_cams.ensure((size_t)B * sizeof(PlCamera)));
        CK(ctx, cudaMemcpyAsync(ws.d_pair_cams.p, cams, (size_t)B * sizeof(PlCamera), cudaMemcpyHostToDevice, ctx->s_h2d));
    }
    int rc = ws_prepare(ctx, ws, cam, cfg, prev, curr, true, priors != nullptr, cams ? ws.d_pair_cams.as<PlCamera>() : nullptr);
    if (rc) return rc;
    const bool have_level = prev->ls_level != nullptr;
    const std::vector<int> bounds = chunk_schedule(B, ctx->sm_count, pipelined);
    for (int k = 0; k + 1 < (int)bounds.size(); ++k) {
        const int p0 = bounds[k], p1 = bounds[k + 1];
        rc = ws_upload_range(ctx, ws, prev, curr, priors, p0, p1, true, ctx->s_h2d);
        if (rc) return rc;
        cudaEvent_t up = next_event(ctx);
        CK(ctx, cudaEventRecord(up, ctx->s_h2d));
        cudaStream_t s = (k & 1) ? ctx->s_alt : ctx->s_main;
        CK(ctx, cudaStreamWaitEvent(s, up, 0));
        rc = ws_launch_match(ctx, ws, p0, p1, s);
        if (rc) return rc;
        rc = ws_launch_solve(ctx, ws, p0, p1, have_level, s);
        if (rc) return rc;
        cudaEvent_t done = next_event(ctx);
        CK(ctx, cudaEventRecord(done, s));
        CK(ctx, cudaStreamWaitEvent(ctx->s_d2h, done, 0));
        rc = ws_download_range(ctx, ws, p0, p1, results, m12_pt, m12_ls, inlier_pt, inlier_ls, ctx->s_d2h);
        if (rc) return rc;
    }
    return 0;
}

int plstvo_track_batch(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                       const PlFrameBatch* curr, const PlPrior* priors, PlPoseResult* results, int32_t* m12_pt,
                       int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    if (!ctx || !cam || !cfg) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = validate_frames(ctx, prev, curr, true);
    if (rc) return rc;
    if (prev->B == 0) return 0;
    rc = track_enqueue(ctx, ctx->ws, cam, cfg, prev, curr, priors, results, m12_pt, m12_ls, inlier_pt, inlier_ls, false);
    if (rc) return rc;
    CK(ctx, cudaStreamSynchronize(ctx->s_d2h));   // every chunk's D2H waited for its compute, which waited for its H2D
    return 0;
}

int plstvo_track_batch_cams(PlContext* ctx, const PlCamera* cams, const PlConfig* cfg, const PlFrameBatch* prev,
                            const PlFrameBatch* curr, const PlPrior* priors, PlPoseResult* results, int32_t* m12_pt,
                            int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    if (!ctx || !cams || !cfg) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = validate_frames(ctx, prev, curr, true);
    if (rc) return rc;
    if (prev->B == 0) return 0;
    rc = track_enqueue(ctx, ctx->ws, &cams[0], cfg, prev, curr, priors, results, m12_pt, m12_ls, inlier_pt, inlier_ls, false,
                       cams);
    if (rc) return rc;
    CK(ctx, cudaStreamSynchronize(ctx->s_d2h));
    return 0;
}

int plstvo_track_batch_async(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                             const PlFrameBatch* curr, const PlPrior* priors, PlPoseResult* results, int32_t* m12_pt,
                             int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    if (!ctx || !cam || !cfg) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = validate_frames(ctx, prev, curr, true);
    if (rc) return rc;
    const int slot = acquire_slot(ctx);
    if (slot < 0) return slot;
    if (prev->B > 0) {
        rc = track_enqueue(ctx, ctx->ws_async[slot], cam, cfg, prev, curr, priors, results, m12_pt, m12_ls, inlier_pt,
                           inlier_ls, true);
        if (rc) return rc;
    }
    CK(ctx, cudaEventRecord(ctx->slot_done[slot], ctx->s_d2h));
    ctx->slot_busy[slot] = true;
    return slot;
}

int plstvo_wait(PlContext* ctx, int ticket) {
    if (!ctx || ticket < 0 || ticket > 1) return PLSTVO_E_INVALID;
    cudaEvent_t ev = nullptr;
    {
        LOCK(ctx);
        CK(ctx, cudaSetDevice(ctx->device));
        if (ctx->slot_busy[ticket]) ev = ctx->slot_done[ticket];
    }
    if (ev) {   // wait outside the lock: other threads may keep enqueueing on this context
        const cudaError_t e = cudaEventSynchronize(ev);
        LOCK(ctx);   // ctx->err is only ever written under the lock
        CK(ctx, e);
        ctx->slot_busy[ticket] = false;
    }
    return 0;
}

// ---- throughput mode ----------------------------------------------------------------------------------
int plstvo_batch_upload(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                        const PlFrameBatch* curr, const PlPrior* priors, PlDeviceBatch** out) {
    if (!ctx || !cam || !cfg || !out) return PLSTVO_E_INVALID;
    LOCK(ctx);
    *out = nullptr;
    CK(ctx, cudaSetDevice(ctx->device));
    int rc = validate_frames(ctx, prev, curr, true);
    if (rc) return rc;
    PlDeviceBatch* db = new PlDeviceBatch();
    rc = ws_prepare(ctx, db->ws, cam, cfg, prev, curr, true, priors != nullptr);
    if (rc == 0 && prev->B > 0) rc = ws_upload_range(ctx, db->ws, prev, curr, priors, 0, prev->B, true, ctx->s_h2d);
    if (rc == 0) {
        cudaError_t e = cudaStreamSynchronize(ctx->s_h2d);
        if (e != cudaSuccess) {
            ctx->err = cudaGetErrorString(e);
            rc = PLSTVO_E_CUDA;
        }
    }
    if (rc) {
        delete db;
        return rc;
    }
    db->ws.have_level = prev->ls_level != nullptr;
    *out = db;
    return 0;
}

int plstvo_batch_run(PlContext* ctx, PlDeviceBatch* db) {
    if (!ctx || !db) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    return ws_run(ctx, db->ws, db->ws.have_level);
}

int plstvo_batch_run_timed(PlContext* ctx, PlDeviceBatch* db, int iters, int flush_l2, float* ms_total) {
    if (!ctx || !db || iters <= 0 || !ms_total) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t flush_bytes = 256u << 20;
    if (flush_l2) CK(ctx, ctx->scratch.ensure(flush_bytes));
    Events<2> ev;
    CK(ctx, ev.create());
    const cudaEvent_t e0 = ev[0], e1 = ev[1];
    double total = 0.0;
    CK(ctx, cudaStreamSynchronize(ctx->s_main));
    if (!flush_l2) {
        CK(ctx, cudaEventRecord(e0, ctx->s_main));
        for (int i = 0; i < iters; ++i) {
                    int rc = ws_run(ctx, db->ws, db->ws.have_level);
            if (rc) return rc;
        }
        CK(ctx, cudaEventRecord(e1, ctx->s_main));
        CK(ctx, cudaEventSynchronize(e1));
        float ms = 0.f;
        CK(ctx, cudaEventElapsedTime(&ms, e0, e1));
        total = ms;
    } else {
        for (int i = 0; i < iters; ++i) {
            CK(ctx, cudaMemsetAsync(ctx->scratch.p, i & 0xFF, flush_bytes, ctx->s_main));
            CK(ctx, cudaEventRecord(e0, ctx->s_main));
                    int rc = ws_run(ctx, db->ws, db->ws.have_level);
            if (rc) return rc;
            CK(ctx, cudaEventRecord(e1, ctx->s_main));
            CK(ctx, cudaEventSynchronize(e1));
            float ms = 0.f;
            CK(ctx, cudaEventElapsedTime(&ms, e0, e1));
            total += ms;
        }
    }
    *ms_total = (float)total;
    return 0;
}

// One solve pass over the resident batch with the solver kernels' cycle counters on; h: [B][PLSTVO_PHASE_SLOTS] on the host.
static int ws_phase_pass(PlContext* ctx, Workspace& ws, long long* h) {
    const size_t bytes = (size_t)ws.B * PLSTVO_PHASE_SLOTS * sizeof(long long);
    CK(ctx, ws.d_phase.ensure(bytes));
    CK(ctx, cudaMemsetAsync(ws.d_phase.p, 0, bytes, ctx->s_main));
    int rc = ws_launch_solve(ctx, ws, 0, ws.B, ws.have_level, ctx->s_main);
    if (rc) return rc;
    CK(ctx, cudaMemcpyAsync(h, ws.d_phase.p, bytes, cudaMemcpyDeviceToHost, ctx->s_main));
    CK(ctx, cudaStreamSynchronize(ctx->s_main));
    ws.d_phase.release();
    return 0;
}

int plstvo_batch_phase_cycles(PlContext* ctx, PlDeviceBatch* db, int64_t* out) {
    if (!ctx || !db || !out) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    if (db->ws.B <= 0) return 0;
    static_assert(sizeof(long long) == sizeof(int64_t), "phase counters");
    return ws_phase_pass(ctx, db->ws, reinterpret_cast<long long*>(out));
}

int plstvo_batch_kernel_times(PlContext* ctx, PlDeviceBatch* db, int iters, double* ms_match, double* ms_solve,
                              int32_t* n_tiles, int32_t* n_pairs) {
    if (!ctx || !db || iters <= 0) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    Workspace& ws = db->ws;
    Events<3> ev;
    CK(ctx, ev.create());
    const cudaEvent_t e0 = ev[0], e1 = ev[1], e2 = ev[2];
    double tm = 0.0, tsv = 0.0;
    const bool lev = ws.have_level;
    for (int i = 0; i < iters; ++i) {
        CK(ctx, cudaEventRecord(e0, ctx->s_main));
        int rc = ws_launch_match(ctx, ws, 0, ws.B, ctx->s_main);
        if (rc) return rc;
        CK(ctx, cudaEventRecord(e1, ctx->s_main));
        rc = ws_launch_solve(ctx, ws, 0, ws.B, lev, ctx->s_main);
        if (rc) return rc;
        CK(ctx, cudaEventRecord(e2, ctx->s_main));
        CK(ctx, cudaEventSynchronize(e2));
        float a = 0.f, b = 0.f;
        CK(ctx, cudaEventElapsedTime(&a, e0, e1));
        CK(ctx, cudaEventElapsedTime(&b, e1, e2));
        tm += a;
        tsv += b;
    }
    if (ms_match) *ms_match = tm / iters;
    if (ms_solve) *ms_solve = tsv / iters;
    if (n_tiles) *n_tiles = (int32_t)std::count_if(ws.problems.begin(), ws.problems.end(),
                                                   [](const MatchProblem& pr) { return pr.enabled != 0; });
    if (n_pairs) *n_pairs = ws.B;
    return 0;
}

int plstvo_batch_stage_times(PlContext* ctx, PlDeviceBatch* db, int iters, double ms[8], int32_t counts[4]) {
    if (!ctx || !db || iters <= 0 || !ms) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    Workspace& ws = db->ws;
    // events: 0 start, 1 before the matcher (operands are expanded inside it: 0 -> 1 is empty), 2 distance done, 3 match done,
    // 4 lists done, 5 GN stage 1 done, 6 outlier pass done, 7 GN stage 2 done, 8 end
    Events<9> evs;
    CK(ctx, evs.create());
    cudaEvent_t* ev = evs.ev;
    double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < iters; ++i) {
        CK(ctx, cudaEventRecord(ev[0], ctx->s_main));
        int rc = ws_launch_match(ctx, ws, 0, ws.B, ctx->s_main, &ev[1]);
        if (rc) return rc;
        CK(ctx, cudaEventRecord(ev[3], ctx->s_main));
        rc = ws_launch_solve(ctx, ws, 0, ws.B, ws.have_level, ctx->s_main, &ev[4]);
        if (rc) return rc;
        CK(ctx, cudaEventRecord(ev[8], ctx->s_main));
        CK(ctx, cudaEventSynchronize(ev[8]));
        auto span = [&](int a, int b, double& out) -> int {
            float t = 0.f;
            CK(ctx, cudaEventElapsedTime(&t, ev[a], ev[b]));
            out += t;
            return 0;
        };
        for (int k = 0; k < 4; ++k)
            if ((rc = span(k, k + 1, acc[k]))) return rc;
        if ((rc = span(4, 8, acc[4])) || (rc = span(4, 5, acc[5])) || (rc = span(5, 6, acc[6])) || (rc = span(6, 7, acc[7]))) return rc;
    }
    for (int k = 0; k < 8; ++k) ms[k] = acc[k] / iters;
    if (counts) {
        int delegated = 0;   // streamed solver: problems it handed to the fp64 kernel in the last pass (its only_if list)
        if (ws.solver.use_stream && ws.B > 0) {
            StreamBufs sb;
            int rc = stream_bufs_prepare(ctx, ws.d_stream, ws.B, (size_t)ws.p_off1[ws.B], (size_t)ws.l_off1[ws.B], &sb);
            if (rc) return rc;
            std::vector<int32_t> act((size_t)ws.B);
            CK(ctx, cudaMemcpy(act.data(), sb.active, (size_t)ws.B * sizeof(int32_t), cudaMemcpyDeviceToHost));
            for (int32_t a : act) delegated += a != 0;
        }
        counts[0] = 1 | (ws.solver.use_stream ? 2 : 0) | (delegated << 8);   // bit 0: the tensor-core matcher, the only form
        counts[1] = (int32_t)(ws.tc_items[0].size() + ws.tc_items[1].size());
        counts[2] = (int32_t)ws.problems.size();
        counts[3] = ws.B;
    }
    return 0;
}

int plstvo_batch_download(PlContext* ctx, PlDeviceBatch* db, PlPoseResult* results, int32_t* m12_pt,
                          int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls) {
    if (!ctx || !db) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    if (db->ws.B == 0) return 0;
    int rc = ws_download_range(ctx, db->ws, 0, db->ws.B, results, m12_pt, m12_ls, inlier_pt, inlier_ls, ctx->s_main);
    if (rc) return rc;
    CK(ctx, cudaStreamSynchronize(ctx->s_main));
    return 0;
}

void plstvo_batch_free(PlContext* ctx, PlDeviceBatch* db) {
    if (!db) return;
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaDeviceSynchronize();
    }
    delete db;
}

int plstvo_debug_select(PlContext* ctx, int n_lists, const int32_t* off, const double* values, const int32_t* k,
                        const double* pivot, int mode, double* out) {
    if (!ctx || n_lists < 0 || !off || !k || !out || (mode != 0 && mode != 1) || (mode == 1 && !pivot)) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (n_lists == 0) return 0;
    const size_t n = (size_t)off[n_lists];
    if (n > 0 && !values) return PLSTVO_E_INVALID;
    for (int p = 0; p < n_lists; ++p) {
        const int len = off[p + 1] - off[p];
        if (len < 0 || (len > 0 && (k[p] < 0 || k[p] >= len))) return PLSTVO_E_INVALID;
    }
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t b_v = (n + 2) * 8, b_o = ((size_t)n_lists + 2) * 4, b_k = (size_t)n_lists * 4 + 8, b_p = (size_t)n_lists * 8;
    CK(ctx, ctx->scratch.ensure(b_v + b_o + b_k + 2 * b_p + 64));
    uint8_t* d = ctx->scratch.as<uint8_t>();
    double* dv = reinterpret_cast<double*>(d);
    double* dp = reinterpret_cast<double*>(d + b_v);
    double* dout = reinterpret_cast<double*>(d + b_v + b_p);
    int32_t* doff = reinterpret_cast<int32_t*>(d + b_v + 2 * b_p);
    int32_t* dk = reinterpret_cast<int32_t*>(d + b_v + 2 * b_p + (b_o + 7) / 8 * 8);
    cudaStream_t s = ctx->s_main;
    if (n) CK(ctx, cudaMemcpyAsync(dv, values, n * 8, cudaMemcpyHostToDevice, s));
    CK(ctx, cudaMemcpyAsync(doff, off, ((size_t)n_lists + 1) * 4, cudaMemcpyHostToDevice, s));
    CK(ctx, cudaMemcpyAsync(dk, k, (size_t)n_lists * 4, cudaMemcpyHostToDevice, s));
    if (pivot) CK(ctx, cudaMemcpyAsync(dp, pivot, b_p, cudaMemcpyHostToDevice, s));
    CK(ctx, cudaMemsetAsync(dout, 0, b_p, s));
    CK(ctx, launch_select_selftest(dv, doff, dk, pivot ? dp : nullptr, mode, n_lists, dout, s));
    ctx->launches++;
    CK(ctx, cudaMemcpyAsync(out, dout, b_p, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

int plstvo_debug_algebra(PlContext* ctx, int n, const double* H, const double* g, double* x, double* lad, double* inv,
                         double* eig) {
    if (!ctx || n < 0 || !H || !g || !x || !lad || !inv || !eig) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (n == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t in_b = (size_t)n * 42 * 8, out_b = (size_t)n * 49 * 8;
    CK(ctx, ctx->scratch.ensure(in_b + out_b));
    double* d = ctx->scratch.as<double>();
    double *dH = d, *dg = d + (size_t)n * 36, *dx = dg + (size_t)n * 6, *dl = dx + (size_t)n * 6, *di = dl + n,
           *de = di + (size_t)n * 36;
    cudaStream_t s = ctx->s_main;
    CK(ctx, cudaMemcpyAsync(dH, H, (size_t)n * 36 * 8, cudaMemcpyHostToDevice, s));
    CK(ctx, cudaMemcpyAsync(dg, g, (size_t)n * 6 * 8, cudaMemcpyHostToDevice, s));
    CK(ctx, launch_algebra_selftest(dH, dg, n, dx, dl, di, de, s));
    ctx->launches++;
    CK(ctx, cudaMemcpyAsync(x, dx, (size_t)n * 6 * 8, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(lad, dl, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(inv, di, (size_t)n * 36 * 8, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(eig, de, (size_t)n * 6 * 8, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

int plstvo_debug_pose_helpers(PlContext* ctx, int n, const double* in, double* out) {
    if (!ctx || n < 0 || !in || !out) return PLSTVO_E_INVALID;
    LOCK(ctx);
    if (n == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t in_b = (size_t)n * PLSTVO_PH_IN * 8, out_b = (size_t)n * PLSTVO_PH_OUT * 8;
    CK(ctx, ctx->scratch.ensure(in_b + out_b));
    double* d = ctx->scratch.as<double>();
    double* dout = d + (size_t)n * PLSTVO_PH_IN;
    cudaStream_t s = ctx->s_main;
    CK(ctx, cudaMemcpyAsync(d, in, in_b, cudaMemcpyHostToDevice, s));
    CK(ctx, launch_pose_helpers_selftest(d, n, dout, s));
    ctx->launches++;
    CK(ctx, cudaMemcpyAsync(out, dout, out_b, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    return 0;
}

int plstvo_popc_rate(PlContext* ctx, double* popc_per_s) {
    if (!ctx || !popc_per_s) return PLSTVO_E_INVALID;
    LOCK(ctx);
    CK(ctx, cudaSetDevice(ctx->device));
    const int blocks = ctx->sm_count * 8, iters = 20000;
    CK(ctx, ctx->scratch.ensure((size_t)blocks * 256 * 4));
    Events<2> ev;
    CK(ctx, ev.create());
    const cudaEvent_t e0 = ev[0], e1 = ev[1];
    CK(ctx, launch_popc_bench(ctx->scratch.as<uint32_t>(), 2000, blocks, ctx->s_main));   // warm-up
    CK(ctx, cudaEventRecord(e0, ctx->s_main));
    CK(ctx, launch_popc_bench(ctx->scratch.as<uint32_t>(), iters, blocks, ctx->s_main));
    CK(ctx, cudaEventRecord(e1, ctx->s_main));
    CK(ctx, cudaEventSynchronize(e1));
    ctx->launches += 2;
    float ms = 0.f;
    CK(ctx, cudaEventElapsedTime(&ms, e0, e1));
    *popc_per_s = (double)blocks * 256.0 * iters * 8.0 / (ms * 1e-3);
    return 0;
}

int plstvo_gn_eval_stream(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m,
                          const double* DT, int iters, double* H, double* g, double* e, float* ms_total) {
    if (!ctx || !cam || !cfg || !m || !DT || iters <= 0) return PLSTVO_E_INVALID;
    LOCK(ctx);
    const int B = m->B;
    if (B <= 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    const size_t n = m->pt_off[B], l = m->ls_off[B];
    cudaStream_t s = ctx->s_main;
    RecPtrs lists;   // resident inputs of the roofline run (context lifetime)
    if (const int rc = upload_matched(ctx, m, ctx->gs_in, s, &lists)) return rc;
    const RowsDev md = rows_dev(ctx->gs_in.pt_off, ctx->gs_in.ls_off, lists);
    // fp32-packed records (SURVEY 8(a) A4/A5: 32 B per point, 64 B per line), packed once on the device
    DevBuf &rec_pt = ctx->gs_rec_pt, &rec_ls = ctx->gs_rec_ls;
    CK(ctx, rec_pt.ensure(std::max<size_t>(n * 32, 32)));
    CK(ctx, rec_ls.ensure(std::max<size_t>(l * 64, 64)));
    CK(ctx, launch_pack_records(md, *cam, B, (int)n, (int)l, rec_pt.as<float4>(), rec_ls.as<float4>(), s));
    ctx->launches++;
    // slices per problem: a work item is ~12 tiles of 16 KB (more slices only when the batch cannot fill the persistent grid)
    int max_tiles = 1;
    for (int p = 0; p < B; ++p)
        max_tiles = std::max(max_tiles, gn_stream_tiles(m->pt_off[p + 1] - m->pt_off[p], m->ls_off[p + 1] - m->ls_off[p]));
    int bpp = std::max(1, std::min(64, max_tiles / 12));
    while ((long)B * bpp < 4L * ctx->sm_count && 2 * bpp <= max_tiles && bpp < 64) ++bpp;
    CK(ctx, ctx->gn_in[0].ensure((size_t)B * 16 * 8));
    CK(ctx, ctx->gn_in[1].ensure((size_t)B * bpp * gn_stream_partials_per_slice() * (ACC_N + 1) * 8));
    CK(ctx, ctx->gn_out[2].ensure((size_t)B * 36 * 8));
    CK(ctx, ctx->gn_out[3].ensure((size_t)B * 7 * 8));
    CK(ctx, cudaMemcpyAsync(ctx->gn_in[0].p, DT, (size_t)B * 16 * 8, cudaMemcpyHostToDevice, s));
    double* dH = ctx->gn_out[2].as<double>();
    double* dg = ctx->gn_out[3].as<double>();
    double* de = dg + (size_t)B * 6;
    Events<2> ev;
    CK(ctx, ev.create());
    const cudaEvent_t e0 = ev[0], e1 = ev[1];
    auto sweep = [&]() {
        return launch_gn_eval_stream(*cam, *cfg, md.pt_off, md.ls_off, rec_pt.as<float4>(),
                                     rec_ls.as<float4>(), B, ctx->gn_in[0].as<double>(), ctx->gn_in[1].as<double>(), bpp,
                                     ctx->sm_count, dH, dg, de, s);
    };
    CK(ctx, sweep());   // warm-up
    CK(ctx, cudaEventRecord(e0, s));
    for (int i = 0; i < iters; ++i) CK(ctx, sweep());
    CK(ctx, cudaEventRecord(e1, s));
    ctx->launches += 2 * (iters + 1);
    if (H) CK(ctx, cudaMemcpyAsync(H, dH, (size_t)B * 36 * 8, cudaMemcpyDeviceToHost, s));
    if (g) CK(ctx, cudaMemcpyAsync(g, dg, (size_t)B * 6 * 8, cudaMemcpyDeviceToHost, s));
    if (e) CK(ctx, cudaMemcpyAsync(e, de, (size_t)B * 8, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    float ms = 0.f;
    CK(ctx, cudaEventElapsedTime(&ms, e0, e1));
    if (ms_total) *ms_total = ms;
    return 0;
}

}  // extern "C"
