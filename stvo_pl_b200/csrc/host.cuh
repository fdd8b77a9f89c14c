// host.cuh — host side of the C-ABI (include/plstvo.h), shared by its three translation units: capi.cu (context, matching,
// tracking, throughput mode, instrumentation), capi_stereo.cu (matchGrid, lifting, matchStereo, tracking from stereo
// features) and capi_features.cu (ORB, LBD, tracking from stereo images).  Not part of the public boundary.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <initializer_list>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "match_tc.cuh"

namespace plstvo {

// Device memory that grows on demand and is freed by its owner's destructor.
struct DevBuf {
    void*  p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Pinned host memory of the size last asked for (when that grew), freed by its owner's destructor.
struct PinnedBuf {
    void*  p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() {
        if (p) cudaFreeHost(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMallocHost(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
};

// N CUDA events, destroyed by their owner's destructor (a context, or the scope of a timing call).
template <int N> struct Events {
    cudaEvent_t ev[N] = {};
    Events() = default;
    Events(const Events&) = delete;
    Events& operator=(const Events&) = delete;
    ~Events() {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
    cudaError_t create(unsigned flags = cudaEventDefault) {   // the ones not created yet
        for (cudaEvent_t& e : ev)
            if (!e) {
                cudaEvent_t t;
                if (const cudaError_t r = cudaEventCreateWithFlags(&t, flags)) return r;
                e = t;
            }
        return cudaSuccess;
    }
    cudaEvent_t& operator[](int k) { return ev[k]; }
};

// One DevBuf carved into slices: take() lays them out (256-byte aligned, in call order), alloc() sizes the buffer, then a
// slice is addressed by its offset.  up / down copy nothing for a null host pointer or zero bytes.
struct Arena {
    size_t off = 0;
    uint8_t* base = nullptr;
    size_t take(size_t bytes) {
        const size_t o = off;
        off += (bytes + 255) / 256 * 256;
        return o;
    }
    cudaError_t alloc(DevBuf& buf) {
        const cudaError_t e = buf.ensure(off);
        base = buf.as<uint8_t>();
        return e;
    }
    template <typename T> T* at(size_t o) const { return reinterpret_cast<T*>(base + o); }
    uint8_t* u8(size_t o) const { return base + o; }
    int32_t* i32(size_t o) const { return at<int32_t>(o); }
    float* f32(size_t o) const { return at<float>(o); }
    double* f64(size_t o) const { return at<double>(o); }
    cudaError_t up(size_t o, const void* src, size_t bytes, cudaStream_t s) const {
        return (src && bytes) ? cudaMemcpyAsync(base + o, src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
    }
    cudaError_t down(void* dst, size_t o, size_t bytes, cudaStream_t s) const {
        return (dst && bytes) ? cudaMemcpyAsync(dst, base + o, bytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
    }
};

// K2's list capacities and where it keeps the lists, and which solver a batch takes (capi.cu: plan_solve)
struct SolvePlan {
    int cap_pt = 1, cap_ls = 1, sort_cap = 1;
    bool feat_in_smem = true;
    bool fits = true;          // K2 can hold the lists, in shared memory or in global scratch
    bool use_stream = false;   // the streamed solver
    size_t feat_stride = 0;    // doubles of global list scratch per pair (0: none needed)
};

// One side of the tracker's device storage: the CSR offsets of its points and lines and one buffer per records.h array, each
// grown on demand to the rows of the call that uses it (a workspace's previous and current frame; explicit matched lists).
// Only the arrays a side's calls use are ever allocated; the others stay null.
struct FrameBufs {
    DevBuf pt_off, ls_off;
    DevBuf rec[N_REC];
    // the buffers of the arrays in role, the other entries null
    template <int N> RecPtrs rows(const int (&role)[N]) const {
        RecPtrs r;
        for (int k : role) r.p[k] = rec[k].p;
        return r;
    }
};

// the solver's view of rows r (device) under offsets pt_off / ls_off
inline RowsDev rows_dev(const DevBuf& pt_off, const DevBuf& ls_off, const RecPtrs& r) {
    RowsDev v;
    v.pt_off = pt_off.as<int32_t>();
    v.ls_off = ls_off.as<int32_t>();
    v.pt_P = r.at<double>(PT_P);
    v.pt_pl = r.at<double>(PT_PL);
    v.pt_sigma2 = r.at<double>(PT_S2);
    v.pt_inlier = r.at<uint8_t>(INL_PT);
    v.ls_sP = r.at<double>(LS_SP);
    v.ls_eP = r.at<double>(LS_EP);
    v.ls_le = r.at<double>(LS_LE);
    v.ls_spl = r.at<double>(LS_SPL);
    v.ls_epl = r.at<double>(LS_EPL);
    v.ls_sigma2 = r.at<double>(LS_S2);
    v.ls_level = r.at<int32_t>(LS_LEVEL);
    v.ls_inlier = r.at<uint8_t>(INL_LS);
    return v;
}

// Work plan + device storage of one batch of frame pairs (also the body of PlDeviceBatch)
struct Workspace {
    int B = 0;
    PlCamera cam{};
    PlConfig cfg{};
    bool has_priors = false;
    bool have_level = false;   // prev->ls_level supplied (null = level 0 everywhere)
    bool planned = false, planned_features = false;   // plan cache (ws_prepare)
    int sm_planned = 0;
    // host copies of the offsets
    std::vector<int32_t> p_off1, p_off2, l_off1, l_off2;
    // plan
    std::vector<MatchProblem> problems;   // [2B]: points, lines
    int max_n2 = 0;
    SolvePlan solver;
    // device storage: the previous frame's PREV_ROLE arrays and the tracker's m12 and inlier rows, the current frame's
    // CURR_ROLE arrays (plstvo_optimize_pose: its explicit lists in prev)
    FrameBufs prev, curr;
    DevBuf d_priors, d_results;
    DevBuf d_rowpart, d_colpart, d_problems, d_feat;
    DevBuf d_phase;   // solver phase cycle counters (plstvo_batch_phase_cycles)
    // K1 (match_tc.cu): per-block value partials, work items
    std::vector<TcProblem> tc_problems;   // [2B], parallel to `problems`
    std::vector<TcItem> tc_items[2];      // work items of the point problems (long) and of the line problems (short)
    std::vector<int32_t> item_start[2];   // [B+1] first work item of each pair in either list
    DevBuf d_tcprob, d_tcitems[2], d_rowp, d_colp, d_sched;
    DevBuf d_stream;       // arena of the streamed solver (frames too large for K2's shared memory)
    const PlCamera* d_cams = nullptr;   // optional device camera of each pair [B] (ws_prepare), else cam for every pair
    DevBuf d_pair_cams;    // plstvo_track_batch_cams: the caller's cameras, uploaded
};

}  // namespace plstvo

struct PlContext {
    std::recursive_mutex mu;   // entry points serialise on it: one context may be shared by the caller's threads
    int device = 0;
    int sm_count = 0;
    size_t smem_optin = 0;
    cudaStream_t s_main = nullptr, s_alt = nullptr, s_h2d = nullptr, s_d2h = nullptr;
    std::vector<cudaEvent_t> events;
    size_t next_event = 0;
    std::string err;
    int64_t launches = 0;
    plstvo::Workspace ws;          // reused by the host-buffer entry points
    plstvo::Workspace ws_async[2]; // double-buffered workspaces of plstvo_track_batch_async
    plstvo::Events<2> slot_done;
    bool slot_busy[2] = {false, false};
    int next_slot = 0;
    plstvo::DevBuf scratch;        // misc (popc bench, L2 flush)
    plstvo::DevBuf gn_in[8], gn_out[4];
    // per-entry-point device arenas (context-owned: a process may hold one context per GPU)
    plstvo::DevBuf arena_grid, arena_lift_pt, arena_lift_ls, arena_stereo;
    plstvo::DevBuf arena_track_stereo[3];   // [0]: blocking calls, [1 + slot]: plstvo_track_stereo_*_async
    plstvo::FrameBufs gs_in;       // resident inputs of the streamed evaluator (plstvo_gn_eval_stream): explicit lists
    plstvo::DevBuf gs_rec_pt, gs_rec_ls;   // their packed records
    plstvo::DevBuf arena_orb;      // plstvo_orb_compute_batch: images, level buffers, key points, outputs
    bool orb_tables = false;
    plstvo::Events<4> orb_ev;
    plstvo::DevBuf arena_orb_kp;   // plstvo_orb_detect_and_compute_batch: per-key-point arrays, sized once the selection is counted
    bool orb_computed = false, orb_detected = false;
    plstvo::Events<5> orb_det_ev;
    plstvo::DevBuf arena_lbd;      // plstvo_lbd_compute_batch: images, gradients, key lines, descriptors
    bool lbd_tables = false, lbd_computed = false;
    plstvo::Events<3> lbd_ev;
    plstvo::DevBuf arena_lsd;      // plstvo_lsd_detect_batch: images, scaled images, per-pixel scratch, regions
    plstvo::DevBuf arena_lsd_seg;  // its per-region arrays, sized once the regions are counted
    plstvo::DevBuf lsd_trig;       // cos / sin table of the gradient angles (lsd.cu), built once
    bool lsd_ran = false;
    plstvo::Events<6> lsd_ev;
    plstvo::DevBuf arena_rect;     // plstvo_rectify_batch / _raw_images_*: raw images (staging), rectified grey images
    bool rect_ran = false;
    plstvo::Events<2> rect_ev;     // the remap (or colour preparation) kernel's start and end
    // plstvo_track_stereo_images_*: [0] first upload, [1] stereo step start, [2] its end, [3] tracking end; the join of the LBD stream
    plstvo::Events<4> img_ev;
    plstvo::Events<1> img_join;
    plstvo::DevBuf arena_run;      // plstvo_stereo_session_run: grey images (no rectifier), threshold and results tables
    float img_ms[5] = {0, 0, 0, 0, 0};
    bool img_timed = false;
    // pinned host scratch (small tables and counters that must not block the enqueueing thread), same indexing as the arenas
    plstvo::PinnedBuf h_staging[3];

    ~PlContext() {   // the owner has synchronised the device; the members free their own memory and events
        for (cudaEvent_t e : events) cudaEventDestroy(e);
        for (cudaStream_t s : {s_main, s_alt, s_h2d, s_d2h})
            if (s) cudaStreamDestroy(s);
    }
};

// A rig's two CV_16SC2 + CV_16UC1 map pairs, resident in HBM (plstvo_rectifier_create).  Where both sides were given the same
// maps they are held once and m1[1], m2[1] alias side 0.  A colour rectifier (plstvo_rectifier_create_color) takes images of
// 3 or 4 interleaved channels and may hold no maps (maps false: the conversion to grey alone).
struct PlRectifier {
    PlContext* ctx = nullptr;
    int width = 0, height = 0;
    int channels = 1;
    bool maps = true;
    plstvo::DevBuf map1[2], map2[2];
    const short2* m1[2] = {nullptr, nullptr};
    const uint16_t* m2[2] = {nullptr, nullptr};
};

namespace plstvo {

#define CK(ctx, call)                                                                            \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess) {                                                                \
            char buf__[512];                                                                     \
            snprintf(buf__, sizeof(buf__), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,         \
                     cudaGetErrorString(e__));                                                   \
            (ctx)->err = buf__;                                                                  \
            return PLSTVO_E_CUDA;                                                                \
        }                                                                                        \
    } while (0)

#define LOCK(ctx) std::lock_guard<std::recursive_mutex> lock__((ctx)->mu)

inline int fail(PlContext* ctx, int code, const char* msg) {
    if (ctx) ctx->err = msg;
    return code;
}

// Cross-stream ordering events.  Each one is recorded and immediately waited on by the enqueuing host code, so a ring
// can be recycled while earlier work is still in flight (a wait captures the record that preceded it).
inline cudaEvent_t next_event(PlContext* ctx) {
    constexpr size_t RING = 512;
    if (ctx->events.size() < RING) {
        cudaEvent_t e;
        cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        ctx->events.push_back(e);
        return e;
    }
    return ctx->events[ctx->next_event++ % RING];
}

// CSR offsets [n + 1] of one or more row sets over the same n frames.  PLSTVO_E_INVALID with `bad` for a null array or (with
// from_zero) a first offset other than 0; then frame by frame, PLSTVO_E_INVALID with `decreasing` for a decreasing offset in
// any set, else PLSTVO_E_TOO_LARGE with `too_large` for more than PLSTVO_MAX_FEATURES rows in any set.
inline int check_offsets(PlContext* ctx, int n, std::initializer_list<const int32_t*> offs, const char* bad,
                         const char* decreasing, const char* too_large, bool from_zero = true) {
    for (const int32_t* off : offs)
        if (!off || (from_zero && off[0] != 0)) return fail(ctx, PLSTVO_E_INVALID, bad);
    for (int p = 0; p < n; ++p) {
        for (const int32_t* off : offs)
            if (off[p + 1] - off[p] < 0) return fail(ctx, PLSTVO_E_INVALID, decreasing);
        for (const int32_t* off : offs)
            if (off[p + 1] - off[p] > PLSTVO_MAX_FEATURES) return fail(ctx, PLSTVO_E_TOO_LARGE, too_large);
    }
    return 0;
}

// matchGrid's per-frame counts: a negative one is the error code of a frame with more than GRID_CAP candidates in a window
inline int check_grid_counts(PlContext* ctx, int n, const int32_t* gcnt) {
    for (int p = 0; p < n; ++p)
        if (gcnt[p] < 0) return fail(ctx, gcnt[p], "matchGrid: more than 128 candidates in one query window");
    return 0;
}

// The end of a blocking call with per-frame counts at d_cnt (device): downloads them on s behind the call's other copies
// (after matchGrid's, d_gcnt, when the call ran it; d_gcnt == d_cnt where they are the result), waits, fails on a negative
// matchGrid count, else fills counts (optional) and returns the total.
inline int counts_total(PlContext* ctx, cudaStream_t s, int n, const int32_t* d_cnt, int32_t* counts,
                        const int32_t* d_gcnt = nullptr) {
    std::vector<int32_t> cnt((size_t)n), gcnt(d_gcnt && d_gcnt != d_cnt ? (size_t)n : 0);
    if (!gcnt.empty()) CK(ctx, cudaMemcpyAsync(gcnt.data(), d_gcnt, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaMemcpyAsync(cnt.data(), d_cnt, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CK(ctx, cudaStreamSynchronize(s));
    if (d_gcnt)
        if (const int rc = check_grid_counts(ctx, n, gcnt.empty() ? cnt.data() : gcnt.data())) return rc;
    long total = 0;
    for (int p = 0; p < n; ++p) {
        if (counts) counts[p] = cnt[p];
        total += cnt[p];
    }
    return (int)total;
}

// The next of the two slots of the async entry points (plstvo_wait's tickets) and its completion event.  A caller that
// skipped plstvo_wait on the batch that used the slot last gets that batch finished first.
inline int acquire_slot(PlContext* ctx) {
    const int slot = ctx->next_slot;
    ctx->next_slot ^= 1;
    if (ctx->slot_busy[slot]) {
        CK(ctx, cudaEventSynchronize(ctx->slot_done[slot]));
        ctx->slot_busy[slot] = false;
    }
    if (!ctx->slot_done[slot]) CK(ctx, cudaEventCreateWithFlags(&ctx->slot_done[slot], cudaEventDisableTiming));
    return slot;
}

// ---- matchGrid (match_grid.cu) on arena scratch ----
constexpr int GRID_CAP = 128;   // candidates per query window (the reference has no limit; typical: ~10)

inline bool grid_ok(int rows, int cols) { return rows > 0 && cols > 0 && rows * cols <= 8192; }

inline size_t grid_cells_per_train(bool lines, int rows, int cols) { return lines ? (size_t)std::max(rows, cols) + 2 : 1; }

// matchGrid's scratch, carved from an arena, for frames of points and / or lines with at most maxN1 query and maxN2 train
// rows in all (max_items: train rows times grid_cells_per_train of their kind); fill() writes the GridProblem table of B
// frames of one kind onto it.
struct GridScratch {
    const Arena& a;
    int rows, cols;
    size_t qcell, tcell, tline, tdir, items, qpairs, qcount, tcount, tstart, tslots, seen, m21;
    GridScratch(Arena& ar, int rows_, int cols_, int B, size_t maxN1, size_t maxN2, size_t max_items, bool points, bool lines)
        : a(ar), rows(rows_), cols(cols_) {
        qcell = ar.take(maxN1 * (lines ? 16 : 8));
        tcell = ar.take(points ? maxN2 * 8 : 0);
        tline = ar.take(lines ? maxN2 * 32 : 0);
        tdir = ar.take(lines ? maxN2 * 16 : 0);
        items = ar.take(max_items * 4);
        qpairs = ar.take(maxN1 * GRID_CAP * 8);
        qcount = ar.take(maxN1 * 4);
        tcount = ar.take(maxN2 * 4);
        tstart = ar.take((maxN2 + B) * 4);
        tslots = ar.take(maxN1 * GRID_CAP * 4);
        seen = ar.take(maxN1 * GRID_CAP);
        m21 = ar.take(maxN2 * 4);
    }
    // frame p: queries q_off[p] .. of d1 (device, 32-byte rows) and m12, trains t_off[p] .. of d2, its count at count[p]
    void fill(GridProblem* probs, int B, bool lines, const int32_t* q_off, const int32_t* t_off, const uint8_t* d1,
              const uint8_t* d2, int32_t* m12, int32_t* count) const {
        const size_t cells = grid_cells_per_train(lines, rows, cols);
        for (int p = 0; p < B; ++p) {
            GridProblem& g = probs[p];
            const size_t qa = q_off[p], tb = t_off[p];
            g.n1 = q_off[p + 1] - q_off[p];
            g.n2 = t_off[p + 1] - t_off[p];
            g.q_cell = a.i32(qcell) + qa * (lines ? 4 : 2);
            g.d1 = d1 + qa * 32;
            g.t_cell = lines ? nullptr : a.i32(tcell) + tb * 2;
            g.t_line = lines ? a.f64(tline) + tb * 4 : nullptr;
            g.t_dir = lines ? a.f64(tdir) + tb * 2 : nullptr;
            g.d2 = d2 + tb * 32;
            g.m12 = m12 + qa;
            g.count = count + p;
            g.grid_items = a.i32(items) + tb * cells;
            g.q_pairs = a.at<int2>(qpairs) + qa * GRID_CAP;
            g.q_count = a.i32(qcount) + qa;
            g.t_count = a.i32(tcount) + tb;
            g.t_start = a.i32(tstart) + tb + p;
            g.t_slots = a.i32(tslots) + qa * GRID_CAP;
            g.seen = a.u8(seen) + qa * GRID_CAP;
            g.m21 = a.i32(m21) + tb;
        }
    }
};

// ---- capi.cu: the tracker's plan and launches, composed by the stereo paths ----
int ws_prepare(PlContext* ctx, Workspace& ws, const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
               const PlFrameBatch* curr, bool with_features, bool has_priors, const PlCamera* d_cams = nullptr);
int ws_launch_match(PlContext* ctx, Workspace& ws, int p0, int p1, cudaStream_t s, cudaEvent_t* marks = nullptr);
int ws_launch_solve(PlContext* ctx, Workspace& ws, int p0, int p1, bool have_level, cudaStream_t s,
                    cudaEvent_t* marks = nullptr);

// ---- the lifted records (records.h) on an arena ----
// Slices of `rows` rows for the record arrays [first, last), taken in table order; off[k] receives array k's offset.
inline void take_records(Arena& a, size_t rows, int first, int last, size_t* off) {
    for (int k = first; k < last; ++k) off[k] = a.take(rows * (size_t)REC_BYTES[k]);
}
// the allocated arena's slices off[first .. last)
inline RecPtrs arena_records(const Arena& a, const size_t* off, int first, int last) {
    RecPtrs r;
    for (int k = first; k < last; ++k) r.p[k] = a.u8(off[k]);
    return r;
}
// downloads `rows` rows of each array [first, last) into dst's non-null entries
inline cudaError_t down_records(const Arena& a, const RecPtrs& dst, const size_t* off, size_t rows, int first, int last,
                                cudaStream_t s) {
    for (int k = first; k < last; ++k)
        if (const cudaError_t e = a.down(dst.p[k], off[k], rows * (size_t)REC_BYTES[k], s)) return e;
    return cudaSuccess;
}

// ---- session.cu: the previous-frame-role records of kept frames (plstvo_stereo_session_*) ----
// One session pool: the kept frames of every stream in the previous-frame role (the PREV_ROLE entries of rows), point rows
// and line rows in stream-id order.
struct SessionPool {
    DevBuf buf;
    size_t cap_pt = 0, cap_ls = 0;   // rows
    RecPtrs rows;
    cudaError_t ensure(size_t n_pt, size_t n_ls);
};
// A block of consecutive rows moved by session_gather_kernel: point rows [src_pt, src_pt + n_pt) of the source to dst_pt ..
// of the destination, and the same for lines.
struct GatherSeg {
    int32_t src_pt, dst_pt, n_pt, src_ls, dst_ls, n_ls;
};
// One block per segment, copying the rows of the PREV_ROLE arrays (prev_role) or of every lifted array (else), unchanged.
// gate (optional, [n_segs]): segment k is copied only where gate[k].new_kf is set.
cudaError_t launch_session_gather(const RecPtrs& src, const RecPtrs& dst, bool prev_role, const GatherSeg* segs, int n_segs,
                                  cudaStream_t s, const PlKeyframeResult* gate = nullptr);

// The records a session call retains for plstvo_stereo_session_read (plstvo_stereo_session_retain): the new frames' full
// point and line records and the insert's m12 / inlier rows, every array of records.h, rows in call order.  lay_out() sizes
// the arena for one call; valid is set only when that call succeeded.
struct SessionRetained {
    DevBuf buf;
    RecPtrs rec;               // where each array starts
    size_t rows[N_REC] = {};   // of every array: the new frames' points / lines, the kept frames' points / lines
    bool valid = false, track = false;
    int n = 0;
    cudaError_t lay_out(size_t new_pt, size_t new_ls, size_t kept_pt, size_t kept_ls);
};

}  // namespace plstvo

// n_streams independent stereo streams, each with the previous-frame-role records of its kept frame in HBM
// (plstvo_stereo_session_create).  pool[cur] holds the kept frames; a call writes pool[cur ^ 1] and flips cur when it succeeds.
struct PlStereoSession {
    PlContext* ctx = nullptr;
    PlCamera cam{};
    PlConfig cfg{};
    PlStereoMatchConfig mc{};
    PlStereoConfig sc{};
    PlOrbDetectConfig oc{};
    PlLsdConfig lc{};
    bool has_lc = false;
    bool fld = false;                       // plstvo_stereo_session_use_fld_lines: the caller's key lines, no LSD
    const PlRectifier* rect = nullptr;
    // plstvo_stereo_session_create_cams: stream i's camera and rectifier (empty: cam and rect for every stream)
    std::vector<PlCamera> cams;
    std::vector<const PlRectifier*> rects;
    plstvo::DevBuf d_cams;                  // this call's camera of each new frame, call order (cams sessions)
    int n_streams = 0;
    std::vector<uint8_t> live;              // [S] the stream has a kept frame
    std::vector<int32_t> n_pt, n_ls;        // [S] its stereo points / lines
    std::vector<int32_t> off_pt, off_ls;    // [S] its first rows in pool[cur]
    plstvo::SessionPool pool[2];
    int cur = 0;
    plstvo::DevBuf d_meta;                  // a call's lift output offsets and gather segments
    // ---- plstvo_stereo_session_retain / _read ----
    bool retain = false;
    plstvo::SessionRetained kept;                    // the last call's records while retain is on
    // ---- plstvo_stereo_session_plot / _read_plot: the last initialize / insert's plotStereoFrame images, [kept.n][H][W][3]
    // (plot_valid: that call succeeded and drew them) ----
    bool plot = false, plot_valid = false;
    plstvo::DevBuf plot_buf;
    // ---- plstvo_stereo_session_run_keyframes / _read_keyframes: per step, every named stream's new rows (the key frames'
    // filled), and the key frames' rows [n_kf][4] (step, stream id, points, lines) with their chunk offsets [n_kf][2] ----
    std::vector<std::unique_ptr<plstvo::SessionRetained>> kf_steps;
    std::vector<int32_t> kf_rows, kf_off;
    bool kf_valid = false;
};

namespace plstvo {

// One call on a session, or one step of a session run, on the entry point's stack: the streams it names, and the plan
// session_plan makes for them, committed to the session by session_commit.
struct SessionCall {
    PlStereoSession* ss = nullptr;
    bool track = false;                     // insert (true) or initialize
    bool retain = false;                    // the call fills the session's retention arena
    int n = 0;
    const int32_t* ids = nullptr;           // the caller's array
    std::vector<int32_t> kept_off_pt, kept_off_ls;   // [n + 1] the named streams' kept frames, compact (insert)
    std::vector<int32_t> next_off_pt, next_off_ls;   // [S] first rows in pool[cur ^ 1]
    std::vector<int32_t> new_pt, new_ls;             // [n] the new frames' stereo points / lines
    std::vector<int32_t> meta;                       // uploaded: out_off_pt [n], out_off_ls [n], GatherSeg named [n], others
    int n_others = 0;
    // plstvo_stereo_session_plot (initialize / insert only, with retain): where the new frames' left images are on the device
    // (the images path fills it before the stereo step)
    bool plot = false;
    const uint8_t* plot_grey = nullptr;   // grey sessions: the grey device copy, the n left images first (null: plot_host)
    const uint8_t* plot_host = nullptr;   // grey sessions where no stage put the images on the device: the caller's left images
    const uint8_t* plot_raw = nullptr;    // colour sessions: the rectifier's staging, the n left images first
};

// plot.cu: plotStereoFrame of c's n new frames into the session's plot arena, enqueued on s: the base image (plot_grey /
// plot_host replicated into B, G, R, or the colour staging remapped with each frame's left maps), then the circles of the
// points and the lines of rec's rows, frame k's at pt_off[k] .. pt_off[k + 1] (ls_off for the lines; device copies d_pt_off,
// d_ls_off).  The images are W x H.
int session_plot(PlContext* ctx, const SessionCall& c, int W, int H, const RecPtrs& rec, const std::vector<int32_t>& pt_off,
                 const std::vector<int32_t>& ls_off, const int32_t* d_pt_off, const int32_t* d_ls_off, cudaStream_t s);

// Lays out pool[cur ^ 1] for the new frames' counts (new_pt, new_ls [n], call order) and the untouched streams' kept frames,
// grows it if need be, and uploads the call's offsets and gather segments on s.  PLSTVO_E_TOO_LARGE: more than INT_MAX rows.
int session_plan(PlContext* ctx, SessionCall& c, const int32_t* new_pt, const int32_t* new_ls, cudaStream_t s);
// The two moves of a planned call, enqueued on s: the named streams' kept frames from pool[cur] into the workspace's
// previous-frame arrays at kept_off_pt / kept_off_ls (insert), and the untouched streams' kept frames from pool[cur] into
// pool[cur ^ 1].  The new frames' previous-frame role goes into pool[cur ^ 1] through the lift kernels, at session_out_off.
int session_gather_named(PlContext* ctx, const SessionCall& c, const RecPtrs& ws_rows, cudaStream_t s);
int session_gather_others(PlContext* ctx, const SessionCall& c, cudaStream_t s);
// device offsets [n] of the new frames' first point / line rows in pool[cur ^ 1]
const int32_t* session_out_off(const SessionCall& c, bool lines);
// the call succeeded: pool[cur ^ 1] becomes the kept frames
void session_commit(const SessionCall& c);
// updateFrame's threshold and the next prior of one session-run step, on s for n streams: from the step's results (ws's
// d_results), th [2 n] (row t of the run's threshold table) -> th + 2 n (row t + 1, both halves), priors [n] (ws's d_priors),
// and the results copied to res_out [n]
cudaError_t launch_session_handler(const PlHandlerConfig& h, int n, const PlPoseResult* results, const int32_t* th,
                                   int32_t* th_next, PlPrior* priors, PlPoseResult* res_out, cudaStream_t s);
// keyframe.cu: needNewKF / currFrameIsKF of one session-run step on s for n streams: from the step's results (ws's
// d_results) and state [n] (updated in place) -> out [n]; where it fires, priors [n] (ws's d_priors, after the handler
// update) take Tfw = I, Tfw_cov = I.  k_entropy = 3 (1 + log 2 pi), as the host computes it.
cudaError_t launch_session_keyframe(const PlKeyframeConfig& cfg, double k_entropy, int n, const PlPoseResult* results,
                                    PlKeyframeState* state, PlKeyframeResult* out, PlPrior* priors, cudaStream_t s);
// KeyframeTest::needNewKF's constant 3 (1 + log 2 pi) (src/stereoFrameHandler.cpp:1144, :1165), as the host computes it: the
// one value every launch_session_keyframe caller passes
inline double keyframe_k_entropy() { return 3.0 * (1.0 + std::log(2.0 * std::acos(-1.0))); }
// plstvo_stereo_session_run_schedule: one entry of a step's initialize or insert group, the call position of its stream
// (its state slot) and, for an initialize, the threshold its frame is detected with
struct SchedEntry {
    int32_t slot, th;
};
// The slots' gather before an insert group's ORB, on s for its n entries: thresholds into th [2 n] (both halves), priors [n]
// (ws's d_priors) and, kfs_slot non-null, the key-frame states into kfs [n]
cudaError_t launch_session_schedule_gather(int n, const SchedEntry* e, const int32_t* th_slot, const PlPrior* prior_slot,
                                           const PlKeyframeState* kfs_slot, int32_t* th, PlPrior* priors, PlKeyframeState* kfs,
                                           cudaStream_t s);
// The slots' update after a group, on s: an insert group's th_next [2 n] (left half read), priors [n] and kfs [n] (kfs_slot
// non-null) into its entries' slots, or (init) the slots reset to what initialize leaves
cudaError_t launch_session_schedule_update(int n, const SchedEntry* e, bool init, const int32_t* th_next, const PlPrior* priors,
                                           const PlKeyframeState* kfs, int32_t* th_slot, PlPrior* prior_slot,
                                           PlKeyframeState* kfs_slot, cudaStream_t s);

// ---- capi_stereo.cu: the stereo step's feature sets, and raw stereo features -> pose, composed by the images path ----
// One feature set: one kind of feature (points or lines) of nf frames.  Offsets and left line angles are host arrays; xy_l,
// xy_r (key points or segments), oct and d1, d2 (descriptors) are host arrays, or with on_device HBM (the images path: ORB's
// and LBD's outputs), where a null oct is octave 0 everywhere.  Stand-alone lifting (lift_only) reads the caller's m12 (host)
// in place of matchGrid's and has no d2.  check() sets N1, N2; take() lays out the set's slices, which the other members read.
struct StereoSet {
    bool lines = false;
    int nf = 0;
    const int32_t *l_off = nullptr, *r_off = nullptr;
    const float* ang = nullptr;
    bool on_device = false;
    const float *xy_l = nullptr, *xy_r = nullptr;
    const int32_t* oct = nullptr;
    const uint8_t *d1 = nullptr, *d2 = nullptr;
    bool lift_only = false;
    const int32_t* m12 = nullptr;
    size_t N1 = 0, N2 = 0;
    size_t o_loff = 0, o_roff = 0, o_xyl = 0, o_xyr = 0, o_ang = 0, o_oct = 0, o_d1 = 0, o_d2 = 0, o_m12 = 0, o_cnt = 0,
           o_gcnt = 0, o_prob = 0;

    // the offsets and the arrays a non-empty side needs
    int check(PlContext* ctx);
    // offsets, host-resident inputs (and zero octaves), m12, lifting's counts and, unless lift_only, matchGrid's counts and
    // problem table
    void take(Arena& a);
    // the host arrays on s, then (g given) the set's GridProblem table, filled at probs, for matchGrid's scratch g
    cudaError_t upload(const Arena& a, cudaStream_t s, const GridScratch* g = nullptr, GridProblem* probs = nullptr) const;
    // grid cells of the key points / segments, then matchGrid with the stereo window, on s
    cudaError_t match(const Arena& a, const GridScratch& g, const PlCamera& cam, const PlStereoMatchConfig& mc,
                      cudaStream_t s) const;
    // the lifting of frames [first, first + n) into out's entries of the set's kind (all null: counts only), at out_off
    // (else the left offsets), with the device camera of each frame (cams) or cam
    cudaError_t lift(const Arena& a, const PlCamera& cam, const PlStereoConfig& sc, int n, int first, const RecPtrs& out,
                     cudaStream_t s, const int32_t* out_off = nullptr, const PlCamera* cams = nullptr) const;
    // where the kernels read input p: HBM when it is there, else its slice o
    template <typename T> const T* in(const Arena& a, const T* p, size_t o) const {
        return on_device && p ? p : a.at<const T>(o);
    }
};

// What a tracking call adds to its feature sets.
struct StereoDevInputs {
    cudaEvent_t lines_ready = nullptr;   // waited on before the first line set's stereo step (LBD's stream, on the device)
    cudaEvent_t* marks = nullptr;        // [3] timing events: stereo step start, its end, tracking end (all on s_main)
    bool priors_resident = false;        // the workspace's d_priors already holds this call's priors (a session run's steps)
    // set: called on s_main once the solver is enqueued, in place of the results' download (results are then not written)
    std::function<int(const Workspace&)> tracked;
};
// prev, curr: [2] the point set and the line set of the previous and the current frames (curr unused with sequence or call)
int track_stereo_common(PlContext* ctx, const PlCamera* cam, const PlConfig* cfg, const PlStereoMatchConfig* mc,
                        const PlStereoConfig* sc, const StereoSet* prev, const StereoSet* curr, const PlPrior* priors,
                        PlPoseResult* results, int32_t* n_stereo, bool sequence, int slot, const StereoDevInputs* dev = nullptr,
                        SessionCall* call = nullptr);

// ---- rectify.cu: rectifyImagesLR on the device, composed by the raw-images path ----
struct ImgPart {   // consecutive host images of one size
    const uint8_t* p; int n;
};
// Enqueues on stream s the upload of n_img raw images of rect's size and channels (parts, in order) into arena_rect's staging
// slot and the grey device copy of them into its rectified slot (*d_out): their remap, in blocks of per_block images that
// alternate left, right maps, and for a colour rectifier the conversion to grey after it.  rects (optional, [per_block], of
// rect's size and channels): image z is prepared by rects[z % per_block] instead, a null entry or one without maps copying
// (grey) or converting (colour) the image.  d_rgb (optional, colour rectifiers only): the same launch also writes the
// COLOR_RGB2GRAY conversion of each remapped (or unmapped) image into a second grey slot, *d_rgb.  d_raw (optional): where the
// staged raw images start, in the order of parts.
int rectify_enqueue(PlContext* ctx, const PlRectifier* rect, int n_img, int per_block, const std::vector<ImgPart>& parts,
                    cudaStream_t s, const uint8_t** d_out, const PlRectifier* const* rects = nullptr,
                    const uint8_t** d_rgb = nullptr, const uint8_t** d_raw = nullptr);

}  // namespace plstvo
