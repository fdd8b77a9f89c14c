// session.cu — the device side of plstvo_stereo_session_*: the session's double-buffered pools of kept frames and the gather
// kernel that moves a list of streams' previous-frame-role rows, byte for byte, from one CSR layout into another.
#include <climits>
#include <cstring>

#include "host.cuh"

namespace plstvo {

namespace {

constexpr int GATHER_THREADS = 256;

constexpr bool lifted_rows_are_words() {
    for (int k = 0; k < N_LIFT; ++k)
        if (REC_BYTES[k] % 4) return false;
    return true;
}
static_assert(lifted_rows_are_words(), "the gather copies 4-byte words");

struct GatherArrays {   // arrays 0 .. n_pt - 1 hold point rows, n_pt .. n - 1 line rows
    int n, n_pt;
    const uint32_t* src[N_LIFT];
    uint32_t* dst[N_LIFT];
    int words[N_LIFT];   // 4-byte words per row
};

// One block per segment: every word of the segment's point rows, then of its line rows, is copied unchanged.  Integer
// copies only (no arithmetic on the values), so the kept records are the lift kernels' bytes.
__global__ void __launch_bounds__(GATHER_THREADS) session_gather_kernel(GatherArrays a, const GatherSeg* __restrict__ segs,
                                                                        const PlKeyframeResult* __restrict__ gate) {
    if (gate && !gate[blockIdx.x].new_kf) return;
    const GatherSeg g = segs[blockIdx.x];
#pragma unroll 1
    for (int k = 0; k < a.n; ++k) {
        const bool pt = k < a.n_pt;
        const int n = pt ? g.n_pt : g.n_ls;
        if (n == 0) continue;
        const int w = a.words[k];
        const size_t words = (size_t)n * w;
        const uint32_t* __restrict__ src = a.src[k] + (size_t)(pt ? g.src_pt : g.src_ls) * w;
        uint32_t* __restrict__ dst = a.dst[k] + (size_t)(pt ? g.dst_pt : g.dst_ls) * w;
        for (size_t i = threadIdx.x; i < words; i += GATHER_THREADS) dst[i] = src[i];
    }
}

// updateFrame of one stream after a session-run step (src/stereoFrameHandler.cpp:62-86, :317-326, :377-378), as
// plstvo.hpp's updateFastThreshold, publishPose and priorOf compute it on the host: comparisons and integer arithmetic only.
// th_next is written into both halves of the next row (ORB reads one threshold per image: [left n][right n]).
__global__ void session_handler_kernel(PlHandlerConfig h, int n, const PlPoseResult* __restrict__ results,
                                       const int32_t* __restrict__ th, int32_t* __restrict__ th_next,
                                       PlPrior* __restrict__ priors, PlPoseResult* __restrict__ res_out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const PlPoseResult& r = results[k];
    const int t = th[k];
    int next = t;
    if (h.adaptative_fast) {
        bool identity = true;   // Eigen's operator==: every coefficient compared exactly
        for (int i = 0; i < 16; ++i) identity = identity && r.DT[i] == ((i % 5 == 0) ? 1.0 : 0.0);
        const int inc = h.fast_inc_th, feat = h.fast_feat_th, n_in = r.n_inliers_pt;
        if (identity || r.err_norm > (double)h.fast_err_th || n_in < feat) next = max(h.fast_min_th, t - 2 * inc);
        else if (n_in < feat * 2) next = max(h.fast_min_th, t - inc);
        else if (n_in > feat * 3) next = min(h.fast_max_th, t + inc);
        // the reference's last branch (> 4 feat: + 2 inc, :84-85) is unreachable behind "> 3 feat"
    }
    th_next[k] = next;
    th_next[n + k] = next;
    PlPrior& p = priors[k];
    for (int i = 0; i < 16; ++i) {
        p.Tfw[i] = r.Tfw[i];
        p.DT[i] = r.DT[i];
    }
    for (int i = 0; i < 36; ++i) {
        p.Tfw_cov[i] = r.Tfw_cov[i];
        p.DT_cov[i] = r.DT_cov[i];
    }
    p.err_norm = r.err_norm;
    res_out[k] = r;
}

// A scheduled run's state gather: entry k of a step's insert group reads its stream's slot, the threshold into both halves
// of ORB's row th [2 n], the prior into the workspace's priors and the key-frame state (kfs non-null) into the step's table.
// Moves only: the slots hold exactly what session_handler_kernel and session_keyframe_kernel wrote.
__global__ void session_schedule_gather_kernel(int n, const SchedEntry* __restrict__ e, const int32_t* __restrict__ th_slot,
                                               const PlPrior* __restrict__ prior_slot,
                                               const PlKeyframeState* __restrict__ kfs_slot, int32_t* __restrict__ th,
                                               PlPrior* __restrict__ priors, PlKeyframeState* __restrict__ kfs) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int s = e[k].slot;
    th[k] = th[n + k] = th_slot[s];
    priors[k] = prior_slot[s];
    if (kfs) kfs[k] = kfs_slot[s];
}

// A scheduled run's state update after a step's group: an insert group writes each entry's next threshold (th_next, row
// layout of session_handler_kernel), prior and key-frame state back into its stream's slot; an initialize group (init)
// resets the slot to what HandlerState::initialize leaves: the entry's threshold, priorOf of a fresh frame (Tfw = I,
// Tfw_cov = I, DT = I, DT_cov = 0, err_norm = -1) and plstvo_initial_keyframe_state.  Slots no entry names stay as they are.
__global__ void session_schedule_update_kernel(int n, const SchedEntry* __restrict__ e, bool init,
                                               const int32_t* __restrict__ th_next, const PlPrior* __restrict__ priors,
                                               const PlKeyframeState* __restrict__ kfs, int32_t* __restrict__ th_slot,
                                               PlPrior* __restrict__ prior_slot, PlKeyframeState* __restrict__ kfs_slot) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int s = e[k].slot;
    if (!init) {
        th_slot[s] = th_next[k];
        prior_slot[s] = priors[k];
        if (kfs_slot) kfs_slot[s] = kfs[k];
        return;
    }
    th_slot[s] = e[k].th;
    PlPrior& p = prior_slot[s];
    for (int i = 0; i < 16; ++i) p.Tfw[i] = p.DT[i] = (i % 5 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 36; ++i) {
        p.Tfw_cov[i] = (i % 7 == 0) ? 1.0 : 0.0;
        p.DT_cov[i] = 0.0;
    }
    p.err_norm = -1.0;
    if (!kfs_slot) return;
    PlKeyframeState& q = kfs_slot[s];
    q.prev_f_iskf = 1;
    q.N_prevKF_currF = 0;
    q.entropy_first_prevKF = 0.0;
    for (int i = 0; i < 16; ++i) q.T_prevKF[i] = (i % 5 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 36; ++i) q.cov_prevKF_currF[i] = 0.0;
}

// offsets into SessionCall::meta
size_t meta_named(const SessionCall& c) { return 2 * (size_t)c.n; }
size_t meta_others(const SessionCall& c) { return meta_named(c) + (size_t)c.n * (sizeof(GatherSeg) / 4); }

}  // namespace

cudaError_t launch_session_gather(const RecPtrs& src, const RecPtrs& dst, bool prev_role, const GatherSeg* segs, int n_segs,
                                  cudaStream_t s, const PlKeyframeResult* gate) {
    if (n_segs <= 0) return cudaSuccess;
    GatherArrays a;
    a.n = prev_role ? N_PREV : N_LIFT;
    a.n_pt = 0;
    for (int j = 0; j < a.n; ++j) {
        const int k = prev_role ? PREV_ROLE[j] : j;
        a.n_pt += rec_is_point(k);
        a.src[j] = src.at<const uint32_t>(k);
        a.dst[j] = dst.at<uint32_t>(k);
        a.words[j] = REC_BYTES[k] / 4;
    }
    session_gather_kernel<<<n_segs, GATHER_THREADS, 0, s>>>(a, segs, gate);
    return cudaGetLastError();
}

cudaError_t launch_session_handler(const PlHandlerConfig& h, int n, const PlPoseResult* results, const int32_t* th,
                                   int32_t* th_next, PlPrior* priors, PlPoseResult* res_out, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    session_handler_kernel<<<(n + 127) / 128, 128, 0, s>>>(h, n, results, th, th_next, priors, res_out);
    return cudaGetLastError();
}

cudaError_t launch_session_schedule_gather(int n, const SchedEntry* e, const int32_t* th_slot, const PlPrior* prior_slot,
                                           const PlKeyframeState* kfs_slot, int32_t* th, PlPrior* priors, PlKeyframeState* kfs,
                                           cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    session_schedule_gather_kernel<<<(n + 127) / 128, 128, 0, s>>>(n, e, th_slot, prior_slot, kfs_slot, th, priors, kfs);
    return cudaGetLastError();
}

cudaError_t launch_session_schedule_update(int n, const SchedEntry* e, bool init, const int32_t* th_next, const PlPrior* priors,
                                           const PlKeyframeState* kfs, int32_t* th_slot, PlPrior* prior_slot,
                                           PlKeyframeState* kfs_slot, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    session_schedule_update_kernel<<<(n + 127) / 128, 128, 0, s>>>(n, e, init, th_next, priors, kfs, th_slot, prior_slot,
                                                                     kfs_slot);
    return cudaGetLastError();
}

cudaError_t SessionPool::ensure(size_t n_pt, size_t n_ls) {
    if (buf.p && n_pt <= cap_pt && n_ls <= cap_ls) return cudaSuccess;
    const size_t want_pt = std::max(n_pt + n_pt / 4, cap_pt) + 64, want_ls = std::max(n_ls + n_ls / 4, cap_ls) + 64;
    Arena a;
    size_t off[N_REC];
    for (int k : PREV_ROLE) off[k] = a.take((rec_is_point(k) ? want_pt : want_ls) * (size_t)REC_BYTES[k]);
    cap_pt = cap_ls = 0;
    rows = RecPtrs{};
    if (const cudaError_t e = a.alloc(buf)) return e;
    for (int k : PREV_ROLE) rows.p[k] = a.u8(off[k]);
    cap_pt = want_pt;
    cap_ls = want_ls;
    return cudaSuccess;
}

cudaError_t SessionRetained::lay_out(size_t new_pt, size_t new_ls, size_t kept_pt, size_t kept_ls) {
    Arena a;
    size_t off[N_REC];
    for (int k = 0; k < N_REC; ++k) {
        rows[k] = k < LS_SPL ? new_pt : k < M12_PT ? new_ls : (k == M12_PT || k == INL_PT) ? kept_pt : kept_ls;
        off[k] = a.take(rows[k] * (size_t)REC_BYTES[k]);
    }
    const cudaError_t e = a.alloc(buf);
    rec = arena_records(a, off, 0, N_REC);
    return e;
}

int session_plan(PlContext* ctx, SessionCall& c, const int32_t* new_pt, const int32_t* new_ls, cudaStream_t s) {
    PlStereoSession* ss = c.ss;
    const int S = ss->n_streams, n = c.n;
    std::vector<int> slot((size_t)S, -1);   // call position of each named stream
    for (int k = 0; k < n; ++k) slot[(size_t)c.ids[k]] = k;
    c.new_pt.assign(new_pt, new_pt + n);
    c.new_ls.assign(new_ls, new_ls + n);
    c.next_off_pt.assign((size_t)S, 0);
    c.next_off_ls.assign((size_t)S, 0);
    std::vector<GatherSeg> others;
    long long tp = 0, tl = 0;
    for (int id = 0; id < S; ++id) {
        const int k = slot[(size_t)id];
        const int np = k >= 0 ? new_pt[k] : ss->live[(size_t)id] ? ss->n_pt[(size_t)id] : 0;
        const int nl = k >= 0 ? new_ls[k] : ss->live[(size_t)id] ? ss->n_ls[(size_t)id] : 0;
        c.next_off_pt[(size_t)id] = (int32_t)tp;
        c.next_off_ls[(size_t)id] = (int32_t)tl;
        if (k < 0 && (np || nl))
            others.push_back(GatherSeg{ss->off_pt[(size_t)id], (int32_t)tp, np, ss->off_ls[(size_t)id], (int32_t)tl, nl});
        tp += np;
        tl += nl;
        if (tp > INT_MAX || tl > INT_MAX) return fail(ctx, PLSTVO_E_TOO_LARGE, "more than INT_MAX kept rows in one session");
    }
    CK(ctx, ss->pool[ss->cur ^ 1].ensure((size_t)tp, (size_t)tl));
    // meta: out_off_pt [n], out_off_ls [n], the named streams' segments (kept frame -> the workspace, compact), the others'
    std::vector<int32_t>& m = c.meta;
    m.assign(meta_others(c), 0);
    for (int k = 0; k < n; ++k) {
        const int id = c.ids[k];
        m[(size_t)k] = c.next_off_pt[(size_t)id];
        m[(size_t)n + k] = c.next_off_ls[(size_t)id];
        if (c.track) {
            const GatherSeg g{ss->off_pt[(size_t)id], c.kept_off_pt[(size_t)k], ss->n_pt[(size_t)id],
                              ss->off_ls[(size_t)id], c.kept_off_ls[(size_t)k], ss->n_ls[(size_t)id]};
            memcpy(m.data() + meta_named(c) + (size_t)k * (sizeof(GatherSeg) / 4), &g, sizeof g);
        }
    }
    c.n_others = (int)others.size();
    const size_t o = m.size();
    m.resize(o + others.size() * (sizeof(GatherSeg) / 4));
    if (!others.empty()) memcpy(m.data() + o, others.data(), others.size() * sizeof(GatherSeg));
    CK(ctx, ss->d_meta.ensure(m.size() * 4));
    CK(ctx, cudaMemcpyAsync(ss->d_meta.p, m.data(), m.size() * 4, cudaMemcpyHostToDevice, s));
    return 0;
}

int session_gather_named(PlContext* ctx, const SessionCall& c, const RecPtrs& ws_rows, cudaStream_t s) {
    const PlStereoSession* ss = c.ss;
    const GatherSeg* segs = reinterpret_cast<const GatherSeg*>(ss->d_meta.as<int32_t>() + meta_named(c));
    CK(ctx, launch_session_gather(ss->pool[ss->cur].rows, ws_rows, true, segs, c.n, s));
    ctx->launches++;
    return 0;
}

int session_gather_others(PlContext* ctx, const SessionCall& c, cudaStream_t s) {
    if (!c.n_others) return 0;
    const PlStereoSession* ss = c.ss;
    const GatherSeg* segs = reinterpret_cast<const GatherSeg*>(ss->d_meta.as<int32_t>() + meta_others(c));
    CK(ctx, launch_session_gather(ss->pool[ss->cur].rows, ss->pool[ss->cur ^ 1].rows, true, segs, c.n_others, s));
    ctx->launches++;
    return 0;
}

const int32_t* session_out_off(const SessionCall& c, bool lines) {
    return c.ss->d_meta.as<int32_t>() + (lines ? c.n : 0);
}

void session_commit(const SessionCall& c) {
    PlStereoSession* ss = c.ss;
    for (int k = 0; k < c.n; ++k) {
        const size_t id = (size_t)c.ids[k];
        ss->live[id] = 1;
        ss->n_pt[id] = c.new_pt[(size_t)k];
        ss->n_ls[id] = c.new_ls[(size_t)k];
    }
    ss->off_pt = c.next_off_pt;
    ss->off_ls = c.next_off_ls;
    ss->cur ^= 1;
}

}  // namespace plstvo
