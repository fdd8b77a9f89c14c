// match_grid.cu — StVO::matchGrid, points and lines (src/matching.cpp:111-177, :179-258): the stereo (left/right)
// matching step one row upstream of the hot path (SURVEY 8(f)-1).  Same 256-bit Hamming primitive, candidates
// restricted to a window of the 64 x 48 bucket grid.
//
// The reference is sequential in the query index because of the bestLRMatches gate (:145-150): a train is considered by
// query i1 only if its distance beats the train's running minimum over all EARLIER queries.  That is a strict
// prefix-minimum per train over ascending query index, so it parallelises as
//   A. one thread per query: enumerate the window's candidates from the train grid (de-duplicated, direction-filtered for
//      lines), compute distances, emit (i2, d) pairs;
//   B. counting sort of the pairs by train;
//   C. one thread per train: a pair is "seen" iff no pair of the same train with a smaller query index has a distance
//      <= its own; the last record-setter is matches_21[i2];
//   D. one thread per query: best / second best over its seen pairs (with multiplicity), ratio test in double, then the
//      mutual filter (:166-174).
// One CTA per frame; a batch of frames runs in parallel.  Integer work and a handful of doubles only.
#include "common.cuh"

namespace plstvo {

namespace {

constexpr int MG_CAP = 128;        // candidates per query window on the fast path (pair keys pack query:16 | slot:7 | distance:9);
                                   // a frame with a fuller window falls back to mg_sequential (no limit)
constexpr int MG_THREADS = 512;    // one CTA per frame: the work is a few thousand short dependent chains, so width buys latency

__device__ __forceinline__ int mg_distance(const uint8_t* a, const uint8_t* b) {   // StVO::distance (:93-109)
    const uint4* pa = reinterpret_cast<const uint4*>(a);
    const uint4* pb = reinterpret_cast<const uint4*>(b);
    const uint4 a0 = __ldg(pa), a1 = __ldg(pa + 1), b0 = __ldg(pb), b1 = __ldg(pb + 1);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// LineIterator (src/lineIterator.cpp:34-77): calls f(x, y) for every visited cell
template <typename F>
__device__ __forceinline__ void mg_line_cells(double x1, double y1, double x2, double y2, F f) {
    const bool steep = fabs(y2 - y1) > fabs(x2 - x1);
    if (steep) { double t = x1; x1 = y1; y1 = t; t = x2; x2 = y2; y2 = t; }
    if (x1 > x2) { double t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    const double dx = x2 - x1, dy = fabs(y2 - y1);
    double error = dx / 2.0;
    const int ystep = (y1 < y2) ? 1 : -1;
    int x = (int)x1, y = (int)y1;
    const int maxX = (int)x2;
    for (; !(x > maxX); ++x) {
        if (steep) f(y, x); else f(x, y);
        error -= dy;
        if (error < 0) { y += ystep; error += dx; }
    }
}

__device__ int mg_block_exclusive_scan(int* data, int n, int* s_tmp /* >= MG_THREADS ints */) {
    // in-place exclusive scan of data[0..n) by the whole block; returns the total
    const int tid = threadIdx.x;
    const int per = (n + MG_THREADS - 1) / MG_THREADS, lo = min(n, tid * per), hi = min(n, lo + per);
    int s = 0;
    for (int i = lo; i < hi; i++) s += data[i];
    s_tmp[tid] = s;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int i = 0; i < MG_THREADS; i++) { const int v = s_tmp[i]; s_tmp[i] = run; run += v; }
        s_tmp[MG_THREADS] = run;
    }
    __syncthreads();
    int run = s_tmp[tid];
    for (int i = lo; i < hi; i++) { const int v = data[i]; data[i] = run; run += v; }
    __syncthreads();
    return s_tmp[MG_THREADS];
}


// ---- overflow path: more than MG_CAP candidates in one query window --------------------------------------------------
// The reference has no limit (the candidates are an unordered_set, src/matching.cpp:128-139, :213-224).  A frame that
// overflows the fixed per-query segments of the fast path is re-run here by the reference's own schedule: queries one
// after the other (the gate's running minimum `distances[i2]` is loop-carried, :145-150), the whole CTA sharing the
// candidates of the current query.  Exact, about 3 us per query: the price is paid only by the dense frame.
template <bool LINES>
__device__ void mg_sequential(const GridProblem& pr, const GridParams& prm, const int* cell_start, int* s_tmp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n1 = pr.n1, n2 = pr.n2;
    int* dist = pr.t_start;      // distances[i2] (:124), INT_MAX = none yet
    int* stamp = pr.t_count;     // last query that enumerated train i2: de-duplicates like the unordered_set
    for (int t = tid; t < n2; t += MG_THREADS) { dist[t] = 0x7FFFFFFF; stamp[t] = -1; pr.m21[t] = -1; }
    __syncthreads();
    int matches = 0;             // thread 0 only
    for (int q = 0; q < n1; ++q) {
        const int* qc = pr.q_cell + (size_t)q * (LINES ? 4 : 2);
        double vx = 0.0, vy = 0.0;
        if (LINES) {
            vx = (double)(qc[2] - qc[0]);
            vy = (double)(qc[3] - qc[1]);
            const double mag = sqrt(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));   // unfused, as dot (matching.h:39-41)
            vx /= mag;
            vy /= mag;
        }
        const uint8_t* dq = pr.d1 + (size_t)q * 32;
        int b1 = 0x7FFFFFFF, b2 = 0x7FFFFFFF, bi = -1, any = 0;
        for (int e = 0; e < (LINES ? 2 : 1); ++e) {
            const int x = qc[2 * e], y = qc[2 * e + 1];
            const int min_x = max(0, x - prm.w.left), max_x = min(prm.cols, x + prm.w.right + 1);
            const int min_y = max(0, y - prm.w.up), max_y = min(prm.rows, y + prm.w.down + 1);
            const int wx = max(0, max_x - min_x), wy = max(0, max_y - min_y);
            for (int c = warp; c < wx * wy; c += MG_THREADS / 32) {   // one warp per cell, one lane per item
                const int cell = (min_x + c / wy) * prm.rows + (min_y + c % wy);
                for (int it = cell_start[cell] + lane; it < cell_start[cell + 1]; it += 32) {
                    const int i2 = pr.grid_items[it];
                    if (atomicExch(&stamp[i2], q) == q) continue;   // already in this query's candidate set
                    any = 1;
                    if (LINES) {
                        const double dt = __dadd_rn(__dmul_rn(vx, pr.t_dir[2 * i2]), __dmul_rn(vy, pr.t_dir[2 * i2 + 1]));
                        if (fabs(dt) < prm.line_sim_th) continue;    // NaN passes (:221); unfused, a fused dot flips |dt| ~ th
                    }
                    const int d = mg_distance(dq, pr.d2 + (size_t)i2 * 32);
                    if (prm.best_lr) {          // each train appears once per query: no race on dist[i2]
                        if (d < dist[i2]) { dist[i2] = d; pr.m21[i2] = q; } else continue;
                    }
                    if (d < b1) { b2 = b1; b1 = d; bi = i2; }
                    else if (d < b2) b2 = d;
                }
            }
        }
        // block-wide best / second best with multiplicity; the smallest distance's train (lowest index on a tie)
        for (int o = 16; o; o >>= 1) {
            const int c1 = __shfl_xor_sync(0xFFFFFFFFu, b1, o), c2 = __shfl_xor_sync(0xFFFFFFFFu, b2, o),
                      ci = __shfl_xor_sync(0xFFFFFFFFu, bi, o), ca = __shfl_xor_sync(0xFFFFFFFFu, any, o);
            const int m2 = min(max(b1, c1), min(b2, c2));
            if (c1 < b1 || (c1 == b1 && ci >= 0 && (bi < 0 || ci < bi))) bi = ci;
            b1 = min(b1, c1);
            b2 = m2;
            any |= ca;
        }
        if (lane == 0) { s_tmp[4 * warp] = b1; s_tmp[4 * warp + 1] = b2; s_tmp[4 * warp + 2] = bi; s_tmp[4 * warp + 3] = any; }
        __syncthreads();
        if (tid == 0) {
            b1 = b2 = 0x7FFFFFFF; bi = -1; any = 0;
            for (int w = 0; w < MG_THREADS / 32; ++w) {
                const int c1 = s_tmp[4 * w], c2 = s_tmp[4 * w + 1], ci = s_tmp[4 * w + 2];
                const int m2 = min(max(b1, c1), min(b2, c2));
                if (c1 < b1 || (c1 == b1 && ci >= 0 && (bi < 0 || ci < bi))) bi = ci;
                b1 = min(b1, c1);
                b2 = m2;
                any |= s_tmp[4 * w + 3];
            }
            int i2 = -1;
            if (any && (double)b1 < (double)b2 * prm.ratio) { i2 = bi; matches++; }   // :160-163
            pr.m12[q] = i2;
        }
        __syncthreads();
    }
    // mutual filter (:166-174)
    __shared__ int s_drop;
    if (tid == 0) s_drop = 0;
    __syncthreads();
    if (prm.best_lr) {
        int drop = 0;
        for (int q = tid; q < n1; q += MG_THREADS) {
            const int i2 = pr.m12[q];
            if (i2 >= 0 && pr.m21[i2] != q) { pr.m12[q] = -1; drop++; }
        }
        if (drop) atomicAdd(&s_drop, drop);
    }
    __syncthreads();
    if (tid == 0 && pr.count) *pr.count = matches - s_drop;
}

template <bool LINES>
__global__ void __launch_bounds__(MG_THREADS) match_grid_kernel(const GridProblem* __restrict__ problems, GridParams prm) {
    extern __shared__ __align__(16) int smem_i[];
    int* cell_start = smem_i;                             // [cells + 1] train grid CSR
    int* cell_fill = smem_i + prm.rows * prm.cols + 1;    // [cells] counts, then fill cursors
    int* s_tmp = cell_fill + prm.rows * prm.cols;         // [MG_THREADS + 1]
    __shared__ int s_flag;
    const GridProblem pr = problems[blockIdx.x];
    const int tid = threadIdx.x, ncell = prm.rows * prm.cols, n1 = pr.n1, n2 = pr.n2;
    constexpr int CAP = MG_CAP;
    if (tid == 0) s_flag = 0;
    for (int q = tid; q < n1; q += MG_THREADS) pr.m12[q] = -1;
    if (n1 == 0 || n2 == 0) {
        if (tid == 0 && pr.count) *pr.count = 0;
        return;
    }

    // ---- train grid (stereoFrame.cpp:135-139 / :326-339): count, scan, fill ----
    for (int c = tid; c < ncell; c += MG_THREADS) cell_fill[c] = 0;
    __syncthreads();
    auto in_grid = [&](int x, int y) { return x >= 0 && x < prm.cols && y >= 0 && y < prm.rows; };
    for (int t = tid; t < n2; t += MG_THREADS) {
        if (!LINES) {
            const int x = pr.t_cell[2 * t], y = pr.t_cell[2 * t + 1];
            if (in_grid(x, y)) atomicAdd(&cell_fill[x * prm.rows + y], 1);
        } else {
            const double* L = pr.t_line + 4 * (size_t)t;
            mg_line_cells(L[0], L[1], L[2], L[3], [&](int x, int y) {
                if (in_grid(x, y)) atomicAdd(&cell_fill[x * prm.rows + y], 1);
            });
        }
    }
    __syncthreads();
    for (int c = tid; c < ncell; c += MG_THREADS) cell_start[c] = cell_fill[c];
    __syncthreads();
    const int n_items = mg_block_exclusive_scan(cell_start, ncell, s_tmp);
    if (tid == 0) cell_start[ncell] = n_items;
    for (int c = tid; c < ncell; c += MG_THREADS) cell_fill[c] = cell_start[c];
    __syncthreads();
    for (int t = tid; t < n2; t += MG_THREADS) {
        if (!LINES) {
            const int x = pr.t_cell[2 * t], y = pr.t_cell[2 * t + 1];
            if (in_grid(x, y)) pr.grid_items[atomicAdd(&cell_fill[x * prm.rows + y], 1)] = t;
        } else {
            const double* L = pr.t_line + 4 * (size_t)t;
            mg_line_cells(L[0], L[1], L[2], L[3], [&](int x, int y) {
                if (in_grid(x, y)) pr.grid_items[atomicAdd(&cell_fill[x * prm.rows + y], 1)] = t;
            });
        }
        pr.t_count[t] = 0;
    }
    __syncthreads();

    // ---- A. candidates of every query (:128-139 / :201-224) ----
    for (int q = tid; q < n1; q += MG_THREADS) {
        int2* seg = pr.q_pairs + (size_t)q * CAP;
        int k = 0;
        bool overflow = false;
        double vx = 0.0, vy = 0.0;
        const int* qc = pr.q_cell + (size_t)q * (LINES ? 4 : 2);
        if (LINES) {   // v = normalize(ep - sp) in INTEGER cell coordinates (:207-211): NaN when both share a cell
            vx = (double)(qc[2] - qc[0]);
            vy = (double)(qc[3] - qc[1]);
            const double mag = sqrt(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));   // unfused, as dot (matching.h:39-41)
            vx /= mag;
            vy /= mag;
        }
        const uint8_t* dq = pr.d1 + (size_t)q * 32;
        for (int e = 0; e < (LINES ? 2 : 1); ++e) {   // GridStructure::get around sp (and ep)
            const int x = qc[2 * e], y = qc[2 * e + 1];
            const int min_x = max(0, x - prm.w.left), max_x = min(prm.cols, x + prm.w.right + 1);
            const int min_y = max(0, y - prm.w.up), max_y = min(prm.rows, y + prm.w.down + 1);
            for (int x_ = min_x; x_ < max_x; ++x_)
                for (int y_ = min_y; y_ < max_y; ++y_) {
                    const int c = x_ * prm.rows + y_;
                    for (int it = cell_start[c]; it < cell_start[c + 1]; ++it) {
                        const int i2 = pr.grid_items[it];
                        if (LINES) {
                            bool dup = false;      // the reference collects into an unordered_set
                            for (int j = 0; j < k; ++j) dup = dup || (seg[j].x == i2);
                            if (dup) continue;
                        }
                        if (k >= CAP) { overflow = true; continue; }
                        int d = -1;                // -1: in the candidate set but dropped by the direction filter
                        bool pass = true;
                        if (LINES) {
                            const double dt = __dadd_rn(__dmul_rn(vx, pr.t_dir[2 * i2]), __dmul_rn(vy, pr.t_dir[2 * i2 + 1]));
                            if (fabs(dt) < prm.line_sim_th) pass = false;   // NaN passes (:221); unfused (see mg_sequential)
                        }
                        if (pass) d = mg_distance(dq, pr.d2 + (size_t)i2 * 32);
                        seg[k++] = make_int2(i2, d);
                        if (pass) atomicAdd(&pr.t_count[i2], 1);
                    }
                }
        }
        pr.q_count[q] = k;
        if (overflow) s_flag = 1;
    }
    __syncthreads();
    if (s_flag) {   // more than CAP candidates in one window: this frame takes the sequential, unbounded path
        mg_sequential<LINES>(pr, prm, cell_start, s_tmp);
        return;
    }

    // ---- B. counting sort of the pairs by train ----
    for (int t = tid; t < n2; t += MG_THREADS) pr.t_start[t] = pr.t_count[t];
    __syncthreads();
    const int n_pairs = mg_block_exclusive_scan(pr.t_start, n2, s_tmp);
    if (tid == 0) pr.t_start[n2] = n_pairs;
    for (int t = tid; t < n2; t += MG_THREADS) pr.t_count[t] = pr.t_start[t];   // fill cursors
    __syncthreads();
    for (int q = tid; q < n1; q += MG_THREADS) {
        const int2* seg = pr.q_pairs + (size_t)q * CAP;
        const int k = pr.q_count[q];
        for (int j = 0; j < k; ++j)   // key = (query << 16) | (slot << 9) | distance: phase C never goes back to q_pairs
            if (seg[j].y >= 0) pr.t_slots[atomicAdd(&pr.t_count[seg[j].x], 1)] = (int)(((uint32_t)q << 16) | ((uint32_t)j << 9) | (uint32_t)seg[j].y);
    }
    __syncthreads();

    // ---- C. the gate (:145-150): strict prefix minimum over ascending query index, per train ----
    for (int t = tid; t < n2; t += MG_THREADS) {
        const int b = pr.t_start[t], e = pr.t_start[t + 1];
        const uint32_t* keys = reinterpret_cast<const uint32_t*>(pr.t_slots);
        int best_key = 0x7FFFFFFF;   // (d << 16 | i1): minimum distance, lowest query index = the last record setter
        for (int a = b; a < e; ++a) {
            const uint32_t ka = keys[a], i1 = ka >> 16, d = ka & 0x1FFu;
            bool seen = true;
            if (prm.best_lr) {
                for (int o = b; o < e; ++o) {
                    const uint32_t ko = keys[o];
                    if ((ko >> 16) < i1 && (ko & 0x1FFu) <= d) seen = false;
                }
            }
            pr.seen[ka >> 9] = seen ? 1 : 0;            // ka >> 9 = query * CAP + slot
            best_key = min(best_key, (int)((d << 16) | i1));
        }
        pr.m21[t] = (e > b) ? (best_key & 0xFFFF) : -1;
    }
    __syncthreads();

    // ---- D. best / second best, ratio test (:152-163), mutual filter (:166-174) ----
    int local = 0;
    for (int q = tid; q < n1; q += MG_THREADS) {
        const int2* seg = pr.q_pairs + (size_t)q * CAP;
        const int k = pr.q_count[q];
        int best_d = 0x7FFFFFFF, best_d2 = 0x7FFFFFFF, best_idx = -1;
        for (int j = 0; j < k; ++j) {
            const int d = seg[j].y;
            if (d < 0 || !pr.seen[(size_t)q * CAP + j]) continue;
            if (d < best_d) { best_d2 = best_d; best_d = d; best_idx = seg[j].x; }
            else if (d < best_d2) best_d2 = d;
        }
        int i2 = -1;
        if (k > 0 && (double)best_d < (double)best_d2 * prm.ratio) {   // int * double (:160)
            i2 = best_idx;
            local++;                                                   // matches++ (:162), whatever best_idx is
        }
        if (prm.best_lr && i2 >= 0 && pr.m21[i2] != q) {
            i2 = -1;
            local--;
        }
        pr.m12[q] = i2;
    }
    // count
    s_tmp[tid] = local;
    __syncthreads();
    if (tid == 0) {
        int tot = 0;
        for (int i = 0; i < MG_THREADS; i++) tot += s_tmp[i];
        if (pr.count) *pr.count = tot;
    }
}

}  // namespace

size_t match_grid_smem_bytes(int rows, int cols) { return ((size_t)2 * rows * cols + 1 + MG_THREADS + 1) * sizeof(int); }

cudaError_t launch_match_grid(const GridProblem* problems, int B, const GridParams& prm, bool lines, cudaStream_t stream) {
    if (B <= 0) return cudaSuccess;
    if (prm.cap != MG_CAP) return cudaErrorInvalidValue;   // the scratch arrays are laid out for MG_CAP candidates per query
    const size_t smem = match_grid_smem_bytes(prm.rows, prm.cols);
    if (lines) {
        if (smem > 48 * 1024) cudaFuncSetAttribute(match_grid_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        match_grid_kernel<true><<<B, MG_THREADS, smem, stream>>>(problems, prm);
    } else {
        if (smem > 48 * 1024) cudaFuncSetAttribute(match_grid_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        match_grid_kernel<false><<<B, MG_THREADS, smem, stream>>>(problems, prm);
    }
    return cudaGetLastError();
}

}  // namespace plstvo
