// gn_stream.cu — optimizeFunctions (src/stereoFrameHandler.cpp:549-694) evaluated for a batch of problems with the
// matched lists STREAMED from HBM: the HBM-roofline kernel of config C5 (1920x1080, 8000 points + 2000 lines,
// B >= 1024 problems resident so that one sweep is far larger than L2).
//
// Records: the fp32-packed layout SURVEY 8(a) A4/A5 defines — the algorithmic bytes of one evaluation are exactly what
// the kernel reads: 32 B per point, 64 B per line.  Pose-independent per-feature quantities are formed once, in double,
// when the batch is packed (gn_stream.cuh, "records": normalised coordinates, the residual at the identity pose, the overlap
// parameters at the identity pose); (oa, ob, oc): StereoFrame::lineSegmentOverlap's parameter lambda of a projected endpoint is
// affine in the endpoint in all three of its branches (src/stereoFrame.cpp:515-612); the coefficients depend on the
// previous-frame segment only.
// Tiles of 16 KB (512 points or 256 lines) are stored plane by plane ([cnt] x float4 per plane), so that a bulk copy of
// one contiguous range lands in shared memory in a bank-conflict-free order.
//
// Kernel: persistent CTAs, 2 per SM, each 8 consumer warps + 1 producer warp.  The producer's elected lane walks the CTA's
// work items (problem, slice) and keeps a ring of 6 x 16 KB stages filled with the TMA engine (cp.async.bulk + full/empty
// mbarriers): ~190 KB in flight per SM, HBM latency decoupled from warp occupancy, no CTA-wide barrier on the data path.
// Per-feature arithmetic is fp32 with MUFU reciprocals / square roots (the survey's precision probe: pose deviation 3e-8
// rad / 8e-7 m); a thread keeps its features' partial sums in fp32 and a warp folds them with a fixed-order shuffle tree;
// warps, slices and the 10 000 features of a problem are summed in fp64 in a fixed order (deterministic).  The solver proper (solve.cu) stays fp64 end to
// end; this kernel is the streamed evaluator of the roofline run.
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "gn_stream.cuh"

namespace plstvo {

namespace {

__device__ __forceinline__ int gs_find_problem(const int32_t* __restrict__ off, int B, int i) {   // off[p] <= i < off[p+1]
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// device-side packing of the double arrays into the tile-planar fp32 records
__global__ void pack_records_kernel(RowsDev m, PlCamera cam, int B, int n_pt, int n_ls, float4* __restrict__ pt,
                                    float4* __restrict__ ls) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const GsCamD c = {cam.fx, cam.fy, cam.cx, cam.cy};
    if (i < n_pt) {
        const int p = gs_find_problem(m.pt_off, B, i), p0 = m.pt_off[p], np = m.pt_off[p + 1] - p0;
        const int j = i - p0, t = j / GS_PT_TILE, r = j % GS_PT_TILE, cnt = min(GS_PT_TILE, np - t * GS_PT_TILE);
        float4* base = pt + 2 * (size_t)(p0 + t * GS_PT_TILE);
        const size_t a = (size_t)i;
        gs_pack_point(c, m.pt_P[3 * a], m.pt_P[3 * a + 1], m.pt_P[3 * a + 2], m.pt_pl[2 * a], m.pt_pl[2 * a + 1],
                      sqrt(m.pt_sigma2[a]), !(m.pt_inlier && !m.pt_inlier[a]), base[r], base[cnt + r]);
    }
    if (i < n_ls) {
        const int p = gs_find_problem(m.ls_off, B, i), l0 = m.ls_off[p], nl = m.ls_off[p + 1] - l0;
        const int j = i - l0, t = j / GS_LS_TILE, r = j % GS_LS_TILE, cnt = min(GS_LS_TILE, nl - t * GS_LS_TILE);
        float4* base = ls + 4 * (size_t)(l0 + t * GS_LS_TILE);
        const size_t a = (size_t)i;
        const double su = m.ls_spl[2 * a], sv = m.ls_spl[2 * a + 1], eu = m.ls_epl[2 * a], ev = m.ls_epl[2 * a + 1];
        double oa, ob, oc;
        overlap_coeffs(su, sv, eu, ev, oa, ob, oc);
        gs_pack_line(c, m.ls_sP[3 * a], m.ls_sP[3 * a + 1], m.ls_sP[3 * a + 2], m.ls_eP[3 * a], m.ls_eP[3 * a + 1], m.ls_eP[3 * a + 2],
                     m.ls_le[3 * a], m.ls_le[3 * a + 1], m.ls_le[3 * a + 2], oa, ob, oc, sqrt(m.ls_sigma2[a]),
                     !(m.ls_inlier && !m.ls_inlier[a]), base[r], base[cnt + r], base[2 * cnt + r], base[3 * cnt + r]);
    }
}

// the tiles of work item `item` = slice `item % bpp` of problem `item / bpp`: whole tiles, points first, then lines
struct GsItem {
    int p0, np, l0, nl, pt_lo, n_ptile, lt_lo, n_tiles;
};
struct GsLists {
    const int32_t* pt_off; const int32_t* ls_off;
};
__device__ __forceinline__ GsItem gs_item(const GsLists& L, int item, int bpp) {
    GsItem it;
    const int prob = item / bpp, blk = item % bpp;
    it.p0 = L.pt_off[prob]; it.np = L.pt_off[prob + 1] - it.p0;
    it.l0 = L.ls_off[prob]; it.nl = L.ls_off[prob + 1] - it.l0;
    const int ptiles = (it.np + GS_PT_TILE - 1) / GS_PT_TILE, ltiles = (it.nl + GS_LS_TILE - 1) / GS_LS_TILE;
    const int pt_per = (ptiles + bpp - 1) / bpp, lt_per = (ltiles + bpp - 1) / bpp;
    it.pt_lo = min(ptiles, blk * pt_per);
    it.lt_lo = min(ltiles, blk * lt_per);
    it.n_ptile = min(ptiles, it.pt_lo + pt_per) - it.pt_lo;
    it.n_tiles = it.n_ptile + min(ltiles, it.lt_lo + lt_per) - it.lt_lo;
    return it;
}

template <class Acc>
__global__ void __launch_bounds__(GS_THREADS, 2)
gn_eval_stream_kernel(PlCamera cam, float homog_th, const GsLists L,
                      const float4* __restrict__ pt, const float4* __restrict__ ls, const double* __restrict__ DTs,
                      double* __restrict__ partial, int bpp, int n_items) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ float sDT[GS_STAGES][12];     // pose of the item whose first tile sits in the stage (written by the producer)
    __shared__ __align__(8) uint64_t full[GS_STAGES], empty[GS_STAGES];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < GS_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], GS_CWARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == GS_CWARPS) {   // ---- producer warp: one elected lane keeps the ring full ----
        if (lane == 0) {
            uint32_t k = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const GsItem it = gs_item(L, item, bpp);
                for (int t = 0; t < it.n_tiles; ++t, ++k) {
                    const uint32_t st = k % GS_STAGES;
                    if (k >= GS_STAGES) mbar_wait(&empty[st], ((k / GS_STAGES) - 1) & 1);
                    if (t == 0) {   // the item's pose rides with its first tile (ordered by the barrier's release / acquire)
                        const double* DT = DTs + (size_t)(item / bpp) * 16;
#pragma unroll
                        for (int i = 0; i < 12; i++) sDT[st][i] = gs_pose_entry(__ldg(DT + i), i);
                    }
                    const void* src;
                    uint32_t bytes;
                    if (t < it.n_ptile) {
                        const int f0 = (it.pt_lo + t) * GS_PT_TILE;
                        src = pt + 2 * (size_t)(it.p0 + f0);
                        bytes = (uint32_t)min(GS_PT_TILE, it.np - f0) * 32u;
                    } else {
                        const int f0 = (it.lt_lo + (t - it.n_ptile)) * GS_LS_TILE;
                        src = ls + 4 * (size_t)(it.l0 + f0);
                        bytes = (uint32_t)min(GS_LS_TILE, it.nl - f0) * 64u;
                    }
                    mbar_arrive_expect_tx(&full[st], bytes);
                    bulk_g2s(smem + (size_t)st * GS_STAGE_BYTES, src, bytes, &full[st]);
                }
            }
        }
        return;
    }

    // ---- consumer warps ----
    GsPose P;
    P.fx = (float)cam.fx; P.fy = (float)cam.fy; P.cx = (float)cam.cx; P.cy = (float)cam.cy;
    P.h = homog_th; P.inv_h = 1.f / homog_th; P.fx_h = P.fx / homog_th;
    uint32_t k = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const GsItem it = gs_item(L, item, bpp);
        if (it.n_tiles > 0) {
            const uint32_t st0 = k % GS_STAGES;
            mbar_wait(&full[st0], (k / GS_STAGES) & 1);
#pragma unroll
            for (int i = 0; i < 12; i++) P.r[i] = sDT[st0][i];
        }
        Acc acc;
        acc.clear();

        for (int t = 0; t < it.n_tiles; ++t, ++k) {
            const uint32_t st = k % GS_STAGES;
            mbar_wait(&full[st], (k / GS_STAGES) & 1);
            const float4* s = reinterpret_cast<const float4*>(smem + (size_t)st * GS_STAGE_BYTES);
            if (t < it.n_ptile) {
                const int cnt = min(GS_PT_TILE, it.np - (it.pt_lo + t) * GS_PT_TILE);
#pragma unroll
                for (int h = 0; h < GS_PT_TILE / GS_CONSUMERS; ++h) {
                    const int idx = tid + h * GS_CONSUMERS;
                    const bool live = idx < cnt;
                    const int ii = live ? idx : 0;
                    const float4 a = s[ii], b = s[cnt + ii];
                    gs_point(P, a, b, live && b.z != 0.f, acc);
                }
            } else {
                const int cnt = min(GS_LS_TILE, it.nl - (it.lt_lo + (t - it.n_ptile)) * GS_LS_TILE);
                const bool live = tid < cnt;
                const int ii = live ? tid : 0;
                const float4 a = s[ii], b = s[cnt + ii], c = s[2 * cnt + ii], d = s[3 * cnt + ii];
                gs_line(P, a, b, c, d, live && b.w != 0.f, acc);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);        // this warp is done with the stage
        }

        // transposed warp reduction (31 shuffles, fixed order): lane L ends with the warp's total of accumulator L (<= 1024
        // features, fp32); everything above a warp — warps, slices, the reduce kernel — is summed in fp64
        float v[32];
        acc.unpack(v);
#pragma unroll
        for (int i = GS_NACC; i < 32; i++) v[i] = 0.f;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < off; i++) {
                const float mine = up ? v[i + off] : v[i];
                const float send = up ? v[i] : v[i + off];
                v[i] = mine + __shfl_xor_sync(0xFFFFFFFFu, send, off);
            }
        }
        if (lane < GS_NACC) partial[((size_t)item * GS_CWARPS + warp) * GS_NACC + lane] = (double)v[0];
    }
}

// Folds the bpp x 8 fp64 partial records of a problem in index order (a per-item fence + counter in the streaming kernel
// costs more than this second launch: measured 82 vs 70 us per sweep).
__global__ void gn_eval_reduce_kernel(const double* __restrict__ partial, int n_part, double* __restrict__ H,
                                      double* __restrict__ g, double* __restrict__ e) {
    const int prob = blockIdx.x, lane = threadIdx.x;
    double sum = 0.0;
    if (lane < GS_NACC)
        for (int b = 0; b < n_part; b++) sum += partial[((size_t)prob * n_part + b) * GS_NACC + lane];
    const double cnt = __shfl_sync(0xFFFFFFFFu, sum, 28);
    if (lane < 21) {            // upper triangle, row-major: lane -> (i, j)
        int i = 0, k = lane;
        while (k >= 6 - i) { k -= 6 - i; i++; }
        const int j = i + k;
        H[(size_t)prob * 36 + i * 6 + j] = sum;
        H[(size_t)prob * 36 + j * 6 + i] = sum;
    } else if (lane < 27) {
        g[(size_t)prob * 6 + (lane - 21)] = sum;
    } else if (lane == 27) {
        e[prob] = sum / cnt;    // :692
    }
}

}  // namespace

int gn_stream_partials_per_slice() { return GS_CWARPS; }
int gn_stream_tiles(int n_pt, int n_ls) {
    return (n_pt + GS_PT_TILE - 1) / GS_PT_TILE + (n_ls + GS_LS_TILE - 1) / GS_LS_TILE;
}

cudaError_t launch_pack_records(const RowsDev& m, const PlCamera& cam, int B, int n_pt, int n_ls, float4* pt, float4* ls,
                                cudaStream_t stream) {
    const int n = n_pt > n_ls ? n_pt : n_ls;
    if (n <= 0 || B <= 0) return cudaSuccess;
    pack_records_kernel<<<(n + 255) / 256, 256, 0, stream>>>(m, cam, B, n_pt, n_ls, pt, ls);
    return cudaGetLastError();
}

cudaError_t launch_gn_eval_stream(const PlCamera& cam, const PlConfig& cfg, const int32_t* pt_off, const int32_t* ls_off,
                                  const float4* pt, const float4* ls, int B, const double* DT, double* partial, int bpp,
                                  int sm_count, double* H, double* g, double* e, cudaStream_t stream) {
    if (B <= 0) return cudaSuccess;
    const size_t smem = (size_t)GS_STAGES * GS_STAGE_BYTES;
    static size_t configured[64] = {};
    cudaError_t err = ensure_dynamic_smem(reinterpret_cast<const void*>(gn_eval_stream_kernel<GsAccScalar>), smem, configured);
    if (err != cudaSuccess) return err;
    const int n_items = B * bpp;
    const int grid = n_items < 2 * sm_count ? n_items : 2 * sm_count;
    const GsLists L{pt_off, ls_off};
    gn_eval_stream_kernel<GsAccScalar><<<grid, GS_THREADS, smem, stream>>>(cam, (float)cfg.homog_th, L, pt, ls, DT, partial, bpp,
                                                                           n_items);
    err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    gn_eval_reduce_kernel<<<B, 32, 0, stream>>>(partial, bpp * GS_CWARPS, H, g, e);
    return cudaGetLastError();
}

}  // namespace plstvo
