// match_tc.cuh — work description of the tensor-core form of K1 (match_tc.cu).  Internal, not part of the boundary.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace plstvo {

constexpr int TC_ROWS = 128;                    // descriptor rows per operand tile (two wgmma M blocks of 64; N = 2 tiles)
constexpr int TC_TILE_BYTES = TC_ROWS * 256;    // 128 rows x 256 e4m3 bytes, swizzled K-major layout
constexpr int TC_CW = 256;                      // trains per work item = per row-partial block (two wgmma N of 128)
constexpr int TC_CWARPS = 8;                    // consumer warps: two warpgroups, 64 query rows of each tile apiece
constexpr int TC_XSTAGES = 4;                   // query tiles in flight (shared memory ring)
constexpr int TC_PTHREADS = 128;                // the producer warpgroup: work distribution and operand expansion
constexpr int TC_THREADS = 32 * TC_CWARPS + TC_PTHREADS;

// one matching problem = StVO::match(desc1, desc2): queries stream through the M side, trains sit on the N side
struct TcProblem {
    const uint8_t* d1;    // [n1][32] query descriptor rows (desc1), 16-byte aligned; expanded in the matcher
    const uint8_t* d2;    // [n2][32] train descriptor rows (desc2), 16-byte aligned
    int32_t n1, n2;
    uint32_t* rowp;       // [ceil(n2 / TC_CW)][n1]: best distance | second << 9 (511 = none) | tag << 18 (parity, chunk group, lane)
    uint32_t* colp;       // [n2]:                 best | second << 9 | tag << 18 (consumer warp)
};

// one work item of the persistent kernel: all query tiles of a problem against 256 trains
struct TcItem {
    int32_t problem;
    int32_t yblk;
};

size_t tc_smem_bytes();
// items_a then items_b form the work list (long items first); sched: two zeroed ints per concurrently running launch
cudaError_t launch_tc_hamming(const TcProblem* problems, const TcItem* items_a, int n_a, const TcItem* items_b, int n_b,
                              int* sched, int grid, cudaStream_t stream);
// writes MatchProblem::rowpart[n1] / colpart[n2]: one resolved key pair per row and per column (dist << 16 | index)
cudaError_t launch_tc_resolve(const MatchProblem* mps, const TcProblem* tps, int n_problems, int slices, cudaStream_t stream);

}  // namespace plstvo
