// match_tc.cu — K1 on the Hopper tensor cores (wgmma): all-pairs 256-bit Hamming 2-NN as a +-1 contraction.
//
// Replaces the arithmetic of StVO::matchNNR / StVO::match (src/matching.cpp:41-91), i.e. OpenCV's
// cv::BFMatcher(NORM_HAMMING)::knnMatch(desc1, desc2, ., 2) per direction.  With descriptor bits mapped to +-1,
//     a . b = (#equal bits) - (#different bits) = 256 - 2 d(a, b)          (exact, |a . b| <= 256)
// so the N1 x N2 distance matrix of one matching problem is a 256-deep GEMM.  Two kernels:
//   tc_hamming_kernel  persistent, warp-specialised: a producer warpgroup loads the raw 32-byte descriptor rows from
//                      global memory and expands them in shared memory to 256 e4m3 bytes each (+1.0 = 0x38, -1.0 = 0xB8)
//                      in the 128-byte-swizzled K-major operand layout wgmma reads; two consumer
//                      warpgroups issue wgmma m64n128k32 (e4m3 operands, f16 accumulators in registers, two columns
//                      per register) on the two 128-train halves of a block, each half folded while the other is on the
//                      tensor pipe, so the top-2 update of BOTH directions costs a few packed min/max per two distances:
//                        row direction   (query -> trains): fold over the columns in registers, then over four lanes;
//                        column direction (train -> queries): element-wise running top-2 over the row tiles in
//                                         registers, one cross-lane reduction per work item (not per tile).
//                      Keys carry no indices in the hot loop: only (best, second) VALUES and a small candidate tag
//                      (which chunk group / lane / warp the best came from);
//   tc_resolve_kernel  merges the per-block partials, converts to distances and recovers the best neighbour's index by
//                      re-evaluating the few tagged candidates with XOR + POPC (exact; ties resolved to the lowest index
//                      as OpenCV does), emitting the packed keys (dist << 16 | index) that everything
//                      downstream (ratio test, mutual filter, K2) reads.
// Integer-exact end to end: the bit-exact parity tests of the matcher are the acceptance test.
#include <cuda_fp16.h>

#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "match_finalize.cuh"
#include "match_tc.cuh"

namespace plstvo {

// ---------------------------------------------------------------------------------------------------------------
// expand: bits -> e4m3 +-1 bytes in the swizzled operand layout
// tile (128 rows) = [slab 0..1][row group 0..15][row 0..7][16-byte chunk position 0..7]; slab = 128 K-bytes;
// logical chunk c of row r sits at position c ^ (r & 7)  (the 128B swizzle: address bits [4,7) ^= bits [7,10))
// The train block of a work item is two such tiles per slab: [slab 0..1][256 rows], the same formula with r = 0..255.
//
// Which descriptor bit lands on which K index is free, as long as queries and trains use the same order: a . b sums
// over K.  The order taken makes the expansion two instructions per output word: 32-bit word i of the row (bits
// 32 i .. 32 i + 31) fills the 32 K-bytes of logical chunks 2 i and 2 i + 1, and byte k of 4-byte group j of those
// holds bit 8 k + j of the word.  Shifting the word left by 7 - j puts bit 8 k + j at bit 7 of byte k, the e4m3 sign.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_nc16(const uint8_t* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// one descriptor row (lo: bytes 0..15, hi: bytes 16..31) into operand row r of the block at shared address `base`
// (1024-byte aligned, slab stride SLAB).  A row past the end of its matrix arrives as all-ones with one = 0 and is
// written as zeros.  The row address carries r & 7 in the chunk bits, so each chunk's swizzled address is one XOR.
template <int SLAB>
__device__ __forceinline__ void expand_row(uint32_t base, int r, const uint4& lo, const uint4& hi, uint32_t one) {
    // r is opaque here: the addresses of a producer thread's rows are loop-invariant, and hoisting them out of the
    // item loop would overflow the producer's 40 registers
    asm volatile("" : "+r"(r));
    const uint32_t row = base + (r >> 3) * 1024 + (r & 7) * 144;   // 128 (r & 7) + 16 (r & 7)
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint32_t o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (~(w[i] << (7 - j)) & 0x80808080u) | one;   // set: 0x38 (+1), clear: 0xB8 (-1)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t c = (2 * i + h) & 7;
            sts128((row ^ (c << 4)) + (i >> 2) * SLAB, o[4 * h], o[4 * h + 1], o[4 * h + 2], o[4 * h + 3]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// PTX helpers (wgmma)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint32_t bar /* shared address */) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { mbar_arrive(smem_u32(bar)); }
// orders this thread's generic-proxy shared-memory stores before later async-proxy (wgmma) reads of them
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (f16, 32 registers) (+)= A[64 x 32] . B[128 x 32]^T, both e4m3 and K-major in shared memory.
// Register d[2i + r] of lane l in warp w of the warpgroup holds row 16 w + l / 4 + 8 r, columns 8 i + 2 (l % 4) + {0, 1}
// (low half = even column), i = 0..15.
__device__ __forceinline__ void wg_mma_f8(uint32_t (&d)[32], uint64_t adesc, uint64_t bdesc, int acc) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.f16.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}
// keeps the compiler from moving reads or writes of one accumulator set across the wgmma fence / wait.  Per set, never
// across both: the other set is in flight meanwhile, and touching its registers makes ptxas serialise the wgmma.
__device__ __forceinline__ void wg_fence_regs(uint32_t (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// packed f16x2 arithmetic on raw 32-bit registers
__device__ __forceinline__ uint32_t hmax2u(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("max.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t hmin2u(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("min.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t hne2mask(uint32_t a, uint32_t b) {   // 0xFFFF per half where a != b
    uint32_t d;
    asm("set.ne.u32.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t hgt2mask(uint32_t a, uint32_t b) {   // 0xFFFF per half where a > b
    uint32_t d;
    asm("set.gt.u32.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t hfma2u(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ uint32_t swap16(uint32_t a) { return __byte_perm(a, a, 0x1032); }
__device__ __forceinline__ uint32_t sel32(uint32_t mask, uint32_t a, uint32_t b) { return (mask & a) | (~mask & b); }   // one LOP3
__device__ __forceinline__ uint32_t h2u_lo(uint32_t p) {   // low half (an integer-valued f16 >= 0) -> uint32
    uint32_t d;
    asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %1; cvt.rni.u32.f16 %0, lo; }" : "=r"(d) : "r"(p));
    return d;
}
__device__ __forceinline__ uint32_t h2u_hi(uint32_t p) {
    uint32_t d;
    asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %1; cvt.rni.u32.f16 %0, hi; }" : "=r"(d) : "r"(p));
    return d;
}

// "no value" sentinel: -1024 (below every dot product, |a . b| <= 256)
constexpr uint32_t NEG2 = 0xE400E400u;
constexpr uint32_t H2_NEGHALF = 0xB800B800u, H2_128 = 0x58005800u, H2_511 = 0x5FFC5FFCu;
// (best, second) dot values packed (lo, hi) -> distances d = (256 - v) / 2 (exact), "none" (sentinel) -> 511
__device__ __forceinline__ uint32_t dots_to_dist(uint32_t pv) { return hmin2u(hfma2u(pv, H2_NEGHALF, H2_128), H2_511); }

// running top-2 update with two new values at once: 5 packed min / max
__device__ __forceinline__ void top2_pair(uint32_t& k1, uint32_t& k2, uint32_t a, uint32_t b) {
    const uint32_t hi = hmax2u(a, b), lo = hmin2u(a, b);
    const uint32_t t = hmin2u(k1, hi);
    k2 = hmax2u(hmax2u(k2, lo), t);
    k1 = hmax2u(hmax2u(k1, a), b);
}
// merges another (best, second) pair into (k1, k2), element-wise
__device__ __forceinline__ void top2_merge(uint32_t& k1, uint32_t& k2, uint32_t o1, uint32_t o2) {
    k2 = hmax2u(hmax2u(hmin2u(k1, o1), k2), o2);
    k1 = hmax2u(k1, o1);
}

// shared-memory operand descriptor: K-major, 128-byte swizzle, 8-row groups 1024 B apart (SBO)
__device__ __forceinline__ uint64_t tc_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// issues one 128-train half of a query tile into accumulator set d as one commit group: 8 K-steps (two 128-byte slabs x
// four k32).  xa: the warpgroup's 64 query rows of the stage (slab 0); yb: the half's train tile in slab 0 of the train block.
// The K-steps' descriptors are the first one's plus a constant: shared addresses stay below 2^18, so the 14-bit start
// address field (address >> 4) never carries into the next field.
__device__ __forceinline__ void wg_issue_half(uint32_t (&d)[32], uint32_t xa, uint32_t yb) {
    const uint64_t da = tc_desc(xa), db = tc_desc(yb);
    wg_fence_regs(d);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
        wg_mma_f8(d, da + (((kk >> 2) * 16384 + (kk & 3) * 32) >> 4), db + (((kk >> 2) * 32768 + (kk & 3) * 32) >> 4), kk > 0);
    wg_commit();
}

// ---------------------------------------------------------------------------------------------------------------
// the matcher
// ---------------------------------------------------------------------------------------------------------------
constexpr int TC_OFF_X = 0;
constexpr int TC_OFF_Y = TC_XSTAGES * TC_TILE_BYTES;                      // [slab 0..1][256 rows]: 64 KB
constexpr int TC_HN = TC_CW / 2;                                          // wgmma N: trains per accumulator set
constexpr int TC_HALF_BYTES = TC_HN * 128;                                // train half 1 within a slab of the train block
constexpr int TC_OFF_MRG = TC_OFF_Y + 2 * TC_TILE_BYTES;                  // [8 consumer warps][256 columns] uint32: 8 KB
constexpr int TC_OFF_BAR = TC_OFF_MRG + TC_CWARPS * TC_CW * 4;
constexpr int TC_IRING = 4;                                               // work items announced ahead
constexpr int TC_NBARS = 2 * TC_XSTAGES + 2 + 2 * TC_IRING;
constexpr int TC_OFF_RING = TC_OFF_BAR + TC_NBARS * 8;
constexpr int TC_SMEM_USED = TC_OFF_RING + TC_IRING * 4;
static_assert(TC_SMEM_USED + 1024 <= 227 * 1024, "tc_hamming_kernel: shared memory");

size_t tc_smem_bytes() { return (size_t)TC_SMEM_USED + 1024; }

// Register budget: the CTA launches with 168 registers per thread (384 threads, 1 CTA / SM), too few for both accumulator
// sets, the column state and the row chains of a consumer thread.  The producer warpgroup, which needs few registers to
// expand one row at a time, hands most of its share to the consumers (setmaxnreg); each of the four SM sub-partitions then
// holds two consumer warps and one producer warp: (2 x 232 + 40) x 32 <= 16384 registers.
constexpr int TC_LAUNCH_REGS = 168, TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;
static_assert(TC_LAUNCH_REGS * TC_THREADS <= 65536 &&
                  TC_CWARPS * TC_CONSUMER_REGS + (TC_THREADS / 32 - TC_CWARPS) * TC_PRODUCER_REGS <= TC_LAUNCH_REGS * TC_THREADS / 32,
              "tc_hamming_kernel: register budget");
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__global__ void __launch_bounds__(TC_THREADS, 1)
tc_hamming_kernel(const TcProblem* __restrict__ problems, const TcItem* __restrict__ items_a, int n_a,
                  const TcItem* __restrict__ items_b, int n_b, int* __restrict__ sched) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t sbase = (raw + 1023u) & ~1023u;
    uint8_t* sm = smem_raw + (sbase - raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + TC_OFF_BAR);
    uint64_t* x_full = bars;
    uint64_t* x_empty = bars + TC_XSTAGES;
    uint64_t* y_full = bars + 2 * TC_XSTAGES;
    uint64_t* y_empty = y_full + 1;
    uint64_t* i_full = y_empty + 1;
    uint64_t* i_empty = i_full + TC_IRING;
    volatile int* iring = reinterpret_cast<volatile int*>(sm + TC_OFF_RING);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_items = n_a + n_b;

    if (tid == 0) {
        for (int i = 0; i < TC_XSTAGES; ++i) {
            mbar_init(&x_full[i], TC_PTHREADS);
            mbar_init(&x_empty[i], TC_CWARPS);
        }
        mbar_init(y_full, TC_PTHREADS);
        mbar_init(y_empty, TC_CWARPS);
        for (int i = 0; i < TC_IRING; ++i) {
            mbar_init(&i_full[i], 1);
            mbar_init(&i_empty[i], TC_CWARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();

    // work items are handed out by an atomic counter (long ones first: list a, then list b) and announced to the
    // consumers through a small ring in shared memory; -1 ends the kernel
    auto item_at = [&](int it) -> TcItem { return it < n_a ? items_a[it] : items_b[it - n_a]; };

    if (warp >= TC_CWARPS) {
        // ===== producer: work distribution + operand expansion =====
        // Thread 0 takes the items and announces them; every producer thread reads them from the ring.  (A slot is
        // reused four items later, when all producer threads have long read it: the item before that needed every
        // producer thread's query rows.)  Each producer thread expands two rows of the train block and one row of every
        // query tile, and arrives on the full barrier after its stores.
        setmaxnreg_dec<TC_PRODUCER_REGS>();
        const int ptid = tid - TC_CWARPS * 32;
        // barriers as shared addresses off the aligned base (fewer live registers than the generic pointers)
        const uint32_t bar_x_full = sbase + TC_OFF_BAR, bar_x_empty = bar_x_full + 8 * TC_XSTAGES,
                       bar_y_full = bar_x_full + 16 * TC_XSTAGES, bar_y_empty = bar_y_full + 8,
                       bar_i_full = bar_y_full + 16, bar_i_empty = bar_i_full + 8 * TC_IRING;
        // The producer has 40 registers.  Rows are opaque (asm) so that a thread's row addresses are not hoisted out of the
        // item loop, and the query side of the problem is re-read after the train block rather than held across it; n <=
        // 65535 rows, so row offsets fit 32 bits.  The read-only (.nc) row loads carry no ordering, so ptxas issues them
        // ahead of the stage wait where registers allow: the ring hides their latency.
        auto row_ptr = [&](const uint8_t* d, int row) {
            asm volatile("" : "+r"(row));
            return d + (uint32_t)row * 32u;
        };
        // a row past the end of its matrix reads as all-ones and is expanded to zeros
        auto expand = [&](auto slab, uint32_t base, int r, const uint8_t* d, int row, int n) {
            const bool v = row < n;
            const uint4 ones = make_uint4(~0u, ~0u, ~0u, ~0u);
            const uint4 lo = v ? ldg_nc16(row_ptr(d, row)) : ones, hi = v ? ldg_nc16(row_ptr(d, row) + 16) : ones;
            expand_row<decltype(slab)::value>(base, r, lo, hi, v ? 0x38383838u : 0u);
        };
        constexpr std::integral_constant<int, TC_TILE_BYTES / 2> XSLAB{};
        constexpr std::integral_constant<int, TC_TILE_BYTES> YSLAB{};
        uint32_t xs = 0, xph = 0;
        auto query_tile = [&](const TcProblem& pr, int t) {
            mbar_wait(bar_x_empty + 8 * xs, xph ^ 1);
            expand(XSLAB, sbase + TC_OFF_X + xs * TC_TILE_BYTES, ptid, pr.d1, t * TC_ROWS + ptid, pr.n1);
            fence_proxy_async_smem();
            mbar_arrive(bar_x_full + 8 * xs);
            if (++xs == TC_XSTAGES) { xs = 0; xph ^= 1; }
        };
        for (uint32_t k = 0;; ++k) {
            const uint32_t slot = k % TC_IRING;
            if (ptid == 0) {
                mbar_wait(bar_i_empty + 8 * slot, ((k / TC_IRING) & 1) ^ 1);
                int it = atomicAdd(sched, 1);
                if (it >= n_items) it = -1;
                iring[slot] = it;
                mbar_arrive(bar_i_full + 8 * slot);
            }
            mbar_wait(bar_i_full + 8 * slot, (k / TC_IRING) & 1);
            const int it = iring[slot];
            if (it < 0) break;
            const TcItem item = item_at(it);
            const TcProblem pr = problems[item.problem];
            mbar_wait(bar_y_empty, (k & 1) ^ 1);
            expand(YSLAB, sbase + TC_OFF_Y, ptid, pr.d2, item.yblk * TC_CW + ptid, pr.n2);
            fence_proxy_async_smem();   // (also keeps the next row's loads from being hoisted into this expansion)
            expand(YSLAB, sbase + TC_OFF_Y, ptid + TC_ROWS, pr.d2, item.yblk * TC_CW + TC_ROWS + ptid, pr.n2);
            fence_proxy_async_smem();
            mbar_arrive(bar_y_full);
            // the query side, re-read through an opaque index: one register across the train block, not a 64-bit pointer
            int pi = item.problem;
            asm volatile("" : "+r"(pi));
            const TcProblem& pq = problems[pi];
            const int nxt = (pq.n1 + TC_ROWS - 1) / TC_ROWS;
            for (int t = 0; t < nxt; ++t) query_tile(pq, t);
        }
    } else {
        // ===== consumers: two warpgroups; warpgroup g multiplies query rows 64 g .. 64 g + 63 of every query tile with the
        // item's 256 trains (f16 accumulators in registers: every partial sum is an integer of magnitude <= 256, exact in
        // f16), then folds the tile into
        //   row direction    (query -> trains): each thread holds 64 columns of two rows; top-2 in registers, then over the
        //                                      four lanes of a row by shuffle;
        //   column direction (train -> queries): element-wise running top-2 over the rows in registers, reduced over lanes,
        //                                      warps and warpgroups once per work item (not per tile).
        // Keys carry no indices in the hot loop: only (best, second) VALUES and a small candidate tag.
        // The 256 trains are two halves of 128 (wgmma m64n128k32), one accumulator set each, software-pipelined so that
        // each half of a tile is folded while the MMA of the next half (t, 1) or (t + 1, 0) is on the tensor pipe.
        setmaxnreg_inc<TC_CONSUMER_REGS>();
        // the warpgroup index through a shuffle from lane 0: ptxas then knows it is warp-uniform and keeps the operand
        // addresses and wgmma descriptors derived from it in uniform registers, off the vector ALU the fold saturates
        const int wg = __shfl_sync(0xFFFFFFFFu, warp >> 2, 0), w = warp & 3, q4 = lane & 3, rl = lane >> 2;
        uint32_t* mrg = reinterpret_cast<uint32_t*>(sm + TC_OFF_MRG);
        uint32_t acc[2][32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[0][i] = acc[1][i] = 0u;
        uint32_t xs = 0, xph = 0;
        for (uint32_t k = 0;; ++k) {
            const uint32_t slot = k % TC_IRING;
            mbar_wait(&i_full[slot], (k / TC_IRING) & 1);
            const int it = iring[slot];
            __syncwarp();
            if (lane == 0) mbar_arrive(&i_empty[slot]);
            if (it < 0) break;
            const TcItem item = item_at(it);
            const TcProblem pr = problems[item.problem];
            const int nxt = (pr.n1 + TC_ROWS - 1) / TC_ROWS;
            const int ycol0 = item.yblk * TC_CW;
            const int nvalid = min(TC_CW, pr.n2 - ycol0);
            uint32_t c1[32], c2[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) c1[i] = c2[i] = NEG2;
            mbar_wait(y_full, k & 1);
            const uint32_t xw = sbase + TC_OFF_X + wg * 8192, ya = sbase + TC_OFF_Y;   // + stage, + half of the trains
            // row direction: one chain per row, carried from half 0 to half 1 of a tile; the tag records which group of
            // four 8-column chunks (0..7 over both halves) raised the best
            uint32_t a1, a2, b1, b2, ta, tb;
            // masks and folds the retired accumulator set h of tile t; after half 1 the row chains are merged and stored
            auto fold = [&](auto hc, int t) {
                constexpr int h = decltype(hc)::value;
                uint32_t (&d)[32] = acc[h];
                const int x0 = t * TC_ROWS + wg * 64 + w * 16 + rl;   // rows x0 (registers 2i) and x0 + 8 (registers 2i + 1)
                if (nvalid < TC_HN * (h + 1) || t * TC_ROWS + wg * 64 + 64 > pr.n1) {
                    // a partial tile or block: rows past the end (zero operand rows) and columns past the end contribute nothing
                    const bool v0 = x0 < pr.n1, v1 = x0 + 8 < pr.n1;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int col = TC_HN * h + 8 * i + 2 * q4;
                        const uint32_t cm = col >= nvalid ? 0xFFFFFFFFu : (col + 1 >= nvalid ? 0xFFFF0000u : 0u);
                        d[2 * i] = v0 ? sel32(cm, NEG2, d[2 * i]) : NEG2;
                        d[2 * i + 1] = v1 ? sel32(cm, NEG2, d[2 * i + 1]) : NEG2;
                    }
                }
                if (h == 0) {
                    a1 = a2 = b1 = b2 = NEG2;
                    ta = tb = 0;
                }
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const uint32_t olda = a1, oldb = b1;
                    top2_pair(a1, a2, d[8 * g + 0], d[8 * g + 2]);
                    top2_pair(b1, b2, d[8 * g + 1], d[8 * g + 3]);
                    top2_pair(a1, a2, d[8 * g + 4], d[8 * g + 6]);
                    top2_pair(b1, b2, d[8 * g + 5], d[8 * g + 7]);
                    ta = sel32(hne2mask(a1, olda), (uint32_t)(4 * h + g) * 0x00010001u, ta);
                    tb = sel32(hne2mask(b1, oldb), (uint32_t)(4 * h + g) * 0x00010001u, tb);
                }
                // column direction: rows x0 and x0 + 8 into the running state of this half's columns
#pragma unroll
                for (int i = 0; i < 16; ++i) top2_pair(c1[16 * h + i], c2[16 * h + i], d[2 * i], d[2 * i + 1]);
                if constexpr (h == 1) {
                    // even- and odd-column streams, then the four lanes of the row; the result sits in the low halves.
                    // tag = parity | chunk group << 1 | lane % 4 << 4
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const uint32_t m1 = r ? b1 : a1, m2 = r ? b2 : a2, tg = r ? tb : ta;
                        const uint32_t s1 = swap16(m1), s2 = swap16(m2), st = swap16(tg);
                        uint32_t f1 = m1, f2 = m2;
                        top2_merge(f1, f2, s1, s2);
                        uint32_t tag = (sel32(hgt2mask(s1, m1), (st << 1) | 1u, tg << 1) & 0xFu) | ((uint32_t)q4 << 4);
#pragma unroll
                        for (int m = 1; m <= 2; m <<= 1) {
                            const uint32_t o1 = __shfl_xor_sync(0xFFFFFFFFu, f1, m), o2 = __shfl_xor_sync(0xFFFFFFFFu, f2, m),
                                           ot = __shfl_xor_sync(0xFFFFFFFFu, tag, m);
                            tag = (hgt2mask(o1, f1) & 1u) ? ot : tag;
                            top2_merge(f1, f2, o1, o2);
                        }
                        const int x = x0 + 8 * r;
                        if (q4 == 0 && x < pr.n1) {
                            const uint32_t dd = dots_to_dist(__byte_perm(f1, f2, 0x5410));
                            pr.rowp[(size_t)item.yblk * pr.n1 + x] = h2u_lo(dd) | (h2u_hi(dd) << 9) | (tag << 18);
                        }
                    }
                }
            };
            constexpr std::integral_constant<int, 0> H0{};
            constexpr std::integral_constant<int, 1> H1{};

            // Each fold runs under the MMA of the other half: (t, 1) is issued before (t, 0) is folded, (t + 1, 0) before
            // (t, 1) is.  Two orderings are load-bearing:
            //  * every commit group is retired inside the iteration that issued it: a group still in flight at the loop's
            //    back edge or exit has no single retiring wait on all paths, and ptxas then treats every accumulator read
            //    as a read of an in-flight register and serialises all the wgmma;
            //  * the fold of set 0 precedes the issue of (t + 1, 0) into the same registers, and the wait for (t, 1)
            //    follows that issue.  ptxas would otherwise hoist the wait above the fold, which no register ties to it.
            mbar_wait(&x_full[xs], xph);
            wg_issue_half(acc[0], xw + xs * TC_TILE_BYTES, ya);   // (0, 0)
            wg_wait<0>();
            wg_fence_regs(acc[0]);
            for (int t = 0; t + 1 < nxt; ++t) {
                const uint32_t nxs = xs + 1 == TC_XSTAGES ? 0 : xs + 1, nxph = nxs == 0 ? xph ^ 1 : xph;
                wg_issue_half(acc[1], xw + xs * TC_TILE_BYTES, ya + TC_HALF_BYTES);   // (t, 1)
                fold(H0, t);
                mbar_wait(&x_full[nxs], nxph);
                wg_issue_half(acc[0], xw + nxs * TC_TILE_BYTES, ya);   // (t + 1, 0)
                wg_wait<1>();   // retires (t, 1)
                wg_fence_regs(acc[1]);
                __syncwarp();
                if (lane == 0) mbar_arrive(&x_empty[xs]);   // both halves of tile t have read the stage
                fold(H1, t);
                wg_wait<0>();   // retires (t + 1, 0)
                wg_fence_regs(acc[0]);
                xs = nxs;
                xph = nxph;
            }
            // the last tile: nothing more to issue after its second half
            wg_issue_half(acc[1], xw + xs * TC_TILE_BYTES, ya + TC_HALF_BYTES);
            fold(H0, nxt - 1);
            wg_wait<0>();
            wg_fence_regs(acc[1]);
            __syncwarp();
            if (lane == 0) {   // the stage and the trains are free
                mbar_arrive(&x_empty[xs]);
                mbar_arrive(y_empty);
            }
            fold(H1, nxt - 1);
            if (++xs == TC_XSTAGES) { xs = 0; xph ^= 1; }

            // ---- column direction: reduce the element-wise state over the eight lanes of a column (shuffles), then over the
            // eight consumer warps (shared memory); the tag is the warp the best came from ----
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                uint32_t m1 = c1[i], m2 = c2[i];
#pragma unroll
                for (int m = 4; m <= 16; m <<= 1)
                    top2_merge(m1, m2, __shfl_xor_sync(0xFFFFFFFFu, m1, m), __shfl_xor_sync(0xFFFFFFFFu, m2, m));
                if (rl == 0) {
                    const int col = 8 * i + 2 * q4;
                    mrg[warp * TC_CW + col] = (m1 & 0xFFFFu) | (m2 << 16);
                    mrg[warp * TC_CW + col + 1] = (m1 >> 16) | (m2 & 0xFFFF0000u);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(TC_CWARPS * 32) : "memory");
            {
                const int col = tid;   // one column per consumer thread
                uint32_t b1 = NEG2, b2 = NEG2, bt = 0;   // only the low halves are meaningful
#pragma unroll
                for (int s = 0; s < TC_CWARPS; ++s) {
                    const uint32_t e = mrg[s * TC_CW + col];
                    const uint32_t a1 = e & 0xFFFFu, a2 = e >> 16;
                    bt = (hgt2mask(a1, b1) & 1u) ? (uint32_t)s : bt;
                    top2_merge(b1, b2, a1, a2);
                }
                if (col < nvalid) {
                    const uint32_t dd = dots_to_dist(__byte_perm(b1, b2, 0x5410));
                    pr.colp[ycol0 + col] = h2u_lo(dd) | (h2u_hi(dd) << 9) | (bt << 18);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(TC_CWARPS * 32) : "memory");
        }
    }

    // the last CTA out re-arms the scheduler words for the next launch on this stream
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(sched + 1, 1) == (int)gridDim.x - 1) {
            sched[0] = 0;
            sched[1] = 0;
            __threadfence();
        }
    }
}

cudaError_t launch_tc_hamming(const TcProblem* problems, const TcItem* items_a, int n_a, const TcItem* items_b, int n_b,
                              int* sched, int grid, cudaStream_t stream) {
    const int n_items = n_a + n_b;
    if (n_items <= 0) return cudaSuccess;
    static size_t configured[64] = {};
    const size_t smem = tc_smem_bytes();
    cudaError_t e = ensure_dynamic_smem(reinterpret_cast<const void*>(tc_hamming_kernel), smem, configured);
    if (e != cudaSuccess) return e;
    if (grid > n_items) grid = n_items;
    if (getenv("PLSTVO_TC_DIAG")) {
        cudaFuncAttributes fa;
        int occ = -1;
        cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(tc_hamming_kernel));
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, tc_hamming_kernel, TC_THREADS, smem);
        fprintf(stderr, "[tc diag] regs %d, maxThreadsPerBlock %d, static smem %zu, local %zu, dynamic smem %zu, occupancy %d\n",
                fa.numRegs, fa.maxThreadsPerBlock, fa.sharedSizeBytes, fa.localSizeBytes, smem, occ);
    }
    tc_hamming_kernel<<<grid, TC_THREADS, smem, stream>>>(problems, items_a, n_a, items_b, n_b, sched);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// resolve: values -> distances, candidate tags -> exact indices, packed keys out
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int hamming256(const uint4& a0, const uint4& a1, const uint8_t* p) {
    const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(p)), b1 = __ldg(reinterpret_cast<const uint4*>(p) + 1);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) +
           __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

__global__ void __launch_bounds__(256) tc_resolve_kernel(const MatchProblem* __restrict__ mps, const TcProblem* __restrict__ tps) {
    const MatchProblem mp = mps[blockIdx.x];
    if (!mp.enabled) return;
    const TcProblem tp = tps[blockIdx.x];
    const int nyh = (mp.n2 + TC_CW - 1) / TC_CW, nxt = (mp.n1 + TC_ROWS - 1) / TC_ROWS;   // row partials: one per TC_CW-train block
    const int slice = blockIdx.y, nslices = gridDim.y;
    // partial word: best distance (9 bits) | second distance << 9 (511 = none) | candidate tag << 18
    // queries: top-2 trains over the 256-train blocks (lowest block wins a tie: its indices are lower)
    for (int x = slice * blockDim.x + threadIdx.x; x < mp.n1; x += nslices * blockDim.x) {
        uint32_t b1 = 511, b2 = 511, btag = 0;
        int bh = 0;
        for (int h = 0; h < nyh; ++h) {
            const uint32_t e = __ldg(&tp.rowp[(size_t)h * mp.n1 + x]);
            const uint32_t a1 = e & 511u, a2 = (e >> 9) & 511u;
            b2 = min(max(b1, a1), min(b2, a2));
            if (a1 < b1) { b1 = a1; bh = h; btag = e >> 18; }
        }
        const int d1 = (int)b1;
        uint32_t k2 = KEY_NONE;
        int idx = 0;
        if (mp.n2 >= 2) {
            const int d2 = (int)b2;
            k2 = ((uint32_t)d2 << 16) | 0xFFFEu;
            if ((float)d1 < __fmul_rn((float)d2, mp.nnr)) {
                const uint4 a0 = __ldg(reinterpret_cast<const uint4*>(mp.d1 + (size_t)x * 32)),
                            a1 = __ldg(reinterpret_cast<const uint4*>(mp.d1 + (size_t)x * 32) + 1);
                idx = -1;
                if (d1 != d2) {   // unique best: it is one of the 4 tagged trains (one lane's columns of a chunk group, one parity)
                    const int base = bh * TC_CW + (int)((btag >> 1) & 7u) * 32 + (int)((btag >> 4) & 3u) * 2 + (int)(btag & 1u);
                    for (int i = 0; i < 4 && idx < 0; ++i) {
                        const int j = base + 8 * i;
                        if (j < mp.n2 && hamming256(a0, a1, mp.d2 + (size_t)j * 32) == d1) idx = j;
                    }
                }
                if (idx < 0) {   // tie accepted (nnr > 1): lowest index among all trains, as OpenCV orders them
                    for (int j = 0; j < mp.n2 && idx < 0; ++j)
                        if (hamming256(a0, a1, mp.d2 + (size_t)j * 32) == d1) idx = j;
                    if (idx < 0) idx = 0;
                }
            }
        }
        mp.rowpart[x] = make_uint2(((uint32_t)d1 << 16) | (uint32_t)idx, k2);
    }
    // trains: top-2 queries
    for (int y = slice * blockDim.x + threadIdx.x; y < mp.n2; y += nslices * blockDim.x) {
        const uint32_t e = __ldg(&tp.colp[y]);
        const int d1 = (int)(e & 511u);
        uint32_t k2 = KEY_NONE;
        int idx = 0;
        if (mp.n1 >= 2) {
            const int d2 = (int)((e >> 9) & 511u);
            k2 = ((uint32_t)d2 << 16) | 0xFFFEu;
            if ((float)d1 < __fmul_rn((float)d2, mp.nnr)) {
                const uint4 a0 = __ldg(reinterpret_cast<const uint4*>(mp.d2 + (size_t)y * 32)),
                            a1 = __ldg(reinterpret_cast<const uint4*>(mp.d2 + (size_t)y * 32) + 1);
                idx = -1;
                if (d1 != d2 && mp.n1 <= (int)M21_DIST) {
                    // unique best: WHICH query it is does not matter to the mutual filter (match_finalize.cuh: a query whose
                    // nearest train is y at distance d1 is that query) — no candidate is re-evaluated
                    idx = (int)KEY_IDX_UNRESOLVED;
                } else if (d1 != d2) {   // (frames beyond 65024 rows) one of the 16 rows per tile the tagged consumer warp holds
                    const int wt = (int)((e >> 18) & 7u), r0 = (wt >> 2) * 64 + (wt & 3) * 16;
                    for (int i = 0; i < nxt && idx < 0; ++i)
                        for (int r = 0; r < 16 && idx < 0; ++r) {
                            const int j = r0 + r + i * TC_ROWS;
                            if (j < mp.n1 && hamming256(a0, a1, mp.d1 + (size_t)j * 32) == d1) idx = j;
                        }
                }
                if (idx < 0) {
                    for (int j = 0; j < mp.n1 && idx < 0; ++j)
                        if (hamming256(a0, a1, mp.d1 + (size_t)j * 32) == d1) idx = j;
                    if (idx < 0) idx = 0;
                }
            }
        }
        mp.colpart[y] = make_uint2(((uint32_t)d1 << 16) | (uint32_t)idx, k2);
    }
}

cudaError_t launch_tc_resolve(const MatchProblem* mps, const TcProblem* tps, int n_problems, int slices, cudaStream_t stream) {
    if (n_problems <= 0) return cudaSuccess;
    tc_resolve_kernel<<<dim3(n_problems, slices > 0 ? slices : 1), 256, 0, stream>>>(mps, tps);
    return cudaGetLastError();
}

}  // namespace plstvo
