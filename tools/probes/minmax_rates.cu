// minmax_rates.cu — issue rates of the packed min/max forms that tc_hamming_kernel's top-2 fold can use on sm_90a.
//
// Standalone: it does not link the library.  tools/probes/minmax_rates.py compiles it into tools/probes/bin/ with the
// library's nvcc flags.  It prints one JSON line: warp instructions per SM cycle per SM sub-partition for each case, at
// two shapes:
//   full     8 blocks of 256 threads per SM (up to 16 warps per sub-partition);
//   matcher  1 block of 256 threads per SM (2 warps per sub-partition), the shape of tc_hamming_kernel's consumer warps.
// Every thread runs 8 independent chains.  One step applies one instruction to each chain; the kind of instruction
// k = 8 s + i (step s, chain i) is pattern[k % length], so a mixed case interleaves its kinds instruction by instruction.
// Operands come from 8 registers derived from the thread index, so nothing is known at compile time.  Two-input kinds
// alternate min and max from step to step, so ptxas cannot merge two of them into one three-input instruction.
// Cycles are the SM's clock64() around the loop: per SM, the span from the first warp's start to the last warp's end.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

enum Kind { F2, F3, U2, U3 };   // HMNMX2, VHMNMX, VIMNMX.U16x2, VIMNMX3.U16x2

constexpr int CHAINS = 8, STEPS = 6;   // 48 instructions per iteration: patterns of length 1, 2 and 3 divide it

template <Kind K>
__device__ __forceinline__ uint32_t apply(uint32_t x, uint32_t a, uint32_t b, bool mx) {
    uint32_t d;
    if constexpr (K == F2) {
        if (mx) asm("max.f16x2 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(a));
        else asm("min.f16x2 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(a));
    } else if constexpr (K == F3) {
        if (mx) asm("{ .reg .b32 t; max.f16x2 t, %1, %2; max.f16x2 %0, t, %3; }" : "=r"(d) : "r"(x), "r"(a), "r"(b));
        else asm("{ .reg .b32 t; min.f16x2 t, %1, %2; min.f16x2 %0, t, %3; }" : "=r"(d) : "r"(x), "r"(a), "r"(b));
    } else if constexpr (K == U2) {
        if (mx) asm("max.u16x2 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(a));
        else asm("min.u16x2 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(a));
    } else {
        if (mx) asm("{ .reg .b32 t; max.u16x2 t, %1, %2; max.u16x2 %0, t, %3; }" : "=r"(d) : "r"(x), "r"(a), "r"(b));
        else asm("{ .reg .b32 t; min.u16x2 t, %1, %2; min.u16x2 %0, t, %3; }" : "=r"(d) : "r"(x), "r"(a), "r"(b));
    }
    return d;
}

template <Kind... P>
__global__ void __launch_bounds__(256) rate_kernel(uint32_t* out, long long* spans, int iters) {
    constexpr Kind pat[] = {P...};
    constexpr int L = sizeof...(P);
    const uint32_t s0 = threadIdx.x * 2654435761u + blockIdx.x;
    uint32_t p[CHAINS], x[CHAINS];
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
        p[i] = (s0 ^ (0x9E3779B9u * (i + 1))) & 0xBFFFBFFFu;   // finite f16 halves
        x[i] = p[i] ^ 0x00400040u;
    }
    __syncwarp();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int s = 0; s < STEPS; ++s) {
#pragma unroll
            for (int i = 0; i < CHAINS; ++i) {
                const uint32_t a = p[(i + s) % CHAINS], b = p[(i + s + 3) % CHAINS];
                const bool mx = s & 1;
                switch (pat[(CHAINS * s + i) % L]) {
                    case F2: x[i] = apply<F2>(x[i], a, b, mx); break;
                    case F3: x[i] = apply<F3>(x[i], a, b, mx); break;
                    case U2: x[i] = apply<U2>(x[i], a, b, mx); break;
                    case U3: x[i] = apply<U3>(x[i], a, b, mx); break;
                }
            }
        }
    }
    __syncwarp();
    const long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) acc ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if ((threadIdx.x & 31) == 0) {
        uint32_t sm;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
        long long* w = spans + 3 * (blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32);
        w[0] = sm;
        w[1] = t0;
        w[2] = t1;
    }
}

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e_ = (x);                                                          \
        if (e_ != cudaSuccess) {                                                       \
            fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); \
            exit(1);                                                                   \
        }                                                                              \
    } while (0)

struct Case {
    const char* name;
    void (*kernel)(uint32_t*, long long*, int);
};

// median over SMs of (warp instructions issued on the SM) / (SM cycles from first start to last end) / 4 sub-partitions
static double measure(const Case& c, int n_sm, int blocks_per_sm, int smem, int iters, uint32_t* d_out, long long* d_spans) {
    const int blocks = n_sm * blocks_per_sm, warps = blocks * 8;
    CK(cudaFuncSetAttribute(c.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    c.kernel<<<blocks, 256, smem>>>(d_out, d_spans, iters / 8);   // warm-up
    c.kernel<<<blocks, 256, smem>>>(d_out, d_spans, iters);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<long long> h(3 * (size_t)warps);
    CK(cudaMemcpy(h.data(), d_spans, h.size() * sizeof(long long), cudaMemcpyDeviceToHost));
    std::vector<long long> lo(n_sm, -1), hi(n_sm, -1), nw(n_sm, 0);
    for (int w = 0; w < warps; ++w) {
        const int sm = (int)h[3 * w];
        if (sm < 0 || sm >= n_sm) continue;
        lo[sm] = lo[sm] < 0 ? h[3 * w + 1] : std::min(lo[sm], h[3 * w + 1]);
        hi[sm] = std::max(hi[sm], h[3 * w + 2]);
        ++nw[sm];
    }
    std::vector<double> r;
    for (int s = 0; s < n_sm; ++s)
        if (nw[s] > 0 && hi[s] > lo[s]) r.push_back((double)nw[s] * iters * CHAINS * STEPS / (double)(hi[s] - lo[s]) / 4.0);
    std::sort(r.begin(), r.end());
    return r.empty() ? 0.0 : r[r.size() / 2];
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 4096;
    const Case cases[] = {
        {"HMNMX2", rate_kernel<F2>},
        {"VHMNMX", rate_kernel<F3>},
        {"VIMNMX.U16x2", rate_kernel<U2>},
        {"VIMNMX3.U16x2", rate_kernel<U3>},
        {"HMNMX2+VIMNMX.U16x2 1:1", rate_kernel<F2, U2>},
        {"HMNMX2+VIMNMX.U16x2 1:2", rate_kernel<F2, U2, U2>},
        {"VHMNMX+VIMNMX3.U16x2 1:1", rate_kernel<F3, U3>},
    };
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int n_sm = prop.multiProcessorCount;
    uint32_t* d_out;
    long long* d_spans;
    CK(cudaMalloc(&d_out, (size_t)n_sm * 8 * 256 * sizeof(uint32_t)));
    CK(cudaMalloc(&d_spans, (size_t)n_sm * 8 * 8 * 3 * sizeof(long long)));
    CK(cudaMemset(d_spans, 0xFF, (size_t)n_sm * 8 * 8 * 3 * sizeof(long long)));
    // the matcher shape reserves more than half of an SM's shared memory per block, so no SM holds two blocks
    const int one_block_smem = (int)(prop.sharedMemPerMultiprocessor / 2 + 1024);
    printf("{\"device\": \"%s\", \"sms\": %d, \"iters\": %d, \"unit\": \"warp instructions per SM cycle per SM sub-partition\"",
           prop.name, n_sm, iters);
    const char* shapes[] = {"full", "matcher"};
    for (int sh = 0; sh < 2; ++sh) {
        printf(", \"%s\": {", shapes[sh]);
        for (size_t c = 0; c < sizeof(cases) / sizeof(cases[0]); ++c) {
            CK(cudaMemset(d_spans, 0xFF, (size_t)n_sm * 8 * 8 * 3 * sizeof(long long)));
            const double r = sh == 0 ? measure(cases[c], n_sm, 8, 0, iters, d_out, d_spans)
                                     : measure(cases[c], n_sm, 1, one_block_smem, iters, d_out, d_spans);
            printf("%s\"%s\": %.4f", c ? ", " : "", cases[c].name, r);
        }
        printf("}");
    }
    printf("}\n");
    CK(cudaFree(d_out));
    CK(cudaFree(d_spans));
    return 0;
}
