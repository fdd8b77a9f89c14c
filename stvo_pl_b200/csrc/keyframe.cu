// keyframe.cu — the PL-SLAM key-frame test of a session run on the device (plstvo_stereo_session_run_keyframes): needNewKF
// and currFrameIsKF of every named stream after each step's optimizePose.  (session_gather_kernel copies the key frames'
// records into the run's retention chunks.)
//
// Precision: every operation follows plstvo.hpp's se3 helpers and KeyframeTest::needNewKF in fp64, in the header's order,
// with its pivoting, loop order and divisions.  Each a * b + c is spelled __dadd_rn(__dmul_rn(a, b), c) so that nvcc forms
// no FMA (the host rounds the product and the sum apart).  Division and sqrt are IEEE-rounded on both sides.  The only
// operations left that can differ from the host are CUDA's log (of the two determinants) and acos (in logmap); the constant
// 3 (1 + log 2 pi) is computed on the host and passed in.
#include "host.cuh"

namespace plstvo {

namespace {

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

__device__ void identity4(double* T) {
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}
// se3::mul: C = A B
__device__ void mul4(const double* A, const double* B, double* C) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc = add(acc, mul(A[4 * i + k], B[4 * k + j]));
            C[4 * i + j] = acc;
        }
}
// se3::inverse: [R^T, -R^T t]
__device__ void inverse4(const double* T, double* Ti) {
    identity4(Ti);
    for (int i = 0; i < 3; ++i) {
        double acc = 0.0;
        for (int k = 0; k < 3; ++k) {
            Ti[4 * i + k] = T[4 * k + i];
            acc = add(acc, mul(-T[4 * k + i], T[4 * k + 3]));
        }
        Ti[4 * i + 3] = acc;
    }
}
// se3::logmap: x = [V^-1 t ; w]
__device__ void logmap(const double* T, double* x) {
    double cosine = sub(add(add(T[0], T[5]), T[10]), 1.0) / 2.0;
    cosine = (-1.0 < cosine) ? cosine : -1.0;   // std::max(-1.0, c), then std::min(1.0, c): NaN becomes -1 as on the host
    cosine = (cosine < 1.0) ? cosine : 1.0;
    double sine = sqrt(sub(1.0, mul(cosine, cosine)));
    sine = (sine < 1.0) ? sine : 1.0;
    const double theta = acos(cosine);   // CUDA's acos: may differ from the host's in the last ulp
    double w[3] = {0, 0, 0}, V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (theta > 0.000001) {
        const double k = theta / mul(2.0, sine);
        w[0] = mul(k, sub(T[9], T[6]));
        w[1] = mul(k, sub(T[2], T[8]));
        w[2] = mul(k, sub(T[4], T[1]));
        const double s[9] = {0, -w[2] / theta, w[1] / theta, w[2] / theta, 0, -w[0] / theta, -w[1] / theta, w[0] / theta, 0};
        const double a = sub(1.0, cosine) / theta, b = sub(theta, sine) / theta;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double ss = 0.0;
                for (int m = 0; m < 3; ++m) ss = add(ss, mul(s[3 * i + m], s[3 * m + j]));
                V[3 * i + j] = add(add(i == j ? 1.0 : 0.0, mul(s[3 * i + j], a)), mul(ss, b));
            }
    }
    const double c00 = sub(mul(V[4], V[8]), mul(V[5], V[7])), c01 = sub(mul(V[5], V[6]), mul(V[3], V[8])),
                 c02 = sub(mul(V[3], V[7]), mul(V[4], V[6]));
    const double det = add(add(mul(V[0], c00), mul(V[1], c01)), mul(V[2], c02));
    const double inv[9] = {c00 / det, sub(mul(V[2], V[7]), mul(V[1], V[8])) / det, sub(mul(V[1], V[5]), mul(V[2], V[4])) / det,
                           c01 / det, sub(mul(V[0], V[8]), mul(V[2], V[6])) / det, sub(mul(V[2], V[3]), mul(V[0], V[5])) / det,
                           c02 / det, sub(mul(V[1], V[6]), mul(V[0], V[7])) / det, sub(mul(V[0], V[4]), mul(V[1], V[3])) / det};
    for (int i = 0; i < 3; ++i) {
        x[i] = add(add(mul(inv[3 * i], T[3]), mul(inv[3 * i + 1], T[7])), mul(inv[3 * i + 2], T[11]));
        x[3 + i] = w[i];
    }
}
// se3::adjoint: [R, skew(t) R; 0, R]
__device__ void adjoint(const double* T, double* A) {
    for (int i = 0; i < 36; ++i) A[i] = 0.0;
    const double t[3] = {T[3], T[7], T[11]};
    const double sk[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            A[6 * i + j] = T[4 * i + j];
            A[6 * (i + 3) + j + 3] = T[4 * i + j];
            double acc = 0.0;
            for (int k = 0; k < 3; ++k) acc = add(acc, mul(sk[3 * i + k], T[4 * k + j]));
            A[6 * i + j + 3] = acc;
        }
}
// se3::sandwich: out = A C A^T (AC scratch)
__device__ void sandwich(const double* A, const double* C, double* AC, double* out) {
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc = add(acc, mul(A[6 * i + k], C[6 * k + j]));
            AC[6 * i + j] = acc;
        }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc = add(acc, mul(AC[6 * i + k], A[6 * j + k]));
            out[6 * i + j] = acc;
        }
}
// se3::det6: partial-pivot LU on a copy (A is overwritten)
__device__ double det6(double* A) {
    double det = 1.0;
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        for (int r = c + 1; r < 6; ++r)
            if (fabs(A[6 * r + c]) > fabs(A[6 * piv + c])) piv = r;
        if (A[6 * piv + c] == 0.0) return 0.0;
        if (piv != c) {
            for (int j = 0; j < 6; ++j) {
                const double v = A[6 * c + j];
                A[6 * c + j] = A[6 * piv + j];
                A[6 * piv + j] = v;
            }
            det = -det;
        }
        det = mul(det, A[6 * c + c]);
        for (int r = c + 1; r < 6; ++r) {
            const double f = A[6 * r + c] / A[6 * c + c];
            for (int j = c + 1; j < 6; ++j) A[6 * r + j] = sub(A[6 * r + j], mul(f, A[6 * c + j]));
        }
    }
    return det;
}

// KeyframeTest::needNewKF (src/stereoFrameHandler.cpp:1136-1187) of stream k on its step's result, then currFrameIsKF
// (:1189-1218) where it fires: the stream's state is reset and the next step's prior takes Tfw = I, Tfw_cov = I.
// The result is read where the solver left it; results keep optimizePose's Tfw.
__global__ void session_keyframe_kernel(PlKeyframeConfig cfg, double k_entropy, int n, const PlPoseResult* __restrict__ results,
                                        PlKeyframeState* __restrict__ state, PlKeyframeResult* __restrict__ out,
                                        PlPrior* __restrict__ priors) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const PlPoseResult& r = results[k];
    PlKeyframeState& s = state[k];
    double A[36], B[36], C[36], D[36], M[16], N[16];
    if (s.prev_f_iskf) {                                 // :1140-1153
        for (int i = 0; i < 36; ++i) A[i] = r.DT_cov[i];
        const double d = det6(A);
        s.entropy_first_prevKF = (d != 0.0) ? add(k_entropy, mul(0.5, log(d))) : -999999999.99;
        s.prev_f_iskf = 0;
    }
    double dX[6];                                        // :1156-1159
    inverse4(r.Tfw, M);
    mul4(M, s.T_prevKF, N);
    logmap(N, dX);
    const double t = sqrt(add(add(mul(dX[0], dX[0]), mul(dX[1], dX[1])), mul(dX[2], dX[2])));
    const double rot = mul(sqrt(add(add(mul(dX[3], dX[3]), mul(dX[4], dX[4])), mul(dX[5], dX[5]))), 180.0) /
                       3.1415926535897932384626433832795;
    inverse4(r.DT, M);                                   // :1162-1164: Ad(T_prevKF) uncTinv(DT, DT_cov) Ad(T_prevKF)^T
    adjoint(M, A);
    sandwich(A, r.DT_cov, B, C);
    adjoint(s.T_prevKF, A);
    sandwich(A, C, B, D);
    for (int i = 0; i < 36; ++i) {
        s.cov_prevKF_currF[i] = add(s.cov_prevKF_currF[i], D[i]);
        A[i] = s.cov_prevKF_currF[i];
    }
    const double entropy_curr = add(k_entropy, mul(0.5, log(det6(A))));
    const double ratio = entropy_curr / s.entropy_first_prevKF;
    bool zero_cov = true, identity = true;
    for (int i = 0; i < 36; ++i) zero_cov = zero_cov && r.DT_cov[i] == 0.0;
    for (int i = 0; i < 16; ++i) identity = identity && r.DT[i] == ((i % 5 == 0) ? 1.0 : 0.0);
    const bool fire = ratio < cfg.min_entropy_ratio || isnan(ratio) || isinf(ratio) || (zero_cov && identity) ||
                      t > cfg.max_kf_t_dist || rot > cfg.max_kf_r_dist || s.N_prevKF_currF > 10;   // :1173-1175
    if (!fire) s.N_prevKF_currF++;
    PlKeyframeResult& o = out[k];
    o.new_kf = fire ? 1 : 0;
    o.N_prevKF_currF = s.N_prevKF_currF;
    o.entropy_curr = entropy_curr;
    o.entropy_ratio = ratio;
    o.t = t;
    o.r = rot;
    if (fire) {                                          // currFrameIsKF
        PlPrior& p = priors[k];
        identity4(p.Tfw);
        for (int i = 0; i < 36; ++i) p.Tfw_cov[i] = (i % 7 == 0) ? 1.0 : 0.0;
        identity4(s.T_prevKF);
        for (int i = 0; i < 36; ++i) s.cov_prevKF_currF[i] = 0.0;
        s.prev_f_iskf = 1;
        s.N_prevKF_currF = 0;
    }
}

}  // namespace

cudaError_t launch_session_keyframe(const PlKeyframeConfig& cfg, double k_entropy, int n, const PlPoseResult* results,
                                    PlKeyframeState* state, PlKeyframeResult* out, PlPrior* priors, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    session_keyframe_kernel<<<(n + 63) / 64, 64, 0, s>>>(cfg, k_entropy, n, results, state, out, priors);
    return cudaGetLastError();
}

}  // namespace plstvo
