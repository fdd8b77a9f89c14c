// gn_stream.cuh — device-side pieces of the streamed GN evaluation (optimizeFunctions, src/stereoFrameHandler.cpp:549-694, on the
// fp32-packed records): shared by the stand-alone sweep kernel (gn_stream.cu) and the per-problem GN loop of the streamed solver
// (solve.cu).  Internal; see gn_stream.cu for the record layout.
#pragma once
#include <math.h>

#include "common.cuh"

namespace plstvo {

namespace {

constexpr int GS_CONSUMERS = 256;
constexpr int GS_CWARPS = GS_CONSUMERS / 32;
constexpr int GS_THREADS = GS_CONSUMERS + 32;          // + producer warp
constexpr int GS_PT_TILE = 512;                        // points per stage (two per consumer thread)
constexpr int GS_LS_TILE = 256;                        // lines per stage (one per consumer thread)
constexpr int GS_STAGE_BYTES = 16384;
constexpr int GS_STAGES = 6;
constexpr int GS_NACC = ACC_N + 1;                     // 21 H + 6 g + e + count

// the approximate SFU forms of division and square root
__device__ __forceinline__ float gs_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float gs_sqrt(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float gs_rsqrt(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// J (+)= the 1x6 Jacobian row of :582-587 / :636-641 with the scale folded into the direction (dxs, dys)
template <bool ADD>
__device__ __forceinline__ void gs_jac(float X, float Y, float Z, float dxs, float dys, float* J) {
    const float t = fmaf(X, dxs, Y * dys), zz = Z * Z;
    const float j0 = dxs * Z, j1 = dys * Z, j3 = fmaf(Y, t, zz * dys), j4 = fmaf(X, t, zz * dxs);
    const float j5 = Z * fmaf(X, dys, -(Y * dxs));
    if (ADD) { J[0] += j0; J[1] += j1; J[2] -= t; J[3] -= j3; J[4] += j4; J[5] += j5; }
    else     { J[0] = j0;  J[1] = j1;  J[2] = -t; J[3] = -j3; J[4] = j4;  J[5] = j5; }
}

// Per-thread accumulators: 21 unique entries of H = sum w J J^T (row-major upper triangle), 6 of g = sum w r J, e, count.
struct GsAccScalar {
    float a[GS_NACC];
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int i = 0; i < GS_NACC; i++) a[i] = 0.f;
    }
    __device__ __forceinline__ void add(const float* J, float r, float w, float one) {
        int k = 0;
#pragma unroll
        for (int i = 0; i < 6; i++) {
            const float Jw = J[i] * w;
#pragma unroll
            for (int j = i; j < 6; j++) a[k] = fmaf(Jw, J[j], a[k]), k++;
            a[21 + i] = fmaf(Jw, r, a[21 + i]);
        }
        a[27] = fmaf(r * w, r, a[27]);
        a[28] += one;
    }
    __device__ __forceinline__ void unpack(float* out) const {
#pragma unroll
        for (int i = 0; i < GS_NACC; i++) out[i] = a[i];
    }
};

// :601-610 on the two parameters.  lo / hi are std::min / std::max, NaN order included: a NaN ls makes the overlap NaN, a NaN
// le is dropped (the reference then compares ls with itself).
__device__ __forceinline__ float gs_overlap_l(float ls, float le) {
    const float lo = (le < ls) ? le : ls, hi = (ls < le) ? le : ls;
    float ov = ((hi > 1.f) ? 1.f : hi) - ((lo < 0.f) ? 0.f : lo);     // covered part of [0, 1]
    ov = (hi < 0.f || lo > 1.f) ? 0.f : ov;
    return ov;
}

// StereoFrame::lineSegmentOverlap (src/stereoFrame.cpp:510-616): for a fixed previous-frame segment (su, sv)-(eu, ev) the
// parameter lambda of a projected endpoint (u, v) is affine in (u, v) in all three branches, lambda = oa u + ob v + oc; the
// coefficients are computed once per matched line when the list is built.  One exception: in the vertical branch a segment
// with ly == 0 (zero length, or |lx| < 1 and ly == 0) has lambda = (v - sv) / ly = +-inf, NaN where v == sv exactly, which no
// finite affine form reproduces.  Its coefficients are ob = 1 / ly = +-inf, oc = -sv, and lambda = ob (v + oc)
// (overlap_lambda / gs_lambda): v + (-sv) rounds exactly as v - sv does.
__device__ __forceinline__ void overlap_coeffs(double su, double sv, double eu, double ev, double& oa, double& ob,
                                               double& oc) {
    const double lx = eu - su, ly = ev - sv;
    if (fabs(su - eu) < 1.0) {          // vertical (:515-544): lambda = (v - sv) / ly
        oa = 0.0; ob = 1.0 / ly; oc = isinf(ob) ? -sv : -sv / ly;
    } else if (fabs(sv - ev) < 1.0) {   // horizontal (:545-574): lambda = (u - su) / lx
        oa = 1.0 / lx; ob = 0.0; oc = -su / lx;
    } else {                            // generic (:575-612): foot of the perpendicular, then (x - su) / lx
        const double a = sv - ev, b = eu - su, c = su * ev - eu * sv;
        const double lxy = 1.0 / (a * a + b * b);
        oa = (b * b * lxy) / lx;
        ob = (-(a * b) * lxy) / lx;
        oc = (-(a * c) * lxy - su) / lx;
    }
}
// lambda of the projected endpoint (u, v) from overlap_coeffs' coefficients
__device__ __forceinline__ double overlap_lambda(double oa, double ob, double oc, double u, double v) {
    return isinf(ob) ? ob * (v + oc) : oa * u + ob * v + oc;
}
// the same on a packed record: (oa, ob) = d.x, d.y, lam0 = the record's lambda term at the identity pose (gs_pack_line), which
// holds v0 - sv where ob is infinite; (du, dv) = the endpoint's projection change
__device__ __forceinline__ float gs_lambda(float oa, float ob, float lam0, float du, float dv) {
    return isinf(ob) ? ob * (dv + lam0) : fmaf(oa, du, fmaf(ob, dv, lam0));
}

// The pose as the evaluator holds it: r[] = the top three rows of DT with the identity taken off the rotation, (R - I | t),
// rounded to fp32 AFTER the subtraction (a frame-to-frame rotation is close to I: its difference from I keeps ~1e-9 of absolute
// accuracy in fp32, R itself only 6e-8).
struct GsPose {
    float r[12];
    float fx, fy, cx, cy, h, inv_h, fx_h;
};
__device__ __forceinline__ float gs_pose_entry(double v, int i) { return (float)((i == 0 || i == 5 || i == 10) ? v - 1.0 : v); }

// ---- records (formed once per list, in double) ------------------------------------------------------------------------------
// Every pose-independent part of a residual is evaluated in fp64 when the record is packed, at the identity pose; the kernel
// adds the pose-dependent CHANGE of the projection, which is a small quantity without cancellation:
//     u(DT) - u_obs = [fx x/z + cx - u_obs]  +  fx (dx - (x/z) dz) / (z + dz),      (dx, dy, dz) = (R - I) P + t
// (the naive fp32 form subtracts two ~1000 px numbers and carries ~2e-4 px of rounding noise into every residual; this form
// carries ~1e-5 px, which matters for the stop tests of the Gauss-Newton loop: they compare errors that differ in the 6th digit).
//   point, 32 B : {x/z, y/z, z, sqrt(sigma2)} {du0, dv0, inlier, -}                du0 = fx x/z + cx - u_obs
//   line,  64 B : {sx/sz, sy/sz, sz, sqrt(sigma2)} {ex/ez, ey/ez, ez, inlier} {l0, l1, ds0, de0} {oa, ob, lam_s0, lam_e0}
//                 ds0 = l . (projection of sP at identity, 1), lam_s0 = (oa, ob, oc) . (that projection, 1)
//                 (lam_s0 = v0 + oc = v0 - sv where ob is infinite: see overlap_coeffs)
struct GsCamD {
    double fx, fy, cx, cy;
};
__device__ __forceinline__ void gs_pack_point(const GsCamD& c, double x, double y, double z, double u, double v, double pss,
                                              bool inl, float4& A, float4& B) {
    const double xn = x / z, yn = y / z;
    A = make_float4((float)xn, (float)yn, (float)z, (float)pss);
    B = make_float4((float)(c.fx * xn + c.cx - u), (float)(c.fy * yn + c.cy - v), inl ? 1.f : 0.f, 0.f);
}
__device__ __forceinline__ void gs_pack_line(const GsCamD& c, double sx, double sy, double sz, double ex, double ey, double ez,
                                             double l0, double l1, double l2, double oa, double ob, double oc, double lss,
                                             bool inl, float4& A, float4& B, float4& C, float4& D) {
    const double sxn = sx / sz, syn = sy / sz, exn = ex / ez, eyn = ey / ez;
    const double spu = c.fx * sxn + c.cx, spv = c.fy * syn + c.cy, epu = c.fx * exn + c.cx, epv = c.fy * eyn + c.cy;
    A = make_float4((float)sxn, (float)syn, (float)sz, (float)lss);
    B = make_float4((float)exn, (float)eyn, (float)ez, inl ? 1.f : 0.f);
    C = make_float4((float)l0, (float)l1, (float)(l0 * spu + l1 * spv + l2), (float)(l0 * epu + l1 * epv + l2));
    if (isinf(ob))   // ly == 0 in the vertical branch (overlap_coeffs): the lambda terms are v0 - sv, gs_lambda scales them by ob
        D = make_float4((float)oa, (float)ob, (float)(spv + oc), (float)(epv + oc));
    else
        D = make_float4((float)oa, (float)ob, (float)(oa * spu + ob * spv + oc), (float)(oa * epu + ob * epv + oc));
}

// one 3D point through the pose: camera-frame coordinates and the change of its projection against the identity pose
struct GsProj {
    float X, Y, Z, iz, du, dv;
};
__device__ __forceinline__ GsProj gs_project(const GsPose& P, float xn, float yn, float z, bool use) {
    const float x = xn * z, y = yn * z;
    const float ddx = fmaf(P.r[0], x, fmaf(P.r[1], y, fmaf(P.r[2], z, P.r[3])));
    const float ddy = fmaf(P.r[4], x, fmaf(P.r[5], y, fmaf(P.r[6], z, P.r[7])));
    const float ddz = fmaf(P.r[8], x, fmaf(P.r[9], y, fmaf(P.r[10], z, P.r[11])));
    GsProj q;
    q.X = x + ddx; q.Y = y + ddy; q.Z = z + ddz;
    q.iz = use ? gs_rcp(q.Z) : 0.f;                      // a dead record contributes exact zeros, never a NaN
    q.du = P.fx * fmaf(-xn, ddz, ddx) * q.iz;
    q.dv = P.fy * fmaf(-yn, ddz, ddy) * q.iz;
    return q;
}

// point block (:563-606); `use` = a live record flagged inlier
template <class Acc>
__device__ __forceinline__ void gs_point(const GsPose& P, const float4 a, const float4 b, bool use, Acc& acc) {
    const GsProj q = gs_project(P, a.x, a.y, a.z, use);
    const float dx = b.x + q.du, dy = b.y + q.dv;
    const float ss = fmaf(dx, dx, dy * dy);
    const float n = gs_sqrt(ss), inv = fminf(P.inv_h, gs_rsqrt(ss));          // 1 / max(homogTh, n)
    const float fg = (q.Z * q.Z > P.h) ? P.fx * q.iz * q.iz : P.fx_h;          // fx / max(homogTh, Z^2)  (:577)
    const float sc = fg * inv;
    float J[6];
    gs_jac<false>(q.X, q.Y, q.Z, sc * dx, sc * dy, J);
    const float r = n * a.w;
    const float w = use ? gs_rcp(fmaf(r, r, 1.f)) : 0.f;
    acc.add(J, r, w, use ? 1.f : 0.f);
}

// line block (:610-684)
template <class Acc>
__device__ __forceinline__ void gs_line(const GsPose& P, const float4 a, const float4 b, const float4 c, const float4 d,
                                        bool use, Acc& acc) {
    const GsProj s = gs_project(P, a.x, a.y, a.z, use), e = gs_project(P, b.x, b.y, b.z, use);
    const float ds = fmaf(c.x, s.du, fmaf(c.y, s.dv, c.z)), de = fmaf(c.x, e.du, fmaf(c.y, e.dv, c.w));
    const float ss = fmaf(ds, ds, de * de);
    const float n = gs_sqrt(ss), iden = fminf(P.inv_h, gs_rsqrt(ss));
    const float ks = ((s.Z * s.Z > P.h) ? P.fx * s.iz * s.iz : P.fx_h) * (ds * iden);
    const float ke = ((e.Z * e.Z > P.h) ? P.fx * e.iz * e.iz : P.fx_h) * (de * iden);
    float J[6];
    gs_jac<false>(s.X, s.Y, s.Z, ks * c.x, ks * c.y, J);
    gs_jac<true>(e.X, e.Y, e.Z, ke * c.x, ke * c.y, J);
    const float r = n * a.w;
    float w = gs_rcp(fmaf(r, r, 1.f));
    w *= gs_overlap_l(gs_lambda(d.x, d.y, d.z, s.du, s.dv), gs_lambda(d.x, d.y, d.w, e.du, e.dv));   // :664-670
    acc.add(J, r, use ? w : 0.f, use ? 1.f : 0.f);
}

}  // namespace

}  // namespace plstvo
