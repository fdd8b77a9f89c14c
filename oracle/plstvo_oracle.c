/*
 * plstvo_oracle.c — CPU ORACLE (test infrastructure, see plstvo_oracle.h for the rules and
 * the parity-pinning statement).  Plain C restatement of the reference's frame-to-frame path;
 * every function cites the reference lines it follows (paths relative to rubengooj/stvo-pl).
 */
#define _GNU_SOURCE
#include "plstvo_oracle.h"

#include <float.h>
#include <limits.h>
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------------------------------
 * small dense helpers (row-major)
 * ---------------------------------------------------------------------------------------------- */
static void mat4_identity(double T[16]) {
    memset(T, 0, 16 * sizeof(double));
    T[0] = T[5] = T[10] = T[15] = 1.0;
}
static void mat4_mul(const double A[16], const double B[16], double C[16]) {
    double R[16];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double s = 0.0;
            for (int k = 0; k < 4; k++) s += A[i * 4 + k] * B[k * 4 + j];
            R[i * 4 + j] = s;
        }
    memcpy(C, R, sizeof(R));
}
static int mat4_is_identity(const double T[16]) { /* `DT != Matrix4d::Identity()` — exact compare */
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            if (T[i * 4 + j] != (i == j ? 1.0 : 0.0)) return 0;
    return 1;
}
static void mat3_mul(const double A[9], const double B[9], double C[9]) {
    double R[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0.0;
            for (int k = 0; k < 3; k++) s += A[i * 3 + k] * B[k * 3 + j];
            R[i * 3 + j] = s;
        }
    memcpy(C, R, sizeof(R));
}
/* src/auxiliar.cpp:29-44 */
static void skew3(const double v[3], double S[9]) {
    S[0] = 0;      S[1] = -v[2];  S[2] = v[1];
    S[3] = v[2];   S[4] = 0;      S[5] = -v[0];
    S[6] = -v[1];  S[7] = v[0];   S[8] = 0;
}
/* Eigen computes a fixed-size 3x3 inverse by cofactors */
static void mat3_inverse(const double A[9], double Ainv[9]) {
    double c00 = A[4] * A[8] - A[5] * A[7];
    double c01 = A[5] * A[6] - A[3] * A[8];
    double c02 = A[3] * A[7] - A[4] * A[6];
    double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
    double id = 1.0 / det;
    Ainv[0] = c00 * id;
    Ainv[1] = (A[2] * A[7] - A[1] * A[8]) * id;
    Ainv[2] = (A[1] * A[5] - A[2] * A[4]) * id;
    Ainv[3] = c01 * id;
    Ainv[4] = (A[0] * A[8] - A[2] * A[6]) * id;
    Ainv[5] = (A[2] * A[3] - A[0] * A[5]) * id;
    Ainv[6] = c02 * id;
    Ainv[7] = (A[1] * A[6] - A[0] * A[7]) * id;
    Ainv[8] = (A[0] * A[4] - A[1] * A[3]) * id;
}

/* ------------------------------------------------------------------------------------------------
 * SE(3) helpers — src/auxiliar.cpp
 * ---------------------------------------------------------------------------------------------- */
void orc_inverse_se3(const double T[16], double Tinv[16]) { /* :113-122 */
    double R[9], t[3];
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) R[i * 3 + j] = T[i * 4 + j];
        t[i] = T[i * 4 + 3];
    }
    double out[16];
    mat4_identity(out);
    for (int i = 0; i < 3; i++) {
        double s = 0.0;
        for (int j = 0; j < 3; j++) {
            out[i * 4 + j] = R[j * 3 + i];
            s += R[j * 3 + i] * t[j];
        }
        out[i * 4 + 3] = -s;
    }
    memcpy(Tinv, out, sizeof(out));
}

void orc_expmap_se3(const double x[6], double T[16]) { /* :124-141, x = [t; w] */
    double w[3] = {x[3], x[4], x[5]};
    double t[3] = {x[0], x[1], x[2]};
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    if (!(theta < 0.000001)) {
        double s[9], ss[9], wn[3] = {w[0] / theta, w[1] / theta, w[2] / theta};
        skew3(wn, s); /* skew(w)/theta: every entry is +-w_i/theta */
        mat3_mul(s, s, ss);
        double sn = sin(theta), cs = cos(theta);
        double V[9];
        for (int i = 0; i < 9; i++) {
            double I = (i % 4 == 0) ? 1.0 : 0.0;
            R[i] = I + s[i] * sn + ss[i] * (1.0 - cs);
            V[i] = I + s[i] * (1.0 - cs) / theta + ss[i] * (theta - sn) / theta;
        }
        double tv[3];
        for (int i = 0; i < 3; i++) tv[i] = V[i * 3] * t[0] + V[i * 3 + 1] * t[1] + V[i * 3 + 2] * t[2];
        memcpy(t, tv, sizeof(tv));
    }
    mat4_identity(T);
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) T[i * 4 + j] = R[i * 3 + j];
        T[i * 4 + 3] = t[i];
    }
}

void orc_logmap_se3(const double T[16], double x[6]) { /* :143-173 */
    double R[9], Vt[3], w[3] = {0, 0, 0};
    double V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) R[i * 3 + j] = T[i * 4 + j];
        Vt[i] = T[i * 4 + 3];
    }
    double cosine = (R[0] + R[4] + R[8] - 1.0) / 2.0;
    if (cosine > 1.0) cosine = 1.0;
    else if (cosine < -1.0) cosine = -1.0;
    double sine = sqrt(1.0 - cosine * cosine);
    if (sine > 1.0) sine = 1.0;
    else if (sine < -1.0) sine = -1.0;
    double theta = acos(cosine);
    if (theta > 0.000001) {
        double w_hat[9];
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++)
                w_hat[i * 3 + j] = theta * (R[i * 3 + j] - R[j * 3 + i]) / (2.0 * sine);
        w[0] = w_hat[2 * 3 + 1]; /* skewcoords: M(2,1), M(0,2), M(1,0)  (:58-62) */
        w[1] = w_hat[0 * 3 + 2];
        w[2] = w_hat[1 * 3 + 0];
        double s[9], ss[9], wn[3] = {w[0] / theta, w[1] / theta, w[2] / theta};
        skew3(wn, s);
        mat3_mul(s, s, ss);
        for (int i = 0; i < 9; i++) {
            double I = (i % 4 == 0) ? 1.0 : 0.0;
            V[i] = I + s[i] * (1.0 - cosine) / theta + ss[i] * (theta - sine) / theta;
        }
    }
    double Vi[9];
    mat3_inverse(V, Vi);
    for (int i = 0; i < 3; i++) x[i] = Vi[i * 3] * Vt[0] + Vi[i * 3 + 1] * Vt[1] + Vi[i * 3 + 2] * Vt[2];
    x[3] = w[0];
    x[4] = w[1];
    x[5] = w[2];
}

void orc_adjoint_se3(const double T[16], double Ad[36]) { /* :175-182 */
    double R[9], t[3], S[9], SR[9];
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) R[i * 3 + j] = T[i * 4 + j];
        t[i] = T[i * 4 + 3];
    }
    skew3(t, S);
    mat3_mul(S, R, SR);
    memset(Ad, 0, 36 * sizeof(double));
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            Ad[i * 6 + j] = R[i * 3 + j];
            Ad[i * 6 + 3 + j] = SR[i * 3 + j];
            Ad[(i + 3) * 6 + 3 + j] = R[i * 3 + j];
        }
}

void orc_unccomp_se3(const double T1[16], const double c1[36], const double cinc[36], double out[36]) { /* :192-197 */
    double Ad[36], tmp[36];
    orc_adjoint_se3(T1, Ad);
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) {
            double s = 0.0;
            for (int k = 0; k < 6; k++) s += Ad[i * 6 + k] * cinc[k * 6 + j];
            tmp[i * 6 + j] = s;
        }
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) {
            double s = 0.0;
            for (int k = 0; k < 6; k++) s += tmp[i * 6 + k] * Ad[j * 6 + k];
            out[i * 6 + j] = c1[i * 6 + j] + s;
        }
}

int orc_is_finite(const double* x, int n) { /* :353-355: ((x-x) == (x-x)).all() */
    for (int i = 0; i < n; i++) {
        double d = x[i] - x[i];
        if (!(d == d)) return 0;
    }
    return 1;
}

/* ------------------------------------------------------------------------------------------------
 * robust statistics — src/auxiliar.cpp
 * ---------------------------------------------------------------------------------------------- */
static int cmp_double(const void* a, const void* b) {
    double x = *(const double*)a, y = *(const double*)b;
    return (x > y) - (x < y);
}

void orc_vector_mean_stdv_mad(const double* res, int n, double* mean, double* stdv) { /* :387-430 */
    *mean = 0.0;
    *stdv = 0.0;
    if (n == 0) return;
    double* r = (double*)malloc((size_t)n * sizeof(double));
    memcpy(r, res, (size_t)n * sizeof(double));
    qsort(r, (size_t)n, sizeof(double), cmp_double);
    double median = r[n / 2];
    for (int i = 0; i < n; i++) r[i] = (double)fabsf((float)(r[i] - median)); /* fabsf: float rounding (:400) */
    qsort(r, (size_t)n, sizeof(double), cmp_double);
    *stdv = 1.4826 * r[n / 2];
    int k = 0;
    double m = 0.0;
    for (int i = 0; i < n; i++)
        if (res[i] < 2.0 * (*stdv)) {
            m += res[i];
            k++;
        }
    if (k >= (int)(0.2 * (double)n))
        m /= (double)k; /* k == 0 can only pass when int(0.2 n) == 0: 0/0 = NaN like the reference */
    else {
        k = 0;
        m = 0.0;
        for (int i = 0; i < n; i++) {
            m += res[i];
            k++;
        }
        m /= (double)k;
    }
    *mean = m;
    free(r);
}

double orc_vector_stdv_mad(const double* res, int n) { /* :444-460 */
    if (n == 0) return 0.0;
    double* r = (double*)malloc((size_t)n * sizeof(double));
    memcpy(r, res, (size_t)n * sizeof(double));
    qsort(r, (size_t)n, sizeof(double), cmp_double);
    double median = r[n / 2];
    for (int i = 0; i < n; i++) r[i] = (double)fabsf((float)(r[i] - median));
    qsort(r, (size_t)n, sizeof(double), cmp_double);
    double mad = r[n / 2];
    free(r);
    return 1.4826 * mad;
}

double orc_robust_weight_cauchy(double r) { return 1.0 / (1.0 + r * r); } /* :556-559 */

/* ------------------------------------------------------------------------------------------------
 * camera — src/pinholeStereoCamera.cpp
 * ---------------------------------------------------------------------------------------------- */
void orc_projection(const PlCamera* cam, const double P[3], double uv[2]) { /* :231-237 */
    uv[0] = cam->cx + cam->fx * P[0] / P[2];
    uv[1] = cam->cy + cam->fy * P[1] / P[2];
}
void orc_back_projection(const PlCamera* cam, double u, double v, double disp, double P[3]) { /* :221-229 */
    double bd = cam->b / disp;
    P[0] = bd * (u - cam->cx);
    P[1] = bd * (v - cam->cy);
    P[2] = bd * cam->fx;
}

/* ------------------------------------------------------------------------------------------------
 * StereoFrame::lineSegmentOverlap — src/stereoFrame.cpp:510-616
 * ---------------------------------------------------------------------------------------------- */
static double overlap_from_lambdas(double lambda_s, double lambda_e) { /* :531-541 et al. */
    double lambda_min = (lambda_e < lambda_s) ? lambda_e : lambda_s; /* std::min(a,b) = (b<a)?b:a */
    double lambda_max = (lambda_s < lambda_e) ? lambda_e : lambda_s; /* std::max(a,b) = (a<b)?b:a */
    double overlap;
    if (lambda_min < 0.0 && lambda_max > 1.0) overlap = 1.0;
    else if (lambda_max < 0.0 || lambda_min > 1.0) overlap = 0.0;
    else if (lambda_min < 0.0) overlap = lambda_max;
    else if (lambda_max > 1.0) overlap = 1.0 - lambda_min;
    else overlap = lambda_max - lambda_min;
    return overlap;
}

double orc_line_segment_overlap(const double spl_obs[2], const double epl_obs[2],
                                const double spl_proj[2], const double epl_proj[2]) {
    double lx = epl_obs[0] - spl_obs[0], ly = epl_obs[1] - spl_obs[1];
    if (fabs(spl_obs[0] - epl_obs[0]) < 1.0) { /* vertical (:515-544) */
        double lambda_s = (spl_proj[1] - spl_obs[1]) / ly;
        double lambda_e = (epl_proj[1] - spl_obs[1]) / ly;
        return overlap_from_lambdas(lambda_s, lambda_e);
    } else if (fabs(spl_obs[1] - epl_obs[1]) < 1.0) { /* horizontal (:545-574) */
        double lambda_s = (spl_proj[0] - spl_obs[0]) / lx;
        double lambda_e = (epl_proj[0] - spl_obs[0]) / lx;
        return overlap_from_lambdas(lambda_s, lambda_e);
    } else { /* generic (:575-612) */
        double a = spl_obs[1] - epl_obs[1];
        double b = epl_obs[0] - spl_obs[0];
        double c = spl_obs[0] * epl_obs[1] - epl_obs[0] * spl_obs[1];
        double lxy = 1.0 / (a * a + b * b);
        double sx = (b * (b * spl_proj[0] - a * spl_proj[1]) - a * c) * lxy;
        double ex = (b * (b * epl_proj[0] - a * epl_proj[1]) - a * c) * lxy;
        double lambda_s = (sx - spl_obs[0]) / lx;
        double lambda_e = (ex - spl_obs[0]) / lx;
        return overlap_from_lambdas(lambda_s, lambda_e);
    }
}

/* ------------------------------------------------------------------------------------------------
 * Eigen pieces restated (agree with Eigen to rounding)
 * ---------------------------------------------------------------------------------------------- */
/* ColPivHouseholderQR<Matrix6d>(H).solve(g) and logAbsDeterminant()
 * (src/stereoFrameHandler.cpp:417-418, :453-455).  Column-pivoted Householder QR, rank decided with
 * Eigen's default threshold (eps * 6 relative to the largest pivot).  Returns the rank. */
int orc_qr6_solve(const double H[36], const double g[6], double x[6], double* log_abs_det) {
    double A[36], c[6];
    int perm[6];
    memcpy(A, H, sizeof(A));
    memcpy(c, g, sizeof(c));
    for (int j = 0; j < 6; j++) perm[j] = j;
    double maxpivot = 0.0;
    for (int k = 0; k < 6; k++) {
        /* pivot: remaining column with the largest norm below row k */
        int best = k;
        double bestn = -1.0;
        for (int j = k; j < 6; j++) {
            double s = 0.0;
            for (int i = k; i < 6; i++) s += A[i * 6 + j] * A[i * 6 + j];
            if (s > bestn) { bestn = s; best = j; }
        }
        if (best != k) {
            for (int i = 0; i < 6; i++) { double t = A[i * 6 + k]; A[i * 6 + k] = A[i * 6 + best]; A[i * 6 + best] = t; }
            int t = perm[k]; perm[k] = perm[best]; perm[best] = t;
        }
        /* Householder vector for column k, rows k..5 (Eigen makeHouseholderInPlace convention) */
        double tail = 0.0;
        for (int i = k + 1; i < 6; i++) tail += A[i * 6 + k] * A[i * 6 + k];
        double c0 = A[k * 6 + k], beta, tau;
        double v[6] = {0, 0, 0, 0, 0, 0};
        if (tail <= DBL_MIN) {
            tau = 0.0;
            beta = c0;
        } else {
            beta = sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            for (int i = k + 1; i < 6; i++) v[i] = A[i * 6 + k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        v[k] = 1.0;
        /* apply (I - tau v v^T) to the trailing columns and to the right-hand side */
        for (int j = k + 1; j < 6; j++) {
            double s = 0.0;
            for (int i = k; i < 6; i++) s += v[i] * A[i * 6 + j];
            s *= tau;
            for (int i = k; i < 6; i++) A[i * 6 + j] -= s * v[i];
        }
        {
            double s = 0.0;
            for (int i = k; i < 6; i++) s += v[i] * c[i];
            s *= tau;
            for (int i = k; i < 6; i++) c[i] -= s * v[i];
        }
        A[k * 6 + k] = beta;
        for (int i = k + 1; i < 6; i++) A[i * 6 + k] = 0.0;
        if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
    }
    int rank = 0;
    double thr = maxpivot * (DBL_EPSILON * 6.0);
    double lad = 0.0;
    for (int k = 0; k < 6; k++) {
        if (fabs(A[k * 6 + k]) > thr) rank++;
        lad += log(fabs(A[k * 6 + k]));
    }
    if (log_abs_det) *log_abs_det = lad;
    double y[6] = {0, 0, 0, 0, 0, 0};
    for (int k = rank - 1; k >= 0; k--) {
        double s = c[k];
        for (int j = k + 1; j < rank; j++) s -= A[k * 6 + j] * y[j];
        y[k] = s / A[k * 6 + k];
    }
    for (int k = 0; k < 6; k++) x[perm[k]] = y[k];
    return rank;
}

/* Matrix6d::inverse() — Eigen uses PartialPivLU for dynamic/large fixed sizes
 * (src/stereoFrameHandler.cpp:429, :470) */
void orc_inv6(const double Ain[36], double Ainv[36]) {
    double A[36], B[36];
    memcpy(A, Ain, sizeof(A));
    memset(B, 0, sizeof(B));
    for (int i = 0; i < 6; i++) B[i * 6 + i] = 1.0;
    for (int k = 0; k < 6; k++) {
        int piv = k;
        double big = fabs(A[k * 6 + k]);
        for (int i = k + 1; i < 6; i++)
            if (fabs(A[i * 6 + k]) > big) { big = fabs(A[i * 6 + k]); piv = i; }
        if (piv != k)
            for (int j = 0; j < 6; j++) {
                double t = A[k * 6 + j]; A[k * 6 + j] = A[piv * 6 + j]; A[piv * 6 + j] = t;
                t = B[k * 6 + j]; B[k * 6 + j] = B[piv * 6 + j]; B[piv * 6 + j] = t;
            }
        double d = A[k * 6 + k];
        for (int i = k + 1; i < 6; i++) {
            double f = A[i * 6 + k] / d;
            A[i * 6 + k] = 0.0;
            for (int j = k + 1; j < 6; j++) A[i * 6 + j] -= f * A[k * 6 + j];
            for (int j = 0; j < 6; j++) B[i * 6 + j] -= f * B[k * 6 + j];
        }
    }
    for (int j = 0; j < 6; j++)
        for (int i = 5; i >= 0; i--) {
            double s = B[i * 6 + j];
            for (int k = i + 1; k < 6; k++) s -= A[i * 6 + k] * Ainv[k * 6 + j];
            Ainv[i * 6 + j] = s / A[i * 6 + i];
        }
}

/* SelfAdjointEigenSolver<Matrix6d>::eigenvalues(): reads the LOWER triangle, ascending
 * (src/stereoFrameHandler.cpp:294-295, :379-380).  Cyclic Jacobi. */
void orc_eig6_sym(const double Ain[36], double w[6]) {
    double A[36];
    for (int i = 0; i < 6; i++)
        for (int j = 0; j <= i; j++) A[i * 6 + j] = A[j * 6 + i] = Ain[i * 6 + j];
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < 6; i++) {
            diag += A[i * 6 + i] * A[i * 6 + i];
            for (int j = 0; j < i; j++) off += 2.0 * A[i * 6 + j] * A[i * 6 + j];
        }
        if (!(off > 1e-30 * diag) || off == 0.0) break;   /* off-diagonal mass at rounding level: eigenvalues settled to ~1e-15 */
        for (int p = 0; p < 5; p++)
            for (int q = p + 1; q < 6; q++) {
                double apq = A[p * 6 + q];
                if (apq == 0.0) continue;
                double app = A[p * 6 + p], aqq = A[q * 6 + q];
                double tau = (aqq - app) / (2.0 * apq);
                double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
                double cs = 1.0 / sqrt(1.0 + t * t), sn = t * cs;
                for (int k = 0; k < 6; k++) { /* columns p,q */
                    double akp = A[k * 6 + p], akq = A[k * 6 + q];
                    A[k * 6 + p] = cs * akp - sn * akq;
                    A[k * 6 + q] = sn * akp + cs * akq;
                }
                for (int k = 0; k < 6; k++) { /* rows p,q */
                    double apk = A[p * 6 + k], aqk = A[q * 6 + k];
                    A[p * 6 + k] = cs * apk - sn * aqk;
                    A[q * 6 + k] = sn * apk + cs * aqk;
                }
            }
    }
    for (int i = 0; i < 6; i++) w[i] = A[i * 6 + i];
    qsort(w, 6, sizeof(double), cmp_double);
    /* NaN input: the sweep test above is false for a NaN off-diagonal mass, so the loop stops at once and w is A's
     * diagonal, which can be finite; the gate below then judges that diagonal.  qsort leaves NaN entries in an arbitrary
     * order, and a NaN w[0] or w[5] passes the gate (both comparisons false).  The device's Jacobi does the same
     * (solve.cu: warp_eig6_sym).  This is NOT what Eigen's solver does with a NaN entry (DESIGN.md §3). */
}

/* ------------------------------------------------------------------------------------------------
 * matching — src/matching.cpp
 * ---------------------------------------------------------------------------------------------- */
int orc_distance(const uint8_t* a, const uint8_t* b) { /* :93-109, SWAR popcount over 8 x int32 */
    int dist = 0;
    for (int i = 0; i < 8; i++) {
        uint32_t pa, pb;
        memcpy(&pa, a + 4 * i, 4);
        memcpy(&pb, b + 4 * i, 4);
        uint32_t v = pa ^ pb;
        v = v - ((v >> 1) & 0x55555555u);
        v = (v & 0x33333333u) + ((v >> 2) & 0x33333333u);
        dist += (int)((((v + (v >> 4)) & 0xF0F0F0Fu) * 0x1010101u) >> 24);
    }
    return dist;
}

/* Hamming norm the way OpenCV's normHamming does it (hardware popcount), used inside knnMatch */
static inline int hamming256(const uint8_t* a, const uint8_t* b) {
    uint64_t x[4], y[4];
    memcpy(x, a, 32);
    memcpy(y, b, 32);
    return __builtin_popcountll(x[0] ^ y[0]) + __builtin_popcountll(x[1] ^ y[1]) +
           __builtin_popcountll(x[2] ^ y[2]) + __builtin_popcountll(x[3] ^ y[3]);
}

/* cv::BFMatcher(NORM_HAMMING,false)::knnMatch(d1, d2, ., 2) -> cv::batchDistance with K = 2
 * (third-party: OpenCV features2d/core, not under /root/reference; call site src/matching.cpp:47-48).
 * Published algorithm: for each query row the integer distances to all train rows are scanned in
 * ascending train index and inserted into a K-long list kept sorted by strict `<` comparisons, so
 * the list ends up ordered by (distance, trainIdx) ascending. */
void orc_knn2(const uint8_t* d1, int n1, const uint8_t* d2, int n2, int32_t* idx, int32_t* dist) {
    for (int i = 0; i < n1; i++) {
        int bd[2] = {INT_MAX, INT_MAX}, bi[2] = {-1, -1};
        const uint8_t* q = d1 + (size_t)i * 32;
        for (int j = 0; j < n2; j++) {
            int d = hamming256(q, d2 + (size_t)j * 32);
            if (d < bd[1]) {
                int k = 0; /* insertion position */
                if (!(bd[0] > d)) k = 1;
                if (k == 0) { bd[1] = bd[0]; bi[1] = bi[0]; }
                bd[k] = d;
                bi[k] = j;
            }
        }
        idx[2 * i] = bi[0];
        idx[2 * i + 1] = bi[1];
        dist[2 * i] = bi[0] >= 0 ? bd[0] : -1;
        dist[2 * i + 1] = bi[1] >= 0 ? bd[1] : -1;
    }
}

int orc_match_nnr(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnr, int32_t* m12) { /* :41-61 */
    int matches = 0;
    for (int i = 0; i < n1; i++) m12[i] = -1; /* matches_12.resize(desc1.rows, -1) (:44) */
    if (n1 <= 0) return 0;
    if (n2 < 2) return 0; /* reference: matches_[idx][1] out of range (UB); defined here as "no match" */
    int32_t* idx = (int32_t*)malloc((size_t)n1 * 2 * sizeof(int32_t));
    int32_t* dist = (int32_t*)malloc((size_t)n1 * 2 * sizeof(int32_t));
    orc_knn2(d1, n1, d2, n2, idx, dist);
    for (int i = 0; i < n1; i++) {
        float dd0 = (float)dist[2 * i], dd1 = (float)dist[2 * i + 1]; /* DMatch::distance is float */
        if (dd0 < dd1 * nnr) { /* float multiply, :54 */
            m12[i] = idx[2 * i];
            matches++;
        }
    }
    free(idx);
    free(dist);
    return matches;
}

typedef struct {
    const uint8_t *d1, *d2;
    int n1, n2;
    float nnr;
    int32_t* out;
    int ret;
} NnrJob;
static void* nnr_thread(void* p) {
    NnrJob* j = (NnrJob*)p;
    j->ret = orc_match_nnr(j->d1, j->n1, j->d2, j->n2, j->nnr, j->out);
    return NULL;
}

int orc_match(const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnr, int best_lr,
              int threads, int32_t* m12) { /* :63-91 */
    if (!best_lr) return orc_match_nnr(d1, n1, d2, n2, nnr, m12);
    int32_t* m21 = (int32_t*)malloc((size_t)(n2 > 0 ? n2 : 1) * sizeof(int32_t));
    int matches;
    if (threads) { /* lrInParallel: two std::async tasks (:68-74) */
        NnrJob a = {d1, d2, n1, n2, nnr, m12, 0}, b = {d2, d1, n2, n1, nnr, m21, 0};
        pthread_t tb;
        pthread_create(&tb, NULL, nnr_thread, &b);
        nnr_thread(&a);
        pthread_join(tb, NULL);
        matches = a.ret;
    } else {
        matches = orc_match_nnr(d1, n1, d2, n2, nnr, m12);
        orc_match_nnr(d2, n2, d1, n1, nnr, m21);
    }
    for (int i1 = 0; i1 < n1; i1++) { /* :80-86 */
        int i2 = m12[i1];
        if (i2 >= 0 && m21[i2] != i1) {
            m12[i1] = -1;
            matches--;
        }
    }
    free(m21);
    return matches;
}

/* ------------------------------------------------------------------------------------------------
 * StVO::matchGrid — the stereo (left/right) step, SURVEY 8(f)-1
 * ---------------------------------------------------------------------------------------------- */
typedef struct {   /* GridStructure: cols x rows lists of train indices (src/gridStructure.cpp:43-63) */
    int rows, cols;
    int* head;     /* [cols*rows] first entry of the cell's list or -1 */
    int* next;     /* linked entries */
    int* item;
    int n, cap;
} OrcGrid;

static void grid_init(OrcGrid* g, int rows, int cols, int cap) {
    g->rows = rows;
    g->cols = cols;
    g->head = (int*)malloc((size_t)rows * cols * sizeof(int));
    for (int i = 0; i < rows * cols; i++) g->head[i] = -1;
    g->cap = cap > 0 ? cap : 1;
    g->next = (int*)malloc((size_t)g->cap * sizeof(int));
    g->item = (int*)malloc((size_t)g->cap * sizeof(int));
    g->n = 0;
}
static void grid_free(OrcGrid* g) { free(g->head); free(g->next); free(g->item); }
static void grid_push(OrcGrid* g, int x, int y, int idx) {   /* grid.at(x, y).push_back(idx); out of bounds -> discarded list */
    if (!(x >= 0 && x < g->cols && y >= 0 && y < g->rows)) return;
    if (g->n == g->cap) {
        g->cap *= 2;
        g->next = (int*)realloc(g->next, (size_t)g->cap * sizeof(int));
        g->item = (int*)realloc(g->item, (size_t)g->cap * sizeof(int));
    }
    g->item[g->n] = idx;
    g->next[g->n] = g->head[x * g->rows + y];
    g->head[x * g->rows + y] = g->n++;
}
/* GridStructure::get (src/gridStructure.cpp:65-76): union of the cells of the window into a set (stamp = dedupe) */
static int grid_get(const OrcGrid* g, int x, int y, PlGridWindow w, int* stamp, int tag, int* out, int n_out) {
    int min_x = x - w.left > 0 ? x - w.left : 0;
    int max_x = x + w.right + 1 < g->cols ? x + w.right + 1 : g->cols;
    int min_y = y - w.up > 0 ? y - w.up : 0;
    int max_y = y + w.down + 1 < g->rows ? y + w.down + 1 : g->rows;
    for (int x_ = min_x; x_ < max_x; ++x_)
        for (int y_ = min_y; y_ < max_y; ++y_)
            for (int e = g->head[x_ * g->rows + y_]; e >= 0; e = g->next[e]) {
                int i2 = g->item[e];
                if (stamp[i2] != tag) {
                    stamp[i2] = tag;
                    out[n_out++] = i2;
                }
            }
    return n_out;
}

int orc_line_cells(double x1, double y1, double x2, double y2, int32_t* cells, int cap) { /* src/lineIterator.cpp:34-77 */
    int steep = fabs(y2 - y1) > fabs(x2 - x1);
    if (steep) { double t = x1; x1 = y1; y1 = t; t = x2; x2 = y2; y2 = t; }
    if (x1 > x2) { double t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    double dx = x2 - x1, dy = fabs(y2 - y1), error = dx / 2.0;
    int ystep = (y1 < y2) ? 1 : -1;
    int x = (int)x1, y = (int)y1, maxX = (int)x2, n = 0;
    while (!(x > maxX)) {
        if (n < cap) {
            cells[2 * n] = steep ? y : x;
            cells[2 * n + 1] = steep ? x : y;
        }
        n++;
        error -= dy;
        if (error < 0) { y += ystep; error += dx; }
        x++;
    }
    return n;
}

/* shared tail of both overloads: candidate loop (:139-158 / :214-239), ratio test (:160 / :241), mutual filter (:166-174) */
static int match_grid_core(int n1, int n2, const uint8_t* d1, const uint8_t* d2, int best_lr, double ratio,
                           const OrcGrid* g, PlGridWindow w, const int32_t* q_cells, int cells_per_query,
                           const double* dirs2, double line_sim_th, int32_t* m12) {
    int matches = 0;
    for (int i = 0; i < n1; i++) m12[i] = -1;
    int* matches_21 = (int*)malloc((size_t)(n2 + 1) * sizeof(int));
    int* distances = (int*)malloc((size_t)(n2 + 1) * sizeof(int));
    int* stamp = (int*)malloc((size_t)(n2 + 1) * sizeof(int));
    int* cand = (int*)malloc((size_t)(n2 + 1) * sizeof(int));
    for (int i = 0; i < n2; i++) { matches_21[i] = -1; distances[i] = INT_MAX; stamp[i] = -1; }
    for (int i1 = 0; i1 < n1; ++i1) {
        int best_d = INT_MAX, best_d2 = INT_MAX, best_idx = -1;
        const int32_t* c = q_cells + (size_t)i1 * 2 * cells_per_query;
        double vx = 0, vy = 0;
        if (cells_per_query == 2) {   /* v = normalize(ep - sp) in INTEGER cell coordinates (:207-211): NaN when equal */
            vx = (double)(c[2] - c[0]);
            vy = (double)(c[3] - c[1]);
            double mag = sqrt(vx * vx + vy * vy);
            vx /= mag;
            vy /= mag;
        }
        int nc = 0;
        for (int k = 0; k < cells_per_query; k++) nc = grid_get(g, c[2 * k], c[2 * k + 1], w, stamp, i1, cand, nc);
        if (nc == 0) continue;
        for (int k = 0; k < nc; k++) {
            int i2 = cand[k];
            if (i2 < 0 || i2 >= n2) continue;
            if (cells_per_query == 2) {
                double dt = vx * dirs2[2 * i2] + vy * dirs2[2 * i2 + 1];
                if (fabs(dt) < line_sim_th) continue;   /* NaN passes (:221) */
            }
            int d = orc_distance(d1 + (size_t)i1 * 32, d2 + (size_t)i2 * 32);
            if (best_lr) {
                if (d < distances[i2]) {
                    distances[i2] = d;
                    matches_21[i2] = i1;
                } else
                    continue;
            }
            if (d < best_d) {
                best_d2 = best_d;
                best_d = d;
                best_idx = i2;
            } else if (d < best_d2)
                best_d2 = d;
        }
        if ((double)best_d < (double)best_d2 * ratio) {   /* int * double (:160) */
            m12[i1] = best_idx;
            matches++;
        }
    }
    if (best_lr)
        for (int i1 = 0; i1 < n1; ++i1) {
            int i2 = m12[i1];
            if (i2 >= 0 && matches_21[i2] != i1) {
                m12[i1] = -1;
                matches--;
            }
        }
    free(matches_21); free(distances); free(stamp); free(cand);
    return matches;
}

int orc_match_grid_points(int rows, int cols, PlGridWindow w, int best_lr, double ratio, const int32_t* q_cell,
                          const uint8_t* d1, int n1, const int32_t* t_cell, const uint8_t* d2, int n2, int32_t* m12) {
    OrcGrid g;
    grid_init(&g, rows, cols, n2);
    for (int idx = 0; idx < n2; ++idx) grid_push(&g, t_cell[2 * idx], t_cell[2 * idx + 1], idx);   /* stereoFrame.cpp:135-139 */
    int r = match_grid_core(n1, n2, d1, d2, best_lr, ratio, &g, w, q_cell, 1, NULL, 0.0, m12);
    grid_free(&g);
    return r;
}

int orc_match_grid_lines(int rows, int cols, PlGridWindow w, int best_lr, double ratio, double line_sim_th,
                         const int32_t* q_line, const uint8_t* d1, int n1, const double* t_line, const double* t_dir,
                         const uint8_t* d2, int n2, int32_t* m12) {
    OrcGrid g;
    grid_init(&g, rows, cols, 4 * n2 + 16);
    int cap = 4 * (rows + cols) + 16;
    int32_t* cells = (int32_t*)malloc((size_t)cap * 2 * sizeof(int32_t));
    for (int idx = 0; idx < n2; ++idx) {   /* stereoFrame.cpp:329-339 */
        int n = orc_line_cells(t_line[4 * idx], t_line[4 * idx + 1], t_line[4 * idx + 2], t_line[4 * idx + 3], cells, cap);
        if (n > cap) n = cap;
        for (int k = 0; k < n; k++) grid_push(&g, cells[2 * k], cells[2 * k + 1], idx);
    }
    int r = match_grid_core(n1, n2, d1, d2, best_lr, ratio, &g, w, q_line, 2, t_dir, line_sim_th, m12);
    free(cells);
    grid_free(&g);
    return r;
}

/* ------------------------------------------------------------------------------------------------
 * 3-D lifting of the stereo matches — SURVEY 8(f)-2
 * ---------------------------------------------------------------------------------------------- */
static double sigma2_of_level(int level, double scale) {   /* PointFeature / LineFeature ctors (src/stereoFeatures.cpp:41-47, :107-115) */
    double sigma2 = 1.0;
    for (int i = 0; i < level; i++) sigma2 *= scale;
    return 1.0 / (sigma2 * sigma2);
}

int orc_stereo_lift_points(const PlCamera* cam, const PlStereoConfig* sc, int n_l, const float* kp_l, const int32_t* octave_l,
                           const uint8_t* desc_l, const float* kp_r, const int32_t* m12, double* pt_pl, double* pt_disp,
                           double* pt_P, double* pt_sigma2, int32_t* pt_level, uint8_t* pdesc_out, int32_t* src_idx) {
    int k = 0;
    for (int i1 = 0; i1 < n_l; ++i1) {   /* src/stereoFrame.cpp:151-170 */
        const int i2 = m12[i1];
        if (i2 < 0) continue;
        const float yl = kp_l[2 * i1 + 1], yr = kp_r[2 * i2 + 1];
        if ((double)fabsf(yl - yr) <= sc->max_dist_epip) {          /* float subtraction (cv::Point2f) */
            const double disp_ = (double)(kp_l[2 * i1] - kp_r[2 * i2]);   /* float - float, then widened */
            if (disp_ >= sc->min_disp) {
                memcpy(pdesc_out + (size_t)k * 32, desc_l + (size_t)i1 * 32, 32);
                const double u = (double)kp_l[2 * i1], v = (double)kp_l[2 * i1 + 1];
                pt_pl[2 * k] = u;
                pt_pl[2 * k + 1] = v;
                pt_disp[k] = disp_;
                orc_back_projection(cam, u, v, disp_, pt_P + 3 * k);
                pt_level[k] = octave_l[i1];
                pt_sigma2[k] = sigma2_of_level(octave_l[i1], sc->orb_scale_factor);
                src_idx[k] = i1;
                k++;
            }
        }
    }
    return k;
}

double orc_line_segment_overlap_stereo(const PlStereoConfig* sc, double spl_obs, double epl_obs, double spl_proj, double epl_proj) {
    double overlap = 1.0;   /* src/stereoFrame.cpp:473-508 */
    if (fabs(epl_obs - spl_obs) > sc->line_horiz_th) {
        double sln = spl_obs < epl_obs ? spl_obs : epl_obs, eln = spl_obs < epl_obs ? epl_obs : spl_obs;
        double spn = spl_proj < epl_proj ? spl_proj : epl_proj, epn = spl_proj < epl_proj ? epl_proj : spl_proj;
        if (epl_obs < spl_obs) { sln = epl_obs; eln = spl_obs; }
        if (epl_proj < spl_proj) { spn = epl_proj; epn = spl_proj; }
        const double length = eln - spn;
        if ((epn < sln) || (spn > eln)) overlap = 0.0;
        else {
            if ((epn > eln) && (spn < sln)) overlap = eln - sln;
            else overlap = (eln < epn ? eln : epn) - (sln < spn ? spn : sln);
        }
        if (length > (double)0.01f) overlap = overlap / length;
        else overlap = 0.0;
        if (overlap > 1.0) overlap = 1.0;
    }
    return overlap;
}

int orc_stereo_lift_lines(const PlCamera* cam, const PlStereoConfig* sc, int n_l, const float* seg_l, const float* angle_l,
                          const int32_t* octave_l, const uint8_t* desc_l, const float* seg_r, const int32_t* m12,
                          double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp, double* ls_sP, double* ls_eP,
                          double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level, uint8_t* ldesc_out,
                          int32_t* src_idx) {
    int k = 0;
    for (int i1 = 0; i1 < n_l; ++i1) {   /* src/stereoFrame.cpp:351-393 */
        const int i2 = m12[i1];
        if (i2 < 0) continue;
        const double sp_l[2] = {seg_l[4 * i1], seg_l[4 * i1 + 1]}, ep_l[2] = {seg_l[4 * i1 + 2], seg_l[4 * i1 + 3]};
        /* le_l = sp_l x ep_l (homogeneous), normalised by sqrt(a^2 + b^2) (:357-358) */
        double le[3] = {sp_l[1] - ep_l[1], ep_l[0] - sp_l[0], sp_l[0] * ep_l[1] - sp_l[1] * ep_l[0]};
        const double nrm = sqrt(le[0] * le[0] + le[1] * le[1]);
        le[0] /= nrm; le[1] /= nrm; le[2] /= nrm;
        double sp_r[2] = {seg_r[4 * i2], seg_r[4 * i2 + 1]}, ep_r[2] = {seg_r[4 * i2 + 2], seg_r[4 * i2 + 3]};
        const double overlap = orc_line_segment_overlap_stereo(sc, sp_l[1], ep_l[1], sp_r[1], ep_r[1]);   /* :362 */
        /* :366-367 — the comma initialiser writes sp_r(0), then sp_r(1); ep_r is then computed from the UPDATED sp_r */
        sp_r[0] = (sp_r[0] * (sp_l[1] - ep_r[1]) + ep_r[0] * (sp_r[1] - sp_l[1])) / (sp_r[1] - ep_r[1]);
        sp_r[1] = sp_l[1];
        ep_r[0] = (sp_r[0] * (ep_l[1] - ep_r[1]) + ep_r[0] * (sp_r[1] - ep_l[1])) / (sp_r[1] - ep_r[1]);
        ep_r[1] = ep_l[1];
        /* filterLineSegmentDisparity (:405-415) */
        double disp_s = sp_l[0] - sp_r[0], disp_e = ep_l[0] - ep_r[0];
        {
            const double mn = disp_e < disp_s ? disp_e : disp_s, mx = disp_s < disp_e ? disp_e : disp_s;
            if (mn / mx < sc->ls_min_disp_ratio) { disp_s = -1.0; disp_e = -1.0; }
        }
        if (disp_s >= sc->min_disp && disp_e >= sc->min_disp && fabs(sp_l[1] - ep_l[1]) > sc->line_horiz_th &&
            fabs(sp_r[1] - ep_r[1]) > sc->line_horiz_th && overlap > sc->stereo_overlap_th) {   /* :371-374 */
            orc_back_projection(cam, sp_l[0], sp_l[1], disp_s, ls_sP + 3 * k);
            orc_back_projection(cam, ep_l[0], ep_l[1], disp_e, ls_eP + 3 * k);
            memcpy(ldesc_out + (size_t)k * 32, desc_l + (size_t)i1 * 32, 32);
            ls_spl[2 * k] = sp_l[0]; ls_spl[2 * k + 1] = sp_l[1];
            ls_epl[2 * k] = ep_l[0]; ls_epl[2 * k + 1] = ep_l[1];
            ls_sdisp[k] = disp_s; ls_edisp[k] = disp_e;
            ls_le[3 * k] = le[0]; ls_le[3 * k + 1] = le[1]; ls_le[3 * k + 2] = le[2];
            ls_angle[k] = (double)angle_l[i1];
            ls_level[k] = octave_l[i1];
            ls_sigma2[k] = sigma2_of_level(octave_l[i1], sc->lsd_scale);
            src_idx[k] = i1;
            k++;
        }
    }
    return k;
}

/* ---- matchStereoPoints / matchStereoLines: the caller-side loops + matchGrid + lifting (src/stereoFrame.cpp:120-173, :309-398) */
int orc_match_stereo_points(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l, const float* kp_l,
                            const int32_t* octave_l, const uint8_t* desc_l, int n_r, const float* kp_r, const uint8_t* desc_r,
                            int32_t* m12, double* pt_pl, double* pt_disp, double* pt_P, double* pt_sigma2, int32_t* pt_level,
                            uint8_t* pdesc_out, int32_t* src_idx) {
    const double inv_width = mc->grid_cols / (double)cam->width, inv_height = mc->grid_rows / (double)cam->height;   /* :47-48 */
    int32_t* q = (int32_t*)malloc(sizeof(int32_t) * 2 * (size_t)(n_l > 0 ? n_l : 1));
    int32_t* t = (int32_t*)malloc(sizeof(int32_t) * 2 * (size_t)(n_r > 0 ? n_r : 1));
    for (int i = 0; i < n_l; ++i) {   /* :131-132: pair<int,int>(kp.pt.x * inv_width, kp.pt.y * inv_height) */
        q[2 * i] = (int)(kp_l[2 * i] * inv_width);
        q[2 * i + 1] = (int)(kp_l[2 * i + 1] * inv_height);
    }
    for (int i = 0; i < n_r; ++i) {   /* :136-139: grid.at(int x, int y) */
        t[2 * i] = (int)(kp_r[2 * i] * inv_width);
        t[2 * i + 1] = (int)(kp_r[2 * i + 1] * inv_height);
    }
    const PlGridWindow w = {mc->matching_s_ws, 0, 0, 0};   /* :141-143 */
    for (int i = 0; i < n_l; ++i) m12[i] = -1;
    if (n_l > 0 && n_r > 0)                                /* :126-127 */
        orc_match_grid_points(mc->grid_rows, mc->grid_cols, w, mc->best_lr_matches, mc->min_ratio_12_p, q, desc_l, n_l, t, desc_r,
                              n_r, m12);
    free(q);
    free(t);
    return orc_stereo_lift_points(cam, sc, n_l, kp_l, octave_l, desc_l, kp_r, m12, pt_pl, pt_disp, pt_P, pt_sigma2, pt_level,
                                  pdesc_out, src_idx);
}

int orc_match_stereo_lines(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int n_l, const float* seg_l,
                           const float* angle_l, const int32_t* octave_l, const uint8_t* desc_l, int n_r, const float* seg_r,
                           const uint8_t* desc_r, int32_t* m12, double* ls_spl, double* ls_epl, double* ls_sdisp, double* ls_edisp,
                           double* ls_sP, double* ls_eP, double* ls_le, double* ls_angle, double* ls_sigma2, int32_t* ls_level,
                           uint8_t* ldesc_out, int32_t* src_idx) {
    const double inv_width = mc->grid_cols / (double)cam->width, inv_height = mc->grid_rows / (double)cam->height;
    int32_t* q = (int32_t*)malloc(sizeof(int32_t) * 4 * (size_t)(n_l > 0 ? n_l : 1));
    double* tl = (double*)malloc(sizeof(double) * 4 * (size_t)(n_r > 0 ? n_r : 1));
    double* td = (double*)malloc(sizeof(double) * 2 * (size_t)(n_r > 0 ? n_r : 1));
    for (int i = 0; i < n_l; ++i) {   /* :320-322 */
        q[4 * i] = (int)(seg_l[4 * i] * inv_width);
        q[4 * i + 1] = (int)(seg_l[4 * i + 1] * inv_height);
        q[4 * i + 2] = (int)(seg_l[4 * i + 2] * inv_width);
        q[4 * i + 3] = (int)(seg_l[4 * i + 3] * inv_height);
    }
    for (int i = 0; i < n_r; ++i) {   /* :328-337 */
        const float sx = seg_r[4 * i], sy = seg_r[4 * i + 1], ex = seg_r[4 * i + 2], ey = seg_r[4 * i + 3];
        double vx = (ex - sx) * inv_width, vy = (ey - sy) * inv_height;   /* float difference, then x double */
        const double magnitude = sqrt(vx * vx + vy * vy);                  /* include/matching.h:43-48 */
        td[2 * i] = vx / magnitude;
        td[2 * i + 1] = vy / magnitude;
        tl[4 * i] = sx * inv_width;
        tl[4 * i + 1] = sy * inv_height;
        tl[4 * i + 2] = ex * inv_width;
        tl[4 * i + 3] = ey * inv_height;
    }
    const PlGridWindow w = {mc->matching_s_ws, 0, 0, 0};
    for (int i = 0; i < n_l; ++i) m12[i] = -1;
    if (n_l > 0 && n_r > 0)
        orc_match_grid_lines(mc->grid_rows, mc->grid_cols, w, mc->best_lr_matches, mc->min_ratio_12_p, mc->line_sim_th, q, desc_l,
                             n_l, tl, td, desc_r, n_r, m12);
    free(q);
    free(tl);
    free(td);
    return orc_stereo_lift_lines(cam, sc, n_l, seg_l, angle_l, octave_l, desc_l, seg_r, m12, ls_spl, ls_epl, ls_sdisp, ls_edisp,
                                 ls_sP, ls_eP, ls_le, ls_angle, ls_sigma2, ls_level, ldesc_out, src_idx);
}

typedef struct {
    const PlCamera* cam; const PlStereoMatchConfig* mc; const PlStereoConfig* sc; int B;
    const int32_t *pl_off, *poct_l, *pr_off, *ll_off, *loct_l, *lr_off;
    const float *kp_l, *kp_r, *seg_l, *angle_l, *seg_r;
    const uint8_t *pdesc_l, *pdesc_r, *ldesc_l, *ldesc_r;
    int32_t* counts; int* next; pthread_mutex_t* mu;
} StereoJob;

static void* stereo_worker(void* arg) {
    StereoJob* j = (StereoJob*)arg;
    for (;;) {
        pthread_mutex_lock(j->mu);
        const int f = (*j->next)++;
        pthread_mutex_unlock(j->mu);
        if (f >= j->B) break;
        const int a = j->pl_off[f], n = j->pl_off[f + 1] - a, b = j->pr_off[f], nr = j->pr_off[f + 1] - b;
        const int c = j->ll_off[f], m = j->ll_off[f + 1] - c, d = j->lr_off[f], mr = j->lr_off[f + 1] - d;
        const size_t cap = (size_t)((n > m ? n : m) > 0 ? (n > m ? n : m) : 1);
        double* buf = (double*)malloc(sizeof(double) * cap * 24);
        int32_t* ib = (int32_t*)malloc(sizeof(int32_t) * cap * 3);
        uint8_t* db = (uint8_t*)malloc(cap * 32);
        j->counts[2 * f] = orc_match_stereo_points(j->cam, j->mc, j->sc, n, j->kp_l + 2 * (size_t)a, j->poct_l + a,
                                                   j->pdesc_l + 32 * (size_t)a, nr, j->kp_r + 2 * (size_t)b,
                                                   j->pdesc_r + 32 * (size_t)b, ib, buf, buf + 2 * cap, buf + 3 * cap, buf + 6 * cap,
                                                   ib + cap, db, ib + 2 * cap);
        j->counts[2 * f + 1] = orc_match_stereo_lines(j->cam, j->mc, j->sc, m, j->seg_l + 4 * (size_t)c, j->angle_l + c, j->loct_l + c,
                                                      j->ldesc_l + 32 * (size_t)c, mr, j->seg_r + 4 * (size_t)d,
                                                      j->ldesc_r + 32 * (size_t)d, ib, buf, buf + 2 * cap, buf + 4 * cap,
                                                      buf + 5 * cap, buf + 6 * cap, buf + 9 * cap, buf + 12 * cap, buf + 15 * cap,
                                                      buf + 16 * cap, ib + cap, db, ib + 2 * cap);
        free(buf);
        free(ib);
        free(db);
    }
    return NULL;
}

int orc_stereo_batch(const PlCamera* cam, const PlStereoMatchConfig* mc, const PlStereoConfig* sc, int B, const int32_t* pl_off,
                     const float* kp_l, const int32_t* poct_l, const uint8_t* pdesc_l, const int32_t* pr_off, const float* kp_r,
                     const uint8_t* pdesc_r, const int32_t* ll_off, const float* seg_l, const float* angle_l, const int32_t* loct_l,
                     const uint8_t* ldesc_l, const int32_t* lr_off, const float* seg_r, const uint8_t* ldesc_r, int threads,
                     int32_t* counts) {
    if (threads < 1) threads = 1;
    if (threads > B) threads = B > 0 ? B : 1;
    int next = 0;
    pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
    StereoJob j = {cam, mc, sc, B, pl_off, poct_l, pr_off, ll_off, loct_l, lr_off, kp_l, kp_r, seg_l, angle_l, seg_r,
                   pdesc_l, pdesc_r, ldesc_l, ldesc_r, counts, &next, &mu};
    pthread_t* th = (pthread_t*)calloc((size_t)threads, sizeof(pthread_t));
    for (int t = 1; t < threads; t++) pthread_create(&th[t], NULL, stereo_worker, &j);
    stereo_worker(&j);
    for (int t = 1; t < threads; t++) pthread_join(th[t], NULL);
    free(th);
    long total = 0;
    for (int f = 0; f < 2 * B; f++) total += counts[f];
    return (int)total;
}

/* ------------------------------------------------------------------------------------------------
 * the handler state (StereoFrameHandler: matched_pt / matched_ls lists, include/stereoFrameHandler.h)
 * ---------------------------------------------------------------------------------------------- */
typedef struct { /* PointFeature fields the path reads (include/stereoFeatures.h:30-58) */
    double P[3], pl_obs[2], sigma2;
    int inlier;
} OrcPoint;
typedef struct { /* LineFeature fields the path reads (include/stereoFeatures.h:60-121) */
    double sP[3], eP[3], le_obs[3], spl[2], epl[2], sigma2;
    int inlier;
} OrcLine;
typedef struct {
    const PlCamera* cam;
    const PlConfig* cfg;
    OrcPoint* pt;
    int n_pt; /* matched_pt */
    OrcLine* ls;
    int n_ls; /* matched_ls */
    int n_inliers, n_inliers_pt, n_inliers_ls;
    int evals; /* instrumentation: optimizeFunctions calls in the current GN run */
} OrcHandler;

static void transform_point(const double DT[16], const double P[3], double out[3]) {
    /* DT.block(0,0,3,3) * P + DT.col(3).head(3)   (src/stereoFrameHandler.cpp:567) */
    for (int i = 0; i < 3; i++)
        out[i] = (DT[i * 4 + 0] * P[0] + DT[i * 4 + 1] * P[1] + DT[i * 4 + 2] * P[2]) + DT[i * 4 + 3];
}

static double dmax(double a, double b) { return (a < b) ? b : a; } /* std::max */

/* the 6-vector of src/stereoFrameHandler.cpp:582-587 / :636-641 with (dx,dy) or (lx,ly) */
static void jac_aux(double fgz2, double gx, double gy, double gz, double dx, double dy, double J[6]) {
    J[0] = +fgz2 * dx * gz;
    J[1] = +fgz2 * dy * gz;
    J[2] = -fgz2 * (gx * dx + gy * dy);
    J[3] = -fgz2 * (gx * gy * dx + gy * gy * dy + gz * gz * dy);
    J[4] = +fgz2 * (gx * gx * dx + gz * gz * dx + gx * gy * dy);
    J[5] = +fgz2 * (gx * gz * dy - gy * gz * dx);
}

static void accumulate(double H[36], double g[6], double* e, const double J[6], double r, double w) {
    /* H += J*J^T*w; g += J*r*w; e += r*r*w   (:601-603) — Eigen evaluates (J*J^T)*w, (J*r)*w */
    for (int i = 0; i < 6; i++) {
        for (int j = 0; j < 6; j++) H[i * 6 + j] += (J[i] * J[j]) * w;
        g[i] += (J[i] * r) * w;
    }
    *e += r * r * w;
}

static double point_residual_norm(const OrcHandler* h, const double DT[16], const OrcPoint* pt,
                                  double P_[3], double err[2]) {
    double uv[2];
    transform_point(DT, pt->P, P_);
    orc_projection(h->cam, P_, uv);
    err[0] = uv[0] - pt->pl_obs[0];
    err[1] = uv[1] - pt->pl_obs[1];
    return sqrt(err[0] * err[0] + err[1] * err[1]);
}

static double line_residual_norm(const OrcHandler* h, const double DT[16], const OrcLine* ls,
                                 double sP_[3], double eP_[3], double sproj[2], double eproj[2],
                                 double err[2]) {
    transform_point(DT, ls->sP, sP_);
    orc_projection(h->cam, sP_, sproj);
    transform_point(DT, ls->eP, eP_);
    orc_projection(h->cam, eP_, eproj);
    err[0] = ls->le_obs[0] * sproj[0] + ls->le_obs[1] * sproj[1] + ls->le_obs[2];
    err[1] = ls->le_obs[0] * eproj[0] + ls->le_obs[1] * eproj[1] + ls->le_obs[2];
    return sqrt(err[0] * err[0] + err[1] * err[1]);
}

/* optimizeFunctions (src/stereoFrameHandler.cpp:549-694) and optimizeFunctionsRobust (:696-962) */
static void optimize_functions(OrcHandler* h, const double DT[16], int robust, double H[36],
                               double g[6], double* e_out) {
    const double homog_th = h->cfg->homog_th, fx = h->cam->fx;
    double H_p[36], H_l[36], g_p[6], g_l[6], e_p = 0.0, e_l = 0.0;
    memset(H_p, 0, sizeof(H_p));
    memset(H_l, 0, sizeof(H_l));
    memset(g_p, 0, sizeof(g_p));
    memset(g_l, 0, sizeof(g_l));
    h->evals++;

    double s_p = 1.0, s_l = 1.0;
    if (robust) { /* pre-weight pass + MAD scales (:707-781) */
        double* res_p = (double*)malloc((size_t)(h->n_pt + 1) * sizeof(double));
        double* res_l = (double*)malloc((size_t)(h->n_ls + 1) * sizeof(double));
        int np = 0, nl = 0;
        for (int i = 0; i < h->n_pt; i++)
            if (h->pt[i].inlier) {
                double P_[3], err[2];
                res_p[np++] = point_residual_norm(h, DT, &h->pt[i], P_, err);
            }
        for (int i = 0; i < h->n_ls; i++)
            if (h->ls[i].inlier) {
                double a[3], b[3], c[2], d[2], err[2];
                res_l[nl++] = line_residual_norm(h, DT, &h->ls[i], a, b, c, d, err);
            }
        const double th_min = 0.0001, th_max = sqrt(7.815);
        s_p = orc_vector_stdv_mad(res_p, np);
        s_l = orc_vector_stdv_mad(res_l, nl);
        if (s_p < th_min) s_p = th_min;
        if (s_p > th_max) s_p = th_max;
        if (s_l < th_min) s_l = th_min;
        if (s_l > th_max) s_l = th_max;
        free(res_p);
        free(res_l);
    }

    int N_p = 0;
    for (int i = 0; i < h->n_pt; i++) { /* point block (:563-606 / :785-870) */
        const OrcPoint* pt = &h->pt[i];
        if (!pt->inlier) continue;
        double P_[3], err[2], J[6];
        double err_norm = point_residual_norm(h, DT, pt, P_, err);
        double gx = P_[0], gy = P_[1], gz = P_[2];
        double gz2 = gz * gz;
        double fgz2 = fx / dmax(homog_th, gz2);
        jac_aux(fgz2, gx, gy, gz, err[0], err[1], J);
        double den = dmax(homog_th, err_norm);
        for (int k = 0; k < 6; k++) J[k] = J[k] / den;
        double s2 = pt->sigma2, r, w;
        if (!robust) {
            r = err_norm * sqrt(s2);
            w = orc_robust_weight_cauchy(r);
        } else {
            r = err_norm;
            w = orc_robust_weight_cauchy(r / s_p);
        }
        accumulate(H_p, g_p, &e_p, J, r, w);
        N_p++;
    }

    int N_l = 0;
    for (int i = 0; i < h->n_ls; i++) { /* line block (:610-684 / :874-952) */
        const OrcLine* ls = &h->ls[i];
        if (!ls->inlier) continue;
        double sP_[3], eP_[3], sproj[2], eproj[2], err[2], Js[6], Je[6], J[6];
        double err_norm = line_residual_norm(h, DT, ls, sP_, eP_, sproj, eproj, err);
        double lx = ls->le_obs[0], ly = ls->le_obs[1];
        double ds = err[0], de = err[1];
        double fgz2 = fx / dmax(homog_th, sP_[2] * sP_[2]);
        jac_aux(fgz2, sP_[0], sP_[1], sP_[2], lx, ly, Js);
        fgz2 = fx / dmax(homog_th, eP_[2] * eP_[2]);
        jac_aux(fgz2, eP_[0], eP_[1], eP_[2], lx, ly, Je);
        double den = dmax(homog_th, err_norm);
        for (int k = 0; k < 6; k++) J[k] = (Js[k] * ds + Je[k] * de) / den;
        double s2 = ls->sigma2, r, w;
        if (!robust) {
            r = err_norm * sqrt(s2);
            w = orc_robust_weight_cauchy(r);
        } else {
            r = err_norm;
            w = orc_robust_weight_cauchy(r / s_l);
        }
        /* overlap with the PREVIOUS frame's endpoints spl/epl (:668, :930) */
        double overlap = orc_line_segment_overlap(ls->spl, ls->epl, sproj, eproj);
        w *= overlap;
        accumulate(H_l, g_l, &e_l, J, r, w);
        N_l++;
    }

    for (int i = 0; i < 36; i++) H[i] = H_p[i] + H_l[i]; /* :687-692 */
    for (int i = 0; i < 6; i++) g[i] = g_p[i] + g_l[i];
    double e = e_p + e_l;
    e /= (double)(N_l + N_p);
    *e_out = e;
}

static double norm3(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

/* DT << DT * inverse_se3( expmap_se3(DT_inc) )   (:419, :460) */
static void apply_increment(double DT[16], const double inc[6]) {
    double E[16], Ei[16];
    orc_expmap_se3(inc, E);
    orc_inverse_se3(E, Ei);
    mat4_mul(DT, Ei, DT);
}

/* gaussNewtonOptimization (src/stereoFrameHandler.cpp:394-431) */
static void gauss_newton(OrcHandler* h, double DT[16], double DT_cov[36], double* err_, int max_iters) {
    double H[36], g[6], inc[6];
    double err = 0.0, err_prev = 999999999.9;
    memset(H, 0, sizeof(H));
    h->evals = 0;
    for (int iters = 0; iters < max_iters; iters++) {
        optimize_functions(h, DT, 0, H, g, &err);
        if (err > err_prev) {
            if (iters > 0) break;
            *err_ = -1.0;
            return;
        }
        if ((err < h->cfg->min_error) || fabs(err - err_prev) < h->cfg->min_error_change) break;
        orc_qr6_solve(H, g, inc, NULL);
        apply_increment(DT, inc);
        if (norm3(inc) < h->cfg->min_error_change && norm3(inc + 3) < h->cfg->min_error_change) break;
        err_prev = err;
    }
    orc_inv6(H, DT_cov);
    *err_ = err;
}

/* gaussNewtonOptimizationRobust (src/stereoFrameHandler.cpp:433-480) */
static void gauss_newton_robust(OrcHandler* h, double DT[16], double DT_cov[36], double* err_, int max_iters) {
    double DT0[16], H[36], g[6], inc[6];
    double err = 0.0, err_prev = 999999999.9;
    int solution_is_good = 1;
    memcpy(DT0, DT, sizeof(DT0));
    memset(H, 0, sizeof(H));
    h->evals = 0;
    for (int iters = 0; iters < max_iters; iters++) {
        optimize_functions(h, DT, 1, H, g, &err);
        if ((fabs(err - err_prev) < h->cfg->min_error_change) || (err < h->cfg->min_error)) break;
        double lad;
        orc_qr6_solve(H, g, inc, &lad);
        if (lad < 0.0) { /* solver.info() is always Success for ColPivHouseholderQR */
            solution_is_good = 0;
            break;
        }
        apply_increment(DT, inc);
        if (sqrt(inc[0] * inc[0] + inc[1] * inc[1] + inc[2] * inc[2] + inc[3] * inc[3] + inc[4] * inc[4] +
                 inc[5] * inc[5]) < h->cfg->min_error_change)
            break;
        err_prev = err;
    }
    if (solution_is_good) {
        orc_inv6(H, DT_cov);
        *err_ = err;
    } else {
        memcpy(DT, DT0, sizeof(DT0));
        *err_ = -1.0;
        memset(DT_cov, 0, 36 * sizeof(double));
        for (int i = 0; i < 6; i++) DT_cov[i * 6 + i] = 1.0;
    }
}

/* isGoodSolution (src/stereoFrameHandler.cpp:292-305) */
static int is_good_solution(const double DT[16], const double DT_cov[36], double err) {
    double w[6];
    orc_eig6_sym(DT_cov, w);
    if (w[0] < 0.0 || w[5] > 1.0 || err < 0.0 || err > 1.0 || !orc_is_finite(DT, 16)) return 0;
    return 1;
}
int orc_is_good_solution(const double DT[16], const double DT_cov[36], double err) { return is_good_solution(DT, DT_cov, err); }

/* removeOutliers (src/stereoFrameHandler.cpp:988-1067) */
static int remove_outliers(OrcHandler* h, const double DT[16]) {
    if (h->cfg->has_points) {
        double* res = (double*)malloc((size_t)(h->n_pt + 1) * sizeof(double));
        for (int i = 0; i < h->n_pt; i++) {
            double P_[3], err[2];
            res[i] = point_residual_norm(h, DT, &h->pt[i], P_, err) * sqrt(h->pt[i].sigma2);
        }
        double mean, stdv;
        orc_vector_mean_stdv_mad(res, h->n_pt, &mean, &stdv);
        double th = h->cfg->inlier_k * stdv;
        for (int i = 0; i < h->n_pt; i++)
            if (h->pt[i].inlier && fabs(res[i] - mean) > th) {
                h->pt[i].inlier = 0;
                h->n_inliers--;
                h->n_inliers_pt--;
            }
        free(res);
    }
    if (h->cfg->has_lines) {
        double* res = (double*)malloc((size_t)(h->n_ls + 1) * sizeof(double));
        for (int i = 0; i < h->n_ls; i++) {
            double a[3], b[3], c[2], d[2], err[2];
            res[i] = line_residual_norm(h, DT, &h->ls[i], a, b, c, d, err) * sqrt(h->ls[i].sigma2);
        }
        double mean, stdv;
        orc_vector_mean_stdv_mad(res, h->n_ls, &mean, &stdv);
        double th = h->cfg->inlier_k * stdv;
        for (int i = 0; i < h->n_ls; i++)
            if (fabs(res[i] - mean) > th && h->ls[i].inlier) {
                h->ls[i].inlier = 0;
                h->n_inliers--;
                h->n_inliers_ls--;
            }
        free(res);
    }
    if (h->n_inliers != h->n_inliers_pt + h->n_inliers_ls) return PLSTVO_E_SIZE; /* :1065-1066 throws */
    return 0;
}

/* optimizePose (src/stereoFrameHandler.cpp:307-392) */
static int optimize_pose(OrcHandler* h, const PlPrior* prior, PlPoseResult* out) {
    const PlConfig* cfg = h->cfg;
    double DT[16], DT_[16], DT_cov[36];
    double err = -1.0;
    int rc = 0;
    memset(DT_cov, 0, sizeof(DT_cov)); /* uninitialised in the reference; only read after a GN call set it,
                                          or together with err == -1 which fails the gate regardless */
    out->status = PLSTVO_ST_REFINED;
    out->iters_stage1 = out->iters_stage2 = 0;

    if (cfg->use_motion_model && prior) { /* :317-324 */
        memcpy(DT, prior->DT, sizeof(DT));
        if (!is_good_solution(DT, prior->DT_cov, prior->err_norm)) mat4_identity(DT);
    } else
        mat4_identity(DT);

    const int mode = cfg->solver_mode; /* hard-wired 0 in the reference (:329) */
    if (h->n_inliers >= cfg->min_features) {
        memcpy(DT_, DT, sizeof(DT));
        if (mode == 0) gauss_newton(h, DT_, DT_cov, &err, cfg->max_iters);
        else gauss_newton_robust(h, DT_, DT_cov, &err, cfg->max_iters);
        out->iters_stage1 = h->evals;
        if (is_good_solution(DT_, DT_cov, err)) {
            rc = remove_outliers(h, DT_);
            if (h->n_inliers >= cfg->min_features) {
                if (mode == 0) gauss_newton(h, DT, DT_cov, &err, cfg->max_iters_ref);
                else gauss_newton_robust(h, DT, DT_cov, &err, cfg->max_iters_ref);
                out->iters_stage2 = h->evals;
            } else {
                mat4_identity(DT);
                out->status = PLSTVO_ST_FEW_AFTER;
            }
        } else {
            gauss_newton_robust(h, DT, DT_cov, &err, cfg->max_iters_ref);
            out->iters_stage2 = h->evals;
            out->status = PLSTVO_ST_ROBUST_FALLBACK;
        }
    } else {
        mat4_identity(DT);
        out->status = PLSTVO_ST_FEW_BEFORE;
    }
    memcpy(out->DT_opt, DT, sizeof(DT));

    double Tfw_prev[16], Tfw_cov_prev[36];
    if (prior) {
        memcpy(Tfw_prev, prior->Tfw, sizeof(Tfw_prev));
        memcpy(Tfw_cov_prev, prior->Tfw_cov, sizeof(Tfw_cov_prev));
    } else { /* initialize(): Tfw = I, Tfw_cov = I (src/stereoFrameHandler.cpp:43-44) */
        mat4_identity(Tfw_prev);
        memset(Tfw_cov_prev, 0, sizeof(Tfw_cov_prev));
        for (int i = 0; i < 6; i++) Tfw_cov_prev[i * 6 + i] = 1.0;
    }

    if (is_good_solution(DT, DT_cov, err) && !mat4_is_identity(DT)) { /* :372-381 */
        double Ti[16], x[6], T2[16];
        orc_inverse_se3(DT, Ti);
        orc_logmap_se3(Ti, x);
        orc_expmap_se3(x, out->DT);
        memcpy(out->DT_cov, DT_cov, sizeof(DT_cov));
        out->err_norm = err;
        mat4_mul(Tfw_prev, out->DT, T2);
        orc_logmap_se3(T2, x);
        orc_expmap_se3(x, out->Tfw);
        orc_unccomp_se3(Tfw_prev, Tfw_cov_prev, DT_cov, out->Tfw_cov);
        orc_eig6_sym(DT_cov, out->DT_cov_eig);
        out->good = 1;
    } else { /* :382-391 */
        mat4_identity(out->DT);
        memset(out->DT_cov, 0, sizeof(out->DT_cov));
        out->err_norm = -1.0;
        memcpy(out->Tfw, Tfw_prev, sizeof(Tfw_prev));
        memcpy(out->Tfw_cov, Tfw_cov_prev, sizeof(Tfw_cov_prev));
        memset(out->DT_cov_eig, 0, sizeof(out->DT_cov_eig));
        out->good = 0;
    }
    out->n_matched_pt = h->n_pt;
    out->n_matched_ls = h->n_ls;
    out->n_inliers_pt = h->n_inliers_pt;
    out->n_inliers_ls = h->n_inliers_ls;
    out->n_inliers = h->n_inliers;
    out->reserved = 0;
    return rc;
}

/* ------------------------------------------------------------------------------------------------
 * public entry points
 * ---------------------------------------------------------------------------------------------- */
static void handler_from_matched(OrcHandler* h, const PlCamera* cam, const PlConfig* cfg,
                                 const PlMatchedBatch* m, int p) {
    int p0 = m->pt_off[p], p1 = m->pt_off[p + 1], l0 = m->ls_off[p], l1 = m->ls_off[p + 1];
    h->cam = cam;
    h->cfg = cfg;
    h->n_pt = p1 - p0;
    h->n_ls = l1 - l0;
    h->pt = (OrcPoint*)calloc((size_t)h->n_pt + 1, sizeof(OrcPoint));
    h->ls = (OrcLine*)calloc((size_t)h->n_ls + 1, sizeof(OrcLine));
    for (int i = 0; i < h->n_pt; i++) {
        OrcPoint* q = &h->pt[i];
        memcpy(q->P, m->pt_P + 3 * (size_t)(p0 + i), 24);
        memcpy(q->pl_obs, m->pt_pl_obs + 2 * (size_t)(p0 + i), 16);
        q->sigma2 = m->pt_sigma2[p0 + i];
        q->inlier = m->pt_inlier ? (m->pt_inlier[p0 + i] != 0) : 1;
    }
    for (int i = 0; i < h->n_ls; i++) {
        OrcLine* q = &h->ls[i];
        memcpy(q->sP, m->ls_sP + 3 * (size_t)(l0 + i), 24);
        memcpy(q->eP, m->ls_eP + 3 * (size_t)(l0 + i), 24);
        memcpy(q->le_obs, m->ls_le_obs + 3 * (size_t)(l0 + i), 24);
        memcpy(q->spl, m->ls_spl + 2 * (size_t)(l0 + i), 16);
        memcpy(q->epl, m->ls_epl + 2 * (size_t)(l0 + i), 16);
        q->sigma2 = m->ls_sigma2[l0 + i];
        q->inlier = m->ls_inlier ? (m->ls_inlier[l0 + i] != 0) : 1;
    }
    /* f2fTracking: n_inliers_* = list sizes (src/stereoFrameHandler.cpp:126-128) */
    h->n_inliers_pt = h->n_pt;
    h->n_inliers_ls = h->n_ls;
    h->n_inliers = h->n_pt + h->n_ls;
    h->evals = 0;
}

void orc_optimize_functions(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* m, int p,
                            const double DT[16], int robust, double H[36], double g[6], double* e) {
    OrcHandler h;
    handler_from_matched(&h, cam, cfg, m, p);
    optimize_functions(&h, DT, robust, H, g, e);
    free(h.pt);
    free(h.ls);
}

int orc_optimize_pose(const PlCamera* cam, const PlConfig* cfg, const PlMatchedBatch* matched,
                      const PlPrior* priors, PlPoseResult* results, uint8_t* inlier_pt,
                      uint8_t* inlier_ls) {
    int rc = 0;
    for (int p = 0; p < matched->B; p++) {
        OrcHandler h;
        handler_from_matched(&h, cam, cfg, matched, p);
        int r = optimize_pose(&h, priors ? &priors[p] : NULL, &results[p]);
        if (r < 0) rc = r;
        if (inlier_pt)
            for (int i = 0; i < h.n_pt; i++) inlier_pt[matched->pt_off[p] + i] = (uint8_t)h.pt[i].inlier;
        if (inlier_ls)
            for (int i = 0; i < h.n_ls; i++) inlier_ls[matched->ls_off[p] + i] = (uint8_t)h.ls[i].inlier;
        free(h.pt);
        free(h.ls);
    }
    return rc;
}

typedef struct {
    const PlConfig* cfg;
    const PlFrameBatch *prev, *curr;
    int p, lines, threads;
    int32_t* m12;
    int ret;
} F2fJob;

static void* f2f_job(void* arg) { /* matchF2FPoints :131-153 / matchF2FLines :155-180 (matching part) */
    F2fJob* j = (F2fJob*)arg;
    const PlFrameBatch *a = j->prev, *b = j->curr;
    const int32_t *oa = j->lines ? a->ls_off : a->pt_off, *ob = j->lines ? b->ls_off : b->pt_off;
    int n1 = oa[j->p + 1] - oa[j->p], n2 = ob[j->p + 1] - ob[j->p];
    int enabled = j->lines ? j->cfg->has_lines : j->cfg->has_points;
    for (int i = 0; i < n1; i++) j->m12[i] = -1;
    j->ret = 0;
    if (!enabled || n1 == 0 || n2 == 0) return NULL; /* :137-138, :160-161 */
    const uint8_t* d1 = (j->lines ? a->ldesc : a->pdesc) + (size_t)oa[j->p] * 32;
    const uint8_t* d2 = (j->lines ? b->ldesc : b->pdesc) + (size_t)ob[j->p] * 32;
    float nnr = (float)(j->lines ? j->cfg->min_ratio_12_l : j->cfg->min_ratio_12_p); /* double -> float at the call */
    j->ret = orc_match(d1, n1, d2, n2, nnr, j->cfg->best_lr_matches, j->threads, j->m12);
    return NULL;
}

static void f2f_pair(const PlConfig* cfg, const PlFrameBatch* prev, const PlFrameBatch* curr, int p,
                     int faithful, int32_t* m12_pt, int32_t* m12_ls, int* n_pt, int* n_ls) {
    F2fJob jp = {cfg, prev, curr, p, 0, faithful, m12_pt, 0};
    F2fJob jl = {cfg, prev, curr, p, 1, faithful, m12_ls, 0};
    if (faithful && cfg->has_points && cfg->has_lines) { /* plInParallel (:113-119) */
        pthread_t t;
        pthread_create(&t, NULL, f2f_job, &jl);
        f2f_job(&jp);
        pthread_join(t, NULL);
    } else {
        f2f_job(&jp);
        f2f_job(&jl);
    }
    *n_pt = jp.ret;
    *n_ls = jl.ret;
}

int orc_f2f_tracking(const PlConfig* cfg, const PlFrameBatch* prev, const PlFrameBatch* curr,
                     int32_t* m12_pt, int32_t* m12_ls, int32_t* n_matched) {
    if (prev->B != curr->B) return PLSTVO_E_SIZE;
    for (int p = 0; p < prev->B; p++) {
        int np, nl;
        f2f_pair(cfg, prev, curr, p, 0, m12_pt + prev->pt_off[p], m12_ls + prev->ls_off[p], &np, &nl);
        if (n_matched) {
            n_matched[2 * p] = np;
            n_matched[2 * p + 1] = nl;
        }
    }
    return 0;
}

static double now_ms(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

/* one (prev, curr) pair: f2fTracking glue (src/stereoFrameHandler.cpp:144-152, :167-179) + optimizePose */
static int track_pair(const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                      const PlFrameBatch* curr, const PlPrior* prior, int p, int faithful,
                      PlPoseResult* res, int32_t* m12_pt, int32_t* m12_ls, uint8_t* inl_pt,
                      uint8_t* inl_ls, double* stage_ms) {
    int n1p = prev->pt_off[p + 1] - prev->pt_off[p], n1l = prev->ls_off[p + 1] - prev->ls_off[p];
    int32_t* mp = m12_pt ? m12_pt : (int32_t*)malloc((size_t)(n1p + 1) * sizeof(int32_t));
    int32_t* ml = m12_ls ? m12_ls : (int32_t*)malloc((size_t)(n1l + 1) * sizeof(int32_t));
    int np, nl;
    double t0 = now_ms();
    f2f_pair(cfg, prev, curr, p, faithful, mp, ml, &np, &nl);
    double t1 = now_ms();

    OrcHandler h;
    h.cam = cam;
    h.cfg = cfg;
    h.pt = (OrcPoint*)calloc((size_t)np + 1, sizeof(OrcPoint));
    h.ls = (OrcLine*)calloc((size_t)nl + 1, sizeof(OrcLine));
    int* ipt = (int*)malloc((size_t)(np + 1) * sizeof(int));
    int* ils = (int*)malloc((size_t)(nl + 1) * sizeof(int));
    h.n_pt = h.n_ls = 0;
    size_t a0 = (size_t)prev->pt_off[p], b0 = (size_t)curr->pt_off[p];
    for (int i1 = 0; i1 < n1p; i1++) { /* :144-152 */
        int i2 = mp[i1];
        if (i2 < 0) continue;
        OrcPoint* q = &h.pt[h.n_pt];
        memcpy(q->P, prev->pt_P + 3 * (a0 + i1), 24);
        memcpy(q->pl_obs, curr->pt_pl + 2 * (b0 + i2), 16); /* pl_obs = curr pl (:148) */
        q->sigma2 = prev->pt_sigma2[a0 + i1];               /* PointFeature::safeCopy keeps sigma2 */
        q->inlier = 1;
        ipt[h.n_pt++] = i1;
    }
    a0 = (size_t)prev->ls_off[p];
    b0 = (size_t)curr->ls_off[p];
    for (int i1 = 0; i1 < n1l; i1++) { /* :167-179 */
        int i2 = ml[i1];
        if (i2 < 0) continue;
        OrcLine* q = &h.ls[h.n_ls];
        memcpy(q->sP, prev->ls_sP + 3 * (a0 + i1), 24);
        memcpy(q->eP, prev->ls_eP + 3 * (a0 + i1), 24);
        memcpy(q->le_obs, curr->ls_le + 3 * (b0 + i2), 24); /* le_obs = curr le (:175) */
        memcpy(q->spl, prev->ls_spl + 2 * (a0 + i1), 16);
        memcpy(q->epl, prev->ls_epl + 2 * (a0 + i1), 16);
        /* LineFeature::safeCopy -> ctor re-applies the level rule on the passed sigma2
         * (src/stereoFeatures.cpp:117-135): for level times sigma2 *= lsdScale; sigma2 = 1/(sigma2*sigma2) */
        double s2 = prev->ls_sigma2[a0 + i1];
        int level = prev->ls_level ? prev->ls_level[a0 + i1] : 0;
        for (int k = 0; k < level; k++) s2 *= cfg->lsd_scale;
        q->sigma2 = 1.0 / (s2 * s2);
        q->inlier = 1;
        ils[h.n_ls++] = i1;
    }
    h.n_inliers_pt = h.n_pt;
    h.n_inliers_ls = h.n_ls;
    h.n_inliers = h.n_pt + h.n_ls;
    h.evals = 0;
    int rc = optimize_pose(&h, prior, res);
    double t2 = now_ms();
    if (stage_ms) {
        stage_ms[0] = t1 - t0;
        stage_ms[1] = t2 - t1;
    }
    if (inl_pt) {
        memset(inl_pt, 0, (size_t)n1p);
        for (int k = 0; k < h.n_pt; k++) inl_pt[ipt[k]] = (uint8_t)h.pt[k].inlier;
    }
    if (inl_ls) {
        memset(inl_ls, 0, (size_t)n1l);
        for (int k = 0; k < h.n_ls; k++) inl_ls[ils[k]] = (uint8_t)h.ls[k].inlier;
    }
    free(h.pt);
    free(h.ls);
    free(ipt);
    free(ils);
    if (!m12_pt) free(mp);
    if (!m12_ls) free(ml);
    return rc;
}

typedef struct {
    const PlCamera* cam;
    const PlConfig* cfg;
    const PlFrameBatch *prev, *curr;
    const PlPrior* priors;
    PlPoseResult* results;
    int32_t *m12_pt, *m12_ls;
    uint8_t *inl_pt, *inl_ls;
    int faithful;
    int* next;
    pthread_mutex_t* mu;
    double stage_ms[2];
    int rc;
} BatchWorker;

static void* batch_worker(void* arg) {
    BatchWorker* w = (BatchWorker*)arg;
    for (;;) {
        pthread_mutex_lock(w->mu);
        int p = (*w->next)++;
        pthread_mutex_unlock(w->mu);
        if (p >= w->prev->B) break;
        double st[2];
        int r = track_pair(w->cam, w->cfg, w->prev, w->curr, w->priors ? &w->priors[p] : NULL, p,
                           w->faithful, &w->results[p],
                           w->m12_pt ? w->m12_pt + w->prev->pt_off[p] : NULL,
                           w->m12_ls ? w->m12_ls + w->prev->ls_off[p] : NULL,
                           w->inl_pt ? w->inl_pt + w->prev->pt_off[p] : NULL,
                           w->inl_ls ? w->inl_ls + w->prev->ls_off[p] : NULL, st);
        if (r < 0) w->rc = r;
        w->stage_ms[0] += st[0];
        w->stage_ms[1] += st[1];
    }
    return NULL;
}

int orc_track_batch(const PlCamera* cam, const PlConfig* cfg, const PlFrameBatch* prev,
                    const PlFrameBatch* curr, const PlPrior* priors, PlPoseResult* results,
                    int32_t* m12_pt, int32_t* m12_ls, uint8_t* inlier_pt, uint8_t* inlier_ls,
                    int threads, int faithful, double* stage_ms) {
    if (prev->B != curr->B) return PLSTVO_E_SIZE;
    if (threads < 1 || faithful) threads = 1;
    if (threads > 1024) threads = 1024;
    int next = 0, rc = 0;
    pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
    BatchWorker* w = (BatchWorker*)calloc((size_t)threads, sizeof(BatchWorker));
    pthread_t* th = (pthread_t*)calloc((size_t)threads, sizeof(pthread_t));
    for (int t = 0; t < threads; t++) {
        BatchWorker b = {cam, cfg, prev, curr, priors, results, m12_pt, m12_ls, inlier_pt, inlier_ls,
                         faithful, &next, &mu, {0, 0}, 0};
        w[t] = b;
    }
    for (int t = 1; t < threads; t++) pthread_create(&th[t], NULL, batch_worker, &w[t]);
    batch_worker(&w[0]);
    for (int t = 1; t < threads; t++) pthread_join(th[t], NULL);
    if (stage_ms) stage_ms[0] = stage_ms[1] = 0.0;
    for (int t = 0; t < threads; t++) {
        if (w[t].rc < 0) rc = w[t].rc;
        if (stage_ms) {
            stage_ms[0] += w[t].stage_ms[0];
            stage_ms[1] += w[t].stage_ms[1];
        }
    }
    free(w);
    free(th);
    return rc;
}

/* ------------------------------------------------------------------------------------------------
 * host-side state machine: adaptive FAST threshold and the key-frame test (SURVEY 8(f)-3)
 * ---------------------------------------------------------------------------------------------- */
void orc_handler_default_config(OrcHandlerConfig* c) {   /* src/config.cpp:40-42, :52, :72-76, :102 */
    c->adaptative_fast = 1; c->fast_min_th = 5; c->fast_max_th = 50; c->fast_inc_th = 5; c->fast_feat_th = 50;
    c->orb_fast_th = 20; c->fast_err_th = 0.5f; c->min_entropy_ratio = 0.85; c->max_kf_t_dist = 5.0; c->max_kf_r_dist = 15.0;
}

static int is_identity4(const double T[16]) {
    for (int i = 0; i < 16; ++i)
        if (T[i] != ((i % 5 == 0) ? 1.0 : 0.0)) return 0;
    return 1;
}

int orc_update_fast_threshold(const OrcHandlerConfig* c, int th, const double DT[16], double err_norm, int n_inliers_pt) {
    if (!c->adaptative_fast) return th;   /* src/stereoFrameHandler.cpp:66-86 */
    const int mn = c->fast_min_th, mx = c->fast_max_th, inc = c->fast_inc_th, feat = c->fast_feat_th;
    if (is_identity4(DT) || err_norm > c->fast_err_th) th = (mn > th - 2 * inc) ? mn : th - 2 * inc;
    else if (n_inliers_pt < feat) th = (mn > th - 2 * inc) ? mn : th - 2 * inc;
    else if (n_inliers_pt < feat * 2) th = (mn > th - inc) ? mn : th - inc;
    else if (n_inliers_pt > feat * 3) th = (mx < th + inc) ? mx : th + inc;
    else if (n_inliers_pt > feat * 4) th = (mx < th + 2 * inc) ? mx : th + 2 * inc;
    return th;
}

void orc_kf_reset(OrcKfState* s) {
    memset(s, 0, sizeof(*s));
    for (int i = 0; i < 4; ++i) s->T_prevKF[5 * i] = 1.0;
    s->prev_f_iskf = 1;
}

double orc_det6(const double Ain[36]) {   /* Eigen: PartialPivLU determinant for fixed sizes above 4 */
    double A[36], det = 1.0;
    memcpy(A, Ain, sizeof(A));
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        for (int r = c + 1; r < 6; ++r)
            if (fabs(A[6 * r + c]) > fabs(A[6 * piv + c])) piv = r;
        if (piv != c) {
            for (int j = 0; j < 6; ++j) { double t = A[6 * c + j]; A[6 * c + j] = A[6 * piv + j]; A[6 * piv + j] = t; }
            det = -det;
        }
        det *= A[6 * c + c];
        if (A[6 * c + c] == 0.0) continue;   /* a zero pivot skips its elimination; the product runs on (0 * inf = NaN) */
        for (int r = c + 1; r < 6; ++r) {
            const double f = A[6 * r + c] / A[6 * c + c];
            for (int j = c + 1; j < 6; ++j) A[6 * r + j] -= f * A[6 * c + j];
        }
    }
    return det;
}

static void sandwich6(const double A[36], const double C[36], double out[36]) {   /* A C A^T */
    double AC[36];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc += A[6 * i + k] * C[6 * k + j];
            AC[6 * i + j] = acc;
        }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 6; ++k) acc += AC[6 * i + k] * A[6 * j + k];
            out[6 * i + j] = acc;
        }
}

void orc_unctinv_se3(const double T[16], const double cov[36], double out[36]) {   /* src/auxiliar.cpp:184-190 */
    double Ti[16], Ad[36];
    orc_inverse_se3(T, Ti);
    orc_adjoint_se3(Ti, Ad);
    sandwich6(Ad, cov, out);
}

int orc_need_new_kf(const OrcHandlerConfig* c, OrcKfState* s, const double Tfw[16], const double DT[16], const double DT_cov[36]) {
    const double k_entropy = 3.0 * (1.0 + log(2.0 * acos(-1)));   /* src/stereoFrameHandler.cpp:1136-1187 */
    if (s->prev_f_iskf) {
        const double d = orc_det6(DT_cov);
        s->entropy_first_prevKF = (d != 0.0) ? k_entropy + 0.5 * log(d) : -999999999.99;
        s->prev_f_iskf = 0;
    }
    double Ti[16], D[16], dX[6];
    orc_inverse_se3(Tfw, Ti);
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += Ti[4 * i + k] * s->T_prevKF[4 * k + j];
            D[4 * i + j] = acc;
        }
    orc_logmap_se3(D, dX);
    s->t = sqrt(dX[0] * dX[0] + dX[1] * dX[1] + dX[2] * dX[2]);
    s->r = sqrt(dX[3] * dX[3] + dX[4] * dX[4] + dX[5] * dX[5]) * 180.f / 3.1415926535897932384626433832795;
    double Ad[36], cinv[36], add[36];
    orc_adjoint_se3(s->T_prevKF, Ad);
    orc_unctinv_se3(DT, DT_cov, cinv);
    sandwich6(Ad, cinv, add);
    for (int i = 0; i < 36; ++i) s->cov_prevKF_currF[i] += add[i];
    s->entropy_curr = k_entropy + 0.5 * log(orc_det6(s->cov_prevKF_currF));
    s->entropy_ratio = s->entropy_curr / s->entropy_first_prevKF;
    int zero_cov = 1;
    for (int i = 0; i < 36; ++i) zero_cov = zero_cov && (DT_cov[i] == 0.0);
    if (s->entropy_ratio < c->min_entropy_ratio || isnan(s->entropy_ratio) || isinf(s->entropy_ratio) ||
        (zero_cov && is_identity4(DT)) || s->t > c->max_kf_t_dist || s->r > c->max_kf_r_dist || s->N_prevKF_currF > 10)
        return 1;
    s->N_prevKF_currF++;
    return 0;
}
