// eigen_standin.h — a small stand-in for the part of Eigen 3 that the pose half of rubengooj/stvo-pl uses.
//
// TEST INFRASTRUCTURE (oracle/_ref).  The reference cannot be built here (no Eigen / OpenCV / Boost / yaml-cpp in the
// image), so oracle/make_ref.py extracts the UNMODIFIED function bodies of the pose path by line range from
// /root/reference and compiles them against this header instead of <eigen3/Eigen/...>.  Everything in this file is
// OURS, written from Eigen's documented semantics; nothing is copied from Eigen or from the reference:
//   * dense value type with eager evaluation (every expression materialises; coefficient arithmetic in the same order as
//     Eigen's lazy coefficient-wise evaluation for the expressions the path uses, e.g. (J J^T) w then +=),
//   * Matrix<double,R,C>, Identity / Zero / Constant, operator()(i,j) / (i), block / col / head / tail as assignable views,
//     the comma initialiser (scalars and matrices, row-major filling as Eigen does), transpose, norm, trace, inverse,
//     products, sums, scalar products / quotients, operator!=, array() == array() with all(),
//   * ColPivHouseholderQR (solve, logAbsDeterminant, info), SelfAdjointEigenSolver (eigenvalues, ascending).
// The 6x6 decompositions are therefore NOT Eigen's code: they are textbook algorithms (Householder QR with column
// pivoting, partial-pivoting LU, cyclic Jacobi) and agree with Eigen's to rounding, not bitwise; tests/test_oracle_ref.py
// cross-checks them against numpy.linalg (LAPACK).
#pragma once
#include <cassert>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <stdexcept>

namespace Eigen {

const int Dynamic = -1;
enum ComputationInfo { Success = 0, NumericalIssue = 1, NoConvergence = 2, InvalidInput = 3 };

class Block;
class CommaInit;
class ArrayView;

// ---- the one concrete value type: up to 6 x 6, row-major storage ---------------------------------------------
class M {
public:
    int r_, c_;
    double d_[36];
    M() : r_(0), c_(0) {}
    M(int r, int c) : r_(r), c_(c) { assert(r * c <= 36); std::memset(d_, 0, sizeof(d_)); }   // Eigen leaves it uninitialised; zero keeps the library deterministic
    int rows() const { return r_; }
    int cols() const { return c_; }
    int size() const { return r_ * c_; }
    double& operator()(int i, int j) { assert(i >= 0 && i < r_ && j >= 0 && j < c_); return d_[i * c_ + j]; }
    double operator()(int i, int j) const { assert(i >= 0 && i < r_ && j >= 0 && j < c_); return d_[i * c_ + j]; }
    double& operator()(int i) { assert(r_ == 1 || c_ == 1); assert(i >= 0 && i < r_ * c_); return d_[i]; }
    double operator()(int i) const { assert(r_ == 1 || c_ == 1); assert(i >= 0 && i < r_ * c_); return d_[i]; }
    double& operator[](int i) { return (*this)(i); }
    double operator[](int i) const { return (*this)(i); }

    M transpose() const {
        M t(c_, r_);
        for (int i = 0; i < r_; ++i)
            for (int j = 0; j < c_; ++j) t.d_[j * r_ + i] = d_[i * c_ + j];
        return t;
    }
    double squaredNorm() const {
        double s = 0.0;
        for (int i = 0; i < r_ * c_; ++i) s += d_[i] * d_[i];
        return s;
    }
    double norm() const { return std::sqrt(squaredNorm()); }
    double trace() const {
        double s = 0.0;
        for (int i = 0; i < r_ && i < c_; ++i) s += d_[i * c_ + i];
        return s;
    }
    double sum() const {
        double s = 0.0;
        for (int i = 0; i < r_ * c_; ++i) s += d_[i];
        return s;
    }
    M cross(const M& o) const {   // 3-vectors: Eigen's coefficient formulas, (1,2), (2,0), (0,1)
        assert(size() == 3 && o.size() == 3);
        M t(r_, c_);
        t.d_[0] = d_[1] * o.d_[2] - d_[2] * o.d_[1];
        t.d_[1] = d_[2] * o.d_[0] - d_[0] * o.d_[2];
        t.d_[2] = d_[0] * o.d_[1] - d_[1] * o.d_[0];
        return t;
    }
    M cwiseAbs() const {
        M t(r_, c_);
        for (int i = 0; i < r_ * c_; ++i) t.d_[i] = std::fabs(d_[i]);
        return t;
    }
    M inverse() const;            // square: partial-pivoting LU
    double determinant() const;   // square: partial-pivoting LU
    ArrayView array() const;

    Block block(int i, int j, int nr, int nc);
    M block(int i, int j, int nr, int nc) const;
    Block col(int j);
    M col(int j) const;
    Block row(int i);
    M row(int i) const;
    Block head(int n);
    M head(int n) const;
    Block tail(int n);
    M tail(int n) const;

    CommaInit operator<<(double v);
    CommaInit operator<<(const M& m);

    M& operator+=(const M& o) {
        assert(r_ == o.r_ && c_ == o.c_);
        for (int i = 0; i < r_ * c_; ++i) d_[i] += o.d_[i];
        return *this;
    }
    M& operator-=(const M& o) {
        assert(r_ == o.r_ && c_ == o.c_);
        for (int i = 0; i < r_ * c_; ++i) d_[i] -= o.d_[i];
        return *this;
    }
    M& operator*=(double s) {
        for (int i = 0; i < r_ * c_; ++i) d_[i] *= s;
        return *this;
    }
    M& operator/=(double s) {
        for (int i = 0; i < r_ * c_; ++i) d_[i] /= s;
        return *this;
    }
};

inline M operator+(const M& a, const M& b) {
    assert(a.r_ == b.r_ && a.c_ == b.c_);
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = a.d_[i] + b.d_[i];
    return t;
}
inline M operator-(const M& a, const M& b) {
    assert(a.r_ == b.r_ && a.c_ == b.c_);
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = a.d_[i] - b.d_[i];
    return t;
}
inline M operator-(const M& a) {
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = -a.d_[i];
    return t;
}
inline M operator*(const M& a, double s) {
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = a.d_[i] * s;
    return t;
}
inline M operator*(double s, const M& a) {
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = s * a.d_[i];
    return t;
}
inline M operator/(const M& a, double s) {
    M t(a.r_, a.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i) t.d_[i] = a.d_[i] / s;
    return t;
}
// matrix product, inner dimension accumulated in index order starting from the first product (Eigen's redux order for
// these small sizes)
inline M operator*(const M& a, const M& b) {
    assert(a.c_ == b.r_);
    M t(a.r_, b.c_);
    for (int i = 0; i < a.r_; ++i)
        for (int j = 0; j < b.c_; ++j) {
            double s = a.d_[i * a.c_] * b.d_[j];
            for (int k = 1; k < a.c_; ++k) s += a.d_[i * a.c_ + k] * b.d_[k * b.c_ + j];
            t.d_[i * b.c_ + j] = s;
        }
    return t;
}
inline bool operator==(const M& a, const M& b) {
    assert(a.r_ == b.r_ && a.c_ == b.c_);
    for (int i = 0; i < a.r_ * a.c_; ++i)
        if (!(a.d_[i] == b.d_[i])) return false;
    return true;
}
inline bool operator!=(const M& a, const M& b) { return !(a == b); }

// ---- array() comparisons: ((x - x).array() == (x - x).array()).all() ------------------------------------------
class BoolArray {
public:
    int n_;
    bool b_[36];
    bool all() const {
        for (int i = 0; i < n_; ++i)
            if (!b_[i]) return false;
        return true;
    }
    bool any() const {
        for (int i = 0; i < n_; ++i)
            if (b_[i]) return true;
        return false;
    }
};
class ArrayView {
public:
    M m_;
    explicit ArrayView(const M& m) : m_(m) {}
};
inline BoolArray operator==(const ArrayView& a, const ArrayView& b) {
    assert(a.m_.r_ == b.m_.r_ && a.m_.c_ == b.m_.c_);
    BoolArray r;
    r.n_ = a.m_.size();
    for (int i = 0; i < r.n_; ++i) r.b_[i] = (a.m_.d_[i] == b.m_.d_[i]);
    return r;
}
inline ArrayView M::array() const { return ArrayView(*this); }

// ---- assignable view of a sub-matrix ------------------------------------------------------------------------------
class Block {
public:
    M* p_;
    int i0_, j0_, nr_, nc_;
    Block(M* p, int i0, int j0, int nr, int nc) : p_(p), i0_(i0), j0_(j0), nr_(nr), nc_(nc) {
        assert(i0 >= 0 && j0 >= 0 && nr >= 0 && nc >= 0 && i0 + nr <= p->r_ && j0 + nc <= p->c_);
    }
    M eval() const {
        M t(nr_, nc_);
        for (int i = 0; i < nr_; ++i)
            for (int j = 0; j < nc_; ++j) t.d_[i * nc_ + j] = (*p_)(i0_ + i, j0_ + j);
        return t;
    }
    operator M() const { return eval(); }
    Block& operator=(const M& m) {
        assert(m.r_ == nr_ && m.c_ == nc_);
        for (int i = 0; i < nr_; ++i)
            for (int j = 0; j < nc_; ++j) (*p_)(i0_ + i, j0_ + j) = m.d_[i * m.c_ + j];
        return *this;
    }
    Block& operator=(const Block& b) { return (*this = b.eval()); }
    double& operator()(int i, int j) { return (*p_)(i0_ + i, j0_ + j); }
    double& operator()(int i) {
        assert(nr_ == 1 || nc_ == 1);
        return nc_ == 1 ? (*p_)(i0_ + i, j0_) : (*p_)(i0_, j0_ + i);
    }
    Block head(int n) { assert(nr_ == 1 || nc_ == 1); return nc_ == 1 ? Block(p_, i0_, j0_, n, 1) : Block(p_, i0_, j0_, 1, n); }
    Block tail(int n) {
        assert(nr_ == 1 || nc_ == 1);
        return nc_ == 1 ? Block(p_, i0_ + nr_ - n, j0_, n, 1) : Block(p_, i0_, j0_ + nc_ - n, 1, n);
    }
    M transpose() const { return eval().transpose(); }
    double norm() const { return eval().norm(); }
    CommaInit operator<<(double v);
    CommaInit operator<<(const M& m);
};
inline Block M::block(int i, int j, int nr, int nc) { return Block(this, i, j, nr, nc); }
inline M M::block(int i, int j, int nr, int nc) const { return Block(const_cast<M*>(this), i, j, nr, nc).eval(); }
inline Block M::col(int j) { return Block(this, 0, j, r_, 1); }
inline M M::col(int j) const { return Block(const_cast<M*>(this), 0, j, r_, 1).eval(); }
inline Block M::row(int i) { return Block(this, i, 0, 1, c_); }
inline M M::row(int i) const { return Block(const_cast<M*>(this), i, 0, 1, c_).eval(); }
inline Block M::head(int n) { assert(r_ == 1 || c_ == 1); return c_ == 1 ? Block(this, 0, 0, n, 1) : Block(this, 0, 0, 1, n); }
inline M M::head(int n) const { return const_cast<M*>(this)->head(n).eval(); }
inline Block M::tail(int n) {
    assert(r_ == 1 || c_ == 1);
    return c_ == 1 ? Block(this, r_ - n, 0, n, 1) : Block(this, 0, c_ - n, 1, n);
}
inline M M::tail(int n) const { return const_cast<M*>(this)->tail(n).eval(); }

// ---- comma initialiser: fills the destination row by row, blocks placed left to right (Eigen::CommaInitializer) ----
class CommaInit {
public:
    Block dst_;
    int row_, col_, cur_rows_;
    CommaInit(const Block& dst) : dst_(dst), row_(0), col_(0), cur_rows_(1) {}
    CommaInit& put(double v) {
        if (col_ == dst_.nc_) { row_ += cur_rows_; col_ = 0; cur_rows_ = 1; }
        assert(row_ < dst_.nr_ && col_ < dst_.nc_);
        dst_(row_, col_++) = v;
        return *this;
    }
    CommaInit& put(const M& m) {
        if (m.r_ == 0 || m.c_ == 0) return *this;
        if (col_ == dst_.nc_) { row_ += cur_rows_; col_ = 0; cur_rows_ = m.r_; }
        if (col_ == 0) cur_rows_ = m.r_;
        assert(m.r_ == cur_rows_ && row_ + m.r_ <= dst_.nr_ && col_ + m.c_ <= dst_.nc_);
        for (int i = 0; i < m.r_; ++i)
            for (int j = 0; j < m.c_; ++j) dst_(row_ + i, col_ + j) = m.d_[i * m.c_ + j];
        col_ += m.c_;
        return *this;
    }
    CommaInit& operator,(double v) { return put(v); }
    CommaInit& operator,(const M& m) { return put(m); }
};
inline CommaInit M::operator<<(double v) { CommaInit c(Block(this, 0, 0, r_, c_)); c.put(v); return c; }
inline CommaInit M::operator<<(const M& m) { const M tmp = m; CommaInit c(Block(this, 0, 0, r_, c_)); c.put(tmp); return c; }
inline CommaInit Block::operator<<(double v) { CommaInit c(*this); c.put(v); return c; }
inline CommaInit Block::operator<<(const M& m) { const M tmp = m; CommaInit c(*this); c.put(tmp); return c; }

// ---- LU with partial pivoting: inverse and determinant -----------------------------------------------------------
inline bool lu_decompose(M& a, int* piv, int& sign) {
    const int n = a.r_;
    sign = 1;
    for (int i = 0; i < n; ++i) piv[i] = i;
    bool ok = true;
    for (int k = 0; k < n; ++k) {
        int p = k;
        double big = std::fabs(a(k, k));
        for (int i = k + 1; i < n; ++i)
            if (std::fabs(a(i, k)) > big) { big = std::fabs(a(i, k)); p = i; }
        if (p != k) {
            for (int j = 0; j < n; ++j) std::swap(a(k, j), a(p, j));
            std::swap(piv[k], piv[p]);
            sign = -sign;
        }
        if (a(k, k) == 0.0) { ok = false; continue; }
        for (int i = k + 1; i < n; ++i) {
            a(i, k) /= a(k, k);
            const double f = a(i, k);
            for (int j = k + 1; j < n; ++j) a(i, j) -= f * a(k, j);
        }
    }
    return ok;
}
inline double M::determinant() const {
    assert(r_ == c_);
    M a = *this;
    int piv[6], sign;
    lu_decompose(a, piv, sign);
    double d = sign;
    for (int i = 0; i < r_; ++i) d *= a(i, i);
    return d;
}
inline M M::inverse() const {
    assert(r_ == c_);
    const int n = r_;
    M a = *this, inv(n, n);
    int piv[6], sign;
    lu_decompose(a, piv, sign);
    for (int c = 0; c < n; ++c) {
        double y[6];
        for (int i = 0; i < n; ++i) {   // L y = P e_c
            double s = (piv[i] == c) ? 1.0 : 0.0;
            for (int k = 0; k < i; ++k) s -= a(i, k) * y[k];
            y[i] = s;
        }
        for (int i = n - 1; i >= 0; --i) {   // U x = y
            double s = y[i];
            for (int k = i + 1; k < n; ++k) s -= a(i, k) * inv(k, c);
            inv(i, c) = s / a(i, i);
        }
    }
    return inv;
}

// ---- Matrix<Scalar, Rows, Cols>: the typed front of M --------------------------------------------------------------
template <typename S, int R, int C>
class Matrix : public M {
public:
    Matrix() : M(R > 0 ? R : 0, C > 0 ? C : 0) {}
    Matrix(const M& m) : M(m) { assert((R < 0 || m.r_ == R) && (C < 0 || m.c_ == C)); }
    Matrix(const Block& b) : M(b.eval()) { assert((R < 0 || r_ == R) && (C < 0 || c_ == C)); }
    Matrix(const Matrix& o) : M(o) {}
    // (rows, cols) for dynamic matrices; (x, y) for fixed 2-vectors
    template <typename A, typename B>
    Matrix(const A& a, const B& b) : M(R > 0 ? R : 0, C > 0 ? C : 0) {
        if (R < 0 || C < 0) { r_ = (int)a; c_ = (int)b; assert(r_ * c_ <= 36); }
        else { assert(R * C == 2); d_[0] = (double)a; d_[1] = (double)b; }
    }
    Matrix(double x, double y, double z) : M(R, C) { assert(R * C == 3); d_[0] = x; d_[1] = y; d_[2] = z; }
    Matrix& operator=(const M& m) {
        assert((R < 0 || m.r_ == R) && (C < 0 || m.c_ == C));
        M::operator=(m);
        return *this;
    }
    Matrix& operator=(const Matrix& o) { M::operator=(o); return *this; }
    Matrix& operator=(const Block& b) { return (*this = b.eval()); }
    static Matrix Zero() { Matrix m; for (int i = 0; i < R * C; ++i) m.d_[i] = 0.0; return m; }
    static Matrix Zero(int r, int c) { Matrix m(r, c); for (int i = 0; i < r * c; ++i) m.d_[i] = 0.0; return m; }
    static Matrix Constant(double v) { Matrix m; for (int i = 0; i < R * C; ++i) m.d_[i] = v; return m; }
    static Matrix Identity() {
        Matrix m = Zero();
        for (int i = 0; i < R && i < C; ++i) m.d_[i * C + i] = 1.0;
        return m;
    }
};
typedef Matrix<double, 2, 2> Matrix2d;
typedef Matrix<double, 3, 3> Matrix3d;
typedef Matrix<double, 4, 4> Matrix4d;
typedef Matrix<double, 2, 1> Vector2d;
typedef Matrix<double, 3, 1> Vector3d;
typedef Matrix<double, 4, 1> Vector4d;
typedef Matrix<double, Dynamic, Dynamic> MatrixXd;
typedef Matrix<double, Dynamic, 1> VectorXd;

// ---- ColPivHouseholderQR: A P = Q R, column pivoting by largest remaining column norm ----------------------------------
template <typename MT>
class ColPivHouseholderQR {
public:
    int n_;
    M qr_;            // R in the upper triangle, Householder vectors below
    double tau_[6];
    int perm_[6];
    int rank_;
    explicit ColPivHouseholderQR(const M& a) : n_(a.r_), qr_(a) {
        assert(a.r_ == a.c_ && n_ <= 6);
        double cn[6];
        for (int j = 0; j < n_; ++j) {
            perm_[j] = j;
            double s = 0.0;
            for (int i = 0; i < n_; ++i) s += qr_(i, j) * qr_(i, j);
            cn[j] = s;
        }
        for (int k = 0; k < n_; ++k) {
            int p = k;
            double big = -1.0;
            for (int j = k; j < n_; ++j) {   // exact remaining norms (recomputed: 6 x 6, no downdating error)
                double s = 0.0;
                for (int i = k; i < n_; ++i) s += qr_(i, j) * qr_(i, j);
                cn[j] = s;
                if (s > big) { big = s; p = j; }
            }
            if (p != k) {
                for (int i = 0; i < n_; ++i) std::swap(qr_(i, k), qr_(i, p));
                std::swap(perm_[k], perm_[p]);
            }
            // Householder reflector for column k, rows k..n-1: H = I - tau v v^T, v(k) = 1
            double tail = 0.0;
            for (int i = k + 1; i < n_; ++i) tail += qr_(i, k) * qr_(i, k);
            const double c0 = qr_(k, k);
            if (tail == 0.0) { tau_[k] = 0.0; continue; }
            double beta = std::sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            for (int i = k + 1; i < n_; ++i) qr_(i, k) /= (c0 - beta);
            tau_[k] = (beta - c0) / beta;
            qr_(k, k) = beta;
            for (int j = k + 1; j < n_; ++j) {
                double s = qr_(k, j);
                for (int i = k + 1; i < n_; ++i) s += qr_(i, k) * qr_(i, j);
                s *= tau_[k];
                qr_(k, j) -= s;
                for (int i = k + 1; i < n_; ++i) qr_(i, j) -= s * qr_(i, k);
            }
        }
        // numerical rank with Eigen's default threshold: |R(i,i)| > eps * n * max|R(j,j)|
        double maxpiv = 0.0;
        for (int i = 0; i < n_; ++i) maxpiv = std::max(maxpiv, std::fabs(qr_(i, i)));
        const double thr = 2.220446049250313e-16 * n_ * maxpiv;
        rank_ = 0;
        for (int i = 0; i < n_; ++i)
            if (std::fabs(qr_(i, i)) > thr) ++rank_;
    }
    M solve(const M& b) const {
        assert(b.r_ == n_ && b.c_ == 1);
        double c[6];
        for (int i = 0; i < n_; ++i) c[i] = b.d_[i];
        for (int k = 0; k < n_; ++k) {   // c = Q^T b
            if (tau_[k] == 0.0) continue;
            double s = c[k];
            for (int i = k + 1; i < n_; ++i) s += qr_(i, k) * c[i];
            s *= tau_[k];
            c[k] -= s;
            for (int i = k + 1; i < n_; ++i) c[i] -= s * qr_(i, k);
        }
        double y[6] = {0, 0, 0, 0, 0, 0};
        for (int i = rank_ - 1; i >= 0; --i) {   // leading rank x rank triangle; the rest of the solution is zero
            double s = c[i];
            for (int k = i + 1; k < rank_; ++k) s -= qr_(i, k) * y[k];
            y[i] = s / qr_(i, i);
        }
        M x(n_, 1);
        for (int i = 0; i < n_; ++i) x.d_[perm_[i]] = y[i];
        return x;
    }
    double logAbsDeterminant() const {
        double s = 0.0;
        for (int i = 0; i < n_; ++i) s += std::log(std::fabs(qr_(i, i)));
        return s;
    }
    ComputationInfo info() const { return Success; }
    int rank() const { return rank_; }
};

// ---- SelfAdjointEigenSolver: eigenvalues of the symmetric matrix given by the LOWER triangle, ascending ---------------
template <typename MT>
class SelfAdjointEigenSolver {
public:
    M w_;
    explicit SelfAdjointEigenSolver(const M& a) : w_(a.r_, 1) {
        const int n = a.r_;
        assert(a.r_ == a.c_ && n <= 6);
        double s[6][6];
        for (int i = 0; i < n; ++i)
            for (int j = 0; j <= i; ++j) s[i][j] = s[j][i] = a(i, j);
        for (int sweep = 0; sweep < 64; ++sweep) {   // cyclic Jacobi
            double off = 0.0;
            for (int i = 0; i < n; ++i)
                for (int j = 0; j < i; ++j) off += s[i][j] * s[i][j];
            if (off == 0.0) break;
            for (int p = 0; p < n - 1; ++p)
                for (int q = p + 1; q < n; ++q) {
                    if (s[p][q] == 0.0) continue;
                    const double theta = (s[q][q] - s[p][p]) / (2.0 * s[p][q]);
                    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                    const double c = 1.0 / std::sqrt(t * t + 1.0), sn = t * c;
                    for (int k = 0; k < n; ++k) {
                        const double kp = s[k][p], kq = s[k][q];
                        s[k][p] = c * kp - sn * kq;
                        s[k][q] = sn * kp + c * kq;
                    }
                    for (int k = 0; k < n; ++k) {
                        const double pk = s[p][k], qk = s[q][k];
                        s[p][k] = c * pk - sn * qk;
                        s[q][k] = sn * pk + c * qk;
                    }
                }
        }
        for (int i = 0; i < n; ++i) w_.d_[i] = s[i][i];
        for (int i = 1; i < n; ++i) {   // insertion sort (NaN-safe: never indexes out of range)
            const double v = w_.d_[i];
            int j = i - 1;
            while (j >= 0 && w_.d_[j] > v) { w_.d_[j + 1] = w_.d_[j]; --j; }
            w_.d_[j + 1] = v;
        }
    }
    const M& eigenvalues() const { return w_; }
    ComputationInfo info() const { return Success; }
};

}  // namespace Eigen
