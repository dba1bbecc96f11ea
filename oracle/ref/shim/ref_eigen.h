// Compile-time stand-in for the part of Eigen the reference's front end and odometry use (fixed-size matrices, quaternions,
// SelfAdjointEigenSolver<Matrix3d>, colPivHouseholderQr().solve).  Element-wise arithmetic is the plain IEEE operation Eigen
// performs; every routine with an order of operations of its own forwards to the oracle's from-knowledge restatement in
// oracle_math.h (qmul, qrot, qinv, qslerp, dot, eigen_sym3, colpiv_qr_solve_nx3), so these headers add no numerics.
#pragma once
#include <cmath>
#include <cstdlib>
#include <initializer_list>
#include "oracle_math.h"

#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define EIGEN_ALIGN16 __attribute__((aligned(16)))

namespace Eigen {

template <class Derived> struct MatrixBase {
    const Derived& derived() const { return static_cast<const Derived&>(*this); }
    Derived& derived() { return static_cast<Derived&>(*this); }
};
template <class Derived> struct QuaternionBase {};

template <class T, int R, int C> struct Matrix;

template <class T, int R, int C> struct CommaInit {
    Matrix<T, R, C>* m; int k;
    CommaInit& operator,(T v) { (*m)(k / C, k % C) = v; ++k; return *this; }
};

template <class T, int R, int C> struct ColPivHouseholderQR;

template <class T, int R, int C> struct Matrix : MatrixBase<Matrix<T, R, C>> {
    typedef T Scalar;
    T a[R * C];   // column-major, as Eigen stores it
    Matrix() { for (int i = 0; i < R * C; ++i) a[i] = T(0); }
    Matrix(T x, T y, T z) { static_assert(R * C == 3, "3-vector"); a[0] = x; a[1] = y; a[2] = z; }
    Matrix(std::initializer_list<T> l) { int i = 0; for (T v : l) a[i++] = v; }
    template <class D> Matrix(const MatrixBase<D>& o) { *this = o.derived(); }
    static Matrix Zero() { return Matrix(); }
    static Matrix Constant(T v) { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = v; return m; }
    static Matrix Ones() { return Constant(T(1)); }
    static Matrix Identity() { Matrix m; for (int i = 0; i < R && i < C; ++i) m(i, i) = T(1); return m; }
    T& operator()(int r, int c) { return a[c * R + r]; }
    const T& operator()(int r, int c) const { return a[c * R + r]; }
    T& operator()(int i) { return a[i]; }
    const T& operator()(int i) const { return a[i]; }
    T& operator[](int i) { return a[i]; }
    const T& operator[](int i) const { return a[i]; }
    T& x() { return a[0]; } T& y() { return a[1]; } T& z() { return a[2]; } T& w() { return a[3]; }
    const T& x() const { return a[0]; } const T& y() const { return a[1]; } const T& z() const { return a[2]; }
    const T& w() const { return a[3]; }
    int rows() const { return R; }
    int cols() const { return C; }
    int size() const { return R * C; }
    CommaInit<T, R, C> operator<<(T v) { a[0] = v; return CommaInit<T, R, C>{this, 1}; }

    Matrix operator+(const Matrix& o) const { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = a[i] + o.a[i]; return m; }
    Matrix operator-(const Matrix& o) const { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = a[i] - o.a[i]; return m; }
    Matrix operator-() const { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = -a[i]; return m; }
    Matrix operator*(T s) const { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = a[i] * s; return m; }
    Matrix operator/(T s) const { Matrix m; for (int i = 0; i < R * C; ++i) m.a[i] = a[i] / s; return m; }
    Matrix& operator+=(const Matrix& o) { for (int i = 0; i < R * C; ++i) a[i] += o.a[i]; return *this; }
    Matrix& operator-=(const Matrix& o) { for (int i = 0; i < R * C; ++i) a[i] -= o.a[i]; return *this; }
    Matrix& operator*=(T s) { for (int i = 0; i < R * C; ++i) a[i] *= s; return *this; }
    Matrix& operator/=(T s) { for (int i = 0; i < R * C; ++i) a[i] /= s; return *this; }
    // a product with an inner dimension of one (the outer products of the covariance sums) is one multiplication per entry;
    // no longer product is evaluated on the paths the harnesses drive
    template <int K> Matrix<T, R, K> operator*(const Matrix<T, C, K>& o) const {
        static_assert(C == 1, "only outer products are used");
        Matrix<T, R, K> m;
        for (int r = 0; r < R; ++r) for (int k = 0; k < K; ++k) m(r, k) = a[r] * o(0, k);
        return m;
    }
    Matrix<T, C, R> transpose() const { Matrix<T, C, R> m; for (int r = 0; r < R; ++r) for (int c = 0; c < C; ++c) m(c, r) = (*this)(r, c); return m; }
    Matrix<T, R, 1> col(int c) const { Matrix<T, R, 1> m; for (int r = 0; r < R; ++r) m.a[r] = (*this)(r, c); return m; }
    T sum() const { T s = a[0]; for (int i = 1; i < R * C; ++i) s += a[i]; return s; }
    T dot(const Matrix& o) const {
        static_assert(R * C == 3, "3-vector");
        return orc::dot(orc::V3{a[0], a[1], a[2]}, orc::V3{o.a[0], o.a[1], o.a[2]});
    }
    T squaredNorm() const { return dot(*this); }
    T norm() const { return orc::norm(orc::V3{a[0], a[1], a[2]}); }
    void normalize() { T z = squaredNorm(); if (z > T(0)) *this /= std::sqrt(z); }
    Matrix normalized() const { Matrix m = *this; m.normalize(); return m; }
    Matrix cross(const Matrix& o) const {
        orc::V3 c = orc::cross(orc::V3{a[0], a[1], a[2]}, orc::V3{o.a[0], o.a[1], o.a[2]});
        return Matrix(c.x, c.y, c.z);
    }
    ColPivHouseholderQR<T, R, C> colPivHouseholderQr() const { return ColPivHouseholderQR<T, R, C>{*this}; }
};

template <class T, int R, int C> Matrix<T, R, C> operator*(T s, const Matrix<T, R, C>& m) {
    Matrix<T, R, C> o; for (int i = 0; i < R * C; ++i) o.a[i] = s * m.a[i]; return o;
}

typedef Matrix<double, 3, 1> Vector3d;
typedef Matrix<float, 3, 1> Vector3f;
typedef Matrix<double, 3, 3> Matrix3d;
typedef Matrix<double, 4, 4> Matrix4d;

// colPivHouseholderQr().solve(b) on an n x 3 matrix: orc::colpiv_qr_solve_nx3
template <class T, int R, int C> struct ColPivHouseholderQR {
    Matrix<T, R, C> A;
    Matrix<T, C, 1> solve(const Matrix<T, R, 1>& b) const {
        static_assert(C == 3 && R <= 8, "n x 3 least squares");
        double rows[R * 3], rhs[R], x[3];
        for (int r = 0; r < R; ++r) { for (int c = 0; c < 3; ++c) rows[r * 3 + c] = A(r, c); rhs[r] = b(r); }
        orc::colpiv_qr_solve_nx3(R, rows, rhs, x);
        return Matrix<T, C, 1>(x[0], x[1], x[2]);
    }
};

// SelfAdjointEigenSolver<Matrix3d>: orc::eigen_sym3 (lower triangle read, ascending eigenvalues)
template <class M> struct SelfAdjointEigenSolver {
    Vector3d ev;
    Matrix3d evec;
    explicit SelfAdjointEigenSolver(const Matrix3d& A) {
        double a[3][3], e[3], v[3][3];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) a[r][c] = A(r, c);
        orc::eigen_sym3(a, e, v);
        for (int r = 0; r < 3; ++r) { ev(r) = e[r]; for (int c = 0; c < 3; ++c) evec(r, c) = v[r][c]; }
    }
    const Vector3d& eigenvalues() const { return ev; }
    const Matrix3d& eigenvectors() const { return evec; }
};

template <class T> struct Quaternion : QuaternionBase<Quaternion<T>> {
    typedef T Scalar;
    T w_, x_, y_, z_;
    Quaternion() : w_(1), x_(0), y_(0), z_(0) {}
    Quaternion(T w, T x, T y, T z) : w_(w), x_(x), y_(y), z_(z) {}
    static Quaternion Identity() { return Quaternion(1, 0, 0, 0); }
    T& w() { return w_; } T& x() { return x_; } T& y() { return y_; } T& z() { return z_; }
    const T& w() const { return w_; } const T& x() const { return x_; } const T& y() const { return y_; } const T& z() const { return z_; }
    Matrix<T, 3, 1> vec() const { return Matrix<T, 3, 1>(x_, y_, z_); }
    static Quaternion of(orc::Quat q) { return Quaternion(q.w, q.x, q.y, q.z); }
    orc::Quat q() const { return orc::Quat{w_, x_, y_, z_}; }
    Quaternion operator*(const Quaternion& o) const { return of(orc::qmul(q(), o.q())); }
    Quaternion& operator*=(const Quaternion& o) { *this = *this * o; return *this; }
    Matrix<T, 3, 1> operator*(const Matrix<T, 3, 1>& v) const {
        orc::V3 r = orc::qrot(q(), orc::V3{v(0), v(1), v(2)});
        return Matrix<T, 3, 1>(r.x, r.y, r.z);
    }
    Quaternion inverse() const { return of(orc::qinv(q())); }
    Quaternion conjugate() const { return Quaternion(w_, -x_, -y_, -z_); }
    Quaternion slerp(T t, const Quaternion& o) const { return of(orc::qslerp(q(), t, o.q())); }
    Matrix<T, 3, 3> toRotationMatrix() const { std::abort(); }
};
typedef Quaternion<double> Quaterniond;
typedef Quaternion<float> Quaternionf;

template <class T> struct AngleAxis {
    template <class M> AngleAxis& fromRotationMatrix(const M&) { std::abort(); }
    T angle() const { std::abort(); }
    Matrix<T, 3, 1> axis() const { std::abort(); }
};

}  // namespace Eigen
