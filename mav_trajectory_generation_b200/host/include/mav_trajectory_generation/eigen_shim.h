// eigen_shim.h -- the few Eigen types the reference's public API exposes (Eigen::VectorXd in
// Vertex/Polynomial/Segment, Eigen::MatrixXd in the debug accessors, Eigen::Matrix<double,N,N>
// in the static helpers of PolynomialOptimization<N>).
//
// When a real Eigen is on the include path it is used and this file defines nothing: callers
// keep their Eigen types and the ABI of this library's headers is unchanged.  This image ships
// no Eigen, so a minimal dense vector / matrix with the same spelling for the members used at
// the API boundary is provided instead.  It is NOT a linear-algebra library: all solving
// happens on the GPU behind include/mtg_b200.h.
#ifndef MAV_TRAJECTORY_GENERATION_EIGEN_SHIM_H_
#define MAV_TRAJECTORY_GENERATION_EIGEN_SHIM_H_

#if defined(__has_include)
#if __has_include(<Eigen/Core>) && !defined(MTG_FORCE_EIGEN_SHIM)
#define MTG_HAVE_EIGEN 1
#endif
#endif

#ifdef MTG_HAVE_EIGEN
#include <Eigen/Core>
#include <Eigen/StdVector>
#else

#include <cmath>
#include <cstddef>
#include <initializer_list>
#include <memory>
#include <complex>
#include <ostream>
#include <vector>

namespace Eigen {

typedef std::ptrdiff_t Index;
const int Dynamic = -1;
enum NoChange_t { NoChange };

template <typename T>
using aligned_allocator = std::allocator<T>;

// Column-major dense storage, like Eigen's default.
template <typename Scalar, int Rows_, int Cols_>
class Matrix {
 public:
  Matrix() : rows_(Rows_ > 0 ? Rows_ : 0), cols_(Cols_ > 0 ? Cols_ : (Cols_ == 1 ? 1 : 0)) {
    data_.assign(size_t(rows_) * cols_, Scalar(0));
  }
  explicit Matrix(Index n) : rows_(Cols_ == 1 ? n : (Rows_ > 0 ? Rows_ : n)), cols_(Cols_ == 1 ? 1 : (Cols_ > 0 ? Cols_ : n)) {
    data_.assign(size_t(rows_) * cols_, Scalar(0));
  }
  Matrix(Index r, Index c) : rows_(r), cols_(c) { data_.assign(size_t(r) * c, Scalar(0)); }
  Matrix(Scalar x, Scalar y, Scalar z) : rows_(3), cols_(1), data_{x, y, z} {}

  Index rows() const { return rows_; }
  Index cols() const { return cols_; }
  Index size() const { return rows_ * cols_; }
  void resize(Index r, Index c) {
    rows_ = r;
    cols_ = c;
    data_.assign(size_t(r) * c, Scalar(0));
  }
  void resize(Index n) { resize(Cols_ == 1 ? n : rows_, Cols_ == 1 ? 1 : n); }
  void resize(Index r, NoChange_t) { resize(r, cols_); }
  void conservativeResize(Index n) {
    data_.resize(size_t(n), Scalar(0));
    rows_ = n;
    cols_ = 1;
  }
  Matrix& setZero() {
    for (auto& v : data_) v = Scalar(0);
    return *this;
  }
  Matrix& setZero(Index n) {
    resize(n);
    return *this;
  }
  Matrix& setConstant(Scalar c) {
    for (auto& v : data_) v = c;
    return *this;
  }
  Matrix& setOnes() { return setConstant(Scalar(1)); }
  static Matrix Zero(Index n) { return Matrix(n); }
  static Matrix Zero(Index r, Index c) { return Matrix(r, c); }
  static Matrix Constant(Index n, Scalar c) {
    Matrix m(n);
    m.setConstant(c);
    return m;
  }
  static Matrix Identity(Index r, Index c) {
    Matrix m(r, c);
    for (Index i = 0; i < (r < c ? r : c); ++i) m(i, i) = Scalar(1);
    return m;
  }

  Scalar& operator()(Index i, Index j) { return data_[size_t(j) * rows_ + i]; }
  const Scalar& operator()(Index i, Index j) const { return data_[size_t(j) * rows_ + i]; }
  Scalar& operator()(Index i) { return data_[size_t(i)]; }
  const Scalar& operator()(Index i) const { return data_[size_t(i)]; }
  Scalar& operator[](Index i) { return data_[size_t(i)]; }
  const Scalar& operator[](Index i) const { return data_[size_t(i)]; }
  Scalar* data() { return data_.data(); }
  const Scalar* data() const { return data_.data(); }
  Scalar& x() { return data_[0]; }
  Scalar& y() { return data_[1]; }
  Scalar& z() { return data_[2]; }
  const Scalar& x() const { return data_[0]; }
  const Scalar& y() const { return data_[1]; }
  const Scalar& z() const { return data_[2]; }

  Scalar squaredNorm() const {
    Scalar s(0);
    for (const auto& v : data_) s += v * v;
    return s;
  }
  Scalar norm() const { return std::sqrt(squaredNorm()); }
  // Eigen's dot, cross, normalize and normalized: sums in index order, cross products as (y z' - z y', ...), and
  // normalisation by one division by sqrt(squaredNorm()) (a zero vector is left as it is)
  template <int R2, int C2>
  Scalar dot(const Matrix<Scalar, R2, C2>& o) const {
    Scalar s = size() > 0 ? data_[0] * o.data()[0] : Scalar(0);
    for (Index i = 1; i < size(); ++i) s += data_[size_t(i)] * o.data()[i];
    return s;
  }
  template <int R2, int C2>
  Matrix cross(const Matrix<Scalar, R2, C2>& o) const {
    Matrix r(*this);
    r[0] = data_[1] * o[2] - data_[2] * o[1];
    r[1] = data_[2] * o[0] - data_[0] * o[2];
    r[2] = data_[0] * o[1] - data_[1] * o[0];
    return r;
  }
  void normalize() {
    const Scalar z = squaredNorm();
    if (z > Scalar(0)) {
      const Scalar n = std::sqrt(z);
      for (auto& v : data_) v /= n;
    }
  }
  Matrix normalized() const {
    Matrix r(*this);
    r.normalize();
    return r;
  }
  Scalar sum() const {
    Scalar s(0);
    for (const auto& v : data_) s += v;
    return s;
  }
  Scalar maxCoeff() const {
    Scalar m = data_.empty() ? Scalar(0) : data_[0];
    for (const auto& v : data_) m = v > m ? v : m;
    return m;
  }
  bool isZero(Scalar tol = Scalar(1e-12)) const {
    for (const auto& v : data_)
      if (std::abs(v) > tol) return false;
    return true;
  }
  template <int R2, int C2>
  bool isApprox(const Matrix<Scalar, R2, C2>& o, Scalar tol = Scalar(1e-12)) const {
    if (o.rows() != rows_ || o.cols() != cols_) return false;
    Scalar d(0), n(0);
    for (Index i = 0; i < size(); ++i) {
      d += (data_[i] - o.data()[i]) * (data_[i] - o.data()[i]);
      n += data_[i] * data_[i];
    }
    return d <= tol * tol * n || d == Scalar(0);
  }
  Matrix<Scalar, Dynamic, Dynamic> transpose() const {
    Matrix<Scalar, Dynamic, Dynamic> t(cols_, rows_);
    for (Index i = 0; i < rows_; ++i)
      for (Index j = 0; j < cols_; ++j) t(j, i) = (*this)(i, j);
    return t;
  }
  Matrix head(Index n) const {
    Matrix r(n);
    for (Index i = 0; i < n; ++i) r[i] = data_[i];
    return r;
  }
  Matrix tail(Index n) const {
    Matrix r(n);
    for (Index i = 0; i < n; ++i) r[i] = data_[size_t(size() - n + i)];
    return r;
  }
  template <int R2, int C2>
  Matrix(const Matrix<Scalar, R2, C2>& o) : rows_(o.rows()), cols_(o.cols()), data_(o.data(), o.data() + o.size()) {}

  bool operator==(const Matrix& o) const { return rows_ == o.rows_ && cols_ == o.cols_ && data_ == o.data_; }
  bool operator!=(const Matrix& o) const { return !(*this == o); }
  Matrix operator+(const Matrix& o) const {
    Matrix r(*this);
    for (Index i = 0; i < size(); ++i) r.data_[i] += o.data_[i];
    return r;
  }
  Matrix operator-(const Matrix& o) const {
    Matrix r(*this);
    for (Index i = 0; i < size(); ++i) r.data_[i] -= o.data_[i];
    return r;
  }
  Matrix operator-() const {
    Matrix r(*this);
    for (auto& v : r.data_) v = -v;
    return r;
  }
  Matrix& operator+=(const Matrix& o) {
    for (Index i = 0; i < size(); ++i) data_[i] += o.data_[i];
    return *this;
  }
  Matrix& operator-=(const Matrix& o) {
    for (Index i = 0; i < size(); ++i) data_[i] -= o.data_[i];
    return *this;
  }
  Matrix operator*(Scalar s) const {
    Matrix r(*this);
    for (auto& v : r.data_) v *= s;
    return r;
  }
  Matrix operator/(Scalar s) const {
    Matrix r(*this);
    for (auto& v : r.data_) v /= s;
    return r;
  }

 private:
  Index rows_, cols_;
  std::vector<Scalar> data_;
};

template <typename S, int R, int C>
Matrix<S, R, C> operator*(S s, const Matrix<S, R, C>& m) {
  return m * s;
}

// matrix * (matrix | vector)
template <typename S, int R1, int C1, int R2, int C2>
Matrix<S, Dynamic, C2> operator*(const Matrix<S, R1, C1>& a, const Matrix<S, R2, C2>& b) {
  Matrix<S, Dynamic, C2> r;
  r.resize(a.rows(), b.cols());
  for (Index i = 0; i < a.rows(); ++i)
    for (Index j = 0; j < b.cols(); ++j) {
      S s(0);
      for (Index k = 0; k < a.cols(); ++k) s += a(i, k) * b(k, j);
      r(i, j) = s;
    }
  return r;
}

template <typename S, int R, int C>
std::ostream& operator<<(std::ostream& os, const Matrix<S, R, C>& m) {
  for (Index i = 0; i < m.rows(); ++i) {
    for (Index j = 0; j < m.cols(); ++j) os << (j ? " " : "") << m(i, j);
    if (i + 1 < m.rows()) os << "\n";
  }
  return os;
}

typedef Matrix<double, Dynamic, 1> VectorXd;
typedef Matrix<double, Dynamic, Dynamic> MatrixXd;
typedef Matrix<double, 3, 1> Vector3d;
typedef Matrix<std::complex<double>, Dynamic, 1> VectorXcd;

}  // namespace Eigen
#endif  // MTG_HAVE_EIGEN
#endif  // MAV_TRAJECTORY_GENERATION_EIGEN_SHIM_H_
