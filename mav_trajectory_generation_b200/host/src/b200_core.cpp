// b200_core.cpp -- host side above the C-ABI: constraint bookkeeping (the reference's
// setupFromVertices / setupConstraintReorderingMatrix, impl/polynomial_optimization_linear_impl.h
// :56-109, :181-260, as flat index arrays), packing/unpacking, and calls into libmtg_b200.so.
#include "mav_trajectory_generation/b200_core.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../csrc/mtg_tables.h"
#include "mtg_b200.h"

namespace mav_trajectory_generation {
namespace b200 {

namespace {
std::mutex g_handle_mutex;
std::recursive_mutex g_call_mutex;
mtg_handle* g_handle = nullptr;

const double kA1Inv2[] = MTG_A1INV_2;
const double kA1Inv4[] = MTG_A1INV_4;
const double kA1Inv6[] = MTG_A1INV_6;
const double kA1Inv8[] = MTG_A1INV_8;
const double kA1Inv10[] = MTG_A1INV_10;
const double kA1Inv12[] = MTG_A1INV_12;
const double* a1inv(int N) {
  switch (N) {
    case 2: return kA1Inv2;
    case 4: return kA1Inv4;
    case 6: return kA1Inv6;
    case 8: return kA1Inv8;
    case 10: return kA1Inv10;
    default: return kA1Inv12;
  }
}
double baseCoeff(int d, int j) {  // j!/(j-d)!
  double b = 1.0;
  for (int k = 0; k < d; ++k) b *= double(j - k);
  return j >= d ? b : 0.0;
}
}  // namespace

mtg_handle* defaultHandle() {
  std::lock_guard<std::mutex> lock(g_handle_mutex);
  if (g_handle == nullptr) {
    int device = 0;
    if (const char* env = std::getenv("MTG_B200_DEVICE")) device = std::atoi(env);
    const int rc = mtg_create(device, &g_handle);
    if (rc != MTG_OK)
      LOG(FATAL) << "mtg_create(device " << device << ") failed (rc=" << rc << "): " << mtg_last_error(nullptr)
                 << " -- the H100 CUDA path is the only solver path; there is no CPU fallback.";
  }
  return g_handle;
}
void lockHandle() { g_call_mutex.lock(); }
void unlockHandle() { g_call_mutex.unlock(); }

namespace {
struct HandleLock {
  HandleLock() { lockHandle(); }
  ~HandleLock() { unlockHandle(); }
};
}  // namespace

void hostMappingMatrix(int N, double T, double* A) {
  const int h = N / 2;
  for (int i = 0; i < N * N; ++i) A[i] = 0.0;
  for (int k = 0; k < h; ++k) {
    A[k * N + k] = baseCoeff(k, k);
    double tp = 1.0;
    for (int j = k; j < N; ++j) {
      A[(h + k) * N + j] = baseCoeff(k, j) * tp;
      tp *= T;
    }
  }
}

void hostInverseMappingMatrix(int N, double T, double* Ai) {
  const int h = N / 2;
  const double* A1 = a1inv(N);
  double tp[MTG_MAX_N], itp[MTG_MAX_N];
  tp[0] = itp[0] = 1.0;
  for (int k = 1; k < N; ++k) {
    tp[k] = tp[k - 1] * T;
    itp[k] = itp[k - 1] / T;
  }
  for (int j = 0; j < N; ++j)
    for (int s = 0; s < N; ++s) Ai[j * N + s] = (j < h ? A1[j * N + s] : itp[j] * A1[j * N + s] * tp[s % h]);
  // for j < h the scaling T^-j * T^(s mod h) acts on a diagonal (s == j) entry only and cancels
}

void hostInvertStructured(int N, const double* A, double* Ai) {
  const int h = N / 2;
  for (int i = 0; i < N * N; ++i) Ai[i] = 0.0;
  // Lambda^-1 (the upper-left block is diagonal)
  for (int k = 0; k < h; ++k) Ai[k * N + k] = 1.0 / A[k * N + k];
  // Dm^-1 by Gauss-Jordan with partial pivoting on the lower-right h x h block
  double M[MTG_MAX_N / 2][MTG_MAX_N];
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < h; ++j) {
      M[i][j] = A[(h + i) * N + (h + j)];
      M[i][h + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < h; ++c) {
    int piv = c;
    for (int i = c + 1; i < h; ++i)
      if (std::abs(M[i][c]) > std::abs(M[piv][c])) piv = i;
    if (piv != c)
      for (int j = 0; j < 2 * h; ++j) std::swap(M[piv][j], M[c][j]);
    const double ip = 1.0 / M[c][c];
    for (int j = 0; j < 2 * h; ++j) M[c][j] *= ip;
    for (int i = 0; i < h; ++i) {
      if (i == c) continue;
      const double f = M[i][c];
      for (int j = 0; j < 2 * h; ++j) M[i][j] -= f * M[c][j];
    }
  }
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < h; ++j) Ai[(h + i) * N + (h + j)] = M[i][h + j];
  // lower-left block: -Dm^-1 C Lambda^-1
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < h; ++j) {
      double s = 0.0;
      for (int k = 0; k < h; ++k) s += M[i][h + k] * A[(h + k) * N + j];
      Ai[(h + i) * N + j] = -s * Ai[j * N + j];
    }
}

void hostCostMatrix(int N, int r, double T, double* Q) {
  for (int i = 0; i < N * N; ++i) Q[i] = 0.0;
  for (int a = r; a < N; ++a)
    for (int b = r; b < N; ++b) {
      const int e = a + b - 2 * r + 1;
      Q[a * N + b] = 2.0 * baseCoeff(r, a) * baseCoeff(r, b) * std::pow(T, double(e)) / double(e);
    }
}

void hostSegmentHessian(int N, int r, double T, double* H) {
  // Same exact-table scaling the kernels use: H(T) = T^(1-2r) S H(1) S.
  static const double k2_0[] = MTG_H1_2_0;
  static const double k4_0[] = MTG_H1_4_0, k4_1[] = MTG_H1_4_1;
  static const double k6_0[] = MTG_H1_6_0, k6_1[] = MTG_H1_6_1, k6_2[] = MTG_H1_6_2;
  static const double k8_0[] = MTG_H1_8_0, k8_1[] = MTG_H1_8_1, k8_2[] = MTG_H1_8_2, k8_3[] = MTG_H1_8_3;
  static const double k10_0[] = MTG_H1_10_0, k10_1[] = MTG_H1_10_1, k10_2[] = MTG_H1_10_2, k10_3[] = MTG_H1_10_3,
                      k10_4[] = MTG_H1_10_4;
  static const double k12_0[] = MTG_H1_12_0, k12_1[] = MTG_H1_12_1, k12_2[] = MTG_H1_12_2, k12_3[] = MTG_H1_12_3,
                      k12_4[] = MTG_H1_12_4, k12_5[] = MTG_H1_12_5;
  static const double* const tab[7][6] = {{nullptr}, {k2_0}, {k4_0, k4_1}, {k6_0, k6_1, k6_2},
                                          {k8_0, k8_1, k8_2, k8_3}, {k10_0, k10_1, k10_2, k10_3, k10_4},
                                          {k12_0, k12_1, k12_2, k12_3, k12_4, k12_5}};
  const int h = N / 2;
  const double* G = tab[h][r];
  double sp[MTG_MAX_N];
  sp[0] = 1.0;
  for (int k = 1; k < h; ++k) sp[k] = sp[k - 1] * T;
  const double rho = std::pow(T, double(1 - 2 * r));
  for (int a = 0; a < N; ++a)
    for (int b = 0; b < N; ++b) H[a * N + b] = rho * sp[a % h] * sp[b % h] * G[a * N + b];
}

void buildTopology(int N, int D, int r, Vertex::Vector* vertices, Topology* topo) {
  const int h = N / 2;
  const int K = static_cast<int>(vertices->size()) - 1;
  topo->N = N;
  topo->K = K;
  topo->D = D;
  topo->r = r;
  topo->mask.assign(size_t(K + 1) * h, 0);
  for (size_t v = 0; v < vertices->size(); ++v) {
    Vertex& vertex = (*vertices)[v];
    CHECK_EQ(vertex.D(), D) << "vertex dimension does not match the optimisation dimension";
    Vertex filtered(static_cast<size_t>(D));
    bool valid = true;
    for (auto it = vertex.cBegin(); it != vertex.cEnd(); ++it) {
      if (it->first > h - 1 || it->first < 0) {
        valid = false;
        LOG(WARNING) << "Invalid constraint on vertex " << v << ": maximum possible derivative is " << h - 1
                     << ", but was set to " << it->first << ". Ignoring constraint";
      } else {
        filtered.addConstraint(it->first, it->second);
        topo->mask[v * h + it->first] = 1;
      }
    }
    if (!valid) vertex = filtered;
  }
  mtg_problem p = {N, r, K, D, topo->mask.data()};
  mtg_layout lay;
  topo->slot_col.assign(size_t(K) * N, 0);
  const int rc = mtg_problem_layout(&p, &lay, topo->slot_col.data());
  CHECK_EQ(rc, MTG_OK) << "mtg_problem_layout rejected the problem";
  topo->n_all = lay.n_all;
  topo->n_fixed = lay.n_fixed;
  topo->n_free = lay.n_free;
  topo->kernel = lay.kernel;
}

void packFixed(const Topology& topo, const Vertex::Vector& vertices, double* d_fixed) {
  const int h = topo.N / 2;
  int col = 0;
  Eigen::VectorXd value;
  for (int v = 0; v <= topo.K; ++v)
    for (int k = 0; k < h; ++k)
      if (topo.mask[size_t(v) * h + k]) {
        CHECK(vertices[v].getConstraint(k, &value)) << "vertex " << v << " lacks constraint " << k;
        for (int d = 0; d < topo.D; ++d) d_fixed[size_t(d) * topo.n_fixed + col] = value[d];
        ++col;
      }
}

bool sameTopology(const Topology& topo, const Vertex::Vector& vertices) {
  const int h = topo.N / 2;
  if (static_cast<int>(vertices.size()) != topo.K + 1) return false;
  for (int v = 0; v <= topo.K; ++v) {
    if (vertices[v].D() != topo.D) return false;
    size_t expected = 0;
    for (int k = 0; k < h; ++k) {
      const bool want = topo.mask[size_t(v) * h + k] != 0;
      if (vertices[v].hasConstraint(k) != want) return false;
      expected += want;
    }
    if (vertices[v].getNumberOfConstraints() != expected) return false;  // a constraint above h-1
  }
  return true;
}

void unpackSegments(const Topology& topo, const double* coeffs, const double* times, Segment::Vector* segments) {
  segments->assign(static_cast<size_t>(topo.K), Segment(topo.N, topo.D));
  Eigen::VectorXd c(topo.N);
  for (int i = 0; i < topo.K; ++i) {
    Segment& seg = (*segments)[i];
    seg.setTime(times[i]);
    for (int d = 0; d < topo.D; ++d) {
      for (int j = 0; j < topo.N; ++j) c[j] = coeffs[(size_t(i) * topo.D + d) * topo.N + j];
      seg[d] = Polynomial(topo.N, c);
    }
  }
}

// ---- LinearCore --------------------------------------------------------------------------
LinearCore::LinearCore(int N, size_t dimension) : N_(N), dimension_(dimension) {
  fixed_constraints_compact_.resize(dimension_);
  free_constraints_compact_.resize(dimension_);
}

bool LinearCore::setupFromVertices(const Vertex::Vector& vertices, const std::vector<double>& times, int r) {
  CHECK(r >= 0 && r <= N_ / 2 - 1) << "You tried to optimize the " << r << "th derivative of position on a " << N_
                                  << "th order polynomial. This is not possible, you either need a higher "
                                     "order polynomial or a smaller derivative to optimize.";
  CHECK(vertices.size() == times.size() + 1) << "Size of times must be one less than positions.";
  CHECK_GE(vertices.size(), 2u);
  vertices_ = vertices;
  buildTopology(N_, static_cast<int>(dimension_), r, &vertices_, &topo_);
  segments_.assign(static_cast<size_t>(topo_.K), Segment(N_, static_cast<int>(dimension_)));
  updateSegmentTimes(times);
  std::vector<double> d_fixed(size_t(topo_.D) * topo_.n_fixed);
  packFixed(topo_, vertices_, d_fixed.data());
  for (size_t d = 0; d < dimension_; ++d) {
    fixed_constraints_compact_[d] = Eigen::VectorXd::Zero(topo_.n_fixed);
    free_constraints_compact_[d] = Eigen::VectorXd::Zero(topo_.n_free);
    for (int c = 0; c < topo_.n_fixed; ++c) fixed_constraints_compact_[d][c] = d_fixed[d * topo_.n_fixed + c];
  }
  return true;
}

void LinearCore::updateSegmentTimes(const std::vector<double>& times) {
  CHECK(times.size() == static_cast<size_t>(topo_.K))
      << "Number of segment times (" << times.size() << ") does not match number of segments (" << topo_.K << ")";
  for (double t : times) CHECK_GT(t, 0) << "Segment times need to be greater than zero";
  segment_times_ = times;
}

void LinearCore::unpack(const std::vector<double>& coeffs) {
  unpackSegments(topo_, coeffs.data(), segment_times_.data(), &segments_);
}

bool LinearCore::solveLinear() {
  CHECK(topo_.r >= 0 && topo_.r <= N_ / 2 - 1);
  const int D = topo_.D;
  std::vector<double> d_fixed(size_t(D) * topo_.n_fixed), d_free(size_t(D) * (topo_.n_free > 0 ? topo_.n_free : 1)),
      coeffs(size_t(topo_.K) * D * N_);
  for (int d = 0; d < D; ++d)
    for (int c = 0; c < topo_.n_fixed; ++c) d_fixed[size_t(d) * topo_.n_fixed + c] = fixed_constraints_compact_[d][c];
  int32_t status = 0;
  mtg_problem p = {N_, topo_.r, topo_.K, D, topo_.mask.data()};
  {
    HandleLock lock;
    mtg_handle* h = defaultHandle();
    const int rc = mtg_solve_linear_batch_host_f64(h, &p, 1, segment_times_.data(), d_fixed.data(), coeffs.data(),
                                                   d_free.data(), &status);
    if (rc != MTG_OK) {
      LOG(ERROR) << "mtg_solve_linear_batch_host_f64 failed (rc=" << rc << "): " << mtg_last_error(h);
      return false;
    }
  }
  last_status_ = status;
  if (status != 0) LOG(WARNING) << "solveLinear: kernel reported status " << status << " (see MTG_STATUS_*)";
  for (int d = 0; d < D; ++d) {
    free_constraints_compact_[d] = Eigen::VectorXd::Zero(topo_.n_free);
    for (int c = 0; c < topo_.n_free; ++c) free_constraints_compact_[d][c] = d_free[size_t(d) * topo_.n_free + c];
  }
  unpack(coeffs);
  return true;
}

void LinearCore::setFreeConstraints(const std::vector<Eigen::VectorXd>& free_constraints) {
  CHECK(free_constraints.size() == dimension_);
  for (const Eigen::VectorXd& v : free_constraints) CHECK(static_cast<int>(v.size()) == topo_.n_free);
  free_constraints_compact_ = free_constraints;
  const int D = topo_.D;
  std::vector<double> d_fixed(size_t(D) * topo_.n_fixed), d_free(size_t(D) * (topo_.n_free > 0 ? topo_.n_free : 1)),
      coeffs(size_t(topo_.K) * D * N_);
  for (int d = 0; d < D; ++d) {
    for (int c = 0; c < topo_.n_fixed; ++c) d_fixed[size_t(d) * topo_.n_fixed + c] = fixed_constraints_compact_[d][c];
    for (int c = 0; c < topo_.n_free; ++c) d_free[size_t(d) * topo_.n_free + c] = free_constraints[d][c];
  }
  mtg_problem p = {N_, topo_.r, topo_.K, D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_coeffs_from_constraints_batch_host_f64(h, &p, 1, segment_times_.data(), d_fixed.data(),
                                                            d_free.data(), coeffs.data());
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
  unpack(coeffs);
}

double LinearCore::computeCost() const {
  CHECK(static_cast<size_t>(topo_.K) == segments_.size());
  const int D = topo_.D;
  std::vector<double> coeffs(size_t(topo_.K) * D * N_);
  for (int i = 0; i < topo_.K; ++i)
    for (int d = 0; d < D; ++d) {
      const Eigen::VectorXd c = segments_[i][d].getCoefficients(0);
      for (int j = 0; j < N_; ++j) coeffs[(size_t(i) * D + d) * N_ + j] = c[j];
    }
  double cost = 0.0;
  mtg_problem p = {N_, topo_.r, topo_.K, D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_compute_cost_batch_host_f64(h, &p, 1, segment_times_.data(), coeffs.data(), &cost);
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
  return cost;
}

void LinearCore::getAInverse(Eigen::MatrixXd* A_inv) const {
  const int n = N_ * topo_.K;
  A_inv->resize(n, n);
  A_inv->setZero();
  std::vector<double> a(size_t(N_) * N_);
  for (int i = 0; i < topo_.K; ++i) {
    hostInverseMappingMatrix(N_, segment_times_[i], a.data());
    for (int r = 0; r < N_; ++r)
      for (int c = 0; c < N_; ++c) (*A_inv)(N_ * i + r, N_ * i + c) = a[size_t(r) * N_ + c];
  }
}

void LinearCore::getA(Eigen::MatrixXd* A) const {
  const int n = N_ * topo_.K;
  A->resize(n, n);
  A->setZero();
  std::vector<double> a(size_t(N_) * N_);
  for (int i = 0; i < topo_.K; ++i) {
    CHECK_GT(segment_times_[i], 0) << "Segment times need to be greater than zero";
    hostMappingMatrix(N_, segment_times_[i], a.data());
    for (int r = 0; r < N_; ++r)
      for (int c = 0; c < N_; ++c) (*A)(N_ * i + r, N_ * i + c) = a[size_t(r) * N_ + c];
  }
}

void LinearCore::getM(Eigen::MatrixXd* M) const {
  M->resize(topo_.n_all, topo_.n_fixed + topo_.n_free);
  M->setZero();
  for (int row = 0; row < topo_.n_all; ++row) (*M)(row, topo_.slot_col[row]) = 1.0;
}

void LinearCore::getMpinv(Eigen::MatrixXd* M_pinv) const {
  // rows of M^T normalised by their sum (reference linear_impl.h:556-565)
  const int cols = topo_.n_fixed + topo_.n_free;
  M_pinv->resize(cols, topo_.n_all);
  M_pinv->setZero();
  std::vector<int> count(cols, 0);
  for (int row = 0; row < topo_.n_all; ++row) count[topo_.slot_col[row]]++;
  for (int row = 0; row < topo_.n_all; ++row) (*M_pinv)(topo_.slot_col[row], row) = 1.0 / count[topo_.slot_col[row]];
}

void LinearCore::getR(Eigen::MatrixXd* R) const {
  const int n = topo_.n_fixed + topo_.n_free;
  R->resize(n, n);
  R->setZero();
  std::vector<double> H(size_t(N_) * N_);
  for (int i = 0; i < topo_.K; ++i) {
    hostSegmentHessian(N_, topo_.r, segment_times_[i], H.data());
    for (int a = 0; a < N_; ++a)
      for (int b = 0; b < N_; ++b)
        (*R)(topo_.slot_col[size_t(i) * N_ + a], topo_.slot_col[size_t(i) * N_ + b]) += H[size_t(a) * N_ + b];
  }
}

// ---- BatchCore ---------------------------------------------------------------------------
BatchCore::BatchCore(int N, size_t dimension) : N_(N), dimension_(dimension) {}
BatchCore::~BatchCore() { release(); }

void BatchCore::release() {
  if (!times_ && !d_fixed_ && !coeffs_ && !d_free_ && !status_) return;
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  mtg_host_free(h, times_);
  mtg_host_free(h, d_fixed_);
  mtg_host_free(h, coeffs_);
  mtg_host_free(h, d_free_);
  mtg_host_free(h, status_);
  times_ = d_fixed_ = coeffs_ = d_free_ = nullptr;
  status_ = nullptr;
}

void BatchCore::allocate(size_t B) {
  release();
  B_ = B;
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const size_t K = topo_.K, D = topo_.D, N = N_;
  times_ = static_cast<double*>(mtg_host_alloc(h, 8 * B * K));
  d_fixed_ = static_cast<double*>(mtg_host_alloc(h, 8 * B * D * topo_.n_fixed));
  coeffs_ = static_cast<double*>(mtg_host_alloc(h, 8 * B * K * D * N));
  d_free_ = static_cast<double*>(mtg_host_alloc(h, 8 * B * D * (topo_.n_free > 0 ? topo_.n_free : 1)));
  status_ = static_cast<int32_t*>(mtg_host_alloc(h, 4 * B));
  CHECK(times_ && d_fixed_ && coeffs_ && d_free_ && status_) << "pinned allocation failed: " << mtg_last_error(h);
}

bool BatchCore::setupFromVertices(const std::vector<Vertex::Vector>& vertices,
                                  const std::vector<std::vector<double> >& times, int r) {
  CHECK(r >= 0 && r <= N_ / 2 - 1);
  CHECK(!vertices.empty());
  CHECK_EQ(vertices.size(), times.size());
  Vertex::Vector first = vertices[0];
  buildTopology(N_, static_cast<int>(dimension_), r, &first, &topo_);
  allocate(vertices.size());
  for (size_t b = 0; b < B_; ++b) {
    CHECK(times[b].size() == static_cast<size_t>(topo_.K)) << "problem " << b << ": wrong number of segment times";
    const Vertex::Vector* vs = &vertices[b];
    Vertex::Vector filtered;
    if (!sameTopology(topo_, *vs)) {
      // tolerate constraints above N/2-1 (dropped like the reference), nothing else
      filtered = *vs;
      Topology t;
      buildTopology(N_, static_cast<int>(dimension_), r, &filtered, &t);
      CHECK(t.mask == topo_.mask) << "problem " << b << " does not share the constraint topology of problem 0";
      vs = &filtered;
    }
    for (int i = 0; i < topo_.K; ++i) {
      CHECK_GT(times[b][i], 0) << "Segment times need to be greater than zero";
      times_[b * topo_.K + i] = times[b][i];
    }
    packFixed(topo_, *vs, d_fixed_ + b * size_t(topo_.D) * topo_.n_fixed);
  }
  return true;
}

bool BatchCore::setupFromWaypoints(size_t B, size_t K, const double* positions, const double* times, int r) {
  CHECK(r >= 0 && r <= N_ / 2 - 1);
  CHECK_GE(K, 1u);
  const int h = N_ / 2, D = static_cast<int>(dimension_);
  topo_ = Topology();
  topo_.N = N_;
  topo_.K = static_cast<int>(K);
  topo_.D = D;
  topo_.r = r;
  topo_.mask.assign((K + 1) * h, 0);
  for (size_t v = 0; v <= K; ++v) {
    topo_.mask[v * h] = 1;
    if (v == 0 || v == K)
      for (int k = 1; k < h; ++k) topo_.mask[v * h + k] = 1;
  }
  mtg_problem p = {N_, r, topo_.K, D, topo_.mask.data()};
  mtg_layout lay;
  topo_.slot_col.assign(K * N_, 0);
  CHECK_EQ(mtg_problem_layout(&p, &lay, topo_.slot_col.data()), MTG_OK);
  topo_.n_all = lay.n_all;
  topo_.n_fixed = lay.n_fixed;
  topo_.n_free = lay.n_free;
  topo_.kernel = lay.kernel;
  allocate(B);
  std::memcpy(times_, times, 8 * B * K);
  const size_t nf = topo_.n_fixed;
  for (size_t b = 0; b < B; ++b) {
    const double* pos = positions + b * (K + 1) * D;
    double* out = d_fixed_ + b * D * nf;
    for (int d = 0; d < D; ++d) {
      double* o = out + d * nf;
      for (size_t c = 0; c < nf; ++c) o[c] = 0.0;
      o[0] = pos[d];
      for (size_t v = 1; v < K; ++v) o[h + v - 1] = pos[v * D + d];
      o[h + K - 1] = pos[K * D + d];
    }
  }
  return true;
}

bool BatchCore::solveLinear() {
  CHECK_GT(B_, 0u) << "setup first";
  mtg_problem p = {N_, topo_.r, topo_.K, topo_.D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_solve_linear_batch_host_f64(h, &p, static_cast<int64_t>(B_), times_, d_fixed_, coeffs_,
                                                 topo_.n_free > 0 ? d_free_ : nullptr, status_);
  if (rc != MTG_OK) {
    LOG(ERROR) << "mtg_solve_linear_batch_host_f64 failed (rc=" << rc << "): " << mtg_last_error(h);
    return false;
  }
  return true;
}

bool BatchCore::solveWaypointsNfabian(size_t B, size_t K, const double* positions, int r, double v_max, double a_max,
                                      double magic) {
  // topology bookkeeping + buffers exactly as setupFromWaypoints (d_fixed_ is still filled so that
  // getFixedConstraints-style consumers see the same data), but times and the solve come from the device
  std::vector<double> dummy_times(B * K, 1.0);
  if (!setupFromWaypoints(B, K, positions, dummy_times.data(), r)) return false;
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_solve_waypoints_nfabian_batch_host_f64(h, N_, r, topo_.K, topo_.D, static_cast<int64_t>(B), positions,
                                                            v_max, a_max, magic, coeffs_, times_, status_);
  if (rc != MTG_OK) {
    LOG(ERROR) << "mtg_solve_waypoints_nfabian_batch_host_f64 failed (rc=" << rc << "): " << mtg_last_error(h);
    return false;
  }
  return true;
}

std::vector<double> BatchCore::computeCosts() const {
  std::vector<double> cost(B_, 0.0);
  mtg_problem p = {N_, topo_.r, topo_.K, topo_.D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_compute_cost_batch_host_f64(h, &p, static_cast<int64_t>(B_), times_, coeffs_, cost.data());
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
  return cost;
}

void BatchCore::costGradientMellinger(std::vector<double>* cost, std::vector<double>* grad) const {
  CHECK_NOTNULL(grad)->assign(B_ * size_t(topo_.K), 0.0);
  if (cost) cost->assign(B_, 0.0);
  mtg_problem p = {N_, topo_.r, topo_.K, topo_.D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_cost_gradient_mellinger_batch_host_f64(h, &p, static_cast<int64_t>(B_), times_, d_fixed_,
                                                            cost ? cost->data() : nullptr, grad->data());
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
}

void BatchCore::evaluateRange(double t_start, double t_end, double dt, const std::vector<int>& derivatives,
                              int max_samples, std::vector<double>* samples, std::vector<int32_t>* n_samples,
                              std::vector<double>* sampling_times) const {
  CHECK(!derivatives.empty() && derivatives.size() <= 8);
  CHECK_GT(dt, 0.0);
  CHECK_NOTNULL(samples)->assign(B_ * size_t(max_samples) * derivatives.size() * topo_.D, 0.0);
  CHECK_NOTNULL(n_samples)->assign(B_, 0);
  if (sampling_times) sampling_times->assign(B_ * size_t(max_samples), 0.0);
  std::vector<int32_t> ders(derivatives.begin(), derivatives.end());
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_evaluate_range_batch_host_f64(h, N_, topo_.K, topo_.D, static_cast<int64_t>(B_), times_, coeffs_,
                                                   t_start, t_end, dt, static_cast<int32_t>(ders.size()), ders.data(),
                                                   max_samples, samples->data(), n_samples->data(),
                                                   sampling_times ? sampling_times->data() : nullptr);
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
}

void BatchCore::computeMaximaOfMagnitude(const std::vector<int>& derivatives, std::vector<Extremum>* maxima) const {
  CHECK(!derivatives.empty() && derivatives.size() <= 8);
  const size_t nd = derivatives.size();
  std::vector<int32_t> ders(derivatives.begin(), derivatives.end());
  std::vector<double> value(B_ * nd), time(B_ * nd);
  std::vector<int32_t> segment(B_ * nd);
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_max_magnitude_batch_host_f64(h, N_, topo_.K, topo_.D, static_cast<int64_t>(B_), times_, coeffs_,
                                                  static_cast<int32_t>(nd), ders.data(), value.data(), time.data(),
                                                  segment.data(), nullptr);
  CHECK_EQ(rc, MTG_OK) << mtg_last_error(h);
  CHECK_NOTNULL(maxima)->resize(B_ * nd);
  for (size_t i = 0; i < B_ * nd; ++i) (*maxima)[i] = Extremum(time[i], value[i], segment[i]);
}

bool BatchCore::timeObjective(const TimeObjectiveParameters& params, const double* d_free, std::vector<double>* objective,
                              std::vector<double>* terms) {
  CHECK_GT(B_, 0u) << "setup first";
  CHECK_LE(params.soft_constraints.size(), 8u);
  std::vector<mtg_soft_constraint> cons;
  for (const auto& c : params.soft_constraints) cons.push_back({c.first, c.second});
  mtg_time_objective obj = {params.richter_time ? 1 : 0, params.time_penalty, params.soft_constraint_weight,
                            params.maximum_cost, static_cast<int32_t>(cons.size()), cons.data()};
  CHECK_NOTNULL(objective)->assign(B_, 0.0);
  if (terms) terms->assign(3 * B_, 0.0);
  mtg_problem p = {N_, topo_.r, topo_.K, topo_.D, topo_.mask.data()};
  HandleLock lock;
  mtg_handle* h = defaultHandle();
  const int rc = mtg_time_objective_batch_host_f64(h, &p, static_cast<int64_t>(B_), times_, d_fixed_, d_free, &obj,
                                                   coeffs_, objective->data(), terms ? terms->data() : nullptr, status_);
  if (rc != MTG_OK) {
    LOG(ERROR) << "mtg_time_objective_batch_host_f64 failed (rc=" << rc << "): " << mtg_last_error(h);
    return false;
  }
  return true;
}

void BatchCore::getSegments(size_t b, Segment::Vector* segments) const {
  CHECK_LT(b, B_);
  unpackSegments(topo_, coeffs_ + b * size_t(topo_.K) * topo_.D * N_, times_ + b * topo_.K, segments);
}

}  // namespace b200
}  // namespace mav_trajectory_generation
