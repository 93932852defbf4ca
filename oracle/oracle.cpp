// oracle.cpp -- CPU restatement of the reference's linear min-derivative solve.
//
// THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load this library.  The
// product path (mav_trajectory_generation_b200/, include/) never links or calls it.
//
// What it restates (paths under mav_trajectory_generation/ of the reference repository):
//   include/mav_trajectory_generation/impl/polynomial_optimization_linear_impl.h
//     :56-109   setupFromVertices      -> Problem::setup
//     :111-121  setupMappingMatrix     -> setup_mapping_matrix
//     :142-179  invertMappingMatrix    -> invert_mapping_matrix (Schur structure, LU of D)
//     :181-260  setupConstraintReorderingMatrix -> Problem::setup_reordering
//     :262-283  updateSegmentsFromCompactConstraints -> Problem::update_segments
//     :285-305  updateSegmentTimes     -> Problem::update_segment_times
//     :307-336  constructR             -> Problem::construct_R
//     :338-379  solveLinear            -> Problem::solve_linear
//     :123-140  computeCost            -> Problem::compute_cost
//     :567-583  computeQuadraticCostJacobian -> cost_jacobian (pow-based, factor 2)
//   include/mav_trajectory_generation/polynomial.h:201-219  baseCoeffsWithTime
//   src/polynomial.cpp:145-160                               computeBaseCoefficients
//   src/vertex.cpp:27-82    createRandomVertices  (std::mt19937 + uniform_real_distribution)
//   src/vertex.cpp:255-272  estimateSegmentTimesNfabian
//
// The reference's arithmetic lives partly in Eigen (eigen_catkin, version unpinned, not
// vendored by the reference): fixed-size .inverse() (PartialPivLU for
// 5x5), dense products, and Eigen::SparseQR<COLAMDOrdering>.  Those calls are restated with
// their published algorithms: partial-pivot LU inverse; row-times-column products evaluated
// left to right ((Ai^T Q) Ai); a Householder QR solve of the full (non-symmetrised) R_pp
// that only skips structural zeros of the band (what a sparse QR does).  The operation
// ORDER of the reference is kept (pow() for Q, A built by baseCoeffsWithTime, H formed from
// A^-T Q A^-1 in floating point, R = C^T H C by summing the two segment contributions of
// interior vertices, general solve, p = A^-1 (C d)).
//
// PARITY PINNING: checked against every golden/known-answer the reference tests hold for
// this path (tests/test_oracle.py): the Matlab coefficients of TwoVerticesSetup
// (test_polynomial_optimization.cpp:776-780), the A^-1 identity (:731-741, 1e-10), checkPath
// (:113-174, 1e-6) on the reference's ten parameter sets (:790-867), ConstraintPacking
// (:505-564) and the mt19937 fixture.  No reference test stores the solved coefficients of
// a problem WITH free constraints, and Eigen cannot be built here, so at the 1e-10 level the
// solve itself is "parity unpinned" by the reference; it is cross-checked instead against a
// 60-digit mpmath solve of the same equations (oracle/truth.py).
//
// Build: see oracle/Makefile (g++ -O3 -march=x86-64-v3 -ffp-contract=off -shared -fPIC -pthread).

#include <sched.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <random>
#include <thread>
#include <vector>

namespace {

constexpr int kMaxN = 12;       // polynomial.h:44  (kMaxN = 12)
constexpr int kTableN = 22;     // polynomial.h:47-50 (kMaxConvolutionSize = 2*kMaxN-2)

// polynomial.cpp:145-160 computeBaseCoefficients, built once (polynomial.cpp:213-214).
struct BaseCoefficients {
  double v[kTableN][kTableN];
  BaseCoefficients() {
    const int N = kTableN;
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) v[i][j] = 0.0;
    for (int j = 0; j < N; ++j) v[0][j] = 1.0;
    const int DEG = N - 1;
    int order = DEG;
    for (int n = 1; n < N; ++n) {
      for (int i = DEG - order; i < N; ++i) v[n][i] = (order - DEG + i) * v[n - 1][i];
      --order;
    }
  }
};
const BaseCoefficients g_base;

// polynomial.h:201-219 baseCoeffsWithTime.
void base_coeffs_with_time(int N, int derivative, double t, double* coeffs) {
  for (int j = 0; j < N; ++j) coeffs[j] = 0.0;
  coeffs[derivative] = g_base.v[derivative][derivative];
  if (std::abs(t) < std::numeric_limits<double>::epsilon()) return;
  double t_power = t;
  for (int j = derivative + 1; j < N; ++j) {
    coeffs[j] = g_base.v[derivative][j] * t_power;
    t_power = t_power * t;
  }
}

// Row-major N x N matrices in flat vectors.
struct Mat {  // fixed storage like the reference's Eigen::Matrix<double, N, N> (no heap)
  int n = 0;
  double a[kMaxN * kMaxN];
  Mat() {}
  explicit Mat(int n_) : n(n_) {
    for (int i = 0; i < n * n; ++i) a[i] = 0.0;
  }
  int size() const { return n * n; }
  double& operator()(int r, int c) { return a[r * n + c]; }
  double operator()(int r, int c) const { return a[r * n + c]; }
};

// linear_impl.h:111-121 setupMappingMatrix: A = [A(t=0); A(t=T)].
void setup_mapping_matrix(int N, double T, Mat* A) {
  const int h = N / 2;
  double row[kMaxN];
  for (int i = 0; i < h; ++i) {
    base_coeffs_with_time(N, i, 0.0, row);
    for (int j = 0; j < N; ++j) (*A)(i, j) = row[j];
    base_coeffs_with_time(N, i, T, row);
    for (int j = 0; j < N; ++j) (*A)(i + h, j) = row[j];
  }
}

// General inverse by LU with partial pivoting (what Eigen's fixed-size inverse() does for
// sizes > 4; sizes <= 4 use cofactor formulas in Eigen -- same result to rounding).
bool lu_inverse(int n, const double* in, double* out) {
  double lu[kMaxN * kMaxN];
  for (int i = 0; i < n * n; ++i) lu[i] = in[i];
  int perm[kMaxN];
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int c = 0; c < n; ++c) {
    int p = c;
    double best = std::abs(lu[size_t(c) * n + c]);
    for (int i = c + 1; i < n; ++i) {
      const double v = std::abs(lu[size_t(i) * n + c]);
      if (v > best) { best = v; p = i; }
    }
    if (best == 0.0) return false;
    if (p != c) {
      for (int j = 0; j < n; ++j) std::swap(lu[size_t(c) * n + j], lu[size_t(p) * n + j]);
      std::swap(perm[c], perm[p]);
    }
    const double piv = lu[size_t(c) * n + c];
    for (int i = c + 1; i < n; ++i) {
      const double f = lu[size_t(i) * n + c] / piv;
      lu[size_t(i) * n + c] = f;
      for (int j = c + 1; j < n; ++j) lu[size_t(i) * n + j] -= f * lu[size_t(c) * n + j];
    }
  }
  for (int col = 0; col < n; ++col) {
    double x[kMaxN];
    for (int i = 0; i < n; ++i) x[i] = (perm[i] == col) ? 1.0 : 0.0;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < i; ++j) x[i] -= lu[size_t(i) * n + j] * x[j];
    for (int i = n - 1; i >= 0; --i) {
      for (int j = i + 1; j < n; ++j) x[i] -= lu[size_t(i) * n + j] * x[j];
      x[i] /= lu[size_t(i) * n + i];
    }
    for (int i = 0; i < n; ++i) out[size_t(i) * n + col] = x[i];
  }
  return true;
}

// linear_impl.h:142-179 invertMappingMatrix: [A_diag 0; C D]^-1 = [A_diag^-1 0; -D^-1 C A_diag^-1, D^-1].
void invert_mapping_matrix(int N, const Mat& A, Mat* Ai) {
  const int h = N / 2;
  double a_inv[kMaxN], C[kMaxN * kMaxN], Dm[kMaxN * kMaxN], Dinv[kMaxN * kMaxN];
  for (int i = 0; i < h; ++i) a_inv[i] = 1.0 / A(i, i);
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < h; ++j) {
      C[size_t(i) * h + j] = A(h + i, j);
      Dm[size_t(i) * h + j] = A(h + i, h + j);
    }
  lu_inverse(h, Dm, Dinv);
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) (*Ai)(i, j) = 0.0;
  for (int i = 0; i < h; ++i) (*Ai)(i, i) = a_inv[i];
  // -D_inv * C * A_inv, evaluated left to right: (-D_inv * C) * A_inv (A_inv diagonal).
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < h; ++j) {
      double s = 0.0;
      for (int k = 0; k < h; ++k) s += (-Dinv[size_t(i) * h + k]) * C[size_t(k) * h + j];
      (*Ai)(h + i, j) = s * a_inv[j];
      (*Ai)(h + i, h + j) = Dinv[size_t(i) * h + j];
    }
}

// linear_impl.h:567-583 computeQuadraticCostJacobian.
void cost_jacobian(int N, int derivative, double t, Mat* Q) {
  for (int i = 0; i < N * N; ++i) Q->a[i] = 0.0;
  for (int col = 0; col < N - derivative; ++col)
    for (int row = 0; row < N - derivative; ++row) {
      const double exponent = (N - 1 - derivative) * 2 + 1 - row - col;
      (*Q)(N - 1 - row, N - 1 - col) = g_base.v[derivative][N - 1 - row] *
                                       g_base.v[derivative][N - 1 - col] * std::pow(t, exponent) * 2.0 /
                                       exponent;
    }
}

// polynomial_optimization_linear.h:287-304 struct Constraint (ordering = (vertex, derivative)).
struct Constraint {
  int vertex_idx;
  int constraint_idx;
  bool operator<(const Constraint& o) const {
    if (vertex_idx != o.vertex_idx) return vertex_idx < o.vertex_idx;
    return constraint_idx < o.constraint_idx;
  }
  bool operator==(const Constraint& o) const {
    return vertex_idx == o.vertex_idx && constraint_idx == o.constraint_idx;
  }
};

// Dense storage, band-limited Householder QR solve of a general square system.
// Restates what Eigen::SparseQR does numerically on R_pp (Householder reflections on the
// full, non-symmetric matrix; structural zeros skipped).  kl/ku = lower/upper bandwidth.
bool qr_solve_banded(int n, int kl, int ku, std::vector<double>& A /* n*n row-major, destroyed */,
                     std::vector<double>& B /* n*nrhs row-major, in/out */, int nrhs) {
  const int kr = std::min(n - 1, kl + ku);  // upper bandwidth of the R factor
  std::vector<double> v(kl + 1);
  for (int j = 0; j < n; ++j) {
    const int i_end = std::min(n - 1, j + kl);
    const int c_end = std::min(n - 1, j + kr);
    double norm2 = 0.0;
    for (int i = j; i <= i_end; ++i) norm2 += A[size_t(i) * n + j] * A[size_t(i) * n + j];
    const double norm = std::sqrt(norm2);
    if (norm == 0.0) return false;
    const double alpha = (A[size_t(j) * n + j] > 0.0) ? -norm : norm;
    for (int i = j; i <= i_end; ++i) v[i - j] = A[size_t(i) * n + j];
    v[0] -= alpha;
    double vnorm2 = 0.0;
    for (int i = j; i <= i_end; ++i) vnorm2 += v[i - j] * v[i - j];
    if (vnorm2 > 0.0) {
      const double beta = 2.0 / vnorm2;
      for (int c = j; c <= c_end; ++c) {
        double s = 0.0;
        for (int i = j; i <= i_end; ++i) s += v[i - j] * A[size_t(i) * n + c];
        s *= beta;
        for (int i = j; i <= i_end; ++i) A[size_t(i) * n + c] -= s * v[i - j];
      }
      for (int c = 0; c < nrhs; ++c) {
        double s = 0.0;
        for (int i = j; i <= i_end; ++i) s += v[i - j] * B[size_t(i) * nrhs + c];
        s *= beta;
        for (int i = j; i <= i_end; ++i) B[size_t(i) * nrhs + c] -= s * v[i - j];
      }
    }
  }
  for (int c = 0; c < nrhs; ++c)
    for (int i = n - 1; i >= 0; --i) {
      double s = B[size_t(i) * nrhs + c];
      const int j_end = std::min(n - 1, i + kr);
      for (int j = i + 1; j <= j_end; ++j) s -= A[size_t(i) * n + j] * B[size_t(j) * nrhs + c];
      B[size_t(i) * nrhs + c] = s / A[size_t(i) * n + i];
    }
  return true;
}

// One PolynomialOptimization<N> object (runtime N).
struct Problem {
  int N, h, D, K = 0, r = -1;
  int n_all = 0, n_fixed = 0, n_free = 0;
  std::vector<double> times;
  std::vector<uint8_t> mask;        // [K+1][h]  1 = vertex has constraint (fixed)
  std::vector<double> values;       // [K+1][h][D]
  std::vector<Mat> Ainv, Q;         // per segment
  std::vector<int> slot_col;        // [K*N]: column of C holding the single 1 of each row
  std::vector<double> d_fixed;      // [D][n_fixed]
  std::vector<double> d_free;       // [D][n_free]
  std::vector<double> coeffs;       // [K][D][N]
  int free_bw = 0;                  // half bandwidth of R_pp

  Problem(int N_, int D_) : N(N_), h(N_ / 2), D(D_) {}

  // linear_impl.h:56-109.  Constraints with derivative > N/2-1 are simply not representable
  // in mask[K+1][h] (the reference drops them with a warning, :84-105).
  bool setup(int K_, const uint8_t* mask_, const double* values_, const double* times_, int r_) {
    if (r_ < 0 || r_ > h - 1) return false;  // CHECK at :60
    K = K_;
    r = r_;
    mask.assign(mask_, mask_ + size_t(K + 1) * h);
    values.assign(values_, values_ + size_t(K + 1) * h * D);
    Ainv.assign(K, Mat(N));
    Q.assign(K, Mat(N));
    coeffs.assign(size_t(K) * D * N, 0.0);
    if (!update_segment_times(times_)) return false;
    setup_reordering();
    return true;
  }

  // linear_impl.h:285-305.
  bool update_segment_times(const double* times_) {
    times.assign(times_, times_ + K);
    Mat A(N);
    for (int i = 0; i < K; ++i) {
      if (!(times[i] > 0.0)) return false;  // CHECK_GT at :297
      cost_jacobian(N, r, times[i], &Q[i]);
      setup_mapping_matrix(N, times[i], &A);
      invert_mapping_matrix(N, A, &Ainv[i]);
    }
    return true;
  }

  // linear_impl.h:181-260.  Same enumeration order and the same nested scans over the
  // sorted-unique fixed / free sets (:238-256); C is stored as one column index per row.
  void setup_reordering() {
    std::vector<Constraint> all, fixed, free_c;
    all.reserve(size_t(K + 1) * h * 2);
    for (int v = 0; v <= K; ++v) {
      const int occ = (v == 0 || v == K) ? 1 : 2;  // :202-204
      for (int co = 0; co < occ; ++co)
        for (int k = 0; k < h; ++k) {
          Constraint c{v, k};
          all.push_back(c);
          (mask[size_t(v) * h + k] ? fixed : free_c).push_back(c);
        }
    }
    auto uniq = [](std::vector<Constraint>& s) {  // std::set semantics
      std::sort(s.begin(), s.end());
      s.erase(std::unique(s.begin(), s.end()), s.end());
    };
    uniq(fixed);
    uniq(free_c);
    n_all = int(all.size());
    n_fixed = int(fixed.size());
    n_free = int(free_c.size());
    slot_col.assign(n_all, -1);
    d_fixed.assign(size_t(D) * n_fixed, 0.0);
    d_free.assign(size_t(D) * n_free, 0.0);
    int row = 0;
    for (const Constraint& ca : all) {
      int col = 0;
      for (const Constraint& cf : fixed) {
        if (ca == cf) {
          slot_col[row] = col;
          for (int d = 0; d < D; ++d)
            d_fixed[size_t(d) * n_fixed + col] = values[(size_t(cf.vertex_idx) * h + cf.constraint_idx) * D + d];
        }
        ++col;
      }
      for (const Constraint& cp : free_c) {
        if (ca == cp) slot_col[row] = col;
        ++col;
      }
      ++row;
    }
    // half bandwidth of R_pp: free columns touched by one segment are contiguous.
    free_bw = 0;
    for (int i = 0; i < K; ++i) {
      int lo = n_free, hi = -1;
      for (int s = 0; s < N; ++s) {
        const int c = slot_col[size_t(i) * N + s] - n_fixed;
        if (c >= 0) { lo = std::min(lo, c); hi = std::max(hi, c); }
      }
      if (hi >= lo) free_bw = std::max(free_bw, hi - lo);
    }
  }

  // linear_impl.h:307-336: H_i = (Ai^T * Q) * Ai ; R = C^T blockdiag(H) C.
  void construct_R(std::vector<double>* R) const {
    const int n = n_fixed + n_free;
    R->assign(size_t(n) * n, 0.0);
    Mat tmp(N), H(N);
    for (int i = 0; i < K; ++i) {
      const Mat& Ai = Ainv[i];
      const Mat& Qi = Q[i];
      for (int a = 0; a < N; ++a)
        for (int b = 0; b < N; ++b) {
          double s = 0.0;
          for (int k = 0; k < N; ++k) s += Ai(k, a) * Qi(k, b);
          tmp(a, b) = s;
        }
      for (int a = 0; a < N; ++a)
        for (int b = 0; b < N; ++b) {
          double s = 0.0;
          for (int k = 0; k < N; ++k) s += tmp(a, k) * Ai(k, b);
          H(a, b) = s;
        }
      for (int a = 0; a < N; ++a) {
        const int ca = slot_col[size_t(i) * N + a];
        for (int b = 0; b < N; ++b) {
          const int cb = slot_col[size_t(i) * N + b];
          (*R)[size_t(ca) * n + cb] += H(a, b);
        }
      }
    }
  }

  // linear_impl.h:262-283.
  void update_segments() {
    const int n = n_fixed + n_free;
    std::vector<double> d_all(n), new_d(N);
    for (int d = 0; d < D; ++d) {
      for (int c = 0; c < n_fixed; ++c) d_all[c] = d_fixed[size_t(d) * n_fixed + c];
      for (int c = 0; c < n_free; ++c) d_all[n_fixed + c] = d_free[size_t(d) * n_free + c];
      for (int i = 0; i < K; ++i) {
        for (int s = 0; s < N; ++s) new_d[s] = d_all[slot_col[size_t(i) * N + s]];
        for (int j = 0; j < N; ++j) {
          double s = 0.0;
          for (int k = 0; k < N; ++k) s += Ainv[i](j, k) * new_d[k];
          coeffs[(size_t(i) * D + d) * N + j] = s;
        }
      }
    }
  }

  // linear_impl.h:338-379.
  bool solve_linear() {
    if (n_free == 0) {  // :343-349
      update_segments();
      return true;
    }
    std::vector<double> R;
    construct_R(&R);
    const int n = n_fixed + n_free;
    std::vector<double> Rpp(size_t(n_free) * n_free), rhs(size_t(n_free) * D);
    for (int a = 0; a < n_free; ++a)
      for (int b = 0; b < n_free; ++b) Rpp[size_t(a) * n_free + b] = R[size_t(n_fixed + a) * n + n_fixed + b];
    for (int d = 0; d < D; ++d)
      for (int a = 0; a < n_free; ++a) {
        double s = 0.0;
        for (int c = 0; c < n_fixed; ++c) s += (-R[size_t(n_fixed + a) * n + c]) * d_fixed[size_t(d) * n_fixed + c];
        rhs[size_t(a) * D + d] = s;  // df = -Rpf * d_f  (:371-372)
      }
    const bool ok = qr_solve_banded(n_free, free_bw, free_bw, Rpp, rhs, D);
    for (int d = 0; d < D; ++d)
      for (int a = 0; a < n_free; ++a) d_free[size_t(d) * n_free + a] = rhs[size_t(a) * D + d];
    update_segments();
    return ok;
  }

  // linear_impl.h:123-140.
  double compute_cost() const {
    double cost = 0.0;
    for (int i = 0; i < K; ++i)
      for (int d = 0; d < D; ++d) {
        const double* c = &coeffs[(size_t(i) * D + d) * N];
        double partial = 0.0;
        for (int a = 0; a < N; ++a) {
          double s = 0.0;
          for (int b = 0; b < N; ++b) s += Q[i](a, b) * c[b];
          partial += c[a] * s;
        }
        cost += partial;
      }
    return 0.5 * cost;
  }
};

// vertex.cpp:27-82 createRandomVertices, positions only (ends get derivatives 1..max fixed
// to zero by makeStartOrEnd, vertex.cpp:147-153; interior vertices position only).
void create_random_positions(int K, int D, const double* pos_min, const double* pos_max, uint64_t seed,
                             double* positions /* [K+1][D] */) {
  std::mt19937 generator(seed);
  std::vector<std::uniform_real_distribution<double>> distribution(D);
  for (int i = 0; i < D; ++i) distribution[i] = std::uniform_real_distribution<double>(pos_min[i], pos_max[i]);
  const double min_distance = 0.2;
  std::vector<double> last(D), pos(D);
  for (int i = 0; i < D; ++i) last[i] = distribution[i](generator);
  for (int d = 0; d < D; ++d) positions[d] = last[d];
  for (int i = 1; i <= K; ++i) {
    while (true) {
      for (int d = 0; d < D; ++d) pos[d] = distribution[d](generator);
      double n2 = 0.0;
      for (int d = 0; d < D; ++d) n2 += (pos[d] - last[d]) * (pos[d] - last[d]);
      if (std::sqrt(n2) > min_distance) break;
    }
    for (int d = 0; d < D; ++d) positions[size_t(i) * D + d] = pos[d];
    last = pos;
  }
}

// vertex.cpp:255-272 estimateSegmentTimesNfabian.
void nfabian(int K, int D, const double* positions, double v_max, double a_max, double magic, double* times) {
  for (int i = 0; i < K; ++i) {
    double n2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double e = positions[size_t(i + 1) * D + d] - positions[size_t(i) * D + d];
      n2 += e * e;
    }
    const double distance = std::sqrt(n2);
    times[i] = distance / v_max * 2 * (1.0 + magic * v_max / a_max * std::exp(-distance / v_max * 2));
  }
}

// Waypoint topology helper: ends fixed 0..h-1 (makeStartOrEnd), interior position only.
void waypoint_problem(int N, int K, int D, const double* positions, std::vector<uint8_t>* mask,
                      std::vector<double>* values) {
  const int h = N / 2;
  mask->assign(size_t(K + 1) * h, 0);
  values->assign(size_t(K + 1) * h * D, 0.0);
  for (int v = 0; v <= K; ++v) {
    (*mask)[size_t(v) * h] = 1;
    for (int d = 0; d < D; ++d) (*values)[(size_t(v) * h) * D + d] = positions[size_t(v) * D + d];
    if (v == 0 || v == K)
      for (int k = 1; k < h; ++k) (*mask)[size_t(v) * h + k] = 1;
  }
}

}  // namespace

extern "C" {

// Full reference lifecycle for one problem: construct + setupFromVertices + solveLinear
// (polynomial_timing_evaluation.cpp:104-110).  Returns 0 on success.
//   mask[K+1][h], values[K+1][h][D], times[K]  ->  coeffs[K][D][N]
//   optional outs: d_fixed[D][n_fixed], d_free[D][n_free], slot_col[K*N], cost, counts[3]
int oracle_solve(int N, int r, int K, int D, const uint8_t* mask, const double* values, const double* times,
                 double* coeffs, double* d_fixed, double* d_free, int32_t* slot_col, double* cost,
                 int32_t* counts) {
  if (N < 2 || N > kMaxN || (N & 1) || K < 1 || D < 1) return -1;
  Problem p(N, D);
  if (!p.setup(K, mask, values, times, r)) return -2;
  const bool ok = p.solve_linear();
  std::memcpy(coeffs, p.coeffs.data(), sizeof(double) * p.coeffs.size());
  if (d_fixed) std::memcpy(d_fixed, p.d_fixed.data(), sizeof(double) * p.d_fixed.size());
  if (d_free && p.n_free) std::memcpy(d_free, p.d_free.data(), sizeof(double) * p.d_free.size());
  if (slot_col)
    for (int i = 0; i < p.n_all; ++i) slot_col[i] = p.slot_col[i];
  if (cost) *cost = p.compute_cost();
  if (counts) {
    counts[0] = p.n_all;
    counts[1] = p.n_fixed;
    counts[2] = p.n_free;
  }
  return ok ? 0 : -3;
}

// Counts only (n_all, n_fixed, n_free) for a mask.
int oracle_counts(int N, int K, const uint8_t* mask, int32_t* counts) {
  const int h = N / 2;
  int nf = 0, np = 0;
  for (int v = 0; v <= K; ++v)
    for (int k = 0; k < h; ++k) (mask[size_t(v) * h + k] ? nf : np)++;
  counts[0] = K * N;
  counts[1] = nf;
  counts[2] = np;
  return 0;
}

void oracle_mapping_matrix(int N, double T, double* A_out) {
  Mat A(N);
  setup_mapping_matrix(N, T, &A);
  std::memcpy(A_out, A.a, sizeof(double) * A.size());
}

void oracle_inverse_mapping_matrix(int N, double T, double* Ai_out) {
  Mat A(N), Ai(N);
  setup_mapping_matrix(N, T, &A);
  invert_mapping_matrix(N, A, &Ai);
  std::memcpy(Ai_out, Ai.a, sizeof(double) * Ai.size());
}

// Plain LU inverse of A(T) ("A.inverse()" in AMatrixInversion, test :731-741).
int oracle_general_inverse(int n, const double* A, double* Ai) { return lu_inverse(n, A, Ai) ? 0 : -1; }

void oracle_cost_matrix(int N, int r, double T, double* Q_out) {
  Mat Q(N);
  cost_jacobian(N, r, T, &Q);
  std::memcpy(Q_out, Q.a, sizeof(double) * Q.size());
}

void oracle_base_coefficients(double* out /* 22*22 */) { std::memcpy(out, g_base.v, sizeof(g_base.v)); }

void oracle_create_random_positions(int K, int D, const double* pos_min, const double* pos_max, uint64_t seed,
                                    double* positions) {
  create_random_positions(K, D, pos_min, pos_max, seed, positions);
}

void oracle_nfabian(int K, int D, const double* positions, double v_max, double a_max, double magic,
                    double* times) {
  nfabian(K, D, positions, v_max, a_max, magic, times);
}

// Batch of waypoint-topology problems (the BASELINE.json fixture): positions[B][K+1][D],
// times[B][K] -> coeffs[B][K][D][N].  n_threads host threads over disjoint slices.
// mode 0: clock covers construct + setupFromVertices + solveLinear per trajectory
//         (polynomial_timing_evaluation.cpp:104-110) -- the headline CPU baseline.
// mode 1: clock covers only updateSegmentTimes + solveLinear on an already set-up object
//         (the nonlinear optimiser's inner step, polynomial_optimization_nonlinear_impl.h:569-570).
// Returns: mode 0 the wall-clock seconds of the whole batch (thread start to join); mode 1 the max
// over threads of the seconds spent inside the clocked calls; < 0 on failure.
double oracle_solve_waypoint_batch(int N, int r, int K, int D, int64_t B, const double* positions,
                                   const double* times, double* coeffs, int n_threads, int mode) {
  if (n_threads < 1) n_threads = 1;
  std::vector<std::thread> pool;
  std::vector<double> spent(n_threads, 0.0);
  std::atomic<int> failures{0};
  std::atomic<int64_t> next_chunk{0};
  constexpr int64_t kChunk = 64;
  const auto wall0 = std::chrono::steady_clock::now();
  for (int t = 0; t < n_threads; ++t) {
    pool.emplace_back([&, t]() {
      using clk = std::chrono::steady_clock;
      std::vector<uint8_t> mask;
      std::vector<double> values;
      double acc = 0.0;
      // dynamic chunks: on a shared host some threads get less CPU than others, and a static split would
      // let the slowest one set the wall clock
      for (;;) {
       const int64_t lo = next_chunk.fetch_add(kChunk), hi = std::min<int64_t>(B, lo + kChunk);
       if (lo >= B) break;
       for (int64_t b = lo; b < hi; ++b) {
        const double* pos = positions + size_t(b) * (K + 1) * D;
        const double* tt = times + size_t(b) * K;
        waypoint_problem(N, K, D, pos, &mask, &values);
        const auto t0 = clk::now();
        Problem p(N, D);
        bool ok = p.setup(K, mask.data(), values.data(), tt, r);
        const auto t1 = clk::now();
        if (mode == 1) ok = ok && p.update_segment_times(tt);
        ok = ok && p.solve_linear();
        const auto t2 = clk::now();
        acc += std::chrono::duration<double>(t2 - (mode == 0 ? t0 : t1)).count();
        if (!ok) failures++;
        if (coeffs) std::memcpy(coeffs + size_t(b) * K * D * N, p.coeffs.data(), sizeof(double) * p.coeffs.size());
       }
      }
      spent[t] = acc;
    });
  }
  for (auto& th : pool) th.join();
  const auto wall1 = std::chrono::steady_clock::now();
  if (failures.load() != 0) return -1.0;
  if (mode == 0) return std::chrono::duration<double>(wall1 - wall0).count();  // whole-batch wall clock
  return *std::max_element(spent.begin(), spent.end());
}

// B fixtures: createRandomVertices(seed = base_seed + b) + estimateSegmentTimesNfabian.
void oracle_make_waypoint_batch(int K, int D, int64_t B, double lo, double hi, uint64_t base_seed, double v_max,
                                double a_max, double* positions /* [B][K+1][D] */, double* times /* [B][K] */) {
  std::vector<double> pmin(D, lo), pmax(D, hi);
  for (int64_t b = 0; b < B; ++b) {
    double* pos = positions + size_t(b) * (K + 1) * D;
    create_random_positions(K, D, pmin.data(), pmax.data(), base_seed + uint64_t(b), pos);
    nfabian(K, D, pos, v_max, a_max, 6.5, times + size_t(b) * K);
  }
}

// getCostAndGradientMellinger (reference impl/polynomial_optimization_nonlinear_impl.h:286-364): cost of the
// current times and the forward-difference gradient with the total-time-preserving perturbation
// (+0.1 s on segment n, -0.1/(K-1) on the others, clamped at kOptimizationTimeLowerBound = 0.1,
// polynomial_optimization_nonlinear.h:31).  Waypoint topology.
int oracle_cost_gradient_mellinger(int N, int r, int K, int D, const double* positions, const double* times,
                                   double* cost, double* grad) {
  std::vector<uint8_t> mask;
  std::vector<double> values;
  waypoint_problem(N, K, D, positions, &mask, &values);
  Problem p(N, D);
  if (!p.setup(K, mask.data(), values.data(), times, r) || !p.solve_linear()) return -1;
  const double J = p.compute_cost();
  *cost = J;
  if (K == 1) {
    grad[0] = 0.0;
    return 0;
  }
  const double increment_time = 0.1, lower = 0.1;
  std::vector<double> bigger(K);
  for (int n = 0; n < K; ++n) {
    const double corr = increment_time / (K - 1.0);
    for (int i = 0; i < K; ++i) bigger[i] = (i == n) ? times[i] + increment_time : times[i] - corr;
    for (double& t : bigger) t = std::max(lower, t);
    if (!p.update_segment_times(bigger.data()) || !p.solve_linear()) return -2;
    grad[n] = (p.compute_cost() - J) / increment_time;
  }
  return 0;
}

// Host threads this process can actually run concurrently: the scheduler affinity mask intersected with the
// cgroup CPU quota (cgroup v2 cpu.max, v1 cpu.cfs_quota_us / cpu.cfs_period_us).  hardware_concurrency()
// alone reports the machine, not the container.  info[0] = hardware_concurrency, [1] = affinity count,
// [2] = cgroup quota in whole CPUs (0 = unlimited), [3] = effective.
int oracle_cpu_info(int32_t* info) {
  const int hw = int(std::thread::hardware_concurrency());
  int aff = hw;
  cpu_set_t set;
  CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof(set), &set) == 0) aff = CPU_COUNT(&set);
  int quota = 0;
  {
    double q = -1.0, per = 0.0;
    if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
      char a[64] = {0};
      if (std::fscanf(f, "%63s %lf", a, &per) == 2 && std::strcmp(a, "max") != 0) q = std::atof(a);
      std::fclose(f);
    } else {
      if (FILE* f1 = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
        if (std::fscanf(f1, "%lf", &q) != 1) q = -1.0;
        std::fclose(f1);
      }
      if (FILE* f2 = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
        if (std::fscanf(f2, "%lf", &per) != 1) per = 0.0;
        std::fclose(f2);
      }
    }
    if (q > 0.0 && per > 0.0) quota = std::max(1, int(std::ceil(q / per)));
  }
  int eff = std::max(1, aff);
  if (quota > 0) eff = std::min(eff, quota);
  if (info) {
    info[0] = hw;
    info[1] = aff;
    info[2] = quota;
    info[3] = eff;
  }
  return eff;
}

int oracle_hardware_threads() { return oracle_cpu_info(nullptr); }

// Trajectory::evaluateRange (reference src/trajectory.cpp:81-141) restated literally, quirks included: the
// sample clock `accumulated_time` starts at the START OF THE SEGMENT that contains t_start (not at t_start),
// advances by dt per sample and is what the loop compares with t_end and reports as the sampling time;
// time_in_segment > T moves to the next segment without consuming a sample; the walk stops after the last
// segment.  Each sample is Segment::evaluate -> Polynomial::evaluate(t, derivative) (polynomial.h:134-149:
// Horner with separate multiply and add).  times [K], coeffs [K][D][N] -> out [n][D], sampling_times [n]
// (nullable); returns n (<= max_samples stored), or -1 when t_start lies beyond the trajectory.
int oracle_evaluate_range(int N, int K, int D, const double* times, const double* coeffs, double t_start, double t_end,
                          double dt, int derivative, int max_samples, double* out, double* sampling_times) {
  double accumulated_time = 0.0;
  int i = 0;
  for (i = 0; i < K; ++i) {
    accumulated_time += times[i];
    if (accumulated_time > t_start) break;
  }
  if (t_start > accumulated_time) return -1;
  if (i >= K) return 0;  // t_start == total time: the reference indexes segments_[size] here (undefined); no samples
  accumulated_time -= times[i];
  double time_in_segment = t_start - accumulated_time;
  int n = 0;
  while (accumulated_time < t_end) {
    if (time_in_segment > times[i]) {
      time_in_segment = time_in_segment - times[i];
      i++;
      if (i >= K) break;
      continue;
    }
    if (n < max_samples) {
      for (int d = 0; d < D; ++d) {
        const double* c = coeffs + (size_t(i) * D + d) * N;
        double result = 0.0;
        if (derivative < N) {
          result = g_base.v[derivative][N - 1] * c[N - 1];
          for (int j = N - 2; j >= derivative; --j) {
            result *= time_in_segment;
            result += g_base.v[derivative][j] * c[j];
          }
        }
        out[size_t(n) * D + d] = result;
      }
      if (sampling_times) sampling_times[n] = accumulated_time;
    }
    ++n;
    time_in_segment += dt;
    accumulated_time += dt;
  }
  return n;
}

}  // extern "C"
