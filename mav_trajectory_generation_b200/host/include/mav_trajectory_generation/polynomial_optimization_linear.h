// polynomial_optimization_linear.h -- PolynomialOptimization<N> with the reference's public
// surface (include/mav_trajectory_generation/polynomial_optimization_linear.h:45-284), backed by
// the H100 kernels.  Behaviour kept from the reference:
//   * value semantics: inputs are copied in, results copied out to caller-owned objects;
//   * argument errors CHECK-abort (impl/...linear_impl.h:60,76,289,297,502-504);
//   * setupFromVertices()/solveLinear() return true (:108,:348,:378);
//   * constraints above derivative N/2-1 are dropped with a warning (:84-105);
//   * compact constraint order = (vertex, derivative) (linear.h:287-295).
// The extrema helpers (computeSegmentMaximumMagnitudeCandidates*, computeMaximumOfMagnitude, linear.h:138-176) are
// provided on top of Segment::computeMinMaxMagnitudeCandidateTimes (host/src/b200_extrema.cpp: Aberth-Ehrlich
// roots instead of the reference's Jenkins-Traub).  setupFromPositons is declared but never defined in the
// reference (linear.h:79-80) and is omitted.
#ifndef MAV_TRAJECTORY_GENERATION_POLYNOMIAL_OPTIMIZATION_LINEAR_H_
#define MAV_TRAJECTORY_GENERATION_POLYNOMIAL_OPTIMIZATION_LINEAR_H_

#include <cmath>
#include <numeric>
#include <ostream>
#include <vector>

#include "mav_trajectory_generation/b200_core.h"
#include "mav_trajectory_generation/motion_defines.h"
#include "mav_trajectory_generation/polynomial.h"
#include "mav_trajectory_generation/segment.h"
#include "mav_trajectory_generation/trajectory.h"
#include "mav_trajectory_generation/vertex.h"

namespace mav_trajectory_generation {

template <int _N>
class PolynomialOptimizationNonLinear;

template <int _N = 10>
class PolynomialOptimization {
  static_assert(_N % 2 == 0, "The number of coefficients has to be even.");
  static_assert(_N >= 2 && _N <= Polynomial::kMaxN, "N must be in [2, 12].");

 public:
  enum { N = _N };
  static constexpr int kHighestDerivativeToOptimize = N / 2 - 1;
  typedef Eigen::Matrix<double, N, N> SquareMatrix;
  typedef std::vector<SquareMatrix, Eigen::aligned_allocator<SquareMatrix> > SquareMatrixVector;

  explicit PolynomialOptimization(size_t dimension) : core_(N, dimension) {}

  bool setupFromVertices(const Vertex::Vector& vertices, const std::vector<double>& segment_times,
                         int derivative_to_optimize = kHighestDerivativeToOptimize) {
    return core_.setupFromVertices(vertices, segment_times, derivative_to_optimize);
  }

  static void setupMappingMatrix(double segment_time, SquareMatrix* A) {
    double a[N * N];
    b200::hostMappingMatrix(N, segment_time, a);
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) (*A)(i, j) = a[i * N + j];
  }
  // Inverts the matrix it is GIVEN, with the reference's Schur structure (linear_impl.h:142-179):
  // A = [[Lambda, 0], [C, Dm]] with Lambda diagonal  =>  A^-1 = [[Lambda^-1, 0], [-Dm^-1 C Lambda^-1, Dm^-1]], the
  // N/2 x N/2 block Dm inverted by Gauss-Jordan with partial pivoting.  (The solver itself never inverts anything:
  // it uses the exact table A(1)^-1 and the time scaling, see csrc/mtg_device.cuh.)
  static void invertMappingMatrix(const SquareMatrix& mapping_matrix, SquareMatrix* inverse_mapping_matrix) {
    double a[N * N], ai[N * N];
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) a[i * N + j] = mapping_matrix(i, j);
    b200::hostInvertStructured(N, a, ai);
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) (*inverse_mapping_matrix)(i, j) = ai[i * N + j];
  }
  static void computeQuadraticCostJacobian(int derivative, double t, SquareMatrix* cost_jacobian) {
    CHECK_LT(derivative, N);
    double q[N * N];
    b200::hostCostMatrix(N, derivative, t, q);
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) (*cost_jacobian)(i, j) = q[i * N + j];
  }

  // ---- extrema of the magnitude of a derivative (reference linear.h:138-176, linear_impl.h:388-470)
  template <int Derivative>
  static bool computeSegmentMaximumMagnitudeCandidates(const Segment& segment, double t_start, double t_stop,
                                                       std::vector<double>* candidates) {
    return computeSegmentMaximumMagnitudeCandidates(Derivative, segment, t_start, t_stop, candidates);
  }
  static bool computeSegmentMaximumMagnitudeCandidates(int derivative, const Segment& segment, double t_start,
                                                       double t_stop, std::vector<double>* candidates) {
    CHECK(candidates);
    CHECK(N - derivative - 1 > 0) << "N-Derivative-1 has to be greater 0";
    std::vector<int> dimensions(segment.D());
    std::iota(dimensions.begin(), dimensions.end(), 0);
    return segment.computeMinMaxMagnitudeCandidateTimes(derivative, t_start, t_stop, dimensions, candidates);
  }
  // Sampling-based variant "meant for debugging / testing" (linear.h:150-160): a sign change of the magnitude's
  // slope between consecutive samples marks a candidate when the next derivative is small there.
  template <int Derivative>
  static void computeSegmentMaximumMagnitudeCandidatesBySampling(const Segment& segment, double t_start,
                                                                 double t_stop, double dt,
                                                                 std::vector<double>* candidates) {
    CHECK_NOTNULL(candidates)->push_back(t_start);
    double t_old = t_start + dt;
    double norm_new = segment.evaluate(t_old, Derivative).norm();
    double direction = norm_new - segment.evaluate(t_start, Derivative).norm();
    bool last_sample = false;
    for (double t = t_start + dt + dt; t <= t_stop; t += dt) {
      const double norm_old = norm_new;
      norm_new = segment.evaluate(t, Derivative).norm();
      const double direction_new = norm_new - norm_old;
      if (std::signbit(direction) != std::signbit(direction_new) &&
          segment.evaluate(t_old, Derivative + 1).norm() < 1e-2)
        candidates->push_back(t_old);  // the extremum was at the previous sample
      direction = direction_new;
      t_old = t;
      if ((t + dt) > t_stop && !last_sample) {  // make sure the last sample before t_stop is taken
        t = t_stop - dt;
        last_sample = true;
      }
    }
    if (candidates->back() != t_stop) candidates->push_back(t_stop);
  }
  template <int Derivative>
  Extremum computeMaximumOfMagnitude(std::vector<Extremum>* candidates) const {
    return computeMaximumOfMagnitude(Derivative, candidates);
  }
  Extremum computeMaximumOfMagnitude(int derivative, std::vector<Extremum>* candidates) const {
    if (candidates != nullptr) candidates->clear();
    Extremum extremum;
    int segment_idx = 0;
    for (const Segment& s : core_.segments_) {
      std::vector<double> times;
      times.push_back(0.0);  // the call below clears and refills: start / end are among its candidates
      computeSegmentMaximumMagnitudeCandidates(derivative, s, 0.0, s.getTime(), &times);
      for (const double t : times) {
        const Extremum candidate(t, s.evaluate(t, derivative).norm(), segment_idx);
        if (extremum < candidate) extremum = candidate;
        if (candidates != nullptr) candidates->emplace_back(candidate);
      }
      ++segment_idx;
    }
    if (!core_.segments_.empty()) {
      const Segment& last = core_.segments_.back();
      const Extremum candidate(last.getTime(), last.evaluate(last.getTime(), derivative).norm(),
                               static_cast<int>(core_.segments_.size()) - 1);
      if (extremum < candidate) extremum = candidate;
      if (candidates != nullptr) candidates->emplace_back(candidate);
    }
    return extremum;
  }

  double computeCost() const { return core_.computeCost(); }
  void updateSegmentTimes(const std::vector<double>& segment_times) { core_.updateSegmentTimes(segment_times); }
  bool solveLinear() { return core_.solveLinear(); }

  void getTrajectory(Trajectory* trajectory) const { CHECK_NOTNULL(trajectory)->setSegments(core_.segments_); }
  void getVertices(Vertex::Vector* vertices) const { *CHECK_NOTNULL(vertices) = core_.vertices_; }
  void getSegments(Segment::Vector* segments) const { *CHECK_NOTNULL(segments) = core_.segments_; }
  void getSegmentTimes(std::vector<double>* segment_times) const {
    CHECK(segment_times != nullptr);
    *segment_times = core_.segment_times_;
  }
  void getFreeConstraints(std::vector<Eigen::VectorXd>* free_constraints) const {
    CHECK(free_constraints != nullptr);
    *free_constraints = core_.free_constraints_compact_;
  }
  void setFreeConstraints(const std::vector<Eigen::VectorXd>& free_constraints) {
    core_.setFreeConstraints(free_constraints);
  }
  void getFixedConstraints(std::vector<Eigen::VectorXd>* fixed_constraints) const {
    CHECK(fixed_constraints != nullptr);
    *fixed_constraints = core_.fixed_constraints_compact_;
  }

  size_t getDimension() const { return core_.dimension_; }
  size_t getNumberSegments() const { return static_cast<size_t>(core_.topo_.K); }
  size_t getNumberAllConstraints() const { return static_cast<size_t>(core_.topo_.n_all); }
  size_t getNumberFixedConstraints() const { return static_cast<size_t>(core_.topo_.n_fixed); }
  size_t getNumberFreeConstraints() const { return static_cast<size_t>(core_.topo_.n_free); }
  int getDerivativeToOptimize() const { return core_.topo_.r; }

  void getAInverse(Eigen::MatrixXd* A_inv) const { core_.getAInverse(CHECK_NOTNULL(A_inv)); }
  void getM(Eigen::MatrixXd* M) const { core_.getM(CHECK_NOTNULL(M)); }
  void getR(Eigen::MatrixXd* R) const { core_.getR(CHECK_NOTNULL(R)); }
  void getA(Eigen::MatrixXd* A) const { core_.getA(CHECK_NOTNULL(A)); }
  void getMpinv(Eigen::MatrixXd* M_pinv) const { core_.getMpinv(CHECK_NOTNULL(M_pinv)); }
  void printReorderingMatrix(std::ostream& stream) const {
    Eigen::MatrixXd M;
    core_.getM(&M);
    stream << "Mapping matrix:\n" << M << std::endl;
  }

  // Extension: status bits of the last solveLinear() (0 = solved; see MTG_STATUS_*).
  int getLastStatus() const { return core_.last_status_; }

 private:
  template <int>
  friend class PolynomialOptimizationNonLinear;  // runs the time optimiser on this problem's core
  b200::LinearCore core_;
};

}  // namespace mav_trajectory_generation
#endif
