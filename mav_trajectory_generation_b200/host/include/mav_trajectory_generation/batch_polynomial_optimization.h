// batch_polynomial_optimization.h -- B independent problems of ONE constraint topology solved in a
// single pass of the H100 kernels.  This is the throughput entry point: the reference solves one
// trajectory per PolynomialOptimization<N> object (its benchmark loops over objects,
// src/polynomial_timing_evaluation.cpp:93-112); here the loop is the GPU grid.
// Buffers are pinned host memory; solveLinear() pipelines H2D / kernels / D2H.
#ifndef MAV_TRAJECTORY_GENERATION_BATCH_POLYNOMIAL_OPTIMIZATION_H_
#define MAV_TRAJECTORY_GENERATION_BATCH_POLYNOMIAL_OPTIMIZATION_H_

#include <vector>

#include "mav_trajectory_generation/b200_core.h"

namespace mav_trajectory_generation {

template <int _N = 10>
class BatchPolynomialOptimization {
  static_assert(_N % 2 == 0, "The number of coefficients has to be even.");

 public:
  enum { N = _N };
  static constexpr int kHighestDerivativeToOptimize = N / 2 - 1;

  explicit BatchPolynomialOptimization(size_t dimension) : core_(N, dimension) {}

  // Every problem must fix the same derivatives at the same vertices as vertices[0]; the
  // constraint values and the segment times are per problem.
  bool setupFromVertices(const std::vector<Vertex::Vector>& vertices,
                         const std::vector<std::vector<double> >& segment_times,
                         int derivative_to_optimize = kHighestDerivativeToOptimize) {
    return core_.setupFromVertices(vertices, segment_times, derivative_to_optimize);
  }
  // createRandomVertices topology straight from flat arrays: positions[B][K+1][D], times[B][K];
  // start/end derivatives 1..N/2-1 are zero (Vertex::makeStartOrEnd).
  bool setupFromWaypoints(size_t batch, size_t n_segments, const double* positions, const double* segment_times,
                          int derivative_to_optimize = kHighestDerivativeToOptimize) {
    return core_.setupFromWaypoints(batch, n_segments, positions, segment_times, derivative_to_optimize);
  }
  bool solveLinear() { return core_.solveLinear(); }
  // SURVEY.md 8f-1: estimateSegmentTimesNfabian(v_max, a_max, magic) + packing + solve fused on the device;
  // afterwards getSegments()/coefficients() hold the result and segmentTimes() the allocated times.
  bool solveWaypointsNfabian(size_t batch, size_t n_segments, const double* positions, double v_max, double a_max,
                             double magic_fabian_constant = 6.5,
                             int derivative_to_optimize = kHighestDerivativeToOptimize) {
    return core_.solveWaypointsNfabian(batch, n_segments, positions, derivative_to_optimize, v_max, a_max,
                                       magic_fabian_constant);
  }
  const double* segmentTimes() const { return core_.times_; }  // [B][K]

  size_t size() const { return core_.B_; }
  size_t getDimension() const { return core_.dimension_; }
  size_t getNumberSegments() const { return static_cast<size_t>(core_.topo_.K); }
  size_t getNumberFixedConstraints() const { return static_cast<size_t>(core_.topo_.n_fixed); }
  size_t getNumberFreeConstraints() const { return static_cast<size_t>(core_.topo_.n_free); }

  void getSegments(size_t b, Segment::Vector* segments) const { core_.getSegments(b, CHECK_NOTNULL(segments)); }
  void getTrajectory(size_t b, Trajectory* trajectory) const {
    Segment::Vector s;
    core_.getSegments(b, &s);
    CHECK_NOTNULL(trajectory)->setSegments(s);
  }
  // Flat results: coefficients()[((b*K + segment)*D + dim)*N + power], status()[b].
  const double* coefficients() const { return core_.coeffs_; }
  const double* freeConstraints() const { return core_.d_free_; }  // [B][D][n_free]
  const int32_t* status() const { return core_.status_; }
  std::vector<double> computeCosts() const { return core_.computeCosts(); }
  // SURVEY.md 8f-2: PolynomialOptimizationNonLinear::getCostAndGradientMellinger (reference
  // impl/polynomial_optimization_nonlinear_impl.h:286-364) for every problem of the batch at its current segment
  // times: cost[b] and grad[b*K + n], the K+1 re-solves per problem fused into one cost-only device pass.
  void costGradientMellinger(std::vector<double>* cost, std::vector<double>* grad) const {
    core_.costGradientMellinger(cost, grad);
  }
  // SURVEY.md 8f-3: Trajectory::evaluateRange (reference src/trajectory.cpp:81-141) of every solved trajectory;
  // derivatives = {0,1,2,3,4} gives the sample set of sampleTrajectoryInRange (src/trajectory_sampling.cpp:45-110).
  // samples[((b*max_samples + s)*n_derivs + q)*D + dim], n_samples[b] as the reference would produce (-1: t_start
  // beyond the trajectory).
  void evaluateRange(double t_start, double t_end, double dt, const std::vector<int>& derivatives, int max_samples,
                     std::vector<double>* samples, std::vector<int32_t>* n_samples,
                     std::vector<double>* sampling_times = nullptr) const {
    core_.evaluateRange(t_start, t_end, dt, derivatives, max_samples, samples, n_samples, sampling_times);
  }
  // PolynomialOptimization::computeMaximumOfMagnitude (reference impl/polynomial_optimization_linear_impl.h:465-497) of
  // every trajectory for each derivative order (each in [0, N-2], at most 8): maxima[b * derivatives.size() + q].
  void computeMaximaOfMagnitude(const std::vector<int>& derivatives, std::vector<Extremum>* maxima) const {
    core_.computeMaximaOfMagnitude(derivatives, maxima);
  }
  // The nonlinear optimiser's objective for every problem at its current segment times (reference
  // impl/polynomial_optimization_nonlinear_impl.h): objectiveFunctionTime when d_free is nullptr (solve), otherwise
  // objectiveFunctionTimeAndConstraints with d_free [B][D][n_free] (setFreeConstraints).  objective[b] is NaN where
  // status()[b] != 0; terms[3 * b + {0, 1, 2}] = trajectory, time and soft-constraint cost.  The evaluated
  // trajectories replace coefficients().
  bool timeObjective(const b200::TimeObjectiveParameters& params, const double* d_free, std::vector<double>* objective,
                     std::vector<double>* terms = nullptr) {
    return core_.timeObjective(params, d_free, objective, terms);
  }

 private:
  b200::BatchCore core_;
};

}  // namespace mav_trajectory_generation
#endif
