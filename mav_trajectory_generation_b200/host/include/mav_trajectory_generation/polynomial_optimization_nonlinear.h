// polynomial_optimization_nonlinear.h -- the reference's PolynomialOptimizationNonLinear<N> (include/
// mav_trajectory_generation/polynomial_optimization_nonlinear.h) for the time allocation method this project
// provides, kMellingerOuterLoop, on the GPU with a batch of one (as PolynomialOptimization<N>).
//
// optimize() runs mtg_optimize_time_mellinger_batch_f64: the projected-gradient descent on the segment times that
// include/mtg_b200.h defines (the reference drives the same outer loop with NLopt), then
// scaleSegmentTimesWithViolation.  The other methods return INVALID_ARGS (-2, nlopt::INVALID_ARGS).
// NonlinearOptimizationParameters has the reference's fields and defaults except `algorithm` and `random_seed`, which
// name NLopt; equality / inequality tolerances, time_penalty and the soft constraints are kept for source
// compatibility and not read by kMellingerOuterLoop (nor by the reference's).
#ifndef MAV_TRAJECTORY_GENERATION_POLYNOMIAL_OPTIMIZATION_NONLINEAR_H_
#define MAV_TRAJECTORY_GENERATION_POLYNOMIAL_OPTIMIZATION_NONLINEAR_H_

#include <limits>
#include <map>
#include <vector>

#include "mav_trajectory_generation/extremum.h"
#include "mav_trajectory_generation/motion_defines.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"

namespace mav_trajectory_generation {

constexpr double kOptimizationTimeLowerBound = 0.1;

struct NonlinearOptimizationParameters {
  double f_abs = -1;
  double f_rel = 0.05;
  double x_rel = -1;
  double x_abs = -1;
  double initial_stepsize_rel = 0.1;
  double equality_constraint_tolerance = 1.0e-3;
  double inequality_constraint_tolerance = 0.1;
  int max_iterations = 3000;
  double time_penalty = 500.0;
  bool use_soft_constraints = true;
  double soft_constraint_weight = 100.0;
  enum TimeAllocMethod {
    kSquaredTime,
    kRichterTime,
    kMellingerOuterLoop,
    kSquaredTimeAndConstraints,
    kRichterTimeAndConstraints,
    kUnknown
  } time_alloc_method = kSquaredTimeAndConstraints;
  bool print_debug_info = false;
  bool print_debug_info_time_allocation = false;
};

struct OptimizationInfo {
  int n_iterations = 0;
  int stopping_reason = -1;  // nlopt::FAILURE
  double cost_trajectory = 0.0;
  double cost_time = 0.0;
  double cost_soft_constraints = 0.0;
  double optimization_time = 0.0;
  std::map<int, Extremum> maxima;
};

template <int _N = 10>
class PolynomialOptimizationNonLinear {
  static_assert(_N % 2 == 0, "The number of coefficients has to be even.");

 public:
  enum { N = _N };
  static constexpr int kInvalidArgs = -2;  // nlopt::INVALID_ARGS

  PolynomialOptimizationNonLinear(size_t dimension, const NonlinearOptimizationParameters& parameters)
      : poly_opt_(dimension), optimization_parameters_(parameters) {}

  bool setupFromVertices(const Vertex::Vector& vertices, const std::vector<double>& segment_times,
                         int derivative_to_optimize = PolynomialOptimization<N>::kHighestDerivativeToOptimize) {
    return poly_opt_.setupFromVertices(vertices, segment_times, derivative_to_optimize);
  }
  // Only the velocity and acceleration limits are read (by scaleSegmentTimesWithViolation), as in the reference.
  bool addMaximumMagnitudeConstraint(int derivative_order, double maximum_value) {
    if (derivative_order < 0 || !(maximum_value > 0.0)) return false;
    constraints_[derivative_order] = maximum_value;
    return true;
  }
  bool solveLinear() { return poly_opt_.solveLinear(); }

  // The time optimisation of time_alloc_method; returns the nlopt_result value (MTG_OPTIMIZE_RESULT_*).
  int optimize() {
    optimization_info_ = OptimizationInfo();
    if (optimization_parameters_.time_alloc_method != NonlinearOptimizationParameters::kMellingerOuterLoop)
      return kInvalidArgs;
    b200::MellingerParameters q;
    q.f_abs = optimization_parameters_.f_abs;
    q.f_rel = optimization_parameters_.f_rel;
    q.x_rel = optimization_parameters_.x_rel;
    q.x_abs = optimization_parameters_.x_abs;
    q.initial_stepsize_rel = optimization_parameters_.initial_stepsize_rel;
    q.max_iterations = optimization_parameters_.max_iterations;
    int result = -1, iterations = 0;
    if (!poly_opt_.core_.optimizeTimeMellinger(q, limit(derivative_order::VELOCITY),
                                               limit(derivative_order::ACCELERATION), &result, &iterations, nullptr))
      return -1;
    optimization_info_.n_iterations = iterations;
    optimization_info_.stopping_reason = result;
    optimization_info_.cost_trajectory = getCost();
    return result;
  }
  // Stretch the segment times until the velocity and acceleration limits hold, then solve again (reference
  // impl/polynomial_optimization_nonlinear_impl.h:366-406).
  void scaleSegmentTimesWithViolation() {
    poly_opt_.core_.scaleSegmentTimesWithViolation(limit(derivative_order::VELOCITY),
                                                   limit(derivative_order::ACCELERATION));
  }

  double getCost() const { return poly_opt_.computeCost(); }
  void getTrajectory(Trajectory* trajectory) const { poly_opt_.getTrajectory(trajectory); }
  const PolynomialOptimization<N>& getPolynomialOptimizationRef() const { return poly_opt_; }
  PolynomialOptimization<N>& getPolynomialOptimizationRef() { return poly_opt_; }
  OptimizationInfo getOptimizationInfo() const { return optimization_info_; }

 private:
  // the limit of one derivative order; a missing constraint is no limit (the reference passes 0 there and divides)
  double limit(int derivative) const {
    const auto it = constraints_.find(derivative);
    return it == constraints_.end() ? std::numeric_limits<double>::infinity() : it->second;
  }

  PolynomialOptimization<N> poly_opt_;
  NonlinearOptimizationParameters optimization_parameters_;
  std::map<int, double> constraints_;
  OptimizationInfo optimization_info_;
};

}  // namespace mav_trajectory_generation
#endif
