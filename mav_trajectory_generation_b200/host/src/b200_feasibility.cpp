// b200_feasibility.cpp -- InputConstraints, FeasibilityBase::checkInputFeasibilityTrajectory,
// FeasibilityAnalytic::checkInputFeasibility, FeasibilityRecursive::checkInputFeasibility and
// FeasibilitySampling::checkInputFeasibility for one segment on the host (reference
// mav_trajectory_generation_ros/src/input_constraints.cpp, feasibility_base.cpp, feasibility_analytic.cpp,
// feasibility_recursive.cpp, feasibility_sampling.cpp), on the extremum candidates and roots of b200_extrema.cpp.  The
// batched GPU forms are mtg_input_feasibility_batch_f64, mtg_input_feasibility_recursive_batch_f64 and
// mtg_input_feasibility_sampling_batch_f64.
#include <algorithm>
#include <cmath>
#include <limits>

#include "mav_trajectory_generation_ros/feasibility_analytic.h"
#include "mav_trajectory_generation_ros/feasibility_recursive.h"
#include "mav_trajectory_generation_ros/feasibility_sampling.h"
#include "mav_trajectory_generation/trajectory_sampling.h"

namespace mav_trajectory_generation {

namespace {
const std::vector<int> kPositionDims = {0, 1, 2};
}

std::string getInputConstraintName(InputConstraintType type) {
  switch (type) {
    case kFMin: return "f_min";
    case kFMax: return "f_max";
    case kVMax: return "v_max";
    case kOmegaXYMax: return "omega_xy_max";
    case kOmegaZMax: return "omega_z_max";
    case kOmegaZDotMax: return "omega_z_dot_max";
  }
  return "Unknown!";
}

void InputConstraints::addConstraint(int constraint_type, double value) {
  value = std::abs(value);
  if (constraint_type == kFMin && hasConstraint(kFMax)) {
    constraints_[kFMax] = std::max(constraints_[kFMax], value);
  } else if (constraint_type == kFMax && hasConstraint(kFMin)) {
    constraints_[kFMin] = std::min(constraints_[kFMin], value);
  }
  constraints_[constraint_type] = value;
}

void InputConstraints::setDefaultValues() {
  const double pi = 3.14159265358979323846;
  constraints_[kFMin] = 0.5 * kGravity;
  constraints_[kFMax] = 1.5 * kGravity;
  constraints_[kVMax] = 3.0;
  constraints_[kOmegaXYMax] = pi / 2.0;
  constraints_[kOmegaZMax] = pi / 2.0;
  constraints_[kOmegaZDotMax] = 2.0 * pi;
}

bool InputConstraints::getConstraint(int constraint_type, double* value) const {
  CHECK_NOTNULL(value);
  const auto it = constraints_.find(constraint_type);
  if (it == constraints_.end()) return false;
  *value = it->second;
  return true;
}

bool InputConstraints::hasConstraint(int constraint_type) const { return constraints_.count(constraint_type) > 0; }

bool InputConstraints::removeConstraint(int constraint_type) { return constraints_.erase(constraint_type) > 0; }

std::string getInputFeasibilityResultName(InputFeasibilityResult fr) {
  switch (fr) {
    case kInputFeasible: return "Feasible";
    case kInputIndeterminable: return "Indeterminable";
    case kInputInfeasibleThrustHigh: return "InfeasibleThrustHigh";
    case kInputInfeasibleThrustLow: return "InfeasibleThrustLow";
    case kInputInfeasibleVelocity: return "InfeasibleVelocity";
    case kInputInfeasibleRollPitchRates: return "InfeasibleRollPitchRates";
    case kInputInfeasibleYawRates: return "InfeasibleYawRates";
    case kInputInfeasibleYawAcc: return "InfeasibleYawAcc";
  }
  return "Unknown!";
}

InputFeasibilityResult FeasibilityBase::checkInputFeasibilityTrajectory(const Trajectory& trajectory) const {
  InputFeasibilityResult result = kInputIndeterminable;
  for (const Segment& segment : trajectory.segments()) {
    result = checkInputFeasibility(segment);
    if (result != kInputFeasible) return result;
  }
  return result;
}

HalfPlane::HalfPlane(const Eigen::Vector3d& point, const Eigen::Vector3d& normal) : point(point), normal(normal) {
  CHECK_GT(normal.norm(), 0.0) << "Invalid normal.";
  this->normal.normalize();
}

HalfPlane::HalfPlane(const Eigen::Vector3d& a, const Eigen::Vector3d& b, const Eigen::Vector3d& c) {
  CHECK(a != b);
  CHECK(a != c);
  point = a;
  normal = (b - a).cross(c - a).normalized();
}

HalfPlane::Vector HalfPlane::createBoundingBox(const Eigen::Vector3d& point, const Eigen::Vector3d& bounding_box_size) {
  const Eigen::Vector3d lower = point - bounding_box_size / 2.0, upper = point + bounding_box_size / 2.0;
  HalfPlane::Vector box;
  for (int axis = 0; axis < 3; ++axis) {
    Eigen::Vector3d inward(0.0, 0.0, 0.0);
    inward[axis] = 1.0;
    box.emplace_back(lower, inward);
    box.emplace_back(upper, -inward);
  }
  return box;
}

bool FeasibilityBase::checkHalfPlaneFeasibility(const Trajectory& trajectory) const {
  for (const Segment& segment : trajectory.segments())
    if (!checkHalfPlaneFeasibility(segment)) return false;
  return true;
}

bool FeasibilityBase::checkHalfPlaneFeasibility(const Segment& segment) const {
  if (segment.D() != 3 && segment.D() != 4) {
    LOG(WARNING) << "Half-plane feasibility needs D = 3 or 4, got " << segment.D() << ".";
    return false;
  }
  for (const HalfPlane& hp : half_plane_constraints_) {
    // the position projected on the normal; its extrema are where the segment comes closest to the plane
    Polynomial projection(segment.N());
    for (int d = 0; d < 3; ++d) projection += segment[d] * hp.normal[d];
    std::vector<double> times;
    projection.computeMinMaxCandidates(0.0, segment.getTime(), derivative_order::POSITION, &times);
    for (const double t : times) {
      const Eigen::VectorXd p = segment.evaluate(t).head(3);
      if ((p - Eigen::VectorXd(hp.point)).dot(hp.normal) <= 0.0) return false;
    }
  }
  return true;
}

InputFeasibilityResult FeasibilityAnalytic::checkInputFeasibility(const Segment& segment) const {
  if (segment.D() != 3 && segment.D() != 4) return kInputIndeterminable;
  const InputConstraints& ic = input_constraints_;
  // thrust (also needed by the roll / pitch bound)
  std::vector<Extremum> thrust_candidates;
  Segment thrust_segment(segment.N() - 2, static_cast<int>(kPositionDims.size()));
  if (ic.hasConstraint(kFMin) || ic.hasConstraint(kFMax) || ic.hasConstraint(kOmegaXYMax)) {
    const InputFeasibilityResult r = thrustFeasibility(segment, &thrust_candidates, &thrust_segment);
    if (r != kInputFeasible) return r;
  }
  // speed over the position dimensions
  double limit;
  if (ic.getConstraint(kVMax, &limit)) {
    std::vector<Extremum> candidates;
    if (!segment.computeMinMaxMagnitudeCandidates(derivative_order::VELOCITY, 0.0, segment.getTime(), kPositionDims,
                                                  &candidates))
      return kInputIndeterminable;
    if (std::max_element(candidates.begin(), candidates.end())->value > limit) return kInputInfeasibleVelocity;
  }
  // yaw rate and acceleration: signed extrema of the yaw polynomial's derivatives
  if (segment.D() == 4) {
    const int orders[2] = {derivative_order::ANGULAR_VELOCITY, derivative_order::ANGULAR_ACCELERATION};
    const int types[2] = {kOmegaZMax, kOmegaZDotMax};
    const InputFeasibilityResult fails[2] = {kInputInfeasibleYawRates, kInputInfeasibleYawAcc};
    for (int q = 0; q < 2; ++q) {
      if (!ic.getConstraint(types[q], &limit)) continue;
      std::pair<double, double> lo, hi;
      if (!segment[3].computeMinMax(0.0, segment.getTime(), orders[q], &lo, &hi)) return kInputIndeterminable;
      if (std::max(std::abs(lo.second), std::abs(hi.second)) > limit) return fails[q];
    }
  }
  // roll / pitch rates
  if (ic.hasConstraint(kOmegaXYMax)) {
    std::vector<Extremum> jerk_candidates;
    if (!segment.computeMinMaxMagnitudeCandidates(derivative_order::JERK, 0.0, segment.getTime(), kPositionDims,
                                                  &jerk_candidates))
      return kInputIndeterminable;
    const InputFeasibilityResult r =
        rollPitchFeasibility(segment, thrust_segment, thrust_candidates, jerk_candidates, 0.0, segment.getTime());
    if (r != kInputFeasible) return r;
  }
  return kInputFeasible;
}

// thrust f = p'' + gravity over the position dimensions: its polynomial has N - 2 coefficients
InputFeasibilityResult FeasibilityAnalytic::thrustFeasibility(const Segment& segment,
                                                              std::vector<Extremum>* thrust_candidates,
                                                              Segment* thrust_segment) const {
  thrust_segment->setTime(segment.getTime());
  for (int i = 0; i < thrust_segment->D(); ++i) {
    Eigen::VectorXd c = segment[i].getCoefficients(derivative_order::ACCELERATION).head(thrust_segment->N());
    c[0] += gravity_[i];
    (*thrust_segment)[i] = Polynomial(c);
  }
  if (!thrust_segment->computeMinMaxMagnitudeCandidates(derivative_order::POSITION, 0.0, thrust_segment->getTime(),
                                                        kPositionDims, thrust_candidates))
    return kInputIndeterminable;
  double limit;
  if (input_constraints_.getConstraint(kFMin, &limit) &&
      std::min_element(thrust_candidates->begin(), thrust_candidates->end())->value < limit)
    return kInputInfeasibleThrustLow;
  if (input_constraints_.getConstraint(kFMax, &limit) &&
      std::max_element(thrust_candidates->begin(), thrust_candidates->end())->value > limit)
    return kInputInfeasibleThrustHigh;
  return kInputFeasible;
}

// Depth first, left half first: a section whose bound sqrt(j_max / f_min) exceeds omega_xy_max is halved, one shorter
// than the minimum section time is Indeterminable.  f_min and j_max come from the candidates inside [t_1, t_2].
InputFeasibilityResult FeasibilityAnalytic::rollPitchFeasibility(const Segment& segment, const Segment& thrust_segment,
                                                                 const std::vector<Extremum>& thrust_candidates,
                                                                 const std::vector<Extremum>& jerk_candidates,
                                                                 double t_1, double t_2) const {
  if (t_2 - t_1 < settings_.getMinSectionTimeS()) return kInputIndeterminable;
  Extremum f_min, f_max, j_min, j_max;
  if (!thrust_segment.selectMinMaxMagnitudeFromCandidates(derivative_order::POSITION, t_1, t_2, kPositionDims,
                                                          thrust_candidates, &f_min, &f_max) ||
      !segment.selectMinMaxMagnitudeFromCandidates(derivative_order::JERK, t_1, t_2, kPositionDims, jerk_candidates,
                                                   &j_min, &j_max))
    return kInputIndeterminable;
  // no jerk candidate leaves j_max at lowest(): the bound is NaN and compares false
  const double bound = f_min.value > 1.0e-6 ? std::sqrt(j_max.value / f_min.value) : std::numeric_limits<double>::max();
  double limit;
  if (!input_constraints_.getConstraint(kOmegaXYMax, &limit)) return kInputFeasible;
  if (!(bound > limit)) return kInputFeasible;
  const double t_half = (t_1 + t_2) / 2;
  const InputFeasibilityResult left =
      rollPitchFeasibility(segment, thrust_segment, thrust_candidates, jerk_candidates, t_1, t_half);
  if (left != kInputFeasible) return left;
  return rollPitchFeasibility(segment, thrust_segment, thrust_candidates, jerk_candidates, t_half, t_2);
}

}  // namespace mav_trajectory_generation

// ---- FeasibilityRecursive (reference src/feasibility_recursive.cpp) -------------------------------------------------
// std::pow(x, 2) of the reference is x * x here: an optimised x86 build computes it with one multiplication.

namespace mav_trajectory_generation {

namespace {
inline double square(double x) { return x * x; }
}  // namespace

InputFeasibilityResult FeasibilityRecursive::checkInputFeasibility(const Segment& segment) const {
  if (segment.D() != 3 && segment.D() != 4) return kInputIndeterminable;
  const InputConstraints& ic = input_constraints_;
  // per position axis, the roots of the derivative of each order the sections bound
  Roots roots_acc, roots_jerk, roots_snap;
  const bool need[3] = {ic.hasConstraint(kVMax),
                        ic.hasConstraint(kFMin) || ic.hasConstraint(kFMax) || ic.hasConstraint(kOmegaXYMax),
                        ic.hasConstraint(kOmegaXYMax)};
  Roots* lists[3] = {&roots_acc, &roots_jerk, &roots_snap};
  const int orders[3] = {derivative_order::ACCELERATION, derivative_order::JERK, derivative_order::SNAP};
  for (int q = 0; q < 3; ++q) {
    if (!need[q]) continue;
    lists[q]->resize(3);
    for (int i = 0; i < 3; ++i)
      if (!segment[i].getRoots(orders[q], &(*lists[q])[i])) return kInputIndeterminable;
  }
  const InputFeasibilityResult result =
      recursiveFeasibility(segment, roots_acc, roots_jerk, roots_snap, 0.0, segment.getTime());
  if (result != kInputFeasible || segment.D() != 4) return result;
  // yaw rate and acceleration over the whole segment (independent of the translation in the rigid-body model)
  const int yaw_orders[2] = {derivative_order::ANGULAR_VELOCITY, derivative_order::ANGULAR_ACCELERATION};
  const int types[2] = {kOmegaZMax, kOmegaZDotMax};
  const InputFeasibilityResult fails[2] = {kInputInfeasibleYawRates, kInputInfeasibleYawAcc};
  for (int q = 0; q < 2; ++q) {
    double limit;
    if (!ic.getConstraint(types[q], &limit)) continue;
    std::pair<double, double> lo, hi;
    if (!segment[3].computeMinMax(0.0, segment.getTime(), yaw_orders[q], &lo, &hi)) return kInputIndeterminable;
    if (std::max(std::abs(lo.second), std::abs(hi.second)) > limit) return fails[q];
  }
  return kInputFeasible;
}

// One section [t_1, t_2]: the end points first, then bounds from the single-axis extrema; a section whose bounds are
// not conclusive is halved, left half first.
InputFeasibilityResult FeasibilityRecursive::recursiveFeasibility(const Segment& segment, const Roots& roots_acc,
                                                                  const Roots& roots_jerk, const Roots& roots_snap,
                                                                  double t_1, double t_2) const {
  if (t_2 - t_1 < settings_.getMinSectionTimeS()) return kInputIndeterminable;
  const InputConstraints& ic = input_constraints_;
  double f_min_limit = 0.0, f_max_limit = 0.0, v_max_limit = 0.0, omega_xy_limit = 0.0;
  const bool has_f_min = ic.getConstraint(kFMin, &f_min_limit), has_f_max = ic.getConstraint(kFMax, &f_max_limit);
  const bool has_v_max = ic.getConstraint(kVMax, &v_max_limit);
  const bool has_omega_xy = ic.getConstraint(kOmegaXYMax, &omega_xy_limit);
  // thrust and speed at the section's ends
  if (has_f_min || has_f_max) {
    const double f_1 = evaluateThrust(segment, t_1), f_2 = evaluateThrust(segment, t_2);
    if (has_f_min && std::min(f_1, f_2) < f_min_limit) return kInputInfeasibleThrustLow;
    if (has_f_max && std::max(f_1, f_2) > f_max_limit) return kInputInfeasibleThrustHigh;
  }
  if (has_v_max) {
    const double v_1 = segment.evaluate(t_1, derivative_order::VELOCITY).head(3).norm();
    const double v_2 = segment.evaluate(t_2, derivative_order::VELOCITY).head(3).norm();
    if (std::max(v_1, v_2) > v_max_limit) return kInputInfeasibleVelocity;
  }
  // squared bounds summed over the axes
  double f_min_sqr = 0.0, f_max_sqr = 0.0, v_max_sqr = 0.0, j_max_sqr = 0.0;
  if (has_v_max) {
    for (int i = 0; i < 3; ++i) {
      std::pair<double, double> lo, hi;
      segment[i].selectMinMaxFromRoots(t_1, t_2, derivative_order::VELOCITY, roots_acc[i], &lo, &hi);
      // one axis alone faster than the limit
      if (std::max(square(lo.second), square(hi.second)) > square(v_max_limit)) return kInputInfeasibleVelocity;
      v_max_sqr += square(std::max(std::abs(lo.second), std::abs(hi.second)));
    }
  }
  if (has_f_min || has_f_max || has_omega_xy) {
    for (int i = 0; i < 3; ++i) {
      std::pair<double, double> lo, hi;
      segment[i].selectMinMaxFromRoots(t_1, t_2, derivative_order::ACCELERATION, roots_jerk[i], &lo, &hi);
      const double f_lo = lo.second + gravity_[i], f_hi = hi.second + gravity_[i];
      // one axis alone above the thrust limit
      if (has_f_max && std::max(std::abs(f_lo), std::abs(f_hi)) > f_max_limit) return kInputInfeasibleThrustHigh;
      // an axis whose thrust changes sign contributes nothing to the lower bound
      if (!(f_lo * f_hi < 0.0)) f_min_sqr += square(std::min(std::abs(f_lo), std::abs(f_hi)));
      f_max_sqr += square(std::max(std::abs(f_lo), std::abs(f_hi)));
    }
  }
  if (has_omega_xy) {
    for (int i = 0; i < 3; ++i) {
      std::pair<double, double> lo, hi;
      segment[i].selectMinMaxFromRoots(t_1, t_2, derivative_order::JERK, roots_snap[i], &lo, &hi);
      j_max_sqr += square(std::max(std::abs(lo.second), std::abs(hi.second)));
    }
  }
  const double f_lower = std::sqrt(f_min_sqr), f_upper = std::sqrt(f_max_sqr), v_upper = std::sqrt(v_max_sqr);
  // Mueller's roll / pitch rate bound |j| / |f|, unbounded where the thrust may vanish
  const double omega_xy_upper =
      f_min_sqr > 1.0e-6 ? std::sqrt(j_max_sqr / f_min_sqr) : std::numeric_limits<double>::max();
  if (has_f_min && f_upper < f_min_limit) return kInputInfeasibleThrustLow;
  if (has_f_max && f_lower > f_max_limit) return kInputInfeasibleThrustHigh;
  if ((has_f_min && f_lower < f_min_limit) || (has_f_max && f_upper > f_max_limit) ||
      (has_v_max && v_upper > v_max_limit) || (has_omega_xy && omega_xy_upper > omega_xy_limit)) {
    const double t_half = (t_1 + t_2) / 2;
    const InputFeasibilityResult left = recursiveFeasibility(segment, roots_acc, roots_jerk, roots_snap, t_1, t_half);
    if (left != kInputFeasible) return left;
    return recursiveFeasibility(segment, roots_acc, roots_jerk, roots_snap, t_half, t_2);
  }
  return kInputFeasible;
}

// |p''(t) + gravity| over the position dimensions, the acceleration evaluated first
double FeasibilityRecursive::evaluateThrust(const Segment& segment, double time) const {
  const Eigen::VectorXd a = segment.evaluate(time, derivative_order::ACCELERATION);
  double sq = 0.0;
  for (int i = 0; i < 3; ++i) sq += square(a[i] + gravity_[i]);
  return std::sqrt(sq);
}

}  // namespace mav_trajectory_generation

// ---- FeasibilitySampling (reference src/feasibility_sampling.cpp) ---------------------------------------------------

namespace mav_trajectory_generation {

InputFeasibilityResult FeasibilitySampling::checkInputFeasibility(const Segment& segment) const {
  if (segment.D() != 3 && segment.D() != 4) return kInputIndeterminable;
  const InputConstraints& ic = input_constraints_;
  double f_min, f_max, v_max, omega_xy_max, omega_z_max, omega_z_dot_max;
  const bool has_f_min = ic.getConstraint(kFMin, &f_min), has_f_max = ic.getConstraint(kFMax, &f_max);
  const bool has_v_max = ic.getConstraint(kVMax, &v_max), has_omega_xy = ic.getConstraint(kOmegaXYMax, &omega_xy_max);
  const bool has_omega_z = ic.getConstraint(kOmegaZMax, &omega_z_max);
  const bool has_omega_z_dot = ic.getConstraint(kOmegaZDotMax, &omega_z_dot_max);
  // the sample times are a running sum, as in the reference (T itself is missed when the sum overshoots it)
  for (double t = 0.0; t <= segment.getTime(); t += settings_.getSamplingIntervalS()) {
    const Eigen::VectorXd position = segment.evaluate(t, derivative_order::POSITION);
    const Eigen::VectorXd velocity = segment.evaluate(t, derivative_order::VELOCITY);
    const Eigen::VectorXd acc = segment.evaluate(t, derivative_order::ACCELERATION);
    mav_msgs::EigenTrajectoryPoint flat_state;
    sampling_detail::head3(position, &flat_state.position_W);
    sampling_detail::head3(velocity, &flat_state.velocity_W);
    sampling_detail::head3(acc, &flat_state.acceleration_W);
    sampling_detail::head3(segment.evaluate(t, derivative_order::JERK), &flat_state.jerk_W);
    flat_state.setFromYawRate(0.0);
    flat_state.setFromYawAcc(0.0);
    if (segment.D() == 4) {
      flat_state.setFromYaw(position[3]);
      flat_state.setFromYawRate(velocity[3]);
      flat_state.setFromYawAcc(acc[3]);
    }
    mav_msgs::EigenMavState state;
    mav_msgs::EigenMavStateFromEigenTrajectoryPoint(flat_state, gravity_[2], &state);
    if (has_f_min || has_f_max) {
      const double thrust = state.acceleration_B.norm();
      if (has_f_min && thrust < f_min) return kInputInfeasibleThrustLow;
      if (has_f_max && thrust > f_max) return kInputInfeasibleThrustHigh;
    }
    if (has_v_max && state.velocity_W.norm() > v_max) return kInputInfeasibleVelocity;
    // roll / pitch and yaw rates assume independent axes (rigid-body model)
    if (has_omega_xy && state.angular_velocity_B.head(2).norm() > omega_xy_max) return kInputInfeasibleRollPitchRates;
    if (has_omega_z && std::fabs(state.angular_velocity_B[2]) > omega_z_max) return kInputInfeasibleYawRates;
    if (has_omega_z_dot && std::fabs(state.angular_acceleration_B[2]) > omega_z_dot_max)
      return kInputInfeasibleYawAcc;
  }
  return kInputFeasible;
}

}  // namespace mav_trajectory_generation
