// b200_feasibility.cpp -- InputConstraints, FeasibilityBase::checkInputFeasibilityTrajectory and
// FeasibilityAnalytic::checkInputFeasibility for one segment on the host (reference
// mav_trajectory_generation_ros/src/input_constraints.cpp, feasibility_base.cpp, feasibility_analytic.cpp), on the
// extremum candidates of b200_extrema.cpp.  The batched GPU form is mtg_input_feasibility_batch_f64.
#include <algorithm>
#include <cmath>
#include <limits>

#include "mav_trajectory_generation_ros/feasibility_analytic.h"

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
