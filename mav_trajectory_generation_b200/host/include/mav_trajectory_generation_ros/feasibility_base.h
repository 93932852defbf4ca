// feasibility_base.h -- input feasibility results and the trajectory-level check (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/feasibility_base.h, src/feasibility_base.cpp).
// Half-plane feasibility is not mirrored.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_
#define MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_

#include <string>

#include "mav_trajectory_generation/trajectory.h"
#include "mav_trajectory_generation_ros/input_constraints.h"

namespace mav_trajectory_generation {

// Equal to the MTG_FEAS_* codes of include/mtg_b200.h.
enum InputFeasibilityResult {
  kInputFeasible = 0,              // within every present limit
  kInputIndeterminable,            // cannot be decided (also: D not 3 or 4, a section below the minimum time)
  kInputInfeasibleThrustHigh,      // failed the maximum thrust test first
  kInputInfeasibleThrustLow,       // failed the minimum thrust test first
  kInputInfeasibleVelocity,        // failed the speed test first
  kInputInfeasibleRollPitchRates,  // failed the roll / pitch rate test first (not returned by FeasibilityAnalytic)
  kInputInfeasibleYawRates,        // failed the yaw rate test first
  kInputInfeasibleYawAcc,          // failed the yaw acceleration test first
};

std::string getInputFeasibilityResultName(InputFeasibilityResult fr);

class FeasibilityBase {
 public:
  FeasibilityBase() : gravity_(0.0, 0.0, kGravity) {}
  explicit FeasibilityBase(const InputConstraints& input_constraints)
      : input_constraints_(input_constraints), gravity_(0.0, 0.0, kGravity) {}
  virtual ~FeasibilityBase() {}

  // The result of the first segment that is not feasible, in order; feasible when every segment is, Indeterminable
  // for a trajectory without segments.
  InputFeasibilityResult checkInputFeasibilityTrajectory(const Trajectory& trajectory) const;
  // The base class cannot decide: Indeterminable.
  virtual InputFeasibilityResult checkInputFeasibility(const Segment& /*segment*/) const {
    return kInputIndeterminable;
  }
  InputConstraints getInputConstraints() const { return input_constraints_; }

  InputConstraints input_constraints_;
  Eigen::Vector3d gravity_;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_
