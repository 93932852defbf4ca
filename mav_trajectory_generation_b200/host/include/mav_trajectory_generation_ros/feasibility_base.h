// feasibility_base.h -- input feasibility results and the trajectory-level check (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/feasibility_base.h, src/feasibility_base.cpp),
// and the half-plane (workspace) check of single segments and trajectories.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_
#define MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_

#include <string>
#include <vector>

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

// A half-space {x : (x - point) . normal > 0}.  The normal is normalised on construction, as in the reference.
class HalfPlane {
 public:
  typedef std::vector<HalfPlane, Eigen::aligned_allocator<HalfPlane>> Vector;
  // point on the plane and a normal pointing into the allowed side (CHECKs that the normal is not zero)
  HalfPlane(const Eigen::Vector3d& point, const Eigen::Vector3d& normal);
  // the plane through a, b and c, normal (b - a) x (c - a) (CHECKs b != a and c != a)
  HalfPlane(const Eigen::Vector3d& a, const Eigen::Vector3d& b, const Eigen::Vector3d& c);
  // six planes bounding the axis-aligned box of the given size around point: for each axis, the lower face (normal
  // +e_axis) and then the upper face (normal -e_axis)
  static HalfPlane::Vector createBoundingBox(const Eigen::Vector3d& point, const Eigen::Vector3d& bounding_box_size);

  Eigen::Vector3d point;
  Eigen::Vector3d normal;
};

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

  // true when every segment passes checkHalfPlaneFeasibility(segment)
  bool checkHalfPlaneFeasibility(const Trajectory& trajectory) const;
  // true when the segment's position stays strictly inside every half-space of half_plane_constraints_ at the extremum
  // candidates of its projection on each normal (0, T and the real critical points in [0, T]); false for D not 3 or 4.
  // Runs on the host; batches go through BatchPolynomialOptimization<N>::checkHalfPlaneFeasibility on the GPU.
  bool checkHalfPlaneFeasibility(const Segment& segment) const;

  InputConstraints input_constraints_;
  HalfPlane::Vector half_plane_constraints_;
  Eigen::Vector3d gravity_;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_BASE_H_
