// feasibility_recursive.h -- recursive input feasibility of one segment (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/feasibility_recursive.h,
// src/feasibility_recursive.cpp): the segment is halved until, on every section, bounds on thrust, speed and the roll /
// pitch rate taken from single-axis extrema are within the limits, then yaw rate and yaw acceleration are checked over
// the whole segment.  This single-object path runs on the host (the mirror's own getRoots); batches of trajectories go
// through BatchPolynomialOptimization<N>::checkInputFeasibilityRecursive on the GPU.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_RECURSIVE_H_
#define MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_RECURSIVE_H_

#include <cmath>
#include <vector>

#include "mav_trajectory_generation/segment.h"
#include "mav_trajectory_generation_ros/feasibility_base.h"

namespace mav_trajectory_generation {

class FeasibilityRecursive : public FeasibilityBase {
 public:
  class Settings {
   public:
    Settings() : min_section_time_s_(0.05) {}
    void setMinSectionTimeS(double min_section_time_s) { min_section_time_s_ = std::abs(min_section_time_s); }
    double getMinSectionTimeS() const { return min_section_time_s_; }

   private:
    // the shortest section the bisection examines; a shorter one is Indeterminable
    double min_section_time_s_;
  };

  FeasibilityRecursive() {}
  explicit FeasibilityRecursive(const Settings& settings) : settings_(settings) {}
  explicit FeasibilityRecursive(const InputConstraints& input_constraints) : FeasibilityBase(input_constraints) {}
  FeasibilityRecursive(const Settings& settings, const InputConstraints& input_constraints)
      : FeasibilityBase(input_constraints), settings_(settings) {}

  InputFeasibilityResult checkInputFeasibility(const Segment& segment) const override;

  Settings settings_;

 private:
  typedef std::vector<Eigen::VectorXcd> Roots;
  InputFeasibilityResult recursiveFeasibility(const Segment& segment, const Roots& roots_acc, const Roots& roots_jerk,
                                              const Roots& roots_snap, double t_1, double t_2) const;
  double evaluateThrust(const Segment& segment, double time) const;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_RECURSIVE_H_
