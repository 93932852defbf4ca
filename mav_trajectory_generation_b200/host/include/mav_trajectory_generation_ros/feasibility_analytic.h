// feasibility_analytic.h -- analytic input feasibility of one segment (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/feasibility_analytic.h,
// src/feasibility_analytic.cpp): thrust, speed, yaw rate and yaw acceleration from their extremum candidates, and the
// roll / pitch rate bound of Mueller, Hehn and D'Andrea (IEEE T-RO 31(6), 2015) on recursively halved sections.
// This single-object path runs on the host (the extremum candidates of b200_extrema.cpp); batches of trajectories go
// through BatchPolynomialOptimization<N>::checkInputFeasibility on the GPU.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_ANALYTIC_H_
#define MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_ANALYTIC_H_

#include <cmath>
#include <vector>

#include "mav_trajectory_generation/segment.h"
#include "mav_trajectory_generation_ros/feasibility_base.h"

namespace mav_trajectory_generation {

class FeasibilityAnalytic : public FeasibilityBase {
 public:
  class Settings {
   public:
    Settings() : min_section_time_s_(0.05) {}
    void setMinSectionTimeS(double min_section_time_s) { min_section_time_s_ = std::abs(min_section_time_s); }
    double getMinSectionTimeS() const { return min_section_time_s_; }

   private:
    // the shortest section the roll / pitch bisection examines; a shorter one is Indeterminable
    double min_section_time_s_;
  };

  FeasibilityAnalytic() {}
  explicit FeasibilityAnalytic(const Settings& settings) : settings_(settings) {}
  explicit FeasibilityAnalytic(const InputConstraints& input_constraints) : FeasibilityBase(input_constraints) {}
  FeasibilityAnalytic(const Settings& settings, const InputConstraints& input_constraints)
      : FeasibilityBase(input_constraints), settings_(settings) {}

  InputFeasibilityResult checkInputFeasibility(const Segment& segment) const override;

  Settings settings_;

 private:
  InputFeasibilityResult thrustFeasibility(const Segment& segment, std::vector<Extremum>* thrust_candidates,
                                           Segment* thrust_segment) const;
  InputFeasibilityResult rollPitchFeasibility(const Segment& segment, const Segment& thrust_segment,
                                              const std::vector<Extremum>& thrust_candidates,
                                              const std::vector<Extremum>& jerk_candidates, double t_1,
                                              double t_2) const;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_ANALYTIC_H_
