// feasibility_sampling.h -- sampling-based input feasibility of one segment (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/feasibility_sampling.h,
// src/feasibility_sampling.cpp): the flat state is sampled every sampling interval from t = 0 while t <= T (a running
// sum), turned into the full state with mav_msgs::EigenMavStateFromEigenTrajectoryPoint, and checked for thrust,
// speed, roll / pitch rate, yaw rate and yaw acceleration.  This single-object path runs on the host; batches of
// trajectories go through BatchPolynomialOptimization<N>::checkInputFeasibilitySampling on the GPU.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_SAMPLING_H_
#define MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_SAMPLING_H_

#include <cmath>

#include "mav_trajectory_generation/segment.h"
#include "mav_trajectory_generation_ros/feasibility_base.h"

namespace mav_trajectory_generation {

class FeasibilitySampling : public FeasibilityBase {
 public:
  class Settings {
   public:
    Settings() : sampling_interval_s_(0.01) {}
    void setSamplingIntervalS(double sampling_interval_s) { sampling_interval_s_ = std::abs(sampling_interval_s); }
    double getSamplingIntervalS() const { return sampling_interval_s_; }

   private:
    double sampling_interval_s_;
  };

  FeasibilitySampling() {}
  explicit FeasibilitySampling(const Settings& settings) : settings_(settings) {}
  explicit FeasibilitySampling(const InputConstraints& input_constraints) : FeasibilityBase(input_constraints) {}
  FeasibilitySampling(const Settings& settings, const InputConstraints& input_constraints)
      : FeasibilityBase(input_constraints), settings_(settings) {}

  // As the reference, a sampling interval of 0 never ends; the batched GPU form refuses it and caps a segment at
  // 2^24 samples.
  InputFeasibilityResult checkInputFeasibility(const Segment& segment) const override;

  Settings settings_;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_FEASIBILITY_SAMPLING_H_
