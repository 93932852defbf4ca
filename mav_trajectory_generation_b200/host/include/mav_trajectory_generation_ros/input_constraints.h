// input_constraints.h -- the dynamic limits of a multicopter that FeasibilityAnalytic checks (reference
// mav_trajectory_generation_ros/include/mav_trajectory_generation_ros/input_constraints.h and src/input_constraints.cpp:
// addConstraint, setDefaultValues, getConstraint, hasConstraint, removeConstraint).  The YAML conversion is not
// mirrored.
#ifndef MAV_TRAJECTORY_GENERATION_ROS_INPUT_CONSTRAINTS_H_
#define MAV_TRAJECTORY_GENERATION_ROS_INPUT_CONSTRAINTS_H_

#include <map>
#include <string>

namespace mav_trajectory_generation {

// Gravity [m/s^2] of the defaults and of FeasibilityBase.  The reference uses mav_msgs::kGravity; mav_comm is not part
// of this project, so this value has not been checked against it.
constexpr double kGravity = 9.81;

enum InputConstraintType {
  kFMin = 0,     // minimum normalized thrust [m/s^2]
  kFMax,         // maximum normalized thrust [m/s^2]
  kVMax,         // maximum speed [m/s]
  kOmegaXYMax,   // maximum roll / pitch rate [rad/s]
  kOmegaZMax,    // maximum yaw rate [rad/s]
  kOmegaZDotMax  // maximum yaw acceleration [rad/s^2]
};

std::string getInputConstraintName(InputConstraintType type);

class InputConstraints {
 public:
  InputConstraints() {}

  // Stores |value|.  Adding f_min above a present f_max raises f_max to it; adding f_max below a present f_min lowers
  // f_min to it.
  void addConstraint(int constraint_type, double value);
  // f_min = 0.5 g, f_max = 1.5 g, v_max = 3 m/s, omega_xy = omega_z = pi / 2 rad/s, omega_z_dot = 2 pi rad/s^2.
  void setDefaultValues();
  // false (value untouched) when the constraint is absent
  bool getConstraint(int constraint_type, double* value) const;
  bool hasConstraint(int constraint_type) const;
  // false when the constraint was absent
  bool removeConstraint(int constraint_type);

 private:
  std::map<int, double> constraints_;
};

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROS_INPUT_CONSTRAINTS_H_
