// trajectory_sampling.h -- single-object sampling of a Trajectory / Segment into flat states (SURVEY.md 8f-3):
// sampleTrajectoryAtTime, sampleTrajectoryInRange, sampleTrajectoryStartDuration, sampleWholeTrajectory,
// sampleSegmentAtTime, sampleFlatStateAtTime (reference include/mav_trajectory_generation/trajectory_sampling.h,
// src/trajectory_sampling.cpp:27-196).  The batched device forms are mtg_sample_flat_states_batch_f64 /
// mtg_sample_flat_state_at_time_batch_f64 (BatchPolynomialOptimization::sampleTrajectoriesInRange,
// sampleWholeTrajectories, sampleTrajectoriesAtTime), which share this mirror's rotation-vector arithmetic
// (rotation_vector_kinematics.h).
//
// mav_msgs is not part of this tree, so mav_msgs::EigenTrajectoryPoint is mirrored as a plain struct with the same
// field names and meaning (mav_msgs/eigen_mav_msgs.h): world-frame position ... snap, orientation quaternion,
// world-frame angular velocity / acceleration, time from start in nanoseconds, degrees of freedom.  A maintainer
// with mav_msgs on the include path deletes the mirror namespace below and includes <mav_msgs/eigen_mav_msgs.h>.
// Same rules as the reference: at least 3 dimensions; a 4th dimension is yaw (orientation about the world z axis,
// yaw rate / acceleration in the z components); 6 dimensions carry a rotation vector in the last three, turned into
// the orientation quaternion and -- through the left Jacobian of SO(3), w = J(phi) phi', w' = J phi'' + J' phi' --
// into world-frame angular velocity / acceleration (the published formulas of mav_msgs' omegaFromRotationVector /
// omegaDotFromRotationVector; pinned here by finite differences of the rotation itself, tests/cpp).
#ifndef MAV_TRAJECTORY_GENERATION_TRAJECTORY_SAMPLING_H_
#define MAV_TRAJECTORY_GENERATION_TRAJECTORY_SAMPLING_H_

#include <cmath>
#include <cstdint>
#include <vector>

#include "mav_trajectory_generation/rotation_vector_kinematics.h"
#include "mav_trajectory_generation/trajectory.h"

namespace mav_msgs {

enum MavActuation { DOF4 = 4, DOF6 = 6 };

struct Quaternion {  // Eigen::Quaterniond's coefficients
  double w = 1.0, x = 0.0, y = 0.0, z = 0.0;
};

struct EigenTrajectoryPoint {
  typedef std::vector<EigenTrajectoryPoint> Vector;
  int64_t time_from_start_ns = 0;
  Eigen::Vector3d position_W, velocity_W, acceleration_W, jerk_W, snap_W;
  Quaternion orientation_W_B;
  Eigen::Vector3d angular_velocity_W, angular_acceleration_W;
  MavActuation degrees_of_freedom = DOF4;

  void setFromYaw(double yaw) {
    orientation_W_B.w = std::cos(0.5 * yaw);
    orientation_W_B.x = orientation_W_B.y = 0.0;
    orientation_W_B.z = std::sin(0.5 * yaw);
  }
  void setFromYawRate(double yaw_rate) {
    angular_velocity_W[0] = angular_velocity_W[1] = 0.0;
    angular_velocity_W[2] = yaw_rate;
  }
  void setFromYawAcc(double yaw_acc) {
    angular_acceleration_W[0] = angular_acceleration_W[1] = 0.0;
    angular_acceleration_W[2] = yaw_acc;
  }
  double getYaw() const {
    return std::atan2(2.0 * (orientation_W_B.w * orientation_W_B.z + orientation_W_B.x * orientation_W_B.y),
                      1.0 - 2.0 * (orientation_W_B.y * orientation_W_B.y + orientation_W_B.z * orientation_W_B.z));
  }
  double getYawRate() const { return angular_velocity_W[2]; }
  double getYawAcc() const { return angular_acceleration_W[2]; }
};
typedef std::vector<EigenTrajectoryPoint> EigenTrajectoryPointVector;

// mav_msgs::EigenMavState (mav_msgs/eigen_mav_msgs.h), mirrored as a plain struct like EigenTrajectoryPoint with the
// fields the conversion below fills: world-frame position and velocity, body-frame acceleration (the thrust direction
// scaled by its magnitude), body-frame angular velocity and acceleration.  The orientation is not mirrored.
struct EigenMavState {
  Eigen::Vector3d position_W, velocity_W, acceleration_B;
  Eigen::Vector3d angular_velocity_B, angular_acceleration_B;
};

// mav_msgs' EigenMavStateFromEigenTrajectoryPoint (mav_msgs/conversions.h), the flat-state to full-state map of
// Mellinger and Kumar (2011) restated here, not checked against mav_msgs:
//   f = a + (0, 0, g), thrust = |f|, zb = f * (1 / thrust), xc = (cos yaw, sin yaw, 0), yb = normalized(zb x xc),
//   xb = yb x zb, acceleration_B = R^T (zb thrust) with R = [xb yb zb], h = (1 / thrust) (j - (zb . j) zb),
//   angular_velocity_B = (-h . yb, h . xb, yaw_rate zb_z), angular_acceleration_B = (0, 0, yaw_acc zb_z)
// with yaw = flat_state.getYaw().  Only the z components of the angular acceleration are part of the restatement; x and
// y are left 0.  A thrust of exactly 0 gives a NaN state.
inline void EigenMavStateFromEigenTrajectoryPoint(const EigenTrajectoryPoint& flat_state, double gravity,
                                                  EigenMavState* state) {
  const double yaw = flat_state.getYaw();
  const Eigen::Vector3d xc(std::cos(yaw), std::sin(yaw), 0.0);
  Eigen::Vector3d f = flat_state.acceleration_W;
  f[2] += gravity;
  const double thrust = f.norm(), inv = 1.0 / thrust;
  const Eigen::Vector3d zb = f * inv;
  const Eigen::Vector3d yb = zb.cross(xc).normalized();
  const Eigen::Vector3d xb = yb.cross(zb);
  const Eigen::Vector3d w = zb * thrust;
  state->position_W = flat_state.position_W;
  state->velocity_W = flat_state.velocity_W;
  state->acceleration_B = Eigen::Vector3d(xb.dot(w), yb.dot(w), zb.dot(w));
  const Eigen::Vector3d h = (flat_state.jerk_W - zb * zb.dot(flat_state.jerk_W)) * inv;
  state->angular_velocity_B = Eigen::Vector3d(-h.dot(yb), h.dot(xb), flat_state.getYawRate() * zb[2]);
  state->angular_acceleration_B = Eigen::Vector3d(0.0, 0.0, flat_state.getYawAcc() * zb[2]);
}

}  // namespace mav_msgs

namespace mav_trajectory_generation {

namespace sampling_detail {
const double kNumNanosecondsPerSecond = 1.e9;

// orientation, world-frame angular velocity and acceleration of the rotation vector phi(t) with derivatives dphi, ddphi
// (rotation_vector_kinematics.h, shared with the batched flat-state kernels)
inline void rotationVectorKinematics(const V3& phi, const V3& dphi, const V3& ddphi, mav_msgs::Quaternion* q, V3* omega,
                                     V3* omega_dot) {
  double c[4];
  rotationVectorKinematics(phi, dphi, ddphi, c, omega, omega_dot);
  q->w = c[0];
  q->x = c[1];
  q->y = c[2];
  q->z = c[3];
}

inline V3 tail3(const Eigen::VectorXd& v) { return {{v[v.size() - 3], v[v.size() - 2], v[v.size() - 1]}}; }
inline void head3(const Eigen::VectorXd& v, Eigen::Vector3d* out) {
  for (int i = 0; i < 3; ++i) (*out)[i] = v[i];
}
inline void store(const V3& a, Eigen::Vector3d* out) {
  for (int i = 0; i < 3; ++i) (*out)[i] = a.v[i];
}

// attitude part shared by the single-time and the range samplers (reference trajectory_sampling.cpp:87-105, 170-188)
inline void fillAttitude(int D, const Eigen::VectorXd& position, const Eigen::VectorXd& velocity,
                         const Eigen::VectorXd& acceleration, mav_msgs::EigenTrajectoryPoint* state) {
  state->degrees_of_freedom = mav_msgs::DOF4;
  if (D == 4) {
    state->setFromYaw(position[3]);
    state->setFromYawRate(velocity[3]);
    state->setFromYawAcc(acceleration[3]);
  } else if (D == 6) {
    V3 omega, omega_dot;
    rotationVectorKinematics(tail3(position), tail3(velocity), tail3(acceleration), &state->orientation_W_B, &omega,
                             &omega_dot);
    store(omega, &state->angular_velocity_W);
    store(omega_dot, &state->angular_acceleration_W);
    state->degrees_of_freedom = mav_msgs::DOF6;
  }
}
}  // namespace sampling_detail

// reference trajectory_sampling.cpp:151-196
template <class T>
bool sampleFlatStateAtTime(const T& type, double sample_time, mav_msgs::EigenTrajectoryPoint* state) {
  CHECK_NOTNULL(state);
  if (type.D() < 3) {
    LOG(ERROR) << "Dimension has to be 3, 4, or 6 but is " << type.D();
    return false;
  }
  const Eigen::VectorXd position = type.evaluate(sample_time, derivative_order::POSITION);
  const Eigen::VectorXd velocity = type.evaluate(sample_time, derivative_order::VELOCITY);
  const Eigen::VectorXd acceleration = type.evaluate(sample_time, derivative_order::ACCELERATION);
  sampling_detail::head3(position, &state->position_W);
  sampling_detail::head3(velocity, &state->velocity_W);
  sampling_detail::head3(acceleration, &state->acceleration_W);
  sampling_detail::head3(type.evaluate(sample_time, derivative_order::JERK), &state->jerk_W);
  sampling_detail::head3(type.evaluate(sample_time, derivative_order::SNAP), &state->snap_W);
  sampling_detail::fillAttitude(type.D(), position, velocity, acceleration, state);
  state->time_from_start_ns = static_cast<int64_t>(sample_time * sampling_detail::kNumNanosecondsPerSecond);
  return true;
}

// reference trajectory_sampling.cpp:27-43
inline bool sampleTrajectoryAtTime(const Trajectory& trajectory, double sample_time,
                                   mav_msgs::EigenTrajectoryPoint* state) {
  CHECK_NOTNULL(state);
  if (sample_time < trajectory.getMinTime() || sample_time > trajectory.getMaxTime()) {
    LOG(ERROR) << "Sample time should be within [" << trajectory.getMinTime() << " " << trajectory.getMaxTime()
               << "] but is " << sample_time;
    return false;
  }
  if (trajectory.D() < 3) {
    LOG(ERROR) << "Dimension has to be at least 3, but is " << trajectory.D();
    return false;
  }
  return sampleFlatStateAtTime<Trajectory>(trajectory, sample_time, state);
}

// reference trajectory_sampling.cpp:45-110: five evaluateRange walks (position .. snap), one state per sample,
// time stamps min_time + i * sampling_interval
inline bool sampleTrajectoryInRange(const Trajectory& trajectory, double min_time, double max_time,
                                    double sampling_interval, mav_msgs::EigenTrajectoryPointVector* states) {
  CHECK_NOTNULL(states);
  if (min_time < trajectory.getMinTime() || max_time > trajectory.getMaxTime()) {
    LOG(ERROR) << "Sample time should be within [" << trajectory.getMinTime() << " " << trajectory.getMaxTime()
               << "] but is [" << min_time << " " << max_time << "]";
    return false;
  }
  if (trajectory.D() < 3) {
    LOG(ERROR) << "Dimension has to be at least 3, but is " << trajectory.D();
    return false;
  }
  std::vector<Eigen::VectorXd> sampled[5];
  for (int derivative = 0; derivative < 5; ++derivative)
    trajectory.evaluateRange(min_time, max_time, sampling_interval, derivative, &sampled[derivative]);
  const size_t n_samples = sampled[0].size();
  states->assign(n_samples, mav_msgs::EigenTrajectoryPoint());
  for (size_t i = 0; i < n_samples; ++i) {
    mav_msgs::EigenTrajectoryPoint& state = (*states)[i];
    sampling_detail::head3(sampled[0][i], &state.position_W);
    sampling_detail::head3(sampled[1][i], &state.velocity_W);
    sampling_detail::head3(sampled[2][i], &state.acceleration_W);
    sampling_detail::head3(sampled[3][i], &state.jerk_W);
    sampling_detail::head3(sampled[4][i], &state.snap_W);
    state.time_from_start_ns =
        static_cast<int64_t>((min_time + sampling_interval * i) * sampling_detail::kNumNanosecondsPerSecond);
    sampling_detail::fillAttitude(trajectory.D(), sampled[0][i], sampled[1][i], sampled[2][i], &state);
  }
  return true;
}

inline bool sampleTrajectoryStartDuration(const Trajectory& trajectory, double start_time, double duration,
                                          double sampling_interval, mav_msgs::EigenTrajectoryPointVector* states) {
  return sampleTrajectoryInRange(trajectory, start_time, start_time + duration, sampling_interval, states);
}

inline bool sampleWholeTrajectory(const Trajectory& trajectory, double sampling_interval,
                                  mav_msgs::EigenTrajectoryPoint::Vector* states) {
  return sampleTrajectoryInRange(trajectory, trajectory.getMinTime(), trajectory.getMaxTime(), sampling_interval, states);
}

// reference trajectory_sampling.cpp:137-149
inline bool sampleSegmentAtTime(const Segment& segment, double sample_time, mav_msgs::EigenTrajectoryPoint* state) {
  CHECK_NOTNULL(state);
  if (sample_time < 0.0 || sample_time > segment.getTime()) {
    LOG(ERROR) << "Sample time should be within [" << 0.0 << " " << segment.getTime() << "] but is " << sample_time;
    return false;
  }
  return sampleFlatStateAtTime<Segment>(segment, sample_time, state);
}

}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_TRAJECTORY_SAMPLING_H_
