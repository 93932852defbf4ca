// rotation_vector_kinematics.h -- orientation, world-frame angular velocity and angular acceleration of a rotation
// vector phi(t) and its derivatives: the arithmetic behind the 6-D flat state of sampleTrajectoryInRange /
// sampleFlatStateAtTime (reference src/trajectory_sampling.cpp:93-106).  Written once for both sides: the host mirror
// (trajectory_sampling.h) and the batched flat-state kernels (csrc/mtg_flat_state_kernel.cuh) include this header, so
// the formula and its branch points (the 1e-4 series switch, the 1e-12 identity cut-off, the w >= 0 sign) cannot drift
// apart.  Plain C++ without Eigen or the standard library's containers, so that nvcc compiles it for the device.
#ifndef MAV_TRAJECTORY_GENERATION_ROTATION_VECTOR_KINEMATICS_H_
#define MAV_TRAJECTORY_GENERATION_ROTATION_VECTOR_KINEMATICS_H_

#include <math.h>

#ifdef __CUDACC__
#define MTG_HOST_DEVICE __host__ __device__ __forceinline__
#else
#define MTG_HOST_DEVICE inline
#endif

namespace mav_trajectory_generation {
namespace sampling_detail {

struct V3 {
  double v[3];
};
MTG_HOST_DEVICE V3 cross(const V3& a, const V3& b) {
  return {{a.v[1] * b.v[2] - a.v[2] * b.v[1], a.v[2] * b.v[0] - a.v[0] * b.v[2], a.v[0] * b.v[1] - a.v[1] * b.v[0]}};
}
MTG_HOST_DEVICE double dot(const V3& a, const V3& b) { return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2]; }
MTG_HOST_DEVICE V3 axpy(double s, const V3& a, const V3& b) {
  return {{s * a.v[0] + b.v[0], s * a.v[1] + b.v[1], s * a.v[2] + b.v[2]}};
}

// coefficients a = (1 - cos t)/t^2, b = (t - sin t)/t^3 of J = I + a [phi]x + b [phi]x^2 and their derivatives in t
MTG_HOST_DEVICE void jacobianCoefficients(double t, double* a, double* b, double* da, double* db) {
  if (t < 1e-4) {  // series: the closed forms cancel catastrophically near 0
    const double t2 = t * t;
    *a = 0.5 - t2 / 24.0;
    *b = 1.0 / 6.0 - t2 / 120.0;
    *da = -t / 12.0;
    *db = -t / 60.0;
    return;
  }
  const double s = sin(t), c = cos(t);
  *a = (1.0 - c) / (t * t);
  *b = (t - s) / (t * t * t);
  *da = (t * s - 2.0 * (1.0 - c)) / (t * t * t);
  *db = ((1.0 - c) * t - 3.0 * (t - s)) / (t * t * t * t);
}

// J x = x + a phi x x + b phi x (phi x x)
MTG_HOST_DEVICE V3 applyLeftJacobian(const V3& phi, double a, double b, const V3& x) {
  const V3 px = cross(phi, x);
  return axpy(b, cross(phi, px), axpy(a, px, x));
}

// Orientation q = (w, x, y, z), world-frame angular velocity and acceleration of the rotation vector phi(t) with
// derivatives dphi, ddphi: w = J(phi) phi', w' = J phi'' + J' phi' (J the left Jacobian of SO(3)).  q has w >= 0, as
// the matrix -> quaternion conversion the reference goes through returns for rotation angles up to 2 pi / 3; past
// that, Eigen's conversion may return the same rotation with the opposite sign.
MTG_HOST_DEVICE void rotationVectorKinematics(const V3& phi, const V3& dphi, const V3& ddphi, double q[4], V3* omega,
                                              V3* omega_dot) {
  const double t = sqrt(dot(phi, phi));
  if (t < 1e-12) {
    q[0] = 1.0;
    q[1] = q[2] = q[3] = 0.0;
  } else {
    const double s = sin(0.5 * t) / t;
    q[0] = cos(0.5 * t);
    q[1] = s * phi.v[0];
    q[2] = s * phi.v[1];
    q[3] = s * phi.v[2];
    if (q[0] < 0.0) {
      for (int k = 0; k < 4; ++k) q[k] = -q[k];
    }
  }
  double a, b, da, db;
  jacobianCoefficients(t, &a, &b, &da, &db);
  *omega = applyLeftJacobian(phi, a, b, dphi);
  // J' dphi with t' = phi . dphi / t:  a' phi x dphi + b' phi x (phi x dphi) + b (dphi x (phi x dphi))   (dphi x dphi = 0)
  const double tdot = t > 1e-12 ? dot(phi, dphi) / t : 0.0;
  const V3 pd = cross(phi, dphi);
  V3 jd = {{0.0, 0.0, 0.0}};
  jd = axpy(da * tdot, pd, jd);
  jd = axpy(db * tdot, cross(phi, pd), jd);
  jd = axpy(b, cross(dphi, pd), jd);
  const V3 jdd = applyLeftJacobian(phi, a, b, ddphi);
  *omega_dot = axpy(1.0, jdd, jd);
}

}  // namespace sampling_detail
}  // namespace mav_trajectory_generation

#endif  // MAV_TRAJECTORY_GENERATION_ROTATION_VECTOR_KINEMATICS_H_
