// mtg_half_plane_kernel.cuh -- FeasibilityBase::checkHalfPlaneFeasibility for one segment and for a trajectory
// (reference mav_trajectory_generation_ros/src/feasibility_base.cpp:109-154) for B trajectories and one set of planes.
//
// A segment stays inside the half-space of plane (q, n) when d(t) = (p(t) - q) . n > 0 at every candidate: 0, T and
// the real roots in [0, T] of the projection's derivative, where the projection n . p(t) has the coefficients
// c_j = ((x_j n_0) + y_j n_1) + z_j n_2.  The first segment with a failing plane decides, and within it the first
// plane.  Every value uses the reference's arithmetic (range_horner per dimension, then the subtraction and the dot
// product in dimension order with explicit round-to-nearest operations), so the value at 0 and at T is bit-identical
// to an x86 build; a NaN compares false and passes.
//
// Per (segment, plane), cheapest first:
//   1. d(0) or d(T) <= 0: the plane fails (both are candidates of every plane).
//   2. The Bernstein coefficients of d(tau T) on [0, 1] (extrema_bernstein) bound d from below.  If their minimum
//      exceeds E = (8N + 16) u S + DBL_MIN (1 + T^(N-1)) (1 + |n|_1), with S = sum_d |n_d| (sum_j |c_dj| T^j + |q_d|),
//      no computed value at any t in [0, T] can be <= 0, so the plane passes without root finding (DESIGN.md §3b).
//   3. Otherwise the interior candidates come from the root isolation of mtg_extrema_kernel.cuh on the derivative of
//      d(tau T); every candidate it visits, safety samples included, is a genuine point of the segment.
// Each step gives exactly the outcome of walking all the candidates.
#pragma once

#include <cfloat>

#include "mtg_feasibility_kernel.cuh"

namespace mtg {

constexpr int kHalfPlaneMax = 64;  // MTG_MAX_HALF_PLANES

struct HalfPlaneParams {
  int K, D, n_planes;
  long long B;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ coeffs;  // [B][K][D][N]
  int* __restrict__ feasible;         // [B]
  int* __restrict__ segment;          // [B] or null
  int* __restrict__ plane;            // [B] or null
  int* __restrict__ status;           // [B] or null
  double planes[kHalfPlaneMax][6];    // point[3], normal[3], as given (3 KB of kernel parameters)
};

// (p(t) - q) . n: Segment::evaluate per dimension, the subtraction, then Eigen's dot in dimension order
template <int N>
__device__ __forceinline__ double half_plane_distance(const double* __restrict__ c, const double* pl, double t) {
  double s = 0.0;
#pragma unroll 1
  for (int d = 0; d < 3; ++d) {
    double cd[N];
#pragma unroll
    for (int j = 0; j < N; ++j) cd[j] = c[d * N + j];
    const double m = __dmul_rn(__dsub_rn(range_horner<N, 0>(cd, t), pl[d]), pl[3 + d]);
    s = d == 0 ? m : __dadd_rn(s, m);
  }
  return s;
}

// The planes of one segment (time T > 0 and finite), in order: 0 when every plane passes, 1 when D is not 3 or 4
// (the reference refuses such a segment before looking at any plane), else 2 + the first failing plane.
template <int N>
__device__ int half_plane_segment(const double* __restrict__ c, double T, const HalfPlaneParams& prm) {
  if (prm.D != 3 && prm.D != 4) return 1;
  constexpr double u = 1.1102230246251565e-16;  // 2^-53
#pragma unroll 1
  for (int p = 0; p < prm.n_planes; ++p) {
    const double* pl = prm.planes[p];
    const double d0 = half_plane_distance<N>(c, pl, 0.0);
    if (d0 <= 0.0 || half_plane_distance<N>(c, pl, T) <= 0.0) return 2 + p;
    // d(tau T) in the power basis (a_0 = the computed d(0)) and the error scale S
    const double n0 = pl[3], n1 = pl[4], n2 = pl[5];
    double a[N];
    a[0] = d0;
    double S = fabs(n0 * pl[0]) + fabs(n1 * pl[1]) + fabs(n2 * pl[2]);
    double tp = 1.0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const double x = c[j], y = c[N + j], z = c[2 * N + j];
      S += (fabs(n0 * x) + fabs(n1 * y) + fabs(n2 * z)) * tp;
      if (j > 0) a[j] = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, n0), __dmul_rn(y, n1)), __dmul_rn(z, n2)), tp);
      if (j < N - 1) tp *= T;
    }
    const double E = (8.0 * N + 16.0) * u * S + DBL_MIN * (1.0 + tp) * (1.0 + fabs(n0) + fabs(n1) + fabs(n2));
    double b[N];
    extrema_bernstein(a, 0.0, 1.0, b);
    bool clear = true;  // a NaN coefficient or bound does not take the shortcut
#pragma unroll
    for (int j = 0; j < N; ++j) clear = clear && b[j] > E;
    if (clear) continue;
    // the interior candidates: roots of d'(tau T) (a positive multiple of the projection's derivative)
    double g[N - 1];
#pragma unroll
    for (int j = 0; j < N - 1; ++j) g[j] = double(j + 1) * a[j + 1];
    bool fail = false;
    extrema_candidates(g, [&](double tau, bool) {
      if (!fail && half_plane_distance<N>(c, pl, tau * T) <= 0.0) fail = true;
    });
    if (fail) return 2 + p;
  }
  return 0;
}

// One thread per (trajectory, segment) runs half_plane_segment; the first failing segment decides.
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) half_plane_kernel(const __grid_constant__ HalfPlaneParams prm,
                                                                        const int tpb) {
  first_failing_segment(
      prm.B, prm.K, prm.times, tpb,
      [&](long long item, double T) { return half_plane_segment<N>(prm.coeffs + item * prm.D * N, T, prm); },
      [&](long long traj, bool bad, int seg, int code) {
        prm.feasible[traj] = !bad && seg < 0 ? 1 : 0;
        if (prm.segment) prm.segment[traj] = seg;
        if (prm.plane) prm.plane[traj] = seg < 0 ? -1 : code - 2;
        if (prm.status) prm.status[traj] = bad ? 1 : 0;  // MTG_STATUS_BAD_TIME
      });
}

}  // namespace mtg
