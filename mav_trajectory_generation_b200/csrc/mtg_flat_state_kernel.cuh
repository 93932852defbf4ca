// mtg_flat_state_kernel.cuh -- batched flat-state sampling: sampleTrajectoryInRange / sampleWholeTrajectory and
// sampleTrajectoryAtTime (reference src/trajectory_sampling.cpp:27-110) for B trajectories at once.
//
// A flat state is one fixed record of MTG_FLAT_STATE_DOUBLES doubles (include/mtg_b200.h): position ... snap of
// dimensions 0..2, the orientation quaternion (w, x, y, z), world-frame angular velocity and angular acceleration.
// Position ... snap are Polynomial::evaluate's arithmetic (range_horner: separate multiply and add), so they are bit
// for bit the values of mtg_evaluate_range_batch_f64 / mtg_evaluate_batch_f64.  The attitude follows D
// (trajectory_sampling.cpp:87-107): ATT = kAttYaw (D = 4) is setFromYaw / setFromYawRate / setFromYawAcc of dimension
// 3; ATT = kAttRotationVector (D = 6) is rotationVectorKinematics of dimensions 3..5 (rotation_vector_kinematics.h,
// the host mirror's own code); any other D >= 3 (kAttNone) gives the identity and zero angular terms.
//
// The range sampler runs after range_walk_kernel (mtg_generic_kernel.cuh), whose one walk gives the segment and local
// time of every sample for all five derivative orders, as the reference's five evaluateRange walks are identical.
// Both kernels run one thread per record and write through a shared-memory tile of blockDim.x records, so a block's
// states leave as one contiguous, coalesced span (a 200-byte record stored per thread touches 7 sectors per lane).
#pragma once

#include "../host/include/mav_trajectory_generation/rotation_vector_kinematics.h"
#include "../../include/mtg_b200.h"
#include "mtg_generic_kernel.cuh"

namespace mtg {

enum FlatAttitude { kAttNone = 0, kAttYaw = 1, kAttRotationVector = 2 };

constexpr int kFlatStateThreads = 128;  // tile: 128 * 25 * 8 = 25 600 bytes of shared memory per block

// The record of the flat state at local time t of the segment whose [D][N] coefficients start at cg.
template <int N, int ATT>
__device__ __forceinline__ void flat_state_record(const double* __restrict__ cg, int D, double t,
                                                  double* __restrict__ o) {
  for (int d = 0; d < 3; ++d) {
    double c[N];
#pragma unroll
    for (int j = 0; j < N; ++j) c[j] = cg[d * N + j];
    o[MTG_FLAT_STATE_POSITION + d] = range_horner<N, 0>(c, t);
    o[MTG_FLAT_STATE_VELOCITY + d] = range_horner<N, 1>(c, t);
    o[MTG_FLAT_STATE_ACCELERATION + d] = range_horner<N, 2>(c, t);
    o[MTG_FLAT_STATE_JERK + d] = range_horner<N, 3>(c, t);
    o[MTG_FLAT_STATE_SNAP + d] = range_horner<N, 4>(c, t);
  }
  double* q = o + MTG_FLAT_STATE_ORIENTATION;
  double* w = o + MTG_FLAT_STATE_ANGULAR_VELOCITY;
  double* wd = o + MTG_FLAT_STATE_ANGULAR_ACCELERATION;
  if constexpr (ATT == kAttNone) {
    q[0] = 1.0;
    q[1] = q[2] = q[3] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = wd[k] = 0.0;
  } else if constexpr (ATT == kAttYaw) {
    double c[N];
#pragma unroll
    for (int j = 0; j < N; ++j) c[j] = cg[3 * N + j];
    const double yaw = range_horner<N, 0>(c, t);
    q[0] = cos(0.5 * yaw);
    q[1] = q[2] = 0.0;
    q[3] = sin(0.5 * yaw);
    w[0] = w[1] = 0.0;
    w[2] = range_horner<N, 1>(c, t);
    wd[0] = wd[1] = 0.0;
    wd[2] = range_horner<N, 2>(c, t);
  } else {
    using mav_trajectory_generation::sampling_detail::V3;
    V3 phi, dphi, ddphi;
    for (int k = 0; k < 3; ++k) {
      double c[N];
#pragma unroll
      for (int j = 0; j < N; ++j) c[j] = cg[(3 + k) * N + j];
      phi.v[k] = range_horner<N, 0>(c, t);
      dphi.v[k] = range_horner<N, 1>(c, t);
      ddphi.v[k] = range_horner<N, 2>(c, t);
    }
    V3 omega, omega_dot;
    mav_trajectory_generation::sampling_detail::rotationVectorKinematics(phi, dphi, ddphi, q, &omega, &omega_dot);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      w[k] = omega.v[k];
      wd[k] = omega_dot.v[k];
    }
  }
}

// Copies `n` records of the tile to `dst` with consecutive threads on consecutive doubles.
__device__ __forceinline__ void flat_state_store_tile(const double* __restrict__ tile, double* __restrict__ dst,
                                                      int n) {
  const int n_out = n * MTG_FLAT_STATE_DOUBLES;
  for (int k = threadIdx.x; k < n_out; k += blockDim.x) dst[k] = tile[k];
}

// sampleTrajectoryInRange: one thread per (trajectory, sample) of the flattened [B][max_samples] index.  The walk
// left n_samples, seg_idx and t_local; samples at or past n_samples[b] (all of a -1 row) are zero records with a zero
// time stamp.  time_ns[s] = (int64)((t_start + dt * s) * 1e9), every operation rounded on its own and truncated toward
// zero, as the reference's static_cast<int64_t>((min_time + sampling_interval * i) * kNumNanosecondsPerSecond).
template <int N, int ATT>
__global__ void __launch_bounds__(kFlatStateThreads) flat_state_range_kernel(const RangeParams prm) {
  __shared__ double tile[kFlatStateThreads * MTG_FLAT_STATE_DOUBLES];
  const int K = prm.K, D = prm.D, S = prm.max_samples;
  const long long total = prm.B * S;
  const double t0 = prm.range_rule == kRangeWhole ? 0.0 : prm.t_start;
  const long long n_tiles = (total + kFlatStateThreads - 1) / kFlatStateThreads;
  for (long long ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const long long idx0 = ti * kFlatStateThreads;
    const long long idx = idx0 + threadIdx.x;
    if (idx < total) {
      const long long b = idx / S;
      const int s = int(idx - b * S);
      double* __restrict__ o = tile + threadIdx.x * MTG_FLAT_STATE_DOUBLES;
      long long ns = 0;
      if (s >= prm.n_samples[b]) {
        for (int q = 0; q < MTG_FLAT_STATE_DOUBLES; ++q) o[q] = 0.0;
      } else {
        const int i = prm.seg_idx[idx];
        flat_state_record<N, ATT>(prm.coeffs + (b * K + i) * D * N, D, prm.t_local[idx], o);
        ns = __double2ll_rz(__dmul_rn(__dadd_rn(t0, __dmul_rn(prm.dt, double(s))), 1e9));
      }
      if (prm.time_ns) prm.time_ns[idx] = ns;
    }
    __syncthreads();
    const long long left = total - idx0;
    flat_state_store_tile(tile, prm.out + idx0 * MTG_FLAT_STATE_DOUBLES,
                          int(left < kFlatStateThreads ? left : kFlatStateThreads));
    __syncthreads();
  }
}

struct FlatAtTimeParams {
  int K, D;
  long long B;
  const double* __restrict__ times;         // [B][K]
  const double* __restrict__ coeffs;        // [B][K][D][N]
  const double* __restrict__ sample_times;  // [B]
  double* __restrict__ states;              // [B][MTG_FLAT_STATE_DOUBLES]
  long long* __restrict__ time_ns;          // [B] or null
  int* __restrict__ ok;                     // [B]
};

// sampleTrajectoryAtTime: one thread per trajectory.  A row is sampled when 0 <= t <= its total time (the left-to-right
// sum of its segment times) and D >= 3; otherwise ok = 0 with a zero record and time stamp.  The segment follows
// Trajectory::evaluate (as evaluate_kernel does): a time on a vertex belongs to the segment on its right, and t equal
// to the total time is the end of the last segment.  time_ns = (int64)(t * 1e9).
template <int N, int ATT>
__global__ void __launch_bounds__(kFlatStateThreads) flat_state_at_time_kernel(const FlatAtTimeParams prm) {
  __shared__ double tile[kFlatStateThreads * MTG_FLAT_STATE_DOUBLES];
  const int K = prm.K, D = prm.D;
  const long long n_tiles = (prm.B + kFlatStateThreads - 1) / kFlatStateThreads;
  for (long long ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const long long b0 = ti * kFlatStateThreads;
    const long long b = b0 + threadIdx.x;
    if (b < prm.B) {
      const double* __restrict__ tt = prm.times + b * K;
      const double t = prm.sample_times[b];
      double total = 0.0;
      for (int k = 0; k < K; ++k) total = __dadd_rn(total, tt[k]);
      double* __restrict__ o = tile + threadIdx.x * MTG_FLAT_STATE_DOUBLES;
      const bool ok = D >= 3 && t >= 0.0 && t <= total;
      long long ns = 0;
      if (!ok) {
        for (int q = 0; q < MTG_FLAT_STATE_DOUBLES; ++q) o[q] = 0.0;
      } else {
        double start = 0.0;
        int i = 0;
        for (; i < K; ++i) {
          const double Ti = tt[i];
          if (__dadd_rn(start, Ti) > t) break;
          start = __dadd_rn(start, Ti);
        }
        if (i == K) {
          i = K - 1;
          start = __dsub_rn(start, tt[i]);
        }
        flat_state_record<N, ATT>(prm.coeffs + (b * K + i) * D * N, D, __dsub_rn(t, start), o);
        ns = __double2ll_rz(__dmul_rn(t, 1e9));
      }
      prm.ok[b] = ok;
      if (prm.time_ns) prm.time_ns[b] = ns;
    }
    __syncthreads();
    const long long left = prm.B - b0;
    flat_state_store_tile(tile, prm.states + b0 * MTG_FLAT_STATE_DOUBLES,
                          int(left < kFlatStateThreads ? left : kFlatStateThreads));
    __syncthreads();
  }
}

}  // namespace mtg
