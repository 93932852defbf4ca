// mtg_feasibility_kernel.cuh -- FeasibilityAnalytic::checkInputFeasibility (reference
// mav_trajectory_generation_ros/src/feasibility_analytic.cpp:42-233) and checkInputFeasibilityTrajectory
// (feasibility_base.cpp:97-107) for B trajectories: thrust within [f_min, f_max], speed, yaw rate and yaw acceleration,
// and Mueller's recursive roll/pitch-rate bound, per segment in the reference's order.
//
// Every extremum comes from the root isolation of mtg_extrema_kernel.cuh (extrema_critical / extrema_candidates):
//   thrust   f = p'' + (0, 0, g) over dims 0..2: |f| at 0, T and the roots of sum_d f_d f_d'
//   velocity |p'| over dims 0..2 (never dim 3)
//   yaw      |yaw'| at 0, T and the roots of yaw'' (rate); |yaw''| at 0, T and the roots of yaw''' (acceleration)
//   jerk     |p'''| over dims 0..2
// The whole-segment extrema (thrust limits, velocity, yaw) also take the isolator's safety samples: they are genuine
// values, so they never move a maximum above or a minimum below the exact one.  The roll/pitch walk selects from the
// thrust and jerk candidates inside each sub-interval, where an extra sample would change the decision, so its two
// lists hold only 0, T, the refined roots and the midpoints of intervals unresolved at the depth cap.
//
// Candidate values use the reference's arithmetic (separate multiply and add, x86 order): the thrust polynomial is
// getCoefficients(ACCELERATION) with gravity added to the z constant term, then Horner; magnitudes sum the squares in
// dimension order and take one sqrt.  Only the root times differ from the reference (exact real roots here, Jenkins-
// Traub there).  The recursion over [t1, t2] is replayed without a stack: the current node is a level and a path of
// left/right bits, and its bounds are recomputed from [0, T] with the reference's (t1 + t2) / 2.
#pragma once

#include <cfloat>

#include "mtg_extrema_kernel.cuh"

namespace mtg {

// InputFeasibilityResult (feasibility_base.h)
enum FeasResult : int {
  kFeasFeasible = 0,
  kFeasIndeterminable = 1,
  kFeasThrustHigh = 2,
  kFeasThrustLow = 3,
  kFeasVelocity = 4,
  kFeasRollPitchRates = 5,  // unreachable in the analytic check
  kFeasYawRates = 6,
  kFeasYawAcc = 7,
};

// bits of FeasParams::present (InputConstraintType order)
constexpr unsigned kFeasFMin = 1u, kFeasFMax = 2u, kFeasVMax = 4u, kFeasOmegaXY = 8u, kFeasOmegaZ = 16u,
                   kFeasOmegaZDot = 32u;

constexpr int kFeasMaxCandidates = 48;  // per list: 0, T, <= 2N - 7 roots, unresolved midpoints
constexpr int kFeasMaxLevel = 64;       // roll/pitch walk depth (a node's path is one 64-bit word)
constexpr int kFeasCapacity = 0x100;    // or-ed into a segment's code when a list or the walk ran out of room

struct FeasParams {
  int K, D;
  unsigned present;
  double f_min, f_max, v_max, omega_xy, omega_z, omega_z_dot;
  double gravity, min_section_time;
  long long B;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ coeffs;  // [B][K][D][N]
  int* __restrict__ result;           // [B]
  int* __restrict__ segment;          // [B] or null
  int* __restrict__ status;           // [B] or null
};

// |p'' + (0, 0, g)| at t over dims 0..2, as Polynomial::evaluate of the thrust segment (coefficients
// B(2, j + 2) c[j + 2], gravity on the z constant term)
template <int N>  // N >= 4
__device__ __forceinline__ double feas_thrust(const double* __restrict__ c, double g, double t) {
  double sq = 0.0;
#pragma unroll 1
  for (int d = 0; d < 3; ++d) {
    double cd[N];
#pragma unroll
    for (int j = 0; j < N; ++j) cd[j] = c[d * N + j];
    double acc = __dmul_rn(range_base_coeff<2>(N - 1), cd[N - 1]);
#pragma unroll
    for (int j = N - 2; j >= 2; --j) {
      double f = __dmul_rn(range_base_coeff<2>(j), cd[j]);
      if (j == 2 && d == 2) f = __dadd_rn(f, g);
      acc = __dadd_rn(__dmul_rn(acc, t), f);
    }
    sq = __dadd_rn(sq, __dmul_rn(acc, acc));
  }
  return sqrt(sq);
}

// The check of one segment (time T > 0 and finite): a FeasResult, or-ed with kFeasCapacity when a candidate list or
// the roll/pitch walk ran out of room (the segment is then reported Indeterminable).
template <int N>
__device__ int feas_segment(const double* __restrict__ c, double T, const FeasParams& prm) {
  constexpr int M = 2 * N - 2;
  if (prm.D != 3 && prm.D != 4) return kFeasIndeterminable;
  const unsigned pr = prm.present;
  double th_t[kFeasMaxCandidates], th_v[kFeasMaxCandidates];  // thrust candidates (roll/pitch walk)
  double jk_t[kFeasMaxCandidates], jk_v[kFeasMaxCandidates];  // jerk candidates
  int n_th = 0, n_jk = 0;
  bool full = false;
  // passes: 0 thrust, 1 velocity, 2 yaw rate, 3 yaw acceleration, 4 jerk -- one inlined copy of the root isolation
#pragma unroll 1
  for (int pass = 0; pass < 5; ++pass) {
    if (pass == 0 && !(pr & (kFeasFMin | kFeasFMax | kFeasOmegaXY))) continue;
    if (pass == 1 && !(pr & kFeasVMax)) continue;
    if (pass == 2 && !(prm.D == 4 && (pr & kFeasOmegaZ))) continue;
    if (pass == 3 && !(prm.D == 4 && (pr & kFeasOmegaZDot))) continue;
    if (pass == 4 && !(pr & kFeasOmegaXY)) continue;
    const bool yaw = pass == 2 || pass == 3;
    const double* __restrict__ cp = yaw ? c + 3 * N : c;
    const int k = pass == 0 ? 2 : pass == 1 ? 1 : pass == 2 ? 1 : pass == 3 ? 2 : 3;
    double g[M];
    extrema_critical<N>(cp, T, yaw ? 1 : 3, k, pass == 0 ? prm.gravity : 0.0, g);
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    double lo = inf, hi = -inf;
    auto take = [&](double t, bool root) {
      double v;
      if (pass == 0) {
        v = feas_thrust<N>(c, prm.gravity, t);
      } else if (yaw) {
        double cy[N];
#pragma unroll
        for (int j = 0; j < N; ++j) cy[j] = cp[j];
        v = fabs(range_horner_any<N>(cy, t, k));
      } else {
        v = extrema_magnitude<N>(c, 3, k, t);
      }
      if (v < lo) lo = v;
      if (hi < v) hi = v;
      if (root && pass == 0) {
        if (n_th < kFeasMaxCandidates) {
          th_t[n_th] = t;
          th_v[n_th++] = v;
        } else {
          full = true;
        }
      } else if (root && pass == 4) {
        if (n_jk < kFeasMaxCandidates) {
          jk_t[n_jk] = t;
          jk_v[n_jk++] = v;
        } else {
          full = true;
        }
      }
    };
    take(0.0, true);
    take(T, true);
    extrema_candidates(g, [&](double tau, bool root) { take(tau * T, root); });
    if (full) return kFeasIndeterminable | kFeasCapacity;
    if (pass == 0) {
      if ((pr & kFeasFMin) && lo < prm.f_min) return kFeasThrustLow;
      if ((pr & kFeasFMax) && hi > prm.f_max) return kFeasThrustHigh;
    } else if (pass == 1) {
      if (hi > prm.v_max) return kFeasVelocity;
    } else if (pass == 2) {
      if (hi > prm.omega_z) return kFeasYawRates;
    } else if (pass == 3) {
      if (hi > prm.omega_z_dot) return kFeasYawAcc;
    }
  }
  if (!(pr & kFeasOmegaXY)) return kFeasFeasible;
  // recursiveRollPitchFeasibility, depth first, left half first.  A node's result is Feasible or Indeterminable, and
  // the first Indeterminable node decides the segment.  Bit l of `path` is 1 when the node at level l + 1 is the
  // right half of its parent.
  const double limit = prm.omega_xy, mst = prm.min_section_time;
  unsigned long long path = 0;
  int level = 0;
  while (true) {
    double t1 = 0.0, t2 = T;
    for (int l = 0; l < level; ++l) {
      const double th = __dmul_rn(__dadd_rn(t1, t2), 0.5);  // (t1 + t2) / 2
      if ((path >> l) & 1ull) t1 = th;
      else t2 = th;
    }
    if (__dsub_rn(t2, t1) < mst) return kFeasIndeterminable;
    double f_min = DBL_MAX, j_max = -DBL_MAX;  // selectMinMaxMagnitudeFromCandidates: closed interval, no end points
    for (int i = 0; i < n_th; ++i)
      if (!(th_t[i] < t1 || th_t[i] > t2) && th_v[i] < f_min) f_min = th_v[i];
    for (int i = 0; i < n_jk; ++i)
      if (!(jk_t[i] < t1 || jk_t[i] > t2) && j_max < jk_v[i]) j_max = jk_v[i];
    // no jerk candidate: sqrt of a negative number is NaN, and NaN > limit is false
    const double bound = f_min > 1.0e-6 ? __dsqrt_rn(__ddiv_rn(j_max, f_min)) : DBL_MAX;
    if (bound > limit) {
      if (level == kFeasMaxLevel) return kFeasIndeterminable | kFeasCapacity;
      ++level;  // the left half (its path bit is 0)
      continue;
    }
    // this node is feasible: a right half completes its parent
    while (level > 0 && ((path >> (level - 1)) & 1ull)) {
      --level;
      path &= ~(1ull << level);
    }
    if (level == 0) return kFeasFeasible;
    path |= 1ull << (level - 1);  // the right half of the same parent
  }
}

// The tile loop of the feasibility kernels.  Work item = (trajectory, segment), as max_magnitude_kernel: each
// segment's code goes to shared memory, then one thread per trajectory takes the first segment whose code is not 0.
// segment_code(item, T) checks one segment with a good time T (item = trajectory * K + segment) and returns 0 when it
// passes; row(traj, bad, seg, code) writes one trajectory's outputs: bad when some segment time is <= 0 or non-finite
// (seg = -1, code = 0 then), else the first failing segment and its code, or seg = -1 and code = 0.
// dynamic shared memory: [tpb * K] codes
template <typename SegmentCode, typename Row>
__device__ __forceinline__ void first_failing_segment(long long B, int K, const double* __restrict__ times, int tpb,
                                                      SegmentCode&& segment_code, Row&& row) {
  extern __shared__ int feas_sm[];
  for (long long t0 = (long long)blockIdx.x * tpb; t0 < B; t0 += (long long)gridDim.x * tpb) {
    const int ntraj = int(B - t0 < tpb ? B - t0 : tpb);
    const int items = ntraj * K;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
      const long long item = t0 * K + it;
      const double T = times[item];
      const bool bad = !(T > 0.0) || !isfinite(T);
      feas_sm[it] = bad ? 0 : segment_code(item, T);
    }
    __syncthreads();
    for (int lt = threadIdx.x; lt < ntraj; lt += blockDim.x) {
      const long long traj = t0 + lt;
      bool bad = false;
      for (int i = 0; i < K; ++i) {
        const double T = times[traj * K + i];
        if (!(T > 0.0) || !isfinite(T)) bad = true;
      }
      int seg = -1, code = 0;
      if (!bad) {
        for (int i = 0; i < K; ++i) {
          const int c = feas_sm[lt * K + i];
          if (c != 0) {
            seg = i;
            code = c;
            break;
          }
        }
      }
      row(traj, bad, seg, code);
    }
    __syncthreads();
  }
}

// One thread per (trajectory, segment) runs feas_segment; the first segment that is not Feasible decides.
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) input_feasibility_kernel(const FeasParams prm, const int tpb) {
  first_failing_segment(
      prm.B, prm.K, prm.times, tpb,
      [&](long long item, double T) { return feas_segment<N>(prm.coeffs + item * prm.D * N, T, prm); },
      [&](long long traj, bool bad, int seg, int code) {
        int res = code & 0xff, st = 0;
        if (bad) {
          res = kFeasIndeterminable;
          st = 1;  // MTG_STATUS_BAD_TIME
        } else if (code & kFeasCapacity) {
          st = 4;  // MTG_STATUS_FEAS_CAPACITY
        }
        prm.result[traj] = res;
        if (prm.segment) prm.segment[traj] = seg;
        if (prm.status) prm.status[traj] = st;
      });
}

}  // namespace mtg
