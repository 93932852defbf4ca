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
  double sampling_interval;  // FeasibilitySampling only
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

constexpr int kFeasSplit = -1;  // a walk node's "halve this section"

// The reference's recursive bisection of [0, T] (recursiveRollPitchFeasibility / recursiveFeasibility), depth first,
// left half first, without a stack: the current node is a level and a path of left/right bits (bit l is 1 when the
// node at level l + 1 is the right half of its parent), and its bounds are recomputed from [0, T] with the reference's
// (t1 + t2) / 2.  A section shorter than min_section_time is Indeterminable; otherwise node(t1, t2) returns kFeasSplit
// or the section's FeasResult.  A split node's result is its left half's when that is not Feasible, else its right
// half's, so the first leaf that is not Feasible decides.  Splitting below level kFeasMaxLevel gives Indeterminable |
// kFeasCapacity.
template <typename Node>
__device__ __forceinline__ int feas_walk(double T, double min_section_time, Node&& node) {
  unsigned long long path = 0;
  int level = 0;
  while (true) {
    double t1 = 0.0, t2 = T;
    for (int l = 0; l < level; ++l) {
      const double th = __dmul_rn(__dadd_rn(t1, t2), 0.5);  // (t1 + t2) / 2
      if ((path >> l) & 1ull) t1 = th;
      else t2 = th;
    }
    if (__dsub_rn(t2, t1) < min_section_time) return kFeasIndeterminable;
    const int r = node(t1, t2);
    if (r == kFeasSplit) {
      if (level == kFeasMaxLevel) return kFeasIndeterminable | kFeasCapacity;
      ++level;  // the left half (its path bit is 0)
      continue;
    }
    if (r != kFeasFeasible) return r;
    // this node is feasible: a right half completes its parent
    while (level > 0 && ((path >> (level - 1)) & 1ull)) {
      --level;
      path &= ~(1ull << level);
    }
    if (level == 0) return kFeasFeasible;
    path |= 1ull << (level - 1);  // the right half of the same parent
  }
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
  // recursiveRollPitchFeasibility: a node whose bound sqrt(j_max / f_min) exceeds omega_xy_max is halved
  const double limit = prm.omega_xy;
  return feas_walk(T, prm.min_section_time, [&](double t1, double t2) {
    double f_min = DBL_MAX, j_max = -DBL_MAX;  // selectMinMaxMagnitudeFromCandidates: closed interval, no end points
    for (int i = 0; i < n_th; ++i)
      if (!(th_t[i] < t1 || th_t[i] > t2) && th_v[i] < f_min) f_min = th_v[i];
    for (int i = 0; i < n_jk; ++i)
      if (!(jk_t[i] < t1 || jk_t[i] > t2) && j_max < jk_v[i]) j_max = jk_v[i];
    // no jerk candidate: sqrt of a negative number is NaN, and NaN > limit is false
    const double bound = f_min > 1.0e-6 ? __dsqrt_rn(__ddiv_rn(j_max, f_min)) : DBL_MAX;
    return bound > limit ? kFeasSplit : int(kFeasFeasible);
  });
}

// The tile loop of the feasibility kernels.  Work item = (trajectory, segment), as max_magnitude_kernel: each
// segment's code goes to shared memory, then one thread per trajectory takes the first segment whose code is not 0.
// W consecutive threads share one work item (W = 1: a thread per segment; W = 32: a warp per segment, every lane
// calling segment_code with the same arguments and lane 0 storing its code).  segment_code(item, T) checks one segment
// with a good time T (item = trajectory * K + segment) and returns 0 when it passes; row(traj, bad, seg, code) writes
// one trajectory's outputs: bad when some segment time is <= 0 or non-finite (seg = -1, code = 0 then), else the first
// failing segment and its code, or seg = -1 and code = 0.
// dynamic shared memory: [tpb * K] codes
template <int W = 1, typename SegmentCode, typename Row>
__device__ __forceinline__ void first_failing_segment(long long B, int K, const double* __restrict__ times, int tpb,
                                                      SegmentCode&& segment_code, Row&& row) {
  extern __shared__ int feas_sm[];
  for (long long t0 = (long long)blockIdx.x * tpb; t0 < B; t0 += (long long)gridDim.x * tpb) {
    const int ntraj = int(B - t0 < tpb ? B - t0 : tpb);
    const int items = ntraj * K;
    for (int it = threadIdx.x / W; it < items; it += blockDim.x / W) {
      const long long item = t0 * K + it;
      const double T = times[item];
      const bool bad = !(T > 0.0) || !isfinite(T);
      const int code = bad ? 0 : segment_code(item, T);
      if (threadIdx.x % W == 0) feas_sm[it] = code;
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

// One trajectory's outputs from first_failing_segment: a bad time gives Indeterminable and MTG_STATUS_BAD_TIME, a
// segment code with kFeasCapacity gives MTG_STATUS_FEAS_CAPACITY.
__device__ __forceinline__ void feas_row(const FeasParams& prm, long long traj, bool bad, int seg, int code) {
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
}

// One thread per (trajectory, segment) runs feas_segment; the first segment that is not Feasible decides.
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) input_feasibility_kernel(const FeasParams prm, const int tpb) {
  first_failing_segment(
      prm.B, prm.K, prm.times, tpb,
      [&](long long item, double T) { return feas_segment<N>(prm.coeffs + item * prm.D * N, T, prm); },
      [&](long long traj, bool bad, int seg, int code) { feas_row(prm, traj, bad, seg, code); });
}

// ---- FeasibilityRecursive::checkInputFeasibility (reference mav_trajectory_generation_ros/src/
// feasibility_recursive.cpp:42-304) -----------------------------------------------------------------------------------
// Per position axis i and order k = 1, 2, 3 (velocity, acceleration, jerk) the roots of p_i^(k+1) in [0, T]: the
// critical polynomial of extrema_critical with D = 1 at its own degree (M = N - 1), and only the points that
// extrema_candidates flags as roots, a halving point where the polynomial is 0 to within rounding included (a
// rest-to-rest segment is symmetric, and its speed peaks exactly at T / 2).  A list holds at most N - 2 - k roots plus kFeasRecSlack midpoints of intervals
// left unresolved at the isolator's depth cap.  Each root's p_i^(k) is evaluated once per segment; a node evaluates
// only its two ends.

constexpr int kFeasRecSlack = 2;

template <int N>
__host__ __device__ constexpr int feas_rec_cap(int k) {  // entries of one (axis, order k) root list
  return (N - 2 - k > 0 ? N - 2 - k : 0) + kFeasRecSlack;
}
template <int N>
__host__ __device__ constexpr int feas_rec_base(int k) {  // first entry of order k's three lists
  return k <= 1 ? 0 : feas_rec_base<N>(k - 1) + 3 * feas_rec_cap<N>(k - 1);
}

// p_i^(k)(t) with Polynomial::evaluate's arithmetic
template <int N>
__device__ __forceinline__ double feas_axis_value(const double* __restrict__ c, int i, int k, double t) {
  double cd[N];
#pragma unroll
  for (int j = 0; j < N; ++j) cd[j] = c[i * N + j];
  return range_horner_any<N>(cd, t, k);
}

// evaluateThrust: |p''(t) + (0, 0, g)|, the acceleration evaluated first and g added to z afterwards
template <int N>
__device__ __forceinline__ double feas_rec_thrust(const double* __restrict__ c, double g, double t) {
  double sq = 0.0;
#pragma unroll 1
  for (int d = 0; d < 3; ++d) {
    double a = feas_axis_value<N>(c, d, 2, t);
    if (d == 2) a = __dadd_rn(a, g);
    sq = __dadd_rn(sq, __dmul_rn(a, a));
  }
  return __dsqrt_rn(sq);
}

// std::max / std::min (the first argument on a tie or a NaN second argument)
__device__ __forceinline__ double feas_max(double a, double b) { return a < b ? b : a; }
__device__ __forceinline__ double feas_min(double a, double b) { return b < a ? b : a; }

// The check of one segment (time T > 0 and finite): a FeasResult, or-ed with kFeasCapacity when a root list or the
// walk ran out of room (the segment is then reported Indeterminable).
template <int N>
__device__ int feas_rec_segment(const double* __restrict__ c, double T, const FeasParams& prm) {
  constexpr int L = feas_rec_base<N>(4);  // entries of all nine lists
  if (prm.D != 3 && prm.D != 4) return kFeasIndeterminable;
  const unsigned pr = prm.present;
  const bool need[4] = {false, (pr & kFeasVMax) != 0, (pr & (kFeasFMin | kFeasFMax | kFeasOmegaXY)) != 0,
                        (pr & kFeasOmegaXY) != 0};
  double rt[L], rv[L];  // root times and their p_i^(k)
  int cnt[9];
  double yaw_max[2] = {0.0, 0.0};  // max |yaw'|, |yaw''| over 0, T and every candidate (computeMinMax on [0, T])
  bool full = false;
  // lists 0..8: (order k = 1 + q / 3, axis q % 3); 9, 10: yaw' and yaw'' (dim 3, D = 4) -- one inlined isolation
#pragma unroll 1
  for (int q = 0; q < 11; ++q) {
    const bool yaw = q >= 9;
    const int k = yaw ? q - 8 : 1 + q / 3, i = yaw ? 3 : q % 3;
    if (!yaw) cnt[q] = 0;
    if (yaw ? !(prm.D == 4 && (pr & (q == 9 ? kFeasOmegaZ : kFeasOmegaZDot))) : !need[k]) continue;
    double g[N - 1];
    extrema_critical<N, N - 1>(c + i * N, T, 1, k, 0.0, g);
    if (yaw) {
      double hi = fmax(fabs(feas_axis_value<N>(c, 3, k, 0.0)), fabs(feas_axis_value<N>(c, 3, k, T)));
      extrema_candidates(g, [&](double tau, bool) { hi = fmax(hi, fabs(feas_axis_value<N>(c, 3, k, tau * T))); });
      yaw_max[q - 9] = hi;
      continue;
    }
    const int cap = feas_rec_cap<N>(k), o = feas_rec_base<N>(k) + i * cap;
    int n = 0;
    extrema_candidates<N - 1, true>(g, [&](double tau, bool root) {
      if (!root) return;
      if (n == cap) {
        full = true;
        return;
      }
      const double t = tau * T;
      rt[o + n] = t;
      rv[o + n] = feas_axis_value<N>(c, i, k, t);
      ++n;
    });
    cnt[q] = n;
  }
  if (full) return kFeasIndeterminable | kFeasCapacity;
  const double g = prm.gravity;
  // recursiveFeasibility on one section [t1, t2]
  const int r = feas_walk(T, prm.min_section_time, [&](double t1, double t2) -> int {
    if (pr & (kFeasFMin | kFeasFMax)) {
      const double f1 = feas_rec_thrust<N>(c, g, t1), f2 = feas_rec_thrust<N>(c, g, t2);
      if ((pr & kFeasFMin) && feas_min(f1, f2) < prm.f_min) return kFeasThrustLow;
      if ((pr & kFeasFMax) && feas_max(f1, f2) > prm.f_max) return kFeasThrustHigh;
    }
    if (pr & kFeasVMax) {
      const double v1 = extrema_magnitude<N>(c, 3, 1, t1), v2 = extrema_magnitude<N>(c, 3, 1, t2);
      if (feas_max(v1, v2) > prm.v_max) return kFeasVelocity;
    }
    double f_min_sqr = 0.0, f_max_sqr = 0.0, v_max_sqr = 0.0, j_max_sqr = 0.0;
#pragma unroll 1
    for (int q = 0; q < 9; ++q) {
      const int k = 1 + q / 3, i = q % 3;
      if (!need[k]) continue;
      // selectMinMaxFromRoots: candidates t1, t2 and the roots in the closed [t1, t2]
      double lo = DBL_MAX, hi = -DBL_MAX;
      auto take = [&](double v) {
        if (v < lo) lo = v;
        if (v > hi) hi = v;
      };
      take(feas_axis_value<N>(c, i, k, t1));
      take(feas_axis_value<N>(c, i, k, t2));
      const int o = feas_rec_base<N>(k) + i * feas_rec_cap<N>(k);
      for (int e = 0; e < cnt[q]; ++e)
        if (!(rt[o + e] < t1 || rt[o + e] > t2)) take(rv[o + e]);
      if (k == 1) {
        if (feas_max(__dmul_rn(lo, lo), __dmul_rn(hi, hi)) > __dmul_rn(prm.v_max, prm.v_max)) return kFeasVelocity;
        const double m = feas_max(fabs(lo), fabs(hi));
        v_max_sqr = __dadd_rn(v_max_sqr, __dmul_rn(m, m));
      } else if (k == 2) {
        const double gi = i == 2 ? g : 0.0;  // gravity_[i]
        const double f_lo = __dadd_rn(lo, gi), f_hi = __dadd_rn(hi, gi);
        const double m = feas_max(fabs(f_lo), fabs(f_hi));
        if ((pr & kFeasFMax) && m > prm.f_max) return kFeasThrustHigh;
        if (!(__dmul_rn(f_lo, f_hi) < 0.0)) {
          const double l = feas_min(fabs(f_lo), fabs(f_hi));
          f_min_sqr = __dadd_rn(f_min_sqr, __dmul_rn(l, l));
        }
        f_max_sqr = __dadd_rn(f_max_sqr, __dmul_rn(m, m));
      } else {
        const double m = feas_max(fabs(lo), fabs(hi));
        j_max_sqr = __dadd_rn(j_max_sqr, __dmul_rn(m, m));
      }
    }
    const double f_lower = __dsqrt_rn(f_min_sqr), f_upper = __dsqrt_rn(f_max_sqr), v_upper = __dsqrt_rn(v_max_sqr);
    const double omega_upper = f_min_sqr > 1.0e-6 ? __dsqrt_rn(__ddiv_rn(j_max_sqr, f_min_sqr)) : DBL_MAX;
    if ((pr & kFeasFMin) && f_upper < prm.f_min) return kFeasThrustLow;
    if ((pr & kFeasFMax) && f_lower > prm.f_max) return kFeasThrustHigh;
    const bool split = ((pr & kFeasFMin) && f_lower < prm.f_min) || ((pr & kFeasFMax) && f_upper > prm.f_max) ||
                       ((pr & kFeasVMax) && v_upper > prm.v_max) || ((pr & kFeasOmegaXY) && omega_upper > prm.omega_xy);
    return split ? kFeasSplit : int(kFeasFeasible);
  });
  if (r != kFeasFeasible || prm.D != 4) return r;
  if ((pr & kFeasOmegaZ) && yaw_max[0] > prm.omega_z) return kFeasYawRates;
  if ((pr & kFeasOmegaZDot) && yaw_max[1] > prm.omega_z_dot) return kFeasYawAcc;
  return kFeasFeasible;
}

// One thread per (trajectory, segment) runs feas_rec_segment; the first segment that is not Feasible decides.
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1)
    input_feasibility_recursive_kernel(const FeasParams prm, const int tpb) {
  first_failing_segment(
      prm.B, prm.K, prm.times, tpb,
      [&](long long item, double T) { return feas_rec_segment<N>(prm.coeffs + item * prm.D * N, T, prm); },
      [&](long long traj, bool bad, int seg, int code) { feas_row(prm, traj, bad, seg, code); });
}

// ---- FeasibilitySampling::checkInputFeasibility (reference mav_trajectory_generation_ros/src/
// feasibility_sampling.cpp) ------------------------------------------------------------------------------------------
// The samples are t = 0, fl(t + dt), ... while t <= T: the reference's running fp64 sum, not k * dt.  At each sample
// the flat state (velocity, acceleration and jerk of dims 0..2; for D = 4 yaw, yaw rate and yaw acceleration of dim 3,
// else 0) goes through mav_msgs' EigenMavStateFromEigenTrajectoryPoint:
//   f = a + (0, 0, g), thrust = |f|, zb = f * (1 / thrust), xc = (cos yaw, sin yaw, 0), yb = normalized(zb x xc),
//   xb = yb x zb, acceleration_B = R^T (zb * thrust) with R = [xb yb zb], h = (1 / thrust) (j - (zb . j) zb),
//   omega_B = (-h . yb, h . xb, yaw_rate zb_z), omega_dot_B,z = yaw_acc zb_z,
// and the reference's checks run in order: |acceleration_B| against f_min, f_max (only when one of them is present),
// |v| against v_max, |omega_B,xy|, |omega_B,z|, |omega_dot_B,z|.  Yaw goes through setFromYaw / getYaw (a quaternion
// about z and atan2 back).  Every operation is rounded on its own (no contraction), dot products and squared norms sum
// in index order.  A thrust of exactly 0 makes the state NaN, and NaN passes every comparison, as in the reference.

constexpr double kFeasSampleCap = 16777216.0;  // 2^24: a segment with fl(T / dt) above it is not sampled
constexpr int kFeasHoist = 12;  // hoisted coefficient rows per warp: (dims 0..2) x (orders 1..3), then yaw orders 0..2

// fl(B(k, j) c_j) of dim d, order k at row (d < 3 ? 3 d + k - 1 : 9 + k); Horner over them is Polynomial::evaluate's
template <int N>
__device__ __forceinline__ int feas_hoist_row(int d, int k) {
  return (d < 3 ? 3 * d + k - 1 : 9 + k) * N;
}

template <int N, int K>
__device__ __forceinline__ double feas_hoisted_horner(const double* __restrict__ h, double t) {
  double acc = h[N - 1];
#pragma unroll
  for (int j = N - 2; j >= K; --j) acc = __dadd_rn(__dmul_rn(acc, t), h[j]);
  return acc;
}

struct FeasVec3 {
  double x, y, z;
};
__device__ __forceinline__ double feas_dot(const FeasVec3& a, const FeasVec3& b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ FeasVec3 feas_cross(const FeasVec3& a, const FeasVec3& b) {
  return {__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
          __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}
__device__ __forceinline__ FeasVec3 feas_scale(double s, const FeasVec3& a) {
  return {__dmul_rn(s, a.x), __dmul_rn(s, a.y), __dmul_rn(s, a.z)};
}

// The check of one sample at time t: 0 (passes) or a FeasResult.  h: this segment's hoisted products.  Only what a
// present limit needs is evaluated.
template <int N>
__device__ __forceinline__ int feas_sample(const double* __restrict__ h, double t, const FeasParams& prm) {
  const unsigned pr = prm.present;
  const bool yaw4 = prm.D == 4;
  const bool thrust_check = (pr & (kFeasFMin | kFeasFMax)) != 0;
  const bool need_r = thrust_check || (pr & kFeasOmegaXY);
  double thrust = 0.0, inv = 0.0;
  FeasVec3 zb = {0.0, 0.0, 0.0}, yb = zb, xb = zb;
  if (need_r || (yaw4 && (pr & (kFeasOmegaZ | kFeasOmegaZDot)))) {
    const FeasVec3 f = {feas_hoisted_horner<N, 2>(h + feas_hoist_row<N>(0, 2), t),
                        feas_hoisted_horner<N, 2>(h + feas_hoist_row<N>(1, 2), t),
                        __dadd_rn(feas_hoisted_horner<N, 2>(h + feas_hoist_row<N>(2, 2), t), prm.gravity)};
    thrust = __dsqrt_rn(feas_dot(f, f));
    inv = __ddiv_rn(1.0, thrust);
    zb = feas_scale(inv, f);
  }
  if (need_r) {
    double cy = 1.0, sy = 0.0;  // D = 3: yaw 0
    if (yaw4) {                 // setFromYaw, then getYaw: atan2(2 (w z + x y), 1 - 2 (y y + z z)) with x = y = 0
      double qz, qw;
      sincos(__dmul_rn(0.5, feas_hoisted_horner<N, 0>(h + feas_hoist_row<N>(3, 0), t)), &qz, &qw);
      const double yaw = atan2(__dmul_rn(2.0, __dadd_rn(__dmul_rn(qw, qz), __dmul_rn(0.0, 0.0))),
                               __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(__dmul_rn(0.0, 0.0), __dmul_rn(qz, qz)))));
      sincos(yaw, &sy, &cy);
    }
    yb = feas_cross(zb, {cy, sy, 0.0});
    const double n2 = feas_dot(yb, yb);
    if (n2 > 0.0) {  // Eigen's normalized(): a zero vector stays as it is
      const double n = __dsqrt_rn(n2);
      yb = {__ddiv_rn(yb.x, n), __ddiv_rn(yb.y, n), __ddiv_rn(yb.z, n)};
    }
    xb = feas_cross(yb, zb);
  }
  if (thrust_check) {
    const FeasVec3 w = feas_scale(thrust, zb), ab = {feas_dot(xb, w), feas_dot(yb, w), feas_dot(zb, w)};
    const double thrust_b = __dsqrt_rn(feas_dot(ab, ab));
    if ((pr & kFeasFMin) && thrust_b < prm.f_min) return kFeasThrustLow;
    if ((pr & kFeasFMax) && thrust_b > prm.f_max) return kFeasThrustHigh;
  }
  if (pr & kFeasVMax) {
    const FeasVec3 v = {feas_hoisted_horner<N, 1>(h + feas_hoist_row<N>(0, 1), t),
                        feas_hoisted_horner<N, 1>(h + feas_hoist_row<N>(1, 1), t),
                        feas_hoisted_horner<N, 1>(h + feas_hoist_row<N>(2, 1), t)};
    if (__dsqrt_rn(feas_dot(v, v)) > prm.v_max) return kFeasVelocity;
  }
  if (pr & kFeasOmegaXY) {
    const FeasVec3 j = {feas_hoisted_horner<N, 3>(h + feas_hoist_row<N>(0, 3), t),
                        feas_hoisted_horner<N, 3>(h + feas_hoist_row<N>(1, 3), t),
                        feas_hoisted_horner<N, 3>(h + feas_hoist_row<N>(2, 3), t)};
    const double zj = feas_dot(zb, j);
    const FeasVec3 hw = feas_scale(inv, {__dsub_rn(j.x, __dmul_rn(zj, zb.x)), __dsub_rn(j.y, __dmul_rn(zj, zb.y)),
                                         __dsub_rn(j.z, __dmul_rn(zj, zb.z))});
    const double wx = -feas_dot(hw, yb), wy = feas_dot(hw, xb);
    if (__dsqrt_rn(__dadd_rn(__dmul_rn(wx, wx), __dmul_rn(wy, wy))) > prm.omega_xy) return kFeasRollPitchRates;
  }
  // D = 3: yaw rate and acceleration are 0, and 0 * zb_z never exceeds a limit >= 0
  if (yaw4 && (pr & kFeasOmegaZ) &&
      fabs(__dmul_rn(feas_hoisted_horner<N, 1>(h + feas_hoist_row<N>(3, 1), t), zb.z)) > prm.omega_z)
    return kFeasYawRates;
  if (yaw4 && (pr & kFeasOmegaZDot) &&
      fabs(__dmul_rn(feas_hoisted_horner<N, 2>(h + feas_hoist_row<N>(3, 2), t), zb.z)) > prm.omega_z_dot)
    return kFeasYawAcc;
  return kFeasFeasible;
}

// The check of one segment (time T > 0 and finite) by one warp: every lane returns the same FeasResult, or
// Indeterminable | kFeasCapacity when fl(T / dt) > 2^24.  The warp first stores the hoisted products fl(B(k, j) c_j) in
// h (kFeasHoist N doubles, rows beyond D unused), then walks the samples in chunks of 32: every lane carries the same
// running sum and keeps the value after `lane` additions, so the times are the reference's bit for bit.  A ballot over
// the chunk's codes gives the first failing sample; a chunk that reaches past T is the last one.  Under the cap the sum
// always advances: dt >= T 2^-24, far above the rounding unit of any t <= T.
template <int N>
__device__ int feas_sampling_segment(const double* __restrict__ c, double T, double* __restrict__ h,
                                     const FeasParams& prm) {
  if (prm.D != 3 && prm.D != 4) return kFeasIndeterminable;
  const double dt = prm.sampling_interval;
  if (__ddiv_rn(T, dt) > kFeasSampleCap) return kFeasIndeterminable | kFeasCapacity;
  const int lane = threadIdx.x & 31;
  const int rows = prm.D == 4 ? kFeasHoist : 9;
  for (int q = lane; q < rows * N; q += 32) {
    const int r = q / N, j = q - r * N;
    const int d = r < 9 ? r / 3 : 3, k = r < 9 ? r % 3 + 1 : r - 9;
    double b = 1.0;  // B(k, j) = j! / (j - k)!, an exact integer
    for (int w = 0; w < k; ++w) b *= double(j - w);
    h[q] = j < k ? 0.0 : __dmul_rn(b, c[d * N + j]);
  }
  __syncwarp();
  double s = 0.0;  // the running sum at the chunk's first sample
  int code = kFeasFeasible;
  while (true) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i == lane) t = s;
      s = __dadd_rn(s, dt);
    }
    const bool in = t <= T;
    const int mine = in ? feas_sample<N>(h, t, prm) : int(kFeasFeasible);
    const unsigned fail = __ballot_sync(0xffffffffu, mine != kFeasFeasible);
    if (fail) {
      code = __shfl_sync(0xffffffffu, mine, __ffs(fail) - 1);
      break;
    }
    if (__ballot_sync(0xffffffffu, !in)) break;
  }
  __syncwarp();  // h is rewritten by the warp's next segment
  return code;
}

// One warp per (trajectory, segment) runs feas_sampling_segment; the first segment that is not Feasible decides.
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1)
    input_feasibility_sampling_kernel(const FeasParams prm, const int tpb) {
  __shared__ double hoist[kExtremaThreads / 32][kFeasHoist * N];
  double* __restrict__ h = hoist[threadIdx.x / 32];
  first_failing_segment<32>(
      prm.B, prm.K, prm.times, tpb,
      [&](long long item, double T) { return feas_sampling_segment<N>(prm.coeffs + item * prm.D * N, T, h, prm); },
      [&](long long traj, bool bad, int seg, int code) { feas_row(prm, traj, bad, seg, code); });
}

}  // namespace mtg
