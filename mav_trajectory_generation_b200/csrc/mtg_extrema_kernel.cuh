// mtg_extrema_kernel.cuh -- PolynomialOptimization::computeMaximumOfMagnitude (reference
// impl/polynomial_optimization_linear_impl.h:465-497) for B trajectories and several derivative orders at once, and the
// soft-constraint time objective of PolynomialOptimizationNonLinear built on it (objectiveFunctionTime /
// objectiveFunctionTimeAndConstraints, impl/polynomial_optimization_nonlinear_impl.h:556-615, 660-742, with
// evaluateMaximumMagnitudeAsSoftConstraint, :766-795).
//
// Candidates of segment i (src/segment.cpp:83-184): 0, T_i and every real root in [0, T_i] of the critical polynomial
// g = sum_d p_d^(k) p_d^(k+1) (D >= 2) or p^(k+1) (D = 1).  Each candidate's value is |p^(k)(t)| with every component
// evaluated by range_horner (bit-identical to Polynomial::evaluate); the largest value wins, the first one on a tie.
//
// Root finding works on G(tau) = g(tau T) (up to a positive factor) over [0, 1]: the Bernstein coefficients of G on a
// dyadic interval are formed from the power coefficients (Taylor shift + basis change, fully unrolled, in registers) and
// Descartes' rule of signs on them bounds the roots inside.  No sign change: no root.  One sign change: exactly one
// root, refined by Newton steps safeguarded by bisection.  More: the interval is halved, depth-first from the left
// without a stack (the next interval follows from its level and index), and every halving point is itself a candidate,
// so a root that rounding hides from both halves still has a candidate next to it.  At the depth cap or the node
// budget an unresolved interval contributes its ends and midpoint.  Extra candidates only cost an evaluation; a missed
// one would be a wrong answer.
#pragma once

#include <cfloat>

#include "mtg_generic_kernel.cuh"

namespace mtg {

constexpr int kExtremaMaxDerivs = 8;
constexpr int kExtremaMaxDepth = 24;   // smallest interval 2^-24 T
constexpr int kExtremaNodeBudget = 512;
constexpr int kExtremaThreads = 128;

struct ExtremaParams {
  int K, D, n_derivs;
  int derivs[kExtremaMaxDerivs];
  long long B;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ coeffs;  // [B][K][D][N]
  double* __restrict__ value;         // [B][n_derivs]
  double* __restrict__ time;          // [B][n_derivs] or null
  int* __restrict__ segment;          // [B][n_derivs] or null
  int* __restrict__ status;           // [B] or null
};

// C(i, j) / C(n, j): the power -> Bernstein weights (exact small rationals, immediates after unrolling)
__host__ __device__ constexpr double bernstein_weight(int n, int i, int j) {
  double w = 1.0;
  for (int q = 0; q < j; ++q) w = w * double(i - q) / double(n - q);
  return w;
}

// Bernstein coefficients on [a, a + h] of the degree-(M-1) polynomial g (power basis, increasing)
template <int M>
__device__ __forceinline__ void extrema_bernstein(const double (&g)[M], double a, double h, double (&b)[M]) {
#pragma unroll
  for (int j = 0; j < M; ++j) b[j] = g[j];
  // Taylor shift to a by repeated synthetic division
#pragma unroll
  for (int i = 0; i < M - 1; ++i)
#pragma unroll
    for (int j = M - 2; j >= i; --j) b[j] = fma(a, b[j + 1], b[j]);
  double hp = h;
#pragma unroll
  for (int j = 1; j < M; ++j) {
    b[j] *= hp;
    hp *= h;
  }
  // power -> Bernstein, highest index first so that b[] can be overwritten in place
#pragma unroll
  for (int i = M - 1; i >= 1; --i) {
    double s = b[0];
#pragma unroll
    for (int j = 1; j <= i; ++j) s = fma(bernstein_weight(M - 1, i, j), b[j], s);
    b[i] = s;
  }
}

template <int M>
__device__ __forceinline__ void extrema_horner2(const double (&g)[M], double x, double* p, double* dp) {
  double a = g[M - 1], d = 0.0;
#pragma unroll
  for (int j = M - 2; j >= 0; --j) {
    d = fma(d, x, a);
    a = fma(a, x, g[j]);
  }
  *p = a;
  *dp = d;
}

// the single root of g in (lo, hi), g(lo) and g(hi) of opposite signs
template <int M>
__device__ double extrema_refine(const double (&g)[M], double lo, double hi) {
  double glo, dummy;
  extrema_horner2(g, lo, &glo, &dummy);
  const bool neg_lo = glo < 0.0;
  double x = 0.5 * (lo + hi);
  for (int it = 0; it < 64; ++it) {
    double gx, dgx;
    extrema_horner2(g, x, &gx, &dgx);
    if (gx == 0.0) break;
    if ((gx < 0.0) == neg_lo) lo = x;
    else hi = x;
    double xn = x - gx / dgx;
    if (!(xn > lo && xn < hi)) xn = 0.5 * (lo + hi);
    const double step = fabs(xn - x);
    x = xn;
    if (step <= 2e-16 || hi - lo <= 4e-16) break;
  }
  return x;
}

// Calls visit(tau, root) for every candidate tau in (0, 1) of the critical polynomial g, in increasing order.  root is
// true for a refined root and for the midpoint of an interval still unresolved at the depth cap or node budget, false
// for the extra safety samples (halving points, the ends of an unresolved interval): a whole-segment extremum may use
// every candidate, a check confined to a sub-interval only the first kind (the reference's candidate set).
// kZeroHalvingRoots: a halving point where g is 0 to within the rounding of its evaluation is also flagged as a root.
// A root on a halving point (a symmetric polynomial's, at 1/2) shows its sign change in neither half, since each half
// rounds g there on its own, so it would otherwise be only a safety sample.
template <int M, bool kZeroHalvingRoots = false, typename Visit>
__device__ void extrema_candidates(const double (&g)[M], Visit&& visit) {
  int level = 0, nodes = 0;
  unsigned idx = 0;
  while (true) {
    const double h = ldexp(1.0, -level), a = double(idx) * h;
    if (idx & 1u) {  // a halving point
      bool root = false;
      if (kZeroHalvingRoots) {
        double v = g[M - 1], s = fabs(g[M - 1]);
#pragma unroll
        for (int j = M - 2; j >= 0; --j) {
          v = fma(v, a, g[j]);
          s = fma(s, a, fabs(g[j]));
        }
        root = fabs(v) <= 4.0 * M * DBL_EPSILON * s;
      }
      visit(a, root);
    }
    double b[M];
    extrema_bernstein(g, a, h, b);
    ++nodes;
    int changes = 0;
    double last = 0.0;
#pragma unroll
    for (int j = 0; j < M; ++j) {
      if (b[j] != 0.0) {
        if (last != 0.0 && ((b[j] < 0.0) != (last < 0.0))) ++changes;
        last = b[j];
      }
    }
    bool descend = false;
    if (changes == 1 && b[0] != 0.0 && b[M - 1] != 0.0) {
      visit(extrema_refine(g, a, a + h), true);
    } else if (changes >= 1) {
      if (level < kExtremaMaxDepth && nodes < kExtremaNodeBudget) {
        descend = true;
      } else {
        visit(a, false);
        visit(a + 0.5 * h, true);
        visit(a + h, false);
      }
    }
    if (descend) {
      ++level;
      idx <<= 1;
      continue;
    }
    while (idx & 1u) {
      idx >>= 1;
      --level;
    }
    if (level == 0) break;
    ++idx;
  }
}

// |p^(k)(t)| of segment (b, i): components by range_horner, squares summed in dimension order
template <int N>
__device__ __forceinline__ double extrema_magnitude(const double* __restrict__ c, int D, int k, double t) {
  double sq = 0.0;
  for (int d = 0; d < D; ++d) {
    double cd[N];
#pragma unroll
    for (int j = 0; j < N; ++j) cd[j] = c[d * N + j];
    const double v = range_horner_any<N>(cd, t, k);
    sq = __dadd_rn(sq, __dmul_rn(v, v));
  }
  return sqrt(sq);
}

// The critical polynomial of |p^(k)| on one segment (coefficients c [D][N], time T), in tau = t / T over [0, 1]:
// G(tau) = sum_d A_d(tau) A_d'(tau), A_d(tau) = p_d^(k)(tau T) (D = 1: A'(tau)); nominal degree 2N - 3.  lift is
// added to the constant term of p_2^(k) first (gravity on z: the thrust polynomial of the feasibility check).  A D = 1
// caller may pass M = N - 1 (the degree of A') to keep its root isolation at that degree.
template <int N, int M = (N >= 2 ? 2 * N - 2 : 1)>
__device__ __forceinline__ void extrema_critical(const double* __restrict__ c, double T, int D, int k, double lift,
                                                 double (&g)[M]) {
#pragma unroll
  for (int j = 0; j < M; ++j) g[j] = 0.0;
  for (int d = 0; d < D; ++d) {
    double a[N];
#pragma unroll
    for (int j = 0; j < N; ++j) a[j] = c[d * N + j];
    for (int s = 0; s < k; ++s) {
#pragma unroll
      for (int j = 0; j < N - 1; ++j) a[j] = double(j + 1) * a[j + 1];
      a[N - 1] = 0.0;
    }
    if (lift != 0.0 && d == 2) a[0] += lift;
    double tp = T;
#pragma unroll
    for (int j = 1; j < N; ++j) {
      a[j] *= tp;
      tp *= T;
    }
    if (D == 1) {
#pragma unroll
      for (int j = 0; j < N - 1; ++j) g[j] = double(j + 1) * a[j + 1];
    } else if constexpr (M >= 2 * N - 2) {
#pragma unroll
      for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = 0; j < N - 1; ++j) g[i + j] = fma(a[i], double(j + 1) * a[j + 1], g[i + j]);
    }
  }
}

// The largest |p^(k)| of one segment (coefficients c [D][N], time T > 0 and finite) and where it is: the candidates
// 0, T and the critical points, in the reference's order (0, T, then the critical points, here increasing).  best_v
// and best_t start at 0: a candidate replaces them only when strictly larger.
template <int N>
__device__ __forceinline__ void extrema_segment_max(const double* __restrict__ c, double T, int D, int k,
                                                    double& best_v, double& best_t) {
  constexpr int M = N >= 2 ? 2 * N - 2 : 1;  // coefficients of the critical polynomial (degree 2N - 3)
  double g[M];
  extrema_critical<N>(c, T, D, k, 0.0, g);
  auto take = [&](double t) {
    const double v = extrema_magnitude<N>(c, D, k, t);
    if (best_v < v) {
      best_v = v;
      best_t = t;
    }
  };
  take(0.0);
  take(T);
  extrema_candidates(g, [&](double tau, bool) { take(tau * T); });
}

// Work item = (trajectory, segment): its best candidate per requested derivative goes to shared memory; one thread per
// (trajectory, derivative) then reduces the segments in order (strict <, so the first maximum wins).
// dynamic shared memory: [tpb * K * n_derivs] values, then as many times
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) max_magnitude_kernel(const ExtremaParams prm, const int tpb) {
  extern __shared__ double extrema_sm[];
  const int K = prm.K, D = prm.D, ND = prm.n_derivs;
  double* pv = extrema_sm;
  double* pt = extrema_sm + size_t(tpb) * K * ND;
  for (long long t0 = (long long)blockIdx.x * tpb; t0 < prm.B; t0 += (long long)gridDim.x * tpb) {
    const int ntraj = int(prm.B - t0 < tpb ? prm.B - t0 : tpb);
    const int items = ntraj * K;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
      const long long item = t0 * K + it;
      const double T = prm.times[item];
      const double* __restrict__ c = prm.coeffs + item * D * N;
      const bool bad = !(T > 0.0) || !isfinite(T);
      for (int q = 0; q < ND; ++q) {
        int k = 0;  // prm.derivs[q] with compile-time indices (a dynamic index copies the parameters to local memory)
#pragma unroll
        for (int j = 0; j < kExtremaMaxDerivs; ++j)
          if (j == q) k = prm.derivs[j];
        double best_v = 0.0, best_t = 0.0;
        if (!bad) extrema_segment_max<N>(c, T, D, k, best_v, best_t);
        pv[size_t(it) * ND + q] = bad ? __longlong_as_double(0x7ff8000000000000LL) : best_v;
        pt[size_t(it) * ND + q] = best_t;
      }
    }
    __syncthreads();
    for (int r = threadIdx.x; r < ntraj * ND; r += blockDim.x) {
      const int lt = r / ND, q = r - lt * ND;
      const long long traj = t0 + lt;
      double bv = 0.0, bt = 0.0;
      int bs = 0;
      bool bad = false;
      for (int i = 0; i < K; ++i) {
        const double v = pv[(size_t(lt) * K + i) * ND + q];
        const double T = prm.times[traj * K + i];
        if (!(T > 0.0) || !isfinite(T)) bad = true;
        if (bv < v) {
          bv = v;
          bt = pt[(size_t(lt) * K + i) * ND + q];
          bs = i;
        }
      }
      const double nan = __longlong_as_double(0x7ff8000000000000LL);
      prm.value[traj * ND + q] = bad ? nan : bv;
      if (prm.time) prm.time[traj * ND + q] = bad ? nan : bt;
      if (prm.segment) prm.segment[traj * ND + q] = bad ? -1 : bs;
      if (prm.status && q == 0) prm.status[traj] = bad ? 1 : 0;  // MTG_STATUS_BAD_TIME
    }
    __syncthreads();
  }
}

// Trajectory::scaleSegmentTimesToMeetConstraints (reference src/trajectory.cpp:382-429, Liu et al., RA-L 2017) for B
// trajectories: up to 20 rounds of (max |v|, max |a|) -> stop when both are within 1e-3 of the limits, else stretch
// every segment by max(1, v / v_max, sqrt(a / a_max)) and rescale its coefficients (Polynomial::scalePolynomialInTime,
// src/polynomial.cpp:199-205).
struct ScaleParams {
  int K, D;
  long long B;
  double v_max, a_max;            // > 0; +inf = no limit on that order
  const double* times;            // [B][K]
  const double* coeffs;           // [B][K][D][N]
  double* times_out;              // [B][K], may equal times
  double* coeffs_out;             // [B][K][D][N], may equal coeffs
  const int* __restrict__ skip;   // [B] or null: rows with a non-zero entry are passed through, and it is ORed into status
  int* __restrict__ within;       // [B] or null
  double* __restrict__ maxima;    // [B][2] or null
  int* __restrict__ status;       // [B] or null
};

constexpr int kScaleMaxRounds = 20;  // kMaxCounter, trajectory.cpp:385

// One CTA owns tpb trajectories at a time (tpb = max(1, 128 / K), as max_magnitude_kernel) and runs the whole loop on
// them: phase A, one thread per (trajectory, segment) of every still-active trajectory, puts the segment's max |p'|
// and max |p''| into shared memory; phase B, one thread per trajectory, reduces over segments in order and decides;
// phase C, the threads of phase A with the same item -> thread mapping, stretch the active trajectories into the
// output buffers.  A trajectory is active in round r only if it was stretched in every earlier round, so round 0 reads
// the inputs and every later round reads what the same thread wrote in the round before: the buffers may alias.
// dynamic shared memory: [tpb * K][2] segment maxima, [tpb] stretch factors, [tpb] stretch counts
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) scale_to_constraints_kernel(const ScaleParams prm, const int tpb) {
  extern __shared__ double extrema_sm[];
  const int K = prm.K, D = prm.D;
  double* pv = extrema_sm;                                          // [tpb * K][2]
  double* scale = extrema_sm + size_t(2) * tpb * K;                 // [tpb]; 0 = not stretched this round
  int* stretched = reinterpret_cast<int*>(scale + tpb);             // [tpb]
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const double limit = 1.0 + 1e-3;  // 1.0 + kTolerance, trajectory.cpp:386
  for (long long t0 = (long long)blockIdx.x * tpb; t0 < prm.B; t0 += (long long)gridDim.x * tpb) {
    const int ntraj = int(prm.B - t0 < tpb ? prm.B - t0 : tpb);
    const int items = ntraj * K;
    for (int lt = threadIdx.x; lt < ntraj; lt += blockDim.x) {
      stretched[lt] = 0;
      scale[lt] = 1.0;  // every row takes part in the first check
    }
    __syncthreads();
    for (int round = 0; round < kScaleMaxRounds; ++round) {
      const double* __restrict__ src_t = round == 0 ? prm.times : prm.times_out;
      const double* __restrict__ src_c = round == 0 ? prm.coeffs : prm.coeffs_out;
      // phase A: computeMaxVelocityAndAcceleration of the active rows, per segment
      for (int it = threadIdx.x; it < items; it += blockDim.x) {
        const int lt = it / K;
        if (scale[lt] == 0.0) continue;
        const long long item = t0 * K + it;
        const double T = src_t[item];
        const double* __restrict__ c = src_c + item * D * N;
        const bool bad = !(T > 0.0) || !isfinite(T);
        // one copy of the root isolation for both orders (two inlined copies run measurably slower)
#pragma unroll 1
        for (int k = 1; k <= 2; ++k) {
          double best_v = 0.0, best_t = 0.0;
          if (!bad) extrema_segment_max<N>(c, T, D, k, best_v, best_t);
          pv[size_t(it) * 2 + (k - 1)] = bad ? nan : best_v;
        }
      }
      __syncthreads();
      // phase B: the reference's decision, one thread per active row
      int any = 0;
      for (int lt = threadIdx.x; lt < ntraj; lt += blockDim.x) {
        if (scale[lt] == 0.0) continue;
        const long long traj = t0 + lt;
        const int pre = prm.skip ? prm.skip[traj] : 0;
        double bv = 0.0, ba = 0.0;
        bool bad = false;
        for (int i = 0; i < K; ++i) {
          const double T = src_t[traj * K + i];
          if (!(T > 0.0) || !isfinite(T)) bad = true;
          const double v = pv[(size_t(lt) * K + i) * 2 + 0], a = pv[(size_t(lt) * K + i) * 2 + 1];
          if (bv < v) bv = v;
          if (ba < a) ba = a;
        }
        double s = 0.0;
        bool within = false;
        if (bad || pre) {
          bv = ba = nan;
        } else {
          const double vv = __ddiv_rn(bv, prm.v_max), av = __ddiv_rn(ba, prm.a_max);
          within = vv <= limit && av <= limit;
          if (!within) {
            const double sa = __dsqrt_rn(av);
            const double m = (vv < sa) ? sa : vv;  // std::max(vv, sqrt(av)): a NaN first argument is kept
            s = (1.0 < m) ? m : 1.0;               // std::max(1.0, m): NaN gives 1
          }
        }
        // the values of this check are the last ones if the row stops here or this is the last round (the reference
        // stretches after its 20th check and returns that check's within_range).  A bad row stops: it is never
        // stretched, so its inputs are passed through.
        if (s == 0.0 || round == kScaleMaxRounds - 1) {
          if (prm.within) prm.within[traj] = within ? 1 : 0;
          if (prm.maxima) {
            prm.maxima[traj * 2 + 0] = bv;
            prm.maxima[traj * 2 + 1] = ba;
          }
          if (prm.status) prm.status[traj] = pre | (bad ? 1 : 0);  // MTG_STATUS_BAD_TIME
        }
        scale[lt] = s;
        if (s != 0.0) {
          stretched[lt] += 1;
          any = 1;
        }
      }
      // phase C: stretch the rows that did not meet the limits (scaleSegmentTimes' arithmetic)
      if (!__syncthreads_or(any)) break;
      for (int it = threadIdx.x; it < items; it += blockDim.x) {
        const int lt = it / K;
        const double s = scale[lt];
        if (s == 0.0) continue;
        const double inv = __ddiv_rn(1.0, s);
        const long long item = t0 * K + it;
        const double* c = src_c + item * D * N;
        double* o = prm.coeffs_out + item * D * N;
        const double T = src_t[item];
        for (int d = 0; d < D; ++d) {
          double f = 1.0;
#pragma unroll
          for (int n = 0; n < N; ++n) {
            o[d * N + n] = __dmul_rn(c[d * N + n], f);
            f = __dmul_rn(f, inv);
          }
        }
        prm.times_out[item] = __dmul_rn(T, s);
      }
      __syncthreads();
    }
    // rows never stretched: pass the inputs through
    if (prm.times_out != prm.times || prm.coeffs_out != prm.coeffs) {
      for (int it = threadIdx.x; it < items; it += blockDim.x) {
        if (stretched[it / K]) continue;
        const long long item = t0 * K + it;
        prm.times_out[item] = prm.times[item];
        for (int j = 0; j < D * N; ++j) prm.coeffs_out[item * D * N + j] = prm.coeffs[item * D * N + j];
      }
    }
    __syncthreads();
  }
}

// b[i] |= a[i]
__global__ void __launch_bounds__(128) or_status_kernel(long long n, const int* __restrict__ a, int* __restrict__ b) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    b[i] |= a[i];
}

// The time objective from the pieces the other kernels computed (one thread per trajectory):
// trajectory cost + time cost + soft constraints, in the reference's order.
struct ObjectiveParams {
  int K, n_constraints, richter;
  double time_penalty, weight, maximum_cost;
  double max_value[kExtremaMaxDerivs];
  long long B;
  const double* __restrict__ times;      // [B][K]
  const double* __restrict__ cost;       // [B] computeCost()
  const double* __restrict__ maxima;     // [B][n_constraints]
  const int* __restrict__ solve_status;  // [B]
  double* __restrict__ objective;        // [B]
  double* __restrict__ terms;            // [B][3] or null
  int* __restrict__ status;              // [B] or null
};

__global__ void __launch_bounds__(128) time_objective_kernel(const ObjectiveParams prm) {
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < prm.B; b += (long long)gridDim.x * blockDim.x) {
    int st = prm.solve_status[b];
    double total_time = 0.0;  // computeTotalTrajectoryTime: left to right
    for (int i = 0; i < prm.K; ++i) {
      const double T = prm.times[b * prm.K + i];
      if (!(T > 0.0) || !isfinite(T)) st |= 1;  // MTG_STATUS_BAD_TIME (the setFreeConstraints path has no solve status)
      total_time = __dadd_rn(total_time, T);
    }
    const double cost_time = prm.richter ? __dmul_rn(total_time, prm.time_penalty)
                                         : __dmul_rn(__dmul_rn(total_time, total_time), prm.time_penalty);
    double soft = 0.0;
    for (int q = 0; q < prm.n_constraints; ++q) {
      const double mv = prm.max_value[q];
      const double relative = __ddiv_rn(__dsub_rn(prm.maxima[b * prm.n_constraints + q], mv), mv);
      const double e = exp(__dmul_rn(relative, prm.weight));
      soft = __dadd_rn(soft, e < prm.maximum_cost ? e : prm.maximum_cost);  // std::min(maximum_cost, e)
    }
    const double cost_traj = prm.cost[b];
    const double total = __dadd_rn(__dadd_rn(cost_traj, cost_time), soft);
    prm.objective[b] = st ? __longlong_as_double(0x7ff8000000000000LL) : total;
    if (prm.terms) {
      prm.terms[b * 3 + 0] = cost_traj;
      prm.terms[b * 3 + 1] = cost_time;
      prm.terms[b * 3 + 2] = soft;
    }
    if (prm.status) prm.status[b] = st;
  }
}

}  // namespace mtg
