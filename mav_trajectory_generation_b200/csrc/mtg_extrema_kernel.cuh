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

// Calls visit(tau) for every candidate tau in (0, 1) of the critical polynomial g, in increasing order.
template <int M, typename Visit>
__device__ void extrema_candidates(const double (&g)[M], Visit&& visit) {
  int level = 0, nodes = 0;
  unsigned idx = 0;
  while (true) {
    const double h = ldexp(1.0, -level), a = double(idx) * h;
    if (idx & 1u) visit(a);  // a halving point
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
      visit(extrema_refine(g, a, a + h));
    } else if (changes >= 1) {
      if (level < kExtremaMaxDepth && nodes < kExtremaNodeBudget) {
        descend = true;
      } else {
        visit(a);
        visit(a + 0.5 * h);
        visit(a + h);
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

// Work item = (trajectory, segment): its best candidate per requested derivative goes to shared memory; one thread per
// (trajectory, derivative) then reduces the segments in order (strict <, so the first maximum wins).
// dynamic shared memory: [tpb * K * n_derivs] values, then as many times
template <int N>
__global__ void __launch_bounds__(kExtremaThreads, 1) max_magnitude_kernel(const ExtremaParams prm, const int tpb) {
  constexpr int M = N >= 2 ? 2 * N - 2 : 1;  // coefficients of the critical polynomial (degree 2N - 3)
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
        if (!bad) {
          // G(tau) = sum_d A_d(tau) A_d'(tau), A_d(tau) = p_d^(k)(tau T) (D = 1: A'(tau)); nominal degree 2N - 3
          double g[M];
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
            double tp = T;
#pragma unroll
            for (int j = 1; j < N; ++j) {
              a[j] *= tp;
              tp *= T;
            }
            if (D == 1) {
#pragma unroll
              for (int j = 0; j < N - 1; ++j) g[j] = double(j + 1) * a[j + 1];
            } else {
#pragma unroll
              for (int i = 0; i < N; ++i)
#pragma unroll
                for (int j = 0; j < N - 1; ++j) g[i + j] = fma(a[i], double(j + 1) * a[j + 1], g[i + j]);
            }
          }
          // candidates in the reference's order: 0, T, then the critical points (here increasing)
          auto take = [&](double t) {
            const double v = extrema_magnitude<N>(c, D, k, t);
            if (best_v < v) {
              best_v = v;
              best_t = t;
            }
          };
          take(0.0);
          take(T);
          extrema_candidates(g, [&](double tau) { take(tau * T); });
        }
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
