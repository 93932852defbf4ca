// mtg_mellinger_loop_kernel.cuh -- the per-row kernels of the Mellinger outer loop
// (mtg_optimize_time_mellinger_batch_f64; the algorithm is stated in include/mtg_b200.h and DESIGN.md).
//
// The loop keeps the rows still iterating in a compact list: position p holds original row idx[p], its times x[p],
// its step alpha[p] and its d_fixed.  Every iteration the gradient and the line search run over the compact rows only;
// mel_update_kernel then decides every row, writes the finished ones to their original index and appends the others
// to the next list (a ballot and one atomic per warp), so a row's position never changes what is computed for it.
#pragma once

#include "mtg_waypoint_kernel.cuh"

namespace mtg {

// nlopt_result values (include/mtg_b200.h MTG_OPTIMIZE_RESULT_*)
constexpr int kOptSuccess = 1, kOptFtol = 3, kOptXtol = 4, kOptMaxeval = 5, kOptFailure = -1, kOptRoundoff = -4;
// internal: row passed through the final scaling (never part of a returned status)
constexpr int kStatusPassThrough = 1 << 8;
constexpr double kArmijo = 1e-4;

struct MelLoopParams {
  int K, dnf;  // segments; doubles of one row's d_fixed
  long long B;
  int max_iterations;
  double f_abs, f_rel, x_rel, x_abs, init_rel, lower;
  int k;  // accepted steps of every active row so far (all rows start together)
  // this iteration's compact rows
  int rows;
  const int* __restrict__ idx;
  const double* __restrict__ x;      // [rows][K]
  const double* __restrict__ g;      // [rows][K]
  const double* __restrict__ J;      // [rows] cost at x (the gradient's)
  const double* __restrict__ alpha;  // [rows]
  const double* __restrict__ dfix;   // [rows][dnf]
  const double* __restrict__ Jc;     // [rows][kLineSearchSteps] candidate costs
  const int* __restrict__ st_g;      // [rows][K+1] status of the gradient's solves
  const int* __restrict__ st_c;      // [rows][kLineSearchSteps] status of the candidates' solves
  // the next iteration's compact rows
  int* __restrict__ idx_next;
  double* __restrict__ x_next;
  double* __restrict__ alpha_next;
  double* __restrict__ dfix_next;
  int* __restrict__ count_next;
  // per original row
  double* rel;                       // [B][K] relative times (may be the caller's seg_times)
  int* __restrict__ iters;           // [B]
  int* __restrict__ result;          // [B]
  int* __restrict__ pass;            // [B] kStatusPassThrough: not scaled
  int* __restrict__ opt_status;      // [B] status bits met by the loop
};

// Append the calling thread's row to a compact list when `keep`: returns its position there (or -1).  Every thread of
// the warp must call it.
__device__ __forceinline__ int append_row(bool keep, int* count) {
  const unsigned ball = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == __ffs(ball) - 1) base = atomicAdd(count, __popc(ball));
  base = __shfl_sync(0xffffffffu, base, __ffs(ball ? ball : 1u) - 1);
  return keep ? base + __popc(ball & ((1u << lane) - 1u)) : -1;
}

// Start: copy seg_times to rel, decide the rows that do not iterate, and list the others.
__global__ void __launch_bounds__(128) mel_init_kernel(const MelLoopParams prm, const double* seg_times,
                                                       const double* __restrict__ dfix_in) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int K = prm.K;
  bool active = false;
  if (b < prm.B) {
    bool bad = false, low = false;
    for (int i = 0; i < K; ++i) {
      const double T = seg_times[b * K + i];
      if (!(T > 0.0) || !isfinite(T)) bad = true;
      else if (T < prm.lower) low = true;
      prm.rel[b * K + i] = T;
    }
    int res = kOptFailure, pass = kStatusPassThrough;
    if (!bad && !low) {
      pass = 0;
      if (prm.max_iterations == 0) res = kOptMaxeval;
      else active = true;
    }
    prm.iters[b] = 0;
    prm.result[b] = res;
    prm.pass[b] = pass;
    prm.opt_status[b] = bad ? kStatusBadTime : 0;
  }
  const int p = append_row(active, prm.count_next);
  if (active) {
    prm.idx_next[p] = int(b);
    for (int i = 0; i < K; ++i) prm.x_next[(long long)p * K + i] = seg_times[b * K + i];
    for (int c = 0; c < prm.dnf; ++c) prm.dfix_next[(long long)p * prm.dnf + c] = dfix_in[b * prm.dnf + c];
  }
}

// First step size: initial_stepsize_rel * max x / max |g| (0.1 for initial_stepsize_rel <= 0).
__global__ void __launch_bounds__(128) mel_alpha0_kernel(const MelLoopParams prm, double* __restrict__ alpha) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= prm.rows) return;
  double mx = 0.0, mg = 0.0;
  for (int i = 0; i < prm.K; ++i) {
    const double x = prm.x[p * prm.K + i], g = fabs(prm.g[p * prm.K + i]);
    if (x > mx) mx = x;
    if (g > mg) mg = g;
  }
  const double rel = prm.init_rel > 0.0 ? prm.init_rel : 0.1;
  alpha[p] = __ddiv_rn(__dmul_rn(rel, mx), mg);
}

// Candidates of the shapes without a fused cost kernel: [rows * kLineSearchSteps] (times, d_fixed), as the
// line-search instantiation of the cost-only kernel generates them.
__global__ void __launch_bounds__(128) line_search_expand_kernel(const MelLoopParams prm, double* __restrict__ times_x,
                                                                 double* __restrict__ dfix_x) {
  const int K = prm.K, dnf = prm.dnf;
  const long long total = (long long)prm.rows * kLineSearchSteps;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += nthreads) {
    const long long p = q / kLineSearchSteps;
    const double step = line_search_step(prm.alpha[p], int(q - p * kLineSearchSteps));
    for (int i = 0; i < K; ++i) times_x[q * K + i] = line_search_time(prm.x[p * K + i], prm.g[p * K + i], step, prm.lower);
    for (int c = 0; c < dnf; ++c) dfix_x[q * dnf + c] = prm.dfix[p * dnf + c];
  }
}

// One iteration's decision for every compact row (section "Iteration" of mtg_optimize_time_mellinger_batch_f64).
__global__ void __launch_bounds__(128) mel_update_kernel(const MelLoopParams prm) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int K = prm.K;
  bool keep = false;
  long long b = 0;
  int res = 0, it = prm.k, acc = -1;
  double step = 0.0;
  if (p < prm.rows) {
    b = prm.idx[p];
    const double* __restrict__ x = prm.x + p * K;
    const double* __restrict__ g = prm.g + p * K;
    const double J = prm.J[p];
    int st_grad = 0, st_cand = 0;
    for (int n = 0; n <= K; ++n) st_grad |= prm.st_g[p * (K + 1) + n];
    bool zero = true;
    for (int i = 0; i < K; ++i) zero = zero && g[i] == 0.0;
    // a zero gradient stops the row before its candidates count (they are not read for K = 1, where none are solved)
    if (!zero)
      for (int j = 0; j < kLineSearchSteps; ++j) st_cand |= prm.st_c[p * kLineSearchSteps + j];
    if ((st_grad | st_cand) & kStatusNotSpd) {
      res = kOptFailure;
      prm.opt_status[b] |= kStatusNotSpd;
    } else if (zero) {
      res = kOptSuccess;
    } else {
      for (int j = 0; j < kLineSearchSteps && acc < 0; ++j) {
        const double s = line_search_step(prm.alpha[p], j);
        double dec = 0.0;
        for (int i = 0; i < K; ++i)
          dec = __dadd_rn(dec, __dmul_rn(g[i], __dsub_rn(line_search_time(x[i], g[i], s, prm.lower), x[i])));
        if (prm.Jc[p * kLineSearchSteps + j] <= __dadd_rn(J, __dmul_rn(kArmijo, dec))) {
          acc = j;
          step = s;
        }
      }
      if (acc < 0) {
        res = kOptRoundoff;
      } else {
        it = prm.k + 1;
        const double Jn = prm.Jc[p * kLineSearchSteps + acc];
        const double dJ = fabs(__dsub_rn(Jn, J));
        bool xtol = prm.x_rel >= 0.0 || prm.x_abs >= 0.0;
        for (int i = 0; i < K; ++i) {
          const double xn = line_search_time(x[i], g[i], step, prm.lower);
          const double dx = fabs(__dsub_rn(xn, x[i]));
          xtol = xtol && ((prm.x_rel >= 0.0 && dx <= __dmul_rn(prm.x_rel, fabs(xn))) ||
                          (prm.x_abs >= 0.0 && dx <= prm.x_abs));
        }
        if (prm.max_iterations >= 0 && it >= prm.max_iterations) res = kOptMaxeval;
        else if ((prm.f_rel >= 0.0 && dJ <= __dmul_rn(prm.f_rel, fabs(Jn))) || (prm.f_abs >= 0.0 && dJ <= prm.f_abs))
          res = kOptFtol;
        else if (xtol) res = kOptXtol;
        else keep = true;
      }
    }
  }
  const int q = append_row(keep, prm.count_next);
  if (p >= prm.rows) return;
  const double* __restrict__ x = prm.x + p * K;
  const double* __restrict__ g = prm.g + p * K;
  if (keep) {
    prm.idx_next[q] = int(b);
    prm.alpha_next[q] = step;
    for (int i = 0; i < K; ++i) prm.x_next[(long long)q * K + i] = line_search_time(x[i], g[i], step, prm.lower);
    for (int c = 0; c < prm.dnf; ++c) prm.dfix_next[(long long)q * prm.dnf + c] = prm.dfix[p * prm.dnf + c];
  } else {
    for (int i = 0; i < K; ++i) prm.rel[b * K + i] = acc >= 0 ? line_search_time(x[i], g[i], step, prm.lower) : x[i];
    prm.iters[b] = it;
    prm.result[b] = res;
  }
}

// The entry's per-row outputs after the final scaling.
__global__ void __launch_bounds__(128) mel_finish_kernel(long long B, const int* __restrict__ iters_in,
                                                         const int* __restrict__ result_in,
                                                         const int* __restrict__ opt_status,
                                                         const int* __restrict__ scale_status, int* __restrict__ iters,
                                                         int* __restrict__ result, int* __restrict__ status) {
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    if (iters) iters[b] = iters_in[b];
    if (result) result[b] = result_in[b];
    if (status) status[b] = (scale_status[b] & ~kStatusPassThrough) | opt_status[b];
  }
}

}  // namespace mtg
