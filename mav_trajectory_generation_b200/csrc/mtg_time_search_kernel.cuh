// mtg_time_search_kernel.cuh -- the per-row kernels of the compass search on the segment times
// (mtg_optimize_time_batch_f64: kSquaredTime / kRichterTime; the search is stated in include/mtg_b200.h).
//
// As in the Mellinger outer loop, the rows still iterating sit in a compact list: position p holds original row
// idx[p], its times x[p], its steps delta[p], its objective f[p] and its d_fixed.  Every poll expands the 2K
// candidates of each listed row, the objective launches evaluate them, and ts_decide_kernel decides each row, writes
// the finished ones to their original index and appends the others to the next list (append_row).  All listed rows
// have run the same number of polls, so the evaluation count is one number per poll, not per row.
#pragma once

#include "mtg_mellinger_loop_kernel.cuh"

namespace mtg {

struct TimeSearchParams {
  int K, dnf;  // segments; doubles of one row's d_fixed
  long long B;
  int max_iterations;  // objective evaluations (NLopt maxeval); < 0: no limit
  double f_abs, f_rel, x_rel, x_abs, init_rel, lower;
  int evals;  // evaluations of every listed row once this poll's candidates are counted
  // this launch's compact rows
  int rows;
  const int* __restrict__ idx;
  const double* __restrict__ x;      // [rows][K]
  const double* __restrict__ delta;  // [rows][K]
  const double* __restrict__ f;      // [rows] objective at x
  const double* __restrict__ dfix;   // [rows][dnf]
  const double* __restrict__ fc;     // [rows][2K] candidate objectives
  const int* __restrict__ st_c;      // [rows][2K] candidate statuses
  // the next poll's compact rows
  int* __restrict__ idx_next;
  double* __restrict__ x_next;
  double* __restrict__ delta_next;
  double* __restrict__ f_next;
  double* __restrict__ dfix_next;
  int* __restrict__ count_next;
  // per original row
  double* x_out;               // [B][K] (may be the caller's seg_times)
  int* __restrict__ evals_out;   // [B]
  int* __restrict__ result;      // [B]
  int* __restrict__ opt_status;  // [B] status bits met by the search
};

__device__ __forceinline__ double ts_clamp(double v, double lower) { return v > lower ? v : lower; }

// Candidate j of a row along its coordinate i = j / 2: x_i + delta_i (j even) or max(l, x_i - delta_i) (j odd).
__device__ __forceinline__ double ts_candidate(double x, double d, int j, double lower) {
  return (j & 1) ? ts_clamp(__dsub_rn(x, d), lower) : __dadd_rn(x, d);
}

// A poll runs only while it fits in max_iterations evaluations.
__device__ __forceinline__ bool ts_poll_fits(const TimeSearchParams& prm, int evals) {
  return prm.max_iterations < 0 || evals + 2 * prm.K <= prm.max_iterations;
}

// Start: copy seg_times to x_out, decide the rows that do not iterate, and list the others with their first steps.
// f0 / st0: the objective and its status at seg_times.
__global__ void __launch_bounds__(128) ts_init_kernel(const TimeSearchParams prm, const double* seg_times,
                                                      const double* __restrict__ f0, const int* __restrict__ st0,
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
      prm.x_out[b * K + i] = T;
    }
    int res = kOptFailure;
    if (!bad && !low && !(st0[b] & kStatusNotSpd)) {
      if (ts_poll_fits(prm, 1)) active = true;
      else res = kOptMaxeval;
    }
    prm.evals_out[b] = bad ? 0 : 1;
    prm.result[b] = res;
    prm.opt_status[b] = bad ? kStatusBadTime : 0;
  }
  const int p = append_row(active, prm.count_next);
  if (active) {
    const double rho = prm.init_rel > 0.0 ? prm.init_rel : 0.1;
    prm.idx_next[p] = int(b);
    prm.f_next[p] = f0[b];
    for (int i = 0; i < K; ++i) {
      const double T = seg_times[b * K + i];
      prm.x_next[(long long)p * K + i] = T;
      prm.delta_next[(long long)p * K + i] = __dmul_rn(rho, T);
    }
    for (int c = 0; c < prm.dnf; ++c) prm.dfix_next[(long long)p * prm.dnf + c] = dfix_in[b * prm.dnf + c];
  }
}

// The candidates of the listed rows: [rows * 2K] (times, d_fixed), candidate j of row p at q = p * 2K + j.
__global__ void __launch_bounds__(128) ts_expand_kernel(const TimeSearchParams prm, double* __restrict__ times_x,
                                                        double* __restrict__ dfix_x) {
  const int K = prm.K, dnf = prm.dnf, C = 2 * prm.K;
  const long long total = (long long)prm.rows * C;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += nthreads) {
    const long long p = q / C;
    const int j = int(q - p * C), ic = j >> 1;
    for (int i = 0; i < K; ++i) {
      const double x = prm.x[p * K + i];
      times_x[q * K + i] = i == ic ? ts_candidate(x, prm.delta[p * K + i], j, prm.lower) : x;
    }
    for (int c = 0; c < dnf; ++c) dfix_x[q * dnf + c] = prm.dfix[p * dnf + c];
  }
}

// One poll's decision for every listed row (steps 4 and 5 of mtg_optimize_time_batch_f64).
__global__ void __launch_bounds__(128) ts_decide_kernel(const TimeSearchParams prm) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int K = prm.K, C = 2 * prm.K;
  bool keep = false;
  long long b = 0;
  int res = 0, best = -1;
  double fn = 0.0;
  bool halve = false;
  if (p < prm.rows) {
    b = prm.idx[p];
    const double* __restrict__ x = prm.x + p * K;
    const double* __restrict__ d = prm.delta + p * K;
    const double f = prm.f[p];
    int st = 0;
    for (int j = 0; j < C; ++j) st |= prm.st_c[p * C + j];
    const bool xtol_on = prm.x_rel >= 0.0 || prm.x_abs >= 0.0;
    if (st & kStatusNotSpd) {
      res = kOptFailure;
      prm.opt_status[b] |= kStatusNotSpd;
    } else {
      // the smallest objective below f, the lowest j on a tie (a NaN never compares below)
      for (int j = 0; j < C; ++j) {
        const double v = prm.fc[p * C + j];
        if (v < f && (best < 0 || v < fn)) {
          best = j;
          fn = v;
        }
      }
      if (best >= 0) {
        const int ib = best >> 1;
        const double xn = ts_candidate(x[ib], d[ib], best, prm.lower);
        const double df = fabs(__dsub_rn(fn, f));
        bool xtol = xtol_on;
        for (int i = 0; i < K; ++i) {
          const double xi = i == ib ? xn : x[i];
          const double dx = fabs(__dsub_rn(xi, x[i]));
          xtol = xtol && ((prm.x_rel >= 0.0 && dx <= __dmul_rn(prm.x_rel, fabs(xi))) ||
                          (prm.x_abs >= 0.0 && dx <= prm.x_abs));
        }
        if ((prm.f_rel >= 0.0 && df <= __dmul_rn(prm.f_rel, fabs(fn))) || (prm.f_abs >= 0.0 && df <= prm.f_abs))
          res = kOptFtol;
        else if (xtol) res = kOptXtol;
        else keep = true;
      } else {
        halve = true;
        bool xtol = xtol_on, still = true;
        for (int i = 0; i < K; ++i) {
          const double dh = __dmul_rn(d[i], 0.5);
          xtol = xtol && ((prm.x_rel >= 0.0 && dh <= __dmul_rn(prm.x_rel, fabs(x[i]))) ||
                          (prm.x_abs >= 0.0 && dh <= prm.x_abs));
          still = still && __dadd_rn(x[i], dh) == x[i] && ts_clamp(__dsub_rn(x[i], dh), prm.lower) == x[i];
        }
        if (xtol) res = kOptXtol;
        else if (still) res = kOptRoundoff;
        else keep = true;
      }
      if (keep && !ts_poll_fits(prm, prm.evals)) {
        keep = false;
        res = kOptMaxeval;
      }
    }
  }
  const int q = append_row(keep, prm.count_next);
  if (p >= prm.rows) return;
  const double* __restrict__ x = prm.x + p * K;
  const double* __restrict__ d = prm.delta + p * K;
  const int ib = best >> 1;
  if (keep) {
    prm.idx_next[q] = int(b);
    prm.f_next[q] = best >= 0 ? fn : prm.f[p];
    for (int i = 0; i < K; ++i) {
      prm.x_next[(long long)q * K + i] = (best >= 0 && i == ib) ? ts_candidate(x[i], d[i], best, prm.lower) : x[i];
      prm.delta_next[(long long)q * K + i] = halve ? __dmul_rn(d[i], 0.5) : d[i];
    }
    for (int c = 0; c < prm.dnf; ++c) prm.dfix_next[(long long)q * prm.dnf + c] = prm.dfix[p * prm.dnf + c];
  } else {
    for (int i = 0; i < K; ++i)
      prm.x_out[b * K + i] = (best >= 0 && i == ib) ? ts_candidate(x[i], d[i], best, prm.lower) : x[i];
    prm.evals_out[b] = prm.evals;
    prm.result[b] = res;
  }
}

// The entry's per-row outputs; st_final is the status of the objective at the returned times.
__global__ void __launch_bounds__(128) ts_finish_kernel(long long B, const int* __restrict__ evals_in,
                                                        const int* __restrict__ result_in,
                                                        const int* __restrict__ opt_status,
                                                        const int* __restrict__ st_final, int* __restrict__ evals,
                                                        int* __restrict__ result, int* __restrict__ status) {
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    if (evals) evals[b] = evals_in[b];
    if (result) result[b] = result_in[b];
    if (status) status[b] = st_final[b] | opt_status[b];
  }
}

}  // namespace mtg
