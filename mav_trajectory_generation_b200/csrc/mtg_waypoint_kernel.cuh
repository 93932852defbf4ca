// mtg_waypoint_kernel.cuh -- K1: fused assemble + factor + solve + back-substitute,
// ONE THREAD PER TRAJECTORY, for the createRandomVertices ("waypoint") topology
// (reference fixture: src/vertex.cpp:27-82): first/last vertex fix derivatives 0..h-1,
// interior vertices fix position only.
//
// Replaces, per trajectory, the reference's
//   updateSegmentTimes()   impl/polynomial_optimization_linear_impl.h:285-305
//   constructR()           :307-336
//   solveLinear()          :338-379   (SparseQR on R_pp -> block-tridiagonal Cholesky)
//   updateSegmentsFromCompactConstraints() :262-283
//
// Mathematics (SURVEY.md appendix B).  h = N/2, m = h-1.  Unknowns: u_v in R^m (derivatives
// 1..m at interior vertex v = 1..K-1), shared by all D dimensions.  R_pp is block
// tridiagonal with m x m blocks:
//   D_v = H_{v-1}[end,end] + H_v[start,start],   E_v = H_v[start,end]   (couples u_v,u_{v+1})
//   b_v = -(H_{v-1}[end,p_s] x_{v-1} + (H_{v-1}[end,p_e] + H_v[start,p_s]) x_v + H_v[start,p_e] x_{v+1})
//         - [v==1] H_0[end,start] u_0  - [v==K-1] E_{K-1} u_K         (u_0, u_K fixed end derivatives)
// with H_i = T_i^(1-2r) S_i H(1) S_i from the exact table.  Forward sweep (block Cholesky):
//   D'_v = D_v - W_{v-1}^T W_{v-1},  L_v = chol(D'_v),  y_v = L_v^-1 (b_v - W_{v-1}^T y_{v-1}),
//   W_v = L_v^-1 E_v
// Backward sweep:  u_v = L_v^-T (y_v - L_v^-1 (E_v u_{v+1})), and as soon as u_v, u_{v+1} are
// known the segment's coefficients p = diag(T^-j) A(1)^-1 diag(T^(s mod h)) d are emitted.
//
// Data layout.  Inputs per trajectory: seg_times[K], d_fixed[D][n_fixed] (reference compact
// order: x_0,u_0(1..m), x_1..x_{K-1}, x_K,u_K(1..m)).  Output coeffs[K][D][N].
// Per-thread sweep state (L_v: m(m+1)/2 doubles, y_v: m*D doubles per interior vertex) lives
// in SHARED memory laid out [vertex][slot][lane] so every access is bank-conflict free
// (consecutive lanes -> consecutive 8-byte words).
#pragma once

#include "mtg_sweep.cuh"

namespace mtg {

struct WaypointParams {
  int K;
  int n_fixed;
  long long B;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ dfix;    // [B][D][n_fixed]
  double* __restrict__ coeffs;        // [B][K][D][N]
  double* __restrict__ dfree;         // [B][D][(K-1)*m] or null
  int* __restrict__ status;           // [B] or null
  // fused time allocation + constraint packing (SURVEY.md 8f-1): when `positions` is set the kernels
  // read waypoints [B][K+1][D] instead of (times, dfix), compute the segment times with
  // estimateSegmentTimesNfabian (reference src/vertex.cpp:255-272) and use zero start/end derivatives
  // (Vertex::makeStartOrEnd, src/vertex.cpp:147-153).
  // The line-search instantiation of the cost-only mode (below) reads its step and gradient pointers in the places of
  // the fused inputs' pointers, which it never reads: the parameter block of every kernel keeps its size.
  union {
    const double* __restrict__ positions;
    const double* __restrict__ ls_grad;   // [rows][K]
  };
  double v_max, a_max, magic;
  union {
    double* __restrict__ times_out;     // [B][K] or null
    const double* __restrict__ ls_alpha;  // [rows]
  };
  // cost-only mode (SURVEY.md 8f-2, the nonlinear optimiser's inner loop): no coefficients are written; the
  // kernel returns computeCost() of every problem.  With mel_k1 = K+1 the batch is the Mellinger expansion
  // (reference impl/polynomial_optimization_nonlinear_impl.h:286-364) generated on the fly: problem q belongs to
  // trajectory q / (K+1); variant n = q % (K+1) - 1 (n = -1: unperturbed) adds mel_inc to segment n, subtracts
  // mel_inc / (K-1) from the others and clamps at mel_lower -- `times` / `dfix` are the UNEXPANDED arrays.
  double* __restrict__ cost;          // [B] or null
  int mel_k1;
  double mel_inc, mel_lower;
  // cost-only mode, line-search instantiation (the Mellinger outer loop's candidates): problem q is candidate
  // j = q % kLineSearchSteps of row q / kLineSearchSteps, at line_search_time(x, g, line_search_step(alpha, j),
  // mel_lower) per segment, where x = `times`, g = ls_grad and alpha = ls_alpha are the UNEXPANDED rows.
};

__device__ __forceinline__ double mellinger_time(double t, int i, int n, double inc, double corr, double lower) {
  if (n < 0) return t;
  const double v = (i == n) ? t + inc : t - corr;
  return v > lower ? v : lower;  // std::max(kOptimizationTimeLowerBound, t)
}

// Step sizes tried per row and iteration by the Mellinger outer loop: alpha * 2^(1 - j), j = 0..kLineSearchSteps-1
constexpr int kLineSearchSteps = 8;
__device__ __forceinline__ double line_search_step(double alpha, int j) { return __dmul_rn(alpha, ldexp(1.0, 1 - j)); }
// max(lower, fl(x - fl(step * g))): two roundings (no FMA), the same max form as mellinger_time
__device__ __forceinline__ double line_search_time(double x, double g, double step, double lower) {
  const double v = __dsub_rn(x, __dmul_rn(step, g));
  return v > lower ? v : lower;
}

// t = distance / v_max * 2 * (1 + magic * v_max / a_max * exp(-distance / v_max * 2)), evaluated in the
// reference's order with no FMA contraction (the CPU oracle is built with -ffp-contract=off).
template <int D>
__device__ __forceinline__ double nfabian_time(const double (&a)[D], const double (&b)[D], double v_max, double a_max,
                                               double magic) {
  double n2 = 0.0;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const double e = __dsub_rn(b[d], a[d]);
    n2 = __dadd_rn(n2, __dmul_rn(e, e));
  }
  const double distance = sqrt(n2);
  const double lead = __dmul_rn(__ddiv_rn(distance, v_max), 2.0);
  const double ex = exp(__dmul_rn(__ddiv_rn(-distance, v_max), 2.0));
  const double fac = __dadd_rn(1.0, __dmul_rn(__ddiv_rn(__dmul_rn(magic, v_max), a_max), ex));
  return __dmul_rn(lead, fac);
}

// Emit the N coefficients of every dimension of one segment.
//   sd[k][d], ed[k][d]: derivative k (0..m) at the segment start / end.
// p_j = T^-j * sum_s A1inv[j][s] * T^(s mod h) * d_s ; for j < h this is d_j / j! exactly as the
// reference computes it (A^-1 is diagonal there, linear_impl.h:173).
// `flip`: the derivative values are given in the time-reversed sign convention (derivative k carries
// (-1)^k); the sign is folded into the time powers (and the 1/k! factors) instead of the data.
template <int N, int D>
__device__ __forceinline__ void emit_segment(double T, double invT, const double (&sd)[N / 2][D],
                                             const double (&ed)[N / 2][D], double* __restrict__ out,
                                             bool valid, bool flip = false) {
  constexpr int h = N / 2;
  double tp[h];     // T^k (times (-1)^k when flip)
  double itp[h];    // T^-(h+j)
  const double Ts = flip ? -T : T;
  tp[0] = 1.0;
#pragma unroll
  for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * Ts;
  itp[0] = pow_int<h>(invT);
#pragma unroll
  for (int j = 1; j < h; ++j) itp[j] = itp[j - 1] * invT;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    double c[N];
    double ss[h], se[h];
#pragma unroll
    for (int k = 0; k < h; ++k) {
      c[k] = sd[k][d] * ((flip && (k & 1)) ? -A1Inv<N>::at(k, k) : A1Inv<N>::at(k, k));
      ss[k] = tp[k] * sd[k][d];
      se[k] = tp[k] * ed[k][d];
    }
#pragma unroll
    for (int j = 0; j < h; ++j) {
      double acc = A1Inv<N>::at(h + j, 0) * ss[0];
#pragma unroll
      for (int k = 1; k < h; ++k) acc = fma(A1Inv<N>::at(h + j, k), ss[k], acc);
#pragma unroll
      for (int k = 0; k < h; ++k) acc = fma(A1Inv<N>::at(h + j, h + k), se[k], acc);
      c[h + j] = acc * itp[j];
    }
    if (valid) {
      // N is even and out is 16-byte aligned (K*D*N*8 and D*N*8 are multiples of 16).
      double2* o2 = reinterpret_cast<double2*>(out + d * N);
#pragma unroll
      for (int j = 0; j < N / 2; ++j) o2[j] = make_double2(c[2 * j], c[2 * j + 1]);
    }
  }
}

// Dynamic shared memory of v1 for a 32-thread CTA: the sweep state of the K-1 interior vertices, [vertex][slot][lane]
template <int N, int D>
struct V1Layout {
  __host__ __device__ static constexpr size_t bytes(int K) {
    return size_t(K - 1) * sweep_state_slots<N, D>() * 32 * sizeof(double);
  }
};

template <int N, int R, int D>
__global__ void __launch_bounds__(32) waypoint_solve_kernel(const WaypointParams prm) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  constexpr int kSlots = sweep_state_slots<N, D>();
  using G = H1<N, R>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  double* st = smem + size_t(threadIdx.x >> 5) * size_t(prm.K - 1) * kSlots * 32 + lane;
  auto SP = [&](int blk, int slot) -> double& { return st[(size_t(blk) * kSlots + slot) * 32]; };

  const int K = prm.K;
  const int nf = prm.n_fixed;
  long long traj = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = traj < prm.B;
  if (!valid) traj = prm.B - 1;  // duplicate work, no stores: keeps the warp convergent

  const double* __restrict__ tt = prm.times + traj * K;
  const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
  // index of the position of vertex v inside one dimension's d_fixed
  auto pidx = [&](int v) -> int { return v == 0 ? 0 : (v < K ? h + v - 1 : h + K - 1); };

  int stat = 0;

  // ---------------------------------------------------------------- forward sweep
  double Wp[m][m];   // W_{v-1} (row k, column a)
  double yp[m][D];   // y_{v-1}
  double Cee[m][m];  // H_{v-1}[end,end] (lower part used)
  double cps[m], cpe[m];  // H_{v-1}[end, p_start], H_{v-1}[end, p_end]
  double bcar[m][D];      // -H_0[end,start] u_0, only non-zero for v == 1
  double xm[D], xc[D];
  {
    const double T0 = __ldg(tt);
    if (bad_segment_time(T0)) stat |= kStatusBadTime;
    const double iT0 = fast_rcp(T0);
    double pw[N - 1];
    segment_powers<N, R>(T0, iT0, pw);
    S::end_blocks(pw, Cee, cps, cpe);
    S::carry_bcar(pw, [&](int b, int d) { return __ldg(fx + d * nf + 1 + b); }, Wp, yp, bcar);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      xm[d] = __ldg(fx + d * nf);
      xc[d] = __ldg(fx + d * nf + pidx(1));
    }
  }

  for (int v = 1; v < K; ++v) {
    const double T = __ldg(tt + v);
    if (bad_segment_time(T)) stat |= kStatusBadTime;
    const double iT = fast_rcp(T);
    double pw[N - 1];
    segment_powers<N, R>(T, iT, pw);
    double xn[D];
    const int pn = pidx(v + 1);
#pragma unroll
    for (int d = 0; d < D; ++d) xn[d] = __ldg(fx + d * nf + pn);

    double Dp[m][m], E[m][m], bb[m][D];
    S::assemble(pw, Cee, cps, cpe, bcar, Wp, yp, xm, xc, xn, Dp, E, bb);
    if (v == K - 1) {  // last interior vertex: coupling to the fixed end derivatives u_K
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double uK[m];
#pragma unroll
        for (int b = 0; b < m; ++b) uK[b] = __ldg(fx + d * nf + h + K + b);
#pragma unroll
        for (int a = 0; a < m; ++a) {
          double s = bb[a][d];
#pragma unroll
          for (int b = 0; b < m; ++b) s = fma(-E[a][b], uK[b], s);
          bb[a][d] = s;
        }
      }
    }

    double L[m][m], inv[m], sv[kSlots];
    S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
    S::pack(L, inv, yp, nullptr, sv);
#pragma unroll
    for (int i = 0; i < kSlots; ++i) SP(v - 1, i) = sv[i];
    // carry the end-side blocks of segment v to the next vertex
    S::end_blocks(pw, Cee, cps, cpe);
#pragma unroll
    for (int a = 0; a < m; ++a)
#pragma unroll
      for (int d = 0; d < D; ++d) bcar[a][d] = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      xm[d] = xc[d];
      xc[d] = xn[d];
    }
  }

  if (valid && prm.status != nullptr) prm.status[traj] = stat;

  // ---------------------------------------------------------------- backward sweep + emission
  double* __restrict__ out = prm.coeffs + traj * (long long)K * D * N;
  const int np = (K - 1) * m;
  double ed[h][D];  // derivatives 0..m at the END of the segment being emitted
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ed[0][d] = xc[d];  // x_K (left in xc by the forward sweep)
#pragma unroll
    for (int b = 0; b < m; ++b) ed[1 + b][d] = __ldg(fx + d * nf + h + K + b);
  }

  for (int v = K - 1; v >= 1; --v) {
    const double T = __ldg(tt + v);
    const double iT = fast_rcp(T);
    double sv[kSlots], L[m][m], inv[m], rhs[m][D];
#pragma unroll
    for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - 1, i);
    S::unpack(sv, L, inv, rhs);
    if (v < K - 1) {  // the last interior vertex's coupling to u_K is already in its right-hand side
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);
      S::uncouple_from(pw, ed, L, inv, rhs);
    }
    double xv[D], sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) xv[d] = __ldg(fx + d * nf + pidx(v));
    S::solve_back(L, inv, rhs, xv, sd);
    if (prm.dfree != nullptr && valid) {
      double* __restrict__ df = prm.dfree + traj * (long long)D * np;
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int j = 0; j < m; ++j) df[d * np + (v - 1) * m + j] = sd[1 + j][d];
    }
    emit_segment<N, D>(T, iT, sd, ed, out + (long long)v * D * N, valid);
#pragma unroll
    for (int d = 0; d < D; ++d)
#pragma unroll
      for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
  }
  {
    const double T = __ldg(tt);
    const double iT = fast_rcp(T);
    double sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d)
#pragma unroll
      for (int k = 0; k < h; ++k) sd[k][d] = __ldg(fx + d * nf + k);
    emit_segment<N, D>(T, iT, sd, ed, out, valid);
  }
}

}  // namespace mtg
