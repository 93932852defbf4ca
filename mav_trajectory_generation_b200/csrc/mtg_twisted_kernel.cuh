// mtg_twisted_kernel.cuh -- K1 (v2): TWO LANES PER TRAJECTORY, twisted ("burn at both ends")
// block-tridiagonal Cholesky for the waypoint topology.
//
// Same mathematics as mtg_waypoint_kernel.cuh, but the K-1 interior vertices are eliminated from
// BOTH ends at once: the even lane of a pair sweeps vertices 1..M-1 forward, the odd lane sweeps
// vertices K-1..M+1 backward, M = (K+1)/2.  The odd lane works in the TIME-REVERSED frame
// (segments and vertices reversed, derivative k scaled by (-1)^k), in which its sweep is again a
// forward sweep -- so both lanes run the SAME code on different index maps.  The two partial
// Schur complements meet at vertex M: each lane sends its half (m(m+1)/2 + m*D doubles) to the
// partner with warp shuffles, both factor the middle block (redundantly, ~3 % extra flops) and
// then back-substitute their own half outward, emitting the coefficients of their own segments.
// Versus one thread per trajectory this halves the serial dependency chain and the per-thread
// sweep state at an identical flop count, which is what the latency-bound C3 shape needs.
//
// Per-lane sweep state (L_v, inverse pivots, y_v of its M-1 vertices) is in shared memory,
// [vertex][slot][lane] (bank-conflict free).
#pragma once

#include "mtg_waypoint_kernel.cuh"

namespace mtg {

// Dynamic shared memory of v2 for a 32-thread CTA: the sweep state of each lane's (K+1)/2-1 vertices,
// [vertex][slot][lane]
template <int N, int D>
struct V2Layout {
  __host__ __device__ static constexpr size_t bytes(int K) {
    return size_t((K + 1) / 2 - 1) * sweep_state_slots<N, D>() * 32 * sizeof(double);
  }
};

template <int N, int R, int D>
__global__ void __launch_bounds__(32) twisted_solve_kernel(const WaypointParams prm) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  constexpr int kSlots = sweep_state_slots<N, D>();
  using G = H1<N, R>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int half = lane & 1;  // 0: forward half (original frame), 1: time-reversed half
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;             // middle vertex (original index)
  const int nh = half ? K - M - 1 : M - 1;  // own number of eliminated vertices
  const int nmax = M - 1;                 // >= nh; state blocks allocated per lane
  double* st = smem + size_t(threadIdx.x >> 5) * size_t(nmax) * kSlots * 32 + lane;
  auto SP = [&](int blk, int slot) -> double& { return st[(size_t(blk) * kSlots + slot) * 32]; };

  long long traj = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 16 + (lane >> 1);
  const bool valid = traj < prm.B;
  if (!valid) traj = prm.B - 1;

  const double* __restrict__ tt = prm.times + traj * K;
  const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
  const sweep::Frame<N> fr{K, half};  // own-frame -> original index maps

  int stat = 0;

  double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], bcar[m][D], xm[D], xc[D];
  double Tn;       // prefetched time of the next own-frame segment
  double xnn[D];   // prefetched position of own-frame vertex v+1 for the next iteration
  {
    const double T0 = __ldg(tt + fr.seg(0));
    if (bad_segment_time(T0)) stat |= kStatusBadTime;
    const double iT0 = fast_rcp(T0);
    double pw[N - 1];
    segment_powers<N, R>(T0, iT0, pw);
    S::end_blocks(pw, Cee, cps, cpe);
    S::carry_bcar(pw, [&](int b, int d) { return fr.sgn(b) * __ldg(fx + d * nf + fr.e0() + b); }, Wp, yp, bcar);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      xm[d] = __ldg(fx + d * nf + fr.pidx(0));
      xc[d] = __ldg(fx + d * nf + fr.pidx(1));
    }
    // prefetch for iteration 1 (always in range: segment 1 and vertex 2 exist because K >= 2;
    // for K == 2 vertex 2 is the far end, harmless)
    Tn = __ldg(tt + fr.seg(K > 1 ? 1 : 0));
    const int p2 = fr.pidx(K >= 2 ? 2 : 1);
#pragma unroll
    for (int d = 0; d < D; ++d) xnn[d] = __ldg(fx + d * nf + p2);
  }

  // ---------------------------------------------------------------- sweep towards the middle
  for (int v = 1; v <= nmax; ++v) {
    if (v <= nh) {
      const double T = Tn;
      double xn[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xn[d] = xnn[d];
      {  // prefetch the next iteration's inputs (clamped indices: never out of bounds)
        const int jn = v + 1 < K ? v + 1 : K - 1;
        const int vn = v + 2 <= K ? v + 2 : K;
        Tn = __ldg(tt + fr.seg(jn));
        const int pn = fr.pidx(vn);
#pragma unroll
        for (int d = 0; d < D; ++d) xnn[d] = __ldg(fx + d * nf + pn);
      }
      if (bad_segment_time(T)) stat |= kStatusBadTime;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);

      double Dp[m][m], E[m][m], bb[m][D], L[m][m], inv[m], sv[kSlots];
      S::assemble(pw, Cee, cps, cpe, bcar, Wp, yp, xm, xc, xn, Dp, E, bb);
      S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
      S::pack(L, inv, yp, nullptr, sv);
#pragma unroll
      for (int i = 0; i < kSlots; ++i) SP(v - 1, i) = sv[i];
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
  }
  __syncwarp();

  // ---------------------------------------------------------------- middle vertex (own-frame nh+1)
  // own half of the Schur complement and right-hand side; xc is the middle position.
  double um[m][D];  // solution at the middle vertex, own frame
  S::middle(Cee, cps, cpe, bcar, Wp, yp, xm, xc, um, stat);
  if (valid && half == 0 && prm.status != nullptr) prm.status[traj] = stat;

  // ---------------------------------------------------------------- outward back-substitution
  double* __restrict__ out = prm.coeffs + traj * (long long)K * D * N;
  const sweep::FreeStore<N, D> store_free(prm.dfree, traj, valid, fr);
  // emit own-frame segment j (start derivatives sd at own vertex j, end derivatives ed at j+1).
  // For the reversed half the ORIGINAL segment starts at own vertex j+1: start = J ed, end = J sd.
  // The swap is a select per value (no divergent code path); J is folded into the time powers.
  auto emit = [&](int j, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D]) {
    double* __restrict__ o = out + (long long)fr.seg(j) * D * N;
    double s2[h][D], e2[h][D];
#pragma unroll
    for (int k = 0; k < h; ++k)
#pragma unroll
      for (int d = 0; d < D; ++d) {
        s2[k][d] = half ? ed[k][d] : sd[k][d];
        e2[k][d] = half ? sd[k][d] : ed[k][d];
      }
    emit_segment<N, D>(T, iT, s2, e2, o, valid, half != 0);
  };

  double ed[h][D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ed[0][d] = xc[d];
#pragma unroll
    for (int j = 0; j < m; ++j) ed[1 + j][d] = um[j][d];
  }
  if (half == 0) store_free(nh + 1, ed);

  // prefetched inputs of the next outward step: time of own segment v, position of own vertex v
  double Tb = __ldg(tt + fr.seg(nh));  // nh == 0: segment 0, used by the final emission
  double xb[D];
#pragma unroll
  for (int d = 0; d < D; ++d) xb[d] = __ldg(fx + d * nf + fr.pidx(nh));

  for (int v = nmax; v >= 1; --v) {
    if (v <= nh) {
      const double T = Tb;
      double xv[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xv[d] = xb[d];
      Tb = __ldg(tt + fr.seg(v - 1));
      {
        const int pn = fr.pidx(v - 1);
#pragma unroll
        for (int d = 0; d < D; ++d) xb[d] = __ldg(fx + d * nf + pn);
      }
      const double iT = fast_rcp(T);
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - 1, i);
      double L[m][m], inv[m], rhs[m][D], pw[N - 1], sd[h][D];
      S::unpack(sv, L, inv, rhs);
      segment_powers<N, R>(T, iT, pw);
      S::uncouple_from(pw, ed, L, inv, rhs);
      S::solve_back(L, inv, rhs, xv, sd);
      store_free(v, sd);
      emit(v, T, iT, sd, ed);
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
    }
  }
  {
    const double T = Tb;
    const double iT = fast_rcp(T);
    double sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      sd[0][d] = xb[d];
#pragma unroll
      for (int b = 0; b < m; ++b) sd[1 + b][d] = fr.sgn(b) * __ldg(fx + d * nf + fr.e0() + b);
    }
    emit(0, T, iT, sd, ed);
  }
}

}  // namespace mtg
