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

template <int N, int R, int D>
__global__ void __launch_bounds__(32) twisted_solve_kernel(const WaypointParams prm) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  constexpr int kL = m * (m + 1) / 2;
  constexpr int kSlots = kL + m * D;
  constexpr unsigned kFull = 0xffffffffu;
  using G = H1<N, R>;

  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int half = lane & 1;  // 0: forward half (original frame), 1: time-reversed half
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;             // middle vertex (original index)
  const int nh = half ? K - M - 1 : M - 1;  // own number of eliminated vertices
  const int nmax = M - 1;                 // >= nh; state blocks allocated per lane
  double* st = smem + size_t(threadIdx.x >> 5) * size_t(nmax) * kSlots * 32 + lane;
  auto S = [&](int blk, int slot) -> double& { return st[(size_t(blk) * kSlots + slot) * 32]; };

  long long traj = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 16 + (lane >> 1);
  const bool valid = traj < prm.B;
  if (!valid) traj = prm.B - 1;

  const double* __restrict__ tt = prm.times + traj * K;
  const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
  // own-frame -> original index maps
  auto seg = [&](int j) -> int { return half ? K - 1 - j : j; };
  auto pidx = [&](int v) -> int {  // position slot of own-frame vertex v inside one dimension's d_fixed
    const int o = half ? K - v : v;
    return o == 0 ? 0 : (o < K ? h + o - 1 : h + K - 1);
  };
  // sign of derivative (idx+1) under time reversal
  auto sgn = [&](int idx) -> double { return (half && !(idx & 1)) ? -1.0 : 1.0; };

  int stat = 0;

  double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], bcar[m][D], xm[D], xc[D];
  double Tn;       // prefetched time of the next own-frame segment
  double xnn[D];   // prefetched position of own-frame vertex v+1 for the next iteration
  {
    const double T0 = __ldg(tt + seg(0));
    if (!(T0 > 0.0)) stat |= kStatusBadTime;
    const double iT0 = fast_rcp(T0);
    double pw[N - 1];
    segment_powers<N, R>(T0, iT0, pw);
    const int e0 = half ? h + K : 1;  // first fixed end-derivative slot of own-frame vertex 0
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b < m; ++b) {
        Cee[a][b] = pw[a + b + 2] * G::at(h + 1 + a, h + 1 + b);
        Wp[a][b] = 0.0;
      }
      cps[a] = pw[a + 1] * G::at(h + 1 + a, 0);
      cpe[a] = pw[a + 1] * G::at(h + 1 + a, h);
    }
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double u0[m];
#pragma unroll
      for (int b = 0; b < m; ++b) u0[b] = sgn(b) * __ldg(fx + d * nf + e0 + b);
#pragma unroll
      for (int a = 0; a < m; ++a) {
        double acc = 0.0;
#pragma unroll
        for (int b = 0; b < m; ++b) acc = fma(pw[a + b + 2] * G::at(h + 1 + a, 1 + b), u0[b], acc);
        bcar[a][d] = -acc;
        yp[a][d] = 0.0;
      }
      xm[d] = __ldg(fx + d * nf + pidx(0));
      xc[d] = __ldg(fx + d * nf + pidx(1));
    }
    // prefetch for iteration 1 (always in range: segment 1 and vertex 2 exist because K >= 2;
    // for K == 2 vertex 2 is the far end, harmless)
    Tn = __ldg(tt + seg(K > 1 ? 1 : 0));
    const int p2 = pidx(K >= 2 ? 2 : 1);
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
        Tn = __ldg(tt + seg(jn));
        const int pn = pidx(vn);
#pragma unroll
        for (int d = 0; d < D; ++d) xnn[d] = __ldg(fx + d * nf + pn);
      }
      if (!(T > 0.0)) stat |= kStatusBadTime;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);

      double Dp[m][m], E[m][m], bb[m][D];
#pragma unroll
      for (int a = 0; a < m; ++a) {
#pragma unroll
        for (int b = 0; b <= a; ++b) {
          double s = fma(pw[a + b + 2], G::at(1 + a, 1 + b), Cee[a][b]);
#pragma unroll
          for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], Wp[k][b], s);
          Dp[a][b] = s;
        }
#pragma unroll
        for (int b = 0; b < m; ++b) E[a][b] = pw[a + b + 2] * G::at(1 + a, h + 1 + b);
        const double gmid = fma(pw[a + 1], G::at(1 + a, 0), cpe[a]);
        const double gnext = pw[a + 1] * G::at(1 + a, h);
#pragma unroll
        for (int d = 0; d < D; ++d) {
          double s = bcar[a][d];
          s = fma(-cps[a], xm[d], s);
          s = fma(-gmid, xc[d], s);
          s = fma(-gnext, xn[d], s);
#pragma unroll
          for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
          bb[a][d] = s;
        }
      }
      double L[m][m], inv[m];
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = Dp[j][j];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], L[j][k], s);
        if (!(s > 0.0)) stat |= kStatusNotSpd;
        inv[j] = fast_rsqrt(s);
#pragma unroll
        for (int i = j + 1; i < m; ++i) {
          double t = Dp[i][j];
#pragma unroll
          for (int k = 0; k < j; ++k) t = fma(-L[i][k], L[j][k], t);
          L[i][j] = t * inv[j];
        }
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
#pragma unroll
        for (int j = 0; j < m; ++j) {
          double s = bb[j][d];
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-L[j][k], yp[k][d], s);
          yp[j][d] = s * inv[j];
        }
      }
#pragma unroll
      for (int c = 0; c < m; ++c) {
#pragma unroll
        for (int j = 0; j < m; ++j) {
          double s = E[j][c];
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-L[j][k], Wp[k][c], s);
          Wp[j][c] = s * inv[j];
        }
      }
      {
        int slot = 0;
#pragma unroll
        for (int i = 1; i < m; ++i)
#pragma unroll
          for (int j = 0; j < i; ++j) S(v - 1, slot++) = L[i][j];
#pragma unroll
        for (int j = 0; j < m; ++j) S(v - 1, slot++) = inv[j];
#pragma unroll
        for (int j = 0; j < m; ++j)
#pragma unroll
          for (int d = 0; d < D; ++d) S(v - 1, slot++) = yp[j][d];
      }
#pragma unroll
      for (int a = 0; a < m; ++a) {
#pragma unroll
        for (int b = 0; b <= a; ++b) Cee[a][b] = pw[a + b + 2] * G::at(h + 1 + a, h + 1 + b);
        cps[a] = pw[a + 1] * G::at(h + 1 + a, 0);
        cpe[a] = pw[a + 1] * G::at(h + 1 + a, h);
#pragma unroll
        for (int d = 0; d < D; ++d) bcar[a][d] = 0.0;
      }
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
  {
    double Dl[m][m], bl[m][D];
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        double s = Cee[a][b];
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], Wp[k][b], s);
        Dl[a][b] = s;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double s = bcar[a][d];
        s = fma(-cps[a], xm[d], s);
        s = fma(-cpe[a], xc[d], s);
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
        bl[a][d] = s;
      }
    }
    // exchange with the partner lane and combine: X_own + J X_partner J  (J = diag((-1)^k))
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        const double o = __shfl_xor_sync(kFull, Dl[a][b], 1);
        Dl[a][b] += ((a + b) & 1) ? -o : o;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const double o = __shfl_xor_sync(kFull, bl[a][d], 1);
        bl[a][d] += (a & 1) ? o : -o;  // derivative order a+1: sign (-1)^(a+1)
      }
    }
    stat |= __shfl_xor_sync(kFull, stat, 1);
    double L[m][m], inv[m];
#pragma unroll
    for (int j = 0; j < m; ++j) {
      double s = Dl[j][j];
#pragma unroll
      for (int k = 0; k < j; ++k) s = fma(-L[j][k], L[j][k], s);
      if (!(s > 0.0)) stat |= kStatusNotSpd;
      inv[j] = fast_rsqrt(s);
#pragma unroll
      for (int i = j + 1; i < m; ++i) {
        double t = Dl[i][j];
#pragma unroll
        for (int k = 0; k < j; ++k) t = fma(-L[i][k], L[j][k], t);
        L[i][j] = t * inv[j];
      }
    }
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double y[m];
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = bl[j][d];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], y[k], s);
        y[j] = s * inv[j];
      }
#pragma unroll
      for (int j = m - 1; j >= 0; --j) {
        double s = y[j];
#pragma unroll
        for (int k = j + 1; k < m; ++k) s = fma(-L[k][j], um[k][d], s);
        um[j][d] = s * inv[j];
      }
    }
  }
  if (valid && half == 0 && prm.status != nullptr) prm.status[traj] = stat;

  // ---------------------------------------------------------------- outward back-substitution
  double* __restrict__ out = prm.coeffs + traj * (long long)K * D * N;
  const int np = (K - 1) * m;
  double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + traj * (long long)D * np : nullptr;
  auto store_free = [&](int v_own, const double (&u)[h][D]) {  // u[1+j][d]: own-frame derivatives
    if (df != nullptr && valid) {
      const int vo = half ? K - v_own : v_own;
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int j = 0; j < m; ++j) df[d * np + (vo - 1) * m + j] = sgn(j) * u[1 + j][d];
    }
  };
  // emit own-frame segment j (start derivatives sd at own vertex j, end derivatives ed at j+1).
  // For the reversed half the ORIGINAL segment starts at own vertex j+1: start = J ed, end = J sd.
  // The swap is a select per value (no divergent code path); J is folded into the time powers.
  auto emit = [&](int j, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D]) {
    double* __restrict__ o = out + (long long)seg(j) * D * N;
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
  double Tb = __ldg(tt + seg(nh));  // nh == 0: segment 0, used by the final emission
  double xb[D];
#pragma unroll
  for (int d = 0; d < D; ++d) xb[d] = __ldg(fx + d * nf + pidx(nh));

  for (int v = nmax; v >= 1; --v) {
    if (v <= nh) {
      const double T = Tb;
      double xv[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xv[d] = xb[d];
      Tb = __ldg(tt + seg(v - 1));
      {
        const int pn = pidx(v - 1);
#pragma unroll
        for (int d = 0; d < D; ++d) xb[d] = __ldg(fx + d * nf + pn);
      }
      const double iT = fast_rcp(T);
      double L[m][m], inv[m], rhs[m][D];
      {
        int slot = 0;
#pragma unroll
        for (int i = 1; i < m; ++i)
#pragma unroll
          for (int j = 0; j < i; ++j) L[i][j] = S(v - 1, slot++);
#pragma unroll
        for (int j = 0; j < m; ++j) inv[j] = S(v - 1, slot++);
#pragma unroll
        for (int j = 0; j < m; ++j)
#pragma unroll
          for (int d = 0; d < D; ++d) rhs[j][d] = S(v - 1, slot++);
      }
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double t[m];
#pragma unroll
        for (int a = 0; a < m; ++a) {
          double s = 0.0;
#pragma unroll
          for (int b = 0; b < m; ++b) s = fma(pw[a + b + 2] * G::at(1 + a, h + 1 + b), ed[1 + b][d], s);
          t[a] = s;
        }
#pragma unroll
        for (int j = 0; j < m; ++j) {
          double s = t[j];
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-L[j][k], t[k], s);
          t[j] = s * inv[j];
          rhs[j][d] -= t[j];
        }
      }
      double sd[h][D];
#pragma unroll
      for (int d = 0; d < D; ++d) {
#pragma unroll
        for (int j = m - 1; j >= 0; --j) {
          double s = rhs[j][d];
#pragma unroll
          for (int k = j + 1; k < m; ++k) s = fma(-L[k][j], sd[1 + k][d], s);
          sd[1 + j][d] = s * inv[j];
        }
        sd[0][d] = xv[d];
      }
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
    const int e0 = half ? h + K : 1;
    double sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      sd[0][d] = xb[d];
#pragma unroll
      for (int b = 0; b < m; ++b) sd[1 + b][d] = sgn(b) * __ldg(fx + d * nf + e0 + b);
    }
    emit(0, T, iT, sd, ed);
  }
}

}  // namespace mtg
