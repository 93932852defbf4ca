// mtg_twisted_chunked_kernel.cuh -- K3: the twisted two-lane sweep for ANY number of segments, with a fixed
// on-chip footprint (large-K kernel; the reference's own timing program runs K = 50 and K = 100,
// src/polynomial_timing_evaluation.cpp:114-129, its test-suite K = 50, test/test_polynomial_optimization.cpp:822-828).
//
// The resident kernels keep the factor of every eliminated vertex in shared memory, which caps the number of
// trajectories in flight per SM as K grows (25 doubles per lane and eliminated vertex at N = 10, D = 3).  Here
// only a CHUNK of C vertex blocks per lane is ever resident -- the host picks C for the most resident CTAs per
// SM -- and the rest is RECOMPUTED (checkpointing):
//
//   round 0   forward sweep over all own vertices 1..n (n = ceil(K/2)-1); only the innermost chunk (n-C, n] is
//             stored; the loop-carried state (W, y: m*m + m*D doubles) is checkpointed to global memory at the
//             start of every other chunk; middle vertex; back-substitution + emission over the innermost chunk;
//   round j   (j = 1 .. nc-1, moving outwards) reload the checkpoint at the chunk's start, re-run the forward
//             sweep over its <= C vertices storing their blocks on chip, back-substitute and emit them.
//
// Cost: the forward sweep runs (2n - C)/n times (1.35x of all FP64 work at K = 50, 1.43x at K = 100); extra HBM
// traffic 2 * (nc-1) * (m*m + m*D) * 8 bytes per lane for the checkpoints (+24 % at K = 100) and one re-read of
// the inputs -- against 2.2x the algorithmic traffic if the whole factor were spilled to HBM.
// CTAs are persistent (static tile assignment) so that the checkpoint area is bounded by the number of resident
// threads, not by the batch.  Arithmetic per vertex is exactly the v3/v4 sequence: results are bitwise equal to
// the resident kernels where both run (tests force tiny chunks on K = 16 to prove it).
#pragma once

#include "mtg_twisted_tmem_v4_kernel.cuh"

namespace mtg {

struct ChunkedLaunch {
  int chunk;          // C: vertex blocks resident per lane (in shared memory)
  double* ckpt;       // [(nc-1)][m*m + m*D][gridDim.x * 128] loop-carried state at chunk starts
};

template <int N, int D>
__host__ __device__ constexpr int chunked_ckpt_slots() {
  return (N / 2 - 1) * (N / 2 - 1) + (N / 2 - 1) * D;
}
// dynamic shared memory: [staging][ring RD x (1+D)][times C+1][stash D+1][restart 1+2D][state blocks]
template <int N, int D, int RD>
__host__ __device__ constexpr size_t chunked_smem_bytes(int C) {
  return size_t(kTmemThreads / 32) * tmem_stage_bytes_per_warp<N, D>() +
         size_t(RD * (1 + D) + (C + 1) + (D + 1) + (1 + 2 * D) + C * v4_state_slots<N, D>()) * kTmemThreads * 8;
}

template <int N, int R, int D, int RD>
__global__ void __launch_bounds__(kTmemThreads, 2)
    twisted_chunked_kernel(const WaypointParams prm, const ChunkedLaunch cl, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  constexpr int kL = m * (m + 1) / 2;
  constexpr int kSlots = kL + m * D + D;
  constexpr int kCk = chunked_ckpt_slots<N, D>();
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = kTmemThreads / 32;
  constexpr double kTiny = 0x1p-600, kHuge = 0x1p+600;
  using G = H1Imm<N, R>;
  using AI = A1InvImm<N>;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int half = lane & 1;
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;
  const int nh = half ? K - M - 1 : M - 1;
  const int n = M - 1;
  const int C = cl.chunk;
  const int nc = n > 0 ? (n + C - 1) / C : 1;

  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);
  double* base = reinterpret_cast<double*>(smem_raw + size_t(kWarps) * tmem_stage_bytes_per_warp<N, D>()) +
                 threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return base + (size_t(buf) * (1 + D) + slot) * kTmemThreads; };
  double* thist = base + size_t(RD) * (1 + D) * kTmemThreads;
  auto HT = [&](int b) -> double& { return thist[size_t(b) * kTmemThreads]; };  // time of the step that made block b
  double* stash = thist + size_t(C + 1) * kTmemThreads;    // x0[D], T0
  double* restart = stash + size_t(D + 1) * kTmemThreads;  // T of own segment lo, x_lo[D], x_{lo+1}[D]
  double* state = restart + size_t(1 + 2 * D) * kTmemThreads;
  auto SP = [&](int blk, int slot) -> double& { return state[(size_t(blk) * kSlots + slot) * kTmemThreads]; };
  auto RS = [&](int slot) -> double* { return restart + size_t(slot) * kTmemThreads; };

  auto put_state = [&](int blk, const double (&sv)[kSlots]) {
#pragma unroll
    for (int i = 0; i < kSlots; ++i) SP(blk, i) = sv[i];
  };
  auto get_state = [&](int blk, double (&sv)[kSlots]) {
#pragma unroll
    for (int i = 0; i < kSlots; ++i) sv[i] = SP(blk, i);
  };

  auto seg = [&](int j) -> int { return half ? K - 1 - j : j; };
  auto pidx = [&](int v) -> int {
    const int o = half ? K - v : v;
    return o == 0 ? 0 : (o < K ? h + o - 1 : h + K - 1);
  };
  auto sgn = [&](int idx) -> double { return (half && !(idx & 1)) ? -1.0 : 1.0; };
  const int e0 = half ? h + K : 1;

  const long long n_wtiles = (prm.B + 15) >> 4;
  const long long wt_stride = (long long)gridDim.x * kWarps;
  const long long gthreads = (long long)gridDim.x * kTmemThreads;
  double* __restrict__ ck = cl.ckpt ? cl.ckpt + ((long long)blockIdx.x * kTmemThreads + threadIdx.x) : nullptr;
  auto CK = [&](int j, int slot) -> double& { return ck[((long long)(j - 1) * kCk + slot) * gthreads]; };

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;

  for (long long wt = (long long)blockIdx.x * kWarps + warp; wt < n_wtiles; wt += wt_stride) {
    long long traj = wt * 16 + (lane >> 1);
    const long long traj0 = wt * 16;
    const bool valid = traj < prm.B;
    if (!valid) traj = prm.B - 1;
    const double* __restrict__ tt = prm.times + traj * K;
    const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
    auto xaddr = [&](int v, int d) -> const double* { return fx + d * nf + pidx(v); };
    auto ring_issue = [&](int v) {
      const int j = v < K ? v : K - 1;
      const int vn = v + 1 <= K ? v + 1 : K;
      const int buf = v % RD;
      cp_async8(PF(buf, 0), tt + seg(j));
#pragma unroll
      for (int d = 0; d < D; ++d) cp_async8(PF(buf, 1 + d), xaddr(vn, d));
    };
    // restart inputs of a chunk that starts after own step lo
    auto restart_issue = [&](int lo) {
      cp_async8(RS(0), tt + seg(lo));
#pragma unroll
      for (int d = 0; d < D; ++d) {
        cp_async8(RS(1 + d), xaddr(lo, d));
        cp_async8(RS(1 + D + d), xaddr(lo + 1, d));
      }
    };

    // emit own-frame segment j for every lane of the warp at once (convergent)
    auto emit_all = [&](int j, int v_step, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D]) {
      double tp[h], itp[h];
      const double Ts = half ? -T : T;
      tp[0] = 1.0;
#pragma unroll
      for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * Ts;
      itp[0] = pow_int<h>(iT);
#pragma unroll
      for (int k = 1; k < h; ++k) itp[k] = itp[k - 1] * iT;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double c[N], ss[h], se[h];
#pragma unroll
        for (int k = 0; k < h; ++k) {
          const double s0 = half ? ed[k][d] : sd[k][d];
          const double e0v = half ? sd[k][d] : ed[k][d];
          c[k] = s0 * ((half && (k & 1)) ? -AI::at(k, k) : AI::at(k, k));
          ss[k] = tp[k] * s0;
          se[k] = tp[k] * e0v;
        }
        double ee[h];
#pragma unroll
        for (int k = 0; k < h; ++k) {
          double acc = se[k] - ss[k];
#pragma unroll
          for (int j2 = k + 1; j2 < h; ++j2) {
            constexpr double kInvFact[6] = {1.0, 1.0, 0.5, 1.0 / 6.0, 1.0 / 24.0, 1.0 / 120.0};
            acc = (j2 - k == 1) ? acc - ss[j2] : fma(-kInvFact[j2 - k], ss[j2], acc);
          }
          ee[k] = acc;
        }
#pragma unroll
        for (int q = 0; q < h; ++q) {
          double acc = AI::at(h + q, h) * ee[0];
#pragma unroll
          for (int k = 1; k < h; ++k) acc = fma(AI::at(h + q, h + k), ee[k], acc);
          c[h + q] = acc * itp[q];
        }
        if (d == 0) {  // the TMA must have finished reading the previous segment's tile
          if (lane == 0) bulk_wait_read();
          __syncwarp();
        }
#pragma unroll
        for (int q = 0; q < h; ++q) my_row[d * h + q] = make_double2(c[2 * q], c[2 * q + 1]);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        if (v_step <= nhF) tma_store_box(&tmap, stage, j * (D * N), (int)traj0);
        if (v_step <= nhB) tma_store_box(&tmap, stage + 16 * (D * h), (K - 1 - j) * (D * N), (int)traj0);
        bulk_commit();
      }
    };


    int stat = 0;
    double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
    double ed[h][D];
    const int np = (K - 1) * m;
    double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + traj * (long long)D * np : nullptr;
    auto store_free = [&](int v_own, const double (&u)[h][D]) {
      if (df != nullptr && valid) {
        const int vo = half ? K - v_own : v_own;
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int j = 0; j < m; ++j) df[d * np + (vo - 1) * m + j] = sgn(j) * u[1 + j][d];
      }
    };

    for (int j = 0; j < nc; ++j) {
      const int hi = n - j * C;
      const int lo = hi - C > 0 ? hi - C : 0;
      const int from = j == 0 ? 0 : lo;  // round 0 sweeps everything, storing only (lo, hi]

      // ---- (re)start state: inputs through the restart slots, carry from the prologue (round 0) or checkpoint
      restart_issue(from);
      cp_async_commit();
#pragma unroll
      for (int q = 1; q < RD; ++q) {
        if (from + q <= nh && from + q <= hi) ring_issue(from + q);
        cp_async_commit();
      }
      if (j > 0) {
#pragma unroll
        for (int a = 0; a < m; ++a) {
#pragma unroll
          for (int b = 0; b < m; ++b) Wp[a][b] = CK(j, a * m + b);
#pragma unroll
          for (int d = 0; d < D; ++d) yp[a][d] = CK(j, m * m + a * D + d);
        }
      }
      cp_async_wait_group<RD - 1>();
      {
        const double Tp = *RS(0);
#pragma unroll
        for (int d = 0; d < D; ++d) {
          xm[d] = *RS(1 + d);
          xc[d] = *RS(1 + D + d);
        }
        if (!(Tp > 0.0)) stat |= kStatusBadTime;
        const double iTp = fast_rcp(Tp);
        double pw[N - 1];
        segment_powers<N, R>(Tp, iTp, pw);
#pragma unroll
        for (int a = 0; a < m; ++a) {
#pragma unroll
          for (int b = 0; b < m; ++b) Cee[a][b] = pw[a + b + 2] * G::at(h + 1 + a, h + 1 + b);
          cps[a] = pw[a + 1] * G::at(h + 1 + a, 0);
          cpe[a] = pw[a + 1] * G::at(h + 1 + a, h);
        }
        if (j == 0) {  // prologue of the tile: initial carry from the fixed end derivatives (exact 2^+-600 scaling)
#pragma unroll
          for (int d = 0; d < D; ++d) stash[size_t(d) * kTmemThreads] = xm[d];
          stash[size_t(D) * kTmemThreads] = Tp;
#pragma unroll
          for (int a = 0; a < m; ++a)
#pragma unroll
            for (int b = 0; b < m; ++b) Wp[a][b] = (a == b) ? kTiny : 0.0;
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
              yp[a][d] = acc * kHuge;
            }
          }
        }
      }

      // ---- forward sweep over (from, hi]
      for (int v = from + 1; v <= hi; ++v) {
        if (j == 0 && nc > 1) {  // checkpoint the carry at the start of every outer chunk (warp-uniform test)
          const int dist = n - (v - 1);
          const bool at0 = (v - 1) == 0;
          if (at0 || (dist % C == 0 && dist >= 2 * C)) {
            const int jc = at0 ? nc - 1 : dist / C - 1;
#pragma unroll
            for (int a = 0; a < m; ++a) {
#pragma unroll
              for (int b = 0; b < m; ++b) CK(jc, a * m + b) = Wp[a][b];
#pragma unroll
              for (int d = 0; d < D; ++d) CK(jc, m * m + a * D + d) = yp[a][d];
            }
          }
        }
        const bool store = v > lo;
        double sv[kSlots];
        if (v <= nh) {
          cp_async_wait_group<RD - 2>();
          double xn[D];
#pragma unroll
          for (int d = 0; d < D; ++d) xn[d] = *PF(v % RD, 1 + d);
          const double T = *PF(v % RD, 0);
          if (store) HT(v - lo - 1) = T;
          if (v + RD - 1 <= nh && v + RD - 1 <= hi) ring_issue(v + RD - 1);
          cp_async_commit();
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
              double s = -cps[a] * xm[d];
              s = fma(-gmid, xc[d], s);
              s = fma(-gnext, xn[d], s);
#pragma unroll
              for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
              bb[a][d] = s;
            }
          }
          double L[m][m], inv[m];
#pragma unroll
          for (int jj = 0; jj < m; ++jj) {
            double s = Dp[jj][jj];
#pragma unroll
            for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], L[jj][k], s);
            if (!(s > 0.0)) stat |= kStatusNotSpd;
            inv[jj] = fast_rsqrt(s);
#pragma unroll
            for (int i = jj + 1; i < m; ++i) {
              double t = Dp[i][jj];
#pragma unroll
              for (int k = 0; k < jj; ++k) t = fma(-L[i][k], L[jj][k], t);
              L[i][jj] = t * inv[jj];
            }
          }
#pragma unroll
          for (int d = 0; d < D; ++d) {
#pragma unroll
            for (int jj = 0; jj < m; ++jj) {
              double s = bb[jj][d];
#pragma unroll
              for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], yp[k][d], s);
              yp[jj][d] = s * inv[jj];
            }
          }
#pragma unroll
          for (int c = 0; c < m; ++c) {
#pragma unroll
            for (int jj = 0; jj < m; ++jj) {
              double s = E[jj][c];
#pragma unroll
              for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], Wp[k][c], s);
              Wp[jj][c] = s * inv[jj];
            }
          }
          {
            int slot = 0;
#pragma unroll
            for (int i = 1; i < m; ++i)
#pragma unroll
              for (int jj = 0; jj < i; ++jj) sv[slot++] = L[i][jj];
#pragma unroll
            for (int jj = 0; jj < m; ++jj) sv[slot++] = inv[jj];
#pragma unroll
            for (int jj = 0; jj < m; ++jj)
#pragma unroll
              for (int d = 0; d < D; ++d) sv[slot++] = yp[jj][d];
#pragma unroll
            for (int d = 0; d < D; ++d) sv[slot++] = xc[d];
          }
#pragma unroll
          for (int a = 0; a < m; ++a) {
#pragma unroll
            for (int b = 0; b <= a; ++b) Cee[a][b] = pw[a + b + 2] * G::at(h + 1 + a, h + 1 + b);
            cps[a] = pw[a + 1] * G::at(h + 1 + a, 0);
            cpe[a] = pw[a + 1] * G::at(h + 1 + a, h);
          }
#pragma unroll
          for (int d = 0; d < D; ++d) {
            xm[d] = xc[d];
            xc[d] = xn[d];
          }
        }
        if (store) {  // warp-uniform
          __syncwarp();
          put_state(v - lo - 1, sv);
        }
      }
      __syncwarp();

      // ---- middle vertex (round 0 only): both halves meet
      if (j == 0) {
        double um[m][D];
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
            double s = -cps[a] * xm[d];
            s = fma(-cpe[a], xc[d], s);
#pragma unroll
            for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
            bl[a][d] = s;
          }
        }
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
            bl[a][d] += (a & 1) ? o : -o;
          }
        }
        stat |= __shfl_xor_sync(kFull, stat, 1);
        double L[m][m], inv[m];
#pragma unroll
        for (int jj = 0; jj < m; ++jj) {
          double s = Dl[jj][jj];
#pragma unroll
          for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], L[jj][k], s);
          if (!(s > 0.0)) stat |= kStatusNotSpd;
          inv[jj] = fast_rsqrt(s);
#pragma unroll
          for (int i = jj + 1; i < m; ++i) {
            double t = Dl[i][jj];
#pragma unroll
            for (int k = 0; k < jj; ++k) t = fma(-L[i][k], L[jj][k], t);
            L[i][jj] = t * inv[jj];
          }
        }
#pragma unroll
        for (int d = 0; d < D; ++d) {
          double y[m];
#pragma unroll
          for (int jj = 0; jj < m; ++jj) {
            double s = bl[jj][d];
#pragma unroll
            for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], y[k], s);
            y[jj] = s * inv[jj];
          }
#pragma unroll
          for (int jj = m - 1; jj >= 0; --jj) {
            double s = y[jj];
#pragma unroll
            for (int k = jj + 1; k < m; ++k) s = fma(-L[k][jj], um[k][d], s);
            um[jj][d] = s * inv[jj];
          }
        }
#pragma unroll
        for (int d = 0; d < D; ++d) {
          ed[0][d] = xc[d];
#pragma unroll
          for (int jj = 0; jj < m; ++jj) ed[1 + jj][d] = um[jj][d];
        }
        if (half == 0) store_free(nh + 1, ed);
      }

      // ---- back-substitution + emission over (lo, hi], outwards
      for (int v = hi; v > lo; --v) {
        const bool act = v <= nh;
        const double T = act ? HT(v - lo - 1) : 1.0;
        const double iT = fast_rcp(T);
        double pw[N - 1];
        segment_powers<N, R>(T, iT, pw);
        double sv[kSlots];
        {
          get_state(v - lo - 1, sv);
        }
        double tE[m][D];  // E_v u_{v+1} (after the wait: this kernel runs at the register limit)
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int a = 0; a < m; ++a) {
            double s = 0.0;
#pragma unroll
            for (int b = 0; b < m; ++b) s = fma(pw[a + b + 2] * G::at(1 + a, h + 1 + b), ed[1 + b][d], s);
            tE[a][d] = s;
          }
        double sd[h][D];
        if (act) {
          double xv[D];
#pragma unroll
          for (int d = 0; d < D; ++d) xv[d] = sv[kL + m * D + d];
          double L[m][m], inv[m], rhs[m][D];
          {
            int slot = 0;
#pragma unroll
            for (int i = 1; i < m; ++i)
#pragma unroll
              for (int jj = 0; jj < i; ++jj) L[i][jj] = sv[slot++];
#pragma unroll
            for (int jj = 0; jj < m; ++jj) inv[jj] = sv[slot++];
#pragma unroll
            for (int jj = 0; jj < m; ++jj)
#pragma unroll
              for (int d = 0; d < D; ++d) rhs[jj][d] = sv[slot++];
          }
#pragma unroll
          for (int d = 0; d < D; ++d) {
            double t[m];
#pragma unroll
            for (int jj = 0; jj < m; ++jj) {
              double s = tE[jj][d];
#pragma unroll
              for (int k = 0; k < jj; ++k) s = fma(-L[jj][k], t[k], s);
              t[jj] = s * inv[jj];
              rhs[jj][d] -= t[jj];
            }
          }
#pragma unroll
          for (int d = 0; d < D; ++d) {
#pragma unroll
            for (int jj = m - 1; jj >= 0; --jj) {
              double s = rhs[jj][d];
#pragma unroll
              for (int k = jj + 1; k < m; ++k) s = fma(-L[k][jj], sd[1 + k][d], s);
              sd[1 + jj][d] = s * inv[jj];
            }
            sd[0][d] = xv[d];
          }
          store_free(v, sd);
        }
        __syncwarp();
        emit_all(v, v, T, iT, sd, ed);
        if (act) {
#pragma unroll
          for (int d = 0; d < D; ++d)
#pragma unroll
            for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
        }
      }
    }
    if (valid && half == 0 && prm.status != nullptr) prm.status[traj] = stat;
    {  // own segment 0: the fixed end vertex
      double sd[h][D];
#pragma unroll
      for (int d = 0; d < D; ++d) {
        sd[0][d] = stash[size_t(d) * kTmemThreads];
#pragma unroll
        for (int b = 0; b < m; ++b) sd[1 + b][d] = sgn(b) * __ldg(fx + d * nf + e0 + b);
      }
      const double T = stash[size_t(D) * kTmemThreads];
      const double iT = fast_rcp(T);
      __syncwarp();
      emit_all(0, 0, T, iT, sd, ed);
    }
  }

  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
