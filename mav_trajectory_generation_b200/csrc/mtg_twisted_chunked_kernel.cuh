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

// Dynamic shared memory of K3 behind the staging tiles, in per-thread slots:
// [input ring RD x (1+D)][times C+1][stash D+1][restart 1+2D][state: C blocks with the vertex position]
template <int N, int D, int RD>
struct ChunkedLayout {
  static constexpr int kSlots = sweep_state_slots<N, D, true>();
  static constexpr int kCkpt = (N / 2 - 1) * (N / 2 - 1) + (N / 2 - 1) * D;  // global checkpoint: W, y
  static constexpr int kHist = RD * (1 + D);      // ring, then the times of the chunk
  static constexpr int kStash = D + 1;             // x0[D], T0
  static constexpr int kRestart = 1 + 2 * D;       // T of own segment lo, x_lo[D], x_{lo+1}[D]
  __host__ __device__ static constexpr int hist_slots(int C) { return C + 1; }
  __host__ __device__ static constexpr size_t stash(int C) { return size_t(kHist) + hist_slots(C); }
  __host__ __device__ static constexpr size_t restart(int C) { return stash(C) + kStash; }
  __host__ __device__ static constexpr size_t state(int C) { return restart(C) + kRestart; }
  __host__ __device__ static constexpr size_t bytes(int C) {
    return tmem_stage_bytes<N, D>() + tmem_slot_bytes(state(C) + size_t(C) * kSlots);
  }
};

template <int N, int R, int D, int RD>
__global__ void __launch_bounds__(kTmemThreads, 2)
    twisted_chunked_kernel(const WaypointParams prm, const ChunkedLaunch cl, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = ChunkedLayout<N, D, RD>;
  constexpr int kSlots = Lay::kSlots;
  constexpr int kCk = Lay::kCkpt;
  constexpr int kWarps = kTmemThreads / 32;
  using G = H1Imm<N, R>;
  using AI = A1InvImm<N>;
  using S = sweep::Sweep<N, D, G>;

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
  double* base = reinterpret_cast<double*>(smem_raw + tmem_stage_bytes<N, D>()) + threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return base + (size_t(buf) * (1 + D) + slot) * kTmemThreads; };
  double* thist = base + size_t(Lay::kHist) * kTmemThreads;
  auto HT = [&](int b) -> double& { return thist[size_t(b) * kTmemThreads]; };  // time of the step that made block b
  double* stash = thist + size_t(Lay::hist_slots(C)) * kTmemThreads;  // x0[D], T0
  double* restart = stash + size_t(Lay::kStash) * kTmemThreads;       // T of own segment lo, x_lo[D], x_{lo+1}[D]
  double* state = restart + size_t(Lay::kRestart) * kTmemThreads;
  auto SP = [&](int blk, int slot) -> double& { return state[(size_t(blk) * kSlots + slot) * kTmemThreads]; };
  auto RS = [&](int slot) -> double* { return restart + size_t(slot) * kTmemThreads; };

  const sweep::Frame<N> fr{K, half};
  const int e0 = fr.e0();

  const long long n_wtiles = (prm.B + 15) >> 4;
  const long long wt_stride = (long long)gridDim.x * kWarps;
  const long long gthreads = (long long)gridDim.x * kTmemThreads;
  double* __restrict__ ck = cl.ckpt ? cl.ckpt + ((long long)blockIdx.x * kTmemThreads + threadIdx.x) : nullptr;
  auto CK = [&](int j, int slot) -> double& { return ck[((long long)(j - 1) * kCk + slot) * gthreads]; };

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB};

  for (long long wt = (long long)blockIdx.x * kWarps + warp; wt < n_wtiles; wt += wt_stride) {
    long long traj = wt * 16 + (lane >> 1);
    const long long traj0 = wt * 16;
    const bool valid = traj < prm.B;
    if (!valid) traj = prm.B - 1;
    const double* __restrict__ tt = prm.times + traj * K;
    const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
    auto xaddr = [&](int v, int d) -> const double* { return fx + d * nf + fr.pidx(v); };
    auto ring_issue = [&](int v) {
      const int j = v < K ? v : K - 1;
      const int vn = v + 1 <= K ? v + 1 : K;
      const int buf = v % RD;
      cp_async8(PF(buf, 0), tt + fr.seg(j));
#pragma unroll
      for (int d = 0; d < D; ++d) cp_async8(PF(buf, 1 + d), xaddr(vn, d));
    };
    // restart inputs of a chunk that starts after own step lo
    auto restart_issue = [&](int lo) {
      cp_async8(RS(0), tt + fr.seg(lo));
#pragma unroll
      for (int d = 0; d < D; ++d) {
        cp_async8(RS(1 + d), xaddr(lo, d));
        cp_async8(RS(1 + D + d), xaddr(lo + 1, d));
      }
    };

    int stat = 0;
    double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
    double ed[h][D];
    const int np = (K - 1) * m;
    double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + traj * (long long)D * np : nullptr;
    auto store_free = [&](int v_own, const double (&u)[h][D]) {
      if (df != nullptr && valid) {
        const int vo = fr.vert(v_own);
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int j = 0; j < m; ++j) df[d * np + (vo - 1) * m + j] = fr.sgn(j) * u[1 + j][d];
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
        S::end_blocks(pw, Cee, cps, cpe);
        if (j == 0) {  // prologue of the tile: initial carry from the fixed end derivatives (exact 2^+-600 scaling)
#pragma unroll
          for (int d = 0; d < D; ++d) stash[size_t(d) * kTmemThreads] = xm[d];
          stash[size_t(D) * kTmemThreads] = Tp;
          S::carry_fold(pw, [&](int b, int d) { return fr.sgn(b) * __ldg(fx + d * nf + e0 + b); }, Wp, yp);
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

          double Dp[m][m], E[m][m], bb[m][D], L[m][m], inv[m];
          S::assemble(pw, Cee, cps, cpe, Wp, yp, xm, xc, xn, Dp, E, bb);
          S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
          S::pack(L, inv, yp, xc, sv);
          S::end_blocks(pw, Cee, cps, cpe);
#pragma unroll
          for (int d = 0; d < D; ++d) {
            xm[d] = xc[d];
            xc[d] = xn[d];
          }
        }
        if (store) {  // warp-uniform
          __syncwarp();
#pragma unroll
          for (int i = 0; i < kSlots; ++i) SP(v - lo - 1, i) = sv[i];
        }
      }
      __syncwarp();

      // ---- middle vertex (round 0 only): both halves meet
      if (j == 0) {
        double um[m][D];
        S::middle(Cee, cps, cpe, Wp, yp, xm, xc, um, stat);
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
#pragma unroll
        for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - lo - 1, i);
        double tE[m][D];  // E_v u_{v+1} (after the wait: this kernel runs at the register limit)
        S::couple(pw, ed, tE);
        double sd[h][D];
        if (act) {
          double xv[D];
#pragma unroll
          for (int d = 0; d < D; ++d) xv[d] = S::position(sv, d);
          S::back_substitute(sv, tE, xv, sd);
          store_free(v, sd);
        }
        __syncwarp();
        out.emit(v, v, T, iT, sd, ed, traj0);
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
        for (int b = 0; b < m; ++b) sd[1 + b][d] = fr.sgn(b) * __ldg(fx + d * nf + e0 + b);
      }
      const double T = stash[size_t(D) * kTmemThreads];
      const double iT = fast_rcp(T);
      __syncwarp();
      out.emit(0, 0, T, iT, sd, ed, traj0);
    }
  }

  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
