// mtg_twisted_chunked_kernel.cuh -- K3: the twisted two-lane sweep for ANY number of segments, with a fixed
// on-chip footprint (large-K kernel; the reference's own timing program runs K = 50 and K = 100,
// src/polynomial_timing_evaluation.cpp:114-129, its test-suite K = 50, test/test_polynomial_optimization.cpp:822-828).
//
// The resident kernels keep the factor of every eliminated vertex in shared memory, which caps the number of
// trajectories in flight per SM as K grows (25 doubles per lane and eliminated vertex at N = 10, D = 3).  Here
// only the C innermost vertex blocks of a lane stay in shared memory -- the host picks C and the warps per SM
// (launch_chunked) -- and the outer ones are PARKED in global memory.  One pass per tile:
//
//   forward   sweep over all own vertices 1..n (n = ceil(K/2)-1); the block of vertex v <= n-C (its pack() slots
//             and the step's segment time) goes to the parking area, the innermost C blocks to shared slot
//             (v-1) % C; then the middle vertex;
//   outward   back-substitution + emission v = n..1 from the shared slots; once vertex v is back-substituted, its
//             slot is refilled by cp.async with parked block v-C, which therefore has C-1 outward steps (and v's
//             emission) to land.
//
// Cost: no recomputation -- every vertex is factorised once, as in the resident kernels.  Extra global traffic
// 2 * (n-C) * (kSlots+1) * 8 bytes per lane (written once, read once); CTAs are persistent (static tile
// assignment), so the parking area is bounded by the number of resident threads, not by the batch (about 0.4 KB
// per thread at K = 16, C = 5: it stays in L2; at K = 50 it spills to HBM).  Every thread owns one column of it,
// laid out [block][slot][thread] so that a warp stores or loads one slot as 256 contiguous bytes.  As in v4, the
// next tile's prologue inputs are prefetched into the dead state region at the end of the outward sweep, and the
// fixed end derivatives of the final emission into the idle input ring.  Arithmetic per vertex is exactly the
// v4 sequence: results are bitwise equal to v4 and independent of C (tests force tiny chunks on K = 16 to prove it),
// of the warps per CTA, of the warps per SM and of the L2 hints.
#pragma once

#include "mtg_twisted_tmem_v4_kernel.cuh"

namespace mtg {

struct ChunkedLaunch {
  int chunk;          // C: vertex blocks resident per lane (in shared memory)
  double* ckpt;       // parking area [n-C][kPark][gridDim.x * blockDim.x]: the outer vertex blocks of the sweep
  int evict_first;    // inputs and coefficient stores marked evict-first in L2, so that the parking area stays there
};

// Dynamic shared memory of K3 behind the staging tiles, in per-thread slots:
// [input ring RD x (1+D)][times C][stash D+1][region: C blocks with the vertex position, or the next tile's prologue]
// for a CTA of W warps
template <int N, int D, int RD, int W>
struct ChunkedLayout {
  static constexpr int kThreads = 32 * W;
  static constexpr int kSlots = sweep_state_slots<N, D, true>();
  static constexpr int kPark = kSlots + 1;                   // a parked block: pack() slots, then the segment time
  static constexpr int kPro = 2 * D + (N / 2 - 1) * D + 1;  // x0, x1, u0[m], T0
  static constexpr int kHist = RD * (1 + D);                 // ring, then the times of the resident blocks
  static constexpr int kStash = D + 1;                       // x0[D], T0
  __host__ __device__ static constexpr int hist_slots(int C) { return C; }
  __host__ __device__ static constexpr size_t stash(int C) { return size_t(kHist) + hist_slots(C); }
  __host__ __device__ static constexpr size_t region(int C) { return stash(C) + kStash; }
  __host__ __device__ static constexpr size_t region_slots(int C) {
    return size_t(C) * kSlots > size_t(kPro) ? size_t(C) * kSlots : size_t(kPro);
  }
  __host__ __device__ static constexpr size_t bytes(int C) {
    return tmem_stage_bytes<N, D, kThreads>() + tmem_slot_bytes(region(C) + region_slots(C), kThreads);
  }
};

// cp.async.wait_group with a run-time bound: waits until at most min(pending, 3) groups are in flight, which is at
// least what `pending` asks for
__device__ __forceinline__ void cp_async_wait_at_most(int pending) {
  if (pending <= 0) cp_async_wait_group<0>();
  else if (pending == 1) cp_async_wait_group<1>();
  else if (pending == 2) cp_async_wait_group<2>();
  else cp_async_wait_group<3>();
}

// W warps per CTA.  The warps of a CTA share nothing but the CTA's shared memory allocation (each has its own staging
// tile, tiles, parking column and TMA group; there is no __syncthreads), so W only sets the granularity in which
// shared memory is allocated: at N = 10, D = 3 one-warp CTAs fit 7 warps per SM at C = 3 where four-warp CTAs
// fit 4.
// Both launch bounds give a register cap of 255.
template <int N, int R, int D, int RD, int W>
__global__ void __launch_bounds__(32 * W, 8 / W)
    twisted_chunked_kernel(const WaypointParams prm, const ChunkedLaunch cl, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = ChunkedLayout<N, D, RD, W>;
  constexpr int kSlots = Lay::kSlots;
  constexpr int kPark = Lay::kPark;
  constexpr int kPro = Lay::kPro;
  constexpr int kThreads = Lay::kThreads;
  static_assert(RD >= 2, "ring depth");
  using G = H1Imm<N, R>;
  using AI = A1InvImm<N>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = W == 1 ? int(threadIdx.x) : int(threadIdx.x & 31);
  const int warp = W == 1 ? 0 : int(threadIdx.x >> 5);
  const int half = lane & 1;
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;
  const int nh = half ? K - M - 1 : M - 1;
  const int n = M - 1;
  const int C = cl.chunk;
  const int npark = n - C;  // vertices 1..npark are parked (none when C >= n)

  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);
  double* base = reinterpret_cast<double*>(smem_raw + tmem_stage_bytes<N, D, kThreads>()) + threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return base + (size_t(buf) * (1 + D) + slot) * kThreads; };
  double* thist = base + size_t(Lay::kHist) * kThreads;
  auto HT = [&](int b) -> double* { return thist + size_t(b) * kThreads; };  // time of the step that made block b
  double* stash = thist + size_t(Lay::hist_slots(C)) * kThreads;  // x0[D], T0
  double* region = stash + size_t(Lay::kStash) * kThreads;        // state blocks; next tile's prologue inputs
  auto SP = [&](int blk, int slot) -> double* { return region + (size_t(blk) * kSlots + slot) * kThreads; };
  auto PRO = [&](int slot) -> double* { return region + size_t(slot) * kThreads; };

  const sweep::Frame<N> fr{K, half};
  const int e0 = fr.e0();

  const long long n_wtiles = (prm.B + 15) >> 4;
  const long long wt_stride = (long long)gridDim.x * W;
  const long long gthreads = (long long)gridDim.x * kThreads;
  double* __restrict__ pk = cl.ckpt ? cl.ckpt + ((long long)blockIdx.x * kThreads + threadIdx.x) : nullptr;
  auto PK = [&](int b, int slot) -> double* { return pk + ((long long)b * kPark + slot) * gthreads; };

  // pointers of a warp tile's trajectory for this lane
  struct Ptrs {
    const double* tt;
    const double* fx;
    long long traj;
    bool valid;
  };
  auto tile_ptrs = [&](long long w) -> Ptrs {
    Ptrs p;
    p.traj = w * 16 + (lane >> 1);
    p.valid = p.traj < prm.B;
    if (!p.valid) p.traj = prm.B - 1;
    p.tt = prm.times + p.traj * K;
    p.fx = prm.dfix + p.traj * (long long)D * nf;
    return p;
  };
  auto xaddr = [&](const Ptrs& p, int v, int d) -> const double* { return p.fx + d * nf + fr.pidx(v); };
  // a tile's prologue inputs -> PRO region (cp.async; the caller commits the group)
  auto pro_issue = [&](const Ptrs& p) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      cp_async8_stream(PRO(d), xaddr(p, 0, d), cl.evict_first);
      cp_async8_stream(PRO(D + d), xaddr(p, 1, d), cl.evict_first);
#pragma unroll
      for (int b = 0; b < m; ++b) cp_async8_stream(PRO(2 * D + b * D + d), p.fx + d * nf + e0 + b, cl.evict_first);
    }
    cp_async8_stream(PRO(kPro - 1), p.tt + fr.seg(0), cl.evict_first);
  };
  // inputs of inward step v (time of own segment v, position of own vertex v+1) -> ring buffer v % RD
  auto ring_issue = [&](const Ptrs& p, int v) {
    const int j = v < K ? v : K - 1;
    const int vn = v + 1 <= K ? v + 1 : K;
    const int buf = v % RD;
    cp_async8_stream(PF(buf, 0), p.tt + fr.seg(j), cl.evict_first);
#pragma unroll
    for (int d = 0; d < D; ++d) cp_async8_stream(PF(buf, 1 + d), xaddr(p, vn, d), cl.evict_first);
  };

  long long wt = (long long)blockIdx.x * W + warp;
  if (wt < n_wtiles) {
    pro_issue(tile_ptrs(wt));
    cp_async_commit();
  }

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB, cl.evict_first != 0};

  for (; wt < n_wtiles; wt += wt_stride) {
    const long long wt_next = wt + wt_stride;  // its prologue is prefetched at the end of this tile
    const Ptrs P = tile_ptrs(wt);
    const long long traj0 = wt * 16;
    const bool valid = P.valid;

    // ---- ring prefetch of the first RD-1 inward steps, then consume the prologue inputs (issued a tile ago)
    // (a group is committed for every step even when it is empty, so that wait_group<RD-2> always means "the data
    // of the current step has landed")
#pragma unroll
    for (int q = 1; q < RD; ++q) {
      if (q <= nh) ring_issue(P, q);
      cp_async_commit();
    }
    cp_async_wait_group<RD - 1>();

    int stat = 0;
    double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
    {
#pragma unroll
      for (int d = 0; d < D; ++d) {
        xm[d] = *PRO(d);
        xc[d] = *PRO(D + d);
        stash[size_t(d) * kThreads] = xm[d];
      }
      const double T0 = *PRO(kPro - 1);
      stash[size_t(D) * kThreads] = T0;
      if (bad_segment_time(T0)) stat |= kStatusBadTime;
      const double iT0 = fast_rcp(T0);
      double pw[N - 1];
      segment_powers<N, R>(T0, iT0, pw);
      S::end_blocks(pw, Cee, cps, cpe);
      // initial carry from the fixed end derivatives (exact 2^+-600 scaling)
      S::carry_fold(pw, [&](int b, int d) { return fr.sgn(b) * *PRO(2 * D + b * D + d); }, Wp, yp);
    }

    // ---------------------------------------------------------------- sweep towards the middle
    for (int v = 1; v <= n; ++v) {
      double sv[kSlots];
      double T;
      if (v <= nh) {
        cp_async_wait_group<RD - 2>();
        double xn[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xn[d] = *PF(v % RD, 1 + d);
        T = *PF(v % RD, 0);
        if (v + RD - 1 <= nh) ring_issue(P, v + RD - 1);  // nothing is left in flight after the last own step
        cp_async_commit();
        if (bad_segment_time(T)) stat |= kStatusBadTime;
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
      __syncwarp();
      if (v <= npark) {  // warp-uniform; every lane is active here (v < n <= nh + 1)
#pragma unroll
        for (int i = 0; i < kSlots; ++i) *PK(v - 1, i) = sv[i];
        *PK(v - 1, kSlots) = T;
      } else {
        const int b = (v - 1) % C;
        if (v <= nh) *HT(b) = T;
#pragma unroll
        for (int i = 0; i < kSlots; ++i) *SP(b, i) = sv[i];
      }
    }
    __syncwarp();

    // ---------------------------------------------------------------- middle vertex: both halves meet
    double um[m][D];
    S::middle(Cee, cps, cpe, Wp, yp, xm, xc, um, stat);
    if (valid && half == 0 && prm.status != nullptr) prm.status[P.traj] = stat;

    // ---------------------------------------------------------------- outward back-substitution
    const int np = (K - 1) * m;
    double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + P.traj * (long long)D * np : nullptr;
    auto store_free = [&](int v_own, const double (&u)[h][D]) {
      if (df != nullptr && valid) {
        const int vo = fr.vert(v_own);
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int j = 0; j < m; ++j) df[d * np + (vo - 1) * m + j] = fr.sgn(j) * u[1 + j][d];
      }
    };

    double ed[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      ed[0][d] = xc[d];
#pragma unroll
      for (int j = 0; j < m; ++j) ed[1 + j][d] = um[j][d];
    }
    if (half == 0) store_free(nh + 1, ed);

    // The ring is idle during the outward sweep: the fixed end derivatives needed by the final emission are
    // fetched into it now (slot q of the flattened ring), many steps ahead of their use.
    constexpr bool kEndInRing = RD * (1 + D) >= m * D;
    if constexpr (kEndInRing) {
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int b = 0; b < m; ++b) cp_async8_stream(base + size_t(b * D + d) * kThreads, P.fx + d * nf + e0 + b, cl.evict_first);
      cp_async_commit();
    }
    // the next tile's prologue inputs go to the state region: issued once every state block has been read back
    auto issue_next_pro = [&]() {
      if (wt_next < n_wtiles) {  // warp-uniform
        pro_issue(tile_ptrs(wt_next));
        cp_async_commit();
      }
    };
    if (n == 0) issue_next_pro();

    for (int v = n; v >= 1; --v) {
      const int b = (v - 1) % C;
      // parked block v was refilled C steps ago; the C-1 refill groups committed since may stay in flight
      if (v <= npark) cp_async_wait_at_most(C - 1);
      const bool act = v <= nh;
      const double T = act ? *HT(b) : 1.0;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = *SP(b, i);
      double tE[m][D];  // E_v u_{v+1} (before the activity test: this kernel runs at the register limit)
      S::couple(pw, ed, tE);
      double sd[h][D];
      if (act) {
        double xv[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xv[d] = S::position(sv, d);
        S::back_substitute(sv, tE, xv, sd);
        store_free(v, sd);
      }
      if (v - C >= 1) {  // warp-uniform: the freed slot takes parked block v-C
#pragma unroll
        for (int i = 0; i < kSlots; ++i) cp_async8(SP(b, i), PK(v - C - 1, i));
        cp_async8(HT(b), PK(v - C - 1, kSlots));
      }
      cp_async_commit();
      __syncwarp();
      out.emit(v, v, T, iT, sd, ed, traj0);
      if (act) {
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
      }
    }
    if (n > 0) issue_next_pro();  // the state region is dead only now
    {  // own segment 0: the fixed end vertex
      double sd[h][D];
      if constexpr (kEndInRing) {
        // everything except (possibly) the next tile's prologue group has landed
        if (wt_next < n_wtiles) cp_async_wait_group<1>(); else cp_async_wait_group<0>();
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        sd[0][d] = stash[size_t(d) * kThreads];
#pragma unroll
        for (int b = 0; b < m; ++b) {
          if constexpr (kEndInRing) {
            sd[1 + b][d] = fr.sgn(b) * base[size_t(b * D + d) * kThreads];
          } else {
            sd[1 + b][d] = fr.sgn(b) * __ldg(P.fx + d * nf + e0 + b);
          }
        }
      }
      const double T = stash[size_t(D) * kThreads];
      const double iT = fast_rcp(T);
      __syncwarp();
      out.emit(0, 0, T, iT, sd, ed, traj0);
    }
  }

  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
