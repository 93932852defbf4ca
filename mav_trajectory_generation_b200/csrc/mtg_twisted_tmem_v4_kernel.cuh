// mtg_twisted_tmem_v4_kernel.cuh -- K1 (v4): the twisted shared-memory-state kernel made PERSISTENT, with every
// global read issued several sweep steps (or half a tile) before it is consumed.
//
// Input reads queue behind the kernel's write bursts (its HBM traffic is mostly coefficient stores), so a read
// issued one sweep step ahead is often not back in time.  v4 therefore
//   * runs a grid of resident CTAs for the whole launch; every WARP loops over its own 16-trajectory tiles
//     (tile = blockIdx.x * 4 + warp, stride gridDim.x * 4), no CTA barrier inside the loop;
//   * prefetches the NEXT tile's prologue inputs (end vertex, its derivatives, first waypoint, first time)
//     with cp.async at the end of the outward sweep, into the part of shared memory that holds the sweep
//     state (dead by then);
//   * deepens the per-thread input ring to RD buffers (prefetch distance RD-1 sweep steps, cp.async groups);
//   * keeps the end vertex position in a 3-double per-thread stash and prefetches the end derivatives for the
//     final emission at the start of the outward sweep -- no exposed global read at the end of a tile;
//   * folds the first step's right-hand-side carry into the (W, y) carry with an exact power-of-two scaling
//     (W = 2^-600 I, y = -2^600 b): the m*D carry registers disappear from the loop.
// The arithmetic of a trajectory is otherwise the v3 sequence (mtg_twisted_tmem_kernel.cuh); results agree to
// rounding (bitwise except for the order in which the first step's carry is added).
#pragma once

#include "mtg_twisted_tmem_kernel.cuh"

namespace mtg {

struct TmemLaunchV4 {
  unsigned long long* tile_counter;  // non-null: warps draw their 16-trajectory tiles from this counter (zeroed by
                                     // the host before the launch); null: static round-robin assignment
};

// Dynamic shared memory of v4 behind the staging tiles, in per-thread slots:
// [input ring RD x (1+D)][time history nmax+1][x0 stash D][region: sweep state, or the next tile's prologue inputs]
template <int N, int D, int RD>
struct V4Layout {
  static constexpr int kSlots = sweep_state_slots<N, D, true>();
  static constexpr int kPro = 2 * D + (N / 2 - 1) * D + 1;  // x0, x1, u0[m], T0
  static constexpr int kHist = RD * (1 + D);                                // ring, then the time history
  __host__ __device__ static constexpr int hist_slots(int nmax) { return nmax + 1; }  // history, then the x0 stash
  __host__ __device__ static constexpr size_t x0(int nmax) { return size_t(kHist) + hist_slots(nmax); }
  __host__ __device__ static constexpr size_t region(int nmax) { return x0(nmax) + D; }
  __host__ __device__ static constexpr size_t bytes(int K) {
    return tmem_stage_bytes<N, D>() + tmem_slot_bytes(region((K + 1) / 2 - 1) + (size_t((K + 1) / 2 - 1) * kSlots > kPro
                                                                                      ? size_t((K + 1) / 2 - 1) * kSlots
                                                                                      : size_t(kPro)));
  }
};

template <int NPEND>
__device__ __forceinline__ void cp_async_wait_group() {
  asm volatile("cp.async.wait_group %0;" ::"n"(NPEND) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

template <int N, int R, int D, bool FUSED, int RD, int MINB>
__global__ void __launch_bounds__(kTmemThreads, MINB)
    twisted_tmem_v4_kernel(const WaypointParams prm, const TmemLaunchV4 tl, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = V4Layout<N, D, RD>;
  constexpr int kSlots = Lay::kSlots;
  constexpr int kPro = Lay::kPro;
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = kTmemThreads / 32;
  static_assert(RD >= 2, "ring depth");
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
  const int nmax = M - 1;

  // ---- shared memory (V4Layout): [staging x kWarps][ring RD x (1+D)][time history nmax+1][x0 stash D][region]
  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);
  double* base = reinterpret_cast<double*>(smem_raw + tmem_stage_bytes<N, D>()) + threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return base + (size_t(buf) * (1 + D) + slot) * kTmemThreads; };
  double* thist = base + size_t(Lay::kHist) * kTmemThreads;
  auto HT = [&](int j) -> double& { return thist[size_t(j) * kTmemThreads]; };
  double* x0s = thist + size_t(Lay::hist_slots(nmax)) * kTmemThreads;
  double* region = x0s + size_t(D) * kTmemThreads;  // sweep state blocks; next tile's prologue inputs
  auto SP = [&](int blk, int slot) -> double& { return region[(size_t(blk) * kSlots + slot) * kTmemThreads]; };
  auto PRO = [&](int slot) -> double* { return region + size_t(slot) * kTmemThreads; };

  const sweep::Frame<N> fr{K, half};
  const int e0 = fr.e0();

  const long long n_wtiles = (prm.B + 15) >> 4;
  const long long wt_stride = (long long)gridDim.x * kWarps;
  const bool dyn = tl.tile_counter != nullptr;
  // lane 0 draws the tile; the broadcast is deferred to the first use so that the atomic's round trip to L2
  // overlaps the sweep
  auto draw_tile = [&]() -> long long { return lane == 0 ? (long long)atomicAdd(tl.tile_counter, 1ULL) : 0; };
  long long wt = dyn ? __shfl_sync(kFull, draw_tile(), 0) : (long long)blockIdx.x * kWarps + warp;

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
    p.tt = FUSED ? nullptr : prm.times + p.traj * K;
    p.fx = FUSED ? prm.positions + p.traj * (long long)(K + 1) * D : prm.dfix + p.traj * (long long)D * nf;
    return p;
  };
  auto xaddr = [&](const Ptrs& p, int v, int d) -> const double* {
    if constexpr (FUSED) {
      return p.fx + fr.vert(v) * D + d;
    } else {
      return p.fx + d * nf + fr.pidx(v);
    }
  };
  // next tile's prologue inputs -> PRO region (cp.async; the caller commits the group)
  auto pro_issue = [&](const Ptrs& p) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      cp_async8(PRO(d), xaddr(p, 0, d));
      cp_async8(PRO(D + d), xaddr(p, 1, d));
      if constexpr (!FUSED) {
#pragma unroll
        for (int b = 0; b < m; ++b) cp_async8(PRO(2 * D + b * D + d), p.fx + d * nf + e0 + b);
      }
    }
    if constexpr (!FUSED) cp_async8(PRO(kPro - 1), p.tt + fr.seg(0));
  };
  // inputs of inward step v (time of own segment v, position of own vertex v+1) -> ring buffer v % RD
  auto ring_issue = [&](const Ptrs& p, int v) {
    const int j = v < K ? v : K - 1;
    const int vn = v + 1 <= K ? v + 1 : K;
    const int buf = v % RD;
    if constexpr (!FUSED) cp_async8(PF(buf, 0), p.tt + fr.seg(j));
#pragma unroll
    for (int d = 0; d < D; ++d) cp_async8(PF(buf, 1 + d), xaddr(p, vn, d));
  };

  if (wt < n_wtiles) {
    const Ptrs p0 = tile_ptrs(wt);
    pro_issue(p0);
    cp_async_commit();
  }

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB};

  while (wt < n_wtiles) {
    long long wt_next = dyn ? draw_tile() : wt + wt_stride;  // known one tile ahead: its prologue is prefetched
    bool next_known = !dyn;
    const Ptrs P = tile_ptrs(wt);
    const long long traj0 = wt * 16;
    const bool valid = P.valid;
    double* __restrict__ tout = (FUSED && prm.times_out != nullptr) ? prm.times_out + P.traj * K : nullptr;

    // ---- ring prefetch of the first RD-1 inward steps, then consume the prologue inputs (issued half a tile ago)
    // (a group is committed for every step even when it is empty -- steps beyond this lane's own range --
    // so that wait_group<RD-2> always means "the data of the current step has landed")
#pragma unroll
    for (int q = 1; q < RD; ++q) {
      if (q <= nh) ring_issue(P, q);
      cp_async_commit();
    }
    cp_async_wait_group<RD - 1>();

    int stat = 0;
    double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
    {
      double T0;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        xm[d] = *PRO(d);
        xc[d] = *PRO(D + d);
        x0s[size_t(d) * kTmemThreads] = xm[d];
      }
      if constexpr (FUSED) {
        T0 = nfabian_time<D>(xm, xc, prm.v_max, prm.a_max, prm.magic);
      } else {
        T0 = *PRO(kPro - 1);
      }
      if (bad_segment_time(T0)) stat |= kStatusBadTime;
      HT(0) = T0;
      const double iT0 = fast_rcp(T0);
      double pw[N - 1];
      segment_powers<N, R>(T0, iT0, pw);
      S::end_blocks(pw, Cee, cps, cpe);
      S::carry_fold(pw, [&](int b, int d) { return FUSED ? 0.0 : fr.sgn(b) * *PRO(2 * D + b * D + d); }, Wp, yp);
    }

    // ---------------------------------------------------------------- sweep towards the middle
    for (int v = 1; v <= nmax; ++v) {
      double sv[kSlots];
      if (v <= nh) {
        cp_async_wait_group<RD - 2>();
        double xn[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xn[d] = *PF(v % RD, 1 + d);
        double T;
        if constexpr (FUSED) {
          T = nfabian_time<D>(xc, xn, prm.v_max, prm.a_max, prm.magic);
        } else {
          T = *PF(v % RD, 0);
        }
        HT(v) = T;
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
#pragma unroll
      for (int i = 0; i < kSlots; ++i) SP(v - 1, i) = sv[i];
    }
    __syncwarp();

    // ---------------------------------------------------------------- middle vertex
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
    constexpr bool kEndInRing = !FUSED && (RD * (1 + D) >= m * D);
    if constexpr (kEndInRing) {
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int b = 0; b < m; ++b) cp_async8(base + size_t(b * D + d) * kTmemThreads, P.fx + d * nf + e0 + b);
      cp_async_commit();
    }
    // the next tile's prologue inputs go to the state region: issued once every state block has been read back
    auto issue_next_pro = [&]() {
      if (!next_known) {
        wt_next = __shfl_sync(kFull, wt_next, 0);
        next_known = true;
      }
      if (wt_next < n_wtiles) {  // warp-uniform
        const Ptrs pn = tile_ptrs(wt_next);
        pro_issue(pn);
        cp_async_commit();
      }
    };
    if (nmax == 0) issue_next_pro();

    for (int v = nmax; v >= 1; --v) {
      const bool act = v <= nh;
      const double T = act ? HT(v) : 1.0;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - 1, i);
      double tE[m][D];
      S::couple(pw, ed, tE);
      double sd[h][D];
      if (act) {
        double xv[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xv[d] = S::position(sv, d);
        if constexpr (FUSED) {
          if (tout != nullptr && valid) tout[fr.seg(v)] = T;
        }
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
    if (nmax > 0) issue_next_pro();  // the state region is dead only now
    {
      double sd[h][D];
      if constexpr (kEndInRing) {
        // everything except (possibly) the next tile's prologue group has landed
        if (wt_next < n_wtiles) cp_async_wait_group<1>(); else cp_async_wait_group<0>();
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        sd[0][d] = x0s[size_t(d) * kTmemThreads];
#pragma unroll
        for (int b = 0; b < m; ++b) {
          if constexpr (FUSED) {
            sd[1 + b][d] = 0.0;
          } else if constexpr (kEndInRing) {
            sd[1 + b][d] = fr.sgn(b) * base[size_t(b * D + d) * kTmemThreads];
          } else {
            sd[1 + b][d] = fr.sgn(b) * __ldg(P.fx + d * nf + e0 + b);
          }
        }
      }
      const double T = HT(0);
      if constexpr (FUSED) {
        if (tout != nullptr && valid) tout[fr.seg(0)] = T;
      }
      const double iT = fast_rcp(T);
      __syncwarp();
      out.emit(0, 0, T, iT, sd, ed, traj0);
    }
    wt = wt_next;
  }

  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
