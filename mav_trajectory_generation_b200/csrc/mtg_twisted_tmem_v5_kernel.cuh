// mtg_twisted_tmem_v5_kernel.cuh -- K1 (v5): the persistent twisted kernel with its INPUTS MOVED BY THE TMA.
//
// The whole input record of a 16-trajectory warp tile -- seg_times[16][K] and d_fixed[16][D][n_fixed], two
// contiguous spans of global memory -- is brought into shared memory by one elected lane with two cp.async.bulk
// copies completing on an mbarrier, and every lane then reads its segment times, waypoints and end derivatives
// from shared memory.  For short trajectories two tiles fit next to the coefficient staging tile and the sweep
// state, and the NEXT tile is fetched a whole tile ahead; for longer ones one tile fits, and the refill is issued
// while the last segment of the current tile is emitted.  The waypoints are not copied into the sweep state (the
// tile stays resident), which shrinks the state to 22 doubles per vertex at N = 10, D = 3.  Compared with v4 this
// removes every per-lane global load, the cp.async ring, the time history, the prologue prefetch region and their
// address arithmetic; what is left on the LSU are shared-memory accesses and the TMA descriptors.  Requirements
// (checked by the host, which otherwise launches v4): B a multiple of 16 and 16-byte aligned seg_times / d_fixed,
// so that every tile is a whole, aligned bulk copy.
// Arithmetic per trajectory is the v3/v4 sequence: results are bitwise identical.
#pragma once

#include "mtg_twisted_tmem_v4_kernel.cuh"

namespace mtg {

struct TmemLaunchV5 {
  int n_buffers;    // input tiles per warp: 2 = next tile fetched a whole tile ahead (K <= 12 at N = 10, D = 3), 1 = the
                    // state of longer trajectories leaves room for one tile only: refilled during the outward sweep
                    // (EARLY template parameter) or while the last segment is emitted
  unsigned long long* tile_counter;  // non-null: dynamic tile assignment
};

// Dynamic shared memory of v5: [staging x kWarps][mbarriers][input tiles: kWarps x nbuf][sweep state: nmax blocks]
// [FUSED: time history nmax+1].  The state blocks hold no positions: the input tile stays resident for the whole tile.
template <int N, int D, bool FUSED>
struct V5Layout {
  static constexpr int kSlots = sweep_state_slots<N, D>();
  static constexpr int kBarBytes = 128;  // two 8-byte mbarriers per warp
  // doubles of one input tile: seg_times[16][K] and d_fixed[16][D][nf], or (FUSED) positions[16][K+1][D]
  __host__ __device__ static constexpr size_t tile_times(int K) { return FUSED ? 0 : size_t(16) * K; }
  __host__ __device__ static constexpr size_t tile_fixed(int K, int nf) {
    return FUSED ? size_t(16) * (K + 1) * D : size_t(16) * D * nf;
  }
  __host__ __device__ static constexpr size_t tile_doubles(int K, int nf) { return tile_times(K) + tile_fixed(K, nf); }
  // per-thread slots behind the input tiles: nmax state blocks, then (FUSED) the time history
  __host__ __device__ static constexpr size_t hist(int nmax) { return size_t(nmax) * kSlots; }
  __host__ __device__ static constexpr size_t bytes(int K, int nf, int nbuf) {
    return tmem_stage_bytes<N, D>() + kBarBytes + size_t(kTmemThreads / 32) * nbuf * tile_doubles(K, nf) * 8 +
           tmem_slot_bytes(hist((K + 1) / 2 - 1) + (FUSED ? (K + 1) / 2 : 0));
  }
  // Early refill E (see below): parking area in the slots of the popped state blocks >= E, per lane:
  // [own step u = E..1: x_u[D], T_u][x_0[D]][u_0[D][m]][T_0]
  __host__ __device__ static constexpr int park_step(int E, int u) { return (E - u) * (D + 1); }
  __host__ __device__ static constexpr int park_x0(int E) { return E * (D + 1); }
  __host__ __device__ static constexpr int park_u0(int E) { return park_x0(E) + D; }
  __host__ __device__ static constexpr int park_T0(int E) { return park_u0(E) + (N / 2 - 1) * D; }
  __host__ __device__ static constexpr int early_stash_slots(int E) { return park_T0(E) + 1; }
  template <int E>
  __host__ __device__ static constexpr bool early_fits(int K) {
    return E <= K - (K + 1) / 2 - 1 && E <= (K + 1) / 2 - 1 &&
           size_t(E) * kSlots + early_stash_slots(E) <= size_t((K + 1) / 2 - 1) * kSlots;
  }
};

namespace bulk {
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy (bytes a multiple of 16, both addresses 16-byte aligned), completion on `bar`
__device__ __forceinline__ void copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
}  // namespace bulk

// EARLY = E > 0 (single tile buffer only): when the outward sweep reaches own vertex E, what its last E steps and the
// closing step still read from the tile ((D+1)*E + D + m*D + 1 doubles per lane) is parked in the shared-memory slots
// of state blocks that are already popped (blocks >= E), and the tile buffer is refilled with the next tile there and
// then: E back-substitution + emission steps of lead for the fetch instead of one.  The host launches this
// instantiation only when n_buffers == 1 and V5Layout::early_fits: both lanes own >= E vertices and the parking area
// lies inside the state.
template <int N, int R, int D, int MINB, bool FUSED = false, int EARLY = 0>
__global__ void __launch_bounds__(kTmemThreads, MINB)
    twisted_tmem_v5_kernel(const WaypointParams prm, const TmemLaunchV5 tl, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = V5Layout<N, D, FUSED>;
  constexpr int kSlots = Lay::kSlots;
  constexpr unsigned kFull = 0xffffffffu;
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
  const int nmax = M - 1;
  const int nbuf = tl.n_buffers;

  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);
  unsigned char* after_stage = smem_raw + tmem_stage_bytes<N, D>();
  const uint32_t bar0 = smem_u32(after_stage) + uint32_t(warp) * 16;  // two 8-byte mbarriers per warp
  // FUSED (SURVEY.md 8f-1): the tile is the waypoint record positions[16][K+1][D]; segment times are computed from it
  // (estimateSegmentTimesNfabian) and kept in a small per-thread history for the outward sweep
  const int tile_t = int(Lay::tile_times(K)), tile_f = int(Lay::tile_fixed(K, nf)), tile_doubles = tile_t + tile_f;
  double* tiles = reinterpret_cast<double*>(after_stage + Lay::kBarBytes) + size_t(warp) * nbuf * tile_doubles;
  // sweep state: state double s (block * kSlots + slot) of this thread at state[s * kTmemThreads]
  double* state =
      reinterpret_cast<double*>(after_stage + Lay::kBarBytes) + size_t(kWarps) * nbuf * tile_doubles + threadIdx.x;
  double* thist = nullptr;  // FUSED only: behind the sweep state
  if constexpr (FUSED) thist = state + Lay::hist(nmax) * kTmemThreads;
  auto TH = [&](int j) -> double& { return thist[size_t(j) * kTmemThreads]; };
  auto ST = [&](int s_global) -> double& { return state[size_t(s_global) * kTmemThreads]; };
  const sweep::Frame<N> fr{K, half};
  const int e0 = fr.e0();

  const long long n_wtiles = prm.B >> 4;  // B is a multiple of 16 (host-checked)
  const long long wt_stride = (long long)gridDim.x * kWarps;
  const bool dyn = tl.tile_counter != nullptr;
  // Dynamic assignment: the FIRST tile of every warp is its static one (no atomic in front of the first fetch); the
  // counter hands out the tiles after those, and is always drawn one tile ahead of its use so that the atomic's
  // round trip to L2 never sits in front of a fetch.
  // (inline PTX: the compiler turns atomicAdd() under `lane == 0` into its warp-aggregated form, ATOMG followed at once
  // by a SHFL of the result -- which puts the round trip back in front of the warp: 2.4 % of all stall samples)
  auto draw_tile = [&]() -> long long {
    unsigned long long old = 0;
    if (lane == 0) asm volatile("atom.global.add.u64 %0, [%1], 1;" : "=l"(old) : "l"(tl.tile_counter) : "memory");
    return (long long)old + wt_stride;
  };
  long long wt = (long long)blockIdx.x * kWarps + warp;
  long long pending = dyn ? draw_tile() : 0;  // lane 0 holds the tile after `wt`

  // one elected lane moves a whole tile: seg_times[16][K] and d_fixed[16][D][nf] are contiguous in global memory
  if (lane == 0) {
    bulk::mbar_init(bar0, 1);
    bulk::mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  auto fetch_tile = [&](long long w, int buf) {
    if (lane == 0) {
      const uint32_t bar = bar0 + 8u * buf;
      double* dst = tiles + size_t(buf) * tile_doubles;
      bulk::mbar_expect_tx(bar, uint32_t(tile_doubles) * 8u);
      if constexpr (FUSED) {
        bulk::copy_g2s(smem_u32(dst), prm.positions + w * 16 * (long long)(K + 1) * D, uint32_t(tile_f) * 8u, bar);
      } else {
        bulk::copy_g2s(smem_u32(dst), prm.times + w * 16 * K, uint32_t(tile_t) * 8u, bar);
        bulk::copy_g2s(smem_u32(dst + tile_t), prm.dfix + w * 16 * (long long)D * nf, uint32_t(tile_f) * 8u, bar);
      }
    }
  };
  if (wt < n_wtiles) fetch_tile(wt, 0);

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;
  const int tl_row = lane >> 1;  // this lane's trajectory inside the tile
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB};

  for (int it = 0; wt < n_wtiles; ++it) {
    const int buf = nbuf == 2 ? (it & 1) : 0;
    long long wt_next = dyn ? __shfl_sync(kFull, pending, 0) : wt + wt_stride;
    if (dyn) pending = draw_tile();
    if (nbuf == 2) {
      // fetch the next tile into the other buffer now: a whole tile of lead.  That buffer was read (generic proxy) by
      // the previous tile; order those reads before the asynchronous-proxy write.
      fence_proxy_async();
      __syncwarp();
      if (wt_next < n_wtiles) fetch_tile(wt_next, buf ^ 1);
    }
    bulk::mbar_wait(bar0 + 8u * buf, nbuf == 2 ? (uint32_t(it >> 1) & 1u) : (uint32_t(it) & 1u));

    const double* __restrict__ tT = tiles + size_t(buf) * tile_doubles + tl_row * K;
    const double* __restrict__ tF =
        tiles + size_t(buf) * tile_doubles + tile_t + tl_row * (FUSED ? (K + 1) * D : D * nf);
    // time of own segment j: from the tile, or (FUSED) from the history filled by the inward sweep
    auto in_T = [&](int j) -> double {
      if constexpr (FUSED) return TH(j);
      return tT[fr.seg(j)];
    };
    auto in_x = [&](int v, int d) -> double {
      if constexpr (FUSED) return tF[fr.vert(v) * D + d];
      return tF[d * nf + fr.pidx(v)];
    };
    auto in_u0 = [&](int b, int d) -> double {  // fixed end derivative b+1 of own vertex 0, own-frame sign
      if constexpr (FUSED) return 0.0;
      return fr.sgn(b) * tF[d * nf + e0 + b];
    };
    const long long traj0 = wt * 16;
    const long long traj = traj0 + tl_row;

    int stat = 0;
    double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
    {
#pragma unroll
      for (int d = 0; d < D; ++d) {
        xm[d] = in_x(0, d);
        xc[d] = in_x(1, d);
      }
      double T0;
      if constexpr (FUSED) {
        T0 = nfabian_time<D>(xm, xc, prm.v_max, prm.a_max, prm.magic);
        TH(0) = T0;
      } else {
        T0 = in_T(0);
      }
      if (bad_segment_time(T0)) stat |= kStatusBadTime;
      const double iT0 = fast_rcp(T0);
      double pw[N - 1];
      segment_powers<N, R>(T0, iT0, pw);
      S::end_blocks(pw, Cee, cps, cpe);
      S::carry_fold(pw, in_u0, Wp, yp);
    }

    // ---------------------------------------------------------------- sweep towards the middle
    for (int v = 1; v <= nmax; ++v) {
      double sv[kSlots];
      if (v <= nh) {
        double xn[D];
#pragma unroll
        for (int d = 0; d < D; ++d) xn[d] = in_x(v + 1, d);
        double T;
        if constexpr (FUSED) {
          T = nfabian_time<D>(xc, xn, prm.v_max, prm.a_max, prm.magic);
          TH(v) = T;
        } else {
          T = in_T(v);
        }
        if (bad_segment_time(T)) stat |= kStatusBadTime;
        const double iT = fast_rcp(T);
        double pw[N - 1];
        segment_powers<N, R>(T, iT, pw);

        double Dp[m][m], E[m][m], bb[m][D], L[m][m], inv[m];
        S::assemble(pw, Cee, cps, cpe, Wp, yp, xm, xc, xn, Dp, E, bb);
        S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
        S::pack(L, inv, yp, nullptr, sv);
        S::end_blocks(pw, Cee, cps, cpe);
#pragma unroll
        for (int d = 0; d < D; ++d) {
          xm[d] = xc[d];
          xc[d] = xn[d];
        }
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < kSlots; ++i) ST((v - 1) * kSlots + i) = sv[i];
    }
    __syncwarp();

    // ---------------------------------------------------------------- middle vertex
    double um[m][D];
    S::middle(Cee, cps, cpe, Wp, yp, xm, xc, um, stat);
    if (half == 0 && prm.status != nullptr) prm.status[traj] = stat;

    // ---------------------------------------------------------------- outward back-substitution
    const int np = (K - 1) * m;
    double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + traj * (long long)D * np : nullptr;
    auto store_free = [&](int v_own, const double (&u)[h][D]) {
      if (df != nullptr) {
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

    constexpr int kStash0 = EARLY * kSlots;  // state slots of the blocks >= EARLY: popped when the sweep reaches vertex EARLY
    auto park = [&](int slot, double val) { ST(kStash0 + slot) = val; };
    for (int v = nmax; v >= 1; --v) {
      if constexpr (EARLY > 0) {
        if (v == EARLY) {
          // park what steps EARLY..1 and the closing step read from the tile, then refill the tile buffer now
#pragma unroll
          for (int u = EARLY; u >= 1; --u) {
#pragma unroll
            for (int d = 0; d < D; ++d) park(Lay::park_step(EARLY, u) + d, in_x(u, d));
            park(Lay::park_step(EARLY, u) + D, in_T(u));
          }
#pragma unroll
          for (int d = 0; d < D; ++d) park(Lay::park_x0(EARLY) + d, in_x(0, d));
#pragma unroll
          for (int d = 0; d < D; ++d)
#pragma unroll
            for (int b = 0; b < m; ++b) park(Lay::park_u0(EARLY) + d * m + b, in_u0(b, d));
          park(Lay::park_T0(EARLY), in_T(0));
          fence_proxy_async();
          __syncwarp();
          if (wt_next < n_wtiles) fetch_tile(wt_next, 0);
        }
      }
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = ST((v - 1) * kSlots + i);
      const bool act = v <= nh;
      double T = 1.0, iT = 1.0;
      double sd[h][D];
      if (act) {
        double xv[D];
        if (EARLY > 0 && v <= EARLY) {
          const int s0 = kStash0 + Lay::park_step(EARLY, v);
#pragma unroll
          for (int d = 0; d < D; ++d) xv[d] = ST(s0 + d);
          T = ST(s0 + D);
        } else {
#pragma unroll
          for (int d = 0; d < D; ++d) xv[d] = in_x(v, d);
          T = in_T(v);
        }
        if constexpr (FUSED) {
          if (prm.times_out != nullptr) prm.times_out[traj * K + fr.seg(v)] = T;
        }
        iT = fast_rcp(T);
        double pw[N - 1];
        segment_powers<N, R>(T, iT, pw);
        double tE[m][D];
        S::couple(pw, ed, tE);
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
    {
      double sd[h][D];
      double T;
      if constexpr (EARLY > 0) {
#pragma unroll
        for (int d = 0; d < D; ++d) {
          sd[0][d] = ST(kStash0 + Lay::park_x0(EARLY) + d);
#pragma unroll
          for (int b = 0; b < m; ++b) sd[1 + b][d] = ST(kStash0 + Lay::park_u0(EARLY) + d * m + b);
        }
        T = ST(kStash0 + Lay::park_T0(EARLY));
      } else {
#pragma unroll
        for (int d = 0; d < D; ++d) {
          sd[0][d] = in_x(0, d);
#pragma unroll
          for (int b = 0; b < m; ++b) sd[1 + b][d] = in_u0(b, d);
        }
        T = in_T(0);
      }
      if constexpr (FUSED) {
        if (prm.times_out != nullptr) prm.times_out[traj * K + fr.seg(0)] = T;
      }
      const double iT = fast_rcp(T);
      if (EARLY == 0 && nbuf == 1) {
        // single buffer: every input of this tile is in registers now -- refill it with the next tile while the last
        // segment is emitted
        fence_proxy_async();
        __syncwarp();
        if (wt_next < n_wtiles) fetch_tile(wt_next, 0);
      }
      __syncwarp();
      out.emit(0, 0, T, iT, sd, ed, traj0);
    }
    wt = wt_next;
  }

  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
