// mtg_twisted_tmem_kernel.cuh -- K1 (v3): twisted two-lanes-per-trajectory sweep with the
// per-thread sweep state held in shared memory and coalesced output.
//
// The sweep state (L_v, inverse pivots, y_v and the vertex position per eliminated vertex; 25 doubles
// per vertex for N=10, D=3) is what bounds the number of trajectories in flight per SM.  It lives in
// shared memory as [vertex][slot][thread] (consecutive threads hit consecutive banks); the host only
// routes a K to this kernel when two CTAs fit on an SM, longer trajectories take the chunked kernel.
//
// Output: each lane writes the D*N coefficients of the segment it has just solved into its row of a
// 128-byte aligned per-warp staging tile ([half][16 trajectories][D*N doubles]); one elected lane then hands
// the two 16-row boxes (forward halves: segment j, reversed halves: segment K-1-j) to the TMA with
// cp.async.bulk.tensor.2d stores against a tensor map of coeffs viewed as [B][K*D*N].  No cooperative
// read-back, no global-store LSU wavefronts, and the ragged last tile is clipped by the tensor map.
//
// Inputs: every lane prefetches the next step's segment time and waypoint with cp.async into a small
// per-thread ring (a register prefetch would share its scoreboard slot with the value being consumed); the
// outward sweep re-reads times from a per-thread shared-memory history and positions from the sweep state.
//
// Mathematics, frames and index maps: see mtg_twisted_kernel.cuh.
#pragma once

#include <cuda.h>  // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)

#include "mtg_twisted_kernel.cuh"

namespace mtg {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

constexpr int kTmemThreads = 128;

// coefficient staging tiles of the warps of a CTA at the start of dynamic shared memory: one whole segment (D*N
// contiguous output doubles) per lane, i.e. two 16-row TMA boxes per warp
template <int N, int D, int kThreads = kTmemThreads>
__host__ __device__ constexpr size_t tmem_stage_bytes() {
  return size_t(kThreads / 32) * 32 * D * (N / 2) * 16;
}
// bytes of `slots` per-thread doubles (slot s of thread t at double s * kThreads + t)
__host__ __device__ constexpr size_t tmem_slot_bytes(size_t slots, int kThreads = kTmemThreads) {
  return slots * kThreads * 8;
}

// Dynamic shared memory of v3 (and its cost-only instantiation) behind the staging tiles, in per-thread slots:
// [prefetch ring 2 x (1+D)][time history nmax+1][sweep state: nmax blocks with the vertex position]
template <int N, int D>
struct V3Layout {
  static constexpr int kSlots = sweep_state_slots<N, D, true>();
  static constexpr int kHist = 2 * (1 + D);                                 // ring, then the time history
  __host__ __device__ static constexpr int hist_slots(int nmax) { return nmax + 1; }  // history, then the state
  __host__ __device__ static constexpr size_t state(int nmax) { return size_t(kHist) + hist_slots(nmax); }
  __host__ __device__ static constexpr size_t bytes(int K) {
    return tmem_stage_bytes<N, D>() + tmem_slot_bytes(state((K + 1) / 2 - 1) + size_t((K + 1) / 2 - 1) * kSlots);
  }
};

__device__ __forceinline__ void cp_async8(const double* smem_dst, const double* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// cp_async8 that, when `evict_first`, marks the line evict-first in L2: for inputs read once, so that they do not
// push out data that is read again (the chunked kernel's parking area)
__device__ __forceinline__ void cp_async8_stream(const double* smem_dst, const double* gsrc, int evict_first) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b64 pol;\n\t"
      "setp.ne.b32 p, %2, 0;\n\t"
      "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
      "@p cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 8, pol;\n\t"
      "@!p cp.async.ca.shared.global [%0], [%1], 8;\n\t}" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(evict_first)
      : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// TMA tensor store of a [16 rows][D*N doubles] shared-memory box to coeffs viewed as a 2-D tensor
// [B trajectories][K*D*N doubles]: (c0 = first double inside the trajectory, c1 = first trajectory).  Rows
// beyond the tensor (ragged last tile) are clipped by the hardware.
__device__ __forceinline__ void tma_store_box(const CUtensorMap* tmap, const void* ssrc, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_u32(ssrc)), "r"(c0), "r"(c1)
               : "memory");
}
// the same store with the written lines marked evict-first in L2 (the output is not read again by the kernel)
__device__ __forceinline__ void tma_store_box_evict_first(const CUtensorMap* tmap, const void* ssrc, int c0, int c1) {
  asm volatile(
      "{\n\t.reg .b64 pol;\n\t"
      "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], pol;\n\t}" ::"l"(
          reinterpret_cast<uint64_t>(tmap)),
      "r"(smem_u32(ssrc)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Output of the twisted TMA kernels: each lane writes the D*N doubles of the segment it emits into row (half*16 +
// trajectory) of the warp's staging tile; one elected lane hands the two 16-row boxes (forward halves: segment j,
// reversed halves: segment K-1-j) to the TMA.  No cooperative read-back and no global-store LSU wavefronts.
template <int N, int D, class AI>
struct TmaEmitter {
  static constexpr int h = N / 2;
  const CUtensorMap* tmap;
  double2* stage;   // this warp's staging tile [half][16][D*h]
  double2* my_row;  // this lane's row of it
  int lane, K;
  int nhF, nhB;  // a half is active in sweep step v iff v <= its nh
  bool evict_first = false;  // stores marked evict-first in L2 (the chunked kernel keeps its parking area in L2)
  __device__ __forceinline__ void store(const void* ssrc, int c0, int c1) const {
    if (evict_first) tma_store_box_evict_first(tmap, ssrc, c0, c1);
    else tma_store_box(tmap, ssrc, c0, c1);
  }
  // emit own-frame segment j for every lane of the warp at once (convergent); v_step: the sweep step (0 = final).
  // Rows of lanes that are not active in v_step are not stored.
  __device__ __forceinline__ void emit(int j, int v_step, double T, double iT, const double (&sd)[h][D],
                                       const double (&ed)[h][D], long long traj0) const {
    using HF = sweep::Hermite<N, AI>;
    const int half = lane & 1;
    double tp[h], itp[h];
    HF::powers(T, iT, half, tp, itp);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double c[N];
      HF::template coeffs<D>(half, tp, itp, sd, ed, d, c);
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
      if (v_step <= nhF) store(stage, j * (D * N), (int)traj0);
      if (v_step <= nhB) store(stage + 16 * (D * h), (K - 1 - j) * (D * N), (int)traj0);
      bulk_commit();
    }
  }
};

template <int N, int R, int D, bool FUSED = false, bool COST = false>
__global__ void __launch_bounds__(kTmemThreads, (N <= 8 ? 3 : 2))
    twisted_tmem_kernel(const WaypointParams prm, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = V3Layout<N, D>;
  // per eliminated vertex: L (strictly lower) + inverse pivots + y + the vertex position (so that the
  // outward sweep does not re-read it from global memory)
  constexpr int kSlots = Lay::kSlots;
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = kTmemThreads / 32;
  using G = H1Imm<N, R>;     // immediates: this kernel is register-bound (see mtg_device.cuh)
  using AI = A1InvImm<N>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ __align__(128) unsigned char smem_raw[];  // TMA tensor stores need 128-byte aligned tiles
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int half = lane & 1;
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;
  const int nh = half ? K - M - 1 : M - 1;
  const int nmax = M - 1;
  const sweep::Frame<N> fr{K, half};

  // ---- shared memory carve-up (V3Layout): [staging: kWarps tiles][prefetch ring][time history][sweep state]
  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);  // [half][16][D*h]
  // per-thread prefetch ring for the next step's inputs (segment time + D positions), filled by
  // cp.async: a register prefetch would share its scoreboard slot with the load being consumed and the
  // consumer would wait for the NEW loads as well (measured: 25 % of all stall samples).
  double* pf = reinterpret_cast<double*>(smem_raw + tmem_stage_bytes<N, D>()) + threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return pf + (size_t(buf) * (1 + D) + slot) * kTmemThreads; };
  // per-thread history of the own-frame segment times seen by the inward sweep (nmax+1 doubles): the
  // outward sweep reads them back from shared memory (in FUSED mode this also saves the sqrt/exp)
  double* thist = pf + size_t(Lay::kHist) * kTmemThreads;
  auto HT = [&](int j) -> double& { return thist[size_t(j) * kTmemThreads]; };
  double* state = thist + size_t(Lay::hist_slots(nmax)) * kTmemThreads;
  auto SP = [&](int blk, int slot) -> double& { return state[(size_t(blk) * kSlots + slot) * kTmemThreads]; };

  const long long traj0 = ((long long)blockIdx.x * kWarps + warp) * 16;  // first trajectory of this warp
  long long traj = traj0 + (lane >> 1);
  const bool valid = traj < prm.B;
  if (!valid) traj = prm.B - 1;

  // cost-only mode with the Mellinger expansion generated on the fly: inputs come from the base trajectory
  long long src = traj;
  int mel_n = -1;
  double mel_corr = 0.0;
  if constexpr (COST) {
    if (prm.mel_k1 > 0) {
      src = traj / prm.mel_k1;
      mel_n = int(traj - src * prm.mel_k1) - 1;
      mel_corr = prm.mel_inc / (K - 1.0);
    }
  }
  auto time_of = [&](double raw, int seg_index) -> double {  // seg_index: ORIGINAL segment index
    if constexpr (COST) return mellinger_time(raw, seg_index, mel_n, prm.mel_inc, mel_corr, prm.mel_lower);
    return raw;
  };
  const double* __restrict__ tt = FUSED ? nullptr : prm.times + src * K;
  const double* __restrict__ fx =
      FUSED ? prm.positions + src * (long long)(K + 1) * D : prm.dfix + src * (long long)D * nf;
  // address of coordinate d of own-frame vertex v
  auto xaddr = [&](int v, int d) -> const double* {
    if constexpr (FUSED) {
      return fx + fr.vert(v) * D + d;
    } else {
      return fx + d * nf + fr.pidx(v);
    }
  };
  // prefetch (time of own segment j, position of own vertex v) into ring buffer `buf`
  auto pf_issue = [&](int buf, int j, int v) {
    if constexpr (!FUSED) cp_async8(PF(buf, 0), tt + fr.seg(j));
#pragma unroll
    for (int d = 0; d < D; ++d) cp_async8(PF(buf, 1 + d), xaddr(v, d));
  };
  double* __restrict__ tout = (FUSED && prm.times_out != nullptr) ? prm.times_out + traj * K : nullptr;

  // ---- issue the first global loads NOW: their latency overlaps the index set-up below
  double T0e = 0.0, x0e[D], x1e[D], u0e[m][D];
  {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      x0e[d] = __ldg(xaddr(0, d));
      x1e[d] = __ldg(xaddr(1, d));
#pragma unroll
      for (int b = 0; b < m; ++b) u0e[b][d] = FUSED ? 0.0 : __ldg(fx + d * nf + fr.e0() + b);
    }
    if constexpr (!FUSED) T0e = __ldg(tt + fr.seg(0));
    pf_issue(1, 1, 2);  // inputs of sweep step v = 1 -> ring buffer (v & 1)
  }

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;  // a half is active in sweep step v iff v <= its nh
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB};

  double cost_acc = 0.0;
  auto emit_all = [&](int j, int v_step, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D]) {
    if constexpr (COST) {
      // 0.5 d^T H(T) d of this segment, d = [start derivatives; end derivatives] in the own frame (the cost is
      // invariant under the time reversal of the odd half): H = T^(1-2r) S G S / scale, S = diag(T^(s mod h)).
      (void)j;
      const int nh_own = half ? nhB : nhF;
      if (v_step <= nh_own) {
        double tp[h];
        tp[0] = 1.0;
#pragma unroll
        for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * T;
        double q = 0.0;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          double u[N];
#pragma unroll
          for (int k = 0; k < h; ++k) {
            u[k] = tp[k] * sd[k][d];
            u[h + k] = tp[k] * ed[k][d];
          }
#pragma unroll
          for (int s2 = 0; s2 < N; ++s2) {
            double row = 0.5 * G::at(s2, s2) * u[s2];
#pragma unroll
            for (int t2 = s2 + 1; t2 < N; ++t2) row = fma(G::at(s2, t2), u[t2], row);
            q = fma(row, u[s2], q);
          }
        }
        // T^(1-2r) = T * (1/T)^(2r)
        cost_acc = fma(q, T * pow_int<2 * R>(iT), cost_acc);
      }
      return;
    }
    out.emit(j, v_step, T, iT, sd, ed, traj0);
  };

  int stat = 0;
  double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], bcar[m][D], xm[D], xc[D];
  {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      xm[d] = x0e[d];
      xc[d] = x1e[d];
    }
    double T0;
    if constexpr (FUSED) {
      T0 = nfabian_time<D>(xm, xc, prm.v_max, prm.a_max, prm.magic);
    } else {
      T0 = time_of(T0e, fr.seg(0));
    }
    if (bad_segment_time(T0)) stat |= kStatusBadTime;
    HT(0) = T0;
    const double iT0 = fast_rcp(T0);
    double pw[N - 1];
    segment_powers<N, R>(T0, iT0, pw);
    S::end_blocks(pw, Cee, cps, cpe);
    S::carry_bcar(pw, [&](int b, int d) { return fr.sgn(b) * u0e[b][d]; }, Wp, yp, bcar);
  }

  // ---------------------------------------------------------------- sweep towards the middle
  for (int v = 1; v <= nmax; ++v) {
    double sv[kSlots];  // lanes with v > nh store whatever is here; they never read it back
    if (v <= nh) {
      cp_async_wait_all();
      double xn[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xn[d] = *PF(v & 1, 1 + d);
      double T;
      if constexpr (FUSED) {
        T = nfabian_time<D>(xc, xn, prm.v_max, prm.a_max, prm.magic);
      } else {
        T = time_of(*PF(v & 1, 0), fr.seg(v));
      }
      HT(v) = T;
      {  // prefetch the next step's inputs (clamped indices: never out of bounds)
        const int jn = v + 1 < K ? v + 1 : K - 1;
        const int vn = v + 2 <= K ? v + 2 : K;
        pf_issue((v + 1) & 1, jn, vn);
      }
      if (bad_segment_time(T)) stat |= kStatusBadTime;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);

      double Dp[m][m], E[m][m], bb[m][D], L[m][m], inv[m];
      S::assemble(pw, Cee, cps, cpe, bcar, Wp, yp, xm, xc, xn, Dp, E, bb);
      S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
      S::pack(L, inv, yp, xc, sv);  // with the position of the vertex just eliminated
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
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kSlots; ++i) SP(v - 1, i) = sv[i];
  }
  __syncwarp();

  // ---------------------------------------------------------------- middle vertex
  double um[m][D];
  S::middle(Cee, cps, cpe, bcar, Wp, yp, xm, xc, um, stat);
  if (valid && half == 0 && prm.status != nullptr) prm.status[traj] = stat;

  // ---------------------------------------------------------------- outward back-substitution
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

  double ed[h][D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ed[0][d] = xc[d];
#pragma unroll
    for (int j = 0; j < m; ++j) ed[1 + j][d] = um[j][d];
  }
  if (half == 0) store_free(nh + 1, ed);

  // outward steps take the vertex position from the sweep state; only the segment time is prefetched
  // (and the position of own vertex 0 for the final emission)
  auto pf_issue_out = [&](int j) {
    if (j == 0) pf_issue(0, 0, 0);  // position of own vertex 0 for the final emission (time comes from HT)
  };
  pf_issue_out(nh);

  for (int v = nmax; v >= 1; --v) {
    double sv[kSlots];
#pragma unroll
    for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - 1, i);
    const bool act = v <= nh;
    double T = 1.0, iT = 1.0;
    double sd[h][D];  // inactive lanes (odd K only) emit garbage rows that are never stored
    if (act) {
      cp_async_wait_all();
      double xv[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xv[d] = S::position(sv, d);
      T = HT(v);
      if constexpr (FUSED) {
        if (tout != nullptr && valid) tout[fr.seg(v)] = T;
      }
      pf_issue_out(v - 1);
      if constexpr (!FUSED) {
        if (v == 1) {  // the final emission re-reads the fixed end derivatives: pull their lines into L1 now
#pragma unroll
          for (int d = 0; d < D; ++d) asm volatile("prefetch.global.L1 [%0];" ::"l"(fx + d * nf + fr.e0()));
        }
      }
      iT = fast_rcp(T);
      double L[m][m], inv[m], rhs[m][D], pw[N - 1];
      S::unpack(sv, L, inv, rhs);
      segment_powers<N, R>(T, iT, pw);
      S::uncouple_from(pw, ed, L, inv, rhs);
      S::solve_back(L, inv, rhs, xv, sd);
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
  {
    cp_async_wait_all();
    double sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      sd[0][d] = *PF(0, 1 + d);
#pragma unroll
      for (int b = 0; b < m; ++b) sd[1 + b][d] = FUSED ? 0.0 : fr.sgn(b) * __ldg(fx + d * nf + fr.e0() + b);
    }
    const double T = HT(0);
    if constexpr (FUSED) {
      if (tout != nullptr && valid) tout[fr.seg(0)] = T;
    }
    const double iT = fast_rcp(T);
    __syncwarp();
    emit_all(0, 0, T, iT, sd, ed);
  }

  if constexpr (COST) {
    // q accumulated sum_{s<=t} (1 or 1/2) G u u = 0.5 u^T G u per segment: cost = sum over both halves / scale
    const double other = __shfl_xor_sync(kFull, cost_acc, 1);
    if (valid && half == 0 && prm.cost != nullptr) prm.cost[traj] = (cost_acc + other) * (1.0 / G::scale);
  }
  if (lane == 0) bulk_wait_all();  // every TMA store issued by this warp has completed
}

}  // namespace mtg
