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
  constexpr bool LSEARCH = false;
#include "mtg_twisted_tmem_body.cuh"
}

// The cost-only form with the line-search time generator (the Mellinger outer loop's candidates, WaypointParams)
template <int N, int R, int D>
__global__ void __launch_bounds__(kTmemThreads, (N <= 8 ? 3 : 2))
    twisted_tmem_line_search_kernel(const WaypointParams prm, const __grid_constant__ CUtensorMap tmap) {
  constexpr bool FUSED = false, COST = true, LSEARCH = true;
#include "mtg_twisted_tmem_body.cuh"
}

}  // namespace mtg
