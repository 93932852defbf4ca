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

#include "mtg_twisted_tmem_v5_kernel.cuh"

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
  using AI = A1InvImm<N>;
  using Tile = sweep::Tile<N, R, D>;

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

    int stat;
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
      Tile::first_segment(T0, [&](int b, int d) { return fr.sgn(b) * *PRO(2 * D + b * D + d); }, stat, Wp, yp, Cee,
                          cps, cpe);
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
        Tile::inward_step(T, xn, stat, Wp, yp, Cee, cps, cpe, xm, xc, sv);
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
    double ed[h][D];
    Tile::meet(stat, Wp, yp, Cee, cps, cpe, xm, xc, ed);
    if (valid && half == 0 && prm.status != nullptr) prm.status[P.traj] = stat;

    // ---------------------------------------------------------------- outward back-substitution
    const sweep::FreeStore<N, D> store_free(prm.dfree, P.traj, valid, fr);
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
      double tE[m][D];  // E_v u_{v+1} (before the activity test: this kernel runs at the register limit)
      const double iT = Tile::outward_couple(T, ed, tE);
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = *SP(b, i);
      double sd[h][D];
      if (act) {
        Tile::outward_solve(sv, tE, sd);
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
      if (act) Tile::advance(ed, sd);
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

// ---- K3 in warp pairs ---------------------------------------------------------------------------------------------
// A 64-thread CTA runs the tiles blockIdx.x, blockIdx.x + gridDim.x, ... of K3 with two warps in lockstep: warp 0
// (inward) runs tile j's prologue, inward sweep and middle vertex while warp 1 (outward) runs tile j-1's outward
// sweep and final segment.  Lane l of both warps works on the same trajectory lane and the same column of shared
// memory, and both call the sweep functions of the one-warp kernel with the same arguments in the same order, so
// the results are bitwise equal to it.
//
// The two tiles in flight share one tile's C resident blocks.  The outward sweep of tile j-1 pops vertex n-k+1 at
// its k-th step; for k > n-C that pop leaves its slot empty (no parked block is refilled into it), and block k of
// tile j -- the first one that is not parked -- takes exactly that slot.  So the slot of vertex v alternates with the
// tile's parity: (v-1) % C on even tiles, (n-v) % C on odd ones.  Parked blocks stay the outer ones of each tile
// (the refill distance stays C-1 steps) and the parking area has one half per parity.
//
// Inputs: the inward warp reads everything from a tile input buffer that holds the tile's seg_times[16][K] and
// d_fixed[16][D][n_fixed] exactly as they lie in global memory.  A whole tile with 16-byte aligned inputs arrives by
// two cp.async.bulk copies (which bypass L1, so the pairs do not compete with their own input lines for it); the
// ragged last tile, or unaligned inputs, fill the same layout with per-lane 8-byte cp.async copies, rows past B
// repeating row B-1.  The buffer is refilled with the next tile once the inward sweep has read its last input, so
// the copy lands while the middle vertex is solved.  Before that refill the inward warp copies what the outward
// warp's final segment reads (x0, u0, T0 of own vertex 0) into END.
//
// Handshakes (mbarriers):
//   freed[s]  outward -> inward, one arrival per lane: the slot s has been read for the last time in this tile; the
//             slot of vertex 1, popped last, is released only after the final segment has read END, so that END is
//             free when the inward warp fills it after step n (which waits for that slot)
//   ready     inward -> outward, one arrival per lane: the middle vertex is done and the handoff (starting ed of each
//             lane) and END written
//   full      the tile buffer holds the next tile: transaction count of the bulk copies (one arrival), or the
//             per-lane copies tracked by cp.async.mbarrier.arrive (one arrival once every lane has issued them)
// Neither side can run two phases ahead of the other: tile j's inward step n waits for tile j-1's last pop, which
// follows that tile's wait on `ready` and the landing of all its refills; this needs n >= 1 (K >= 3).
// tests/test_k3_pair_schedule.py walks this schedule on the host.
//
// Output: TmaPairEmitter, or TmaEmitter where the staging of TmaPairEmitter does not fit (ChunkedPairLayout).
//
// RD does not enter the paired form (it has no input ring): it is the ring depth of the one-warp instantiations
// built beside it, kept in the name so that each registry row has one paired kernel of a fixed name.
template <int N, int D, int RD>
struct ChunkedPairLayout {
  static constexpr int h = N / 2;
  static constexpr int m = h - 1;
  static constexpr int kSlots = sweep_state_slots<N, D, true>();
  static constexpr int kPark = kSlots + 1;
  static constexpr int kEnd = D + m * D + 1;         // outward warp: x0, u0[m], T0 of the final segment
  static constexpr int kHand = h * D;                // handoff: the starting ed of the outward sweep
  static constexpr int kMaxChunk = 30;               // mbarriers: freed[C], ready, full
  static constexpr size_t kBarBytes = 8 * (kMaxChunk + 2);
  static constexpr int end = 0;
  static constexpr int hand = end + kEnd;
  static constexpr int times = hand + kHand;         // then C slot times, then C blocks
  // The outward warp stores two segments per box (TmaPairEmitter) from two buffers of [half][16 rows][two segments],
  // four times the staging of one segment per box (TmaEmitter).  It does so where two CTAs per SM still fit with that
  // staging at K = 16 with all 7 blocks of a lane resident: the default route runs the paired form there at two pairs
  // per SM (plan_chunked), and the wider staging must not push a shape off it.  That holds up to D*N = 32; N = 10 at
  // D = 4 and N = 12 at D >= 3 store one segment per box.
  static constexpr size_t kTile = tmem_stage_bytes<N, D, 32>();
  static constexpr size_t kPairCtaAtK16 = 4 * kTile + kBarBytes + 8 * (16 * 16 + 16 * D * (2 * h + 15)) +
                                          tmem_slot_bytes(times + 7 + 7 * kSlots, 32);
  static constexpr bool kStorePairs = 2 * (kPairCtaAtK16 + 1024) <= 228 * 1024;
  static constexpr size_t stage_bytes = (kStorePairs ? 4 : 1) * kTile;
  static constexpr size_t tile_offset = stage_bytes + kBarBytes;      // 16-byte aligned: the bulk copies land here
  static_assert(tile_offset % 16 == 0, "tile input buffer alignment");
  // doubles of the tile input buffer: seg_times[16][K], then d_fixed[16][D][nf] (both multiples of 16 bytes)
  __host__ __device__ static constexpr size_t tile_doubles(int K, int nf) { return size_t(16) * K + size_t(16) * D * nf; }
  __host__ __device__ static constexpr size_t region(int C) { return size_t(times) + C; }
  __host__ __device__ static constexpr size_t bytes(int C, int K, int nf) {
    return tile_offset + tile_doubles(K, nf) * 8 + tmem_slot_bytes(region(C) + size_t(C) * kSlots, 32);
  }
};

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// the mbarrier's current phase also waits for every cp.async this thread has issued so far (its pending count is
// raised by one now and lowered when they have landed)
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// bulk::mbar_wait with the loop in C++, so that one kernel can wait at several places
__device__ __forceinline__ void mbar_wait_parity(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done)
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
}

// waits until at most one bulk group of this thread is still reading shared memory
__device__ __forceinline__ void bulk_wait_read_1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }

// Output of the paired kernel's outward warp.  A half stores its segments in boxes of two consecutive global
// segments (2i, 2i+1): 16 rows x 2*D*N doubles against `tmap2`.  Its pieces are 16*D*N bytes apart, so at N = 10,
// D = 3 and even K every one starts on a 32-byte sector of the output (one segment, 240 bytes, starts every other
// one 16 bytes into a sector, and its neighbour follows a step later).  The forward half emits ..., 3, 2 | 1, 0 and the backward half M, M+1 | ... | K-2, K-1 (M = ceil(K/2)); a
// segment whose partner belongs to the other half (n even; M odd; K-1 even) is stored alone, 16 rows x D*N against
// `tmap`.  Each half alternates between two staging buffers box by box, and lane `half` issues its half's stores
// into its own bulk groups (one per box), so the first write of a box waits only until the store of the box before
// the last one has read its buffer.
template <int N, int D, class AI>
struct TmaPairEmitter {
  static constexpr int h = N / 2;
  static constexpr int kSeg = D * h;  // double2 of one segment
  const CUtensorMap* tmap;            // box 16 x D*N
  const CUtensorMap* tmap2;           // box 16 x 2*D*N
  double2* stage;                     // the warp's staging [buffer][half][16 rows][2 * kSeg]
  int lane, K;
  int nh;                             // this lane's half is active in sweep step v iff v <= nh
  bool evict_first;                   // stores marked evict-first in L2
  int nbox = 0;                       // boxes stored by this lane's half (its buffer is nbox % 2)
  __device__ __forceinline__ void store(const CUtensorMap* map, const void* ssrc, int c0, int c1) const {
    if (evict_first) tma_store_box_evict_first(map, ssrc, c0, c1);
    else tma_store_box(map, ssrc, c0, c1);
  }
  // emit own-frame segment v (sweep step v; 0 = final) for every lane of the warp at once (convergent)
  __device__ __forceinline__ void emit(int v, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D],
                                       long long traj0) {
    using HF = sweep::Hermite<N, AI>;
    const int half = lane & 1;
    const int g = half ? K - 1 - v : v;  // global segment
    const bool act = v <= nh;
    const bool next = (g & 1) != half;  // the partner g^1 is this half's segment of step v-1 (else of step v+1)
    const bool open = act && next && v >= 1;
    const bool close = act && !next && v + 1 <= nh;
    double2* buf = stage + size_t((nbox & 1) * 2 + half) * 16 * (2 * kSeg);
    double2* row = open || close ? buf + (lane >> 1) * (2 * kSeg) + (g & 1) * kSeg : buf + (lane >> 1) * kSeg;
    double tp[h], itp[h];
    HF::powers(T, iT, half, tp, itp);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double c[N];
      HF::template coeffs<D>(half, tp, itp, sd, ed, d, c);
      if (d == 0) {  // a box's buffer is free once the store of the box before the last one has read it
        if (lane == half && act && !close) bulk_wait_read_1();
        __syncwarp();
      }
      if (act) {
#pragma unroll
        for (int q = 0; q < h; ++q) row[d * h + q] = make_double2(c[2 * q], c[2 * q + 1]);
      }
    }
    fence_proxy_async();
    __syncwarp();
    if (act && !open) {
      if (lane == half) {
        if (close) store(tmap2, buf, (g & ~1) * (D * N), (int)traj0);
        else store(tmap, buf, g * (D * N), (int)traj0);
        bulk_commit();
      }
      ++nbox;
    }
  }
};

// 64 threads, at most 4 CTAs per SM by registers (cap 255)
template <int N, int R, int D, int RD>
__global__ void __launch_bounds__(64, 4)
    twisted_chunked_pair_kernel(const WaypointParams prm, const ChunkedLaunch cl,
                                const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap2) {
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = ChunkedPairLayout<N, D, RD>;
  constexpr int kSlots = Lay::kSlots;
  constexpr int kPark = Lay::kPark;
  using G = H1Imm<N, R>;
  using AI = A1InvImm<N>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = int(threadIdx.x & 31);
  const bool inward = threadIdx.x < 32;
  const int half = lane & 1;
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;
  const int nh = half ? K - M - 1 : M - 1;
  const int n = M - 1;
  const int C = cl.chunk;
  const int npark = n - C;

  double2* stage = reinterpret_cast<double2*>(smem_raw);
  // freed[s] at bar0 + 8 s, ready at bar0 + 8 C, full at bar0 + 8 (C + 1)
  const uint32_t bar0 = smem_u32(smem_raw + Lay::stage_bytes);
  const uint32_t ready = bar0 + 8u * uint32_t(C);
  const uint32_t full = ready + 8u;
  const int tile_t = 16 * K, tile_f = 16 * D * nf;
  double* tile = reinterpret_cast<double*>(smem_raw + Lay::tile_offset);
  double* base = tile + tile_t + tile_f + lane;
  auto SL = [&](int slot) -> double* { return base + size_t(slot) * 32; };
  auto END = [&](int slot) -> double* { return SL(Lay::end + slot); };
  auto HAND = [&](int slot) -> double* { return SL(Lay::hand + slot); };
  auto HT = [&](int b) -> double* { return SL(Lay::times + b); };
  auto SP = [&](int blk, int slot) -> double* { return SL(int(Lay::region(C)) + blk * kSlots + slot); };
  // slot of vertex v in the j-th tile of this CTA
  auto slot_of = [&](int v, long long j) -> int { return (j & 1) ? (n - v) % C : (v - 1) % C; };

  if (threadIdx.x == 0) {
    for (int s = 0; s <= C; ++s) bulk::mbar_init(bar0 + 8u * uint32_t(s), 32);
    bulk::mbar_init(full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const sweep::Frame<N> fr{K, half};
  const int e0 = fr.e0();
  const long long n_wtiles = (prm.B + 15) >> 4;
  const long long wt_stride = gridDim.x;
  const long long gthreads = (long long)gridDim.x * 64;
  // parking column of this lane in the half of tile parity p
  auto PK = [&](long long j, int b, int slot) -> double* {
    return cl.ckpt + ((long long)b * kPark + slot) * gthreads + ((long long)blockIdx.x * 64 + (j & 1) * 32 + lane);
  };
  // this lane's trajectory in warp tile w (past B: row B-1, whose results are not stored)
  struct Row {
    long long traj;
    bool valid;
  };
  auto row_of = [&](long long w) -> Row {
    Row r;
    r.traj = w * 16 + (lane >> 1);
    r.valid = r.traj < prm.B;
    if (!r.valid) r.traj = prm.B - 1;
    return r;
  };
  const int np = (K - 1) * m;

  if (inward) {
    // ================================================================ warp 0: prologue, inward sweep, middle
    const bool inputs_a16 = ((reinterpret_cast<uintptr_t>(prm.times) | reinterpret_cast<uintptr_t>(prm.dfix)) & 15u) == 0;
    // warp tile w -> the tile buffer, completing the current phase of `full`
    auto fill = [&](long long w) {
      const double* gt = prm.times + w * tile_t;
      const double* gf = prm.dfix + w * (long long)tile_f;
      // the reads of the last tile (generic proxy) before the writes of the bulk copies (async proxy)
      fence_proxy_async();
      __syncwarp();
      if (inputs_a16 && (w + 1) * 16 <= prm.B) {  // warp-uniform
        if (lane == 0) {
          bulk::mbar_expect_tx(full, uint32_t(tile_t + tile_f) * 8u);
          bulk::copy_g2s(smem_u32(tile), gt, uint32_t(tile_t) * 8u, full);
          bulk::copy_g2s(smem_u32(tile + tile_t), gf, uint32_t(tile_f) * 8u, full);
        }
      } else {
        // element i of the buffer is element i of the tile's inputs; in rows past B, the same column of row B-1
        const int rows = int(prm.B - w * 16 < 16 ? prm.B - w * 16 : 16);
        const int last_t = rows * K - K, last_f = (rows - 1) * D * nf;
        for (int i = lane; i < tile_t; i += 32) cp_async8(tile + i, gt + (i < rows * K ? i : last_t + i % K));
        for (int i = lane; i < tile_f; i += 32)
          cp_async8(tile + tile_t + i, gf + (i < rows * D * nf ? i : last_f + i % (D * nf)));
        cp_async_mbar_arrive(full);
        __syncwarp();  // every lane's pending count is raised before the phase can complete
        if (lane == 0) mbar_arrive(full);
      }
    };
    const double* __restrict__ tT = tile + (lane >> 1) * K;
    const double* __restrict__ tF = tile + tile_t + (lane >> 1) * D * nf;
    auto in_x = [&](int v, int d) -> double { return tF[d * nf + fr.pidx(v)]; };  // position of own vertex v
    auto in_u0 = [&](int b, int d) -> double { return tF[d * nf + e0 + b]; };     // fixed end derivative b+1, raw

    long long wt = blockIdx.x;
    if (wt < n_wtiles) fill(wt);
    for (long long j = 0; wt < n_wtiles; wt += wt_stride, ++j) {
      const Row P = row_of(wt);
      mbar_wait_parity(full, uint32_t(j & 1));

      int stat = 0;
      double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], xm[D], xc[D];
      {
#pragma unroll
        for (int d = 0; d < D; ++d) {
          xm[d] = in_x(0, d);
          xc[d] = in_x(1, d);
        }
        const double T0 = tT[fr.seg(0)];
        if (bad_segment_time(T0)) stat |= kStatusBadTime;
        const double iT0 = fast_rcp(T0);
        double pw[N - 1];
        segment_powers<N, R>(T0, iT0, pw);
        S::end_blocks(pw, Cee, cps, cpe);
        S::carry_fold(pw, [&](int b, int d) { return fr.sgn(b) * in_u0(b, d); }, Wp, yp);
      }

      for (int v = 1; v <= n; ++v) {
        double sv[kSlots];
        double T;
        if (v <= nh) {
          double xn[D];
#pragma unroll
          for (int d = 0; d < D; ++d) xn[d] = in_x(v + 1, d);
          T = tT[fr.seg(v)];
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
        if (v <= npark) {  // warp-uniform
#pragma unroll
          for (int i = 0; i < kSlots; ++i) *PK(j, v - 1, i) = sv[i];
          *PK(j, v - 1, kSlots) = T;
        } else {
          const int b = slot_of(v, j);
          if (j > 0) mbar_wait_parity(bar0 + 8u * uint32_t(b), uint32_t((j - 1) & 1));  // freed by the last tile
          if (v <= nh) *HT(b) = T;
#pragma unroll
          for (int i = 0; i < kSlots; ++i) *SP(b, i) = sv[i];
        }
      }
      // the last tile's final segment has read END (step n waited for the slot released after it): the final
      // segment's inputs of this tile go there, then the buffer takes the next tile, which lands during the middle
      // vertex
#pragma unroll
      for (int d = 0; d < D; ++d) {
        *END(d) = in_x(0, d);
#pragma unroll
        for (int b = 0; b < m; ++b) *END(D + b * D + d) = in_u0(b, d);
      }
      *END(Lay::kEnd - 1) = tT[fr.seg(0)];
      if (wt + wt_stride < n_wtiles) fill(wt + wt_stride);

      double um[m][D];
      S::middle(Cee, cps, cpe, Wp, yp, xm, xc, um, stat);
      if (P.valid && half == 0 && prm.status != nullptr) prm.status[P.traj] = stat;
      if (half == 0 && prm.dfree != nullptr && P.valid) {
        double* __restrict__ df = prm.dfree + P.traj * (long long)D * np;
        const int vo = fr.vert(nh + 1);
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int q = 0; q < m; ++q) df[d * np + (vo - 1) * m + q] = fr.sgn(q) * um[q][d];
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        *HAND(d) = xc[d];
#pragma unroll
        for (int q = 0; q < m; ++q) *HAND((1 + q) * D + d) = um[q][d];
      }
      mbar_arrive(ready);
    }
    return;
  }

  // ================================================================== warp 1: outward sweep, final segment
  const TmaEmitter<N, D, AI> out1{&tmap, stage, stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h), lane, K, M - 1,
                                  K - M - 1, cl.evict_first != 0};
  TmaPairEmitter<N, D, AI> out2{&tmap, &tmap2, stage, lane, K, nh, cl.evict_first != 0};
  auto emit = [&](int v, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D], long long traj0) {
    if constexpr (Lay::kStorePairs) out2.emit(v, T, iT, sd, ed, traj0);
    else out1.emit(v, v, T, iT, sd, ed, traj0);
  };

  long long j = 0;
  for (long long wt = blockIdx.x; wt < n_wtiles; wt += wt_stride, ++j) {
    const Row P = row_of(wt);
    const long long traj0 = wt * 16;
    const bool valid = P.valid;

    double* __restrict__ df = prm.dfree != nullptr ? prm.dfree + P.traj * (long long)D * np : nullptr;
    auto store_free = [&](int v_own, const double (&u)[h][D]) {
      if (df != nullptr && valid) {
        const int vo = fr.vert(v_own);
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int q = 0; q < m; ++q) df[d * np + (vo - 1) * m + q] = fr.sgn(q) * u[1 + q][d];
      }
    };

    mbar_wait_parity(ready, uint32_t(j & 1));
    double ed[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d)
#pragma unroll
      for (int k = 0; k < h; ++k) ed[k][d] = *HAND(k * D + d);

    for (int v = n; v >= 1; --v) {
      const int b = slot_of(v, j);
      if (v <= npark) cp_async_wait_at_most(C - 1);
      const bool act = v <= nh;
      const double T = act ? *HT(b) : 1.0;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);
      double sv[kSlots];
#pragma unroll
      for (int i = 0; i < kSlots; ++i) sv[i] = *SP(b, i);
      if (v - C >= 1) {  // warp-uniform: the slot takes parked block v-C
#pragma unroll
        for (int i = 0; i < kSlots; ++i) cp_async8(SP(b, i), PK(j, v - C - 1, i));
        cp_async8(HT(b), PK(j, v - C - 1, kSlots));
      } else if (v > 1) {
        mbar_arrive(bar0 + 8u * uint32_t(b));  // the slot is the next tile's (vertex 1's: after the final segment)
      }
      cp_async_commit();
      double tE[m][D];
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
      emit(v, T, iT, sd, ed, traj0);
      if (act) {
#pragma unroll
        for (int d = 0; d < D; ++d)
#pragma unroll
          for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
      }
    }
    {  // own segment 0: the fixed end vertex
      double sd[h][D];
#pragma unroll
      for (int d = 0; d < D; ++d) {
        sd[0][d] = *END(d);
#pragma unroll
        for (int b = 0; b < m; ++b) sd[1 + b][d] = fr.sgn(b) * *END(D + b * D + d);
      }
      const double T = *END(Lay::kEnd - 1);
      mbar_arrive(bar0 + 8u * uint32_t(slot_of(1, j)));  // vertex 1's slot and END are the next tile's
      const double iT = fast_rcp(T);
      __syncwarp();
      emit(0, T, iT, sd, ed, traj0);
    }
  }
  if (lane < (Lay::kStorePairs ? 2 : 1)) bulk_wait_all();  // lane `half` stores each half's pairs
}

}  // namespace mtg
