// mtg_capi.cu -- the C-ABI (include/mtg_b200.h): handle, host-side constraint layout,
// kernel routing and the pipelined host-buffer entry points.  No CPU compute path exists
// here: every mtg_*_batch_* call launches sm_90a kernels or returns an error.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/mtg_b200.h"
#include "mtg_extrema_kernel.cuh"
#include "mtg_feasibility_kernel.cuh"
#include "mtg_flat_state_kernel.cuh"
#include "mtg_generic_kernel.cuh"
#include "mtg_half_plane_kernel.cuh"
#include "mtg_mellinger_loop_kernel.cuh"
#include "mtg_time_search_kernel.cuh"
#include "mtg_twisted_kernel.cuh"
#include "mtg_twisted_tmem_kernel.cuh"
#include "mtg_twisted_tmem_v4_kernel.cuh"
#include "mtg_twisted_chunked_kernel.cuh"
#include "mtg_twisted_tmem_v5_kernel.cuh"
#include "mtg_masked_block_kernel.cuh"
#include "mtg_waypoint_kernel.cuh"

namespace {

thread_local std::string g_create_error;

struct Layout {
  int n_all = 0, n_fixed = 0, n_free = 0, bw = 0;
  bool waypoint = false;
  std::vector<int32_t> slot_col;
  std::vector<int32_t> vcol;  // [(K+1)*h] column of (vertex, derivative)
};

struct CachedTopology {
  std::vector<uint8_t> mask;  // canonical mask
  int N = 0, K = 0;
  Layout layout;
  int32_t* d_slot_col = nullptr;
  int32_t* d_vcol = nullptr;
};

}  // namespace

struct mtg_handle {
  int device = 0;
  int sm_count = 0;
  int cc_major = 0;
  size_t smem_optin = 0;
  std::string error;
  int64_t launches = 0;
  int waypoint_variant = 0;  // MTG_OPT_WAYPOINT_VARIANT
  int early_steps = 0;       // MTG_OPT_EARLY_REFILL (v5, single tile buffer): 0 = on (kV5Early steps of lead), -1 = off
  int ctas_per_sm = 0;       // MTG_OPT_CTAS_PER_SM (v4 kernel: 0 = as many as fit, 9 = one CTA per tile, not persistent;
                             // chunked kernel: cap on resident warps per SM)
  int tma_inputs = 2;       // MTG_OPT_TMA_INPUTS (default routing prefers the TMA-input kernel v5 when eligible)
  int mellinger_unfused = 0; // MTG_OPT_MELLINGER_UNFUSED (1 = expand + solve + cost kernels, the round-1 path)
  int generic_variant = 0;   // MTG_OPT_GENERIC_VARIANT (0 = masked block kernel, 1 = banded kernel in global scratch)
  int chunk_blocks = 0;      // MTG_OPT_CHUNK_BLOCKS (chunked kernel: resident vertex blocks per lane, 0 = auto)
  int chunk_warps = 0;       // MTG_OPT_CHUNK_WARPS (chunked kernel: warps per CTA, 1 or 4; 0 = auto)
  int l2_hints = 0;          // MTG_OPT_L2_HINTS (chunked kernel: 0 = no cache hints, 1 = streamed data evict-first in L2)
  int dynamic_tiles = 0;     // MTG_OPT_DYNAMIC_TILES (v4 kernel: warps draw tiles from a global counter)
  std::vector<CachedTopology> topologies;
  // host-pointer pipeline
  static constexpr int kPipe = 3;
  // Scratch arenas are PER PIPELINE SLOT (index kPipe = launches on a caller-supplied stream): two chunks
  // of the host pipeline run concurrently on different streams and must never share band / pack scratch.
  // On the caller-stream slot consecutive users on DIFFERENT streams are ordered with an event.
  struct Arena {
    double* p = nullptr;
    size_t bytes = 0;
    cudaEvent_t ev = nullptr;       // recorded after the last kernel that used the arena
    cudaStream_t last = nullptr;
    bool used = false;
  };
  Arena scratch[kPipe + 1];  // generic kernel: banded factor + right-hand sides
  Arena pack[kPipe + 1];     // times + d_fixed produced by nfabian_pack_kernel; Mellinger expansion
  Arena counters[kPipe + 1]; // dynamic tile counter of the persistent kernels (event-ordered like the scratch arenas: two
                             // launches of one slot on different caller streams must not share a live counter)
  Arena optim[kPipe + 1];    // Mellinger outer loop and compass search: compact row lists and per-row state across
                             // their iterations; the compass search's candidate chunk too (up to kTimeSearchBudget)
  int* pinned_count = nullptr;        // the outer loop's active-row count, read back once per iteration
  cudaEvent_t count_ev = nullptr;
  // What is known about each kernel function launched so far, queried or set once per function so that a repeated
  // B = 1 solveLinear() call makes no attribute call.  The dynamic shared memory limit is a property of the function
  // (shared by every K routed to it): only ever raised.
  struct FnInfo {
    const void* fn;
    int regs;             // cudaFuncGetAttributes().numRegs
    size_t max_dyn_smem;  // cudaFuncAttributeMaxDynamicSharedMemorySize, at most its real value (0: not yet known)
    int carveout;         // cudaFuncAttributePreferredSharedMemoryCarveout as last set (-1: never)
  };
  std::vector<FnInfo> fns;
  // cached residency of the chunked kernel per (function, dynamic shared memory, CTA cap)
  struct ChunkedPlan {
    const void* fn = nullptr;
    size_t smem = 0;
    int cap = 0;
    int ctas = 0;
    int carveout = 0;  // cudaFuncAttributePreferredSharedMemoryCarveout for these CTAs
  };
  std::vector<ChunkedPlan> chunked_plans;
  // last encoded coefficient tensor map of each cache slot (B = 1 solveLinear() calls re-use the same output buffer):
  // slot 0 holds boxes of one segment or less, slot 1 the paired chunked kernel's boxes of two segments
  struct TmapKey {
    const void* base = nullptr;
    int64_t B = 0;
    int K = 0, D = 0, N = 0, box = 0;
  } tmap_key[2];
  CUtensorMap tmap_cached[2];
  cudaStream_t streams[kPipe] = {nullptr, nullptr, nullptr};
  void* dev_buf[kPipe] = {nullptr, nullptr, nullptr};
  size_t dev_buf_bytes[kPipe] = {0, 0, 0};
};

namespace {

bool set_err(mtg_handle* h, const char* what, cudaError_t e) {
  if (e == cudaSuccess) return false;
  if (h) h->error = std::string(what) + ": " + cudaGetErrorString(e);
  return true;
}

#define MTG_CUDA(h, call)                         \
  do {                                            \
    cudaError_t e__ = (call);                     \
    if (set_err(h, #call, e__)) return MTG_ERR_CUDA; \
  } while (0)

// return the status of `expr` unless it is MTG_OK
#define MTG_TRY(expr)                  \
  do {                                 \
    const int rc__ = (expr);           \
    if (rc__ != MTG_OK) return rc__;   \
  } while (0)

bool valid_problem(const mtg_problem* p) {
  if (!p) return false;
  if (p->N < 2 || p->N > MTG_MAX_N || (p->N & 1)) return false;
  if (p->r < 0 || p->r > p->N / 2 - 1) return false;  // CHECK at linear_impl.h:60
  if (p->K < 1 || p->D < 1) return false;
  return true;
}

std::vector<uint8_t> canonical_mask(const mtg_problem* p) {
  const int h = p->N / 2;
  std::vector<uint8_t> m(size_t(p->K + 1) * h, 0);
  if (p->fixed_mask) {
    for (size_t i = 0; i < m.size(); ++i) m[i] = p->fixed_mask[i] ? 1 : 0;
  } else {
    for (int v = 0; v <= p->K; ++v) {
      m[size_t(v) * h] = 1;
      if (v == 0 || v == p->K)
        for (int k = 1; k < h; ++k) m[size_t(v) * h + k] = 1;
    }
  }
  return m;
}

// The constraint reordering of linear_impl.h:181-260 in O(n): columns are the ranks of
// (vertex, derivative) inside the sorted fixed / free sets (linear.h:287-295); row i*N+s is
// slot s of segment i (s < h: vertex i, s >= h: vertex i+1; interior vertices appear twice,
// :202-205).
void compute_layout(int N, int K, const std::vector<uint8_t>& mask, Layout* L) {
  const int h = N / 2;
  std::vector<int32_t> col(size_t(K + 1) * h);
  int nf = 0, np = 0;
  for (size_t i = 0; i < mask.size(); ++i) (mask[i] ? nf : np)++;
  int cf = 0, cp = 0;
  for (size_t i = 0; i < mask.size(); ++i) col[i] = mask[i] ? cf++ : nf + cp++;
  L->vcol = col;
  L->n_all = K * N;
  L->n_fixed = nf;
  L->n_free = np;
  L->slot_col.resize(size_t(K) * N);
  L->bw = 0;
  for (int i = 0; i < K; ++i) {
    int lo = 1 << 30, hi = -1;
    for (int s = 0; s < N; ++s) {
      const int v = s < h ? i : i + 1, k = s < h ? s : s - h;
      const int c = col[size_t(v) * h + k];
      L->slot_col[size_t(i) * N + s] = c;
      if (c >= nf) { lo = std::min(lo, c); hi = std::max(hi, c); }
    }
    if (hi >= lo) L->bw = std::max(L->bw, hi - lo);
  }
  bool wp = K >= 2;
  for (int v = 0; v <= K && wp; ++v)
    for (int k = 0; k < h; ++k) {
      const bool want = (k == 0) || v == 0 || v == K;
      if ((mask[size_t(v) * h + k] != 0) != want) { wp = false; break; }
    }
  L->waypoint = wp && h >= 2;
}

// ---- waypoint kernel table: one row per compiled (N, r, D) -----------------------------------
// depth of the cp.async input ring of the v4 and chunked instantiations (their layouts depend on it)
constexpr int kRingDepth = 3;
// lead (outward-sweep steps) of v5's single-buffer tile refill
constexpr int kV5Early = 2;
// v4 is the default for short trajectories (K <= 8), where the per-tile prologue of v3 is a large share of a tile
constexpr int kV4MaxK = 8;
// warps per CTA of the chunked kernel's instantiations (WaypointEntry::k3)
constexpr int kChunkedWarps[2] = {1, 4};
// the paired form has mbarriers for the largest C that plan_chunked() picks
static_assert(mtg::ChunkedPairLayout<10, 3, kRingDepth>::kMaxChunk >= 24, "paired K3: C up to 24");
typedef void (*SweepKernel)(const mtg::WaypointParams);                    // v1, v2
typedef void (*TmemKernel)(const mtg::WaypointParams, const CUtensorMap);  // v3, cost-only
typedef void (*V4Kernel)(const mtg::WaypointParams, const mtg::TmemLaunchV4, const CUtensorMap);
typedef void (*V5Kernel)(const mtg::WaypointParams, const mtg::TmemLaunchV5, const CUtensorMap);
typedef void (*ChunkedKernel)(const mtg::WaypointParams, const mtg::ChunkedLaunch, const CUtensorMap);
typedef void (*ChunkedPairKernel)(const mtg::WaypointParams, const mtg::ChunkedLaunch, const CUtensorMap,
                                  const CUtensorMap);
struct WaypointEntry {
  int N, R, D;
  SweepKernel v2;                 // two lanes per trajectory (twisted factorisation), state in shared memory
  size_t (*v2_smem)(int K);
  TmemKernel v3, v3_fused;        // + 128-thread CTAs, TMA tensor stores; fused Nfabian
  size_t (*v3_smem)(int K);
  ChunkedKernel k3[2];            // K3: any K, kChunkedWarps[i] warps per CTA
  size_t (*k3_smem[2])(int C);    // with C resident blocks per lane
  int k3_park;                    // doubles per thread of one vertex block that K3 parks in global memory
  ChunkedPairKernel k3_pair;      // K3 in warp pairs (one tile's inward sweep beside the last tile's outward one)
  size_t (*k3_pair_smem)(int C, int K, int nf);  // with C resident blocks per lane and its tile input buffer
  // null where the shape has no such instantiation
  SweepKernel v1;                 // one thread per trajectory (cross-checks and profiles)
  size_t (*v1_smem)(int K);
  V4Kernel v4, v4_fused;          // persistent, deep input prefetch
  size_t (*v4_smem)(int K);
  V5Kernel v5, v5_fused;          // v4 with the inputs moved by TMA bulk copies
  V5Kernel v5_early, v5_fused_early;  // the EARLY = kV5Early instantiations
  size_t (*v5_smem)(int K, int nf, int nbuf), (*v5_fused_smem)(int K, int nf, int nbuf);
  bool (*early_fits)(int K);      // the EARLY instantiations may run for this K
  TmemKernel cost;                // computeCost of the solution without writing coefficients (v3 layout)
  TmemKernel cost_ls;             // the same with the line-search time generator (Mellinger outer loop)
};
enum : int { kV1 = 1, kCost = 2 };
// The row of (N, R, D).  FLAGS adds v1 and the cost-only kernel; MINB > 0 adds v4 and v5 with MINB blocks per SM in
// their launch bounds.
template <int N, int R, int D, int FLAGS = 0, int MINB = 0>
WaypointEntry waypoint_row() {
  WaypointEntry e{};
  e.N = N;
  e.R = R;
  e.D = D;
  e.v2 = mtg::twisted_solve_kernel<N, R, D>;
  e.v2_smem = mtg::V2Layout<N, D>::bytes;
  e.v3 = mtg::twisted_tmem_kernel<N, R, D>;
  e.v3_fused = mtg::twisted_tmem_kernel<N, R, D, true>;
  e.v3_smem = mtg::V3Layout<N, D>::bytes;
  e.k3[0] = mtg::twisted_chunked_kernel<N, R, D, kRingDepth, 1>;
  e.k3[1] = mtg::twisted_chunked_kernel<N, R, D, kRingDepth, 4>;
  e.k3_smem[0] = mtg::ChunkedLayout<N, D, kRingDepth, 1>::bytes;
  e.k3_smem[1] = mtg::ChunkedLayout<N, D, kRingDepth, 4>::bytes;
  e.k3_park = mtg::ChunkedLayout<N, D, kRingDepth, 4>::kPark;
  e.k3_pair = mtg::twisted_chunked_pair_kernel<N, R, D, kRingDepth>;
  e.k3_pair_smem = mtg::ChunkedPairLayout<N, D, kRingDepth>::bytes;
  if constexpr ((FLAGS & kV1) != 0) {
    e.v1 = mtg::waypoint_solve_kernel<N, R, D>;
    e.v1_smem = mtg::V1Layout<N, D>::bytes;
  }
  if constexpr (MINB > 0) {
    e.v4 = mtg::twisted_tmem_v4_kernel<N, R, D, false, kRingDepth, MINB>;
    e.v4_fused = mtg::twisted_tmem_v4_kernel<N, R, D, true, kRingDepth, MINB>;
    e.v4_smem = mtg::V4Layout<N, D, kRingDepth>::bytes;
    e.v5 = mtg::twisted_tmem_v5_kernel<N, R, D, MINB, false>;
    e.v5_fused = mtg::twisted_tmem_v5_kernel<N, R, D, MINB, true>;
    e.v5_early = mtg::twisted_tmem_v5_kernel<N, R, D, MINB, false, kV5Early>;
    e.v5_fused_early = mtg::twisted_tmem_v5_kernel<N, R, D, MINB, true, kV5Early>;
    e.v5_smem = mtg::V5Layout<N, D, false>::bytes;
    e.v5_fused_smem = mtg::V5Layout<N, D, true>::bytes;
    e.early_fits = mtg::V5Layout<N, D, false>::template early_fits<kV5Early>;
  }
  if constexpr ((FLAGS & kCost) != 0) {
    e.cost = mtg::twisted_tmem_kernel<N, R, D, false, true>;
    e.cost_ls = mtg::twisted_tmem_line_search_kernel<N, R, D>;
  }
  return e;
}
const WaypointEntry kWaypoints[] = {
    // min snap, N = 10
    waypoint_row<10, 4, 3, kV1 | kCost, 2>(), waypoint_row<10, 4, 1, kV1 | kCost, 2>(), waypoint_row<10, 4, 2>(),
    waypoint_row<10, 4, 4, kCost>(),
    // jerk / acceleration on N = 10
    waypoint_row<10, 3, 3, kV1 | kCost, 2>(), waypoint_row<10, 3, 1>(), waypoint_row<10, 2, 3, kV1 | kCost, 2>(),
    waypoint_row<10, 2, 1>(),
    // min jerk, N = 8
    waypoint_row<8, 3, 3, kV1 | kCost, 3>(), waypoint_row<8, 3, 1, kV1>(), waypoint_row<8, 3, 2>(),
    waypoint_row<8, 3, 4>(),
    // N = 12 (feasibility tests)
    waypoint_row<12, 5, 3, kV1 | kCost, 2>(), waypoint_row<12, 5, 1>(), waypoint_row<12, 5, 4>(),
    // min acceleration, N = 6
    waypoint_row<6, 2, 3>(), waypoint_row<6, 2, 1>(),
};

const WaypointEntry* find_waypoint(const mtg_problem* p, const Layout& L) {
  if (!L.waypoint) return nullptr;
  for (const auto& e : kWaypoints)
    if (e.N == p->N && e.R == p->r && e.D == p->D) return &e;  // any K: the chunked kernel has a fixed footprint
  return nullptr;
}

int route(const mtg_problem* p, const Layout& L) {
  if (L.n_free == 0) return MTG_KERNEL_NOFREE;
  if (find_waypoint(p, L)) return MTG_KERNEL_WAYPOINT;
  return MTG_KERNEL_GENERIC;
}

CachedTopology* get_topology(mtg_handle* h, const mtg_problem* p) {
  std::vector<uint8_t> mask = canonical_mask(p);
  for (auto& t : h->topologies)
    if (t.N == p->N && t.K == p->K && t.mask == mask) return &t;
  CachedTopology t;
  t.N = p->N;
  t.K = p->K;
  t.mask = mask;
  compute_layout(p->N, p->K, mask, &t.layout);
  if (set_err(h, "cudaMalloc(slot_col)", cudaMalloc(&t.d_slot_col, sizeof(int32_t) * t.layout.slot_col.size())))
    return nullptr;
  if (set_err(h, "cudaMemcpy(slot_col)",
              cudaMemcpy(t.d_slot_col, t.layout.slot_col.data(), sizeof(int32_t) * t.layout.slot_col.size(),
                         cudaMemcpyHostToDevice)))
    return nullptr;
  if (set_err(h, "cudaMalloc(vcol)", cudaMalloc(&t.d_vcol, sizeof(int32_t) * t.layout.vcol.size()))) return nullptr;
  if (set_err(h, "cudaMemcpy(vcol)", cudaMemcpy(t.d_vcol, t.layout.vcol.data(), sizeof(int32_t) * t.layout.vcol.size(),
                                                cudaMemcpyHostToDevice)))
    return nullptr;
  if (h->topologies.size() >= 64) {  // bound the cache
    cudaFree(h->topologies.front().d_vcol);
    cudaFree(h->topologies.front().d_slot_col);
    h->topologies.erase(h->topologies.begin());
  }
  h->topologies.push_back(std::move(t));
  return &h->topologies.back();
}

// Grow-only arena.  acquire(): make the arena usable by a kernel about to be launched on `stream` (orders it
// after the previous user when that one ran on another stream); release(): note the new last user.
int arena_acquire(mtg_handle* h, mtg_handle::Arena& a, size_t bytes, cudaStream_t stream) {
  if (bytes > a.bytes) {
    if (a.p) {
      MTG_CUDA(h, cudaDeviceSynchronize());
      cudaFree(a.p);
      a.p = nullptr;
      a.bytes = 0;
    }
    MTG_CUDA(h, cudaMalloc(&a.p, bytes));
    a.bytes = bytes;
    a.used = false;
  }
  if (a.used && a.last != stream) MTG_CUDA(h, cudaStreamWaitEvent(stream, a.ev, 0));
  return MTG_OK;
}
int arena_release(mtg_handle* h, mtg_handle::Arena& a, cudaStream_t stream) {
  if (!a.ev) MTG_CUDA(h, cudaEventCreateWithFlags(&a.ev, cudaEventDisableTiming));
  MTG_CUDA(h, cudaEventRecord(a.ev, stream));
  a.last = stream;
  a.used = true;
  return MTG_OK;
}

// zeroed dynamic-tile counter of pipeline slot `slot`, ordered after the previous launch that used it
int tile_counter_acquire(mtg_handle* h, int slot, cudaStream_t stream, unsigned long long** out) {
  mtg_handle::Arena& a = h->counters[slot];
  MTG_TRY(arena_acquire(h, a, 256, stream));
  *out = reinterpret_cast<unsigned long long*>(a.p);
  MTG_CUDA(h, cudaMemsetAsync(*out, 0, sizeof(unsigned long long), stream));
  return MTG_OK;
}

// The cached facts of `fn`: its registers are queried on first use.  Null (and h->error set) when the query fails.
mtg_handle::FnInfo* fn_info(mtg_handle* h, const void* fn) {
  for (auto& f : h->fns)
    if (f.fn == fn) return &f;
  cudaFuncAttributes attr;
  if (set_err(h, "cudaFuncGetAttributes", cudaFuncGetAttributes(&attr, fn))) return nullptr;
  h->fns.push_back({fn, attr.numRegs, 0, -1});
  return &h->fns.back();
}

// Make sure `fn` may be launched with `bytes` of dynamic shared memory (raises the function attribute when needed).
// The attribute belongs to the function in the device's context, so every handle of the process shares it, while
// each handle caches what it knows.  It is therefore only ever raised: under one process-wide lock, to `bytes` when
// its current value is smaller.  A handle's cached value then stays at or below the real one, even after another
// handle has needed less (setting the smaller value would make this handle's next larger launch fail).
int ensure_dyn_smem(mtg_handle* h, const void* fn, size_t bytes) {
  mtg_handle::FnInfo* f = fn_info(h, fn);
  if (!f) return MTG_ERR_CUDA;
  if (bytes <= f->max_dyn_smem) return MTG_OK;
  static std::mutex attr_lock;
  std::lock_guard<std::mutex> lock(attr_lock);
  cudaFuncAttributes attr;
  MTG_CUDA(h, cudaFuncGetAttributes(&attr, fn));
  const size_t current = size_t(std::max(attr.maxDynamicSharedSizeBytes, 0));
  if (current < bytes)
    MTG_CUDA(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  f->max_dyn_smem = std::max(current, bytes);
  return MTG_OK;
}

// Set the shared memory carveout of `fn` (percent of the SM's maximum), unless it already has that value.
int set_carveout(mtg_handle* h, const void* fn, int percent) {
  mtg_handle::FnInfo* f = fn_info(h, fn);
  if (!f) return MTG_ERR_CUDA;
  if (f->carveout == percent) return MTG_OK;
  MTG_CUDA(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, percent));
  f->carveout = percent;
  return MTG_OK;
}

// ---- launches: every kernel of the library goes through launch_kernel() -------------------------------------------
// Blocks of `per_block` items for `work` items, at most `per_sm` resident or grid-strided blocks per SM.
int64_t capped_grid(const mtg_handle* h, int64_t work, int64_t per_block, int per_sm) {
  return std::min<int64_t>((work + per_block - 1) / per_block, int64_t(per_sm) * h->sm_count);
}

// fn<<<grid, block, smem, s>>>(args...), its launch error checked and the launch counted (mtg_launch_count).  A launch
// with dynamic shared memory first raises fn's limit to `smem` (ensure_dyn_smem); one without makes no attribute call.
template <class... P, class... A>
int launch_kernel(mtg_handle* h, void (*fn)(P...), int64_t grid, int block, size_t smem, cudaStream_t s, A&&... args) {
  if (smem > 0) MTG_TRY(ensure_dyn_smem(h, (const void*)fn, smem));
  fn<<<(unsigned)grid, block, smem, s>>>(std::forward<A>(args)...);
  MTG_CUDA(h, cudaGetLastError());
  h->launches++;
  return MTG_OK;
}

// The segment-parallel kernels (extrema, time scaling, input feasibility, half planes): kExtremaThreads threads per
// block in rows of K threads, one trajectory per row, with `row_smem` bytes of dynamic shared memory per row.  When
// the rows of a block need more shared memory than a block may have, `entry` fails with "<entry>: <what> too large".
template <class Params>
int launch_segment_parallel(mtg_handle* h, void (*fn)(Params, int), const Params& prm, int K, int64_t B,
                            size_t row_smem, const char* entry, const char* what, cudaStream_t s) {
  const int tpb = std::max(1, mtg::kExtremaThreads / K);
  const size_t smem = size_t(tpb) * row_smem;
  if (smem > h->smem_optin) {
    h->error = std::string(entry) + ": " + what + " too large";
    return MTG_ERR_BAD_ARG;
  }
  return launch_kernel(h, fn, capped_grid(h, B, tpb, 16), mtg::kExtremaThreads, smem, s, prm, tpb);
}

// ---- kernel tables: one instantiation per order N -----------------------------------------------------------------
// The (N, A) of one instantiation; A is the second template parameter where a kernel has one (the flat-state
// attitude case, the masked kernel's dimension group).
template <int N_, int A_>
struct Inst {
  static constexpr int N = N_, A = A_;
};
template <int N0, int STEP, int A0, int NA, class Pick, size_t... I>
auto kernel_table(Pick pick, std::index_sequence<I...>) {
  return std::array{pick(Inst<N0 + STEP * int(I / NA), A0 + int(I % NA)>{})...};
}
// The kernel `pick(Inst<n, a>{})` from a table, built on first use, of one instantiation per N in {N0, N0 + STEP, ...,
// N1} and A in [A0, A1].  Takes arguments in those ranges.
template <int N0, int N1, int STEP = 1, int A0 = 0, int A1 = 0, class Pick>
auto kernel_by_n(Pick pick, int n, int a = A0) {
  constexpr int NA = A1 - A0 + 1;
  static const auto table =
      kernel_table<N0, STEP, A0, NA>(pick, std::make_index_sequence<((N1 - N0) / STEP + 1) * NA>{});
  return table[size_t((n - N0) / STEP * NA + (a - A0))];
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// coeffs as a 2-D fp64 tensor [B][K*D*N] for the TMA stores (box = 16 trajectories x `box` doubles: at most one
// segment, or two for the paired chunked kernel).  The last encoded map of each size class is kept: repeated calls
// on the same output buffer encode it once.
int coeff_tmap(mtg_handle* h, double* coeffs, int64_t B, const mtg_problem* p, int box, const CUtensorMap** out) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                               const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  // function-local static with a lambda initialiser: initialised exactly once, thread-safe (C++11)
  static const EncodeFn encode = []() -> EncodeFn {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeFn>(fp);
  }();
  const int slot = box > p->D * p->N ? 1 : 0;
  mtg_handle::TmapKey& key = h->tmap_key[slot];
  CUtensorMap* map = &h->tmap_cached[slot];
  *out = map;
  if (key.base == coeffs && key.B == B && key.K == p->K && key.D == p->D && key.N == p->N && key.box == box)
    return MTG_OK;
  key.base = nullptr;
  if (!encode) {
    h->error = "cuTensorMapEncodeTiled is not available from the driver";
    return MTG_ERR_CUDA;
  }
  const cuuint64_t row = cuuint64_t(p->K) * p->D * p->N;
  const cuuint64_t dims[2] = {row, cuuint64_t(B)};
  const cuuint64_t strides[1] = {row * sizeof(double)};
  const cuuint32_t boxdim[2] = {cuuint32_t(box), 16u};
  const cuuint32_t estr[2] = {1u, 1u};
  const CUresult cr = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, coeffs, dims, strides, boxdim, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    h->error = "cuTensorMapEncodeTiled failed (" + std::to_string(int(cr)) + ")";
    return MTG_ERR_CUDA;
  }
  key = {coeffs, B, p->K, p->D, p->N, box};
  return MTG_OK;
}

struct FusedInput {
  const double* positions;
  double v_max, a_max, magic;
  double* times_out;
};

// shared memory of an SM that resident CTAs share (H100: 228 KB; every CTA also reserves 1 KB of it)
constexpr int kSmemPerSm = 228 * 1024;

// Resident CTAs per SM of a `threads`-thread kernel with `smem` bytes of dynamic shared memory: limited by its
// registers, by shared memory and by `cap`; 0 when `smem` exceeds the per-block opt-in limit.
int resident_ctas(mtg_handle* h, const void* fn, size_t smem, int cap, int threads, int* ctas) {
  const mtg_handle::FnInfo* f = fn_info(h, fn);
  if (!f) return MTG_ERR_CUDA;
  const int by_regs = std::max(1, 65536 / (std::max(f->regs, 1) * threads));
  *ctas = smem > h->smem_optin ? 0 : std::min(std::min<int>(by_regs, int(kSmemPerSm / (smem + 1024))), cap);
  return MTG_OK;
}

// v3 and its cost-only form run while their factor leaves at least two CTAs of `fn` per SM (of at most 16); beyond,
// the chunked kernel (K3) takes the solve.
int v3_fits(mtg_handle* h, const void* fn, size_t smem, bool* fits) {
  int ctas = 0;
  MTG_TRY(resident_ctas(h, fn, smem, 16, mtg::kTmemThreads, &ctas));
  *fits = ctas >= 2;
  return MTG_OK;
}

// Resident CTAs per SM of the chunked kernel `fn` (`threads` per CTA, `smem` bytes of dynamic shared memory, at most
// `cap`) and the shared memory carveout those CTAs need (*carveout, percent): the rest of the SM's 256 KB stays L1,
// which serves the 8-byte cp.async input reads.  On the first use of a configuration the hand-computed residency is
// checked against the occupancy calculator at that carveout, so that the planned warps per SM are the ones that run.
int chunked_residency(mtg_handle* h, const void* fn, size_t smem, int cap, int threads, int* ctas, int* carveout) {
  for (const auto& pl : h->chunked_plans)
    if (pl.fn == fn && pl.smem == smem && pl.cap == cap) {
      *ctas = pl.ctas;
      *carveout = pl.carveout;
      return MTG_OK;
    }
  mtg_handle::ChunkedPlan np;
  np.fn = fn;
  np.smem = smem;
  np.cap = cap;
  MTG_TRY(resident_ctas(h, fn, smem, cap, threads, &np.ctas));
  if (np.ctas > 0) {
    MTG_TRY(ensure_dyn_smem(h, fn, smem));
    const size_t need = size_t(np.ctas) * (smem + 1024);
    np.carveout = int(std::min<size_t>(100, (need * 100 + kSmemPerSm - 1) / kSmemPerSm));
    MTG_TRY(set_carveout(h, fn, np.carveout));
    int occ = 0;
    MTG_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem));
    np.ctas = std::min(np.ctas, occ);
  }
  h->chunked_plans.push_back(np);
  *ctas = np.ctas;
  *carveout = np.carveout;
  return MTG_OK;
}

// ---- waypoint launches: plan_waypoint() decides, launch_waypoint() launches -------------------
enum class Family { Sweep, Tmem, V4, V5, Chunked, ChunkedPair };  // v1 and v2, v3, v4, v5, K3, paired K3: fixes the
                                                                 // argument list
struct WaypointPlan {
  Family family = Family::Sweep;
  const void* fn = nullptr;
  int64_t blocks = 0;
  int threads = 0;
  size_t smem = 0;            // dynamic shared memory
  int n_buffers = 0;          // v5: input tile buffers per warp
  bool tile_counter = false;  // v4, v5: warps draw their tiles from a zeroed global counter
  int chunk = 0;              // K3: vertex blocks resident per lane
  size_t park_bytes = 0;      // K3: parking area of the outer vertex blocks (0: nothing is parked)
  int carveout = -1;          // K3: shared memory carveout in percent (-1: left as it is)
  int evict_first = 0;        // K3: streamed data marked evict-first in L2
};

// K3: the chunked twisted kernel -- any K, fixed on-chip footprint; the vertex blocks beyond the C resident ones
// are parked in global memory.
// With `pairs` (the default route), the paired form takes the solve where it fits: see below.
int plan_chunked(mtg_handle* h, const mtg_problem* p, const WaypointEntry& e, int64_t B, int nf, bool pairs,
                 WaypointPlan* pl) {
  const int nmax = (p->K + 1) / 2 - 1;
  // Auto: one-warp CTAs (shared memory then comes in 31-52 KB steps instead of 124-206 KB ones), no L2 hints, at
  // most kAutoParkWarps warps per SM while any block is parked and as many as fit otherwise; among the chunks up to
  // the auto chunk, the one with the most warps, the largest on a tie.  The auto chunk is 5 while that parks at most
  // kAutoParkedMax blocks per lane (K <= 16 at N = 10), 4 beyond.  Each resident block takes 3.2 KB of shared
  // memory per warp away from L1 and saves one round trip of a parked block through L2: it pays while the parked
  // blocks are few.  Measured with tools/k3_sweep.py on an H100 SXM at N = 10, D = 3, 4 warps per SM (ms per solve,
  // 700 W power limit, spread of the round medians <= 0.02 ms):
  //   K = 16  (1 048 576): C = 3 2.93, C = 4 2.72, C = 5 2.60, C = 6 2.98
  //   K = 50  (246 272):   C = 3 3.15, C = 4 3.09, C = 5 3.10, C = 6 3.48
  //   K = 100 (113 664):   C = 3 3.11, C = 4 3.08, C = 5 3.14, C = 6 3.60
  // More warps pay only when nothing is parked (400 W: K = 8, C = 3 runs 1.28 ms at 6-7 warps against 1.51 ms at 4);
  // with parked blocks they lose (C = 3, K = 16: 2.93 ms at 4 warps, 3.52 at 7), with or without evict-first hints on
  // the streamed data, and the hints themselves cost 2-20 %.  Four-warp CTAs at the same warps run 1-3 % slower.
  constexpr int kAutoParkWarps = 4;
  constexpr int kAutoParkedMax = 2;
  const int auto_chunk = nmax - 5 <= kAutoParkedMax ? 5 : 4;
  const int cmax = std::max(1, std::min(nmax, h->chunk_blocks > 0 ? 24 : auto_chunk));
  int best_warps = 0, best_C = 0, best_i = 0, best_ctas = 0, best_carveout = 0;
  size_t best_smem = 0;
  for (int C = cmax; C >= 1; --C) {
    if (h->chunk_blocks > 0 && C != std::min(h->chunk_blocks, cmax)) continue;
    for (int i = 0; i < 2; ++i) {
      const int W = kChunkedWarps[i];
      if (h->chunk_warps > 0 ? W != h->chunk_warps : W != 1) continue;
      // cap on resident warps per SM
      const int wcap = h->ctas_per_sm > 0 ? h->ctas_per_sm : (nmax > C ? kAutoParkWarps : 64);
      const size_t smem = e.k3_smem[i](C);
      int ctas = 0, carveout = 0;
      MTG_TRY(chunked_residency(h, (const void*)e.k3[i], smem, std::max(1, wcap / W), 32 * W, &ctas, &carveout));
      if (ctas * W > best_warps) {
        best_warps = ctas * W;
        best_ctas = ctas;
        best_carveout = carveout;
        best_C = C;
        best_i = i;
        best_smem = smem;
      }
    }
  }
  if (best_warps == 0) {
    h->error = "chunked kernel: no launch configuration fits";
    return MTG_ERR_ALLOC;
  }
  pl->family = Family::Chunked;
  pl->evict_first = h->l2_hints;
  // The paired form (twisted_chunked_pair_kernel): 64-thread CTAs that run one tile's inward sweep beside the last
  // tile's outward sweep on one tile's resident blocks.  Auto: while every block of a lane fits in shared memory
  // (nmax <= kPairMaxBlocks, K <= 16), C = nmax -- nothing parked -- at kAutoPairs pairs per SM.  Measured with
  // tools/k3_sweep.py on an H100 80GB HBM3 at N = 10, D = 3, 700 W power limit, SM clock 1980 MHz (ms per solve,
  // spread of the round medians <= 0.02 ms but one 0.34), with the inputs in tile buffers filled by bulk copies, at
  // 2 / 3 / 4 pairs per SM where they fit:
  //   K = 8  (1 048 576): C = 3: 1.128 / 1.111 / 1.148
  //   K = 12 (1 048 576): C = 3: 1.808 / 1.975 / 2.134   C = 5: 1.593 / 1.662
  //   K = 16 (1 048 576): C = 3: 2.720 / 3.134 / 3.397   C = 5: 2.340 / 2.567   C = 7: 2.054 / 2.183
  // A third pair loses even though the inputs no longer pass through L1 (only at K = 8 is it 1.5 % ahead, within
  // twice the spread).  Before the tile buffers (per-lane cp.async gathers through L1), K = 16 ran C = 7 at 2.20 / 2.36
  // and, with blocks parked, K = 50 and K = 100 at 3.1-3.3 ms against 3.09 and 3.08 for the one-warp plan, which
  // keeps those K.  Forced,
  // CHUNK_BLOCKS sets C and CTAS_PER_SM caps the warps per SM (pairs = CTAS_PER_SM / 2) at any K.  The pairs need an
  // inward sweep (K >= 3); CHUNK_WARPS or L2_HINTS select the one-warp form.
  constexpr int kPairMaxBlocks = 7;
  constexpr int kAutoPairs = 2;
  static_assert(kPairMaxBlocks == 7 && kAutoPairs == 2 && kSmemPerSm == 228 * 1024,
                "ChunkedPairLayout::kStorePairs is sized for two pairs per SM at C = 7");
  const bool forced = h->chunk_blocks > 0 || h->ctas_per_sm > 0;
  if (pairs && h->chunk_warps == 0 && h->l2_hints == 0 && nmax >= 1 && (forced || nmax <= kPairMaxBlocks)) {
    const int C = h->chunk_blocks > 0 || nmax > kPairMaxBlocks ? best_C : nmax;
    const size_t smem = e.k3_pair_smem(C, p->K, nf);
    const int cap = h->ctas_per_sm > 0 ? h->ctas_per_sm / 2 : kAutoPairs;
    int ctas = 0, carveout = 0;
    if (cap >= 1) MTG_TRY(chunked_residency(h, (const void*)e.k3_pair, smem, cap, 64, &ctas, &carveout));
    if (ctas >= (forced ? 1 : kAutoPairs)) {
      pl->family = Family::ChunkedPair;
      pl->fn = (const void*)e.k3_pair;
      pl->threads = 64;
      pl->smem = smem;
      pl->blocks = capped_grid(h, B, 16, ctas);
      pl->chunk = C;
      if (nmax > C) pl->park_bytes = size_t(nmax - C) * e.k3_park * size_t(pl->blocks) * 64 * sizeof(double);
      pl->carveout = carveout;
      return MTG_OK;
    }
  }
  const int npark = nmax - best_C;  // parked vertex blocks per lane
  pl->chunk = best_C;
  const int W = kChunkedWarps[best_i];
  pl->fn = (const void*)e.k3[best_i];
  pl->threads = 32 * W;
  pl->smem = best_smem;
  pl->blocks = capped_grid(h, B, 16 * W, best_ctas);
  if (npark > 0) pl->park_bytes = size_t(npark) * e.k3_park * size_t(pl->blocks) * pl->threads * sizeof(double);
  pl->carveout = best_carveout;
  return MTG_OK;
}

// Waypoint routing.  a16 = 16-byte aligned, V = MTG_OPT_WAYPOINT_VARIANT.  Every kernel here stores coefficients in
// 16-byte units (TMA tensor stores / double2), so a plain call whose output is not a16 (e.g. a tensor slice) has
// already gone to the banded generic kernel, which stores scalar doubles.  The first rule that applies decides:
//  1. A fused call whose output is not a16: no fused kernel; the caller packs the inputs and solves.
//  2. V = 5, plain call: K3.
//  3. v5 when V = 6, or V = 0 and TMA_INPUTS != 0, with B % 16 == 0, a16 inputs and a v5 instantiation.  Of two and
//     one input tile buffers per warp, the one with more resident CTAs per SM wins (at most 8; two on a tie).  V = 6
//     takes it at >= 1 CTA; V = 0 at >= 2 CTAs (with fewer, K3 keeps more warps in flight) and with two buffers, or
//     with one when TMA_INPUTS = 2.  One buffer is refilled early (EARLY instantiation) unless EARLY_REFILL = -1,
//     where K leaves room for it and the EARLY kernel's registers keep as many CTAs resident.
//  4. v4 when V = 4, or V = 0 and K <= 8, with a v4 instantiation, at >= 2 resident CTAs per SM of at most 8 (V = 4:
//     >= 1), then at most CTAS_PER_SM; CTAS_PER_SM = 9 launches one CTA per tile instead of persistent CTAs.
//  5. For V in {0, 3, 4, 5, 6}, every fused call, V = 2 when v2's state does not fit in shared memory and V = 1 when
//     neither v1's nor v2's does: v3 while its factor leaves >= 2 CTAs per SM (counted with the plain kernel's
//     registers, fused calls too); beyond, K3 for a plain call (with V = 0 its paired form where plan_chunked
//     takes it) and no fused kernel for a fused one.
//  6. V = 1 where v1 is compiled and fits: v1.  Otherwise v2.
// v5 and v4 draw tiles from a global counter when DYNAMIC_TILES = 1, and in auto mode when every warp has many tiles
// (v5: >= 8 and K > 8; v4: >= 16), where the counter balances the tail; otherwise tiles go round-robin, since the
// counter's round trip to L2 is not small against a short tile or amortised over few.  CTAS_PER_SM also caps K3's
// resident warps (plan_chunked), and has no effect on v5.
int plan_waypoint(mtg_handle* h, const mtg_problem* p, const Layout& L, const WaypointEntry& e,
                  const mtg::WaypointParams& prm, bool fused, WaypointPlan* pl) {
  const auto a16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  const int V = h->waypoint_variant, K = p->K;
  const int64_t B = prm.B;
  if (!a16(prm.coeffs)) return MTG_ERR_ALLOC;
  if (V == 5 && !fused) return plan_chunked(h, p, e, B, prm.n_fixed, false, pl);
  const bool inputs_a16 = fused ? a16(prm.positions) : a16(prm.times) && a16(prm.dfix);
  if ((V == 6 || (V == 0 && h->tma_inputs != 0)) && B % 16 == 0 && inputs_a16 && e.v5) {
    const void* fn = (const void*)(fused ? e.v5_fused : e.v5);
    int ctas = 0, nbuf = 0;
    size_t smem = 0;
    for (int nb = 2; nb >= 1; --nb) {
      const size_t s = (fused ? e.v5_fused_smem : e.v5_smem)(K, L.n_fixed, nb);
      int c = 0;
      MTG_TRY(resident_ctas(h, fn, s, 8, mtg::kTmemThreads, &c));
      if (c > ctas) {
        ctas = c;
        nbuf = nb;
        smem = s;
      }
    }
    if (ctas >= (V == 6 ? 1 : 2) && (V == 6 || nbuf == 2 || h->tma_inputs == 2)) {
      pl->family = Family::V5;
      pl->fn = fn;
      pl->threads = mtg::kTmemThreads;
      pl->smem = smem;
      pl->n_buffers = nbuf;
      if (nbuf == 1 && h->early_steps >= 0 && e.early_fits(K)) {
        const void* fe = (const void*)(fused ? e.v5_fused_early : e.v5_early);
        const mtg_handle::FnInfo* f = fn_info(h, fe);
        if (!f) return MTG_ERR_CUDA;
        if (65536 / (std::max(f->regs, 1) * mtg::kTmemThreads) >= ctas) pl->fn = fe;
      }
      pl->blocks = capped_grid(h, B, 64, ctas);
      const int64_t tiles_per_warp = (B / 16) / std::max<int64_t>(1, pl->blocks * 4);
      pl->tile_counter = h->dynamic_tiles == 1 || (h->dynamic_tiles == 0 && tiles_per_warp >= 8 && K > kV4MaxK);
      return MTG_OK;
    }
  }
  if ((V == 4 || (V == 0 && K <= kV4MaxK)) && e.v4) {
    const void* fn = (const void*)(fused ? e.v4_fused : e.v4);
    const size_t smem = e.v4_smem(K);
    int ctas = 0;
    MTG_TRY(resident_ctas(h, fn, smem, 8, mtg::kTmemThreads, &ctas));
    if (ctas >= (V == 4 ? 1 : 2)) {
      const bool per_tile = h->ctas_per_sm == 9;
      if (h->ctas_per_sm > 0 && !per_tile) ctas = std::min(ctas, h->ctas_per_sm);
      const int64_t tiles = (B + 63) / 64;
      const int64_t tiles_per_warp = ((B + 15) / 16) / std::max<int64_t>(1, int64_t(ctas) * h->sm_count * 4);
      pl->family = Family::V4;
      pl->fn = fn;
      pl->threads = mtg::kTmemThreads;
      pl->smem = smem;
      pl->blocks = per_tile ? tiles : capped_grid(h, B, 64, ctas);
      pl->tile_counter = !per_tile && (h->dynamic_tiles == 1 || (h->dynamic_tiles == 0 && tiles_per_warp >= 16));
      return MTG_OK;
    }
  }
  const bool v1_fits = e.v1 && e.v1_smem(K) <= h->smem_optin;
  const bool v2_fits = e.v2_smem(K) <= h->smem_optin;
  if (fused || (V != 1 && V != 2) || (V == 2 && !v2_fits) || (V == 1 && !v1_fits && !v2_fits)) {
    const size_t smem = e.v3_smem(K);
    bool fits = false;
    MTG_TRY(v3_fits(h, (const void*)e.v3, smem, &fits));
    if (!fits) return fused ? MTG_ERR_ALLOC : plan_chunked(h, p, e, B, prm.n_fixed, V == 0, pl);
    pl->family = Family::Tmem;
    pl->fn = (const void*)(fused ? e.v3_fused : e.v3);
    pl->blocks = (B + 63) / 64;
    pl->threads = mtg::kTmemThreads;
    pl->smem = smem;
  } else if (V == 1 && v1_fits) {
    pl->fn = (const void*)e.v1;
    pl->blocks = (B + 31) / 32;
    pl->threads = 32;
    pl->smem = e.v1_smem(K);
  } else {
    pl->fn = (const void*)e.v2;
    pl->blocks = (B + 15) / 16;
    pl->threads = 32;
    pl->smem = e.v2_smem(K);
  }
  return MTG_OK;
}

// The one launch site of the waypoint kernels: tile counter or parking area, function attributes, tensor map,
// launch, and the release that orders the next user of the counter or parking area after this launch.
int launch_waypoint(mtg_handle* h, const mtg_problem* p, const WaypointPlan& pl, const mtg::WaypointParams& prm,
                    cudaStream_t stream, int slot) {
  mtg_handle::Arena* held = nullptr;
  unsigned long long* counter = nullptr;
  if (pl.tile_counter) {
    MTG_TRY(tile_counter_acquire(h, slot, stream, &counter));
    held = &h->counters[slot];
  }
  if (pl.park_bytes > 0) {
    held = &h->scratch[slot];
    MTG_TRY(arena_acquire(h, *held, pl.park_bytes, stream));
  }
  // raised before the carveout and the tensor map (launch_kernel() then finds it raised)
  MTG_TRY(ensure_dyn_smem(h, pl.fn, pl.smem));
  if (pl.carveout >= 0) MTG_TRY(set_carveout(h, pl.fn, pl.carveout));
  const CUtensorMap* tmap = nullptr;
  if (pl.family != Family::Sweep) MTG_TRY(coeff_tmap(h, prm.coeffs, prm.B, p, p->D * p->N, &tmap));
  const int64_t grid = pl.blocks;
  const int block = pl.threads;
  switch (pl.family) {
    case Family::Sweep:
      MTG_TRY(launch_kernel(h, (SweepKernel)pl.fn, grid, block, pl.smem, stream, prm));
      break;
    case Family::Tmem:
      MTG_TRY(launch_kernel(h, (TmemKernel)pl.fn, grid, block, pl.smem, stream, prm, *tmap));
      break;
    case Family::V4:
      MTG_TRY(launch_kernel(h, (V4Kernel)pl.fn, grid, block, pl.smem, stream, prm, mtg::TmemLaunchV4{counter}, *tmap));
      break;
    case Family::V5: {
      const mtg::TmemLaunchV5 v5{pl.n_buffers, counter};
      MTG_TRY(launch_kernel(h, (V5Kernel)pl.fn, grid, block, pl.smem, stream, prm, v5, *tmap));
      break;
    }
    case Family::Chunked: {
      const mtg::ChunkedLaunch cl{pl.chunk, pl.park_bytes > 0 ? held->p : nullptr, pl.evict_first};
      MTG_TRY(launch_kernel(h, (ChunkedKernel)pl.fn, grid, block, pl.smem, stream, prm, cl, *tmap));
      break;
    }
    case Family::ChunkedPair: {
      const CUtensorMap* tmap2 = nullptr;
      MTG_TRY(coeff_tmap(h, prm.coeffs, prm.B, p, 2 * p->D * p->N, &tmap2));
      const mtg::ChunkedLaunch cl{pl.chunk, pl.park_bytes > 0 ? held->p : nullptr, pl.evict_first};
      MTG_TRY(launch_kernel(h, (ChunkedPairKernel)pl.fn, grid, block, pl.smem, stream, prm, cl, *tmap, *tmap2));
      break;
    }
  }
  return held ? arena_release(h, *held, stream) : MTG_OK;
}

// ---- K4: masked block-tridiagonal kernel, any mask; N in {2..12}, dimension groups of 1..4
int launch_masked(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B, const double* times,
                  const double* dfix, double* coeffs, double* dfree, int32_t* status, cudaStream_t stream, int slot) {
  const Layout& L = topo->layout;
  const int hh = p->N / 2;
  mtg::MaskedParams prm;
  prm.N = p->N;
  prm.r = p->r;
  prm.K = p->K;
  prm.D = p->D;
  prm.n_fixed = L.n_fixed;
  prm.n_free = L.n_free;
  prm.B = B;
  prm.vcol = topo->d_vcol;
  prm.times = times;
  prm.dfix = dfix;
  prm.coeffs = coeffs;
  prm.dfree = dfree;
  prm.status = status;
  mtg_handle::Arena& ar = h->scratch[slot];
  for (int d0 = 0; d0 < p->D;) {
    const int rem = p->D - d0;
    const int dg = rem > 4 ? (rem == 5 ? 3 : 4) : rem;  // 5 = 3 + 2 rather than 4 + 1
    const auto fn = kernel_by_n<2, MTG_MAX_N, 2, 1, 4>(
        [](auto k) { return mtg::masked_block_kernel<decltype(k)::N, decltype(k)::A>; }, p->N, dg);
    const int kslots = hh * (hh + 1) / 2 + hh * dg;
    const size_t smem = size_t(4) * 32 * dg * p->N * sizeof(double);  // staging tiles of the four warps
    MTG_TRY(ensure_dyn_smem(h, (const void*)fn, smem));  // before the occupancy query
    int per_sm = 0;
    MTG_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)fn, 128, smem));
    per_sm = std::max(per_sm, 1);
    const int64_t blocks = capped_grid(h, B, 128, per_sm);
    const size_t bytes = size_t(p->K + 1) * kslots * size_t(blocks) * 128 * sizeof(double);
    MTG_TRY(arena_acquire(h, ar, bytes, stream));
    prm.lifo = ar.p;
    prm.d0 = d0;
    const CUtensorMap* tmap = nullptr;
    MTG_TRY(coeff_tmap(h, coeffs, B, p, dg * p->N, &tmap));
    MTG_TRY(launch_kernel(h, fn, blocks, 128, smem, stream, prm, *tmap));
    MTG_TRY(arena_release(h, ar, stream));
    d0 += dg;
  }
  return MTG_OK;
}

// Fused cost-only solve (SURVEY.md 8f-2): nx problems -> cost_x[nx].  With mel_k1 > 0 the nx = B * mel_k1 problems
// are the Mellinger expansion of the B trajectories in (times, dfix), generated inside the kernel.
// Returns MTG_ERR_ALLOC when no fused kernel / launch configuration exists (caller falls back).
// With ls_grad set the nx = rows * kLineSearchSteps problems are the line-search candidates of the rows in (times, dfix)
// at steps ls_alpha (mtg::WaypointParams).  status_x [nx] or null: every problem's solve status.
int launch_cost_fused(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t nx, const double* times,
                      const double* dfix, double* cost_x, int mel_k1, double inc, double lower, cudaStream_t stream,
                      int32_t* status_x = nullptr, const double* ls_grad = nullptr, const double* ls_alpha = nullptr) {
  const Layout& L = topo->layout;
  const WaypointEntry* e = find_waypoint(p, L);
  if (!e || !e->cost || L.n_free == 0) return MTG_ERR_ALLOC;
  const TmemKernel fn = ls_grad ? e->cost_ls : e->cost;
  const size_t smem = e->v3_smem(p->K);
  bool fits = false;
  MTG_TRY(v3_fits(h, (const void*)fn, smem, &fits));
  if (!fits) return MTG_ERR_ALLOC;  // large K: unfused path (chunked kernel + cost kernel)
  mtg::WaypointParams prm{};  // no coefficient output, no fused inputs
  prm.K = p->K;
  prm.n_fixed = L.n_fixed;
  prm.B = nx;
  prm.times = times;
  prm.dfix = dfix;
  prm.cost = cost_x;
  prm.status = status_x;
  prm.mel_k1 = mel_k1;
  prm.mel_inc = inc;
  prm.mel_lower = lower;
  prm.ls_grad = ls_grad;
  prm.ls_alpha = ls_alpha;
  CUtensorMap tmap;
  std::memset(&tmap, 0, sizeof(tmap));  // unused by the cost-only instantiations
  return launch_kernel(h, fn, (nx + 63) / 64, mtg::kTmemThreads, smem, stream, prm, tmap);
}

int launch_solve(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B, const double* times,
                 const double* dfix, const double* dfree_in, double* coeffs, double* dfree, int32_t* status,
                 cudaStream_t stream, bool backsub_only, const FusedInput* fused = nullptr,
                 int slot = mtg_handle::kPipe) {
  const Layout& L = topo->layout;
  int kind = backsub_only ? MTG_KERNEL_NOFREE : route(p, L);
  // Every specialised kernel stores coefficients in 16-byte units (TMA tensor stores / double2): an output that
  // is only 8-byte aligned (e.g. a tensor slice) takes the banded generic kernel, which stores scalar doubles.
  const bool out_aligned = (reinterpret_cast<uintptr_t>(coeffs) & 15u) == 0;
  if (kind == MTG_KERNEL_WAYPOINT && !fused && !out_aligned) kind = MTG_KERNEL_GENERIC;
  if (kind == MTG_KERNEL_WAYPOINT) {
    mtg::WaypointParams prm{};  // not cost-only
    prm.K = p->K;
    prm.n_fixed = L.n_fixed;
    prm.B = B;
    prm.times = times;
    prm.dfix = dfix;
    prm.coeffs = coeffs;
    prm.dfree = dfree;
    prm.status = status;
    if (fused) {
      prm.positions = fused->positions;
      prm.v_max = fused->v_max;
      prm.a_max = fused->a_max;
      prm.magic = fused->magic;
      prm.times_out = fused->times_out;
    }
    WaypointPlan plan;
    MTG_TRY(plan_waypoint(h, p, L, *find_waypoint(p, L), prm, fused != nullptr, &plan));
    return launch_waypoint(h, p, plan, prm, stream, slot);
  }
  if (kind == MTG_KERNEL_GENERIC && out_aligned && h->generic_variant == 0)
    return launch_masked(h, p, topo, B, times, dfix, coeffs, dfree, status, stream, slot);
  mtg::GenericParams prm;
  prm.N = p->N;
  prm.r = p->r;
  prm.K = p->K;
  prm.D = p->D;
  prm.n_fixed = L.n_fixed;
  prm.n_free = L.n_free;
  prm.bw = L.bw;
  prm.B = B;
  prm.slot_col = topo->d_slot_col;
  prm.times = times;
  prm.dfix = dfix;
  prm.dfree_in = dfree_in;
  prm.coeffs = coeffs;
  prm.dfree = dfree;
  prm.status = status;
  prm.scratch = nullptr;
  prm.scratch_stride = 0;
  const int threads = 128;
  int64_t blocks = (B + threads - 1) / threads;
  const int64_t max_blocks = int64_t(h->sm_count) * 8;
  if (blocks > max_blocks) blocks = max_blocks;
  if (kind == MTG_KERNEL_NOFREE) return launch_kernel(h, mtg::backsub_kernel, blocks, threads, 0, stream, prm);
  const size_t per_thread = size_t(L.n_free) * (L.bw + 1 + p->D);
  const size_t bytes = per_thread * size_t(blocks) * threads * sizeof(double);
  mtg_handle::Arena& ar = h->scratch[slot];
  MTG_TRY(arena_acquire(h, ar, bytes, stream));
  prm.scratch = ar.p;
  prm.scratch_stride = blocks * threads;
  MTG_TRY(launch_kernel(h, mtg::generic_solve_kernel, blocks, threads, 0, stream, prm));
  return arena_release(h, ar, stream);
}

int ensure_pipe(mtg_handle* h, int i, size_t bytes) {
  if (!h->streams[i]) MTG_CUDA(h, cudaStreamCreateWithFlags(&h->streams[i], cudaStreamNonBlocking));
  if (bytes > h->dev_buf_bytes[i]) {
    if (h->dev_buf[i]) {
      MTG_CUDA(h, cudaStreamSynchronize(h->streams[i]));
      cudaFree(h->dev_buf[i]);
      h->dev_buf[i] = nullptr;
      h->dev_buf_bytes[i] = 0;
    }
    MTG_CUDA(h, cudaMalloc(&h->dev_buf[i], bytes));
    h->dev_buf_bytes[i] = bytes;
  }
  return MTG_OK;
}

size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }
// element counts of sub-buffers carved out of one allocation: keep every sub-buffer 256-byte aligned
// (the TMA tensor map of the coefficient buffer needs >= 16 bytes)
size_t align_doubles(size_t n) { return (n + 31) & ~size_t(31); }

// B >= 0, and every array that a batch of B > 0 rows needs is given
bool valid_rows(int64_t B, std::initializer_list<const void*> required) {
  if (B < 0) return false;
  if (B > 0)
    for (const void* q : required)
      if (!q) return false;
  return true;
}

// The opening of every compute entry point: a null handle, the entry's argument check (`valid`), an empty batch
// (`rows` == 0); then `body` runs with the handle's device current.
template <class Body>
int run_entry(mtg_handle* h, bool valid, int64_t rows, Body&& body) {
  if (!h) return MTG_ERR_BAD_ARG;
  if (!valid) {
    h->error = "bad argument";
    return MTG_ERR_BAD_ARG;
  }
  if (rows == 0) return MTG_OK;
  DeviceGuard g(h->device);
  // Clear a stale (non-sticky) error that an earlier failed runtime call left behind: the cudaGetLastError() after
  // our launches must report OUR launch only.  The CUDA runtime is linked in statically and keeps its own last
  // error, so such a call is one of this library's (e.g. an mtg_device_alloc that could not be satisfied).
  (void)cudaGetLastError();
  return body();
}

// run_entry for an entry of one constraint problem: `body` gets the problem's cached layout
template <class Body>
int run_problem_entry(mtg_handle* h, bool valid, const mtg_problem* p, int64_t B, Body&& body) {
  return run_entry(h, valid, B, [&]() -> int {
    CachedTopology* topo = get_topology(h, p);
    return topo ? body(topo) : MTG_ERR_CUDA;
  });
}

// ---- host-pointer entry points: copy in, launch, copy out ---------------------------------------------------
// One host buffer of a host-pointer entry, rows of `row_bytes`: `in` is copied to the device before the launch, the
// device copy to `out` after it.  Either may be null, and both may be the same buffer.
struct HostBuf {
  const void* in;
  void* out;
  size_t row_bytes;
};

// The device copy of a HostBuf (null when both its host pointers are); converts to the launcher's pointer type.
struct DevBuf {
  void* p;
  template <class T>
  operator T*() const {
    return static_cast<T*>(p);
  }
};

// Every exit of a host-pointer entry point -- error returns included -- waits for all pipeline streams:
// copies into caller-owned (possibly pinned) buffers must not be in flight when the caller gets control back.
struct PipeSyncGuard {
  mtg_handle* h;
  ~PipeSyncGuard() {
    for (int i = 0; i < mtg_handle::kPipe; ++i)
      if (h->streams[i]) cudaStreamSynchronize(h->streams[i]);
  }
};

// OneChunk: the whole batch on streams[0], launched with the caller-stream arenas (slot kPipe).  Pipelined: one chunk
// up to 4096 rows; beyond, chunks of ceil(B / kPipe) rows (at most 32768, so that the pipeline has work for every
// stream but stays in a few tens of MB) round-robin over the kPipe streams, each launched with its slot's arenas.
enum class Staging { OneChunk, Pipelined };

// Runs `launch(dev, rows, stream, slot)` on device copies of `bufs` (dev[i] is the copy of bufs[i]), chunk by chunk.
// The sub-buffers of a chunk are 256-byte aligned in its slot's dev_buf.  Every copy in of a chunk is queued before
// any of its copies out, so aliased host buffers stay correct; zero-byte copies are skipped.
template <size_t NB, class Launch>
int stage_host(mtg_handle* h, int64_t B, Staging staging, const HostBuf (&bufs)[NB], Launch&& launch) {
  constexpr int kPipe = mtg_handle::kPipe;
  const bool pipelined = staging == Staging::Pipelined;
  const int64_t chunk =
      pipelined && B > 4096 ? std::max<int64_t>(1, std::min<int64_t>((B + kPipe - 1) / kPipe, 32768)) : B;
  PipeSyncGuard sync_on_exit{h};
  int slot = 0;
  for (int64_t b0 = 0; b0 < B; b0 += chunk, slot = (slot + 1) % kPipe) {
    const int64_t nb = std::min<int64_t>(chunk, B - b0);
    size_t off[NB], total = 0;
    for (size_t i = 0; i < NB; ++i) {
      off[i] = total;
      if (bufs[i].in || bufs[i].out) total = align_up(total + bufs[i].row_bytes * nb);
    }
    MTG_TRY(ensure_pipe(h, slot, total));
    const cudaStream_t s = h->streams[slot];
    char* base = static_cast<char*>(h->dev_buf[slot]);
    DevBuf dev[NB];
    for (size_t i = 0; i < NB; ++i) {
      const HostBuf& b = bufs[i];
      dev[i].p = b.in || b.out ? base + off[i] : nullptr;
      if (b.in && b.row_bytes)
        MTG_CUDA(h, cudaMemcpyAsync(dev[i].p, static_cast<const char*>(b.in) + b0 * b.row_bytes, b.row_bytes * nb,
                                    cudaMemcpyHostToDevice, s));
    }
    MTG_TRY(launch(dev, nb, s, pipelined ? slot : kPipe));
    for (size_t i = 0; i < NB; ++i) {
      const HostBuf& b = bufs[i];
      if (b.out && b.row_bytes)
        MTG_CUDA(h, cudaMemcpyAsync(static_cast<char*>(b.out) + b0 * b.row_bytes, dev[i].p, b.row_bytes * nb,
                                    cudaMemcpyDeviceToHost, s));
    }
    // the buffer of this slot is reused kPipe chunks later: wait for it then
    const int next = (slot + 1) % kPipe;
    if (b0 + chunk < B && h->streams[next]) MTG_CUDA(h, cudaStreamSynchronize(h->streams[next]));
  }
  for (int i = 0; i < kPipe; ++i)
    if (h->streams[i]) MTG_CUDA(h, cudaStreamSynchronize(h->streams[i]));
  return MTG_OK;
}

}  // namespace

extern "C" {

int mtg_version(void) { return 100; }

int mtg_create(int device, mtg_handle** out) {
  if (!out) return MTG_ERR_BAD_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e);
    return MTG_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= count) {
    g_create_error = "device index out of range";
    return MTG_ERR_BAD_ARG;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) {
    g_create_error = std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e);
    return MTG_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    g_create_error = "this library contains sm_90a code only; device is sm_" + std::to_string(prop.major) +
                     std::to_string(prop.minor);
    return MTG_ERR_NO_DEVICE;
  }
  mtg_handle* h = new (std::nothrow) mtg_handle();
  if (!h) return MTG_ERR_ALLOC;
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  h->cc_major = prop.major;
  h->smem_optin = prop.sharedMemPerBlockOptin;
  *out = h;
  return MTG_OK;
}

void mtg_destroy(mtg_handle* h) {
  if (!h) return;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  for (auto& t : h->topologies) {
    cudaFree(t.d_slot_col);
    cudaFree(t.d_vcol);
  }
  for (int i = 0; i <= mtg_handle::kPipe; ++i) {
    for (mtg_handle::Arena* a : {&h->scratch[i], &h->pack[i], &h->counters[i], &h->optim[i]}) {
      if (a->p) cudaFree(a->p);
      if (a->ev) cudaEventDestroy(a->ev);
    }
  }
  for (int i = 0; i < mtg_handle::kPipe; ++i) {
    if (h->dev_buf[i]) cudaFree(h->dev_buf[i]);
    if (h->streams[i]) cudaStreamDestroy(h->streams[i]);
  }
  if (h->pinned_count) cudaFreeHost(h->pinned_count);
  if (h->count_ev) cudaEventDestroy(h->count_ev);
  delete h;
}

const char* mtg_last_error(const mtg_handle* h) { return h ? h->error.c_str() : g_create_error.c_str(); }

int64_t mtg_launch_count(const mtg_handle* h) { return h ? h->launches : 0; }

int mtg_device_is_sm90(const mtg_handle* h) { return h && h->cc_major == 9; }

int mtg_set_option(mtg_handle* h, int key, int value) {
  if (!h) return MTG_ERR_BAD_ARG;
  if (key == MTG_OPT_MELLINGER_UNFUSED && (value == 0 || value == 1)) {
    h->mellinger_unfused = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_GENERIC_VARIANT && (value == 0 || value == 1)) {
    h->generic_variant = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_CHUNK_BLOCKS && value >= 0 && value <= 64) {
    h->chunk_blocks = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_CHUNK_WARPS && (value == 0 || value == 1 || value == 4)) {
    h->chunk_warps = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_L2_HINTS && (value == 0 || value == 1)) {
    h->l2_hints = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_TMA_INPUTS && value >= 0 && value <= 2) {
    h->tma_inputs = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_WAYPOINT_VARIANT && value >= 0 && value <= 6) {
    h->waypoint_variant = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_EARLY_REFILL && value >= -1 && value <= 0) {
    h->early_steps = value;
    return MTG_OK;
  }
  // reserved keys: accepted in their documented ranges, no effect
  if ((key == MTG_OPT_RING_DEPTH && value >= 2 && value <= 4) ||
      (key == MTG_OPT_STAGGER_US && value >= 0 && value <= 1000))
    return MTG_OK;
  if (key == MTG_OPT_CTAS_PER_SM && value >= 0 && value <= 9) {
    h->ctas_per_sm = value;
    return MTG_OK;
  }
  if (key == MTG_OPT_DYNAMIC_TILES && value >= 0 && value <= 2) {  // 0 = auto, 1 = always, 2 = never
    h->dynamic_tiles = value;
    return MTG_OK;
  }
  h->error = "unknown option";
  return MTG_ERR_BAD_ARG;
}

int mtg_problem_layout(const mtg_problem* p, mtg_layout* out, int32_t* slot_col) {
  if (!valid_problem(p) || !out) return MTG_ERR_BAD_ARG;
  Layout L;
  compute_layout(p->N, p->K, canonical_mask(p), &L);
  out->n_all = L.n_all;
  out->n_fixed = L.n_fixed;
  out->n_free = L.n_free;
  out->kernel = route(p, L);
  if (slot_col) std::memcpy(slot_col, L.slot_col.data(), sizeof(int32_t) * L.slot_col.size());
  return MTG_OK;
}

// ---- the compute entry points ------------------------------------------------------------------------------------
// Each kind has one argument check, shared by its device entry and its host twin, and one launcher, which takes
// checked arguments and launches on `s` (with the arenas of pipeline slot `slot` where it uses any).  A device entry
// is run_entry() around its launcher; a host entry is run_entry() around stage_host() around the same launcher.  Each
// launcher starts its kernels with launch_kernel(), sized by capped_grid() (the segment-parallel ones through
// launch_segment_parallel()), and picks an order's instantiation with kernel_by_n().

// the entries of one constraint problem with three arrays that every row needs (solve, setFreeConstraints,
// computeCost, the Mellinger gradient)
static bool valid_problem_args(const mtg_problem* p, int64_t B, const double* a, const double* b, const double* c) {
  return valid_problem(p) && valid_rows(B, {a, b, c});
}

// setFreeConstraints needs d_free whenever the problem has free constraints
static int check_d_free(mtg_handle* h, const Layout& L, const double* d_free) {
  if (L.n_free == 0 || d_free) return MTG_OK;
  h->error = "d_free is required for back-substitution of a problem with free constraints";
  return MTG_ERR_BAD_ARG;
}

// solveLinear (backsub_only = false) and setFreeConstraints (backsub_only = true)
static int solve_device(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times, const double* d_fixed,
                        const double* d_free_in, double* coeffs, double* d_free, int32_t* status, void* stream,
                        bool backsub_only) {
  return run_problem_entry(h, valid_problem_args(p, B, seg_times, d_fixed, coeffs), p, B, [&](CachedTopology* topo) {
    if (backsub_only) MTG_TRY(check_d_free(h, topo->layout, d_free_in));
    return launch_solve(h, p, topo, B, seg_times, d_fixed, d_free_in, coeffs, d_free, status, (cudaStream_t)stream,
                        backsub_only);
  });
}

int mtg_solve_linear_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                               const double* d_fixed, double* coeffs, double* d_free, int32_t* status,
                               void* stream) {
  return solve_device(h, p, B, seg_times, d_fixed, nullptr, coeffs, d_free, status, stream, false);
}

static bool valid_nfabian(const mtg_problem* p, int64_t B, const double* positions, double v_max, double a_max,
                          const double* coeffs) {
  return valid_problem(p) && v_max > 0.0 && a_max > 0.0 && valid_rows(B, {positions, coeffs});
}

static int launch_nfabian(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B, const double* positions,
                          double v_max, double a_max, double magic, double* coeffs, double* seg_times_out,
                          int32_t* status, cudaStream_t s, int slot) {
  const Layout& L = topo->layout;
  if (route(p, L) == MTG_KERNEL_WAYPOINT) {
    FusedInput f = {positions, v_max, a_max, magic, seg_times_out};
    const int rc = launch_solve(h, p, topo, B, nullptr, nullptr, nullptr, coeffs, nullptr, status, s, false, &f, slot);
    if (rc != MTG_ERR_ALLOC) return rc;
  }
  // no fused specialisation: pack (times, d_fixed) with a small kernel, then the regular path
  const size_t n_t = align_doubles(size_t(B) * p->K), n_f = size_t(B) * p->D * L.n_fixed;
  mtg_handle::Arena& ar = h->pack[slot];
  MTG_TRY(arena_acquire(h, ar, (n_t + n_f) * 8, s));
  double* t_buf = seg_times_out ? seg_times_out : ar.p;
  double* f_buf = ar.p + n_t;
  mtg::PackParams pk;
  pk.N = p->N;
  pk.K = p->K;
  pk.D = p->D;
  pk.n_fixed = L.n_fixed;
  pk.B = B;
  pk.positions = positions;
  pk.v_max = v_max;
  pk.a_max = a_max;
  pk.magic = magic;
  pk.times = t_buf;
  pk.dfix = f_buf;
  MTG_TRY(launch_kernel(h, mtg::nfabian_pack_kernel, capped_grid(h, B, 128, 16), 128, 0, s, pk));
  MTG_TRY(launch_solve(h, p, topo, B, t_buf, f_buf, nullptr, coeffs, nullptr, status, s, false, nullptr, slot));
  return arena_release(h, ar, s);  // the solve was the last reader of the packed inputs
}

int mtg_solve_waypoints_nfabian_batch_f64(mtg_handle* h, int32_t N, int32_t r, int32_t K, int32_t D, int64_t B,
                                          const double* positions, double v_max, double a_max, double magic,
                                          double* coeffs, double* seg_times_out, int32_t* status, void* stream) {
  const mtg_problem p = {N, r, K, D, nullptr};
  return run_problem_entry(h, valid_nfabian(&p, B, positions, v_max, a_max, coeffs), &p, B, [&](CachedTopology* topo) {
    return launch_nfabian(h, &p, topo, B, positions, v_max, a_max, magic, coeffs, seg_times_out, status,
                          (cudaStream_t)stream, mtg_handle::kPipe);
  });
}

int mtg_coeffs_from_constraints_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                          const double* seg_times, const double* d_fixed,
                                          const double* d_free, double* coeffs, void* stream) {
  return solve_device(h, p, B, seg_times, d_fixed, d_free, coeffs, nullptr, nullptr, stream, true);
}

static int launch_cost(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times, const double* coeffs,
                       double* cost, cudaStream_t s) {
  mtg::CostParams prm;
  prm.N = p->N;
  prm.r = p->r;
  prm.K = p->K;
  prm.D = p->D;
  prm.B = B;
  prm.times = seg_times;
  prm.coeffs = coeffs;
  prm.cost = cost;
  const int threads = 256;
  const int KD = p->K * p->D;
  const int tpb = std::max(1, threads / KD);
  const size_t smem = (size_t(36) + size_t(tpb) * KD) * sizeof(double);
  if (smem > h->smem_optin) {
    h->error = "mtg_compute_cost_batch_f64: K * D too large";
    return MTG_ERR_BAD_ARG;
  }
  typedef void (*CostFn)(const mtg::CostParams, const int);
  struct CostKernelEntry {
    int N, r;
    CostFn fn;
  };
  static const CostKernelEntry kComputeCostKernels[] = {
      {10, 4, mtg::cost_kernel<10, 4>}, {10, 3, mtg::cost_kernel<10, 3>}, {10, 2, mtg::cost_kernel<10, 2>},
      {8, 3, mtg::cost_kernel<8, 3>},   {12, 5, mtg::cost_kernel<12, 5>}, {12, 4, mtg::cost_kernel<12, 4>},
      {6, 2, mtg::cost_kernel<6, 2>},   {4, 1, mtg::cost_kernel<4, 1>}};
  CostFn fn = mtg::cost_kernel<0, 0>;
  for (const auto& e : kComputeCostKernels)
    if (e.N == p->N && e.r == p->r) fn = e.fn;
  return launch_kernel(h, fn, capped_grid(h, B, tpb, 16), threads, smem, s, prm, tpb);
}

int mtg_compute_cost_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                               const double* coeffs, double* cost, void* stream) {
  return run_entry(h, valid_problem_args(p, B, seg_times, coeffs, cost), B,
                   [&] { return launch_cost(h, p, B, seg_times, coeffs, cost, (cudaStream_t)stream); });
}

int mtg_evaluate_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                           const double* coeffs, int32_t derivative, double t_start, double dt, int32_t n_samples,
                           double* out, void* stream) {
  const bool valid = N >= 1 && N <= MTG_MAX_N && K >= 1 && D >= 1 && B >= 0 && derivative >= 0 && n_samples >= 0 &&
                     (n_samples == 0 || valid_rows(B, {seg_times, coeffs, out}));
  return run_entry(h, valid, n_samples > 0 ? B : 0, [&]() -> int {
    mtg::EvalParams ep;
    ep.N = N;
    ep.K = K;
    ep.D = D;
    ep.derivative = derivative;
    ep.n_samples = n_samples;
    ep.B = B;
    ep.t_start = t_start;
    ep.dt = dt;
    ep.times = seg_times;
    ep.coeffs = coeffs;
    ep.out = out;
    if (size_t(32) * D * 8 > size_t(160) * 1024) {
      h->error = "mtg_evaluate_batch_f64: D too large for the output tile";
      return MTG_ERR_BAD_ARG;
    }
    const int threads = std::max(32, std::min(256, int((40 * 1024) / (D * 8)) / 32 * 32));
    const size_t smem = size_t(threads) * D * sizeof(double);
    const auto fn = kernel_by_n<1, MTG_MAX_N>([](auto k) { return mtg::evaluate_kernel<decltype(k)::N>; }, N);
    return launch_kernel(h, fn, capped_grid(h, B * int64_t(n_samples), threads, 32), threads, smem,
                         (cudaStream_t)stream, ep);
  });
}

// evaluateRange: 1..8 derivative orders, each >= 0, dt > 0; out may be null while max_samples is 0
static bool valid_range(int32_t N, int32_t K, int32_t D, int64_t B, double dt, int32_t n_derivs, const int32_t* derivs,
                        int32_t max_samples, const double* seg_times, const double* coeffs, const double* out,
                        const int32_t* n_samples) {
  if (N < 1 || N > MTG_MAX_N || K < 1 || D < 1 || n_derivs < 1 || n_derivs > 8 || !derivs || max_samples < 0 ||
      !(dt > 0.0))
    return false;
  for (int q = 0; q < n_derivs; ++q)
    if (derivs[q] < 0) return false;
  return valid_rows(B, {seg_times, coeffs, n_samples}) && (B == 0 || max_samples == 0 || out);
}

// range_walk_kernel over the rows of `rp`: each sample's segment and local time, into rp.t_local and rp.seg_idx in
// pipeline slot `slot`'s pack arena, which this acquires.  The caller evaluates the samples and releases the arena.
static int walk_range(mtg_handle* h, mtg::RangeParams& rp, cudaStream_t s, int slot) {
  const size_t ns = size_t(rp.B) * size_t(std::max(rp.max_samples, 1));
  mtg_handle::Arena& ar = h->pack[slot];
  const size_t o_idx = align_doubles(ns);  // t_local first (doubles), then seg_idx (int32)
  MTG_TRY(arena_acquire(h, ar, (o_idx + align_doubles((ns + 1) / 2)) * 8, s));
  rp.t_local = ar.p;
  rp.seg_idx = reinterpret_cast<int*>(ar.p + o_idx);
  return launch_kernel(h, mtg::range_walk_kernel, capped_grid(h, rp.B, 128, 16), 128, 0, s, rp);
}

static int launch_range(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                        const double* coeffs, double t_start, double t_end, double dt, int32_t n_derivs,
                        const int32_t* derivs, int32_t max_samples, double* out, int32_t* n_samples,
                        double* sampling_times, cudaStream_t s, int slot) {
  mtg::RangeParams rp;
  rp.N = N;
  rp.K = K;
  rp.D = D;
  rp.n_derivs = n_derivs;
  rp.max_samples = max_samples;
  for (int q = 0; q < 8; ++q) rp.derivs[q] = q < n_derivs ? derivs[q] : 0;
  rp.B = B;
  rp.t_start = t_start;
  rp.t_end = t_end;
  rp.dt = dt;
  rp.times = seg_times;
  rp.coeffs = coeffs;
  rp.n_samples = n_samples;
  rp.sampling_times = sampling_times;
  rp.out = out;
  rp.range_rule = mtg::kRangePlain;
  rp.time_ns = nullptr;
  MTG_TRY(walk_range(h, rp, s, slot));
  mtg_handle::Arena& ar = h->pack[slot];
  if (max_samples > 0) {
    // block size: the output tile (threads * n_derivs * D doubles) stays under 40 KB of shared memory
    const int rec = n_derivs * D;
    if (size_t(32) * rec * 8 > size_t(160) * 1024) {
      h->error = "mtg_evaluate_range_batch_f64: n_derivs * D too large for the output tile";
      arena_release(h, ar, s);
      return MTG_ERR_BAD_ARG;
    }
    const int threads = std::max(32, std::min(256, int((40 * 1024) / (rec * 8)) / 32 * 32));
    const size_t smem = size_t(threads) * rec * sizeof(double);
    const auto fn = kernel_by_n<1, MTG_MAX_N>([](auto k) { return mtg::range_eval_kernel<decltype(k)::N>; }, N);
    MTG_TRY(launch_kernel(h, fn, capped_grid(h, B * int64_t(max_samples), threads, 32), threads, smem, s, rp));
  }
  return arena_release(h, ar, s);
}

int mtg_evaluate_range_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                 const double* coeffs, double t_start, double t_end, double dt, int32_t n_derivs,
                                 const int32_t* derivs, int32_t max_samples, double* out, int32_t* n_samples,
                                 double* sampling_times, void* stream) {
  return run_entry(h, valid_range(N, K, D, B, dt, n_derivs, derivs, max_samples, seg_times, coeffs, out, n_samples), B,
                   [&] {
                     return launch_range(h, N, K, D, B, seg_times, coeffs, t_start, t_end, dt, n_derivs, derivs,
                                         max_samples, out, n_samples, sampling_times, (cudaStream_t)stream,
                                         mtg_handle::kPipe);
                   });
}

// ---- flat-state samplers ------------------------------------------------------------------------------------------
static int flat_attitude(int32_t D) { return D == 4 ? mtg::kAttYaw : D == 6 ? mtg::kAttRotationVector : mtg::kAttNone; }

static bool valid_flat_range(int32_t N, int32_t K, int32_t D, int64_t B, double dt, int32_t max_samples, const double* seg_times,
                             const double* coeffs, const double* states, const int32_t* n_samples) {
  return N >= 1 && N <= MTG_MAX_N && K >= 1 && D >= 1 && max_samples >= 0 && dt > 0.0 && std::isfinite(dt) &&
         valid_rows(B, {seg_times, coeffs, n_samples}) && (B == 0 || max_samples == 0 || states);
}

// range_walk_kernel under sampleTrajectoryInRange's rule, then flat_state_range_kernel
static int launch_flat_range(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                             const double* coeffs, double min_time, double max_time, double dt, int32_t whole,
                             int32_t max_samples, double* states, int64_t* time_ns, int32_t* n_samples, cudaStream_t s,
                             int slot) {
  mtg::RangeParams rp = {};
  rp.N = N;
  rp.K = K;
  rp.D = D;
  rp.max_samples = max_samples;
  rp.B = B;
  rp.t_start = min_time;
  rp.t_end = max_time;
  rp.dt = dt;
  rp.times = seg_times;
  rp.coeffs = coeffs;
  rp.n_samples = n_samples;
  rp.sampling_times = nullptr;
  rp.out = states;
  rp.range_rule = whole ? mtg::kRangeWhole : mtg::kRangeChecked;
  rp.time_ns = reinterpret_cast<long long*>(time_ns);
  MTG_TRY(walk_range(h, rp, s, slot));
  if (max_samples > 0) {
    const auto fn = kernel_by_n<1, MTG_MAX_N, 1, mtg::kAttNone, mtg::kAttRotationVector>(
        [](auto k) { return mtg::flat_state_range_kernel<decltype(k)::N, decltype(k)::A>; }, N, flat_attitude(D));
    const int threads = mtg::kFlatStateThreads;
    MTG_TRY(launch_kernel(h, fn, capped_grid(h, B * int64_t(max_samples), threads, 16), threads, 0, s, rp));
  }
  return arena_release(h, h->pack[slot], s);
}

int mtg_sample_flat_states_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                     const double* coeffs, double min_time, double max_time, double sampling_interval,
                                     int32_t whole, int32_t max_samples, double* states, int64_t* time_ns,
                                     int32_t* n_samples, void* stream) {
  return run_entry(
      h, valid_flat_range(N, K, D, B, sampling_interval, max_samples, seg_times, coeffs, states, n_samples), B, [&] {
        return launch_flat_range(h, N, K, D, B, seg_times, coeffs, min_time, max_time, sampling_interval, whole,
                                 max_samples, states, time_ns, n_samples, (cudaStream_t)stream, mtg_handle::kPipe);
      });
}

static int launch_flat_at_time(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                               const double* coeffs, const double* sample_times, double* states, int64_t* time_ns,
                               int32_t* ok, cudaStream_t s) {
  mtg::FlatAtTimeParams prm;
  prm.K = K;
  prm.D = D;
  prm.B = B;
  prm.times = seg_times;
  prm.coeffs = coeffs;
  prm.sample_times = sample_times;
  prm.states = states;
  prm.time_ns = reinterpret_cast<long long*>(time_ns);
  prm.ok = ok;
  const auto fn = kernel_by_n<1, MTG_MAX_N, 1, mtg::kAttNone, mtg::kAttRotationVector>(
      [](auto k) { return mtg::flat_state_at_time_kernel<decltype(k)::N, decltype(k)::A>; }, N, flat_attitude(D));
  const int threads = mtg::kFlatStateThreads;
  return launch_kernel(h, fn, capped_grid(h, B, threads, 16), threads, 0, s, prm);
}

static bool valid_flat_at_time(int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times, const double* coeffs,
                               const double* sample_times, const double* states, const int32_t* ok) {
  return N >= 1 && N <= MTG_MAX_N && K >= 1 && D >= 1 && valid_rows(B, {seg_times, coeffs, sample_times, states, ok});
}

int mtg_sample_flat_state_at_time_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                            const double* seg_times, const double* coeffs, const double* sample_times,
                                            double* states, int64_t* time_ns, int32_t* ok, void* stream) {
  return run_entry(h, valid_flat_at_time(N, K, D, B, seg_times, coeffs, sample_times, states, ok), B, [&] {
    return launch_flat_at_time(h, N, K, D, B, seg_times, coeffs, sample_times, states, time_ns, ok,
                               (cudaStream_t)stream);
  });
}

// status_x [B][K+1] or null: the status of every solve (the unperturbed one first)
static int launch_mellinger(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B,
                            const double* seg_times, const double* d_fixed, double* cost, double* grad, cudaStream_t s,
                            int slot, int32_t* status_x = nullptr) {
  const Layout& L = topo->layout;
  const size_t K = p->K, D = p->D, N = p->N, nf = L.n_fixed;
  mtg_handle::Arena& ar = h->pack[slot];
  if (p->K > 1 && h->mellinger_unfused == 0) {
    // fused path: one cost-only launch over the B*(K+1) expanded problems (expansion generated in the kernel, no
    // perturbed inputs or coefficients ever written), then the finite differences
    MTG_TRY(arena_acquire(h, ar, size_t(B) * (K + 1) * 8, s));
    const int rc =
        launch_cost_fused(h, p, topo, B * int64_t(K + 1), seg_times, d_fixed, ar.p, int(K + 1), 0.1, 0.1, s, status_x);
    if (rc == MTG_OK) {
      MTG_TRY(launch_kernel(h, mtg::mellinger_gradient_kernel, capped_grid(h, B, 128, 16), 128, 0, s, B, p->K, ar.p,
                            cost, grad, 0.1));
      return arena_release(h, ar, s);
    }
    if (rc != MTG_ERR_ALLOC) return rc;
  }
  const size_t per_x = (K + D * nf + K * D * N + 1) * 8;  // times + d_fixed + coeffs + cost of one expanded problem
  int64_t chunk = std::max<int64_t>(1, int64_t((size_t(384) << 20) / (per_x * (K + 1))));
  chunk = std::min<int64_t>(chunk, B);
  const size_t nx_max = size_t(chunk) * (K + 1);
  const size_t o_f = align_doubles(nx_max * K), o_c = o_f + align_doubles(nx_max * D * nf),
               o_j = o_c + align_doubles(nx_max * K * D * N), need = (o_j + align_doubles(nx_max)) * 8;
  MTG_TRY(arena_acquire(h, ar, need, s));
  for (int64_t b0 = 0; b0 < B; b0 += chunk) {
    const int64_t nb = std::min<int64_t>(chunk, B - b0), nx = nb * int64_t(K + 1);
    double* t_x = ar.p;
    double* f_x = ar.p + o_f;
    double* c_x = ar.p + o_c;
    double* j_x = ar.p + o_j;
    mtg::MellingerParams mp;
    mp.K = p->K;
    mp.D = p->D;
    mp.n_fixed = L.n_fixed;
    mp.B = nb;
    mp.times = seg_times + b0 * K;
    mp.dfix = d_fixed + b0 * D * nf;
    mp.times_x = t_x;
    mp.dfix_x = f_x;
    mp.increment = 0.1;  // reference: increment_time (nonlinear_impl.h:310)
    mp.lower = 0.1;      // kOptimizationTimeLowerBound (polynomial_optimization_nonlinear.h:31)
    MTG_TRY(launch_kernel(h, mtg::mellinger_expand_kernel, capped_grid(h, nx, 128, 16), 128, 0, s, mp));
    MTG_TRY(launch_solve(h, p, topo, nx, t_x, f_x, nullptr, c_x, nullptr,
                         status_x ? status_x + b0 * int64_t(K + 1) : nullptr, s, false, nullptr, slot));
    MTG_TRY(launch_cost(h, p, nx, t_x, c_x, j_x, s));
    MTG_TRY(launch_kernel(h, mtg::mellinger_gradient_kernel, capped_grid(h, nb, 128, 16), 128, 0, s, nb, p->K, j_x,
                          cost ? cost + b0 : nullptr, grad + b0 * K, mp.increment));
  }
  return arena_release(h, ar, s);
}

int mtg_cost_gradient_mellinger_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                          const double* d_fixed, double* cost, double* grad, void* stream) {
  return run_problem_entry(h, valid_problem_args(p, B, seg_times, d_fixed, grad), p, B, [&](CachedTopology* topo) {
    return launch_mellinger(h, p, topo, B, seg_times, d_fixed, cost, grad, (cudaStream_t)stream, mtg_handle::kPipe);
  });
}

// computeMaximumOfMagnitude: N even in [2, 12], 1..8 derivative orders, each in [0, N-2] (linear_impl.h:401 CHECKs
// N - k - 1 > 0)
static bool valid_extrema_args(int32_t N, int32_t K, int32_t D, int64_t B, int32_t n_derivs, const int32_t* derivs,
                               const double* seg_times, const double* coeffs, const double* value) {
  if (N < 2 || N > MTG_MAX_N || (N & 1) || K < 1 || D < 1) return false;
  if (n_derivs < 1 || n_derivs > mtg::kExtremaMaxDerivs || !derivs) return false;
  for (int q = 0; q < n_derivs; ++q)
    if (derivs[q] < 0 || derivs[q] > N - 2) return false;
  return valid_rows(B, {seg_times, coeffs, value});
}

static int launch_max_magnitude(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                const double* coeffs, int32_t n_derivs, const int32_t* derivs, double* value,
                                double* time, int32_t* segment, int32_t* status, cudaStream_t s) {
  mtg::ExtremaParams ep;
  ep.K = K;
  ep.D = D;
  ep.n_derivs = n_derivs;
  for (int q = 0; q < mtg::kExtremaMaxDerivs; ++q) ep.derivs[q] = q < n_derivs ? derivs[q] : 0;
  ep.B = B;
  ep.times = seg_times;
  ep.coeffs = coeffs;
  ep.value = value;
  ep.time = time;
  ep.segment = segment;
  ep.status = status;
  const auto fn = kernel_by_n<2, MTG_MAX_N, 2>([](auto k) { return mtg::max_magnitude_kernel<decltype(k)::N>; }, N);
  return launch_segment_parallel(h, fn, ep, K, B, size_t(2) * K * n_derivs * sizeof(double),
                                 "mtg_max_magnitude_batch_f64", "K * n_derivs", s);
}

int mtg_max_magnitude_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                const double* coeffs, int32_t n_derivs, const int32_t* derivs, double* value,
                                double* time, int32_t* segment, int32_t* status, void* stream) {
  return run_entry(h, valid_extrema_args(N, K, D, B, n_derivs, derivs, seg_times, coeffs, value), B, [&] {
    return launch_max_magnitude(h, N, K, D, B, seg_times, coeffs, n_derivs, derivs, value, time, segment, status,
                                (cudaStream_t)stream);
  });
}

static bool valid_objective(const mtg_problem* p, int64_t B, const mtg_time_objective* obj, const double* seg_times,
                            const double* d_fixed, const double* coeffs, const double* objective) {
  if (!valid_problem(p) || !obj || (obj->time_cost != 0 && obj->time_cost != 1)) return false;
  if (obj->n_constraints < 0 || obj->n_constraints > mtg::kExtremaMaxDerivs) return false;
  if (obj->n_constraints > 0 && !obj->constraints) return false;
  for (int q = 0; q < obj->n_constraints; ++q) {
    const mtg_soft_constraint& c = obj->constraints[q];
    // max_value == 0 would divide by zero in the reference (nonlinear_impl.h:785)
    if (c.derivative < 0 || c.derivative > p->N - 2 || !(c.max_value > 0.0) || !std::isfinite(c.max_value)) return false;
  }
  return valid_rows(B, {seg_times, d_fixed, coeffs, objective});
}

static int launch_time_objective(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B,
                                 const double* seg_times, const double* d_fixed, const double* d_free,
                                 const mtg_time_objective* obj, double* coeffs, double* objective, double* terms,
                                 int32_t* status, cudaStream_t s, int slot) {
  const int nc = obj->n_constraints;
  // scratch: computeCost [B], maxima [B][nc], solve status [B]
  const size_t o_max = align_doubles(size_t(B)), o_st = o_max + align_doubles(size_t(B) * nc),
               need = (o_st + align_doubles((size_t(B) + 1) / 2)) * 8;
  mtg_handle::Arena& ar = h->pack[slot];
  MTG_TRY(arena_acquire(h, ar, need, s));
  double* cost = ar.p;
  double* maxima = ar.p + o_max;
  int32_t* solve_status = reinterpret_cast<int32_t*>(ar.p + o_st);
  MTG_CUDA(h, cudaMemsetAsync(solve_status, 0, sizeof(int32_t) * size_t(B), s));
  // the same launches as mtg_solve_linear_batch_f64 / mtg_coeffs_from_constraints_batch_f64
  if (!d_free)
    MTG_TRY(launch_solve(h, p, topo, B, seg_times, d_fixed, nullptr, coeffs, nullptr, solve_status, s, false, nullptr,
                         slot));
  else
    MTG_TRY(launch_solve(h, p, topo, B, seg_times, d_fixed, d_free, coeffs, nullptr, nullptr, s, true, nullptr, slot));
  MTG_TRY(launch_cost(h, p, B, seg_times, coeffs, cost, s));
  mtg::ObjectiveParams op;
  op.K = p->K;
  op.n_constraints = nc;
  op.richter = obj->time_cost;
  op.time_penalty = obj->time_penalty;
  op.weight = obj->soft_constraint_weight;
  op.maximum_cost = obj->maximum_cost;
  if (nc > 0) {
    int32_t derivs[mtg::kExtremaMaxDerivs];
    for (int q = 0; q < nc; ++q) {
      derivs[q] = obj->constraints[q].derivative;
      op.max_value[q] = obj->constraints[q].max_value;
    }
    MTG_TRY(launch_max_magnitude(h, p->N, p->K, p->D, B, seg_times, coeffs, nc, derivs, maxima, nullptr, nullptr, nullptr,
                                 s));
  }
  op.B = B;
  op.times = seg_times;
  op.cost = cost;
  op.maxima = maxima;
  op.solve_status = solve_status;
  op.objective = objective;
  op.terms = terms;
  op.status = status;
  MTG_TRY(launch_kernel(h, mtg::time_objective_kernel, capped_grid(h, B, 128, 16), 128, 0, s, op));
  return arena_release(h, ar, s);
}

int mtg_time_objective_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                 const double* d_fixed, const double* d_free, const mtg_time_objective* obj,
                                 double* coeffs, double* objective, double* terms, int32_t* status, void* stream) {
  return run_problem_entry(h, valid_objective(p, B, obj, seg_times, d_fixed, coeffs, objective), p, B,
                           [&](CachedTopology* topo) {
                             return launch_time_objective(h, p, topo, B, seg_times, d_fixed, d_free, obj, coeffs,
                                                          objective, terms, status, (cudaStream_t)stream,
                                                          mtg_handle::kPipe);
                           });
}

// scaleSegmentTimesToMeetConstraints: N even in [4, 12] (N = 2 has no acceleration), limits > 0 (+inf = no limit)
static bool valid_scale_args(int32_t N, int32_t K, int32_t D, int64_t B, double v_max, double a_max) {
  return N >= 4 && N <= MTG_MAX_N && !(N & 1) && K >= 1 && D >= 1 && B >= 0 && v_max > 0.0 && a_max > 0.0;
}

static bool valid_scale(int32_t N, int32_t K, int32_t D, int64_t B, double v_max, double a_max, const double* seg_times,
                        const double* coeffs, const double* seg_times_out, const double* coeffs_out) {
  return valid_scale_args(N, K, D, B, v_max, a_max) && valid_rows(B, {seg_times, coeffs, seg_times_out, coeffs_out});
}

static int launch_scale_to_constraints(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                       const double* seg_times, const double* coeffs, double v_max, double a_max,
                                       double* seg_times_out, double* coeffs_out, const int32_t* skip,
                                       int32_t* within_range, double* maxima, int32_t* status, cudaStream_t s) {
  mtg::ScaleParams sp;
  sp.K = K;
  sp.D = D;
  sp.B = B;
  sp.v_max = v_max;
  sp.a_max = a_max;
  sp.times = seg_times;
  sp.coeffs = coeffs;
  sp.times_out = seg_times_out;
  sp.coeffs_out = coeffs_out;
  sp.skip = skip;
  sp.within = within_range;
  sp.maxima = maxima;
  sp.status = status;
  const auto fn =
      kernel_by_n<4, MTG_MAX_N, 2>([](auto k) { return mtg::scale_to_constraints_kernel<decltype(k)::N>; }, N);
  return launch_segment_parallel(h, fn, sp, K, B, size_t(2) * K * sizeof(double) + sizeof(double) + sizeof(int),
                                 "mtg_scale_to_constraints_batch_f64", "K", s);
}

int mtg_scale_to_constraints_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                       const double* seg_times, const double* coeffs, double v_max, double a_max,
                                       double* seg_times_out, double* coeffs_out, int32_t* within_range,
                                       double* maxima, int32_t* status, void* stream) {
  return run_entry(h, valid_scale(N, K, D, B, v_max, a_max, seg_times, coeffs, seg_times_out, coeffs_out), B, [&] {
    return launch_scale_to_constraints(h, N, K, D, B, seg_times, coeffs, v_max, a_max, seg_times_out, coeffs_out,
                                       nullptr, within_range, maxima, status, (cudaStream_t)stream);
  });
}

static bool valid_violation(const mtg_problem* p, int64_t B, double v_max, double a_max, const double* seg_times,
                            const double* d_fixed, const double* coeffs, const double* seg_times_out) {
  return valid_problem(p) && valid_scale_args(p->N, p->K, p->D, B, v_max, a_max) &&
         valid_rows(B, {seg_times, d_fixed, coeffs, seg_times_out});
}

static int launch_scale_with_violation(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B,
                                       const double* seg_times, const double* d_fixed, double v_max, double a_max,
                                       double* coeffs, double* seg_times_out, int32_t* within_range, double* maxima,
                                       int32_t* status, cudaStream_t s, int slot, const int32_t* pass = nullptr) {
  // scratch: status of the first solve [B], of the scaling [B], of the re-solve [B]
  const size_t o_sc = align_doubles((size_t(B) + 1) / 2), o_re = 2 * o_sc;
  mtg_handle::Arena& ar = h->pack[slot];
  MTG_TRY(arena_acquire(h, ar, 3 * o_sc * 8, s));
  int32_t* st_solve = reinterpret_cast<int32_t*>(ar.p);
  int32_t* st_scale = reinterpret_cast<int32_t*>(ar.p + o_sc);
  int32_t* st_resolve = reinterpret_cast<int32_t*>(ar.p + o_re);
  MTG_CUDA(h, cudaMemsetAsync(st_solve, 0, sizeof(int32_t) * size_t(B), s));
  MTG_CUDA(h, cudaMemsetAsync(st_resolve, 0, sizeof(int32_t) * size_t(B), s));
  // nonlinear_impl.h:366-406: the solve at the given times (trajectory_.scaleSegmentTimesToMeetConstraints acts on
  // the solved trajectory), the stretch in place on coeffs, then solveLinear() at the stretched times
  MTG_TRY(launch_solve(h, p, topo, B, seg_times, d_fixed, nullptr, coeffs, nullptr, st_solve, s, false, nullptr, slot));
  const int64_t blocks = capped_grid(h, B, 128, 16);
  if (pass)  // rows with a non-zero pass[] are not stretched (the scaling passes failed solves through)
    MTG_TRY(launch_kernel(h, mtg::or_status_kernel, blocks, 128, 0, s, B, pass, st_solve));
  MTG_TRY(launch_scale_to_constraints(h, p->N, p->K, p->D, B, seg_times, coeffs, v_max, a_max, seg_times_out, coeffs,
                                      st_solve, within_range, maxima, st_scale, s));
  MTG_TRY(launch_solve(h, p, topo, B, seg_times_out, d_fixed, nullptr, coeffs, nullptr, st_resolve, s, false, nullptr,
                       slot));
  if (status) {
    MTG_CUDA(h, cudaMemcpyAsync(status, st_scale, sizeof(int32_t) * size_t(B), cudaMemcpyDeviceToDevice, s));
    MTG_TRY(launch_kernel(h, mtg::or_status_kernel, blocks, 128, 0, s, B, st_resolve, status));
  }
  return arena_release(h, ar, s);
}

int mtg_scale_times_with_violation_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                             const double* d_fixed, double v_max, double a_max, double* coeffs,
                                             double* seg_times_out, int32_t* within_range, double* maxima,
                                             int32_t* status, void* stream) {
  return run_problem_entry(
      h, valid_violation(p, B, v_max, a_max, seg_times, d_fixed, coeffs, seg_times_out), p, B, [&](CachedTopology* topo) {
        return launch_scale_with_violation(h, p, topo, B, seg_times, d_fixed, v_max, a_max, coeffs, seg_times_out,
                                           within_range, maxima, status, (cudaStream_t)stream, mtg_handle::kPipe);
      });
}

// ---- the Mellinger outer loop (PolynomialOptimizationNonLinear::optimize with kMellingerOuterLoop) -----------------
static bool valid_mellinger_params(const mtg_mellinger_params* q) {
  if (!q) return false;
  const bool any_tol = q->f_rel >= 0.0 || q->f_abs >= 0.0 || q->x_rel >= 0.0 || q->x_abs >= 0.0;
  return any_tol || q->max_iterations >= 0;  // otherwise nothing would stop a row
}

static bool valid_optimize(const mtg_problem* p, int64_t B, const mtg_mellinger_params* q, double v_max, double a_max,
                           const double* seg_times, const double* d_fixed, const double* coeffs,
                           const double* seg_times_out) {
  return valid_violation(p, B, v_max, a_max, seg_times, d_fixed, coeffs, seg_times_out) && valid_mellinger_params(q);
}

// The candidate costs Jc [rows][kLineSearchSteps] and solve statuses st_c of the compact rows in `lp`: one cost-only
// launch where the fused kernel exists, else expand + solve + cost in chunks (as launch_mellinger's unfused path).
static int launch_line_search(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, const mtg::MelLoopParams& lp,
                              double* Jc, int32_t* st_c, cudaStream_t s, int slot) {
  constexpr int kL = mtg::kLineSearchSteps;
  const int64_t rows = lp.rows;
  if (h->mellinger_unfused == 0) {  // MTG_OPT_MELLINGER_UNFUSED selects the unfused path here as for the gradient
    const int rc =
        launch_cost_fused(h, p, topo, rows * kL, lp.x, lp.dfix, Jc, 0, 0.0, lp.lower, s, st_c, lp.g, lp.alpha);
    if (rc != MTG_ERR_ALLOC) return rc;
  }
  const size_t K = p->K, D = p->D, N = p->N, dnf = lp.dnf;
  const size_t per_x = (K + dnf + K * D * N) * 8;  // times + d_fixed + coeffs of one candidate
  int64_t chunk = std::max<int64_t>(1, int64_t((size_t(384) << 20) / (per_x * kL)));
  chunk = std::min<int64_t>(chunk, rows);
  const size_t nx_max = size_t(chunk) * kL;
  const size_t o_f = align_doubles(nx_max * K), o_c = o_f + align_doubles(nx_max * dnf),
               need = (o_c + align_doubles(nx_max * K * D * N)) * 8;
  mtg_handle::Arena& ar = h->pack[slot];
  MTG_TRY(arena_acquire(h, ar, need, s));
  for (int64_t r0 = 0; r0 < rows; r0 += chunk) {
    const int64_t nr = std::min<int64_t>(chunk, rows - r0), nx = nr * kL;
    mtg::MelLoopParams cp = lp;
    cp.rows = int(nr);
    cp.x = lp.x + r0 * K;
    cp.g = lp.g + r0 * K;
    cp.alpha = lp.alpha + r0;
    cp.dfix = lp.dfix + r0 * dnf;
    MTG_TRY(launch_kernel(h, mtg::line_search_expand_kernel, capped_grid(h, nx, 128, 16), 128, 0, s, cp, ar.p,
                          ar.p + o_f));
    MTG_TRY(launch_solve(h, p, topo, nx, ar.p, ar.p + o_f, nullptr, ar.p + o_c, nullptr, st_c + r0 * kL, s, false,
                         nullptr, slot));
    MTG_TRY(launch_cost(h, p, nx, ar.p, ar.p + o_c, Jc + r0 * kL, s));
  }
  return arena_release(h, ar, s);
}

// The number of compact rows the last kernel on `s` listed: one copy into pinned memory and one event wait.
static int read_count(mtg_handle* h, const int32_t* d_count, cudaStream_t s, int* out) {
  if (!h->pinned_count) MTG_CUDA(h, cudaHostAlloc((void**)&h->pinned_count, sizeof(int), cudaHostAllocDefault));
  if (!h->count_ev) MTG_CUDA(h, cudaEventCreateWithFlags(&h->count_ev, cudaEventDisableTiming));
  MTG_CUDA(h, cudaMemcpyAsync(h->pinned_count, d_count, sizeof(int), cudaMemcpyDeviceToHost, s));
  MTG_CUDA(h, cudaEventRecord(h->count_ev, s));
  MTG_CUDA(h, cudaEventSynchronize(h->count_ev));
  *out = *h->pinned_count;
  return MTG_OK;
}

static int launch_optimize_mellinger(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B,
                                     const double* seg_times, const double* d_fixed, const mtg_mellinger_params* q,
                                     double v_max, double a_max, double* coeffs, double* seg_times_out,
                                     double* relative_times, double* cost, int32_t* iterations, int32_t* result,
                                     int32_t* within_range, double* maxima, int32_t* status, cudaStream_t s, int slot) {
  constexpr int kL = mtg::kLineSearchSteps;
  const size_t K = p->K, dnf = size_t(p->D) * topo->layout.n_fixed, nB = size_t(B);
  const size_t ni = align_doubles((nB + 1) / 2);  // one int32 per row, in doubles
  // arena: [2][B][K] x, [2][B] alpha, [2][B][dnf] d_fixed, [B][K] g, [B] J, [B][kL] Jc | int32: [2][B] idx, [B][K+1]
  // st_g, [B][kL] st_c, [B] iters, result, pass, opt_status, scale status, and the count
  size_t off = 0;
  auto take = [&](size_t doubles) {
    const size_t o = off;
    off += align_doubles(doubles);
    return o;
  };
  const size_t o_x[2] = {take(nB * K), take(nB * K)}, o_a[2] = {take(nB), take(nB)},
               o_f[2] = {take(nB * dnf), take(nB * dnf)}, o_g = take(nB * K), o_J = take(nB), o_Jc = take(nB * kL),
               o_idx[2] = {take((nB + 1) / 2), take((nB + 1) / 2)}, o_stg = take((nB * (K + 1) + 1) / 2),
               o_stc = take((nB * kL + 1) / 2), o_it = take(ni), o_res = take(ni), o_pass = take(ni),
               o_ost = take(ni), o_sst = take(ni), o_cnt = take(1);
  mtg_handle::Arena& ar = h->optim[slot];
  MTG_TRY(arena_acquire(h, ar, off * 8, s));
  double* base = ar.p;
  auto ip = [&](size_t o) { return reinterpret_cast<int32_t*>(base + o); };
  int32_t* d_count = ip(o_cnt);

  mtg::MelLoopParams lp{};
  lp.K = p->K;
  lp.dnf = int(dnf);
  lp.B = B;
  lp.max_iterations = q->max_iterations;
  lp.f_abs = q->f_abs;
  lp.f_rel = q->f_rel;
  lp.x_rel = q->x_rel;
  lp.x_abs = q->x_abs;
  lp.init_rel = q->initial_stepsize_rel;
  lp.lower = 0.1;  // kOptimizationTimeLowerBound (polynomial_optimization_nonlinear.h)
  lp.rel = seg_times_out;
  lp.iters = ip(o_it);
  lp.result = ip(o_res);
  lp.pass = ip(o_pass);
  lp.opt_status = ip(o_ost);
  lp.J = base + o_J;
  lp.g = base + o_g;
  lp.Jc = base + o_Jc;
  lp.st_g = ip(o_stg);
  lp.st_c = ip(o_stc);
  lp.count_next = d_count;
  const int threads = 128;
  int cur = 0;
  auto set_lists = [&](int c) {
    lp.idx = ip(o_idx[c]);
    lp.x = base + o_x[c];
    lp.alpha = base + o_a[c];
    lp.dfix = base + o_f[c];
    lp.idx_next = ip(o_idx[c ^ 1]);
    lp.x_next = base + o_x[c ^ 1];
    lp.alpha_next = base + o_a[c ^ 1];
    lp.dfix_next = base + o_f[c ^ 1];
  };
  // the start lists the iterating rows into list 0
  set_lists(1);
  MTG_CUDA(h, cudaMemsetAsync(d_count, 0, sizeof(int32_t), s));
  MTG_TRY(launch_kernel(h, mtg::mel_init_kernel, (B + threads - 1) / threads, threads, 0, s, lp, seg_times, d_fixed));
  int rows = 0;
  MTG_TRY(read_count(h, d_count, s, &rows));
  for (int k = 0; rows > 0; ++k) {
    set_lists(cur);
    lp.rows = rows;
    lp.k = k;
    const int blocks = (rows + threads - 1) / threads;
    MTG_CUDA(h, cudaMemsetAsync(ip(o_stg), 0, sizeof(int32_t) * size_t(rows) * (K + 1), s));
    MTG_CUDA(h, cudaMemsetAsync(ip(o_stc), 0, sizeof(int32_t) * size_t(rows) * kL, s));
    MTG_TRY(launch_mellinger(h, p, topo, rows, lp.x, lp.dfix, base + o_J, base + o_g, s, slot, ip(o_stg)));
    if (k == 0) MTG_TRY(launch_kernel(h, mtg::mel_alpha0_kernel, blocks, threads, 0, s, lp, base + o_a[cur]));
    // K = 1: every gradient is zero (getCostAndGradientMellinger), so every row stops with SUCCESS: no candidates
    if (p->K > 1) MTG_TRY(launch_line_search(h, p, topo, lp, base + o_Jc, ip(o_stc), s, slot));
    MTG_CUDA(h, cudaMemsetAsync(d_count, 0, sizeof(int32_t), s));
    MTG_TRY(launch_kernel(h, mtg::mel_update_kernel, blocks, threads, 0, s, lp));
    MTG_TRY(read_count(h, d_count, s, &rows));
    cur ^= 1;
  }
  if (relative_times)
    MTG_CUDA(h, cudaMemcpyAsync(relative_times, seg_times_out, sizeof(double) * nB * K, cudaMemcpyDeviceToDevice, s));
  MTG_TRY(launch_scale_with_violation(h, p, topo, B, seg_times_out, d_fixed, v_max, a_max, coeffs, seg_times_out,
                                      within_range, maxima, ip(o_sst), s, slot, ip(o_pass)));
  if (cost) MTG_TRY(launch_cost(h, p, B, seg_times_out, coeffs, cost, s));
  MTG_TRY(launch_kernel(h, mtg::mel_finish_kernel, capped_grid(h, B, threads, 16), threads, 0, s, B, ip(o_it),
                        ip(o_res), ip(o_ost), ip(o_sst), iterations, result, status));
  return arena_release(h, ar, s);
}

int mtg_optimize_time_mellinger_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                          const double* d_fixed, const mtg_mellinger_params* params, double v_max,
                                          double a_max, double* coeffs, double* seg_times_out, double* relative_times,
                                          double* cost, int32_t* iterations, int32_t* result, int32_t* within_range,
                                          double* maxima, int32_t* status, void* stream) {
  return run_problem_entry(
      h, valid_optimize(p, B, params, v_max, a_max, seg_times, d_fixed, coeffs, seg_times_out), p, B,
      [&](CachedTopology* topo) {
        return launch_optimize_mellinger(h, p, topo, B, seg_times, d_fixed, params, v_max, a_max, coeffs,
                                         seg_times_out, relative_times, cost, iterations, result, within_range, maxima,
                                         status, (cudaStream_t)stream, mtg_handle::kPipe);
      });
}

// ---- the compass search on the segment times (optimize() with kSquaredTime / kRichterTime) -------------------------
// Device memory for one poll's candidates (times, d_fixed, coefficients, objective, status): larger batches are
// evaluated in chunks of at most this many bytes (DESIGN.md section 3f).
constexpr size_t kTimeSearchBudget = size_t(512) << 20;

static bool valid_optimize_time(const mtg_problem* p, int64_t B, const mtg_time_objective* obj,
                                const mtg_mellinger_params* q, const double* seg_times, const double* d_fixed,
                                const double* coeffs, const double* seg_times_out) {
  return valid_objective(p, B, obj, seg_times, d_fixed, coeffs, seg_times_out) && valid_mellinger_params(q);
}

static int launch_optimize_time(mtg_handle* h, const mtg_problem* p, CachedTopology* topo, int64_t B,
                                const double* seg_times, const double* d_fixed, const mtg_time_objective* obj,
                                const mtg_mellinger_params* q, double* coeffs, double* seg_times_out,
                                double* objective, double* terms, int32_t* evaluations, int32_t* result,
                                int32_t* status, cudaStream_t s, int slot) {
  const size_t K = p->K, D = p->D, N = p->N, C = 2 * K, dnf = D * topo->layout.n_fixed, nB = size_t(B);
  // candidates per chunk: a multiple of 16 (8 rows), so that the expanded batch keeps the TMA-input route
  const size_t per_x = (K + dnf + K * D * N + 1) * 8 + 4;
  size_t chunk = std::max<size_t>(8, kTimeSearchBudget / (per_x * C) / 8 * 8);
  chunk = std::min(chunk, nB);
  const size_t nx = chunk * C, ni = (nB + 1) / 2;
  // arena (optim; launch_time_objective takes pack): [B] f0, [2] lists of ([B] idx, [B][K] x, [B][K] delta, [B] f,
  // [B][dnf] d_fixed), [B] evals, result, opt_status, st0, st_final, the count, then one chunk's candidates
  size_t off = 0;
  auto take = [&](size_t doubles) {
    const size_t o = off;
    off += align_doubles(doubles);
    return o;
  };
  const size_t o_f0 = take(nB), o_idx[2] = {take(ni), take(ni)}, o_x[2] = {take(nB * K), take(nB * K)},
               o_d[2] = {take(nB * K), take(nB * K)}, o_f[2] = {take(nB), take(nB)},
               o_df[2] = {take(nB * dnf), take(nB * dnf)}, o_ev = take(ni), o_res = take(ni), o_ost = take(ni),
               o_st0 = take(ni), o_stf = take(ni), o_cnt = take(1), o_tx = take(nx * K), o_fx = take(nx * dnf),
               o_cx = take(nx * K * D * N), o_fc = take(nx), o_stc = take((nx + 1) / 2);
  mtg_handle::Arena& ar = h->optim[slot];
  MTG_TRY(arena_acquire(h, ar, off * 8, s));
  double* base = ar.p;
  auto ip = [&](size_t o) { return reinterpret_cast<int32_t*>(base + o); };
  int32_t* d_count = ip(o_cnt);

  mtg::TimeSearchParams tp{};
  tp.K = p->K;
  tp.dnf = int(dnf);
  tp.B = B;
  tp.max_iterations = q->max_iterations;
  tp.f_abs = q->f_abs;
  tp.f_rel = q->f_rel;
  tp.x_rel = q->x_rel;
  tp.x_abs = q->x_abs;
  tp.init_rel = q->initial_stepsize_rel;
  tp.lower = 0.1;  // kOptimizationTimeLowerBound (polynomial_optimization_nonlinear.h)
  tp.x_out = seg_times_out;
  tp.evals_out = ip(o_ev);
  tp.result = ip(o_res);
  tp.opt_status = ip(o_ost);
  tp.count_next = d_count;
  const int threads = 128;
  auto set_lists = [&](int c) {
    tp.idx = ip(o_idx[c]);
    tp.x = base + o_x[c];
    tp.delta = base + o_d[c];
    tp.f = base + o_f[c];
    tp.dfix = base + o_df[c];
    tp.idx_next = ip(o_idx[c ^ 1]);
    tp.x_next = base + o_x[c ^ 1];
    tp.delta_next = base + o_d[c ^ 1];
    tp.f_next = base + o_f[c ^ 1];
    tp.dfix_next = base + o_df[c ^ 1];
  };
  // f(x0) for every row (coeffs is scratch until the final evaluation), then the start lists the iterating rows
  // into list 0
  MTG_TRY(launch_time_objective(h, p, topo, B, seg_times, d_fixed, nullptr, obj, coeffs, base + o_f0, nullptr,
                                ip(o_st0), s, slot));
  set_lists(1);
  MTG_CUDA(h, cudaMemsetAsync(d_count, 0, sizeof(int32_t), s));
  MTG_TRY(launch_kernel(h, mtg::ts_init_kernel, (B + threads - 1) / threads, threads, 0, s, tp, seg_times,
                        base + o_f0, ip(o_st0), d_fixed));
  int rows = 0;
  MTG_TRY(read_count(h, d_count, s, &rows));
  int cur = 0;
  for (int polls = 1; rows > 0; ++polls) {
    set_lists(cur);
    tp.evals = 1 + int(C) * polls;
    MTG_CUDA(h, cudaMemsetAsync(d_count, 0, sizeof(int32_t), s));
    for (int64_t r0 = 0; r0 < rows; r0 += int64_t(chunk)) {
      const int64_t nr = std::min<int64_t>(int64_t(chunk), rows - r0), ncx = nr * int64_t(C);
      mtg::TimeSearchParams cp = tp;
      cp.rows = int(nr);
      cp.idx = tp.idx + r0;
      cp.x = tp.x + r0 * K;
      cp.delta = tp.delta + r0 * K;
      cp.f = tp.f + r0;
      cp.dfix = tp.dfix + r0 * dnf;
      cp.fc = base + o_fc;
      cp.st_c = ip(o_stc);
      MTG_TRY(launch_kernel(h, mtg::ts_expand_kernel, capped_grid(h, ncx, threads, 16), threads, 0, s, cp,
                            base + o_tx, base + o_fx));
      MTG_TRY(launch_time_objective(h, p, topo, ncx, base + o_tx, base + o_fx, nullptr, obj, base + o_cx, base + o_fc,
                                    nullptr, ip(o_stc), s, slot));
      MTG_TRY(launch_kernel(h, mtg::ts_decide_kernel, (nr + threads - 1) / threads, threads, 0, s, cp));
    }
    MTG_TRY(read_count(h, d_count, s, &rows));
    cur ^= 1;
  }
  // the returned point's solve, objective and terms
  MTG_TRY(launch_time_objective(h, p, topo, B, seg_times_out, d_fixed, nullptr, obj, coeffs,
                                objective ? objective : base + o_f0, terms, ip(o_stf), s, slot));
  MTG_TRY(launch_kernel(h, mtg::ts_finish_kernel, capped_grid(h, B, threads, 16), threads, 0, s, B, ip(o_ev),
                        ip(o_res), ip(o_ost), ip(o_stf), evaluations, result, status));
  return arena_release(h, ar, s);
}

int mtg_optimize_time_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                const double* d_fixed, const mtg_time_objective* obj,
                                const mtg_mellinger_params* params, double* coeffs, double* seg_times_out,
                                double* objective, double* terms, int32_t* evaluations, int32_t* result,
                                int32_t* status, void* stream) {
  return run_problem_entry(
      h, valid_optimize_time(p, B, obj, params, seg_times, d_fixed, coeffs, seg_times_out), p, B,
      [&](CachedTopology* topo) {
        return launch_optimize_time(h, p, topo, B, seg_times, d_fixed, obj, params, coeffs, seg_times_out, objective,
                                    terms, evaluations, result, status, (cudaStream_t)stream, mtg_handle::kPipe);
      });
}

// Every input-feasibility entry: N even in [4, 12]; the limits are final values (the host mirror's InputConstraints
// applies addConstraint's corrections), each present one not NaN and >= 0 (+inf never fails); gravity finite.  Any D:
// rows with D not 3 or 4 are Indeterminable, as in the reference.
static bool valid_input_limits(int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                               const double* coeffs, const mtg_input_constraints* ic, const int32_t* result) {
  if (N < 4 || N > MTG_MAX_N || (N & 1) || K < 1 || D < 1 || !ic) return false;
  if (ic->present & ~uint32_t(MTG_INPUT_ALL)) return false;
  const double limits[6] = {ic->f_min, ic->f_max, ic->v_max, ic->omega_xy_max, ic->omega_z_max, ic->omega_z_dot_max};
  for (int q = 0; q < 6; ++q)
    if ((ic->present >> q & 1u) && !(limits[q] >= 0.0)) return false;
  if (!std::isfinite(ic->gravity)) return false;
  return valid_rows(B, {seg_times, coeffs, result});
}

// FeasibilityAnalytic and FeasibilityRecursive: also min_section_time > 0 and finite
static bool valid_feasibility(int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                              const double* coeffs, const mtg_input_constraints* ic, const int32_t* result) {
  return valid_input_limits(N, K, D, B, seg_times, coeffs, ic, result) && ic->min_section_time > 0.0 &&
         std::isfinite(ic->min_section_time);
}

// FeasibilitySampling: also sampling_interval > 0 and finite; min_section_time is not read
static bool valid_sampling(int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times, const double* coeffs,
                           const mtg_input_constraints* ic, double sampling_interval, const int32_t* result) {
  return valid_input_limits(N, K, D, B, seg_times, coeffs, ic, result) && sampling_interval > 0.0 &&
         std::isfinite(sampling_interval);
}

enum class FeasKind { Analytic, Recursive, Sampling };

// Analytic: input_feasibility_kernel; Recursive: input_feasibility_recursive_kernel; Sampling:
// input_feasibility_sampling_kernel (a warp per segment) at sampling_interval.  `entry` names the public entry point
// in the error of a K too large.
static int launch_input_feasibility(mtg_handle* h, const char* entry, int32_t N, int32_t K, int32_t D, int64_t B,
                                    const double* seg_times, const double* coeffs, const mtg_input_constraints* ic,
                                    int32_t* result, int32_t* segment, int32_t* status, cudaStream_t s,
                                    FeasKind kind = FeasKind::Analytic, double sampling_interval = 0.0) {
  mtg::FeasParams fp;
  fp.K = K;
  fp.D = D;
  fp.present = ic->present;
  fp.f_min = ic->f_min;
  fp.f_max = ic->f_max;
  fp.v_max = ic->v_max;
  fp.omega_xy = ic->omega_xy_max;
  fp.omega_z = ic->omega_z_max;
  fp.omega_z_dot = ic->omega_z_dot_max;
  fp.gravity = ic->gravity;
  fp.min_section_time = ic->min_section_time;
  fp.sampling_interval = sampling_interval;
  fp.B = B;
  fp.times = seg_times;
  fp.coeffs = coeffs;
  fp.result = result;
  fp.segment = segment;
  fp.status = status;
  const auto fn = kernel_by_n<4, MTG_MAX_N, 2, 0, 2>(
      [](auto k) {
        constexpr int n = decltype(k)::N;
        if constexpr (decltype(k)::A == int(FeasKind::Recursive)) return mtg::input_feasibility_recursive_kernel<n>;
        else if constexpr (decltype(k)::A == int(FeasKind::Sampling)) return mtg::input_feasibility_sampling_kernel<n>;
        else return mtg::input_feasibility_kernel<n>;
      },
      N, int(kind));
  return launch_segment_parallel(h, fn, fp, K, B, size_t(K) * sizeof(int), entry, "K", s);
}

int mtg_input_feasibility_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                    const double* coeffs, const mtg_input_constraints* constraints, int32_t* result,
                                    int32_t* segment, int32_t* status, void* stream) {
  return run_entry(h, valid_feasibility(N, K, D, B, seg_times, coeffs, constraints, result), B, [&] {
    return launch_input_feasibility(h, "mtg_input_feasibility_batch_f64", N, K, D, B, seg_times, coeffs, constraints,
                                    result, segment, status, (cudaStream_t)stream);
  });
}

// FeasibilityRecursive: the same arguments, refused by the same check
int mtg_input_feasibility_recursive_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                              const double* seg_times, const double* coeffs,
                                              const mtg_input_constraints* constraints, int32_t* result,
                                              int32_t* segment, int32_t* status, void* stream) {
  return run_entry(h, valid_feasibility(N, K, D, B, seg_times, coeffs, constraints, result), B, [&] {
    return launch_input_feasibility(h, "mtg_input_feasibility_recursive_batch_f64", N, K, D, B, seg_times, coeffs,
                                    constraints, result, segment, status, (cudaStream_t)stream, FeasKind::Recursive);
  });
}

// FeasibilitySampling: the analytic entry's arguments, sampling_interval instead of min_section_time
int mtg_input_feasibility_sampling_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                             const double* seg_times, const double* coeffs,
                                             const mtg_input_constraints* constraints, double sampling_interval,
                                             int32_t* result, int32_t* segment, int32_t* status, void* stream) {
  return run_entry(h, valid_sampling(N, K, D, B, seg_times, coeffs, constraints, sampling_interval, result), B, [&] {
    return launch_input_feasibility(h, "mtg_input_feasibility_sampling_batch_f64", N, K, D, B, seg_times, coeffs,
                                    constraints, result, segment, status, (cudaStream_t)stream, FeasKind::Sampling,
                                    sampling_interval);
  });
}

// checkHalfPlaneFeasibility: N even in [2, 12]; 0 <= n_planes <= MTG_MAX_HALF_PLANES, the planes (a host array)
// finite with a non-zero normal.  Any D: rows with D not 3 or 4 are infeasible, as in the reference.
static bool valid_half_plane(int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                             const double* coeffs, int32_t n_planes, const mtg_half_plane* planes,
                             const int32_t* feasible) {
  if (N < 2 || N > MTG_MAX_N || (N & 1) || K < 1 || D < 1) return false;
  if (n_planes < 0 || n_planes > MTG_MAX_HALF_PLANES || (n_planes > 0 && !planes)) return false;
  for (int p = 0; p < n_planes; ++p) {
    bool zero = true;
    for (int d = 0; d < 3; ++d) {
      if (!std::isfinite(planes[p].point[d]) || !std::isfinite(planes[p].normal[d])) return false;
      if (planes[p].normal[d] != 0.0) zero = false;
    }
    if (zero) return false;
  }
  return valid_rows(B, {seg_times, coeffs, feasible});
}

static int launch_half_plane(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                             const double* coeffs, int32_t n_planes, const mtg_half_plane* planes, int32_t* feasible,
                             int32_t* segment, int32_t* plane, int32_t* status, cudaStream_t s) {
  static_assert(mtg::kHalfPlaneMax == MTG_MAX_HALF_PLANES, "plane table size");
  mtg::HalfPlaneParams hp;  // the planes travel by value in the kernel parameters
  hp.K = K;
  hp.D = D;
  hp.n_planes = n_planes;
  hp.B = B;
  hp.times = seg_times;
  hp.coeffs = coeffs;
  hp.feasible = feasible;
  hp.segment = segment;
  hp.plane = plane;
  hp.status = status;
  for (int p = 0; p < mtg::kHalfPlaneMax; ++p)
    for (int d = 0; d < 3; ++d) {
      hp.planes[p][d] = p < n_planes ? planes[p].point[d] : 0.0;
      hp.planes[p][3 + d] = p < n_planes ? planes[p].normal[d] : 0.0;
    }
  const auto fn = kernel_by_n<2, MTG_MAX_N, 2>([](auto k) { return mtg::half_plane_kernel<decltype(k)::N>; }, N);
  return launch_segment_parallel(h, fn, hp, K, B, size_t(K) * sizeof(int), "mtg_half_plane_feasibility_batch_f64", "K",
                                 s);
}

int mtg_half_plane_feasibility_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                         const double* seg_times, const double* coeffs, int32_t n_planes,
                                         const mtg_half_plane* planes, int32_t* feasible, int32_t* segment,
                                         int32_t* plane, int32_t* status, void* stream) {
  return run_entry(h, valid_half_plane(N, K, D, B, seg_times, coeffs, n_planes, planes, feasible), B, [&] {
    return launch_half_plane(h, N, K, D, B, seg_times, coeffs, n_planes, planes, feasible, segment, plane, status,
                             (cudaStream_t)stream);
  });
}

// ---- host-pointer entry points: the device entry's check and launcher, around stage_host() ------------------------

static int solve_host(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times, const double* d_fixed,
                      const double* d_free_in, double* coeffs, double* d_free, int32_t* status, bool backsub_only) {
  return run_problem_entry(h, valid_problem_args(p, B, seg_times, d_fixed, coeffs), p, B, [&](CachedTopology* topo) {
    const Layout& L = topo->layout;
    if (backsub_only) MTG_TRY(check_d_free(h, L, d_free_in));
    const size_t K = p->K, D = p->D, N = p->N;
    const HostBuf bufs[] = {{seg_times, nullptr, K * 8},           {d_fixed, nullptr, D * L.n_fixed * 8},
                            {d_free_in, nullptr, D * L.n_free * 8}, {nullptr, coeffs, K * D * N * 8},
                            {nullptr, d_free, D * L.n_free * 8},    {nullptr, status, 4}};
    return stage_host(h, B, Staging::Pipelined, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
      return launch_solve(h, p, topo, nb, d[0], d[1], d[2], d[3], d[4], d[5], s, backsub_only, nullptr, slot);
    });
  });
}

int mtg_solve_linear_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                    const double* d_fixed, double* coeffs, double* d_free, int32_t* status) {
  return solve_host(h, p, B, seg_times, d_fixed, nullptr, coeffs, d_free, status, false);
}

int mtg_solve_waypoints_nfabian_batch_host_f64(mtg_handle* h, int32_t N, int32_t r, int32_t K, int32_t D, int64_t B,
                                               const double* positions, double v_max, double a_max, double magic,
                                               double* coeffs, double* seg_times_out, int32_t* status) {
  const mtg_problem p = {N, r, K, D, nullptr};
  return run_problem_entry(h, valid_nfabian(&p, B, positions, v_max, a_max, coeffs), &p, B, [&](CachedTopology* topo) {
    const HostBuf bufs[] = {{positions, nullptr, size_t(K + 1) * D * 8},
                            {nullptr, coeffs, size_t(K) * D * N * 8},
                            {nullptr, seg_times_out, size_t(K) * 8},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::Pipelined, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
      return launch_nfabian(h, &p, topo, nb, d[0], v_max, a_max, magic, d[1], d[2], d[3], s, slot);
    });
  });
}

int mtg_coeffs_from_constraints_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                               const double* seg_times, const double* d_fixed,
                                               const double* d_free, double* coeffs) {
  return solve_host(h, p, B, seg_times, d_fixed, d_free, coeffs, nullptr, nullptr, true);
}

int mtg_compute_cost_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                    const double* coeffs, double* cost) {
  return run_entry(h, valid_problem_args(p, B, seg_times, coeffs, cost), B, [&] {
    const size_t K = p->K, D = p->D, N = p->N;
    const HostBuf bufs[] = {{seg_times, nullptr, K * 8}, {coeffs, nullptr, K * D * N * 8}, {nullptr, cost, 8}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_cost(h, p, nb, d[0], d[1], d[2], s);
    });
  });
}

int mtg_cost_gradient_mellinger_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                               const double* d_fixed, double* cost, double* grad) {
  return run_problem_entry(h, valid_problem_args(p, B, seg_times, d_fixed, grad), p, B, [&](CachedTopology* topo) {
    const size_t K = p->K, D = p->D;
    const HostBuf bufs[] = {{seg_times, nullptr, K * 8},
                            {d_fixed, nullptr, D * topo->layout.n_fixed * 8},
                            {nullptr, cost, 8},
                            {nullptr, grad, K * 8}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
      return launch_mellinger(h, p, topo, nb, d[0], d[1], d[2], d[3], s, slot);
    });
  });
}

int mtg_evaluate_range_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                      const double* coeffs, double t_start, double t_end, double dt, int32_t n_derivs,
                                      const int32_t* derivs, int32_t max_samples, double* out, int32_t* n_samples,
                                      double* sampling_times) {
  return run_entry(h, valid_range(N, K, D, B, dt, n_derivs, derivs, max_samples, seg_times, coeffs, out, n_samples), B,
                   [&] {
                     const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                                             {coeffs, nullptr, size_t(K) * D * N * 8},
                                             {nullptr, out, size_t(max_samples) * n_derivs * D * 8},
                                             {nullptr, n_samples, 4},
                                             {nullptr, sampling_times, size_t(max_samples) * 8}};
                     return stage_host(h, B, Staging::OneChunk, bufs,
                                       [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
                                         return launch_range(h, N, K, D, nb, d[0], d[1], t_start, t_end, dt, n_derivs,
                                                             derivs, max_samples, d[2], d[3], d[4], s, slot);
                                       });
                   });
}

int mtg_sample_flat_states_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                          const double* seg_times, const double* coeffs, double min_time,
                                          double max_time, double sampling_interval, int32_t whole, int32_t max_samples,
                                          double* states, int64_t* time_ns, int32_t* n_samples) {
  return run_entry(
      h, valid_flat_range(N, K, D, B, sampling_interval, max_samples, seg_times, coeffs, states, n_samples), B, [&] {
        const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                                {coeffs, nullptr, size_t(K) * D * N * 8},
                                {nullptr, states, size_t(max_samples) * MTG_FLAT_STATE_DOUBLES * 8},
                                {nullptr, time_ns, size_t(max_samples) * 8},
                                {nullptr, n_samples, 4}};
        return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
          return launch_flat_range(h, N, K, D, nb, d[0], d[1], min_time, max_time, sampling_interval, whole,
                                   max_samples, d[2], d[3], d[4], s, slot);
        });
      });
}

int mtg_sample_flat_state_at_time_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                 const double* seg_times, const double* coeffs,
                                                 const double* sample_times, double* states, int64_t* time_ns,
                                                 int32_t* ok) {
  return run_entry(h, valid_flat_at_time(N, K, D, B, seg_times, coeffs, sample_times, states, ok), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                            {coeffs, nullptr, size_t(K) * D * N * 8},
                            {sample_times, nullptr, 8},
                            {nullptr, states, size_t(MTG_FLAT_STATE_DOUBLES) * 8},
                            {nullptr, time_ns, 8},
                            {nullptr, ok, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_flat_at_time(h, N, K, D, nb, d[0], d[1], d[2], d[3], d[4], d[5], s);
    });
  });
}

int mtg_max_magnitude_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                     const double* coeffs, int32_t n_derivs, const int32_t* derivs, double* value,
                                     double* time, int32_t* segment, int32_t* status) {
  return run_entry(h, valid_extrema_args(N, K, D, B, n_derivs, derivs, seg_times, coeffs, value), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},       {coeffs, nullptr, size_t(K) * D * N * 8},
                            {nullptr, value, size_t(n_derivs) * 8},    {nullptr, time, size_t(n_derivs) * 8},
                            {nullptr, segment, size_t(n_derivs) * 4},  {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_max_magnitude(h, N, K, D, nb, d[0], d[1], n_derivs, derivs, d[2], d[3], d[4], d[5], s);
    });
  });
}

int mtg_time_objective_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                      const double* d_fixed, const double* d_free, const mtg_time_objective* obj,
                                      double* coeffs, double* objective, double* terms, int32_t* status) {
  return run_problem_entry(
      h, valid_objective(p, B, obj, seg_times, d_fixed, coeffs, objective), p, B, [&](CachedTopology* topo) {
        const Layout& L = topo->layout;
        const size_t K = p->K, D = p->D, N = p->N;
        const HostBuf bufs[] = {{seg_times, nullptr, K * 8},      {d_fixed, nullptr, D * L.n_fixed * 8},
                                {d_free, nullptr, D * L.n_free * 8}, {nullptr, coeffs, K * D * N * 8},
                                {nullptr, objective, 8},          {nullptr, terms, 24},
                                {nullptr, status, 4}};
        return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
          return launch_time_objective(h, p, topo, nb, d[0], d[1], d[2], obj, d[3], d[4], d[5], d[6], s, slot);
        });
      });
}

int mtg_scale_to_constraints_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                            const double* seg_times, const double* coeffs, double v_max, double a_max,
                                            double* seg_times_out, double* coeffs_out, int32_t* within_range,
                                            double* maxima, int32_t* status) {
  return run_entry(h, valid_scale(N, K, D, B, v_max, a_max, seg_times, coeffs, seg_times_out, coeffs_out), B, [&] {
    // the stretch runs in place on the device copies of the times and coefficients
    const HostBuf bufs[] = {{seg_times, seg_times_out, size_t(K) * 8},
                            {coeffs, coeffs_out, size_t(K) * D * N * 8},
                            {nullptr, within_range, 4},
                            {nullptr, maxima, 16},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_scale_to_constraints(h, N, K, D, nb, d[0], d[1], v_max, a_max, d[0], d[1], nullptr, d[2], d[3],
                                         d[4], s);
    });
  });
}

int mtg_scale_times_with_violation_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                                  const double* seg_times, const double* d_fixed, double v_max,
                                                  double a_max, double* coeffs, double* seg_times_out,
                                                  int32_t* within_range, double* maxima, int32_t* status) {
  return run_problem_entry(
      h, valid_violation(p, B, v_max, a_max, seg_times, d_fixed, coeffs, seg_times_out), p, B, [&](CachedTopology* topo) {
        const size_t K = p->K, D = p->D, N = p->N;
        // the times go in from seg_times and come back, stretched in place, into seg_times_out
        const HostBuf bufs[] = {{seg_times, seg_times_out, K * 8},
                                {d_fixed, nullptr, D * topo->layout.n_fixed * 8},
                                {nullptr, coeffs, K * D * N * 8},
                                {nullptr, within_range, 4},
                                {nullptr, maxima, 16},
                                {nullptr, status, 4}};
        return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
          return launch_scale_with_violation(h, p, topo, nb, d[0], d[1], v_max, a_max, d[2], d[0], d[3], d[4], d[5], s,
                                             slot);
        });
      });
}

int mtg_optimize_time_mellinger_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                               const double* d_fixed, const mtg_mellinger_params* params, double v_max,
                                               double a_max, double* coeffs, double* seg_times_out,
                                               double* relative_times, double* cost, int32_t* iterations,
                                               int32_t* result, int32_t* within_range, double* maxima,
                                               int32_t* status) {
  return run_problem_entry(
      h, valid_optimize(p, B, params, v_max, a_max, seg_times, d_fixed, coeffs, seg_times_out), p, B,
      [&](CachedTopology* topo) {
        const size_t K = p->K, D = p->D, N = p->N;
        // the times go in from seg_times and come back, optimised and stretched in place, into seg_times_out
        const HostBuf bufs[] = {{seg_times, seg_times_out, K * 8},
                                {d_fixed, nullptr, D * topo->layout.n_fixed * 8},
                                {nullptr, coeffs, K * D * N * 8},
                                {nullptr, relative_times, K * 8},
                                {nullptr, cost, 8},
                                {nullptr, iterations, 4},
                                {nullptr, result, 4},
                                {nullptr, within_range, 4},
                                {nullptr, maxima, 16},
                                {nullptr, status, 4}};
        return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
          return launch_optimize_mellinger(h, p, topo, nb, d[0], d[1], params, v_max, a_max, d[2], d[0], d[3], d[4],
                                           d[5], d[6], d[7], d[8], d[9], s, slot);
        });
      });
}

int mtg_optimize_time_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                     const double* d_fixed, const mtg_time_objective* obj,
                                     const mtg_mellinger_params* params, double* coeffs, double* seg_times_out,
                                     double* objective, double* terms, int32_t* evaluations, int32_t* result,
                                     int32_t* status) {
  return run_problem_entry(
      h, valid_optimize_time(p, B, obj, params, seg_times, d_fixed, coeffs, seg_times_out), p, B,
      [&](CachedTopology* topo) {
        const size_t K = p->K, D = p->D, N = p->N;
        // the times go in from seg_times and come back, optimised in place, into seg_times_out
        const HostBuf bufs[] = {{seg_times, seg_times_out, K * 8},
                                {d_fixed, nullptr, D * topo->layout.n_fixed * 8},
                                {nullptr, coeffs, K * D * N * 8},
                                {nullptr, objective, 8},
                                {nullptr, terms, 24},
                                {nullptr, evaluations, 4},
                                {nullptr, result, 4},
                                {nullptr, status, 4}};
        return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int slot) {
          return launch_optimize_time(h, p, topo, nb, d[0], d[1], obj, params, d[2], d[0], d[3], d[4], d[5], d[6], d[7],
                                      s, slot);
        });
      });
}

int mtg_input_feasibility_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                         const double* seg_times, const double* coeffs,
                                         const mtg_input_constraints* constraints, int32_t* result, int32_t* segment,
                                         int32_t* status) {
  return run_entry(h, valid_feasibility(N, K, D, B, seg_times, coeffs, constraints, result), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                            {coeffs, nullptr, size_t(K) * D * N * 8},
                            {nullptr, result, 4},
                            {nullptr, segment, 4},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_input_feasibility(h, "mtg_input_feasibility_batch_f64", N, K, D, nb, d[0], d[1], constraints, d[2],
                                      d[3], d[4], s);
    });
  });
}

int mtg_input_feasibility_recursive_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                   const double* seg_times, const double* coeffs,
                                                   const mtg_input_constraints* constraints, int32_t* result,
                                                   int32_t* segment, int32_t* status) {
  return run_entry(h, valid_feasibility(N, K, D, B, seg_times, coeffs, constraints, result), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                            {coeffs, nullptr, size_t(K) * D * N * 8},
                            {nullptr, result, 4},
                            {nullptr, segment, 4},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_input_feasibility(h, "mtg_input_feasibility_recursive_batch_f64", N, K, D, nb, d[0], d[1],
                                      constraints, d[2], d[3], d[4], s, FeasKind::Recursive);
    });
  });
}

int mtg_input_feasibility_sampling_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                  const double* seg_times, const double* coeffs,
                                                  const mtg_input_constraints* constraints, double sampling_interval,
                                                  int32_t* result, int32_t* segment, int32_t* status) {
  return run_entry(h, valid_sampling(N, K, D, B, seg_times, coeffs, constraints, sampling_interval, result), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                            {coeffs, nullptr, size_t(K) * D * N * 8},
                            {nullptr, result, 4},
                            {nullptr, segment, 4},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_input_feasibility(h, "mtg_input_feasibility_sampling_batch_f64", N, K, D, nb, d[0], d[1],
                                      constraints, d[2], d[3], d[4], s, FeasKind::Sampling, sampling_interval);
    });
  });
}

int mtg_half_plane_feasibility_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                              const double* seg_times, const double* coeffs, int32_t n_planes,
                                              const mtg_half_plane* planes, int32_t* feasible, int32_t* segment,
                                              int32_t* plane, int32_t* status) {
  return run_entry(h, valid_half_plane(N, K, D, B, seg_times, coeffs, n_planes, planes, feasible), B, [&] {
    const HostBuf bufs[] = {{seg_times, nullptr, size_t(K) * 8},
                            {coeffs, nullptr, size_t(K) * D * N * 8},
                            {nullptr, feasible, 4},
                            {nullptr, segment, 4},
                            {nullptr, plane, 4},
                            {nullptr, status, 4}};
    return stage_host(h, B, Staging::OneChunk, bufs, [&](const DevBuf* d, int64_t nb, cudaStream_t s, int) {
      return launch_half_plane(h, N, K, D, nb, d[0], d[1], n_planes, planes, d[2], d[3], d[4], d[5], s);
    });
  });
}

void* mtg_host_alloc(mtg_handle* h, uint64_t bytes) {
  void* p = nullptr;
  if (!h) return nullptr;
  DeviceGuard g(h->device);
  if (set_err(h, "cudaMallocHost", cudaMallocHost(&p, bytes ? bytes : 1))) return nullptr;
  return p;
}
void mtg_host_free(mtg_handle* h, void* ptr) {
  if (h && ptr) {
    DeviceGuard g(h->device);
    cudaFreeHost(ptr);
  }
}
void* mtg_device_alloc(mtg_handle* h, uint64_t bytes) {
  void* p = nullptr;
  if (!h) return nullptr;
  DeviceGuard g(h->device);
  if (set_err(h, "cudaMalloc", cudaMalloc(&p, bytes ? bytes : 1))) return nullptr;
  return p;
}
void mtg_device_free(mtg_handle* h, void* ptr) {
  if (h && ptr) {
    DeviceGuard g(h->device);
    cudaFree(ptr);
  }
}
int mtg_memcpy_h2d(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream) {
  if (!h) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  MTG_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return MTG_OK;
}
int mtg_memcpy_d2h(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream) {
  if (!h) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  MTG_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return MTG_OK;
}
int mtg_memcpy_d2d(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream) {
  if (!h) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  MTG_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return MTG_OK;
}

// ---- peer memory (NVLink): export / import a device allocation between the one-process-per-GPU ranks ----------
int mtg_ipc_export(mtg_handle* h, const void* ptr, uint8_t handle_out[64], uint64_t* offset_out) {
  if (!h || !ptr || !handle_out || !offset_out) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  typedef CUresult (*RangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
  static const RangeFn range = []() -> RangeFn {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<RangeFn>(fp);
  }();
  if (!range) {
    h->error = "cuMemGetAddressRange is not available from the driver";
    return MTG_ERR_CUDA;
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, reinterpret_cast<CUdeviceptr>(ptr)) != CUDA_SUCCESS) {
    h->error = "cuMemGetAddressRange failed";
    return MTG_ERR_CUDA;
  }
  cudaIpcMemHandle_t hd;
  MTG_CUDA(h, cudaIpcGetMemHandle(&hd, reinterpret_cast<void*>(base)));
  static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
  std::memcpy(handle_out, &hd, 64);
  *offset_out = uint64_t(reinterpret_cast<CUdeviceptr>(ptr) - base);
  return MTG_OK;
}

int mtg_ipc_import(mtg_handle* h, const uint8_t handle[64], uint64_t offset, void** ptr_out, void** base_out) {
  if (!h || !handle || !ptr_out || !base_out) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);  // opened with THIS handle's device current: peer access to the owner is enabled lazily
  cudaIpcMemHandle_t hd;
  std::memcpy(&hd, handle, 64);
  void* base = nullptr;
  MTG_CUDA(h, cudaIpcOpenMemHandle(&base, hd, cudaIpcMemLazyEnablePeerAccess));
  *base_out = base;
  *ptr_out = static_cast<char*>(base) + offset;
  return MTG_OK;
}

int mtg_ipc_close(mtg_handle* h, void* base) {
  if (!h || !base) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  MTG_CUDA(h, cudaIpcCloseMemHandle(base));
  return MTG_OK;
}

int mtg_stream_synchronize(mtg_handle* h, void* stream) {
  if (!h) return MTG_ERR_BAD_ARG;
  DeviceGuard g(h->device);
  MTG_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
  return MTG_OK;
}

}  // extern "C"
