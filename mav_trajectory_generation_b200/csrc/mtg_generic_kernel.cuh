// mtg_generic_kernel.cuh -- K4: arbitrary per-vertex constraint masks (any Vertex::Vector the
// reference accepts), runtime N / r / K / D; plus the back-substitution-only and cost kernels.
//
// One thread per trajectory, grid-stride.  The reduced system R_pp d_p = -R_pf d_f
// (impl/polynomial_optimization_linear_impl.h:360-375) is assembled directly in banded
// lower storage (free constraints sorted by (vertex, derivative) couple only inside one
// segment, so the half bandwidth is <= 2h-1), factorised by a banded Cholesky and solved for
// all D right-hand sides.  Scratch lives in global memory, interleaved by thread
// (element e of thread t at scratch[e * stride + t]) so warp accesses coalesce.
// The 0/1 reordering matrix C of the reference (linear_impl.h:181-260) is passed as one column
// index per row (slot_col), built once per topology on the host.
#pragma once

#include "mtg_device.cuh"

namespace mtg {

__device__ __forceinline__ const double* a1inv_table(int N) {
  switch (N) {
    case 2: return c_a1inv_2;
    case 4: return c_a1inv_4;
    case 6: return c_a1inv_6;
    case 8: return c_a1inv_8;
    case 10: return c_a1inv_10;
    default: return c_a1inv_12;
  }
}

__device__ __forceinline__ const double* h1_table(int N, int r) {
  switch (N * 8 + r) {
    case 2 * 8 + 0: return c_h1_2_0;
    case 4 * 8 + 0: return c_h1_4_0;
    case 4 * 8 + 1: return c_h1_4_1;
    case 6 * 8 + 0: return c_h1_6_0;
    case 6 * 8 + 1: return c_h1_6_1;
    case 6 * 8 + 2: return c_h1_6_2;
    case 8 * 8 + 0: return c_h1_8_0;
    case 8 * 8 + 1: return c_h1_8_1;
    case 8 * 8 + 2: return c_h1_8_2;
    case 8 * 8 + 3: return c_h1_8_3;
    case 10 * 8 + 0: return c_h1_10_0;
    case 10 * 8 + 1: return c_h1_10_1;
    case 10 * 8 + 2: return c_h1_10_2;
    case 10 * 8 + 3: return c_h1_10_3;
    case 10 * 8 + 4: return c_h1_10_4;
    case 12 * 8 + 0: return c_h1_12_0;
    case 12 * 8 + 1: return c_h1_12_1;
    case 12 * 8 + 2: return c_h1_12_2;
    case 12 * 8 + 3: return c_h1_12_3;
    case 12 * 8 + 4: return c_h1_12_4;
    default: return c_h1_12_5;
  }
}

struct GenericParams {
  int N, r, K, D;
  int n_fixed, n_free, bw;
  long long B;
  const int* __restrict__ slot_col;   // [K*N]
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ dfix;    // [B][D][n_fixed]
  const double* __restrict__ dfree_in;  // [B][D][n_free] (back-substitution-only kernel) or null
  double* __restrict__ coeffs;        // [B][K][D][N]
  double* __restrict__ dfree;         // [B][D][n_free] or null
  int* __restrict__ status;           // [B] or null
  double* __restrict__ scratch;       // per-thread interleaved scratch
  long long scratch_stride;           // number of threads of the launch
};

// p = diag(T^-j) A(1)^-1 diag(T^(s mod h)) (C_i d)   (linear_impl.h:270-280), all segments.
// value(col, d) supplies d_all[col].
template <typename ValueFn>
__device__ __forceinline__ void back_substitute(const GenericParams& prm, long long traj, ValueFn value) {
  const int N = prm.N, h = N / 2, K = prm.K, D = prm.D;
  const double* __restrict__ A1 = a1inv_table(N);
  double* __restrict__ out = prm.coeffs + traj * (long long)K * D * N;
  for (int i = 0; i < K; ++i) {
    const double T = prm.times[traj * K + i];
    const double iT = 1.0 / T;
    double tp[MTG_MAX_N_HALF];
    tp[0] = 1.0;
    for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * T;
    for (int d = 0; d < D; ++d) {
      double sv[2 * MTG_MAX_N_HALF];
      for (int s = 0; s < N; ++s) sv[s] = value(prm.slot_col[i * N + s], d);
      double ip = 1.0;  // T^-j
      for (int j = 0; j < N; ++j) {
        double acc;
        if (j < h) {
          acc = sv[j] * A1[j * N + j];  // d_j / j!  (A^-1 is diagonal here)
        } else {
          acc = 0.0;
          for (int s = 0; s < N; ++s) acc = fma(A1[j * N + s], tp[s < h ? s : s - h] * sv[s], acc);
          acc *= ip;
        }
        out[((long long)i * D + d) * N + j] = acc;
        ip *= iT;
      }
    }
  }
}

// n_free == 0 shortcut (linear_impl.h:343-349) and setFreeConstraints (:499-508).
__global__ void __launch_bounds__(128) backsub_kernel(const GenericParams prm) {
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long traj = (long long)blockIdx.x * blockDim.x + threadIdx.x; traj < prm.B; traj += nthreads) {
    const double* __restrict__ fx = prm.dfix + traj * (long long)prm.D * prm.n_fixed;
    const double* __restrict__ fr =
        prm.dfree_in ? prm.dfree_in + traj * (long long)prm.D * prm.n_free : nullptr;
    const int nf = prm.n_fixed, np = prm.n_free;
    int stat = 0;
    for (int i = 0; i < prm.K; ++i)
      if (bad_segment_time(prm.times[traj * prm.K + i])) stat |= kStatusBadTime;
    back_substitute(prm, traj, [&](int col, int d) -> double {
      return col < nf ? fx[d * nf + col] : fr[d * np + (col - nf)];
    });
    if (prm.status) prm.status[traj] = stat;
  }
}

__global__ void __launch_bounds__(128) generic_solve_kernel(const GenericParams prm) {
  const int N = prm.N, h = N / 2, K = prm.K, D = prm.D;
  const int nf = prm.n_fixed, np = prm.n_free, bw = prm.bw, bw1 = prm.bw + 1;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const double* __restrict__ G = h1_table(N, prm.r);
  double* __restrict__ scr = prm.scratch + tid;
  const long long ss = prm.scratch_stride;
  const long long rhs0 = (long long)np * bw1;
#define BAND(i, k) scr[((long long)(i)*bw1 + (k)) * ss]
#define RHS(i, d) scr[(rhs0 + (long long)(i)*D + (d)) * ss]

  for (long long traj = tid; traj < prm.B; traj += nthreads) {
    const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
    int stat = 0;
    for (long long e = 0; e < rhs0 + (long long)np * D; ++e) scr[e * ss] = 0.0;

    // ---- assemble R_pp (banded lower) and -R_pf d_f
    for (int i = 0; i < K; ++i) {
      const double T = prm.times[traj * K + i];
      if (bad_segment_time(T)) stat |= kStatusBadTime;
      const double iT = 1.0 / T;
      double sp[MTG_MAX_N_HALF];
      sp[0] = 1.0;
      for (int k = 1; k < h; ++k) sp[k] = sp[k - 1] * T;
      double rho = T;  // T^(1-2r)
      for (int k = 0; k < 2 * prm.r; ++k) rho *= iT;
      for (int a = 0; a < N; ++a) {
        const int ca = prm.slot_col[i * N + a] - nf;
        if (ca < 0) continue;
        const double fa = rho * sp[a < h ? a : a - h];
        for (int b = 0; b < N; ++b) {
          const int cb = prm.slot_col[i * N + b];
          const double Hab = fa * sp[b < h ? b : b - h] * G[a * N + b];
          if (cb >= nf) {
            const int j = cb - nf;
            if (j <= ca) BAND(ca, ca - j) += Hab;
          } else {
            for (int d = 0; d < D; ++d) RHS(ca, d) -= Hab * fx[d * nf + cb];
          }
        }
      }
    }

    // ---- banded Cholesky, BAND(i,0) keeps the inverse pivot
    for (int i = 0; i < np; ++i) {
      const int j0 = i - bw > 0 ? i - bw : 0;
      for (int j = j0; j <= i; ++j) {
        double s = BAND(i, i - j);
        for (int k = j0; k < j; ++k) {
          if (j - k <= bw) s = fma(-BAND(i, i - k), BAND(j, j - k), s);
        }
        if (j < i) {
          BAND(i, i - j) = s * BAND(j, 0);
        } else {
          if (!(s > 0.0) || isinf(s)) stat |= kStatusNotSpd;
          BAND(i, 0) = rsqrt(s);
        }
      }
    }
    // ---- forward / backward substitution for the D right-hand sides
    for (int d = 0; d < D; ++d) {
      for (int i = 0; i < np; ++i) {
        const int j0 = i - bw > 0 ? i - bw : 0;
        double s = RHS(i, d);
        for (int k = j0; k < i; ++k) s = fma(-BAND(i, i - k), RHS(k, d), s);
        RHS(i, d) = s * BAND(i, 0);
      }
      for (int i = np - 1; i >= 0; --i) {
        const int k1 = i + bw < np - 1 ? i + bw : np - 1;
        double s = RHS(i, d);
        for (int k = i + 1; k <= k1; ++k) s = fma(-BAND(k, k - i), RHS(k, d), s);
        RHS(i, d) = s * BAND(i, 0);
      }
    }
    if (prm.dfree) {
      double* __restrict__ df = prm.dfree + traj * (long long)D * np;
      for (int d = 0; d < D; ++d)
        for (int i = 0; i < np; ++i) df[d * np + i] = RHS(i, d);
    }
    back_substitute(prm, traj, [&](int col, int d) -> double {
      return col < nf ? fx[d * nf + col] : RHS(col - nf, d);
    });
    if (prm.status) prm.status[traj] = stat;
  }
#undef BAND
#undef RHS
}

// estimateSegmentTimesNfabian (reference src/vertex.cpp:255-272) + the waypoint-topology d_fixed packing
// (linear_impl.h:233-247) for configurations without a fused specialised kernel.
struct PackParams {
  int N, K, D, n_fixed;
  long long B;
  const double* __restrict__ positions;  // [B][K+1][D]
  double v_max, a_max, magic;
  double* __restrict__ times;            // [B][K]
  double* __restrict__ dfix;             // [B][D][n_fixed]
};

__global__ void __launch_bounds__(128) nfabian_pack_kernel(const PackParams prm) {
  const int K = prm.K, D = prm.D, h = prm.N / 2, nf = prm.n_fixed;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long traj = (long long)blockIdx.x * blockDim.x + threadIdx.x; traj < prm.B; traj += nthreads) {
    const double* __restrict__ pos = prm.positions + traj * (long long)(K + 1) * D;
    double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;
    for (int d = 0; d < D; ++d) {
      for (int c = 0; c < nf; ++c) fx[d * nf + c] = 0.0;
      fx[d * nf] = pos[d];
      for (int v = 1; v < K; ++v) fx[d * nf + h + v - 1] = pos[v * D + d];
      fx[d * nf + h + K - 1] = pos[K * D + d];
    }
    for (int i = 0; i < K; ++i) {
      double n2 = 0.0;
      for (int d = 0; d < D; ++d) {
        const double e = __dsub_rn(pos[(i + 1) * D + d], pos[i * D + d]);
        n2 = __dadd_rn(n2, __dmul_rn(e, e));
      }
      const double distance = sqrt(n2);
      const double lead = __dmul_rn(__ddiv_rn(distance, prm.v_max), 2.0);
      const double ex = exp(__dmul_rn(__ddiv_rn(-distance, prm.v_max), 2.0));
      prm.times[traj * K + i] =
          __dmul_rn(lead, __dadd_rn(1.0, __dmul_rn(__ddiv_rn(__dmul_rn(prm.magic, prm.v_max), prm.a_max), ex)));
    }
  }
}

// Batched getCostAndGradientMellinger (reference impl/polynomial_optimization_nonlinear_impl.h:286-364):
// every trajectory is expanded into K+1 problems -- the current segment times and, for each segment n,
// the times with +increment on n and -increment/(K-1) on the others, clamped at `lower` -- which are then
// solved and costed by the regular kernels in ONE launch each; the gradient is the forward difference.
struct MellingerParams {
  int K, D, n_fixed;
  long long B;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ dfix;    // [B][D][n_fixed]
  double* __restrict__ times_x;       // [B*(K+1)][K]
  double* __restrict__ dfix_x;        // [B*(K+1)][D][n_fixed]
  double increment, lower;
};

__global__ void __launch_bounds__(128) mellinger_expand_kernel(const MellingerParams prm) {
  const int K = prm.K, dnf = prm.D * prm.n_fixed;
  const long long total = prm.B * (K + 1);
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < total; row += nthreads) {
    const long long b = row / (K + 1);
    const int n = int(row - b * (K + 1)) - 1;  // -1: unperturbed
    const double* __restrict__ t = prm.times + b * K;
    double* __restrict__ tx = prm.times_x + row * K;
    const double corr = prm.increment / (K - 1.0);
    for (int i = 0; i < K; ++i) {
      double v = t[i];
      if (n >= 0) {
        v = (i == n) ? v + prm.increment : v - corr;
        v = v > prm.lower ? v : prm.lower;  // std::max(lower, t)
      }
      tx[i] = v;
    }
    const double* __restrict__ f = prm.dfix + b * dnf;
    double* __restrict__ fxp = prm.dfix_x + row * dnf;
    for (int c = 0; c < dnf; ++c) fxp[c] = f[c];
  }
}

__global__ void __launch_bounds__(128) mellinger_gradient_kernel(long long B, int K, const double* __restrict__ cost_x,
                                                                 double* __restrict__ cost, double* __restrict__ grad,
                                                                 double increment) {
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += nthreads) {
    const double J = cost_x[b * (K + 1)];
    if (cost) cost[b] = J;
    for (int n = 0; n < K; ++n) grad[b * K + n] = K == 1 ? 0.0 : (cost_x[b * (K + 1) + 1 + n] - J) / increment;
  }
}

// Batched Trajectory::evaluate on a uniform time grid (reference src/trajectory.cpp:48-79 semantics per
// sample; Polynomial::evaluate Horner form, polynomial.h:134-149).  One thread per (trajectory, sample),
// samples fastest so that the [B][S][D] output is written coalesced.
struct EvalParams {
  int N, K, D, derivative, n_samples;
  long long B;
  double t_start, dt;
  const double* __restrict__ times;   // [B][K]
  const double* __restrict__ coeffs;  // [B][K][D][N]
  double* __restrict__ out;           // [B][n_samples][D]
};

// Compile-time polynomial order (host switch) and derivative order (warp-uniform switch): base coefficients are
// immediates; results leave through a shared-memory tile as coalesced stores (dynamic shared memory: [blockDim.x][D]).
template <int N, int DER>
__device__ __forceinline__ double eval_horner_fused(const double (&c)[N], double t) {
  double acc = 0.0;
  if constexpr (DER < N) {
#pragma unroll
    for (int j = N - 1; j >= DER; --j) {
      double bc = 1.0;  // B(der, j) = j!/(j-der)!
#pragma unroll
      for (int q = 0; q < DER; ++q) bc *= double(j - q);
      acc = fma(acc, t, bc * c[j]);
    }
  }
  return acc;
}
template <int N>
__device__ __forceinline__ double eval_horner_fused_any(const double (&c)[N], double t, int der) {
  switch (der) {  // warp-uniform
    case 0: return eval_horner_fused<N, 0>(c, t);
    case 1: return eval_horner_fused<N, 1>(c, t);
    case 2: return eval_horner_fused<N, 2>(c, t);
    case 3: return eval_horner_fused<N, 3>(c, t);
    case 4: return eval_horner_fused<N, 4>(c, t);
    case 5: return eval_horner_fused<N, 5>(c, t);
    case 6: return eval_horner_fused<N, 6>(c, t);
    case 7: return eval_horner_fused<N, 7>(c, t);
    case 8: return eval_horner_fused<N, 8>(c, t);
    case 9: return eval_horner_fused<N, 9>(c, t);
    case 10: return eval_horner_fused<N, 10>(c, t);
    case 11: return eval_horner_fused<N, 11>(c, t);
    default: return 0.0;
  }
}

template <int N>
__global__ void __launch_bounds__(256) evaluate_kernel(const EvalParams prm) {
  extern __shared__ double eval_tile[];
  const int K = prm.K, D = prm.D, S = prm.n_samples, der = prm.derivative;
  const long long total = prm.B * S;
  const long long n_tiles = (total + blockDim.x - 1) / blockDim.x;
  for (long long ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const long long idx0 = ti * blockDim.x;
    const long long idx = idx0 + threadIdx.x;
    if (idx < total) {
      const long long b = idx / S;
      const int sidx = int(idx - b * S);
      // t_start + s * dt rounded twice, as the header and every host-side caller compute it: a contracted fma would
      // land an ulp away on some grids and take a sample on a vertex from the other segment
      const double t = __dadd_rn(prm.t_start, __dmul_rn(double(sidx), prm.dt));
      const double* __restrict__ tt = prm.times + b * K;
      double start = 0.0;
      int i = 0;
      for (; i < K; ++i) {
        const double Ti = tt[i];
        if (start + Ti > t) break;
        start += Ti;
      }
      bool in_range = true;
      if (i == K) {
        if (t > start) in_range = false;
        i = K - 1;
        start -= tt[i];
      }
      const double tl = t - start;
      double* __restrict__ o = eval_tile + threadIdx.x * D;
      for (int d = 0; d < D; ++d) {
        double acc = 0.0;
        if (in_range) {
          const double* __restrict__ cg = prm.coeffs + ((b * K + i) * D + d) * N;
          double c[N];
#pragma unroll
          for (int j = 0; j < N; ++j) c[j] = cg[j];
          acc = eval_horner_fused_any<N>(c, tl, der);
        }
        o[d] = acc;
      }
    }
    __syncthreads();
    const long long left = total - idx0;
    const int n_out = int(left < (long long)blockDim.x ? left : (long long)blockDim.x) * D;
    double* __restrict__ og = prm.out + idx0 * D;
    for (int k = threadIdx.x; k < n_out; k += blockDim.x) og[k] = eval_tile[k];
    __syncthreads();
  }
}

// Batched Trajectory::evaluateRange (reference src/trajectory.cpp:81-141) / sampleTrajectoryInRange
// (src/trajectory_sampling.cpp:45-110).  The reference walks the segments SEQUENTIALLY with a running
// `time_in_segment += dt` / `accumulated_time += dt` (so sample k is not t_start + k*dt in floating point, the
// sample clock starts at the start of the segment containing t_start, and a sample exactly on a segment end
// belongs to the left segment).  Phase 1 replays that walk, one thread per trajectory, and records for every
// sample its segment and local time; phase 2 evaluates all requested derivative orders of all dimensions, one
// thread per (trajectory, sample), with Polynomial::evaluate's own arithmetic (polynomial.h:134-149: Horner
// with a separate multiply and add -- no FMA contraction, so the samples are bit-identical to an x86 build of
// the reference).
struct RangeParams {
  int N, K, D, n_derivs, max_samples;
  int derivs[8];
  long long B;
  double t_start, t_end, dt;
  const double* __restrict__ times;    // [B][K]
  const double* __restrict__ coeffs;   // [B][K][D][N]
  int* __restrict__ seg_idx;           // [B][max_samples] scratch
  double* __restrict__ t_local;        // [B][max_samples] scratch
  int* __restrict__ n_samples;         // [B]; -1: t_start beyond the trajectory (reference logs an error, no samples)
  double* __restrict__ sampling_times; // [B][max_samples] or null
  double* __restrict__ out;            // [B][max_samples][n_derivs][D]
  // sampleTrajectoryInRange's rule around the walk (flat-state samplers only; kRangePlain for evaluateRange)
  int range_rule;
  long long* __restrict__ time_ns;     // flat-state samplers: [B][max_samples] or null
};
// kRangeChecked: n = -1 where t_start < 0, t_end exceeds the row's total time (the left-to-right sum of its segment
// times, Trajectory::max_time_) or D < 3; a t_start beyond the trajectory gives 0 samples (the reference's
// evaluateRange logs an error and sampleTrajectoryInRange still succeeds).  kRangeWhole: the same over [0, the row's
// total] (sampleWholeTrajectory), t_start and t_end are not read.
enum RangeRule { kRangePlain = 0, kRangeChecked = 1, kRangeWhole = 2 };

// The walk is sequential per trajectory (the reference accumulates `+= dt`), so a thread owns a trajectory; its samples
// are parked in shared memory 16 at a time and leave as row-contiguous runs written by half-warps (a lane storing its
// own [b][n] element touches 32 different sectors per instruction: the stores, not the walk, were the 0.17 ms).
constexpr int kRangeChunk = 16;
__global__ void __launch_bounds__(128) range_walk_kernel(const RangeParams prm) {
  __shared__ int s_si[4][32][kRangeChunk + 1];
  __shared__ double s_tl[4][32][kRangeChunk + 1];
  __shared__ double s_st[4][32][kRangeChunk + 1];
  const int K = prm.K, S = prm.max_samples;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long rounds = (prm.B + nthreads - 1) / nthreads;
  for (long long rnd = 0; rnd < rounds; ++rnd) {
    const long long b = rnd * nthreads + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long b0 = b - lane;  // first trajectory of this warp
    bool done = b >= prm.B;
    const double* __restrict__ tt = prm.times + (done ? 0 : b) * K;
    double accumulated = 0.0, Ti = 0.0, tis = 0.0;
    double t_start = prm.t_start, t_end = prm.t_end;
    int i = 0, n = 0;
    if (!done && prm.range_rule != kRangePlain) {
      double total = 0.0;
      for (int k = 0; k < K; ++k) total = __dadd_rn(total, tt[k]);
      if (prm.range_rule == kRangeWhole) {
        t_start = 0.0;
        t_end = total;
      }
      if (prm.D < 3 || t_start < 0.0 || t_end > total) {
        n = -1;
        done = true;
      }
    }
    if (!done) {
      for (i = 0; i < K; ++i) {
        accumulated = __dadd_rn(accumulated, tt[i]);
        if (accumulated > t_start) break;
      }
      if (t_start > accumulated) {
        n = prm.range_rule == kRangePlain ? -1 : 0;
        done = true;
      } else if (i >= K) {
        done = true;
      } else {
        Ti = tt[i];
        accumulated = __dsub_rn(accumulated, Ti);
        tis = __dsub_rn(t_start, accumulated);
      }
    }
    for (int n0 = 0;; n0 += kRangeChunk) {
      int cnt = 0;
      while (!done && cnt < kRangeChunk) {
        if (!(accumulated < t_end)) {
          done = true;
          break;
        }
        if (tis > Ti) {
          tis = __dsub_rn(tis, Ti);
          ++i;
          if (i >= K) {
            done = true;
            break;
          }
          Ti = tt[i];
          continue;
        }
        s_si[warp][lane][cnt] = i;
        s_tl[warp][lane][cnt] = tis;
        s_st[warp][lane][cnt] = accumulated;
        ++cnt;
        ++n;
        tis = __dadd_rn(tis, prm.dt);
        accumulated = __dadd_rn(accumulated, prm.dt);
      }
      __syncwarp();
      if (n0 < S) {
        const int col = lane & (kRangeChunk - 1), sub = lane / kRangeChunk;
#pragma unroll 4
        for (int r2 = 0; r2 < 32; r2 += 32 / kRangeChunk) {
          const int row = r2 + sub;
          const int row_cnt = __shfl_sync(0xffffffffu, cnt, row);
          if (col < row_cnt && n0 + col < S) {
            const long long at = (b0 + row) * S + n0 + col;
            prm.seg_idx[at] = s_si[warp][row][col];
            prm.t_local[at] = s_tl[warp][row][col];
            if (prm.sampling_times) prm.sampling_times[at] = s_st[warp][row][col];
          }
        }
      }
      __syncwarp();
      if (!__any_sync(0xffffffffu, !done)) break;
    }
    if (b < prm.B) prm.n_samples[b] = n;
  }
}

// One thread per sample; a block owns `blockDim.x` consecutive samples of the flattened [B][max_samples] index, i.e. one
// CONTIGUOUS span of blockDim.x * n_derivs * D output doubles: results go to a shared-memory tile and leave as fully
// coalesced stores (the per-thread 120-byte records written directly cost 4-5x the store transactions).
// The polynomial order and the derivative order are compile-time (host switch on N, warp-uniform switch on the
// derivative), so the base coefficients B(der, j) = j!/(j-der)! are immediates (exact small integers, the same
// successive products as Polynomial::base_coefficients_) and the Horner recurrence is the reference's, unfused, with no
// wasted steps -- the runtime-order form spent 2800 instructions per sample, 0.90 ms of the 1.07 ms call.
// dynamic shared memory: [blockDim.x][n_derivs * D] tile
template <int DER>
__host__ __device__ constexpr double range_base_coeff(int j) {
  double b = 1.0;
  for (int w = 0; w < DER; ++w) b *= double(j - w);
  return b;
}
template <int N, int DER>
__device__ __forceinline__ double range_horner(const double (&c)[N], double t) {
  if constexpr (DER >= N) {
    return 0.0;
  } else {
    double acc = __dmul_rn(range_base_coeff<DER>(N - 1), c[N - 1]);
#pragma unroll
    for (int j = N - 2; j >= DER; --j) {
      acc = __dmul_rn(acc, t);
      acc = __dadd_rn(acc, __dmul_rn(range_base_coeff<DER>(j), c[j]));
    }
    return acc;
  }
}
template <int N>
__device__ __forceinline__ double range_horner_any(const double (&c)[N], double t, int der) {
  switch (der) {  // warp-uniform
    case 0: return range_horner<N, 0>(c, t);
    case 1: return range_horner<N, 1>(c, t);
    case 2: return range_horner<N, 2>(c, t);
    case 3: return range_horner<N, 3>(c, t);
    case 4: return range_horner<N, 4>(c, t);
    case 5: return range_horner<N, 5>(c, t);
    case 6: return range_horner<N, 6>(c, t);
    case 7: return range_horner<N, 7>(c, t);
    case 8: return range_horner<N, 8>(c, t);
    case 9: return range_horner<N, 9>(c, t);
    case 10: return range_horner<N, 10>(c, t);
    case 11: return range_horner<N, 11>(c, t);
    default: return 0.0;
  }
}

template <int N>
__global__ void __launch_bounds__(256) range_eval_kernel(const RangeParams prm) {
  extern __shared__ double range_tile[];
  const int K = prm.K, D = prm.D, S = prm.max_samples, ND = prm.n_derivs;
  const int rec = ND * D;
  const long long total = prm.B * S;
  const long long n_tiles = (total + blockDim.x - 1) / blockDim.x;
  for (long long ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const long long idx0 = ti * blockDim.x;
    const long long idx = idx0 + threadIdx.x;
    if (idx < total) {
      const long long b = idx / S;
      const int s = int(idx - b * S);
      const int n = prm.n_samples[b];
      double* __restrict__ o = range_tile + threadIdx.x * rec;
      if (s >= n) {  // beyond this trajectory's sample count: defined output (zeros)
        for (int q = 0; q < rec; ++q) o[q] = 0.0;
      } else {
        const int i = prm.seg_idx[idx];
        const double t = prm.t_local[idx];
        for (int d = 0; d < D; ++d) {
          const double* __restrict__ cg = prm.coeffs + ((b * K + i) * D + d) * N;
          double c[N];
#pragma unroll
          for (int j = 0; j < N; ++j) c[j] = cg[j];
          for (int q = 0; q < ND; ++q) o[q * D + d] = range_horner_any<N>(c, t, prm.derivs[q]);
        }
      }
    }
    __syncthreads();
    const long long left = total - idx0;
    const int n_out = int(left < (long long)blockDim.x ? left : (long long)blockDim.x) * rec;
    double* __restrict__ og = prm.out + idx0 * rec;
    for (int k = threadIdx.x; k < n_out; k += blockDim.x) og[k] = range_tile[k];
    __syncthreads();
  }
}

// computeCost() (linear_impl.h:123-140): 0.5 * sum c^T Q(T) c with
// Q[a][b] = 2 B(r,a) B(r,b) T^(a+b-2r+1) / (a+b-2r+1)   (:567-583).
struct CostParams {
  int N, r, K, D;
  long long B;
  const double* __restrict__ times;
  const double* __restrict__ coeffs;
  double* __restrict__ cost;
};

// Work item = (trajectory, segment, dimension): its N coefficients are contiguous and consecutive items are contiguous,
// so a block reads one contiguous span of the coefficient tensor (the thread-per-trajectory form walked 3 840-byte
// rows with a 3 840-byte stride between lanes and kept q[] in local memory).  The per-item sum is the reference-order
// double loop; the trajectory's total is then accumulated by ONE thread in (segment, dimension) order with the same
// fma, so the result is bitwise what the thread-per-trajectory kernel produced.
// dynamic shared memory: [12] B(r,a), [24] 1/k, [tpb * K * D] per-item sums   (tpb = trajectories per block pass)
// NT, RT > 0: compile-time order / derivative (the double loop is (N-r)^2 fused multiply-adds with immediate 1/k);
// NT = 0: any (N, r) with predicated 12 x 12 loops.
template <int NT, int RT>
__global__ void __launch_bounds__(256) cost_kernel(const CostParams prm, const int tpb) {
  extern __shared__ double cost_sm[];
  double* bcoef = cost_sm;
  double* inv = cost_sm + 12;
  double* partial = cost_sm + 36;
  const int N = NT > 0 ? NT : prm.N, r = NT > 0 ? RT : prm.r, K = prm.K, D = prm.D, KD = K * D;
  if (threadIdx.x < 12) {
    double bc = 1.0;  // B(r,a) = a!/(a-r)!
    for (int k = 0; k < r; ++k) bc *= double(int(threadIdx.x) - k);
    bcoef[threadIdx.x] = bc;
  }
  if (threadIdx.x < 24) inv[threadIdx.x] = threadIdx.x ? 1.0 / double(threadIdx.x) : 0.0;
  __syncthreads();
  for (long long t0 = (long long)blockIdx.x * tpb; t0 < prm.B; t0 += (long long)gridDim.x * tpb) {
    const int ntraj = int(prm.B - t0 < tpb ? prm.B - t0 : tpb);
    const int items = ntraj * KD;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
      const int lt = it / KD, i = (it - lt * KD) / D;
      const double T = prm.times[(t0 + lt) * K + i];
      const double* __restrict__ c = prm.coeffs + (t0 * KD + it) * N;
      double sum = 0.0;
      if constexpr (NT > 0) {
        double q[NT];
        double tpow = 1.0;
#pragma unroll
        for (int a = RT; a < NT; ++a) {
          q[a] = bcoef[a] * c[a] * tpow;
          tpow *= T;
        }
#pragma unroll
        for (int a = RT; a < NT; ++a)
#pragma unroll
          for (int b = RT; b < NT; ++b) sum = fma(q[a] * q[b], 1.0 / double(a + b - 2 * RT + 1), sum);
      } else {
        double q[12];
        double tpow = 1.0;
#pragma unroll
        for (int a = 0; a < 12; ++a) {
          q[a] = 0.0;
          if (a >= r && a < N) {
            q[a] = bcoef[a] * c[a] * tpow;
            tpow *= T;
          }
        }
#pragma unroll
        for (int a = 0; a < 12; ++a) {
          if (a >= r && a < N) {
#pragma unroll
            for (int b = 0; b < 12; ++b)
              if (b >= r && b < N) sum = fma(q[a] * q[b], inv[a + b - 2 * r + 1], sum);
          }
        }
      }
      partial[it] = sum;
    }
    __syncthreads();
    if (threadIdx.x < ntraj) {
      const long long traj = t0 + threadIdx.x;
      double total = 0.0;
      for (int i = 0; i < K; ++i) {
        const double T = prm.times[traj * K + i];
        for (int d = 0; d < D; ++d) total = fma(partial[threadIdx.x * KD + i * D + d], T, total);  // 0.5 * 2 * T * sum
      }
      prm.cost[traj] = total;
    }
    __syncthreads();
  }
}

}  // namespace mtg
