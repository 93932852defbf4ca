// mtg_masked_block_kernel.cuh -- K4 (v2): arbitrary per-vertex constraint masks (any Vertex::Vector the reference
// accepts) as a MASKED BLOCK-TRIDIAGONAL solve, everything in registers, no local memory, no zero-initialised
// band, TMA tensor stores of the coefficients.
//
// Reference path replaced: setupConstraintReorderingMatrix + constructR + solveLinear +
// updateSegmentsFromCompactConstraints (impl/polynomial_optimization_linear_impl.h:181-379) for masks that are
// not the createRandomVertices topology.
//
// Formulation.  Every vertex v = 0..K owns h = N/2 slots z_v (derivatives 0..h-1), fixed or free by the
// topology's mask (uniform over the batch).  Over ALL slots the cost matrix R = C^T H C is block tridiagonal
// with h x h blocks:  A_v = H_{v-1}[end,end] + H_v[start,start],  B_v = H_v[start,end].  With P = diag(free),
//     M = P R P + (I - P),      f = (I - P) d - P R (I - P) d
// is SPD block tridiagonal with the SAME uniform block structure for any mask, its solution carries the free
// derivatives in the free slots (R_pp d_p = -R_pf d_f, linear_impl.h:360-375) and reproduces the fixed values in
// the fixed slots (identity rows) -- so one branch-free code path serves every mask: the mask only enters as 0/1
// factors, warp-uniform because the topology is shared by the batch.  Block Cholesky forward sweep v = 0..K
//     D'_v = M_vv - W_{v-1}^T W_{v-1},  L_v = chol(D'_v),  y_v = L_v^-1 (f_v - W_{v-1}^T y_{v-1}),
//     W_v = L_v^-1 M_{v,v+1}
// and backward sweep  z_v = L_v^-T (y_v - W_v z_{v+1})  emitting segment v = [z_v, z_{v+1}] as soon as both ends
// are known (p = A^-1 C d, linear_impl.h:262-283, with the exact scaled table A(1)^-1).  H_i comes from the exact
// table H(1;r) and powers of T_i (mtg_device.cuh).
//
// Mapping: one thread per trajectory, 128-thread CTAs, persistent grid-stride over 32-trajectory warp tiles.
// The factor (L_v: h(h+1)/2, y_v: h*D doubles per vertex; W_v is recomputed from T_v on the way back) is a LIFO in
// global memory, [vertex][slot][resident thread] so that every access is coalesced; it is written once and read
// once (8*(K+1)*(h(h+1)/2 + h*D)*2 bytes per trajectory -- for N = 10, D = 3, K = 16: 8.2 KB next to 4.9 KB of
// algorithmic traffic), which bounds this kernel well below the HBM roofline.  Dimensions are processed in
// groups of DG <= 4 (template), larger D re-runs the sweep per group.
#pragma once

#include "mtg_generic_kernel.cuh"
#include "mtg_twisted_tmem_kernel.cuh"

namespace mtg {

struct MaskedParams {
  int N, r, K, D;
  int n_fixed, n_free;
  int d0;                                // first dimension of this pass (D > DG)
  long long B;
  const int* __restrict__ vcol;          // [(K+1)*h]: column of (vertex, derivative): < n_fixed fixed, else free
  const double* __restrict__ times;      // [B][K]
  const double* __restrict__ dfix;       // [B][D][n_fixed]
  double* __restrict__ coeffs;           // [B][K][D][N]
  double* __restrict__ dfree;            // [B][D][n_free] or null
  int* __restrict__ status;              // [B] or null
  double* __restrict__ lifo;             // [(K+1)][slots][gridDim.x * 128]
};

template <int N, int DG>
__host__ __device__ constexpr int masked_state_slots() {
  return (N / 2) * (N / 2 + 1) / 2 + (N / 2) * DG;
}

// TMA store of DG dimensions of one segment for 16 trajectories: coeffs viewed as [B][K*D*N], box [16][DG*N]
template <int N, int DG>
__global__ void __launch_bounds__(128, 2)
    masked_block_kernel(const MaskedParams prm, const __grid_constant__ CUtensorMap tmap) {
  constexpr int h = N / 2;
  constexpr int kL = h * (h + 1) / 2;
  constexpr int kSlots = kL + h * DG;
  constexpr int kWarps = 4;
  using AI = A1InvImm<N>;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int K = prm.K, nf = prm.n_fixed, np = prm.n_free, D = prm.D, d0 = prm.d0;
  const double* __restrict__ Gt = h1_table(N, prm.r);  // H(1;r), constant memory, warp-uniform reads
  auto G = [&](int a, int b) -> double { return Gt[a * N + b]; };

  // staging tile of this warp: [32 trajectories][DG*N doubles], two 16-row TMA boxes
  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (DG * h);
  double2* my_row = stage + lane * (DG * h);

  const long long gthreads = (long long)gridDim.x * blockDim.x;
  double* __restrict__ lifo = prm.lifo + ((long long)blockIdx.x * blockDim.x + threadIdx.x);
  auto ST = [&](int v, int slot) -> double& { return lifo[((long long)v * kSlots + slot) * gthreads]; };

  const long long n_wtiles = (prm.B + 31) >> 5;
  for (long long wt = (long long)blockIdx.x * kWarps + warp; wt < n_wtiles; wt += (long long)gridDim.x * kWarps) {
    long long traj = wt * 32 + lane;
    const long long traj0 = wt * 32;
    const bool valid = traj < prm.B;
    if (!valid) traj = prm.B - 1;
    const double* __restrict__ tt = prm.times + traj * K;
    const double* __restrict__ fx = prm.dfix + traj * (long long)D * nf;

    // free-slot bit mask of a vertex (warp-uniform) and the fixed value of (vertex, derivative k, dimension d)
    auto free_mask = [&](int v) -> unsigned {
      unsigned mk = 0;
#pragma unroll
      for (int k = 0; k < h; ++k) mk |= (__ldg(prm.vcol + v * h + k) >= nf ? 1u : 0u) << k;
      return mk;
    };
    auto is_free = [](unsigned mk, int k) -> bool { return (mk >> k) & 1u; };
    auto fixed_value = [&](int v, int k, int d) -> double { return __ldg(fx + (d0 + d) * nf + __ldg(prm.vcol + v * h + k)); };
    auto seg_powers = [&](double T, double (&pw)[N - 1]) {
      const double iT = 1.0 / T;
      double p0 = T;  // T^(1-2r)
      for (int q = 0; q < 2 * prm.r; ++q) p0 *= iT;
      pw[0] = p0;
#pragma unroll
      for (int e = 1; e < N - 1; ++e) pw[e] = pw[e - 1] * T;
    };

    int stat = 0;
    double pwp[N - 1], pwc[N - 1];  // powers of T_{v-1} and T_v (zero where the segment does not exist)
    double Wp[h][h], yp[h][DG];     // W_{v-1}, y_{v-1}
#pragma unroll
    for (int a = 0; a < h; ++a) {
#pragma unroll
      for (int b = 0; b < h; ++b) Wp[a][b] = 0.0;
#pragma unroll
      for (int d = 0; d < DG; ++d) yp[a][d] = 0.0;
    }
#pragma unroll
    for (int e = 0; e < N - 1; ++e) pwp[e] = 0.0;
    unsigned mm = 0, mc = free_mask(0), mn = 0;  // free masks of vertices v-1, v, v+1

    // ------------------------------------------------------------ forward sweep, vertices 0..K
    for (int v = 0; v <= K; ++v) {
      if (v < K) {
        const double T = __ldg(tt + v);
        if (bad_segment_time(T)) stat |= kStatusBadTime;  // +inf too: a segment between two fully fixed
                                                          // vertices reaches no pivot
        seg_powers(T, pwc);
        mn = free_mask(v + 1);
      } else {
#pragma unroll
        for (int e = 0; e < N - 1; ++e) pwc[e] = 0.0;
        mn = 0;
      }
      // f = (I - P) d - P (B_{v-1}^T g_{v-1} + A_v g_v + B_v g_{v+1}) - W_{v-1}^T y_{v-1}, g = fixed values (0 at
      // free slots), streamed: one (vertex, derivative) at a time so that no g vector stays live
      double Dp[h][h], f[h][DG];
#pragma unroll
      for (int a = 0; a < h; ++a)
#pragma unroll
        for (int d = 0; d < DG; ++d) {
          double s = 0.0;
#pragma unroll
          for (int k = 0; k < h; ++k) s = fma(-Wp[k][a], yp[k][d], s);
          f[a][d] = s;
        }
#pragma unroll
      for (int b = 0; b < h; ++b) {
        if (v > 0 && !is_free(mm, b)) {  // warp-uniform
#pragma unroll
          for (int d = 0; d < DG; ++d) {
            const double g = fixed_value(v - 1, b, d);
#pragma unroll
            for (int a = 0; a < h; ++a)
              if (is_free(mc, a)) f[a][d] = fma(-(pwp[a + b] * G(b, h + a)), g, f[a][d]);  // (B_{v-1}^T)[a][b]
          }
        }
        if (!is_free(mc, b)) {
#pragma unroll
          for (int d = 0; d < DG; ++d) {
            const double g = fixed_value(v, b, d);
#pragma unroll
            for (int a = 0; a < h; ++a) {
              if (a == b) {
                f[a][d] += g;  // identity row of a fixed slot
              } else if (is_free(mc, a)) {
                f[a][d] = fma(-fma(pwp[a + b], G(h + a, h + b), pwc[a + b] * G(a, b)), g, f[a][d]);  // A_v[a][b]
              }
            }
          }
        }
        if (v < K && !is_free(mn, b)) {
#pragma unroll
          for (int d = 0; d < DG; ++d) {
            const double g = fixed_value(v + 1, b, d);
#pragma unroll
            for (int a = 0; a < h; ++a)
              if (is_free(mc, a)) f[a][d] = fma(-(pwc[a + b] * G(a, h + b)), g, f[a][d]);  // B_v[a][b]
          }
        }
      }
      // D'_v = P A_v P + (I - P) - W_{v-1}^T W_{v-1}
#pragma unroll
      for (int a = 0; a < h; ++a)
#pragma unroll
        for (int b = 0; b <= a; ++b) {
          double s = (is_free(mc, a) && is_free(mc, b)) ? fma(pwp[a + b], G(h + a, h + b), pwc[a + b] * G(a, b))
                                                        : ((a == b) ? 1.0 : 0.0);
#pragma unroll
          for (int k = 0; k < h; ++k) s = fma(-Wp[k][a], Wp[k][b], s);
          Dp[a][b] = s;
        }
      double inv[h];
#pragma unroll
      for (int j = 0; j < h; ++j) {  // in-place Cholesky: Dp becomes L (strictly lower), inv = 1 / diagonal
        double s = Dp[j][j];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-Dp[j][k], Dp[j][k], s);
        if (!(s > 0.0) || isinf(s)) stat |= kStatusNotSpd;
        inv[j] = fast_rsqrt(s);
#pragma unroll
        for (int i = j + 1; i < h; ++i) {
          double t = Dp[i][j];
#pragma unroll
          for (int k = 0; k < j; ++k) t = fma(-Dp[i][k], Dp[j][k], t);
          Dp[i][j] = t * inv[j];
        }
      }
#pragma unroll
      for (int d = 0; d < DG; ++d) {
#pragma unroll
        for (int j = 0; j < h; ++j) {
          double s = f[j][d];
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-Dp[j][k], yp[k][d], s);
          yp[j][d] = s * inv[j];
        }
      }
      // W_v = L_v^-1 (P_v B_v P_{v+1})
#pragma unroll
      for (int c = 0; c < h; ++c) {
#pragma unroll
        for (int j = 0; j < h; ++j) {
          double s = (is_free(mc, j) && is_free(mn, c)) ? pwc[j + c] * G(j, h + c) : 0.0;
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-Dp[j][k], Wp[k][c], s);
          Wp[j][c] = s * inv[j];
        }
      }
      {  // push (L_v, 1/pivots, y_v)
        int slot = 0;
#pragma unroll
        for (int i = 1; i < h; ++i)
#pragma unroll
          for (int j = 0; j < i; ++j) ST(v, slot++) = Dp[i][j];
#pragma unroll
        for (int j = 0; j < h; ++j) ST(v, slot++) = inv[j];
#pragma unroll
        for (int j = 0; j < h; ++j)
#pragma unroll
          for (int d = 0; d < DG; ++d) ST(v, slot++) = yp[j][d];
      }
      mm = mc;
      mc = mn;
#pragma unroll
      for (int e = 0; e < N - 1; ++e) pwp[e] = pwc[e];
    }
    if (valid && prm.status != nullptr && d0 == 0) prm.status[traj] = stat;

    // ------------------------------------------------------------ backward sweep, vertices K..0
    double zn[h][DG];  // z_{v+1}
#pragma unroll
    for (int a = 0; a < h; ++a)
#pragma unroll
      for (int d = 0; d < DG; ++d) zn[a][d] = 0.0;
    for (int v = K; v >= 0; --v) {
      double L[h][h], inv[h], y[h][DG];
      {
        int slot = 0;
#pragma unroll
        for (int i = 1; i < h; ++i)
#pragma unroll
          for (int j = 0; j < i; ++j) L[i][j] = ST(v, slot++);
#pragma unroll
        for (int j = 0; j < h; ++j) inv[j] = ST(v, slot++);
#pragma unroll
        for (int j = 0; j < h; ++j)
#pragma unroll
          for (int d = 0; d < DG; ++d) y[j][d] = ST(v, slot++);
      }
      double T = 1.0, pw[N - 1];
      const unsigned mv = free_mask(v), mv1 = v < K ? free_mask(v + 1) : 0u;
      if (v < K) {
        T = __ldg(tt + v);
        seg_powers(T, pw);
      } else {
#pragma unroll
        for (int e = 0; e < N - 1; ++e) pw[e] = 0.0;
      }
      double z[h][DG];
#pragma unroll
      for (int d = 0; d < DG; ++d) {
        // t = L^-1 (M_{v,v+1} z_{v+1});  z_v = L^-T (y_v - t)
        double t[h];
#pragma unroll
        for (int a = 0; a < h; ++a) {
          double s = 0.0;
#pragma unroll
          for (int b = 0; b < h; ++b)
            if (is_free(mv, a) && is_free(mv1, b)) s = fma(pw[a + b] * G(a, h + b), zn[b][d], s);
          t[a] = s;
        }
#pragma unroll
        for (int j = 0; j < h; ++j) {
          double s = t[j];
#pragma unroll
          for (int k = 0; k < j; ++k) s = fma(-L[j][k], t[k], s);
          t[j] = s * inv[j];
          y[j][d] -= t[j];
        }
#pragma unroll
        for (int j = h - 1; j >= 0; --j) {
          double s = y[j][d];
#pragma unroll
          for (int k = j + 1; k < h; ++k) s = fma(-L[k][j], z[k][d], s);
          z[j][d] = s * inv[j];
        }
      }
      if (prm.dfree != nullptr && valid) {  // getFreeConstraints order: (vertex, derivative) rank among the free ones
#pragma unroll
        for (int k = 0; k < h; ++k) {
          const int col = __ldg(prm.vcol + v * h + k);
          if (col >= nf) {
#pragma unroll
            for (int d = 0; d < DG; ++d)
              if (d0 + d < D) prm.dfree[traj * (long long)D * np + (long long)(d0 + d) * np + (col - nf)] = z[k][d];
          }
        }
      }
      if (v < K) {
        // ---- emit segment v: start z_v, end z_{v+1}   (A(1)^-1 in Hermite form, as the waypoint kernels)
        const double iT = 1.0 / T;
        double tp[h], itp[h];
        sweep::Hermite<N, AI>::powers(T, iT, false, tp, itp);
        if (lane == 0) bulk_wait_read();
        __syncwarp();
#pragma unroll
        for (int d = 0; d < DG; ++d) {
          double c[N];
          sweep::Hermite<N, AI>::template coeffs<DG>(false, tp, itp, z, zn, d, c);
#pragma unroll
          for (int q = 0; q < h; ++q) my_row[d * h + q] = make_double2(c[2 * q], c[2 * q + 1]);
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          const int c0 = (v * D + d0) * N;  // first double of (segment v, dimension d0) inside the trajectory row
          tma_store_box(&tmap, stage, c0, (int)traj0);
          tma_store_box(&tmap, stage + 16 * (DG * h), c0, (int)traj0 + 16);
          bulk_commit();
        }
      }
#pragma unroll
      for (int a = 0; a < h; ++a)
#pragma unroll
        for (int d = 0; d < DG; ++d) zn[a][d] = z[a][d];
    }
  }
  if (lane == 0) bulk_wait_all();
}

}  // namespace mtg
