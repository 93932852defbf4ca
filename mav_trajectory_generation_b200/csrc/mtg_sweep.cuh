// mtg_sweep.cuh -- the per-vertex arithmetic of the waypoint (block-tridiagonal) sweep, written once for every kernel
// that runs it (v1 one-thread, v2 twisted, v3, v4, v5 and the chunked kernel K3) and the Hermite-form emission of the
// twisted TMA kernels and the masked kernel.
//
// Mathematics: see mtg_waypoint_kernel.cuh; twisted frames and index maps: mtg_twisted_kernel.cuh.  Each piece fixes
// one operation order; the kernels only choose where they call it.  Two differences between kernels are deliberate
// and change rounding:
//   * the first step's right-hand-side carry is an explicit term `bcar` (v1, v2, v3) or is folded into the (W, y)
//     carry with an exact power-of-two scaling (v4, v5, K3): carry_bcar / carry_fold and the two overloads of
//     assemble() and middle().  The fold form starts the right-hand side with -cps*xm, which is not
//     fma(-cps, xm, 0.0): the latter can flip the sign of a zero.
//   * where the outward step's E u product is computed: couple() before the activity test in v4 and K3 (K3 runs
//     at the register limit), inside it in v5; uncouple_from() interleaves it with the solve per dimension (v1-v3).
// v1 sweeps the whole trajectory in one thread: it folds the far end's fixed derivatives u_K into the last
// right-hand side between assemble() and factor(), and its last outward step has no coupling term.
#pragma once

#include "mtg_device.cuh"

namespace mtg {

// doubles of one eliminated vertex's sweep-state block: L (strictly lower), inverse pivots, y, and optionally the
// vertex position
template <int N, int D, bool kPos = false>
__host__ __device__ constexpr int sweep_state_slots() {
  return (N / 2 - 1) * (N / 2) / 2 + (N / 2 - 1) * D + (kPos ? D : 0);
}

namespace sweep {

// own-frame -> original index maps of lane `half` (1: the time-reversed half) of a K-segment trajectory
template <int N>
struct Frame {
  int K, half;
  __device__ __forceinline__ int seg(int j) const { return half ? K - 1 - j : j; }
  __device__ __forceinline__ int vert(int v) const { return half ? K - v : v; }
  // position slot of own-frame vertex v inside one dimension's d_fixed
  __device__ __forceinline__ int pidx(int v) const {
    const int o = half ? K - v : v;
    return o == 0 ? 0 : (o < K ? N / 2 + o - 1 : N / 2 + K - 1);
  }
  // sign of derivative (idx+1) under time reversal
  __device__ __forceinline__ double sgn(int idx) const { return (half && !(idx & 1)) ? -1.0 : 1.0; }
  // first fixed end-derivative slot of own-frame vertex 0
  __device__ __forceinline__ int e0() const { return half ? N / 2 + K : 1; }
};

template <int N, int D, class G>
struct Sweep {
  static constexpr int h = N / 2;
  static constexpr int m = h - 1;
  static constexpr int kL = m * (m + 1) / 2;
  static constexpr unsigned kFull = 0xffffffffu;

  // blocks of the segment just stepped over that couple its end vertex (the next one to eliminate): H[end, end]
  // (lower triangle), H[end, start position], H[end, end position]
  static __device__ __forceinline__ void end_blocks(const double (&pw)[N - 1], double (&Cee)[m][m], double (&cps)[m],
                                                    double (&cpe)[m]) {
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) Cee[a][b] = pw[a + b + 2] * G::at(h + 1 + a, h + 1 + b);
      cps[a] = pw[a + 1] * G::at(h + 1 + a, 0);
      cpe[a] = pw[a + 1] * G::at(h + 1 + a, h);
    }
  }

  // carry of the fixed end derivatives u0(b, d) (derivative b+1 of own vertex 0, own-frame sign) into the first step:
  // an explicit right-hand-side term bcar = -H_0[end, start] u0, with W = 0 and y = 0
  template <class U0>
  static __device__ __forceinline__ void carry_bcar(const double (&pw)[N - 1], const U0& u0, double (&Wp)[m][m],
                                                    double (&yp)[m][D], double (&bcar)[m][D]) {
#pragma unroll
    for (int a = 0; a < m; ++a)
#pragma unroll
      for (int b = 0; b < m; ++b) Wp[a][b] = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double u[m];
#pragma unroll
      for (int b = 0; b < m; ++b) u[b] = u0(b, d);
#pragma unroll
      for (int a = 0; a < m; ++a) {
        double acc = 0.0;
#pragma unroll
        for (int b = 0; b < m; ++b) acc = fma(pw[a + b + 2] * G::at(h + 1 + a, 1 + b), u[b], acc);
        bcar[a][d] = -acc;
        yp[a][d] = 0.0;
      }
    }
  }
  // the same carry stored as y = 2^600 * (H u0) against W = 2^-600 I, so that -W^T y reproduces it exactly and W^T W
  // underflows to zero: the m*D carry registers disappear from the loop
  template <class U0>
  static __device__ __forceinline__ void carry_fold(const double (&pw)[N - 1], const U0& u0, double (&Wp)[m][m],
                                                    double (&yp)[m][D]) {
    constexpr double kTiny = 0x1p-600, kHuge = 0x1p+600;
#pragma unroll
    for (int a = 0; a < m; ++a)
#pragma unroll
      for (int b = 0; b < m; ++b) Wp[a][b] = (a == b) ? kTiny : 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double u[m];
#pragma unroll
      for (int b = 0; b < m; ++b) u[b] = u0(b, d);
#pragma unroll
      for (int a = 0; a < m; ++a) {
        double acc = 0.0;
#pragma unroll
        for (int b = 0; b < m; ++b) acc = fma(pw[a + b + 2] * G::at(h + 1 + a, 1 + b), u[b], acc);
        yp[a][d] = acc * kHuge;
      }
    }
  }

  // inward step, assembly: the Schur-complemented diagonal block D' (lower triangle), the coupling E to the next
  // vertex and the right-hand side b' (xm, xc, xn: positions of the previous, current and next vertex)
  static __device__ __forceinline__ void assemble(const double (&pw)[N - 1], const double (&Cee)[m][m],
                                                  const double (&cps)[m], const double (&cpe)[m],
                                                  const double (&Wp)[m][m], const double (&yp)[m][D],
                                                  const double (&xm)[D], const double (&xc)[D], const double (&xn)[D],
                                                  double (&Dp)[m][m], double (&E)[m][m], double (&bb)[m][D]) {
    assemble_impl<false>(pw, Cee, cps, cpe, nullptr, Wp, yp, xm, xc, xn, Dp, E, bb);
  }
  // ... with the explicit first-step carry term bcar
  static __device__ __forceinline__ void assemble(const double (&pw)[N - 1], const double (&Cee)[m][m],
                                                  const double (&cps)[m], const double (&cpe)[m],
                                                  const double (&bcar)[m][D], const double (&Wp)[m][m],
                                                  const double (&yp)[m][D], const double (&xm)[D],
                                                  const double (&xc)[D], const double (&xn)[D], double (&Dp)[m][m],
                                                  double (&E)[m][m], double (&bb)[m][D]) {
    assemble_impl<true>(pw, Cee, cps, cpe, bcar, Wp, yp, xm, xc, xn, Dp, E, bb);
  }

  // Cholesky of a symmetric block (lower triangle read) with inverse pivots; a pivot that is not > 0 or is infinite sets
  // kStatusNotSpd
  static __device__ __forceinline__ void cholesky(const double (&A)[m][m], double (&L)[m][m], double (&inv)[m],
                                                  int& stat) {
#pragma unroll
    for (int j = 0; j < m; ++j) {
      double s = A[j][j];
#pragma unroll
      for (int k = 0; k < j; ++k) s = fma(-L[j][k], L[j][k], s);
      if (!(s > 0.0) || isinf(s)) stat |= kStatusNotSpd;
      inv[j] = fast_rsqrt(s);
#pragma unroll
      for (int i = j + 1; i < m; ++i) {
        double t = A[i][j];
#pragma unroll
        for (int k = 0; k < j; ++k) t = fma(-L[i][k], L[j][k], t);
        L[i][j] = t * inv[j];
      }
    }
  }

  // inward step, factorisation: D' = L L^T, y <- L^-1 b', W <- L^-1 E
  static __device__ __forceinline__ void factor(const double (&Dp)[m][m], const double (&E)[m][m],
                                                const double (&bb)[m][D], double (&L)[m][m], double (&inv)[m],
                                                double (&Wp)[m][m], double (&yp)[m][D], int& stat) {
    cholesky(Dp, L, inv, stat);
#pragma unroll
    for (int d = 0; d < D; ++d) {
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = bb[j][d];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], yp[k][d], s);
        yp[j][d] = s * inv[j];
      }
    }
#pragma unroll
    for (int c = 0; c < m; ++c) {
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = E[j][c];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], Wp[k][c], s);
        Wp[j][c] = s * inv[j];
      }
    }
  }

  // state block of an eliminated vertex: strictly lower L, then the inverse pivots, then y, then (S == kL + m*D + D)
  // the vertex position
  template <int S>
  static __device__ __forceinline__ void pack(const double (&L)[m][m], const double (&inv)[m], const double (&yp)[m][D],
                                              const double* xpos, double (&sv)[S]) {
    static_assert(S == kL + m * D || S == kL + m * D + D, "state block size");
    int slot = 0;
#pragma unroll
    for (int i = 1; i < m; ++i)
#pragma unroll
      for (int j = 0; j < i; ++j) sv[slot++] = L[i][j];
#pragma unroll
    for (int j = 0; j < m; ++j) sv[slot++] = inv[j];
#pragma unroll
    for (int j = 0; j < m; ++j)
#pragma unroll
      for (int d = 0; d < D; ++d) sv[slot++] = yp[j][d];
    if constexpr (S > kL + m * D) {
#pragma unroll
      for (int d = 0; d < D; ++d) sv[slot++] = xpos[d];
    }
  }
  template <int S>
  static __device__ __forceinline__ void unpack(const double (&sv)[S], double (&L)[m][m], double (&inv)[m],
                                                double (&rhs)[m][D]) {
    int slot = 0;
#pragma unroll
    for (int i = 1; i < m; ++i)
#pragma unroll
      for (int j = 0; j < i; ++j) L[i][j] = sv[slot++];
#pragma unroll
    for (int j = 0; j < m; ++j) inv[j] = sv[slot++];
#pragma unroll
    for (int j = 0; j < m; ++j)
#pragma unroll
      for (int d = 0; d < D; ++d) rhs[j][d] = sv[slot++];
  }
  template <int S>
  static __device__ __forceinline__ double position(const double (&sv)[S], int d) {
    static_assert(S == kL + m * D + D, "the state block holds no position");
    return sv[kL + m * D + d];
  }

  // middle vertex: own half of the Schur complement and right-hand side, exchanged with the partner lane and combined
  // (X_own + J X_partner J, J = diag((-1)^k)), then solved for the middle derivatives um.  stat becomes the status of
  // the whole trajectory.
  static __device__ __forceinline__ void middle(const double (&Cee)[m][m], const double (&cps)[m],
                                                const double (&cpe)[m], const double (&Wp)[m][m],
                                                const double (&yp)[m][D], const double (&xm)[D],
                                                const double (&xc)[D], double (&um)[m][D], int& stat) {
    middle_impl<false>(Cee, cps, cpe, nullptr, Wp, yp, xm, xc, um, stat);
  }
  // ... with the explicit first-step carry term bcar (still live when the half eliminated no vertex)
  static __device__ __forceinline__ void middle(const double (&Cee)[m][m], const double (&cps)[m],
                                                const double (&cpe)[m], const double (&bcar)[m][D],
                                                const double (&Wp)[m][m], const double (&yp)[m][D],
                                                const double (&xm)[D], const double (&xc)[D], double (&um)[m][D],
                                                int& stat) {
    middle_impl<true>(Cee, cps, cpe, bcar, Wp, yp, xm, xc, um, stat);
  }

  // outward step, coupling: tE = E_v u_{v+1} (ed: the derivatives of the vertex solved last)
  static __device__ __forceinline__ void couple(const double (&pw)[N - 1], const double (&ed)[h][D],
                                                double (&tE)[m][D]) {
#pragma unroll
    for (int d = 0; d < D; ++d)
#pragma unroll
      for (int a = 0; a < m; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < m; ++b) s = fma(pw[a + b + 2] * G::at(1 + a, h + 1 + b), ed[1 + b][d], s);
        tE[a][d] = s;
      }
  }
  // outward step, back-substitution: u_v = L^-T (y - L^-1 tE) from the vertex's state block sv; sd = [xv; u_v]
  template <int S>
  static __device__ __forceinline__ void back_substitute(const double (&sv)[S], const double (&tE)[m][D],
                                                         const double (&xv)[D], double (&sd)[h][D]) {
    double L[m][m], inv[m], rhs[m][D];
    unpack(sv, L, inv, rhs);
    uncouple(L, inv, tE, rhs);
    solve_back(L, inv, rhs, xv, sd);
  }
  // rhs <- y - L^-1 E_v u_{v+1} one dimension at a time: the product and the solve interleaved, for kernels that
  // cannot keep the whole tE live (v1, v2, v3)
  static __device__ __forceinline__ void uncouple_from(const double (&pw)[N - 1], const double (&ed)[h][D],
                                                       const double (&L)[m][m], const double (&inv)[m],
                                                       double (&rhs)[m][D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double t[m];
#pragma unroll
      for (int a = 0; a < m; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < m; ++b) s = fma(pw[a + b + 2] * G::at(1 + a, h + 1 + b), ed[1 + b][d], s);
        t[a] = s;
      }
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = t[j];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], t[k], s);
        t[j] = s * inv[j];
        rhs[j][d] -= t[j];
      }
    }
  }
  // rhs <- y - L^-1 tE
  static __device__ __forceinline__ void uncouple(const double (&L)[m][m], const double (&inv)[m],
                                                  const double (&tE)[m][D], double (&rhs)[m][D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double t[m];
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = tE[j][d];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], t[k], s);
        t[j] = s * inv[j];
        rhs[j][d] -= t[j];
      }
    }
  }
  // u_v = L^-T rhs; sd = [xv; u_v]
  static __device__ __forceinline__ void solve_back(const double (&L)[m][m], const double (&inv)[m],
                                                    const double (&rhs)[m][D], const double (&xv)[D],
                                                    double (&sd)[h][D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
#pragma unroll
      for (int j = m - 1; j >= 0; --j) {
        double s = rhs[j][d];
#pragma unroll
        for (int k = j + 1; k < m; ++k) s = fma(-L[k][j], sd[1 + k][d], s);
        sd[1 + j][d] = s * inv[j];
      }
      sd[0][d] = xv[d];
    }
  }

 private:
  template <bool kBcar>
  static __device__ __forceinline__ void assemble_impl(const double (&pw)[N - 1], const double (&Cee)[m][m],
                                                       const double (&cps)[m], const double (&cpe)[m],
                                                       const double (*bcar)[D], const double (&Wp)[m][m],
                                                       const double (&yp)[m][D], const double (&xm)[D],
                                                       const double (&xc)[D], const double (&xn)[D],
                                                       double (&Dp)[m][m], double (&E)[m][m], double (&bb)[m][D]) {
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        double s = fma(pw[a + b + 2], G::at(1 + a, 1 + b), Cee[a][b]);
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], Wp[k][b], s);
        Dp[a][b] = s;
      }
#pragma unroll
      for (int b = 0; b < m; ++b) E[a][b] = pw[a + b + 2] * G::at(1 + a, h + 1 + b);
      const double gmid = fma(pw[a + 1], G::at(1 + a, 0), cpe[a]);
      const double gnext = pw[a + 1] * G::at(1 + a, h);
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double s;
        if constexpr (kBcar) {
          s = bcar[a][d];
          s = fma(-cps[a], xm[d], s);
        } else {
          s = -cps[a] * xm[d];
        }
        s = fma(-gmid, xc[d], s);
        s = fma(-gnext, xn[d], s);
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
        bb[a][d] = s;
      }
    }
  }

  template <bool kBcar>
  static __device__ __forceinline__ void middle_impl(const double (&Cee)[m][m], const double (&cps)[m],
                                                     const double (&cpe)[m], const double (*bcar)[D],
                                                     const double (&Wp)[m][m], const double (&yp)[m][D],
                                                     const double (&xm)[D], const double (&xc)[D],
                                                     double (&um)[m][D], int& stat) {
    double Dl[m][m], bl[m][D];
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        double s = Cee[a][b];
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], Wp[k][b], s);
        Dl[a][b] = s;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double s;
        if constexpr (kBcar) {
          s = bcar[a][d];
          s = fma(-cps[a], xm[d], s);
        } else {
          s = -cps[a] * xm[d];
        }
        s = fma(-cpe[a], xc[d], s);
#pragma unroll
        for (int k = 0; k < m; ++k) s = fma(-Wp[k][a], yp[k][d], s);
        bl[a][d] = s;
      }
    }
#pragma unroll
    for (int a = 0; a < m; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        const double o = __shfl_xor_sync(kFull, Dl[a][b], 1);
        Dl[a][b] += ((a + b) & 1) ? -o : o;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const double o = __shfl_xor_sync(kFull, bl[a][d], 1);
        bl[a][d] += (a & 1) ? o : -o;  // derivative order a+1: sign (-1)^(a+1)
      }
    }
    stat |= __shfl_xor_sync(kFull, stat, 1);
    double L[m][m], inv[m];
    cholesky(Dl, L, inv, stat);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double y[m];
#pragma unroll
      for (int j = 0; j < m; ++j) {
        double s = bl[j][d];
#pragma unroll
        for (int k = 0; k < j; ++k) s = fma(-L[j][k], y[k], s);
        y[j] = s * inv[j];
      }
#pragma unroll
      for (int j = m - 1; j >= 0; --j) {
        double s = y[j];
#pragma unroll
        for (int k = j + 1; k < m; ++k) s = fma(-L[k][j], um[k][d], s);
        um[j][d] = s * inv[j];
      }
    }
  }
};

// Hermite-form emission of one segment from its start derivatives sd and end derivatives ed ([h][D]).  flip: the lane
// works in the time-reversed frame, so the original segment starts at its own end vertex (start = J ed, end = J sd,
// J folded into the time powers).
template <int N, class AI>
struct Hermite {
  static constexpr int h = N / 2;
  // tp[k] = (+-T)^k, itp[k] = iT^(h+k)
  static __device__ __forceinline__ void powers(double T, double iT, bool flip, double (&tp)[h], double (&itp)[h]) {
    const double Ts = flip ? -T : T;
    tp[0] = 1.0;
#pragma unroll
    for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * Ts;
    itp[0] = pow_int<h>(iT);
#pragma unroll
    for (int k = 1; k < h; ++k) itp[k] = itp[k - 1] * iT;
  }
  // the N coefficients of dimension d
  template <int D>
  static __device__ __forceinline__ void coeffs(bool flip, const double (&tp)[h], const double (&itp)[h],
                                                const double (&sd)[h][D], const double (&ed)[h][D], int d,
                                                double (&c)[N]) {
    double ss[h], se[h];
#pragma unroll
    for (int k = 0; k < h; ++k) {
      const double s0 = flip ? ed[k][d] : sd[k][d];
      const double e0 = flip ? sd[k][d] : ed[k][d];
      c[k] = s0 * ((flip && (k & 1)) ? -AI::at(k, k) : AI::at(k, k));
      ss[k] = tp[k] * s0;
      se[k] = tp[k] * e0;
    }
    // Upper coefficients in Hermite form: A(1)^-1 = [[L^-1, 0], [-D^-1 C L^-1, D^-1]] and (C L^-1)[k][j] =
    // 1/(j-k)! (derivative k of the Taylor part at tau = 1), so  q = D^-1 (se - C L^-1 ss):
    // h(h+1)/2 + h^2 operations instead of 2 h^2, and the 1/(j-k)! factors are mostly dyadic immediates.
    double ee[h];
#pragma unroll
    for (int k = 0; k < h; ++k) {
      double acc = se[k] - ss[k];
#pragma unroll
      for (int j = k + 1; j < h; ++j) {
        constexpr double kInvFact[6] = {1.0, 1.0, 0.5, 1.0 / 6.0, 1.0 / 24.0, 1.0 / 120.0};
        acc = (j - k == 1) ? acc - ss[j] : fma(-kInvFact[j - k], ss[j], acc);
      }
      ee[k] = acc;
    }
#pragma unroll
    for (int q = 0; q < h; ++q) {
      double acc = AI::at(h + q, h) * ee[0];
#pragma unroll
      for (int k = 1; k < h; ++k) acc = fma(AI::at(h + q, h + k), ee[k], acc);
      c[h + q] = acc * itp[q];
    }
  }
};

}  // namespace sweep
}  // namespace mtg
