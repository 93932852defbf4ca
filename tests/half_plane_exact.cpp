// half_plane_exact.cpp -- replay of FeasibilityBase::checkHalfPlaneFeasibility with binary128 roots and values: the
// exact reference for mtg_half_plane_feasibility_batch_f64.  TEST INFRASTRUCTURE ONLY (tests/half_plane_oracle.py);
// never linked by the product.
//
// Per segment and plane, in order: the projection n . p(t) is formed in fp64 in the reference's order
// (c_j = ((x_j n_0) + y_j n_1) + z_j n_2), the real roots in [0, T] of its derivative are isolated in binary128 with the
// Taylor-bound subdivision of extrema_exact.cpp, and d(t) = (p(t) - q) . n is evaluated in binary128 at 0, T and those
// roots.  A value <= 0 fails the plane.
//
// Per row it also returns a margin: over the visited (segment, plane) pairs, the smallest |min_t d(t)| relative to the
// scale S(t) = sum_d |n_d| (sum_j |c_dj| t^j + |q_d|) at the minimiser, less the fp64 evaluation's error factor
// (2N + 4) 2^-52.  A row whose margin is positive is decided identically by any evaluation within that forward error.
#include "extrema_exact.cpp"

#include <cfloat>
#include <limits>

namespace {

struct PlaneCheck {
  int N;
  const double* c;  // [D][N]
  double T;
  const double* pl;  // point[3], normal[3]

  double err_factor() const { return (2.0 * N + 4.0) * std::ldexp(1.0, -52); }

  Q distance(Q t) const {
    Q s = 0;
    for (int d = 0; d < 3; ++d) {
      std::vector<Q> p(N);
      for (int j = 0; j < N; ++j) p[j] = Q(c[d * N + j]);
      s += Q(pl[3 + d]) * (horner(p, t) - Q(pl[d]));
    }
    return s;
  }

  double scale(double t) const {
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
      double acc = 0.0;
      for (int j = N - 1; j >= 0; --j) acc = acc * t + std::abs(c[d * N + j]);
      s += std::abs(pl[3 + d]) * (acc + std::abs(pl[d]));
    }
    return s;
  }

  // true when the plane passes; *margin gets the pair's relative margin
  bool run(double* margin) const {
    volatile double n0 = pl[3], n1 = pl[4], n2 = pl[5];  // no contraction: the reference's separate roundings
    std::vector<Q> g(N > 1 ? N - 1 : 1, Q(0));
    for (int j = 1; j < N; ++j) {
      volatile double x = c[j] * n0, y = c[N + j] * n1, z = c[2 * N + j] * n2;
      volatile double xy = x + y;
      const double cj = xy + z;
      g[j - 1] = Q(double(j)) * Q(cj);
    }
    bool finite = true;  // a NaN or infinite derivative: every interior value is NaN or infinite too
    for (const Q& x : g) finite = finite && double(x) == double(x) && std::isfinite(double(x));
    std::vector<Q> roots;
    if (finite) real_roots(g, Q(T), &roots);
    std::vector<Q> times = {Q(0), Q(T)};
    times.insert(times.end(), roots.begin(), roots.end());
    bool pass = true;
    Q lo = 0;
    Q t_lo = 0;
    for (size_t q = 0; q < times.size(); ++q) {
      const Q v = distance(times[q]);
      if (v <= 0) pass = false;  // NaN passes, as in the reference
      if (q == 0 || v < lo) {
        lo = v;
        t_lo = times[q];
      }
    }
    const double s = scale(double(t_lo));
    *margin = (s > 0 ? double(qabs(lo)) / s : std::numeric_limits<double>::infinity()) - err_factor();
    return pass;
  }
};


// Which step of the GPU kernel decides this (segment, plane), with its fp64 arithmetic replayed: 1 = d(0) or d(T) <= 0,
// 2 = the Bernstein shortcut, 4 = the root isolation.  (The bound's scale S may differ from the kernel's in its last
// bits where nvcc contracts, so a pair right at the bound can be classified differently; only used for statistics.)
int kernel_path(int N, double T, const double* c, const double* pl) {
  auto dist = [&](double t) {
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
      volatile double acc = c[d * N + N - 1];
      for (int j = N - 2; j >= 0; --j) {
        volatile double m = acc * t;
        acc = m + c[d * N + j];
      }
      volatile double e = acc - pl[d];
      volatile double m = e * pl[3 + d];
      s = d == 0 ? double(m) : double(s + m);
    }
    return s;
  };
  const double d0 = dist(0.0);
  if (d0 <= 0.0 || dist(T) <= 0.0) return 1;
  std::vector<double> a(N);
  a[0] = d0;
  double S = std::abs(pl[3] * pl[0]) + std::abs(pl[4] * pl[1]) + std::abs(pl[5] * pl[2]);
  double tp = 1.0;
  for (int j = 0; j < N; ++j) {
    const double x = c[j], y = c[N + j], z = c[2 * N + j];
    S += (std::abs(pl[3] * x) + std::abs(pl[4] * y) + std::abs(pl[5] * z)) * tp;
    if (j > 0) {
      volatile double px = x * pl[3], py = y * pl[4], pz = z * pl[5];
      volatile double sxy = px + py;
      volatile double cj = sxy + pz;
      a[j] = cj * tp;
    }
    if (j < N - 1) tp *= T;
  }
  const double E = (8.0 * N + 16.0) * std::ldexp(1.0, -53) * S +
                   DBL_MIN * (1.0 + tp) * (1.0 + std::abs(pl[3]) + std::abs(pl[4]) + std::abs(pl[5]));
  const int n = N - 1;
  bool clear = true;
  for (int i = 0; i <= n; ++i) {
    double s = a[0];
    for (int j = 1; j <= i; ++j) {
      double w = 1.0;
      for (int q = 0; q < j; ++q) w = w * double(i - q) / double(n - q);
      s = std::fma(w, a[j], s);
    }
    clear = clear && s > E;
  }
  return clear ? 2 : 4;
}

}  // namespace

extern "C" {

// times [B][K], coeffs [B][K][D][N], planes [P][6] (point, normal, used as given) -> feasible [B] (1 / 0), segment [B]
// and plane [B] (the first failing pair, -1 when none), margin [B], paths [B] (the OR of kernel_path over the visited
// pairs).  D not 3 or 4: feasible 0, segment 0, plane -1.
// A row with a segment time <= 0 or non-finite: feasible 0, segment and plane -1, margin +inf.  Returns 0, or -1 on
// a bad argument.
int exact_half_plane(int N, int K, int D, int64_t B, const double* times, const double* coeffs, int P,
                     const double* planes, int32_t* feasible, int32_t* segment, int32_t* plane, double* margin,
                     int32_t* paths, int n_threads) {
  if (N < 1 || N > 12 || K < 1 || D < 1 || B < 0 || P < 0) return -1;
  std::atomic<int64_t> next(0);
  auto work = [&]() {
    for (int64_t b = next++; b < B; b = next++) {
      bool bad = false;
      for (int i = 0; i < K; ++i) {
        const double T = times[b * K + i];
        if (!(T > 0.0) || !std::isfinite(T)) bad = true;
      }
      feasible[b] = 1;
      segment[b] = plane[b] = -1;
      paths[b] = 0;
      margin[b] = std::numeric_limits<double>::infinity();
      if (bad) {
        feasible[b] = 0;
        continue;
      }
      for (int i = 0; i < K && feasible[b]; ++i) {
        if (D != 3 && D != 4) {
          feasible[b] = 0;
          segment[b] = i;
          break;
        }
        for (int p = 0; p < P; ++p) {
          PlaneCheck pc{N, coeffs + (size_t(b) * K + i) * D * N, times[b * K + i], planes + 6 * p};
          double m;
          const bool pass = pc.run(&m);
          margin[b] = std::min(margin[b], m);
          paths[b] |= kernel_path(N, times[b * K + i], coeffs + (size_t(b) * K + i) * D * N, planes + 6 * p);
          if (!pass) {
            feasible[b] = 0;
            segment[b] = i;
            plane[b] = p;
            break;
          }
        }
      }
    }
  };
  const int nt = n_threads > 1 ? n_threads : 1;
  std::vector<std::thread> pool;
  for (int i = 1; i < nt; ++i) pool.emplace_back(work);
  work();
  for (auto& th : pool) th.join();
  return 0;
}

// The shortcut's bound, checked exactly: for one segment and plane, the fp64 Bernstein coefficients b of d(tau T) on
// [0, 1] and the bound E computed as the kernel computes them, the exact minimum of d over the roots and end points, and
// the largest |fp64 reference-arithmetic value - exact value| over `n_t` given times in [0, T].  out: [0] min b,
// [1] E, [2] exact minimum of d on [0, T], [3] largest evaluation error, [4] largest |b_fp64 - b_exact|.
void exact_half_plane_bound(int N, double T, const double* c, const double* pl, int n_t, const double* ts,
                            double* out) {
  PlaneCheck pc{N, c, T, pl};
  auto fp64_distance = [&](double t) {
    volatile double s = 0.0;
    for (int d = 0; d < 3; ++d) {
      volatile double acc = c[d * N + N - 1];
      for (int j = N - 2; j >= 0; --j) {
        volatile double m = acc * t;
        acc = m + c[d * N + j];
      }
      volatile double e = acc - pl[d];
      volatile double m = e * pl[3 + d];
      s = d == 0 ? double(m) : double(s + m);
    }
    return double(s);
  };
  // the kernel's coefficients: a_0 = d(0) computed, a_j = c_j T^j
  std::vector<double> a(N);
  std::vector<Q> ae(N);
  a[0] = fp64_distance(0.0);
  ae[0] = pc.distance(Q(0));
  double S = std::abs(pl[3] * pl[0]) + std::abs(pl[4] * pl[1]) + std::abs(pl[5] * pl[2]);
  double tp = 1.0;
  Q tq = 1;
  for (int j = 0; j < N; ++j) {
    const double x = c[j], y = c[N + j], z = c[2 * N + j];
    S += (std::abs(pl[3] * x) + std::abs(pl[4] * y) + std::abs(pl[5] * z)) * tp;
    if (j > 0) {
      volatile double px = x * pl[3], py = y * pl[4], pz = z * pl[5];
      volatile double sxy = px + py;
      volatile double cj = sxy + pz;
      volatile double aj = cj * tp;
      a[j] = aj;
      ae[j] = (Q(x) * Q(pl[3]) + Q(y) * Q(pl[4]) + Q(z) * Q(pl[5])) * tq;
    }
    if (j < N - 1) {
      tp *= T;
      tq *= Q(T);
    }
  }
  const double u = std::ldexp(1.0, -53);
  const double E = (8.0 * N + 16.0) * u * S + DBL_MIN * (1.0 + tp) * (1.0 + std::abs(pl[3]) + std::abs(pl[4]) +
                                                                      std::abs(pl[5]));
  // power -> Bernstein on [0, 1] as extrema_bernstein (fma chains over the same weights)
  const int n = N - 1;
  double bmin = std::numeric_limits<double>::infinity(), berr = 0.0;
  for (int i = 0; i <= n; ++i) {
    double s = a[0];
    Q se = ae[0];
    for (int j = 1; j <= i; ++j) {
      double w = 1.0;
      for (int q = 0; q < j; ++q) w = w * double(i - q) / double(n - q);
      s = std::fma(w, a[j], s);
      Q we = 1;
      for (int q = 0; q < j; ++q) we = we * Q(double(i - q)) / Q(double(n - q));
      se += we * ae[j];
    }
    bmin = std::min(bmin, s);
    berr = std::max(berr, double(qabs(Q(s) - se)));
  }
  // exact minimum over 0, T and the roots of the exact derivative
  std::vector<Q> g(N > 1 ? N - 1 : 1, Q(0));
  for (int j = 1; j < N; ++j) g[j - 1] = Q(double(j)) * ae[j];
  std::vector<Q> roots;
  real_roots(g, Q(1), &roots);
  Q mn = pc.distance(Q(0));
  const Q dT = pc.distance(Q(T));
  if (dT < mn) mn = dT;
  for (const Q& r : roots) {
    const Q v = pc.distance(r * Q(T));
    if (v < mn) mn = v;
  }
  double eerr = 0.0;
  for (int k = 0; k < n_t; ++k) eerr = std::max(eerr, double(qabs(Q(fp64_distance(ts[k])) - pc.distance(Q(ts[k])))));
  out[0] = bmin;
  out[1] = E;
  out[2] = double(mn);
  out[3] = eerr;
  out[4] = berr;
}

}  // extern "C"
