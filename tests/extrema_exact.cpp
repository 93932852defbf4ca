// extrema_exact.cpp -- binary128 maximum of |p^(k)(t)| over every segment of a trajectory: the exact reference for
// mtg_max_magnitude_batch_f64.  TEST INFRASTRUCTURE ONLY (tests/extrema_oracle.py); never linked by the product.
//
// For each segment the critical polynomial of the given fp64 coefficients, sum_d p_d^(k) p_d^(k+1) (p^(k+1) for
// D = 1), is formed in binary128 (a product of two doubles is exact there; the integer derivative factors cost at most
// one rounding at 2^-113).  Its real roots in [0, T] are isolated by interval subdivision with Taylor bounds taken at
// each interval's midpoint m with radius r:
//   |g(m)| > sum_{j>=1} |g^(j)(m)/j!| r^j       -> no root in the interval;
//   |g'(m)| > sum_{j>=2} j |g^(j)(m)/j!| r^(j-1) -> g is monotone there: at most one root, found by bisection.
// An interval that is neither and narrower than 1e-22 T (a multiple or clustered root) contributes its midpoint.
// This is a different method from the kernel's (Bernstein coefficients, Descartes' rule, Newton) on purpose.
// Candidates are 0, T and the roots; values are evaluated in binary128 and rounded once.
#include <stdint.h>

#include <atomic>
#include <cmath>
#include <thread>
#include <vector>

namespace {

typedef __float128 Q;

inline Q qabs(Q x) { return x < 0 ? -x : x; }

double base_coeff(int k, int j) {  // j! / (j - k)!
  if (j < k) return 0.0;
  double v = 1.0;
  for (int q = 0; q < k; ++q) v *= double(j - q);
  return v;
}

Q horner(const std::vector<Q>& c, Q x) {
  Q a = 0;
  for (int j = int(c.size()) - 1; j >= 0; --j) a = a * x + c[j];
  return a;
}

// Taylor coefficients g^(j)(m) / j! by repeated synthetic division
std::vector<Q> taylor(std::vector<Q> c, Q m) {
  const int n = int(c.size()) - 1;
  for (int i = 0; i < n; ++i)
    for (int j = n - 1; j >= i; --j) c[j] += m * c[j + 1];
  return c;
}

void real_roots(std::vector<Q> g, Q T, std::vector<Q>* roots) {
  while (!g.empty() && g.back() == 0) g.pop_back();
  if (g.size() < 2) return;
  const int n = int(g.size()) - 1;
  const Q min_width = T * Q(1e-22);
  std::vector<std::pair<Q, Q>> stack = {{Q(0), T}};
  while (!stack.empty()) {
    const Q a = stack.back().first, b = stack.back().second;
    stack.pop_back();
    const Q m = (a + b) / 2, r = (b - a) / 2;
    const std::vector<Q> t = taylor(g, m);
    Q s1 = 0, s2 = 0, rp = r;
    for (int j = 1; j <= n; ++j) {
      s1 += qabs(t[j]) * rp;
      if (j >= 2) s2 += Q(j) * qabs(t[j]) * (rp / r);
      rp *= r;
    }
    if (qabs(t[0]) > s1) continue;
    if (qabs(t[1]) > s2) {
      const Q ga = horner(g, a), gb = horner(g, b);
      if (ga == 0) roots->push_back(a);
      if (gb == 0) roots->push_back(b);
      if ((ga < 0 && gb > 0) || (ga > 0 && gb < 0)) {
        Q lo = a, hi = b;
        for (int it = 0; it < 240 && hi - lo > 0; ++it) {
          const Q mid = (lo + hi) / 2;
          if (mid <= lo || mid >= hi) break;
          const Q gm = horner(g, mid);
          if (gm == 0) {
            lo = hi = mid;
            break;
          }
          if ((gm < 0) == (ga < 0)) lo = mid;
          else hi = mid;
        }
        roots->push_back((lo + hi) / 2);
      }
      continue;
    }
    if (b - a < min_width) {
      roots->push_back(m);
      continue;
    }
    stack.emplace_back(m, b);
    stack.emplace_back(a, m);
  }
}

struct SegmentPolys {
  std::vector<std::vector<Q>> pk;  // [D] p_d^(k), power basis in t
};

Q magnitude_sq(const SegmentPolys& s, Q t) {
  Q sq = 0;
  for (const auto& p : s.pk) {
    const Q v = horner(p, t);
    sq += v * v;
  }
  return sq;
}

double qsqrt_to_double(Q x) {
  if (x <= 0) return 0.0;
  Q y = std::sqrt(double(x));
  y = (y + x / y) / 2;  // one Newton step from the fp64 root: binary128 accurate
  return double(y);
}

// Horner forward-error scale of the fp64 evaluation: sum_d sum_j |B(k,j) c_dj| t^(j-k)
double horner_scale(const SegmentPolys& s, double t) {
  double total = 0.0;
  for (const auto& p : s.pk) {
    double acc = 0.0;
    for (int j = int(p.size()) - 1; j >= 0; --j) acc = acc * t + double(qabs(p[j]));
    total += acc;
  }
  return total;
}

}  // namespace

extern "C" {

// times [B][K], coeffs [B][K][D][N] -> per trajectory: value, time (in segment), segment of the maximum of |p^(k)|,
// runner_up (largest candidate value more than 1e-6 T away from the maximiser or in another segment; -1 if none) and
// scale (the Horner forward-error scale at the maximiser).  Trajectories with a segment time <= 0 or non-finite get
// value NaN.  Returns 0, or -1 on a bad argument.
int exact_max_magnitude(int N, int K, int D, int64_t B, const double* times, const double* coeffs, int k, double* value,
                        double* time, int32_t* segment, double* runner_up, double* scale, int n_threads) {
  if (N < 2 || N > 12 || k < 0 || k > N - 2 || K < 1 || D < 1 || B < 0) return -1;
  std::atomic<int64_t> next(0);
  auto work = [&]() {
    for (int64_t b = next++; b < B; b = next++) {
      struct Cand {
        double t;
        Q v2;
        int seg;
      };
      std::vector<Cand> cands;
      bool bad = false;
      std::vector<SegmentPolys> polys(K);
      for (int i = 0; i < K; ++i) {
        const double T = times[b * K + i];
        if (!(T > 0.0) || !std::isfinite(T)) {
          bad = true;
          break;
        }
        const double* c = coeffs + (size_t(b) * K + i) * D * N;
        SegmentPolys& s = polys[i];
        s.pk.assign(D, std::vector<Q>(N - k, Q(0)));
        std::vector<Q> g(D == 1 ? N - k - 1 : 2 * (N - k) - 2, Q(0));
        for (int d = 0; d < D; ++d) {
          for (int j = 0; j < N - k; ++j) s.pk[d][j] = Q(base_coeff(k, j + k)) * Q(c[d * N + j + k]);
          std::vector<Q> p1(N - k - 1);
          for (int j = 0; j < N - k - 1; ++j) p1[j] = Q(base_coeff(k + 1, j + k + 1)) * Q(c[d * N + j + k + 1]);
          if (D == 1) {
            g = p1;
          } else {
            for (int a = 0; a < N - k; ++a)
              for (int j = 0; j < N - k - 1; ++j) g[a + j] += s.pk[d][a] * p1[j];
          }
        }
        std::vector<Q> roots;
        real_roots(g, Q(T), &roots);
        cands.push_back({0.0, magnitude_sq(s, 0), i});
        cands.push_back({T, magnitude_sq(s, Q(T)), i});
        for (const Q& r : roots) cands.push_back({double(r), magnitude_sq(s, r), i});
      }
      if (bad) {
        value[b] = time[b] = runner_up[b] = scale[b] = NAN;
        segment[b] = -1;
        continue;
      }
      size_t best = 0;
      Q best_v2 = 0;
      bool any = false;
      for (size_t q = 0; q < cands.size(); ++q)
        if (cands[q].v2 > best_v2) {
          best_v2 = cands[q].v2;
          best = q;
          any = true;
        }
      if (!any) {  // Extremum(): every value is 0
        value[b] = 0.0;
        time[b] = 0.0;
        segment[b] = 0;
        runner_up[b] = -1.0;
        scale[b] = 0.0;
        continue;
      }
      const Cand& w = cands[best];
      const double Tw = times[b * K + w.seg];
      Q second = -1;
      for (const Cand& c : cands)
        if (c.seg != w.seg || std::abs(c.t - w.t) > 1e-6 * Tw)
          if (c.v2 > second) second = c.v2;
      value[b] = qsqrt_to_double(best_v2);
      time[b] = w.t;
      segment[b] = w.seg;
      runner_up[b] = second < 0 ? -1.0 : qsqrt_to_double(second);
      scale[b] = horner_scale(polys[w.seg], w.t);
    }
  };
  const int nt = n_threads > 1 ? n_threads : 1;
  std::vector<std::thread> pool;
  for (int i = 1; i < nt; ++i) pool.emplace_back(work);
  work();
  for (auto& th : pool) th.join();
  return 0;
}

}  // extern "C"
