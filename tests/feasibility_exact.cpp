// feasibility_exact.cpp -- replay of FeasibilityAnalytic::checkInputFeasibilityTrajectory with binary128 roots and
// values: the exact reference for mtg_input_feasibility_batch_f64.  TEST INFRASTRUCTURE ONLY
// (tests/feasibility_oracle.py); never linked by the product.
//
// The critical polynomials (thrust sum_d f_d f_d' with f = p'' + (0, 0, g), speed and jerk sum_d p_d^(k) p_d^(k+1) over
// dims 0..2, yaw'' and yaw''') are formed in binary128 from the fp64 coefficients, and their real roots in [0, T] are
// isolated with the Taylor-bound subdivision of extrema_exact.cpp (an unresolved interval narrower than 1e-22 T
// contributes its midpoint).  Candidates are 0, T and those roots; values are binary128.  The roll/pitch interval walk
// runs in fp64 exactly as the reference does ((t1 + t2) / 2, t2 - t1 < min_section_time), comparing binary128
// candidate times and values against it.
//
// Per row it also returns a decision margin: the smallest relative gap of any comparison the replay made -- each value
// against its limit, the bound against omega_xy_max at every visited node, f_min against 1e-6, and the time of every
// root whose side of a visited boundary moves that interval's f_min or j_max, against that boundary (relative to T) --
// and an error scale: the largest Horner
// forward-error scale sum_j |a_j| t^j (over the compared candidates, relative to the limit).  A row whose margin is
// well above u times its scale is decided identically by any evaluation within that forward error.
#include "extrema_exact.cpp"

#include <cfloat>
#include <limits>

namespace {

struct Cand {
  Q t, v;
  double scale;  // forward-error scale of v: sum_d sum_j |a_dj| t^j
  bool root;     // false for the end points 0 and T, which both implementations take exactly
};

struct Checker {
  int N, D;
  const double* c;  // [D][N]
  double T;
  Q TQ;
  uint32_t present;
  const double* lim;  // [6]
  double gravity, mst;
  double margin = std::numeric_limits<double>::infinity();

  double err_factor() const { return (4.0 * N + 16.0) * std::ldexp(1.0, -52); }

  // relative gap of a against b (reference |ref|), less err (already relative)
  void gap(Q a, Q b, Q ref, double err = 0.0) {
    ref = qabs(ref);
    if (ref == 0) ref = 1;
    const double g = double(qabs(a - b) / ref) - err;
    if (g < margin) margin = g;
  }

  // p_d^(k) of dims [d0, d0 + nd) (power basis in t), thrust: + gravity on dim 2
  std::vector<std::vector<Q>> polys(int d0, int nd, int k, bool thrust) const {
    std::vector<std::vector<Q>> p(nd, std::vector<Q>(N - k, Q(0)));
    for (int d = 0; d < nd; ++d)
      for (int j = 0; j < N - k; ++j) p[d][j] = Q(base_coeff(k, j + k)) * Q(c[(d0 + d) * N + j + k]);
    if (thrust) p[2][0] += Q(gravity);
    return p;
  }

  static std::vector<Q> deriv(const std::vector<Q>& p) {
    std::vector<Q> q(p.size() > 1 ? p.size() - 1 : 1, Q(0));
    for (size_t j = 1; j < p.size(); ++j) q[j - 1] = Q(double(j)) * p[j];
    return q;
  }

  // candidates of |p| (nd = 3: magnitude over the dims; nd = 1: |p| of the one polynomial)
  std::vector<Cand> candidates(const std::vector<std::vector<Q>>& p) const {
    std::vector<Q> g;
    if (p.size() == 1) {
      g = deriv(p[0]);
    } else {
      g.assign(2 * p[0].size(), Q(0));
      for (const auto& pd : p) {
        const std::vector<Q> dp = deriv(pd);
        for (size_t a = 0; a < pd.size(); ++a)
          for (size_t j = 0; j < dp.size(); ++j) g[a + j] += pd[a] * dp[j];
      }
    }
    std::vector<Q> roots;
    real_roots(g, TQ, &roots);
    std::vector<Q> times = {Q(0), TQ};
    times.insert(times.end(), roots.begin(), roots.end());
    std::vector<Cand> out;
    for (size_t q = 0; q < times.size(); ++q) {
      const Q t = times[q];
      Q sq = 0;
      double s = 0.0;
      for (const auto& pd : p) {
        const Q v = horner(pd, t);
        sq += v * v;
        double acc = 0.0;
        for (int j = int(pd.size()) - 1; j >= 0; --j) acc = acc * double(t) + double(qabs(pd[j]));
        s += acc;
      }
      Q v = sq > 0 ? Q(qsqrt_to_double(sq)) : Q(0);
      if (sq > 0) v = (v + sq / v) / 2;  // binary128 sqrt: one Newton step from the fp64 root
      out.push_back({t, v, s, q >= 2 && t != 0 && t != TQ});  // a root on an end point repeats that end point
    }
    return out;
  }

  // the largest value, and the forward error of any candidate's evaluation relative to `limit`
  Q max_of(const std::vector<Cand>& cs, double limit, double* err) const {
    Q m = cs[0].v;
    double s = 0.0;
    for (const Cand& x : cs) {
      if (x.v > m) m = x.v;
      s = std::max(s, x.scale);
    }
    *err = limit > 0 ? err_factor() * s / limit : 0.0;
    return m;
  }

  int run() {
    if (D != 3 && D != 4) return 1;
    std::vector<Cand> th, jk;
    const bool thrust = present & (1u | 2u | 8u);
    if (thrust) {
      th = candidates(polys(0, 3, 2, true));
      Q lo = th[0].v, hi = th[0].v;
      for (const Cand& x : th) {
        lo = x.v < lo ? x.v : lo;
        hi = x.v > hi ? x.v : hi;
      }
      double err;
      if (present & 1u) {
        max_of(th, lim[0], &err);
        gap(lo, Q(lim[0]), Q(lim[0]), err);
        if (lo < Q(lim[0])) return 3;
      }
      if (present & 2u) {
        max_of(th, lim[1], &err);
        gap(hi, Q(lim[1]), Q(lim[1]), err);
        if (hi > Q(lim[1])) return 2;
      }
    }
    if (present & 4u) {
      const std::vector<Cand> v = candidates(polys(0, 3, 1, false));
      double err;
      const Q m = max_of(v, lim[2], &err);
      gap(m, Q(lim[2]), Q(lim[2]), err);
      if (m > Q(lim[2])) return 4;
    }
    if (D == 4) {
      for (int q = 0; q < 2; ++q) {
        if (!(present & (16u << q))) continue;
        const std::vector<Cand> y = candidates(polys(3, 1, 1 + q, false));
        double err;
        const Q m = max_of(y, lim[4 + q], &err);
        gap(m, Q(lim[4 + q]), Q(lim[4 + q]), err);
        if (m > Q(lim[4 + q])) return 6 + q;
      }
    }
    if (!(present & 8u)) return 0;
    jk = candidates(polys(0, 3, 3, false));
    return walk(th, jk, 0.0, T);
  }

  // recursiveRollPitchFeasibility (recursion depth is at most ~log2(T / min_section_time) + 2)
  int walk(const std::vector<Cand>& th, const std::vector<Cand>& jk, double t1, double t2) {
    if (t2 - t1 < mst) return 1;
    // a root's side of a boundary matters only where its membership moves the interval's extreme by more than 1e-12
    // of the list's largest value (below any evaluation error): a root in a cluster at an end point repeats that end
    // point, and a jerk root next to a zero-jerk end point is zero to rounding
    for (int list = 0; list < 2; ++list) {
      const std::vector<Cand>& xs = list == 0 ? th : jk;
      Q top = 0;
      for (const Cand& x : xs) top = x.v > top ? x.v : top;
      for (size_t q = 0; q < xs.size(); ++q) {
        const Cand& x = xs[q];
        if (!x.root) continue;
        bool any = false;
        Q ext = 0;
        for (size_t o = 0; o < xs.size(); ++o) {
          if (o == q || xs[o].t < Q(t1) || xs[o].t > Q(t2)) continue;
          if (!any || (list == 0 ? xs[o].v < ext : xs[o].v > ext)) ext = xs[o].v;
          any = true;
        }
        const Q tol = top * Q(1e-12);
        if (any && (list == 0 ? !(x.v < ext - tol) : !(x.v > ext + tol))) continue;
        gap(x.t, Q(t1), TQ);
        gap(x.t, Q(t2), TQ);
      }
    }
    Q f_min = Q(DBL_MAX), j_max = Q(std::numeric_limits<double>::lowest());
    bool any_f = false, any_j = false;
    double s_f = 0.0, s_j = 0.0;
    for (const Cand& x : th)
      if (!(x.t < Q(t1) || x.t > Q(t2)) && x.v < f_min) {
        f_min = x.v;
        s_f = x.scale;
        any_f = true;
      }
    for (const Cand& x : jk)
      if (!(x.t < Q(t1) || x.t > Q(t2)) && x.v > j_max) {
        j_max = x.v;
        s_j = x.scale;
        any_j = true;
      }
    const double limit = lim[3];
    bool split;
    if (any_f) gap(f_min, Q(1.0e-6), Q(1.0e-6), err_factor() * s_f / 1.0e-6);
    if (!(f_min > Q(1.0e-6))) {
      split = DBL_MAX > limit;
    } else if (!any_j) {
      split = false;  // sqrt of a negative number: NaN > limit is false
    } else {
      const Q r = j_max / f_min;
      Q b = r > 0 ? Q(std::sqrt(double(r))) : Q(0);
      if (r > 0) b = (b + r / b) / 2;
      // the bound's error from j_max and f_min each off by their forward error
      const double jq = double(j_max), fq = double(f_min);
      const double lo_f = std::max(fq - err_factor() * s_f, 1.0e-300);
      const double b_hi = std::sqrt((jq + err_factor() * s_j) / lo_f);
      const double b_lo = std::sqrt(std::max(jq - err_factor() * s_j, 0.0) / (fq + err_factor() * s_f));
      gap(b, Q(limit), Q(limit), std::max(b_hi - double(b), double(b) - b_lo) / limit);
      split = b > Q(limit);
    }
    if (!split) return 0;
    const double th_ = (t1 + t2) / 2;
    const int r1 = walk(th, jk, t1, th_);
    if (r1 != 0) return r1;
    return walk(th, jk, th_, t2);
  }
};

}  // namespace

extern "C" {

// times [B][K], coeffs [B][K][D][N], limits [6] (InputConstraintType order, used where `present` has the bit) ->
// result [B] (InputFeasibilityResult), segment [B] (-1: Feasible or a bad time), margin [B].  A row with a
// segment time <= 0 or non-finite: result 1, segment -1, margin +inf.  Returns 0, or -1 on a bad argument.
int exact_input_feasibility(int N, int K, int D, int64_t B, const double* times, const double* coeffs, uint32_t present,
                            const double* limits, double gravity, double min_section_time, int32_t* result,
                            int32_t* segment, double* margin, int n_threads) {
  if (N < 4 || N > 12 || K < 1 || D < 1 || B < 0 || !(min_section_time > 0)) return -1;
  std::atomic<int64_t> next(0);
  auto work = [&]() {
    for (int64_t b = next++; b < B; b = next++) {
      bool bad = false;
      for (int i = 0; i < K; ++i) {
        const double T = times[b * K + i];
        if (!(T > 0.0) || !std::isfinite(T)) bad = true;
      }
      result[b] = 0;
      segment[b] = -1;
      margin[b] = std::numeric_limits<double>::infinity();
      if (bad) {
        result[b] = 1;
        continue;
      }
      for (int i = 0; i < K; ++i) {
        Checker ck{N, D, coeffs + (size_t(b) * K + i) * D * N, times[b * K + i], Q(times[b * K + i]), present, limits,
                   gravity, min_section_time};
        const int r = ck.run();
        margin[b] = std::min(margin[b], ck.margin);
        if (r != 0) {
          result[b] = r;
          segment[b] = i;
          break;
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

}  // extern "C"
