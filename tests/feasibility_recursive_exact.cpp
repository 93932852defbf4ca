// feasibility_recursive_exact.cpp -- replay of FeasibilityRecursive::checkInputFeasibilityTrajectory with binary128
// roots: the exact reference for mtg_input_feasibility_recursive_batch_f64.  TEST INFRASTRUCTURE ONLY
// (tests/feasibility_recursive_oracle.py); never linked by the product.
//
// The real roots in [0, T] of p_i'', p_i''' and p_i'''' (i = 0..2) are isolated in binary128 with the Taylor-bound
// subdivision of extrema_exact.cpp, and each root's p_i^(k) is evaluated in binary128 and rounded once.  The section
// walk then runs in fp64 exactly as the reference does: (t1 + t2) / 2, t2 - t1 < min_section_time, end-point values by
// Polynomial::evaluate's Horner (separate multiply and add), squares as x * x, sums in axis order, one sqrt.  The
// yaw checks take 0, T and the binary128 roots of yaw'' / yaw''' with binary128 values.
//
// Per row it also returns a decision margin: the smallest relative gap of any comparison the replay made, less the
// forward error the compared values can carry.  Every fp64 quantity of the walk carries an error radius: 0 for what
// both sides compute bit for bit from the same inputs (end-point values and everything derived only from them), the
// Horner forward error (4N + 16) u sum_j |a_j| t^j for a root's value, propagated through min / max, squares, sums,
// sqrt and the division with one extra rounding per operation.  A comparison whose operands both have radius 0 is
// decided identically by both sides and does not count; the sign test f_i_min * f_i_max < 0 never counts, since where
// it is within rounding of 0 both of its branches add the same bound to within the radius.  The time of every root whose side of a visited section end
// moves that section's per-axis minimum or maximum counts too, as its distance to that end relative to T.
#include "extrema_exact.cpp"

#include <algorithm>
#include <cfloat>
#include <limits>

namespace {

const double kInf = std::numeric_limits<double>::infinity();
const double kUlp = std::ldexp(1.0, -52);

// an fp64 value as both sides compute it, and the radius within which the device's value lies
struct V {
  double v, e;
};

// one rounding of a result whose inputs were perturbed (nothing when they were not)
inline V rounded(double v, double e) { return {v, e > 0 ? e + kUlp * std::abs(v) : 0.0}; }
inline V sq(V x) { return rounded(x.v * x.v, 2.0 * std::abs(x.v) * x.e + x.e * x.e); }
inline V add(V a, V b) { return rounded(a.v + b.v, a.e + b.e); }
inline V vabs(V x) { return {std::abs(x.v), x.e}; }
inline V vmax(V a, V b) { return {a.v < b.v ? b.v : a.v, std::max(a.e, b.e)}; }  // std::max
inline V vmin(V a, V b) { return {b.v < a.v ? b.v : a.v, std::max(a.e, b.e)}; }  // std::min
inline V vsqrt(V x) {
  const double r = std::sqrt(x.v);
  return rounded(r, x.e > 0 ? (r > 0 ? std::min(std::sqrt(x.e), x.e / r) : std::sqrt(x.e)) : 0.0);
}

struct Root {
  Q t;
  double v, e;  // p_i^(k)(t) rounded once, and the device's evaluation error bound
};

struct Checker {
  int N, D;
  const double* c;  // [D][N]
  double T;
  Q TQ;
  uint32_t present;
  const double* lim;  // [6]
  double gravity, mst;
  double margin = kInf;
  std::vector<Root> roots[9];  // (order k = 1 + q / 3, axis q % 3)

  double err_factor() const { return (4.0 * N + 16.0) * kUlp; }

  // the relative gap of a against b (a limit or threshold), less both radii; +inf when both sides compute both
  // operands bit for bit
  static double gap(V a, V b, double ref) {
    const double e = a.e + b.e;
    if (e == 0) return kInf;
    ref = std::abs(ref) > 0 ? std::abs(ref) : 1.0;
    return (std::abs(a.v - b.v) - e) / ref;
  }
  void cmp(V a, V b, double ref) { margin = std::min(margin, gap(a, b, ref)); }
  void gap_q(Q a, Q b, Q ref, double err) {
    ref = qabs(ref);
    if (ref == 0) ref = 1;
    margin = std::min(margin, double(qabs(a - b) / ref) - err);
  }

  // Polynomial::evaluate(t, k) of dim d
  double ev(int d, int k, double t) const {
    if (k >= N) return 0.0;
    const double* a = c + d * N;
    double r = base_coeff(k, N - 1) * a[N - 1];
    for (int j = N - 2; j >= k; --j) {
      r = r * t;
      r = r + base_coeff(k, j) * a[j];
    }
    return r;
  }

  std::vector<Q> poly(int d, int k) const {  // p_d^(k), power basis in t
    std::vector<Q> p(N - k > 0 ? N - k : 1, Q(0));
    for (int j = 0; j < N - k; ++j) p[j] = Q(base_coeff(k, j + k)) * Q(c[d * N + j + k]);
    return p;
  }
  static std::vector<Q> deriv(const std::vector<Q>& p) {
    std::vector<Q> q(p.size() > 1 ? p.size() - 1 : 1, Q(0));
    for (size_t j = 1; j < p.size(); ++j) q[j - 1] = Q(double(j)) * p[j];
    return q;
  }
  static double scale(const std::vector<Q>& p, Q t) {
    double acc = 0.0;
    for (int j = int(p.size()) - 1; j >= 0; --j) acc = acc * double(t) + double(qabs(p[j]));
    return acc;
  }

  void find_roots(int q) {
    const int k = 1 + q / 3, i = q % 3;
    const std::vector<Q> p = poly(i, k);
    std::vector<Q> rs;
    real_roots(deriv(p), TQ, &rs);
    for (const Q& t : rs) roots[q].push_back({t, double(horner(p, t)), err_factor() * scale(p, t)});
  }

  int run() {
    if (D != 3 && D != 4) return 1;
    const bool need[3] = {(present & 4u) != 0, (present & (1u | 2u | 8u)) != 0, (present & 8u) != 0};
    for (int q = 0; q < 9; ++q)
      if (need[q / 3]) find_roots(q);
    const int r = walk(0.0, T);
    if (r != 0 || D != 4) return r;
    for (int q = 0; q < 2; ++q) {
      if (!(present & (16u << q))) continue;
      const std::vector<Q> p = poly(3, 1 + q);
      std::vector<Q> ts = {Q(0), TQ};
      real_roots(deriv(p), TQ, &ts);
      Q m = 0;
      double s = 0.0;
      for (const Q& t : ts) {
        m = std::max(m, qabs(horner(p, t)));
        s = std::max(s, scale(p, t));
      }
      const double limit = lim[4 + q];
      gap_q(m, Q(limit), Q(limit), limit > 0 ? err_factor() * s / limit : 0.0);
      if (m > Q(limit)) return 6 + q;
    }
    return 0;
  }

  // selectMinMaxFromRoots of list q on [t1, t2]: the end points (exact) and the roots inside
  void minmax(int q, double t1, double t2, V* lo, V* hi) {
    const int k = 1 + q / 3, i = q % 3;
    const double a = ev(i, k, t1), b = ev(i, k, t2);
    *lo = {DBL_MAX, 0.0};
    *hi = {std::numeric_limits<double>::lowest(), 0.0};
    auto take = [&](double v, double e) {
      if (v < lo->v) lo->v = v;
      if (v > hi->v) hi->v = v;
      lo->e = std::max(lo->e, e);
      hi->e = std::max(hi->e, e);
    };
    take(a, 0.0);
    take(b, 0.0);
    const std::vector<Root>& rs = roots[q];
    for (size_t n = 0; n < rs.size(); ++n)
      if (!(rs[n].t < Q(t1) || rs[n].t > Q(t2))) take(rs[n].v, rs[n].e);
    // a root whose membership moves this section's minimum or maximum: its time against both ends
    for (size_t n = 0; n < rs.size(); ++n) {
      double o_lo = std::min(a, b), o_hi = std::max(a, b);
      for (size_t o = 0; o < rs.size(); ++o)
        if (o != n && !(rs[o].t < Q(t1) || rs[o].t > Q(t2))) {
          o_lo = std::min(o_lo, rs[o].v);
          o_hi = std::max(o_hi, rs[o].v);
        }
      const double tol = 1e-12 * std::max({std::abs(o_lo), std::abs(o_hi), std::abs(rs[n].v)}) + rs[n].e;
      if (!(rs[n].v < o_lo - tol || rs[n].v > o_hi + tol)) continue;
      gap_q(rs[n].t, Q(t1), TQ, 0.0);
      gap_q(rs[n].t, Q(t2), TQ, 0.0);
    }
  }

  // recursiveFeasibility on [t1, t2]
  int walk(double t1, double t2) {
    if (t2 - t1 < mst) return 1;
    const bool f_min = present & 1u, f_max = present & 2u, v_max = present & 4u, omega = present & 8u;
    if (f_min || f_max) {
      double f[2];
      for (int s = 0; s < 2; ++s) {
        const double t = s == 0 ? t1 : t2;
        double acc = 0.0;
        for (int d = 0; d < 3; ++d) {
          double a = ev(d, 2, t);
          if (d == 2) a = a + gravity;
          acc = acc + a * a;
        }
        f[s] = std::sqrt(acc);
      }
      if (f_min && std::min(f[0], f[1]) < lim[0]) return 3;
      if (f_max && std::max(f[0], f[1]) > lim[1]) return 2;
    }
    if (v_max) {
      double v[2];
      for (int s = 0; s < 2; ++s) {
        const double t = s == 0 ? t1 : t2;
        double acc = 0.0;
        for (int d = 0; d < 3; ++d) {
          const double a = ev(d, 1, t);
          acc = acc + a * a;
        }
        v[s] = std::sqrt(acc);
      }
      if (std::max(v[0], v[1]) > lim[2]) return 4;
    }
    V f_min_sqr = {0, 0}, f_max_sqr = {0, 0}, v_max_sqr = {0, 0}, j_max_sqr = {0, 0};
    if (v_max) {
      const V limit_sq = {lim[2] * lim[2], 0.0};
      for (int i = 0; i < 3; ++i) {
        V lo, hi;
        minmax(i, t1, t2, &lo, &hi);
        const V m2 = vmax(sq(lo), sq(hi));
        cmp(m2, limit_sq, limit_sq.v);
        if (m2.v > limit_sq.v) return 4;
        v_max_sqr = add(v_max_sqr, sq(vmax(vabs(lo), vabs(hi))));
      }
    }
    if (f_min || f_max || omega) {
      for (int i = 0; i < 3; ++i) {
        V lo, hi;
        minmax(3 + i, t1, t2, &lo, &hi);
        const double gi = i == 2 ? gravity : 0.0;
        const V f_lo = rounded(lo.v + gi, lo.e), f_hi = rounded(hi.v + gi, hi.e);
        const V m = vmax(vabs(f_lo), vabs(f_hi));
        if (f_max) {
          cmp(m, {lim[1], 0.0}, lim[1]);
          if (m.v > lim[1]) return 2;
        }
        const V prod =
            rounded(f_lo.v * f_hi.v, std::abs(f_lo.v) * f_hi.e + std::abs(f_hi.v) * f_lo.e + f_lo.e * f_hi.e);
        // a sign change adds nothing to the lower bound, otherwise the smaller magnitude squared; when the sign is
        // within rounding of 0 the smaller magnitude is too, and the other branch only widens the radius
        const V lower = sq(vmin(vabs(f_lo), vabs(f_hi)));
        if (!(prod.v < 0.0)) f_min_sqr = add(f_min_sqr, lower);
        if (prod.e > 0 && !(std::abs(prod.v) > prod.e)) f_min_sqr.e += lower.v + lower.e;
        f_max_sqr = add(f_max_sqr, sq(m));
      }
    }
    if (omega) {
      for (int i = 0; i < 3; ++i) {
        V lo, hi;
        minmax(6 + i, t1, t2, &lo, &hi);
        j_max_sqr = add(j_max_sqr, sq(vmax(vabs(lo), vabs(hi))));
      }
    }
    const V f_lower = vsqrt(f_min_sqr), f_upper = vsqrt(f_max_sqr), v_upper = vsqrt(v_max_sqr);
    V omega_upper = {DBL_MAX, 0.0};
    double omega_gap = kInf;  // f_min_sqr against 1e-6 decides between DBL_MAX and the computed bound
    if (omega) omega_gap = gap(f_min_sqr, {1.0e-6, 0.0}, 1.0e-6);
    if (f_min_sqr.v > 1.0e-6) {
      const double qv = j_max_sqr.v / f_min_sqr.v;
      double qe = 0.0;
      if (j_max_sqr.e > 0 || f_min_sqr.e > 0) {
        const double den = f_min_sqr.v - f_min_sqr.e;
        qe = den > 0 ? std::max((j_max_sqr.v + j_max_sqr.e) / den - qv,
                                qv - std::max(j_max_sqr.v - j_max_sqr.e, 0.0) / (f_min_sqr.v + f_min_sqr.e))
                     : kInf;
      }
      omega_upper = vsqrt(rounded(qv, qe));
    }
    if (f_min) {
      cmp(f_upper, {lim[0], 0.0}, lim[0]);
      if (f_upper.v < lim[0]) return 3;
    }
    if (f_max) {
      cmp(f_lower, {lim[1], 0.0}, lim[1]);
      if (f_lower.v > lim[1]) return 2;
    }
    // the split: true operands make it robust when the clearest of them is; when none is true, any could flip
    bool split = false;
    double true_gap = -kInf, false_gap = kInf;
    auto operand = [&](bool present_, bool value, double g) {
      if (!present_) return;
      split = split || value;
      if (value) true_gap = std::max(true_gap, g);
      else false_gap = std::min(false_gap, g);
    };
    operand(f_min, f_lower.v < lim[0], gap(f_lower, {lim[0], 0.0}, lim[0]));
    operand(f_max, f_upper.v > lim[1], gap(f_upper, {lim[1], 0.0}, lim[1]));
    operand(v_max, v_upper.v > lim[2], gap(v_upper, {lim[2], 0.0}, lim[2]));
    operand(omega, omega_upper.v > lim[3], std::min(omega_gap, gap(omega_upper, {lim[3], 0.0}, lim[3])));
    margin = std::min(margin, split ? true_gap : false_gap);
    if (!split) return 0;
    const double th = (t1 + t2) / 2;
    const int r1 = walk(t1, th);
    if (r1 != 0) return r1;
    return walk(th, t2);
  }
};

}  // namespace

extern "C" {

// times [B][K], coeffs [B][K][D][N], limits [6] (InputConstraintType order, used where `present` has the bit) ->
// result [B] (InputFeasibilityResult), segment [B] (-1: Feasible or a bad time), margin [B].  A row with a
// segment time <= 0 or non-finite: result 1, segment -1, margin +inf.  Returns 0, or -1 on a bad argument.
int exact_input_feasibility_recursive(int N, int K, int D, int64_t B, const double* times, const double* coeffs,
                                      uint32_t present, const double* limits, double gravity, double min_section_time,
                                      int32_t* result, int32_t* segment, double* margin, int n_threads) {
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
      margin[b] = kInf;
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
