// feasibility_sampling_exact.cpp -- replay of FeasibilitySampling::checkInputFeasibilityTrajectory with binary128
// sample values: the exact reference for mtg_input_feasibility_sampling_batch_f64.  TEST INFRASTRUCTURE ONLY
// (tests/feasibility_sampling_oracle.py); never linked by the product.
//
// The sample times are the reference's running fp64 sum t = 0, fl(t + dt), ... while t <= T, so they are the device's
// bit for bit.  At each sample the flat state (velocity, acceleration, jerk of dims 0..2; yaw, yaw rate and yaw
// acceleration of dim 3 when D = 4) is evaluated from the fp64 coefficients, and the full state of mav_msgs'
// EigenMavStateFromEigenTrajectoryPoint is formed from it, in binary128: the real-number value of what the device
// rounds step by step.  The quaternion round trip of setFromYaw / getYaw is the identity on cos and sin of the yaw, so
// xc = (cos yaw, sin yaw, 0) directly.  The checks run in the reference's order and the first failing sample and check
// decide.  A thrust of exactly 0 makes the state NaN, which passes every comparison.
//
// Each sample is first evaluated in long double (x87, 64-bit significand); a comparison whose relative gap to its limit
// is below kScreen (or a NaN operand) sends the whole sample to binary128, whose values then decide it.  Per row the
// replay also returns the decision margin: the smallest relative gap |q - limit| / limit (|q| for a limit of 0) of every
// comparison made up to the deciding one.  A segment with fl(T / dt) > 2^24 is not sampled: Indeterminable with the capacity status, as on
// the device.
#include <stdint.h>

#include <atomic>
#include <cmath>
#include <limits>
#include <thread>
#include <vector>

namespace {

typedef __float128 Q;
typedef long double L;

const double kInf = std::numeric_limits<double>::infinity();
const double kScreen = 1e-6;       // gaps below this are decided in binary128
const double kSampleCap = 16777216.0;  // 2^24

// binary128 sqrt, sin and cos without libquadmath: Newton from the fp64 root; sin and cos of the argument reduced to
// [-pi, pi] (pi as the sum of three doubles), Taylor series at a / 8 and three double-angle steps.  A few units of
// binary128 rounding are far below anything the margin resolves.
Q xsqrt(Q x) {
  if (!(x > 0)) return x == 0 ? Q(0) : Q(std::numeric_limits<double>::quiet_NaN());
  if (x > Q(1e300) || x < Q(1e-300)) return Q(std::sqrt(double(x)));  // beyond fp64's range: never decided here
  Q r = Q(std::sqrt(double(x)));
  for (int i = 0; i < 3; ++i) r = (r + x / r) / 2;
  return r;
}
void xsincos(Q x, Q* s, Q* c) {
  const Q pi = Q(3.141592653589793116) + Q(1.2246467991473532e-16) + Q(-2.9947698097183397e-33);
  const Q k = Q(std::nearbyint(double(x / (2 * pi))));
  x = x - k * 2 * pi;
  const Q a = x / 8, a2 = a * a;
  Q ts = a, tc = 1, ps = a, pc = 1;
  for (int n = 1; n < 30; ++n) {
    ps = -ps * a2 / Q(double((2 * n) * (2 * n + 1)));
    pc = -pc * a2 / Q(double((2 * n - 1) * (2 * n)));
    ts += ps;
    tc += pc;
  }
  for (int i = 0; i < 3; ++i) {
    const Q s2 = 2 * ts * tc, c2 = tc * tc - ts * ts;
    ts = s2;
    tc = c2;
  }
  *s = ts;
  *c = tc;
}
inline L xsqrt(L x) { return sqrtl(x); }
inline void xsincos(L x, L* s, L* c) {
  *s = sinl(x);
  *c = cosl(x);
}
inline bool xnan(L x) { return x != x; }
inline bool xnan(Q x) { return x != x; }

template <typename R>
struct V3 {
  R x, y, z;
};
template <typename R>
R dot(const V3<R>& a, const V3<R>& b) {
  return a.x * b.x + a.y * b.y + a.z * b.z;
}
template <typename R>
V3<R> cross(const V3<R>& a, const V3<R>& b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <typename R>
V3<R> scale(R s, const V3<R>& a) {
  return {s * a.x, s * a.y, s * a.z};
}

double base_coeff(int k, int j) {  // j! / (j - k)!
  if (j < k) return 0.0;
  double v = 1.0;
  for (int q = 0; q < k; ++q) v *= double(j - q);
  return v;
}

struct Checker {
  int N, D;
  const double* c;  // [D][N]
  uint32_t present;
  const double* lim;  // [6]
  double gravity;
  double margin = kInf;

  template <typename R>
  R ev(int d, int k, double t) const {  // p_d^(k)(t) of the fp64 coefficients
    if (k >= N) return R(0);
    const double* a = c + d * N;
    R r = R(base_coeff(k, N - 1)) * R(a[N - 1]);
    for (int j = N - 2; j >= k; --j) r = r * R(t) + R(base_coeff(k, j)) * R(a[j]);
    return r;
  }

  // the quantities the present limits compare, in the reference's order: q[i] against lim[which[i]], with "<" for
  // f_min (which 0) and ">" otherwise
  template <typename R>
  int quantities(double t, R* q, int* which) const {
    int n = 0;
    const bool yaw4 = D == 4;
    const bool thrust_check = present & 3u, need_r = thrust_check || (present & 8u);
    V3<R> zb = {0, 0, 0}, xb = zb, yb = zb;
    R thrust = 0;
    if (need_r || (yaw4 && (present & 48u))) {
      const V3<R> f = {ev<R>(0, 2, t), ev<R>(1, 2, t), ev<R>(2, 2, t) + R(gravity)};
      thrust = xsqrt(dot(f, f));
      zb = scale(R(1) / thrust, f);
    }
    if (need_r) {
      R cy = 1, sy = 0;
      if (yaw4) {
        xsincos(ev<R>(3, 0, t), &sy, &cy);
      }
      yb = cross(zb, V3<R>{cy, sy, R(0)});
      const R n2 = dot(yb, yb);
      if (n2 > 0) yb = scale(R(1) / xsqrt(n2), yb);
      xb = cross(yb, zb);
    }
    if (thrust_check) {
      const V3<R> w = scale(thrust, zb), ab = {dot(xb, w), dot(yb, w), dot(zb, w)};
      const R tb = xsqrt(dot(ab, ab));
      if (present & 1u) q[n] = tb, which[n++] = 0;
      if (present & 2u) q[n] = tb, which[n++] = 1;
    }
    if (present & 4u) {
      const V3<R> v = {ev<R>(0, 1, t), ev<R>(1, 1, t), ev<R>(2, 1, t)};
      q[n] = xsqrt(dot(v, v)), which[n++] = 2;
    }
    if (present & 8u) {
      const V3<R> j = {ev<R>(0, 3, t), ev<R>(1, 3, t), ev<R>(2, 3, t)};
      const R zj = dot(zb, j);
      const V3<R> h = scale(R(1) / thrust, V3<R>{j.x - zj * zb.x, j.y - zj * zb.y, j.z - zj * zb.z});
      const R wx = -dot(h, yb), wy = dot(h, xb);
      q[n] = xsqrt(wx * wx + wy * wy), which[n++] = 3;
    }
    if (present & 16u) {
      const R r = yaw4 ? ev<R>(3, 1, t) * zb.z : R(0);
      q[n] = r < 0 ? -r : r, which[n++] = 4;
    }
    if (present & 32u) {
      const R r = yaw4 ? ev<R>(3, 2, t) * zb.z : R(0);
      q[n] = r < 0 ? -r : r, which[n++] = 5;
    }
    return n;
  }

  static constexpr int kCode[6] = {3, 2, 4, 5, 6, 7};  // ThrustLow, ThrustHigh, Velocity, RollPitch, YawRates, YawAcc

  // the comparisons of one sample: 0 or the failing code; gaps[] receives each comparison's relative gap
  template <typename R>
  int decide(const R* q, const int* which, int n, double* gaps, int* used, bool* clear) const {
    *clear = true;
    for (int i = 0; i < n; ++i) {
      const int w = which[i];
      const double l = lim[w];
      used[0] = i + 1;
      if (xnan(q[i])) {
        gaps[i] = kInf;
        *clear = false;
        continue;
      }
      const R d = q[i] - R(l);
      gaps[i] = l == kInf ? kInf : double((d < 0 ? -d : d) / R(l > 0 ? l : 1.0));
      if (!(gaps[i] > kScreen)) *clear = false;
      if (w == 0 ? q[i] < R(l) : q[i] > R(l)) return kCode[w];
    }
    return 0;
  }

  int sample(double t) {
    L ql[6];
    Q qq[6];
    int which[6];
    double gaps[6];
    int used = 0;
    bool clear;
    const int n = quantities<L>(t, ql, which);
    int r = decide<L>(ql, which, n, gaps, &used, &clear);
    if (!clear) {
      quantities<Q>(t, qq, which);
      r = decide<Q>(qq, which, n, gaps, &used, &clear);
    }
    for (int i = 0; i < used; ++i) margin = std::min(margin, gaps[i]);
    return r;
  }

  // 0 passes, else a FeasResult; *capacity when the segment is over the sample cap
  int run(double T, double dt, bool* capacity) {
    *capacity = false;
    if (D != 3 && D != 4) return 1;
    if (T / dt > kSampleCap) {
      *capacity = true;
      return 1;
    }
    for (double t = 0.0; t <= T; t += dt) {
      const int r = sample(t);
      if (r) return r;
    }
    return 0;
  }
};
constexpr int Checker::kCode[6];

}  // namespace

extern "C" {

// times [B][K], coeffs [B][K][D][N], limits [6] (InputConstraintType order, used where `present` has the bit) ->
// result [B] (InputFeasibilityResult), segment [B] (-1: Feasible or a bad time), status [B] (0, 1 bad time, 4 over
// the sample cap), margin [B].  A row with a segment time <= 0 or non-finite: result 1, segment -1, margin +inf.
// Returns 0, or -1 on a bad argument.
int exact_input_feasibility_sampling(int N, int K, int D, int64_t B, const double* times, const double* coeffs,
                                     uint32_t present, const double* limits, double gravity, double dt,
                                     int32_t* result, int32_t* segment, int32_t* status, double* margin,
                                     int n_threads) {
  if (N < 4 || N > 12 || K < 1 || D < 1 || B < 0 || !(dt > 0) || !std::isfinite(dt)) return -1;
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
      status[b] = 0;
      margin[b] = kInf;
      if (bad) {
        result[b] = 1;
        status[b] = 1;
        continue;
      }
      for (int i = 0; i < K; ++i) {
        Checker ck{N, D, coeffs + (size_t(b) * K + i) * D * N, present, limits, gravity};
        bool capacity;
        const int r = ck.run(times[b * K + i], dt, &capacity);
        margin[b] = std::min(margin[b], ck.margin);
        if (r != 0) {
          result[b] = r;
          segment[b] = i;
          status[b] = capacity ? 4 : 0;
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
