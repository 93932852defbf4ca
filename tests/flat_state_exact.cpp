// flat_state_exact.cpp -- the attitude of a flat state in binary128: the exact reference for the orientation, angular
// velocity and angular acceleration of mtg_sample_flat_states_batch_f64 / mtg_sample_flat_state_at_time_batch_f64 and
// of the host mirror (trajectory_sampling.h).  TEST INFRASTRUCTURE ONLY (tests/flat_state_oracle.py); never linked by
// the product.
//
// Inputs are the fp64 attitude-dimension values of each sample (bit for bit what every side evaluates, since the
// polynomial values are Polynomial::evaluate's arithmetic everywhere); from them the state is formed in binary128:
//   yaw (D = 4):           q = (cos y/2, 0, 0, sin y/2), omega = (0, 0, y'), omega_dot = (0, 0, y'')
//   rotation vector (D = 6): q = (cos t/2, sin(t/2)/t phi) with t = |phi|, negated when w < 0;
//                          omega = J phi',  omega_dot = J phi'' + J' phi'  with J = I + a [phi]x + b [phi]x^2,
//                          a = (1 - cos t)/t^2, b = (t - sin t)/t^3,
//                          J' phi' = (a'/t)(phi.phi')(phi x phi') + (b'/t)(phi.phi') phi x (phi x phi') + b phi' x (phi x phi')
// a, b, a'/t and b'/t are their power series below t = 1 (no cancellation, and t = 0 needs no special case) and the
// closed forms above it.  Results are rounded once to fp64.
#include <stdint.h>

#include <cmath>

namespace {

typedef __float128 Q;

// binary128 sqrt, sin and cos without libquadmath: Newton from the fp64 root; sin and cos of the argument reduced to
// [-pi, pi] (pi as the sum of three doubles), Taylor series at x / 8 and three double-angle steps.
Q xsqrt(Q x) {
  if (!(x > 0)) return Q(0);
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

struct V {
  Q x, y, z;
};
V cross(const V& a, const V& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
Q dot(const V& a, const V& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
V add(const V& a, const V& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
V scale(Q s, const V& a) { return {s * a.x, s * a.y, s * a.z}; }
V load(const double* p) { return {Q(p[0]), Q(p[1]), Q(p[2])}; }
void store(const V& a, double* p) {
  p[0] = double(a.x);
  p[1] = double(a.y);
  p[2] = double(a.z);
}

// a, b, a'/t, b'/t of t
void coefficients(Q t, Q* a, Q* b, Q* a1, Q* b1) {
  if (t < 1) {
    // a = sum (-1)^k t^2k / (2k+2)!, b = sum (-1)^k t^2k / (2k+3)!, and the term-wise derivatives over t
    const Q t2 = t * t;
    Q sa = 0, sb = 0, sa1 = 0, sb1 = 0;
    Q p = 1, pm = -1;  // (-1)^k t^2k, and (-1)^k t^(2k-2) = its derivative over 2k t
    Q fa = 2, fb = 6;  // (2k+2)!, (2k+3)!
    for (int k = 0; k < 24; ++k) {
      sa += p / fa;
      sb += p / fb;
      if (k > 0) {
        sa1 += Q(2 * k) * pm / fa;
        sb1 += Q(2 * k) * pm / fb;
        pm *= -t2;
      }
      p *= -t2;
      fa *= Q(double((2 * k + 3) * (2 * k + 4)));
      fb *= Q(double((2 * k + 4) * (2 * k + 5)));
    }
    *a = sa;
    *b = sb;
    *a1 = sa1;
    *b1 = sb1;
    return;
  }
  Q s, c;
  xsincos(t, &s, &c);
  const Q t2 = t * t, t3 = t2 * t, t4 = t3 * t;
  *a = (1 - c) / t2;
  *b = (t - s) / t3;
  *a1 = (t * s - 2 * (1 - c)) / t4;
  *b1 = ((1 - c) * t - 3 * (t - s)) / (t4 * t);
}

}  // namespace

extern "C" {

// M samples of a rotation vector phi [M][3] and its derivatives -> q [M][4] (w, x, y, z), omega, omega_dot [M][3]
int exact_rotation_vector_state(int64_t M, const double* phi, const double* dphi, const double* ddphi, double* q,
                                double* omega, double* omega_dot) {
  for (int64_t m = 0; m < M; ++m) {
    const V p = load(phi + 3 * m), d = load(dphi + 3 * m), dd = load(ddphi + 3 * m);
    const Q t = xsqrt(dot(p, p));
    Q a, b, a1, b1;
    coefficients(t, &a, &b, &a1, &b1);
    Q w = 1, x = 0, y = 0, z = 0;
    if (t > 0) {
      Q s, c;
      xsincos(t / 2, &s, &c);
      const Q k = s / t;
      w = c;
      x = k * p.x;
      y = k * p.y;
      z = k * p.z;
      if (w < 0) {
        w = -w;
        x = -x;
        y = -y;
        z = -z;
      }
    }
    q[4 * m + 0] = double(w);
    q[4 * m + 1] = double(x);
    q[4 * m + 2] = double(y);
    q[4 * m + 3] = double(z);
    auto applyJ = [&](const V& v) {
      const V pv = cross(p, v);
      return add(v, add(scale(a, pv), scale(b, cross(p, pv))));
    };
    store(applyJ(d), omega + 3 * m);
    const Q pd = dot(p, d);
    const V c1 = cross(p, d);
    const V jd = add(add(scale(a1 * pd, c1), scale(b1 * pd, cross(p, c1))), scale(b, cross(d, c1)));
    store(add(applyJ(dd), jd), omega_dot + 3 * m);
  }
  return 0;
}

// M samples of yaw, yaw rate, yaw acceleration -> q [M][4], omega, omega_dot [M][3]
int exact_yaw_state(int64_t M, const double* yaw, const double* yaw_rate, const double* yaw_acc, double* q,
                    double* omega, double* omega_dot) {
  for (int64_t m = 0; m < M; ++m) {
    Q s, c;
    xsincos(Q(yaw[m]) / 2, &s, &c);
    q[4 * m + 0] = double(c);
    q[4 * m + 1] = q[4 * m + 2] = 0.0;
    q[4 * m + 3] = double(s);
    omega[3 * m] = omega[3 * m + 1] = 0.0;
    omega[3 * m + 2] = yaw_rate[m];
    omega_dot[3 * m] = omega_dot[3 * m + 1] = 0.0;
    omega_dot[3 * m + 2] = yaw_acc[m];
  }
  return 0;
}

// the series coefficients at t, for the closed-form tests: out = {a, b, a'/t, b'/t}
int exact_jacobian_coefficients(double t, double* out) {
  Q a, b, a1, b1;
  coefficients(Q(t), &a, &b, &a1, &b1);
  out[0] = double(a);
  out[1] = double(b);
  out[2] = double(a1);
  out[3] = double(b1);
  return 0;
}
}
