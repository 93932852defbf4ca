// The host mirror's flat-state samplers (trajectory_sampling.h) and the batched
// BatchPolynomialOptimization<N>::sampleTrajectoriesInRange / sampleWholeTrajectories / sampleTrajectoriesAtTime, driven
// by tests/test_flat_state_sampling.py.
//   test_flat_state_sampling mirror IN OUT
//       host only: IN = int32 B, K, D, N, mode (0 sampleTrajectoryInRange, 1 sampleWholeTrajectory,
//       2 sampleTrajectoryAtTime), S; double min_time, max_time, sampling_interval; times [B][K]; coeffs [B][K][D][N];
//       sample_times [B] (mode 2) -> OUT = int32 n [B] (-1 where the sampler returns false; mode 2: 1 or -1),
//       double records [B][S][25] (the first S states, zero beyond), int64 time_ns [B][S]
//   test_flat_state_sampling batch
//       needs the GPU: solves random-vertex problems (N = 10, K = 5, D = 3, 4 and 6), runs the three batch samplers
//       and the mirror on every trajectory and compares them: position ... snap and time stamps equal, attitude within
//       kAttitudeBound, the quaternion up to sign where |w| is within rounding of 0.  Exit 0 when all agree.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"
#include "mav_trajectory_generation/trajectory_sampling.h"
#include "mtg_b200.h"

using namespace mav_trajectory_generation;

static void to_record(const mav_msgs::EigenTrajectoryPoint& p, double* r) {
  const Eigen::Vector3d* vecs[] = {&p.position_W, &p.velocity_W, &p.acceleration_W, &p.jerk_W, &p.snap_W};
  for (int f = 0; f < 5; ++f)
    for (int k = 0; k < 3; ++k) r[3 * f + k] = (*vecs[f])[k];
  r[MTG_FLAT_STATE_ORIENTATION + 0] = p.orientation_W_B.w;
  r[MTG_FLAT_STATE_ORIENTATION + 1] = p.orientation_W_B.x;
  r[MTG_FLAT_STATE_ORIENTATION + 2] = p.orientation_W_B.y;
  r[MTG_FLAT_STATE_ORIENTATION + 3] = p.orientation_W_B.z;
  for (int k = 0; k < 3; ++k) {
    r[MTG_FLAT_STATE_ANGULAR_VELOCITY + k] = p.angular_velocity_W[k];
    r[MTG_FLAT_STATE_ANGULAR_ACCELERATION + k] = p.angular_acceleration_W[k];
  }
}

static Trajectory trajectory_of(const double* times, const double* coeffs, int K, int D, int N) {
  Segment::Vector segs;
  for (int i = 0; i < K; ++i) {
    Segment s(N, D);
    s.setTime(times[i]);
    for (int d = 0; d < D; ++d) {
      Eigen::VectorXd c(N);
      for (int n = 0; n < N; ++n) c[n] = coeffs[(size_t(i) * D + d) * N + n];
      s[d] = Polynomial(c);
    }
    segs.push_back(s);
  }
  Trajectory t;
  t.setSegments(segs);
  return t;
}

static bool read_all(FILE* f, void* p, size_t bytes) { return std::fread(p, 1, bytes, f) == bytes; }

// attitude of the batch against the mirror: |difference| <= kAttitudeBound * (1 + |mirror value|) per component
static const double kAttitudeBound = 1e-13;

static int compare(const mav_msgs::EigenTrajectoryPoint& a, const mav_msgs::EigenTrajectoryPoint& b, const char* what,
                   int row, int i) {
  double ra[MTG_FLAT_STATE_DOUBLES], rb[MTG_FLAT_STATE_DOUBLES];
  to_record(a, ra);
  to_record(b, rb);
  bool ok = a.time_from_start_ns == b.time_from_start_ns && a.degrees_of_freedom == b.degrees_of_freedom;
  for (int k = 0; k < MTG_FLAT_STATE_ORIENTATION; ++k) ok = ok && std::memcmp(&ra[k], &rb[k], 8) == 0;
  // |w| within rounding of 0: the two sides may hold the same rotation with opposite signs
  const double sign = std::fabs(rb[MTG_FLAT_STATE_ORIENTATION]) < 1e-12 &&
                              ra[MTG_FLAT_STATE_ORIENTATION + 1] * rb[MTG_FLAT_STATE_ORIENTATION + 1] +
                                      ra[MTG_FLAT_STATE_ORIENTATION + 2] * rb[MTG_FLAT_STATE_ORIENTATION + 2] +
                                      ra[MTG_FLAT_STATE_ORIENTATION + 3] * rb[MTG_FLAT_STATE_ORIENTATION + 3] <
                                  0
                          ? -1.0
                          : 1.0;
  for (int k = MTG_FLAT_STATE_ORIENTATION; k < MTG_FLAT_STATE_DOUBLES; ++k) {
    const double s = k < MTG_FLAT_STATE_ANGULAR_VELOCITY ? sign : 1.0;
    ok = ok && std::fabs(s * ra[k] - rb[k]) <= kAttitudeBound * (1.0 + std::fabs(rb[k]));
  }
  if (!ok) std::printf("%s: row %d state %d differs\n", what, row, i);
  return ok ? 0 : 1;
}

int main(int argc, char** argv) {
  if (argc == 4 && !std::strcmp(argv[1], "mirror")) {
    FILE* in = std::fopen(argv[2], "rb");
    if (!in) return 2;
    int32_t hdr[6];
    double rng[3];
    if (!read_all(in, hdr, sizeof(hdr)) || !read_all(in, rng, sizeof(rng))) return 2;
    const int B = hdr[0], K = hdr[1], D = hdr[2], N = hdr[3], mode = hdr[4], S = hdr[5];
    std::vector<double> times(size_t(B) * K), coeffs(size_t(B) * K * D * N), at(B);
    if (!read_all(in, times.data(), times.size() * 8) || !read_all(in, coeffs.data(), coeffs.size() * 8)) return 2;
    if (mode == 2 && !read_all(in, at.data(), at.size() * 8)) return 2;
    std::fclose(in);
    std::vector<int32_t> n(B);
    std::vector<double> rec(size_t(B) * S * MTG_FLAT_STATE_DOUBLES, 0.0);
    std::vector<int64_t> ns(size_t(B) * S, 0);
    for (int b = 0; b < B; ++b) {
      const Trajectory t = trajectory_of(&times[size_t(b) * K], &coeffs[size_t(b) * K * D * N], K, D, N);
      mav_msgs::EigenTrajectoryPointVector states;
      bool ok;
      if (mode == 2) {
        mav_msgs::EigenTrajectoryPoint p;
        ok = sampleTrajectoryAtTime(t, at[b], &p);
        if (ok) states.push_back(p);
      } else if (mode == 1) {
        ok = sampleWholeTrajectory(t, rng[2], &states);
      } else {
        ok = sampleTrajectoryInRange(t, rng[0], rng[1], rng[2], &states);
      }
      n[b] = ok ? static_cast<int32_t>(states.size()) : -1;
      for (int i = 0; i < S && i < int(states.size()); ++i) {
        to_record(states[i], &rec[(size_t(b) * S + i) * MTG_FLAT_STATE_DOUBLES]);
        ns[size_t(b) * S + i] = states[i].time_from_start_ns;
      }
    }
    FILE* out = std::fopen(argv[3], "wb");
    if (!out) return 2;
    std::fwrite(n.data(), 4, B, out);
    std::fwrite(rec.data(), 8, rec.size(), out);
    std::fwrite(ns.data(), 8, ns.size(), out);
    std::fclose(out);
    return 0;
  }
  if (argc == 2 && !std::strcmp(argv[1], "batch")) {
    constexpr int N = 10;
    const int K = 5, B = 48;
    int bad = 0, checked = 0;
    for (int D : {3, 4, 6}) {
      std::vector<Vertex::Vector> all_v;
      std::vector<std::vector<double> > all_t;
      for (int b = 0; b < B; ++b) {
        Eigen::VectorXd lo = Eigen::VectorXd::Constant(D, -4.0), hi = Eigen::VectorXd::Constant(D, 4.0);
        all_v.push_back(createRandomVertices(derivative_order::SNAP, K, lo, hi, 7100 + 10 * D + b));
        all_t.push_back(estimateSegmentTimes(all_v.back(), 2.0 + 0.05 * (b % 40), 3.0 + 0.1 * (b % 50)));
      }
      BatchPolynomialOptimization<N> batch(D);
      batch.setupFromVertices(all_v, all_t, derivative_order::SNAP);
      if (!batch.solveLinear()) return 3;
      std::vector<mav_msgs::EigenTrajectoryPointVector> range, whole;
      std::vector<uint8_t> range_ok, whole_ok, at_ok;
      const double t0 = 0.37, t1 = 2.9, dt = 0.05;
      batch.sampleTrajectoriesInRange(t0, t1, dt, &range, &range_ok);
      batch.sampleWholeTrajectories(dt, &whole, &whole_ok);
      std::vector<double> at_times(B);
      for (int b = 0; b < B; ++b) {
        Trajectory t;
        batch.getTrajectory(b, &t);
        at_times[b] = b % 7 == 0 ? t.getMaxTime() : b % 7 == 1 ? t.getMaxTime() * 1.5 : 0.13 * (b % 11);
      }
      mav_msgs::EigenTrajectoryPointVector at;
      batch.sampleTrajectoriesAtTime(at_times, &at, &at_ok);
      for (int b = 0; b < B; ++b) {
        Trajectory t;
        batch.getTrajectory(b, &t);
        mav_msgs::EigenTrajectoryPointVector hr, hw;
        const bool hr_ok = sampleTrajectoryInRange(t, t0, t1, dt, &hr);
        const bool hw_ok = sampleWholeTrajectory(t, dt, &hw);
        mav_msgs::EigenTrajectoryPoint ha;
        const bool ha_ok = sampleTrajectoryAtTime(t, at_times[b], &ha);
        if (hr_ok != bool(range_ok[b]) || hr.size() != range[b].size() || hw_ok != bool(whole_ok[b]) ||
            hw.size() != whole[b].size() || ha_ok != bool(at_ok[b])) {
          std::printf("D=%d row %d: ok or count differs\n", D, b);
          ++bad;
          continue;
        }
        for (size_t i = 0; i < hr.size(); ++i) bad += compare(range[b][i], hr[i], "range", b, int(i));
        for (size_t i = 0; i < hw.size(); ++i) bad += compare(whole[b][i], hw[i], "whole", b, int(i));
        if (ha_ok) bad += compare(at[b], ha, "at time", b, 0);
        checked += int(hr.size() + hw.size()) + ha_ok;
      }
    }
    std::printf("batch class: %d states checked, %d differ\n", checked, bad);
    return bad == 0 && checked > 1000 ? 0 : 4;
  }
  std::fprintf(stderr, "usage: %s mirror IN OUT | batch\n", argv[0]);
  return 1;
}
