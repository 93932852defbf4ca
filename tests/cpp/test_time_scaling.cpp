// BatchPolynomialOptimization<N>::scaleSegmentTimesToMeetConstraints / scaleSegmentTimesWithViolation against the
// single-object host mirror: Trajectory::scaleSegmentTimesToMeetConstraints (host Aberth root finder) and a
// PolynomialOptimization<N> solved again at the stretched times.  The two find the maxima with different root finders,
// so a trajectory whose violation lies within 1e-9 of the 1.001 threshold may stop one round apart: such rows are
// counted and skipped.  Needs the GPU.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"

using namespace mav_trajectory_generation;

static int g_failures = 0, g_checks = 0;
#define EXPECT_TRUE(c)                                                  \
  do {                                                                  \
    ++g_checks;                                                         \
    if (!(c)) {                                                         \
      ++g_failures;                                                     \
      std::printf("EXPECT_TRUE failed %s:%d: %s\n", __FILE__, __LINE__, #c); \
    }                                                                   \
  } while (0)
#define EXPECT_NEAR(a, b, tol)                                                                                    \
  do {                                                                                                            \
    ++g_checks;                                                                                                   \
    if (!(std::abs((a) - (b)) <= (tol))) {                                                                        \
      ++g_failures;                                                                                               \
      std::printf("EXPECT_NEAR failed %s:%d: %.17g vs %.17g (tol %g)\n", __FILE__, __LINE__, double(a), double(b), \
                  double(tol));                                                                                   \
    }                                                                                                             \
  } while (0)

constexpr int N = 10;

// true when a check of the mirror's trajectory lies within 1e-9 of the decision threshold
static bool near_threshold(const Trajectory& t, double v_max, double a_max) {
  double v = 0.0, a = 0.0;
  t.computeMaxVelocityAndAcceleration(&v, &a);
  return std::abs(v / v_max - 1.001) <= 1e-9 || std::abs(a / a_max - 1.001) <= 1e-9;
}

int main() {
  const int D = 3, K = 6, B = 23;
  const double v_max = 1.5, a_max = 2.5;  // the fixture's times are allocated for (3, 5): most rows stretch
  std::vector<Vertex::Vector> all_v;
  std::vector<std::vector<double> > all_t;
  for (int b = 0; b < B; ++b) {
    Eigen::VectorXd lo = Eigen::VectorXd::Constant(D, -10.0), hi = Eigen::VectorXd::Constant(D, 10.0);
    all_v.push_back(createRandomVertices(getHighestDerivativeFromN(N), K, lo, hi, 1700 + b));
    all_t.push_back(estimateSegmentTimes(all_v.back(), 3.0, 5.0));
  }
  BatchPolynomialOptimization<N> batch(D), batch_nl(D);
  batch.setupFromVertices(all_v, all_t, derivative_order::SNAP);
  batch_nl.setupFromVertices(all_v, all_t, derivative_order::SNAP);
  EXPECT_TRUE(batch.solveLinear());
  std::vector<uint8_t> within, within_nl;
  EXPECT_TRUE(batch.scaleSegmentTimesToMeetConstraints(v_max, a_max, &within));
  EXPECT_TRUE(batch_nl.scaleSegmentTimesWithViolation(v_max, a_max, &within_nl));
  int skipped = 0, stretched = 0;
  for (int b = 0; b < B; ++b) {
    PolynomialOptimization<N> opt(D);
    opt.setupFromVertices(all_v[b], all_t[b], derivative_order::SNAP);
    opt.solveLinear();
    Trajectory traj;
    opt.getTrajectory(&traj);
    Trajectory first = traj;
    if (near_threshold(first, v_max, a_max)) {
      ++skipped;
      continue;
    }
    const bool ok = traj.scaleSegmentTimesToMeetConstraints(v_max, a_max);
    if (near_threshold(traj, v_max, a_max)) {
      ++skipped;
      continue;
    }
    EXPECT_TRUE(within[b] == (ok ? 1 : 0));
    EXPECT_TRUE(within_nl[b] == (ok ? 1 : 0));
    EXPECT_TRUE(batch_nl.status()[b] == 0);
    const std::vector<double> ref_t = traj.getSegmentTimes();
    if (ref_t[0] != all_t[b][0]) ++stretched;
    Segment::Vector segs;
    traj.getSegments(&segs);
    // the re-solve at the stretched times
    PolynomialOptimization<N> again(D);
    again.setupFromVertices(all_v[b], ref_t, derivative_order::SNAP);
    again.solveLinear();
    Segment::Vector resolved;
    again.getSegments(&resolved);
    double cmax = 0.0, rmax = 0.0;
    for (int i = 0; i < K; ++i)
      for (int d = 0; d < D; ++d) {
        const Eigen::VectorXd c = segs[i][d].getCoefficients(0), r = resolved[i][d].getCoefficients(0);
        for (int n = 0; n < N; ++n) {
          cmax = std::max(cmax, std::abs(c[n]));
          rmax = std::max(rmax, std::abs(r[n]));
        }
      }
    for (int i = 0; i < K; ++i) {
      EXPECT_NEAR(batch.segmentTimes()[b * K + i], ref_t[i], 1e-10 * ref_t[i]);
      EXPECT_NEAR(batch_nl.segmentTimes()[b * K + i], ref_t[i], 1e-10 * ref_t[i]);
      for (int d = 0; d < D; ++d) {
        const Eigen::VectorXd c = segs[i][d].getCoefficients(0), r = resolved[i][d].getCoefficients(0);
        for (int n = 0; n < N; ++n) {
          EXPECT_NEAR(batch.coefficients()[((size_t(b) * K + i) * D + d) * N + n], c[n], 1e-10 * cmax);
          EXPECT_NEAR(batch_nl.coefficients()[((size_t(b) * K + i) * D + d) * N + n], r[n], 1e-10 * rmax);
        }
      }
    }
  }
  EXPECT_TRUE(stretched >= B / 2);
  std::printf("time scaling: %d stretched, %d near the threshold skipped, %d checks, %d failures\n", stretched, skipped,
              g_checks, g_failures);
  return g_failures == 0 ? 0 : 1;
}
