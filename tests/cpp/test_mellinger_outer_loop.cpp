// PolynomialOptimizationNonLinear<10>::optimize() with kMellingerOuterLoop, and
// BatchPolynomialOptimization<10>::optimizeTimeMellingerOuterLoop, at the reference suite's OptimizationParams: the
// TimeScaling test's sequence (velocity-ramp times for (v, a), scaleSegmentTimesWithViolation, then optimize()) must end
// within 1e-3 of both limits (host root finder, double precision) with a cost no higher than after the scaling.  The
// batch class must give the same times and coefficients as the single object, bit for bit, and the other time
// allocation methods must return INVALID_ARGS.  Needs the GPU.
#include <cmath>
#include <cstdio>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_nonlinear.h"

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

constexpr int N = 10;

struct Case {
  int D, r, K, seed;
  double bounds, v_max, a_max;
};
// the reference suite's OptimizationParams (tests/test_oracle.py REF_PARAMS)
static const Case kCases[] = {{1, 4, 1, 100, 10.0, 3.0, 5.0}, {1, 4, 10, 102, 10.0, 3.0, 5.0},
                              {1, 4, 50, 103, 10.0, 3.0, 5.0}, {3, 4, 1, 104, 10.0, 3.0, 5.0},
                              {3, 4, 10, 105, 10.0, 3.0, 5.0}, {3, 4, 50, 106, 10.0, 3.0, 5.0},
                              {1, 2, 5, 107, 10.0, 1.0, 2.0},  {3, 2, 1, 108, 10.0, 1.0, 2.0},
                              {3, 2, 5, 109, 10.0, 1.0, 2.0},  {3, 3, 5, 110, 10.0, 1.0, 2.0}};

int main() {
  NonlinearOptimizationParameters params;
  params.time_alloc_method = NonlinearOptimizationParameters::kMellingerOuterLoop;
  for (const Case& c : kCases) {
    const Eigen::VectorXd lo = Eigen::VectorXd::Constant(c.D, -c.bounds), hi = Eigen::VectorXd::Constant(c.D, c.bounds);
    const Vertex::Vector vertices = createRandomVertices(getHighestDerivativeFromN(N), c.K, lo, hi, c.seed);
    const std::vector<double> ramp = estimateSegmentTimesVelocityRamp(vertices, c.v_max, c.a_max);

    PolynomialOptimizationNonLinear<N> opt(c.D, params);
    EXPECT_TRUE(opt.setupFromVertices(vertices, ramp, c.r));
    EXPECT_TRUE(opt.addMaximumMagnitudeConstraint(derivative_order::VELOCITY, c.v_max));
    EXPECT_TRUE(opt.addMaximumMagnitudeConstraint(derivative_order::ACCELERATION, c.a_max));
    EXPECT_TRUE(opt.solveLinear());
    opt.scaleSegmentTimesWithViolation();
    const double scaled_cost = opt.getCost();
    std::vector<double> scaled_times;
    opt.getPolynomialOptimizationRef().getSegmentTimes(&scaled_times);
    const int result = opt.optimize();
    EXPECT_TRUE(result > 0 || result == -4);  // SUCCESS / FTOL / XTOL / MAXEVAL, or ROUNDOFF_LIMITED
    EXPECT_TRUE(opt.getOptimizationInfo().stopping_reason == result);
    EXPECT_TRUE(opt.getPolynomialOptimizationRef().getLastStatus() == 0);
    const double cost = opt.getCost();
    EXPECT_TRUE(cost <= scaled_cost);
    Trajectory traj;
    opt.getTrajectory(&traj);
    double v = 0.0, a = 0.0;
    traj.computeMaxVelocityAndAcceleration(&v, &a);
    EXPECT_TRUE(v <= c.v_max + 1e-3 && a <= c.a_max + 1e-3);
    std::vector<double> times;
    opt.getPolynomialOptimizationRef().getSegmentTimes(&times);
    Segment::Vector segs;
    opt.getPolynomialOptimizationRef().getSegments(&segs);

    // the batch class on the same start (the scaled times), two copies of the problem
    BatchPolynomialOptimization<N> batch(c.D);
    std::vector<Vertex::Vector> all_v(2, vertices);
    std::vector<std::vector<double> > all_t(2, scaled_times);
    EXPECT_TRUE(batch.setupFromVertices(all_v, all_t, c.r));
    b200::MellingerParameters q;
    std::vector<int> res, iters;
    EXPECT_TRUE(batch.optimizeTimeMellingerOuterLoop(q, c.v_max, c.a_max, &res, &iters));
    for (int b = 0; b < 2; ++b) {
      EXPECT_TRUE(res[b] == result && iters[b] == opt.getOptimizationInfo().n_iterations);
      EXPECT_TRUE(batch.status()[b] == 0);
      for (int i = 0; i < c.K; ++i) {
        EXPECT_TRUE(batch.segmentTimes()[b * c.K + i] == times[i]);
        for (int d = 0; d < c.D; ++d) {
          const Eigen::VectorXd co = segs[i][d].getCoefficients(0);
          for (int n = 0; n < N; ++n)
            EXPECT_TRUE(batch.coefficients()[((size_t(b) * c.K + i) * c.D + d) * N + n] == co[n]);
        }
      }
    }
    std::printf("D=%d r=%d K=%d: result %d after %d steps, cost %.6g -> %.6g, v %.6g / %.3g, a %.6g / %.3g\n", c.D,
                c.r, c.K, result, opt.getOptimizationInfo().n_iterations, scaled_cost, cost, v, c.v_max, a, c.a_max);
  }
  // every other time allocation method: INVALID_ARGS
  for (auto m : {NonlinearOptimizationParameters::kSquaredTime, NonlinearOptimizationParameters::kRichterTime,
                 NonlinearOptimizationParameters::kSquaredTimeAndConstraints,
                 NonlinearOptimizationParameters::kRichterTimeAndConstraints}) {
    NonlinearOptimizationParameters p;
    p.time_alloc_method = m;
    PolynomialOptimizationNonLinear<N> opt(3, p);
    const Eigen::VectorXd lo = Eigen::VectorXd::Constant(3, -10.0), hi = Eigen::VectorXd::Constant(3, 10.0);
    const Vertex::Vector vertices = createRandomVertices(getHighestDerivativeFromN(N), 4, lo, hi, 7);
    opt.setupFromVertices(vertices, estimateSegmentTimes(vertices, 3.0, 5.0));
    EXPECT_TRUE(opt.optimize() == -2);
  }
  std::printf("mellinger outer loop: %d checks, %d failures\n", g_checks, g_failures);
  return g_failures == 0 ? 0 : 1;
}
