// BatchPolynomialOptimization<N>::computeMaximaOfMagnitude / timeObjective against the single-object host mirror:
// PolynomialOptimization<N>::computeMaximumOfMagnitude (host Aberth root finder) and computeCost().  Needs the GPU.
#include <cmath>
#include <cstdio>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"

using namespace mav_trajectory_generation;

static int g_failures = 0, g_checks = 0;
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

int main() {
  const int D = 3, K = 6, B = 23;
  std::vector<Vertex::Vector> all_v;
  std::vector<std::vector<double> > all_t;
  for (int b = 0; b < B; ++b) {
    Eigen::VectorXd lo = Eigen::VectorXd::Constant(D, -10.0), hi = Eigen::VectorXd::Constant(D, 10.0);
    all_v.push_back(createRandomVertices(getHighestDerivativeFromN(N), K, lo, hi, 900 + b));
    all_t.push_back(estimateSegmentTimes(all_v.back(), 3.0, 5.0));
  }
  BatchPolynomialOptimization<N> batch(D);
  batch.setupFromVertices(all_v, all_t, derivative_order::SNAP);
  b200::TimeObjectiveParameters params;
  params.soft_constraints = {{derivative_order::VELOCITY, 3.0}, {derivative_order::ACCELERATION, 5.0}};
  std::vector<double> objective, terms;
  if (!batch.timeObjective(params, nullptr, &objective, &terms)) ++g_failures;
  const std::vector<int> ders = {0, 1, 2, 3};
  std::vector<Extremum> maxima;
  batch.computeMaximaOfMagnitude(ders, &maxima);
  for (int b = 0; b < B; ++b) {
    PolynomialOptimization<N> opt(D);
    opt.setupFromVertices(all_v[b], all_t[b], derivative_order::SNAP);
    opt.solveLinear();
    const double J = opt.computeCost();
    EXPECT_NEAR(terms[3 * b], J, 1e-12 * std::abs(J));
    double soft = 0.0;
    for (size_t q = 0; q < ders.size(); ++q) {
      const Extremum ref = opt.computeMaximumOfMagnitude(ders[q], nullptr);
      const Extremum& got = maxima[b * ders.size() + q];
      EXPECT_NEAR(got.value, ref.value, 1e-12 * ref.value);
      if (ders[q] == 1) soft += std::min(1e12, std::exp((ref.value - 3.0) / 3.0 * 100.0));
      if (ders[q] == 2) soft += std::min(1e12, std::exp((ref.value - 5.0) / 5.0 * 100.0));
    }
    EXPECT_NEAR(terms[3 * b + 2], soft, 1e-9 * soft + 1e-300);
    double total = 0.0;
    for (double t : all_t[b]) total += t;
    EXPECT_NEAR(objective[b], J + total * total * 500.0 + terms[3 * b + 2], 1e-12 * objective[b]);
  }
  std::printf("time objective: %d checks, %d failures\n", g_checks, g_failures);
  return g_failures == 0 ? 0 : 1;
}
