// BatchPolynomialOptimization<10>::optimizeTime (kSquaredTime and kRichterTime as the compass search of
// mtg_optimize_time_batch_f64) against the C-ABI entry called directly on the same rows: times, coefficients, result,
// evaluations, objective and status must be equal bit for bit, row by row.  Needs the GPU.
#include <cstdio>
#include <cstring>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mtg_b200.h"

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

static bool sameBits(double a, double b) { return std::memcmp(&a, &b, sizeof(double)) == 0; }

int main() {
  const int D = 3, K = 7, B = 41, h = N / 2, nf = 2 * h + K - 1;
  std::vector<Vertex::Vector> all_v;
  std::vector<std::vector<double> > all_t;
  std::vector<double> times, d_fixed(size_t(B) * D * nf, 0.0);
  for (int b = 0; b < B; ++b) {
    const Eigen::VectorXd lo = Eigen::VectorXd::Constant(D, -10.0), hi = Eigen::VectorXd::Constant(D, 10.0);
    all_v.push_back(createRandomVertices(getHighestDerivativeFromN(N), K, lo, hi, 1300 + b));
    all_t.push_back(estimateSegmentTimes(all_v.back(), 3.0, 5.0));
    times.insert(times.end(), all_t.back().begin(), all_t.back().end());
    // d_fixed in the reference's compact order: x_0, its derivatives (zero), x_1 .. x_{K-1}, x_K, its derivatives
    for (int v = 0; v <= K; ++v) {
      Eigen::VectorXd pos;
      all_v.back()[v].getConstraint(derivative_order::POSITION, &pos);
      const int slot = v == 0 ? 0 : (v < K ? h + v - 1 : h + K - 1);
      for (int d = 0; d < D; ++d) d_fixed[(size_t(b) * D + d) * nf + slot] = pos[d];
    }
  }
  mtg_handle* handle = nullptr;
  EXPECT_TRUE(mtg_create(0, &handle) == MTG_OK);
  for (bool richter : {false, true}) {
    BatchPolynomialOptimization<N> batch(D);
    EXPECT_TRUE(batch.setupFromVertices(all_v, all_t, derivative_order::SNAP));
    b200::TimeObjectiveParameters op;
    op.richter_time = richter;
    op.soft_constraints = {{derivative_order::VELOCITY, 3.0}, {derivative_order::ACCELERATION, 5.0}};
    b200::MellingerParameters q;
    q.x_rel = 0.1;
    std::vector<int> res, ev;
    std::vector<double> obj;
    EXPECT_TRUE(batch.optimizeTime(op, q, &res, &ev, &obj));

    const mtg_soft_constraint cons[2] = {{derivative_order::VELOCITY, 3.0}, {derivative_order::ACCELERATION, 5.0}};
    const mtg_time_objective o = {richter ? 1 : 0, 500.0, 100.0, 1e12, 2, cons};
    const mtg_mellinger_params prm = {q.f_abs, q.f_rel, q.x_rel, q.x_abs, q.initial_stepsize_rel, q.max_iterations};
    const mtg_problem p = {N, derivative_order::SNAP, K, D, nullptr};
    std::vector<double> coeffs(size_t(B) * K * D * N), t_out(size_t(B) * K), objective(B);
    std::vector<int32_t> res2(B), ev2(B), st2(B);
    EXPECT_TRUE(mtg_optimize_time_batch_host_f64(handle, &p, B, times.data(), d_fixed.data(), &o, &prm, coeffs.data(),
                                                 t_out.data(), objective.data(), nullptr, ev2.data(), res2.data(),
                                                 st2.data()) == MTG_OK);
    int improved = 0;
    for (int b = 0; b < B; ++b) {
      EXPECT_TRUE(res[b] == res2[b] && ev[b] == ev2[b] && batch.status()[b] == st2[b]);
      EXPECT_TRUE(sameBits(obj[b], objective[b]));
      EXPECT_TRUE(res[b] > 0 || res[b] == MTG_OPTIMIZE_RESULT_ROUNDOFF_LIMITED);
      bool moved = false;
      for (int i = 0; i < K; ++i) {
        EXPECT_TRUE(sameBits(batch.segmentTimes()[b * K + i], t_out[b * K + i]));
        moved = moved || t_out[b * K + i] != times[b * K + i];
      }
      for (size_t c = 0; c < size_t(K) * D * N; ++c)
        EXPECT_TRUE(sameBits(batch.coefficients()[b * size_t(K) * D * N + c], coeffs[b * size_t(K) * D * N + c]));
      improved += moved;
    }
    EXPECT_TRUE(improved > B / 2);
    std::printf("%s: %d of %d rows moved, evaluations of row 0: %d, result %d\n",
                richter ? "kRichterTime" : "kSquaredTime", improved, B, ev[0], res[0]);
  }
  mtg_destroy(handle);
  std::printf("optimize time: %d checks, %d failures\n", g_checks, g_failures);
  return g_failures == 0 ? 0 : 1;
}
