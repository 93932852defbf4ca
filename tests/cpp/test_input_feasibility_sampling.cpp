// The single-object host FeasibilitySampling and the batched
// BatchPolynomialOptimization<N>::checkInputFeasibilitySampling, driven by tests/test_input_feasibility_sampling.py,
// which compares both against the binary128 replay on the rows whose decision margin is clear of rounding.
//   test_input_feasibility_sampling mirror IN OUT
//       host only: IN = int32 B, K, D, N, present; double limits[6], gravity, sampling_interval, times [B][K],
//       coeffs [B][K][D][N] -> OUT = int32 result [B], segment [B] of FeasibilitySampling
//   test_input_feasibility_sampling batch OUT
//       needs the GPU: solves B = 96 random-vertex problems (N = 10, D = 3, K = 5) and writes int32 B, K, D, N; times;
//       coeffs; the batch's result and segment; the host FeasibilitySampling's result and segment (default limits,
//       sampling interval 0.05 s)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"
#include "mav_trajectory_generation_ros/feasibility_sampling.h"

using namespace mav_trajectory_generation;

// result and first failing segment (-1 when feasible) of the host checker on one trajectory
static void check_host(const FeasibilitySampling& f, const Segment::Vector& segs, int32_t* result,
                       int32_t* segment) {
  Trajectory t;
  t.setSegments(segs);
  *result = f.checkInputFeasibilityTrajectory(t);
  *segment = -1;
  for (size_t i = 0; i < segs.size(); ++i)
    if (f.checkInputFeasibility(segs[i]) != kInputFeasible) {
      *segment = static_cast<int32_t>(i);
      break;
    }
}

static Segment::Vector segments_of(const double* times, const double* coeffs, int K, int D, int N) {
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
  return segs;
}

static bool read_all(FILE* f, void* p, size_t bytes) { return std::fread(p, 1, bytes, f) == bytes; }

int main(int argc, char** argv) {
  if (argc == 4 && !std::strcmp(argv[1], "mirror")) {
    FILE* in = std::fopen(argv[2], "rb");
    if (!in) return 2;
    int32_t hdr[5];
    double lim[6], gravity, dt;
    if (!read_all(in, hdr, sizeof(hdr)) || !read_all(in, lim, sizeof(lim)) || !read_all(in, &gravity, 8) ||
        !read_all(in, &dt, 8))
      return 2;
    const int B = hdr[0], K = hdr[1], D = hdr[2], N = hdr[3];
    std::vector<double> times(size_t(B) * K), coeffs(size_t(B) * K * D * N);
    if (!read_all(in, times.data(), times.size() * 8) || !read_all(in, coeffs.data(), coeffs.size() * 8)) return 2;
    std::fclose(in);
    InputConstraints ic;
    for (int q = 0; q < 6; ++q)
      if (hdr[4] >> q & 1) ic.addConstraint(q, lim[q]);
    FeasibilitySampling::Settings settings;
    settings.setSamplingIntervalS(dt);
    FeasibilitySampling f(settings, ic);
    f.gravity_ = Eigen::Vector3d(0.0, 0.0, gravity);
    std::vector<int32_t> res(B), seg(B);
    for (int b = 0; b < B; ++b)
      check_host(f, segments_of(&times[size_t(b) * K], &coeffs[size_t(b) * K * D * N], K, D, N), &res[b], &seg[b]);
    FILE* out = std::fopen(argv[3], "wb");
    if (!out) return 2;
    std::fwrite(res.data(), 4, B, out);
    std::fwrite(seg.data(), 4, B, out);
    std::fclose(out);
    return 0;
  }
  if (argc == 3 && !std::strcmp(argv[1], "batch")) {
    constexpr int N = 10;
    const int D = 3, K = 5, B = 96;
    std::vector<Vertex::Vector> all_v;
    std::vector<std::vector<double> > all_t;
    for (int b = 0; b < B; ++b) {
      Eigen::VectorXd lo = Eigen::VectorXd::Constant(D, -5.0), hi = Eigen::VectorXd::Constant(D, 5.0);
      all_v.push_back(createRandomVertices(derivative_order::SNAP, K, lo, hi, 5300 + b));
      all_t.push_back(estimateSegmentTimes(all_v.back(), 2.0 + 0.05 * (b % 40), 3.0 + 0.1 * (b % 50)));
    }
    BatchPolynomialOptimization<N> batch(D);
    batch.setupFromVertices(all_v, all_t, derivative_order::SNAP);
    if (!batch.solveLinear()) return 3;
    InputConstraints ic;
    ic.setDefaultValues();
    std::vector<InputFeasibilityResult> res;
    std::vector<int> seg;
    if (!batch.checkInputFeasibilitySampling(ic, 0.05, &res, &seg)) return 3;
    FeasibilitySampling::Settings settings;
    settings.setSamplingIntervalS(-0.05);  // abs() is taken, as in the reference
    FeasibilitySampling f(settings, ic);
    std::vector<int32_t> hr(B), hs(B), br(res.begin(), res.end()), bs(seg.begin(), seg.end());
    for (int b = 0; b < B; ++b) {
      Segment::Vector segs;
      batch.getSegments(b, &segs);
      check_host(f, segs, &hr[b], &hs[b]);
    }
    FILE* out = std::fopen(argv[2], "wb");
    if (!out) return 2;
    const int32_t hdr[4] = {B, K, D, N};
    std::fwrite(hdr, 4, 4, out);
    std::fwrite(batch.segmentTimes(), 8, size_t(B) * K, out);
    std::fwrite(batch.coefficients(), 8, size_t(B) * K * D * N, out);
    std::fwrite(br.data(), 4, B, out);
    std::fwrite(bs.data(), 4, B, out);
    std::fwrite(hr.data(), 4, B, out);
    std::fwrite(hs.data(), 4, B, out);
    std::fclose(out);
    std::printf("batch class: %d trajectories checked\n", B);
    return 0;
  }
  std::fprintf(stderr, "usage: %s mirror IN OUT | batch OUT\n", argv[0]);
  return 1;
}
