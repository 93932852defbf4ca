// The single-object host half-plane check (HalfPlane, createBoundingBox, FeasibilityBase::checkHalfPlaneFeasibility)
// and the batched BatchPolynomialOptimization<N>::checkHalfPlaneFeasibility, driven by tests/test_half_plane_cpu.py
// and tests/test_half_plane_feasibility.py.
//   test_half_plane reference        host only: the reference test's parabola (x = t, z = t^2, T = 1, N = 3 and N = 4
//                                    with a zero cubic term) against a plane shifted down by z -= 0.05 and a box grown
//                                    by l += 0.05, with the reference test's expectations; exit 0 when all hold
//   test_half_plane planes IN OUT    host only: IN = int32 n, then n records of int32 kind and double[9]
//                                    (0: point, normal; 1: a, b, c; 2: box center, size) -> OUT = the planes, [rows][6]
//   test_half_plane mirror IN OUT    host only: IN = int32 B, K, D, N, P; double planes [P][6] (used as given), times
//                                    [B][K], coeffs [B][K][D][N] -> OUT = int32 feasible [B], segment [B], plane [B]
//   test_half_plane batch OUT        needs the GPU: solves B = 96 random-vertex problems (N = 10, D = 3, K = 5) and
//                                    writes int32 B, K, D, N, P; planes; times; coeffs; the batch's feasible, segment
//                                    and plane; the host check's feasible, segment and plane
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "mav_trajectory_generation/batch_polynomial_optimization.h"
#include "mav_trajectory_generation/polynomial_optimization_linear.h"
#include "mav_trajectory_generation_ros/feasibility_base.h"

using namespace mav_trajectory_generation;

// feasible, first failing segment and plane (-1 when none) of the host check on one trajectory
static void check_host(const FeasibilityBase& f, const Segment::Vector& segs, int32_t* ok, int32_t* segment,
                       int32_t* plane) {
  Trajectory t;
  t.setSegments(segs);
  *ok = f.checkHalfPlaneFeasibility(t) ? 1 : 0;
  *segment = *plane = -1;
  for (size_t i = 0; i < segs.size() && *segment < 0; ++i) {
    if (segs[i].D() != 3 && segs[i].D() != 4) {
      *segment = static_cast<int32_t>(i);
      break;
    }
    for (size_t p = 0; p < f.half_plane_constraints_.size(); ++p) {
      FeasibilityBase one;
      one.half_plane_constraints_.push_back(f.half_plane_constraints_[p]);
      if (!one.checkHalfPlaneFeasibility(segs[i])) {
        *segment = static_cast<int32_t>(i);
        *plane = static_cast<int32_t>(p);
        break;
      }
    }
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

// a plane exactly as given (HalfPlane's constructor would normalise the normal)
static HalfPlane as_given(const double* row) {
  HalfPlane hp(Eigen::Vector3d(0.0, 0.0, 0.0), Eigen::Vector3d(1.0, 0.0, 0.0));
  for (int d = 0; d < 3; ++d) {
    hp.point[d] = row[d];
    hp.normal[d] = row[3 + d];
  }
  return hp;
}

static bool read_all(FILE* f, void* p, size_t bytes) { return std::fread(p, 1, bytes, f) == bytes; }

static int reference_test() {
  int failures = 0;
  for (int N : {3, 4}) {
    Segment segment(N, 3);
    Eigen::VectorXd cx = Eigen::VectorXd::Zero(N), cy = Eigen::VectorXd::Zero(N), cz = Eigen::VectorXd::Zero(N);
    cx[1] = 1.0;  // x = t
    cz[2] = 1.0;  // z = t^2
    segment[0] = Polynomial(cx);
    segment[1] = Polynomial(cy);
    segment[2] = Polynomial(cz);
    segment.setTime(1.0);
    FeasibilityBase check;
    Eigen::Vector3d point(0.0, 0.0, 0.0);
    const Eigen::Vector3d normal(-1.0, 0.0, 1.0);
    int steps = 0;
    while (point.z() > -1.0) {
      check.half_plane_constraints_.clear();
      check.half_plane_constraints_.emplace_back(point, normal);
      const bool feasible = check.checkHalfPlaneFeasibility(segment);
      if (feasible != !(point.z() >= -0.25)) {
        std::printf("N=%d plane z=%.17g: feasible=%d\n", N, point.z(), int(feasible));
        ++failures;
      }
      point.z() -= 0.05;
      ++steps;
    }
    FeasibilityBase box;
    double l = 0.0;
    int boxes = 0;
    while (l < 4.0) {
      box.half_plane_constraints_ = HalfPlane::createBoundingBox(Eigen::Vector3d(0.0, 0.0, 0.0),
                                                                 Eigen::Vector3d(l, l, l));
      const bool feasible = box.checkHalfPlaneFeasibility(segment);
      if (feasible != !(l <= 2.0)) {
        std::printf("N=%d box l=%.17g: feasible=%d\n", N, l, int(feasible));
        ++failures;
      }
      l += 0.05;
      ++boxes;
    }
    std::printf("reference test N=%d: %d planes, %d boxes\n", N, steps, boxes);
  }
  return failures ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc == 2 && !std::strcmp(argv[1], "reference")) return reference_test();
  if (argc == 4 && !std::strcmp(argv[1], "planes")) {
    FILE* in = std::fopen(argv[2], "rb");
    if (!in) return 2;
    int32_t n;
    if (!read_all(in, &n, 4)) return 2;
    std::vector<double> out;
    for (int i = 0; i < n; ++i) {
      int32_t kind;
      double v[9];
      if (!read_all(in, &kind, 4) || !read_all(in, v, sizeof(v))) return 2;
      const Eigen::Vector3d a(v[0], v[1], v[2]), b(v[3], v[4], v[5]), c(v[6], v[7], v[8]);
      HalfPlane::Vector planes;
      if (kind == 0) planes.emplace_back(a, b);
      else if (kind == 1) planes.emplace_back(a, b, c);
      else planes = HalfPlane::createBoundingBox(a, b);
      for (const HalfPlane& hp : planes)
        for (int d = 0; d < 6; ++d) out.push_back(d < 3 ? hp.point[d] : hp.normal[d - 3]);
    }
    std::fclose(in);
    FILE* o = std::fopen(argv[3], "wb");
    if (!o) return 2;
    std::fwrite(out.data(), 8, out.size(), o);
    std::fclose(o);
    return 0;
  }
  if (argc == 4 && !std::strcmp(argv[1], "mirror")) {
    FILE* in = std::fopen(argv[2], "rb");
    if (!in) return 2;
    int32_t hdr[5];
    if (!read_all(in, hdr, sizeof(hdr))) return 2;
    const int B = hdr[0], K = hdr[1], D = hdr[2], N = hdr[3], P = hdr[4];
    std::vector<double> planes(size_t(P) * 6), times(size_t(B) * K), coeffs(size_t(B) * K * D * N);
    if (!read_all(in, planes.data(), planes.size() * 8) || !read_all(in, times.data(), times.size() * 8) ||
        !read_all(in, coeffs.data(), coeffs.size() * 8))
      return 2;
    std::fclose(in);
    FeasibilityBase f;
    for (int p = 0; p < P; ++p) f.half_plane_constraints_.push_back(as_given(&planes[size_t(p) * 6]));
    std::vector<int32_t> ok(B), seg(B), pl(B);
    for (int b = 0; b < B; ++b)
      check_host(f, segments_of(&times[size_t(b) * K], &coeffs[size_t(b) * K * D * N], K, D, N), &ok[b], &seg[b],
                 &pl[b]);
    FILE* out = std::fopen(argv[3], "wb");
    if (!out) return 2;
    std::fwrite(ok.data(), 4, B, out);
    std::fwrite(seg.data(), 4, B, out);
    std::fwrite(pl.data(), 4, B, out);
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
      all_v.push_back(createRandomVertices(derivative_order::SNAP, K, lo, hi, 6100 + b));
      all_t.push_back(estimateSegmentTimes(all_v.back(), 2.0 + 0.05 * (b % 40), 3.0 + 0.1 * (b % 50)));
    }
    BatchPolynomialOptimization<N> batch(D);
    batch.setupFromVertices(all_v, all_t, derivative_order::SNAP);
    if (!batch.solveLinear()) return 3;
    FeasibilityBase f;
    f.half_plane_constraints_ = HalfPlane::createBoundingBox(Eigen::Vector3d(0.0, 0.0, 0.0),
                                                             Eigen::Vector3d(10.5, 10.5, 10.5));
    f.half_plane_constraints_.emplace_back(Eigen::Vector3d(0.0, 0.0, -4.0), Eigen::Vector3d(0.3, -0.2, 1.0));
    std::vector<uint8_t> ok;
    std::vector<int> seg, pl;
    if (!batch.checkHalfPlaneFeasibility(f.half_plane_constraints_, &ok, &seg, &pl)) return 3;
    const int P = static_cast<int>(f.half_plane_constraints_.size());
    std::vector<int32_t> hf(B), hs(B), hp(B), bf(ok.begin(), ok.end()), bs(seg.begin(), seg.end()),
        bp(pl.begin(), pl.end());
    for (int b = 0; b < B; ++b) {
      Segment::Vector segs;
      batch.getSegments(b, &segs);
      check_host(f, segs, &hf[b], &hs[b], &hp[b]);
    }
    FILE* out = std::fopen(argv[2], "wb");
    if (!out) return 2;
    const int32_t hdr[5] = {B, K, D, N, P};
    std::fwrite(hdr, 4, 5, out);
    for (const HalfPlane& h : f.half_plane_constraints_) {
      std::fwrite(h.point.data(), 8, 3, out);
      std::fwrite(h.normal.data(), 8, 3, out);
    }
    std::fwrite(batch.segmentTimes(), 8, size_t(B) * K, out);
    std::fwrite(batch.coefficients(), 8, size_t(B) * K * D * N, out);
    for (const std::vector<int32_t>* v : {&bf, &bs, &bp, &hf, &hs, &hp}) std::fwrite(v->data(), 4, B, out);
    std::fclose(out);
    std::printf("batch class: %d trajectories checked against %d planes\n", B, P);
    return 0;
  }
  std::fprintf(stderr, "usage: %s reference | planes IN OUT | mirror IN OUT | batch OUT\n", argv[0]);
  return 1;
}
