// The reference README's 3-vertex example (README.md:105-139 of ethz-asl/mav_trajectory_generation), unchanged
// apart from the include root: solveLinear() runs on the H100 behind include/mtg_b200.h.
//
//   g++ -std=c++17 -I mav_trajectory_generation_b200/host/include -I include examples/readme_example.cpp \
//       -L mav_trajectory_generation_b200 -lmtg_host -lmtg_b200 -Wl,-rpath,$PWD/mav_trajectory_generation_b200 -o readme_example
#include <cstdio>

#include <mav_trajectory_generation/polynomial_optimization_linear.h>

using namespace mav_trajectory_generation;

int main() {
  Vertex::Vector vertices;
  const int dimension = 3;
  const int derivative_to_optimize = derivative_order::SNAP;
  Vertex start(dimension), middle(dimension), end(dimension);

  start.makeStartOrEnd(Eigen::Vector3d(0, 0, 1), derivative_to_optimize);
  vertices.push_back(start);
  middle.addConstraint(derivative_order::POSITION, Eigen::Vector3d(1, 2, 3));
  vertices.push_back(middle);
  end.makeStartOrEnd(Eigen::Vector3d(2, 1, 5), derivative_to_optimize);
  vertices.push_back(end);

  const double v_max = 2.0, a_max = 2.0;
  std::vector<double> segment_times = estimateSegmentTimes(vertices, v_max, a_max);

  const int N = 10;
  PolynomialOptimization<N> opt(dimension);
  opt.setupFromVertices(vertices, segment_times, derivative_to_optimize);
  opt.solveLinear();

  Segment::Vector segments;
  opt.getSegments(&segments);
  Trajectory trajectory;
  opt.getTrajectory(&trajectory);

  std::printf("segments: %d, total time %.6f s, cost %.6f\n", trajectory.K(), trajectory.getMaxTime(), opt.computeCost());
  for (double t = 0.0; t <= trajectory.getMaxTime(); t += trajectory.getMaxTime() / 4.0) {
    const Eigen::VectorXd p = trajectory.evaluate(t, derivative_order::POSITION);
    std::printf("t = %.3f  position = (%.4f, %.4f, %.4f)\n", t, p[0], p[1], p[2]);
  }
  return 0;
}
