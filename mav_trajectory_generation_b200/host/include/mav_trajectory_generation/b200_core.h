// b200_core.h -- non-template implementation behind PolynomialOptimization<N> and
// BatchPolynomialOptimization<N>: packs Vertex constraints into the flat buffers of the C-ABI
// (include/mtg_b200.h), calls the sm_90a kernels, unpacks Segment::Vector.
// There is no host solve in here -- only index bookkeeping and the small debug matrices the
// reference exposes (getA/getAInverse/getM/getR), which are built from the same exact tables
// the kernels use.
#ifndef MAV_TRAJECTORY_GENERATION_B200_CORE_H_
#define MAV_TRAJECTORY_GENERATION_B200_CORE_H_

#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "mav_trajectory_generation/segment.h"
#include "mav_trajectory_generation/trajectory.h"
#include "mav_trajectory_generation/vertex.h"

struct mtg_handle;

namespace mav_trajectory_generation {
namespace b200 {

// Process-wide handle (device from env MTG_B200_DEVICE, default 0), created on first use.
// Aborts with a clear message when no sm_90 device / library is available: the GPU path is
// the only path.
mtg_handle* defaultHandle();
// Serialises callers of the shared handle (a handle is single-caller, include/mtg_b200.h).
void lockHandle();
void unlockHandle();

// Row-major N x N host matrices built from the exact tables (debug accessors / static helpers).
void hostMappingMatrix(int N, double T, double* A);
void hostInverseMappingMatrix(int N, double T, double* Ai);
// A^-1 of a GIVEN row-major N x N mapping matrix A = [[Lambda, 0], [C, Dm]] (reference linear_impl.h:142-179)
void hostInvertStructured(int N, const double* A, double* Ai);
void hostCostMatrix(int N, int derivative, double T, double* Q);
void hostSegmentHessian(int N, int derivative, double T, double* H);  // A^-T Q A^-1

struct Topology {
  int N = 0, K = 0, D = 0, r = -1;
  int n_all = 0, n_fixed = 0, n_free = 0, kernel = 0;
  std::vector<uint8_t> mask;       // [K+1][N/2]
  std::vector<int32_t> slot_col;   // [K*N]
};

// Drops constraints above N/2-1 (with a warning, like the reference linear_impl.h:84-105) and fills topo.
void buildTopology(int N, int D, int r, Vertex::Vector* vertices, Topology* topo);
// d_fixed[D][n_fixed] of one problem, reference compact order.
void packFixed(const Topology& topo, const Vertex::Vector& vertices, double* d_fixed);
// Checks that `vertices` fixes exactly the derivatives topo.mask says.
bool sameTopology(const Topology& topo, const Vertex::Vector& vertices);
void unpackSegments(const Topology& topo, const double* coeffs, const double* times, Segment::Vector* segments);

class LinearCore {
 public:
  LinearCore(int N, size_t dimension);
  bool setupFromVertices(const Vertex::Vector& vertices, const std::vector<double>& times, int r);
  void updateSegmentTimes(const std::vector<double>& times);
  bool solveLinear();
  void setFreeConstraints(const std::vector<Eigen::VectorXd>& free_constraints);
  double computeCost() const;
  void getAInverse(Eigen::MatrixXd* A_inv) const;
  void getA(Eigen::MatrixXd* A) const;
  void getM(Eigen::MatrixXd* M) const;
  void getMpinv(Eigen::MatrixXd* M_pinv) const;
  void getR(Eigen::MatrixXd* R) const;

  int N_;
  size_t dimension_;
  Topology topo_;
  Vertex::Vector vertices_;
  Segment::Vector segments_;
  std::vector<double> segment_times_;
  std::vector<Eigen::VectorXd> fixed_constraints_compact_, free_constraints_compact_;
  int last_status_ = 0;

 private:
  void unpack(const std::vector<double>& coeffs);
};

// The time objective of PolynomialOptimizationNonLinear (reference NonlinearOptimizationParameters fields and defaults)
struct TimeObjectiveParameters {
  bool richter_time = false;  // kRichterTime*: time_penalty * T_total; otherwise time_penalty * T_total^2
  double time_penalty = 500.0;
  double soft_constraint_weight = 100.0;
  double maximum_cost = 1e12;  // clamp of each soft term (1e9 in getTotalCostWithSoftConstraints)
  std::vector<std::pair<int, double> > soft_constraints;  // (derivative, max value > 0), summed in this order; <= 8
};

class BatchCore {
 public:
  BatchCore(int N, size_t dimension);
  ~BatchCore();
  BatchCore(const BatchCore&) = delete;
  BatchCore& operator=(const BatchCore&) = delete;
  bool setupFromVertices(const std::vector<Vertex::Vector>& vertices, const std::vector<std::vector<double>>& times,
                         int r);
  bool setupFromWaypoints(size_t B, size_t K, const double* positions, const double* times, int r);
  bool solveLinear();
  // time allocation (Nfabian) + packing + solve in one device pass; fills times_ and coeffs_
  bool solveWaypointsNfabian(size_t B, size_t K, const double* positions, int r, double v_max, double a_max,
                             double magic);
  std::vector<double> computeCosts() const;
  // batched getCostAndGradientMellinger at the current segment times (grad: [B][K])
  void costGradientMellinger(std::vector<double>* cost, std::vector<double>* grad) const;
  // batched Trajectory::evaluateRange of the solved trajectories (samples: [B][max_samples][n_derivs][D])
  void evaluateRange(double t_start, double t_end, double dt, const std::vector<int>& derivatives, int max_samples,
                     std::vector<double>* samples, std::vector<int32_t>* n_samples,
                     std::vector<double>* sampling_times) const;
  // batched computeMaximumOfMagnitude of the current coefficients (maxima: [B][n_derivs])
  void computeMaximaOfMagnitude(const std::vector<int>& derivatives, std::vector<Extremum>* maxima) const;
  // objectiveFunctionTime (d_free == nullptr) / objectiveFunctionTimeAndConstraints at the current segment times;
  // the solved coefficients replace coeffs_ (objective: [B], terms: [B][3] or nullptr)
  bool timeObjective(const TimeObjectiveParameters& params, const double* d_free, std::vector<double>* objective,
                     std::vector<double>* terms);
  void getSegments(size_t b, Segment::Vector* segments) const;

  int N_;
  size_t dimension_;
  size_t B_ = 0;
  Topology topo_;
  // pinned host buffers (mtg_host_alloc)
  double* times_ = nullptr;     // [B][K]
  double* d_fixed_ = nullptr;   // [B][D][n_fixed]
  double* coeffs_ = nullptr;    // [B][K][D][N]
  double* d_free_ = nullptr;    // [B][D][n_free]
  int32_t* status_ = nullptr;   // [B]

 private:
  void allocate(size_t B);
  void release();
};

}  // namespace b200
}  // namespace mav_trajectory_generation
#endif
