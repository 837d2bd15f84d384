// Reference-side binding #1 (INTEGRATION.md section 1): karto::ScanSolver implemented on the b200slam C ABI.
// In a slam_toolbox workspace this class is exported with PLUGINLIB_EXPORT_CLASS and listed in
// solver_plugins.xml; here it is compiled against the reference headers (+ oracle/stubs for the absent
// Boost / Eigen / rclcpp headers) and driven by the reference's own karto::Mapper in integration/replay_driver.cpp.
#pragma once
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "karto_sdk/Mapper.h"
#include "b200slam.h"

namespace solver_plugins {

class B200Solver : public karto::ScanSolver
{
public:
  B200Solver() { b200pg_create(nullptr, &h_); }
  ~B200Solver() override { b200pg_destroy(h_); }

  // CeresSolver::Configure (solvers/ceres_solver.cpp:25-193) reads the `ceres_*` ROS parameters.  With rclcpp present
  // (B200_WITH_ROS, see INTEGRATION.md) the node's parameters are read here; the mapping itself is ConfigureFromStrings so
  // that it can be exercised without ROS (integration/replay_driver.cpp: krep_solver_configure).
  void Configure(rclcpp_lifecycle::LifecycleNode::SharedPtr node) override
  {
#ifdef B200_WITH_ROS
    std::map<std::string, std::string> kv;
    for (const char * k : {"ceres_linear_solver", "ceres_preconditioner", "ceres_trust_strategy", "ceres_dogleg_type", "ceres_loss_function",
                           "b200_linear_solver"}) {
      std::string v;
      if (!node->has_parameter(k)) node->declare_parameter(k, std::string(""));
      if (node->get_parameter(k, v) && !v.empty()) kv[k] = v;
    }
    ConfigureFromStrings(kv);
#else
    (void)node;
#endif
  }
  // Returns the number of keys that were understood and applied; the rest are reported on stderr like the reference's
  // RCLCPP_WARN fall-backs (ceres_solver.cpp:44-94).  The linear solver / preconditioner / dogleg keys select Ceres internals
  // that have one counterpart here (block-sparse PCG with a two-level preconditioner inside Levenberg-Marquardt).
  int ConfigureFromStrings(const std::map<std::string, std::string> & kv)
  {
    std::lock_guard<std::mutex> lock(mu_);
    b200pg_opts o;
    b200pg_get_opts(h_, &o);
    int applied = 0;
    for (const auto & e : kv) {
      const std::string & k = e.first, & v = e.second;
      if (k == "ceres_loss_function") {   // ceres_solver.cpp:82-94
        if (v == "None") { o.loss_function = 0; ++applied; }
        else if (v == "HuberLoss") { o.loss_function = 1; o.loss_scale = 0.7; ++applied; }
        else if (v == "CauchyLoss") { o.loss_function = 2; o.loss_scale = 0.7; ++applied; }
        else fprintf(stderr, "B200Solver: unknown ceres_loss_function '%s', keeping the squared loss\n", v.c_str());
      } else if (k == "ceres_trust_strategy") {   // :68-76
        if (v == "LEVENBERG_MARQUARDT") ++applied;
        else fprintf(stderr, "B200Solver: trust strategy '%s' is not available, using LEVENBERG_MARQUARDT\n", v.c_str());
      } else if (k == "b200_linear_solver") {   // this library's own choice; ceres_linear_solver does not select it
        if (v == "PCG") { o.linear_solver_type = 0; ++applied; }
        else if (v == "SPARSE_NORMAL_CHOLESKY") { o.linear_solver_type = 1; ++applied; }
        else fprintf(stderr, "B200Solver: unknown b200_linear_solver '%s', keeping the current linear solver\n", v.c_str());
      } else if (k == "ceres_linear_solver" || k == "ceres_preconditioner" || k == "ceres_dogleg_type") {
        ++applied;   // accepted: the linear solve is the library's block-sparse PCG whatever Ceres back end is named
      } else if (k == "max_num_iterations") { o.max_num_iterations = atoi(v.c_str()); ++applied; }
      else if (k == "function_tolerance") { o.function_tolerance = atof(v.c_str()); ++applied; }
      else if (k == "gradient_tolerance") { o.gradient_tolerance = atof(v.c_str()); ++applied; }
      else if (k == "parameter_tolerance") { o.parameter_tolerance = atof(v.c_str()); ++applied; }
      else fprintf(stderr, "B200Solver: unknown option '%s'\n", k.c_str());
    }
    if (b200pg_set_opts(h_, &o) != B200_OK) return -1;
    return applied;
  }

  // the options ConfigureFromStrings left on the handle
  b200pg_opts GetOptions() const
  {
    std::lock_guard<std::mutex> lock(mu_);
    b200pg_opts o;
    b200pg_get_opts(h_, &o);
    return o;
  }

  void Compute() override   // solvers/ceres_solver.cpp:214-269
  {
    std::lock_guard<std::mutex> lock(mu_);   // CeresSolver takes nodes_mutex_ in every method (ceres_solver.cpp:217 ...)
    ++computes_;
    b200pg_summary s;
    if (b200pg_solve(h_, &s) != B200_OK) return;   // unusable: corrections untouched, like the reference
    solve_ms_ += s.solve_ms;
    compute_log_.push_back({s.solve_ms, s.uploaded_edges});
    const int n = b200pg_num_nodes(h_);
    std::vector<int32_t> ids(n);
    std::vector<double> p(3 * (size_t)n);
    const int m = b200pg_get_corrections(h_, ids.data(), p.data(), n);
    corrections_.clear();
    corrections_.reserve(m);
    for (int i = 0; i < m; ++i) corrections_.emplace_back(ids[i], karto::Pose2(p[3 * i], p[3 * i + 1], p[3 * i + 2]));
  }
  const karto::ScanSolver::IdPoseVector & GetCorrections() const override { return corrections_; }
  void Clear() override { std::lock_guard<std::mutex> lock(mu_); corrections_.clear(); b200pg_clear(h_); }
  void Reset() override { std::lock_guard<std::mutex> lock(mu_); corrections_.clear(); ids_.clear(); b200pg_reset(h_); }

  void AddNode(karto::Vertex<karto::LocalizedRangeScan> * v) override   // ceres_solver.cpp:317-336
  {
    if (!v) return;
    std::lock_guard<std::mutex> lock(mu_);
    const karto::Pose2 p = v->GetObject()->GetCorrectedPose();
    const double pose[3] = {p.GetX(), p.GetY(), p.GetHeading()};
    if (b200pg_add_node(h_, v->GetObject()->GetUniqueId(), pose) == B200_OK) ids_.push_back(v->GetObject()->GetUniqueId());
  }
  void AddConstraint(karto::Edge<karto::LocalizedRangeScan> * e) override   // ceres_solver.cpp:339-392
  {
    if (!e) return;
    std::lock_guard<std::mutex> lock(mu_);
    karto::LinkInfo * li = static_cast<karto::LinkInfo *>(e->GetLabel());
    const karto::Pose2 d = li->GetPoseDifference();
    const karto::Matrix3 c = li->GetCovariance();
    const double z[3] = {d.GetX(), d.GetY(), d.GetHeading()};
    double cov[9];
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) cov[3 * r + k] = c(r, k);
    b200pg_add_edge(h_, e->GetSource()->GetObject()->GetUniqueId(), e->GetTarget()->GetObject()->GetUniqueId(), z, cov);
  }
  void RemoveNode(kt_int32s id) override
  {
    std::lock_guard<std::mutex> lock(mu_);
    if (b200pg_remove_node(h_, id) != B200_OK) return;
    for (size_t i = 0; i < ids_.size(); ++i)
      if (ids_[i] == id) { ids_.erase(ids_.begin() + i); break; }
  }
  void RemoveConstraint(kt_int32s a, kt_int32s b) override { std::lock_guard<std::mutex> lock(mu_); b200pg_remove_edge(h_, a, b); }
  void ModifyNode(const int & id, Eigen::Vector3d pose) override
  {
    std::lock_guard<std::mutex> lock(mu_);
    const double p[3] = {pose(0), pose(1), pose(2)};
    b200pg_modify_node(h_, id, p);
  }
  void GetNodeOrientation(const int & id, double & yaw) override
  {
    std::lock_guard<std::mutex> lock(mu_);
    double p[3];
    if (b200pg_get_node(h_, id, p) == B200_OK) yaw = p[2];
  }

  // the raw node store for visualisation (ceres_solver.cpp:474-479, used by src/loop_closure_assistant.cpp:161):
  // a host copy of the nodes as the library holds them now, refreshed on every call.  The returned pointer stays valid
  // until the next getGraph() call (the reference hands out a pointer into its live store under the same rule).
  std::unordered_map<int, Eigen::Vector3d> * getGraph() override
  {
    std::lock_guard<std::mutex> lock(mu_);
    graph_.clear();
    for (int id : ids_) {
      double p[3];
      if (b200pg_get_node(h_, id, p) != B200_OK) continue;
      Eigen::Vector3d v;
      v(0) = p[0]; v(1) = p[1]; v(2) = p[2];
      graph_[id] = v;
    }
    return &graph_;
  }

  int computes() const { return computes_; }
  double solve_ms() const { return solve_ms_; }
  // one record per successful Compute: device ms of the solve and the constraints it uploaded (all of them after a removal)
  struct ComputeRecord { double solve_ms; int uploaded_edges; };
  const std::vector<ComputeRecord> & compute_log() const { return compute_log_; }
  int num_nodes() const { std::lock_guard<std::mutex> lock(mu_); return b200pg_num_nodes(h_); }
  int num_edges() const { std::lock_guard<std::mutex> lock(mu_); return b200pg_num_edges(h_); }

private:
  mutable std::mutex mu_;                                 // mirrors CeresSolver::nodes_mutex_
  b200pg * h_ = nullptr;
  karto::ScanSolver::IdPoseVector corrections_;
  std::vector<int> ids_;                                  // node ids in insertion order
  std::unordered_map<int, Eigen::Vector3d> graph_;
  int computes_ = 0;
  double solve_ms_ = 0.0;
  std::vector<ComputeRecord> compute_log_;
};

}  // namespace solver_plugins
