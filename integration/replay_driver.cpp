// cfg3 replay driver: the reference's own karto::Mapper::Process (Mapper.cpp:2679-2749) fed with posed
// scans, with the GPU ScanSolver adapter installed through Mapper::SetScanSolver and -- when linked into
// libreplay_b200.so -- every MatchScan redirected to the GPU by scan_matcher_b200.cpp.
// libreplay_ref.so is the same driver linked WITHOUT the matcher shim (reference CPU matcher).
// Localization mode (src/slam_toolbox_localization.cpp:176-237) runs through the same mapper: ProcessLocalization,
// ProcessAgainstNodesNearBy and ClearLocalizationBuffer.  There the mapper deletes the scans it drops from its rolling
// buffer, so the driver holds no scan pointers of its own: every readout walks the mapper's current processed set.
#include <chrono>
#include <csignal>
#include <cstdlib>
#include <execinfo.h>
#include <string>
#include <unistd.h>

#include "karto_sdk/Mapper.h"
#include "b200_solver.hpp"
#include "occupancy_b200.hpp"

using namespace karto;

namespace {
struct Replay {
  Mapper mapper;
  solver_plugins::B200Solver * solver = nullptr;
  double process_seconds = 0.0;
};
const char * kLaser = "laser0";

// a new scan at the odometric pose, corrected pose = odometric pose (SlamToolbox::getLocalizedRangeScan)
LocalizedRangeScan * make_scan(const double * ranges, int n, const double odom[3], int id)
{
  RangeReadingsVector rr(ranges, ranges + n);
  LocalizedRangeScan * s = new LocalizedRangeScan(Name(kLaser), rr);
  Pose2 p(odom[0], odom[1], odom[2]);
  s->SetOdometricPose(p);
  s->SetCorrectedPose(p);
  s->SetTime(static_cast<double>(id));
  return s;
}

// the scans the mapper holds now (Mapper::GetAllProcessedScans: unique-id order, which is processing order)
LocalizedRangeScanVector processed_scans(Replay * r) { return r->mapper.GetAllProcessedScans(); }

// The localization calls remove nodes through m_pScanOptimizer without a check (Mapper.cpp:2977, 3003), and a rolling
// buffer of 0 scans would delete the scan being processed before the caller reads its pose.
bool can_localize(Replay * r) { return r->solver != nullptr && r->mapper.getParamScanBufferSize() >= 1; }

// runs one mapper call on a new scan; the scan is the mapper's once processed, else deleted.  Writes the corrected pose and
// the covariance the localization node publishes (slam_toolbox_localization.cpp:195-233).
template <class F>
int run_scan(Replay * r, LocalizedRangeScan * s, const char * what, F && call, double * out_pose, double * out_cov)
{
  Matrix3 cov;
  cov.SetToIdentity();
  auto t0 = std::chrono::steady_clock::now();
  bool ok = false;
  try {
    ok = call(s, &cov);
  } catch (const std::exception & e) {
    std::fprintf(stderr, "%s: %s\n", what, e.what());
  }
  r->process_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (!ok) { delete s; return 0; }
  if (out_pose) {
    const Pose2 & p = s->GetCorrectedPose();
    out_pose[0] = p.GetX(); out_pose[1] = p.GetY(); out_pose[2] = p.GetHeading();
  }
  if (out_cov) for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) out_cov[3 * i + j] = cov(i, j);
  return 1;
}
}

static void segv_handler(int)
{
  void * frames[64];
  int n = backtrace(frames, 64);
  backtrace_symbols_fd(frames, n, 2);
  _exit(139);
}

extern "C" {

int krep_init_laser(double min_angle, double max_angle, double ang_res, double min_range, double max_range, double range_threshold)
{
  if (getenv("B200_TRACE")) signal(SIGSEGV, segv_handler);
  Name nm(kLaser);
  LaserRangeFinder * l = LaserRangeFinder::CreateLaserRangeFinder(LaserRangeFinder_Custom, nm);
  l->SetMinimumRange(min_range); l->SetMaximumRange(max_range);
  l->SetMinimumAngle(min_angle); l->SetMaximumAngle(max_angle);
  l->SetAngularResolution(ang_res); l->SetRangeThreshold(range_threshold);
  l->SetOffsetPose(Pose2(0.0, 0.0, 0.0));
  SensorManager::GetInstance()->RegisterSensor(l);
  return static_cast<int>(l->GetNumberOfRangeReadings());
}

void * krep_create(int use_solver)
{
  Replay * r = new Replay();
  if (use_solver) {
    r->solver = new solver_plugins::B200Solver();
    r->mapper.SetScanSolver(r->solver);
  }
  return r;
}

// B200Solver::ConfigureFromStrings (the mapping CeresSolver::Configure applies to the ceres_* ROS parameters): returns the
// number of keys applied, -1 without a solver
int krep_solver_configure(void * rp, const char * key, const char * value)
{
  Replay * r = static_cast<Replay *>(rp);
  if (!r->solver) return -1;
  return r->solver->ConfigureFromStrings({{std::string(key), std::string(value)}});
}

// b200pg_opts.linear_solver_type of the adapter's handle (what b200_linear_solver selected), -1 without a solver
int krep_solver_linear_solver_type(void * rp)
{
  Replay * r = static_cast<Replay *>(rp);
  return r->solver ? r->solver->GetOptions().linear_solver_type : -1;
}

// Mapper::Reset (Mapper.cpp:2656-2677) deletes both scan matchers; krep_destroy deletes the mapper.  With the matcher shim
// linked, b200_shim_live_handles() must drop to 0 afterwards (no leaked device state).
void krep_reset_mapper(void * rp) { static_cast<Replay *>(rp)->mapper.Reset(); }
void krep_destroy(void * rp)
{
  Replay * r = static_cast<Replay *>(rp);
  solver_plugins::B200Solver * s = r->solver;
  delete r;
  delete s;
}

int krep_set(void * rp, const char * name, double v)
{
  Mapper * m = &static_cast<Replay *>(rp)->mapper;
  std::string n(name);
  if (n == "coarse_search_angle_offset") m->setParamCoarseSearchAngleOffset(v);
  else if (n == "coarse_angle_resolution") m->setParamCoarseAngleResolution(v);
  else if (n == "fine_search_angle_offset") m->setParamFineSearchAngleOffset(v);
  else if (n == "distance_variance_penalty") m->setParamDistanceVariancePenalty(v);
  else if (n == "angle_variance_penalty") m->setParamAngleVariancePenalty(v);
  else if (n == "minimum_distance_penalty") m->setParamMinimumDistancePenalty(v);
  else if (n == "minimum_angle_penalty") m->setParamMinimumAnglePenalty(v);
  else if (n == "use_response_expansion") m->setParamUseResponseExpansion(v != 0.0);
  else if (n == "correlation_search_space_dimension") m->setParamCorrelationSearchSpaceDimension(v);
  else if (n == "correlation_search_space_resolution") m->setParamCorrelationSearchSpaceResolution(v);
  else if (n == "correlation_search_space_smear_deviation") m->setParamCorrelationSearchSpaceSmearDeviation(v);
  else if (n == "loop_search_space_dimension") m->setParamLoopSearchSpaceDimension(v);
  else if (n == "loop_search_space_resolution") m->setParamLoopSearchSpaceResolution(v);
  else if (n == "loop_search_space_smear_deviation") m->setParamLoopSearchSpaceSmearDeviation(v);
  else if (n == "minimum_travel_distance") m->setParamMinimumTravelDistance(v);
  else if (n == "minimum_travel_heading") m->setParamMinimumTravelHeading(v);
  else if (n == "scan_buffer_size") m->setParamScanBufferSize(static_cast<int>(v));
  else if (n == "scan_buffer_maximum_scan_distance") m->setParamScanBufferMaximumScanDistance(v);
  else if (n == "link_match_minimum_response_fine") m->setParamLinkMatchMinimumResponseFine(v);
  else if (n == "link_scan_maximum_distance") m->setParamLinkScanMaximumDistance(v);
  else if (n == "loop_search_maximum_distance") m->setParamLoopSearchMaximumDistance(v);
  else if (n == "do_loop_closing") m->setParamDoLoopClosing(v != 0.0);
  else if (n == "loop_match_minimum_chain_size") m->setParamLoopMatchMinimumChainSize(static_cast<int>(v));
  else if (n == "loop_match_maximum_variance_coarse") m->setParamLoopMatchMaximumVarianceCoarse(v);
  else if (n == "loop_match_minimum_response_coarse") m->setParamLoopMatchMinimumResponseCoarse(v);
  else if (n == "loop_match_minimum_response_fine") m->setParamLoopMatchMinimumResponseFine(v);
  else if (n == "use_scan_matching") m->setParamUseScanMatching(v != 0.0);
  else if (n == "use_scan_barycenter") m->setParamUseScanBarycenter(v != 0.0);
  else if (n == "minimum_time_interval") m->setParamMinimumTimeInterval(v);
  else return -1;
  // After the first scan the running-scan buffer has its own copy of the two buffer limits.  Hand it the new ones as
  // Mapper::Initialize does for a loaded map (Mapper.cpp:2620-2623), the way the localization node starts on a map:
  // a localization buffer shorter than the running buffer would otherwise leave deleted scans among the running scans.
  if (MapperSensorManager * sm = m->GetMapperSensorManager()) {
    if (n == "scan_buffer_size") sm->SetRunningScanBufferSize(static_cast<kt_int32u>(v));
    else if (n == "scan_buffer_maximum_scan_distance") sm->SetRunningScanBufferMaximumDistance(v);
  }
  return 0;
}

// feeds one scan with its odometric pose; returns 1 if the mapper processed (kept) it
int krep_process(void * rp, const double * ranges, int n, const double odom[3], int id)
{
  Replay * r = static_cast<Replay *>(rp);
  return run_scan(r, make_scan(ranges, n, odom, id), "krep_process",
                  [r](LocalizedRangeScan * s, Matrix3 *) { return r->mapper.Process(s); }, nullptr, nullptr);
}

// Mapper::ProcessLocalization (Mapper.cpp:2831-2909), the localization node's PROCESS_LOCALIZATION step.  Returns 1 if the
// scan was processed (out_pose = its corrected pose, out_cov = the published covariance), 0 if not, -1 (nothing done)
// without a solver or with scan_buffer_size < 1.
int krep_process_localization(void * rp, const double * ranges, int n, const double odom[3], int id, double out_pose[3],
                              double out_cov[9])
{
  Replay * r = static_cast<Replay *>(rp);
  if (!can_localize(r)) return -1;
  return run_scan(r, make_scan(ranges, n, odom, id), "krep_process_localization",
                  [r](LocalizedRangeScan * s, Matrix3 * c) { return r->mapper.ProcessLocalization(s, c); }, out_pose, out_cov);
}

// PROCESS_NEAR_REGION (slam_toolbox_localization.cpp:197-212): the scan's odometric and corrected pose are set to the
// requested pose, then Mapper::ProcessAgainstNodesNearBy(scan, true, &cov) matches it against the map scan nearest to it
// and puts it in the rolling buffer.  Returns as krep_process_localization.
int krep_process_near(void * rp, const double * ranges, int n, const double odom[3], int id, const double pose[3],
                      double out_pose[3], double out_cov[9])
{
  Replay * r = static_cast<Replay *>(rp);
  if (!can_localize(r)) return -1;
  LocalizedRangeScan * s = make_scan(ranges, n, odom, id);
  const Pose2 p(pose[0], pose[1], pose[2]);
  s->SetOdometricPose(p);
  s->SetCorrectedPose(p);
  return run_scan(r, s, "krep_process_near",
                  [r](LocalizedRangeScan * s, Matrix3 * c) { return r->mapper.ProcessAgainstNodesNearBy(s, true, c); },
                  out_pose, out_cov);
}

// Mapper::ClearLocalizationBuffer (Mapper.cpp:2937-2962): every buffered scan leaves the graph and the solver, and the
// running and last scans are cleared.  0 on success, -1 (nothing done) without a solver or before the first scan.
int krep_clear_localization_buffer(void * rp)
{
  Replay * r = static_cast<Replay *>(rp);
  if (!can_localize(r) || !r->mapper.GetMapperSensorManager()) return -1;
  r->mapper.ClearLocalizationBuffer();
  return 0;
}

int krep_num_scans(void * rp) { return static_cast<int>(processed_scans(static_cast<Replay *>(rp)).size()); }

// corrected poses (after all loop closures) of the scans the mapper holds, in processing order; ids (if not NULL) receives
// their unique ids.  krep_num_scans gives the count.
void krep_poses(void * rp, double * out, int * ids)
{
  const LocalizedRangeScanVector v = processed_scans(static_cast<Replay *>(rp));
  for (size_t i = 0; i < v.size(); ++i) {
    const Pose2 & p = v[i]->GetCorrectedPose();
    out[3 * i] = p.GetX(); out[3 * i + 1] = p.GetY(); out[3 * i + 2] = p.GetHeading();
    if (ids) ids[i] = v[i]->GetUniqueId();
  }
}

// the mapper's graph edges (MapperGraph::GetEdges, insertion order): source / target unique ids, LinkInfo pose difference
// and covariance (row-major), filled up to cap.  Returns the number of edges.
int krep_edges(void * rp, int * src, int * dst, double * diff, double * cov, int cap)
{
  Replay * r = static_cast<Replay *>(rp);
  if (!r->mapper.GetGraph()) return 0;
  const std::vector<Edge<LocalizedRangeScan> *> & edges = r->mapper.GetGraph()->GetEdges();
  int k = 0;
  for (Edge<LocalizedRangeScan> * e : edges) {
    if (k < cap) {
      LinkInfo * li = static_cast<LinkInfo *>(e->GetLabel());
      src[k] = e->GetSource()->GetObject()->GetUniqueId();
      dst[k] = e->GetTarget()->GetObject()->GetUniqueId();
      const Pose2 d = li->GetPoseDifference();
      const Matrix3 c = li->GetCovariance();
      diff[3 * k] = d.GetX(); diff[3 * k + 1] = d.GetY(); diff[3 * k + 2] = d.GetHeading();
      for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) cov[9 * k + 3 * i + j] = c(i, j);
    }
    ++k;
  }
  return k;
}

// graph sizes: mapper vertices, mapper edges, solver nodes, solver edges (the solver's are -1 without one)
void krep_counts(void * rp, int out[4])
{
  Replay * r = static_cast<Replay *>(rp);
  MapperGraph * g = r->mapper.GetGraph();
  int nv = 0;
  if (g)
    for (const auto & kv : g->GetVertices()) nv += static_cast<int>(kv.second.size());
  out[0] = nv;
  out[1] = g ? static_cast<int>(g->GetEdges().size()) : 0;
  out[2] = r->solver ? r->solver->num_nodes() : -1;
  out[3] = r->solver ? r->solver->num_edges() : -1;
}

// per Compute of the adapter, in call order: device ms of the solve and the constraints it uploaded; filled up to cap.
// Returns the number of computes.
int krep_solver_computes(void * rp, double * ms, int * uploaded, int cap)
{
  Replay * r = static_cast<Replay *>(rp);
  if (!r->solver) return 0;
  const auto & log = r->solver->compute_log();
  for (size_t i = 0; i < log.size() && static_cast<int>(i) < cap; ++i) { ms[i] = log[i].solve_ms; uploaded[i] = log[i].uploaded_edges; }
  return static_cast<int>(log.size());
}

// ScanSolver::getGraph() of the adapter: number of nodes; ids / poses filled up to cap
int krep_solver_graph(void * rp, int * ids, double * poses, int cap)
{
  Replay * r = static_cast<Replay *>(rp);
  if (!r->solver) return 0;
  std::unordered_map<int, Eigen::Vector3d> * g = r->solver->getGraph();
  int k = 0;
  for (const auto & kv : *g) {
    if (k < cap) { ids[k] = kv.first; poses[3 * k] = kv.second(0); poses[3 * k + 1] = kv.second(1); poses[3 * k + 2] = kv.second(2); }
    ++k;
  }
  return k;
}

// stats: process seconds, solver computes, solver device ms, graph edges, graph vertices
void krep_stats(void * rp, double out[5])
{
  Replay * r = static_cast<Replay *>(rp);
  out[0] = r->process_seconds;
  out[1] = r->solver ? r->solver->computes() : 0;
  out[2] = r->solver ? r->solver->solve_ms() : 0;
  out[3] = static_cast<double>(r->mapper.GetGraph() ? r->mapper.GetGraph()->GetEdges().size() : 0);
  out[4] = static_cast<double>(processed_scans(r).size());
}

// map publish over all processed scans (SMapper::getOccupancyGrid, src/slam_mapper.cpp:63-69):
// use_gpu = 0 the reference's OccupancyGrid::CreateFromScans, 1 the b200og binding.  info = {width, height,
// width step}; cells (if not NULL, cap bytes) receives the grid bytes.  Returns wall seconds, < 0 on failure.
double krep_occupancy(void * rp, double resolution, int use_gpu, int info[3], double offset[2], unsigned char * cells, long cap)
{
  Replay * r = static_cast<Replay *>(rp);
  const LocalizedRangeScanVector v = processed_scans(r);
  auto t0 = std::chrono::steady_clock::now();
  OccupancyGrid * g = use_gpu ? karto::b200::CreateOccupancyGridFromScans(v, resolution) : OccupancyGrid::CreateFromScans(v, resolution);
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (!g) return -1.0;
  info[0] = g->GetWidth(); info[1] = g->GetHeight(); info[2] = g->GetWidthStep();
  offset[0] = g->GetCoordinateConverter()->GetOffset().GetX();
  offset[1] = g->GetCoordinateConverter()->GetOffset().GetY();
  if (cells && cap >= static_cast<long>(g->GetDataSize())) std::memcpy(cells, g->GetDataPointer(), g->GetDataSize());
  delete g;
  return sec;
}

}  // extern "C"
