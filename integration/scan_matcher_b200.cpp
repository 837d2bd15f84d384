// Reference-side binding #2 (INTEGRATION.md section 2): link-time replacement of
// karto::ScanMatcher::Create and karto::ScanMatcher::MatchScan<T> by the b200slam C ABI.
//
// Mapper.o reaches both through PLT relocations by symbol name (objdump -dr: 3 x Create, 8 x MatchScan),
// so linking THIS object ahead of the unmodified Mapper.o (with -Wl,--allow-multiple-definition for the
// strong Create; the MatchScan instantiations in Mapper.o are weak) redirects every match the
// reference's Mapper / MapperGraph performs -- sequential match, near-chain links, loop closure --
// to the GPU, with no change to the reference sources.
#include <cstdio>
#include <mutex>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "karto_sdk/Mapper.h"
#include "b200slam.h"

namespace karto {

namespace {
std::unordered_map<const ScanMatcher *, b200sm *> & handles()
{
  static std::unordered_map<const ScanMatcher *, b200sm *> h;
  return h;
}
std::mutex & handles_mutex()
{
  static std::mutex m;
  return m;
}
b200sm * handle_of(const ScanMatcher * m)
{
  std::lock_guard<std::mutex> lock(handles_mutex());
  return handles().at(m);
}
long g_match_calls = 0;
long g_correct_poses_calls = 0;

b200_scan to_scan(LocalizedRangeScan * s)
{
  b200_scan o;
  const PointVectorDouble & pts = s->GetPointReadings(false);   // unfiltered (Karto.h:5613-5628)
  o.n = static_cast<int32_t>(s->GetNumberOfRangeReadings());
  o.ranges = s->GetRangeReadings();
  static_assert(sizeof(Vector2<kt_double>) == 2 * sizeof(double), "Vector2<double> must be {x, y}");
  o.points_xy = reinterpret_cast<const double *>(pts.data());
  const Pose2 p = s->GetSensorPose();
  o.sensor_pose[0] = p.GetX(); o.sensor_pose[1] = p.GetY(); o.sensor_pose[2] = p.GetHeading();
  return o;
}
inline LocalizedRangeScan * deref(LocalizedRangeScanVector::const_iterator it) { return *it; }
inline LocalizedRangeScan * deref(LocalizedRangeScanMap::const_iterator it) { return it->second; }
}  // namespace

extern "C" long b200_shim_match_calls() { return g_match_calls; }
// MapperGraph::CorrectPoses calls so far: a resident map store (integration/occupancy_b200.hpp) reloads after each one
extern "C" long b200_shim_correct_poses_calls() { return g_correct_poses_calls; }
extern "C" long b200_shim_live_handles()
{
  std::lock_guard<std::mutex> lock(handles_mutex());
  return static_cast<long>(handles().size());
}

// Releases the device state of a matcher.  Called by the destructor below; also exported for hosts that tear the mapper
// down through other paths.
extern "C" void b200_shim_release(const void * matcher)
{
  b200sm * h = nullptr;
  {
    std::lock_guard<std::mutex> lock(handles_mutex());
    auto it = handles().find(static_cast<const ScanMatcher *>(matcher));
    if (it == handles().end()) return;
    h = it->second;
    handles().erase(it);
  }
  b200sm_destroy(h);
}

// ScanMatcher::~ScanMatcher (Mapper.cpp:464-475) is a strong symbol in Mapper.o; this definition is linked first (like
// Create, -Wl,--allow-multiple-definition), frees what the reference's destructor frees -- nothing is allocated on this
// path, the three members stay NULL -- and releases the b200sm handle, so Mapper::Reset / lifelong mode do not leak.
ScanMatcher::~ScanMatcher()
{
  if (m_pCorrelationGrid) delete m_pCorrelationGrid;
  if (m_pSearchSpaceProbs) delete m_pSearchSpaceProbs;
  if (m_pGridLookup) delete m_pGridLookup;
  b200_shim_release(this);
}

ScanMatcher * ScanMatcher::Create(Mapper * pMapper, kt_double searchSize, kt_double resolution,
                                  kt_double smearDeviation, kt_double rangeThreshold)
{
  b200sm_params p{searchSize, resolution, smearDeviation, rangeThreshold,
      pMapper->m_pCoarseSearchAngleOffset->GetValue(), pMapper->m_pCoarseAngleResolution->GetValue(),
      pMapper->m_pFineSearchAngleOffset->GetValue(), pMapper->m_pDistanceVariancePenalty->GetValue(),
      pMapper->m_pAngleVariancePenalty->GetValue(), pMapper->m_pMinimumDistancePenalty->GetValue(),
      pMapper->m_pMinimumAnglePenalty->GetValue(), pMapper->m_pUseResponseExpansion->GetValue() ? 1 : 0};
  b200sm * h = nullptr;
  if (b200sm_create(&p, &h) != B200_OK) {
    std::fprintf(stderr, "ScanMatcher::Create (b200): %s\n", b200_last_error());
    return NULL;   // Mapper.cpp:481-493 returns NULL on invalid parameters
  }
  ScanMatcher * m = new ScanMatcher(pMapper);
  b200sm * stale = nullptr;
  {
    std::lock_guard<std::mutex> lock(handles_mutex());
    auto it = handles().find(m);
    if (it != handles().end()) stale = it->second;   // a matcher freed without its destructor reused the address
    handles()[m] = h;
  }
  if (stale) b200sm_destroy(stale);
  return m;
}

// MapperGraph::CorrectPoses (Mapper.cpp:2012-2030), linked ahead of the reference's definition like Create: the same calls in the
// same order, except that the per-scan SetCorrectedPoseAndUpdate -- 1081 sin / cos per scan, every scan of the map after every loop
// closure, most of a long replay once matching and solving run on the GPU -- is spread over the library's host threads.  Scans are
// independent objects and the arithmetic is the reference's own inline code (same libm), so the poses and point readings are
// bit-identical.
void MapperGraph::CorrectPoses()
{
  ++g_correct_poses_calls;
  ScanSolver * pSolver = m_pMapper->m_pScanOptimizer;
  if (pSolver != NULL) {
    pSolver->Compute();
    struct Job { LocalizedRangeScan * scan; Pose2 pose; };
    std::vector<Job> jobs;
    const ScanSolver::IdPoseVector & corr = pSolver->GetCorrections();
    jobs.reserve(corr.size());
    for (ScanSolver::IdPoseVector::const_iterator it = corr.begin(); it != corr.end(); ++it) {
      LocalizedRangeScan * scan = m_pMapper->m_pMapperSensorManager->GetScan(it->first);
      if (scan == NULL) continue;
      jobs.push_back(Job{scan, it->second});
    }
    b200_parallel_for(static_cast<int32_t>(jobs.size()),
                      [](int32_t i, void * ctx) {
                        Job & j = (*static_cast<std::vector<Job> *>(ctx))[i];
                        j.scan->SetCorrectedPoseAndUpdate(j.pose);
                      },
                      &jobs);
    pSolver->Clear();
  }
}

template<class T>
kt_double ScanMatcher::MatchScan(LocalizedRangeScan * pScan, const T & rBaseScans, Pose2 & rMean,
                                 Matrix3 & rCovariance, kt_bool doPenalize, kt_bool doRefineMatch)
{
  ++g_match_calls;
  std::vector<b200_scan> base;
  for (auto it = rBaseScans.begin(); it != rBaseScans.end(); ++it) {
    LocalizedRangeScan * s = deref(it);
    if (s) base.push_back(to_scan(s));   // NULL scans are skipped (Mapper.cpp:1039); order preserved
  }
  const b200_scan q = to_scan(pScan);
  double mean[3], cov[9], resp = 0.0;
  if (b200sm_match(handle_of(this), &q, base.data(), static_cast<int32_t>(base.size()), doPenalize ? 1 : 0,
                   doRefineMatch ? 1 : 0, mean, cov, &resp) != B200_OK) {
    throw std::runtime_error(b200_last_error());   // the reference throws std::runtime_error too (Mapper.cpp:789-828)
  }
  rMean = Pose2(mean[0], mean[1], mean[2]);
  // MatchScan leaves entries it does not compute untouched; the callers pass zero / identity matrices and
  // the ABI returns the full matrix the reference would have produced from a zero-initialised one
  for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) rCovariance(r, k) = cov[3 * r + k];
  return resp;
}

template kt_double ScanMatcher::MatchScan<LocalizedRangeScanVector>(LocalizedRangeScan *, const LocalizedRangeScanVector &,
                                                                    Pose2 &, Matrix3 &, kt_bool, kt_bool);
template kt_double ScanMatcher::MatchScan<LocalizedRangeScanMap>(LocalizedRangeScan *, const LocalizedRangeScanMap &,
                                                                 Pose2 &, Matrix3 &, kt_bool, kt_bool);

}  // namespace karto
