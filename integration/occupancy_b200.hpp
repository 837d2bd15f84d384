// Reference-side binding #3 (INTEGRATION.md section 3): karto::OccupancyGrid::CreateFromScans
// (Karto.h:5946-5961) through the b200slam C ABI.
//
// CreateFromScans is a static INLINE member of a header class, so there is no symbol to interpose: the
// binding is a drop-in function with the same signature and result type that a maintainer calls from the
// one place slam_toolbox builds its map, SMapper::getOccupancyGrid (src/slam_mapper.cpp:63-69):
//
//     return karto::b200::CreateOccupancyGridFromScans(mapper_->GetAllProcessedScans(), resolution);
//
// The returned karto::OccupancyGrid has the reference's width / height / offset / resolution and cell
// bytes, which is everything its consumers read (vis_utils::toNavMap, include/slam_toolbox/
// visualization_utils.hpp:108-146; map_saver; RayCast / IsFree).  The hit / pass counter grids inside it
// stay empty: they are scratch of the CPU build (fetch them with b200og_fetch when wanted).
//
// Every scan is stored with its own laser's limits (scan->GetLaserRangeFinder(): range threshold, minimum and maximum
// range), as the reference's AddScan and LocalizedRangeScan::Update read them (Karto.h:6146-6151, :5646-5698), so a map of
// several lasers equals the reference's.
//
// ResidentOccupancyMap is the same publish with the scans kept on the device between calls (section 3a).
#pragma once
#include <cstdio>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "karto_sdk/Karto.h"
#include "b200slam.h"

namespace karto {
namespace b200 {

namespace detail {

// a laser's limits as the store keeps them
inline b200og_laser Limits(const LaserRangeFinder * l)
{
  return b200og_laser{l->GetRangeThreshold(), l->GetMinimumRange(), l->GetMaximumRange()};
}

inline bool SameLimits(const b200og_laser & a, const b200og_laser & b)
{
  return a.range_threshold == b.range_threshold && a.minimum_range == b.minimum_range && a.maximum_range == b.maximum_range;
}

// the non-NULL scans of rScans as the C ABI takes them (pointers into the scans), each scan's own laser limits
// (GetLaserRangeFinder looks the laser up by the scan's sensor name, Karto.h:5304-5306), and the laser of the first one
inline std::vector<b200_scan> CollectScans(const LocalizedRangeScanVector & rScans, std::vector<b200og_laser> * lasers,
                                           LaserRangeFinder ** laser)
{
  std::vector<b200_scan> scans;
  static_assert(sizeof(Vector2<kt_double>) == 2 * sizeof(double), "Vector2<double> must be {x, y}");
  for (LocalizedRangeScan * s : rScans) {
    if (s == nullptr) continue;                                   // Karto.h:6094, :6123
    LaserRangeFinder * l = s->GetLaserRangeFinder();
    if (laser && !*laser) *laser = l;
    if (lasers) lasers->push_back(Limits(l));
    b200_scan o;
    const PointVectorDouble & pts = s->GetPointReadings(false);  // Karto.h:6149
    o.n = static_cast<int32_t>(pts.size());
    o.ranges = s->GetRangeReadings();
    o.points_xy = reinterpret_cast<const double *>(pts.data());
    const Pose2 p = s->GetSensorPose();
    o.sensor_pose[0] = p.GetX(); o.sensor_pose[1] = p.GetY(); o.sensor_pose[2] = p.GetHeading();
    scans.push_back(o);
  }
  return scans;
}

inline b200og_params GridParams(kt_double resolution, LaserRangeFinder * laser)
{
  b200og_params p;
  b200og_default_params(&p);                                      // MinPassThrough 2, OccupancyThreshold 0.1
  p.resolution = resolution;
  if (laser) {
    p.range_threshold = laser->GetRangeThreshold();
    p.minimum_range = laser->GetMinimumRange();
    p.maximum_range = laser->GetMaximumRange();
  }
  return p;
}

// the karto grid of a successful build of h; NULL, with the error printed under `who`, when it cannot be fetched
inline OccupancyGrid * FetchGrid(b200og * h, const b200og_info & info, kt_double resolution,
                                 const char * who = "OccupancyGrid::CreateFromScans")
{
  OccupancyGrid * g = new OccupancyGrid(info.width, info.height, Vector2<kt_double>(info.offset[0], info.offset[1]), resolution);
  if (g->GetWidthStep() != info.stride || b200og_fetch(h, g->GetDataPointer(), nullptr, nullptr) != B200_OK) {
    std::fprintf(stderr, "%s (b200): %s\n", who, b200_last_error());
    delete g;
    g = NULL;
  }
  return g;
}

}  // namespace detail

inline OccupancyGrid * CreateOccupancyGridFromScans(const LocalizedRangeScanVector & rScans, kt_double resolution,
                                                     float * device_ms = nullptr)
{
  LaserRangeFinder * laser = nullptr;
  std::vector<b200og_laser> lasers;
  const std::vector<b200_scan> scans = detail::CollectScans(rScans, &lasers, &laser);
  if (rScans.empty()) return NULL;                                // Karto.h:5950-5952
  const b200og_params p = detail::GridParams(resolution, laser);
  b200og * h = nullptr;
  b200og_info info;
  if (b200og_create(&p, &h) != B200_OK ||
      b200og_add_scans_lasers(h, scans.data(), static_cast<int32_t>(scans.size()), lasers.data()) != B200_OK ||
      b200og_build(h, &info) != B200_OK) {
    std::fprintf(stderr, "OccupancyGrid::CreateFromScans (b200): %s\n", b200_last_error());
    b200og_destroy(h);
    return NULL;
  }
  OccupancyGrid * g = detail::FetchGrid(h, info, resolution);
  if (device_ms) b200og_kernel_ms(h, device_ms);
  b200og_destroy(h);
  return g;
}

// The map publish with the scans resident on the device between publishes.  The store holds the scans of the last publish,
// matched to the mapper's by unique id, in the order they were uploaded.  That need not be rScans' order (with several lasers
// GetAllProcessedScans returns them sensor by sensor), and need not be: the grid does not depend on the scans' order (the
// counters are integer sums, the box a min / max).  A publish
//   - removes, in place (b200og_remove_scans), the stored scans the mapper no longer holds, such as the localization rolling
//     buffer's oldest scans;
//   - appends the scans whose unique ids are not stored;
//   - reloads every scan when poses_corrected is set, i.e. when MapperGraph::CorrectPoses has run since the last publish
//     (b200_shim_correct_poses_calls() of integration/scan_matcher_b200.cpp counts its calls), since that moves stored scans'
//     points;
//   - reloads every scan when the limits of a laser with stored scans changed since they were uploaded: the reference reads
//     the laser's limits on every CreateFromScans, and every stored scan holds the limits of its upload.
// The store is keyed on the resolution only: scans of any number of lasers share it, each with its own laser's limits.
// The grid equals CreateOccupancyGridFromScans over the same scans.  One instance per map; not thread-safe.
class ResidentOccupancyMap {
 public:
  struct Stats { int32_t removed = 0, appended = 0, reloaded = 0; };

  ResidentOccupancyMap() = default;
  ResidentOccupancyMap(const ResidentOccupancyMap &) = delete;
  ResidentOccupancyMap & operator=(const ResidentOccupancyMap &) = delete;
  ~ResidentOccupancyMap() { if (h_) b200og_destroy(h_); }

  OccupancyGrid * Publish(const LocalizedRangeScanVector & rScans, kt_double resolution, bool poses_corrected, Stats * stats = nullptr,
                          float * device_ms = nullptr)
  {
    Stats st;
    std::vector<LocalizedRangeScan *> live;
    for (LocalizedRangeScan * s : rScans)
      if (s) live.push_back(s);
    if (rScans.empty()) { if (stats) *stats = st; return NULL; }  // Karto.h:5950-5952
    // the store is built for one resolution; another one starts a fresh store.  The handle's own limits are never used: every
    // scan is added with its laser's limits.
    if (!h_ || resolution != resolution_) {
      if (h_) b200og_destroy(h_);
      h_ = nullptr;
      ids_.clear();
      uploaded_.clear();
      const b200og_params p = detail::GridParams(resolution, nullptr);
      if (b200og_create(&p, &h_) != B200_OK) return Fail();
      resolution_ = resolution;
      poses_corrected = true;
    }
    // the limits every laser of the live scans has now; a stored sensor whose limits changed since its upload reloads the store
    std::map<std::string, b200og_laser> now;
    for (LocalizedRangeScan * s : live) {
      const std::string name = s->GetSensorName().ToString();
      if (now.count(name)) continue;
      now[name] = detail::Limits(s->GetLaserRangeFinder());
    }
    bool limits_changed = false;
    for (const auto & kv : uploaded_) {
      auto it = now.find(kv.first);
      if (it != now.end() && !detail::SameLimits(it->second, kv.second)) limits_changed = true;
    }
    // stored scans that are gone, and the ones that stay
    std::set<kt_int32s> live_ids, kept_ids;
    for (LocalizedRangeScan * s : live) live_ids.insert(s->GetUniqueId());
    std::vector<int32_t> gone;
    const bool reload = poses_corrected || limits_changed;
    for (size_t k = 0; k < ids_.size() && !reload; ++k) {
      if (live_ids.count(ids_[k])) kept_ids.insert(ids_[k]);
      else gone.push_back(static_cast<int32_t>(k));
    }
    if (reload) {
      if (b200og_clear_scans(h_) != B200_OK) return Fail();
      ids_.clear();
      uploaded_.clear();
      st.reloaded = 1;
    } else if (!gone.empty()) {
      if (b200og_remove_scans(h_, gone.data(), static_cast<int32_t>(gone.size())) != B200_OK) return Fail();
      std::vector<kt_int32s> kept;
      kept.reserve(ids_.size() - gone.size());
      for (size_t k = 0, r = 0; k < ids_.size(); ++k) {
        if (r < gone.size() && gone[r] == static_cast<int32_t>(k)) { ++r; continue; }
        kept.push_back(ids_[k]);
      }
      ids_.swap(kept);
      st.removed = static_cast<int32_t>(gone.size());
    }
    LocalizedRangeScanVector added;
    for (LocalizedRangeScan * s : live)
      if (!kept_ids.count(s->GetUniqueId())) added.push_back(s);
    std::vector<b200og_laser> lasers;
    const std::vector<b200_scan> scans = detail::CollectScans(added, &lasers, nullptr);
    if (!scans.empty() && b200og_add_scans_lasers(h_, scans.data(), static_cast<int32_t>(scans.size()), lasers.data()) != B200_OK)
      return Fail();
    for (LocalizedRangeScan * s : added) {
      ids_.push_back(s->GetUniqueId());
      const std::string name = s->GetSensorName().ToString();
      uploaded_[name] = now[name];
    }
    st.appended = static_cast<int32_t>(scans.size());
    if (stats) *stats = st;
    b200og_info info;
    if (b200og_build(h_, &info) != B200_OK) return Fail();
    if (device_ms) b200og_kernel_ms(h_, device_ms);
    return detail::FetchGrid(h_, info, resolution);
  }

 private:
  // after a failed call the store's contents are unknown: the next publish starts from a fresh handle
  OccupancyGrid * Fail()
  {
    std::fprintf(stderr, "ResidentOccupancyMap (b200): %s\n", b200_last_error());
    if (h_) b200og_destroy(h_);
    h_ = nullptr;
    ids_.clear();
    uploaded_.clear();
    return NULL;
  }

  b200og * h_ = nullptr;
  kt_double resolution_ = 0.0;                   // what h_ was created with
  std::vector<kt_int32s> ids_;                   // unique ids of the stored scans, in store order
  std::map<std::string, b200og_laser> uploaded_;   // sensor name -> the limits its stored scans were uploaded with
};

}  // namespace b200
}  // namespace karto
