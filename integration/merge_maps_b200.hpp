// Reference-side binding #4 (INTEGRATION.md section 3): slam_toolbox's map-merge tool (MergeMapsKinematic,
// src/merge_maps_kinematic.cpp) on the b200slam occupancy store.
//
// The tool keeps every loaded submap's scans (scans_vec_) and, on each merge, corrects all of them in place with
// transformScan (:195-248) and builds one grid with OccupancyGrid::CreateFromScans (:294-310).  A SubmapStore holds the
// same scans on the device instead: the tool calls
//
//     karto::b200::SubmapStore store(resolution_);                             // a member of the tool
//     id = store.AddSubmap(mapper->GetAllProcessedScans(), &grid);            // addSubmapCallback, :94-113
//     store.ApplyCorrection(id, submap_correction.getBasis(), submap_correction.getOrigin());   // per submap, :262-273
//     karto::OccupancyGrid * g = store.Merge(resolution_);                    // :275-278
//
// where ApplyCorrection takes the correction as tf2 holds it (any type with operator[](r)[c] / operator[](r) of doubles,
// so no tf2 type appears here).  The grids equal the reference's bit for bit: width, height, offset, cell bytes.  The
// corrected scans stay on the device, so the karto scans the tool keeps are not corrected by this path; the sensor
// position takes the points' formula, which is exact for a laser at the robot origin (GetSensorPose adds a zero offset).
// Every scan is stored with its own laser's limits (each pose-graph file the tool loads brings its own laser), as the
// reference's CreateFromScans reads them per scan.
#pragma once
#include <cstdio>
#include <vector>

#include "karto_sdk/Karto.h"
#include "b200slam.h"
#include "occupancy_b200.hpp"

namespace karto {
namespace b200 {

class SubmapStore {
public:
  // resolution = the tool's resolution_ parameter: every grid of this store is built at it
  explicit SubmapStore(kt_double resolution) : resolution_(resolution) {}
  SubmapStore(const SubmapStore &) = delete;
  SubmapStore & operator=(const SubmapStore &) = delete;
  ~SubmapStore() { if (h_) b200og_destroy(h_); }

  // addSubmapCallback: stores the submap's scans and returns its id (0, 1, ...), -1 on failure.  *grid (if not NULL)
  // receives the submap's own grid (caller deletes; NULL for a submap without scans).
  int AddSubmap(const LocalizedRangeScanVector & rScans, OccupancyGrid ** grid = nullptr)
  {
    if (grid) *grid = NULL;
    std::vector<b200og_laser> lasers;
    const std::vector<b200_scan> scans = detail::CollectScans(rScans, &lasers, &laser_);
    if (!h_) {
      const b200og_params p = detail::GridParams(resolution_, laser_);
      if (b200og_create(&p, &h_) != B200_OK) return Fail();
    }
    const int32_t first = b200og_num_scans(h_);
    if (b200og_add_scans_lasers(h_, scans.data(), static_cast<int32_t>(scans.size()), lasers.data()) != B200_OK) return Fail();
    submaps_.push_back({first, static_cast<int32_t>(scans.size())});
    if (grid && !scans.empty()) *grid = Build(first, static_cast<int32_t>(scans.size()));
    return static_cast<int>(submaps_.size()) - 1;
  }

  // transformScan on every scan of submap `id`, with the values of submap_correction.getBasis() (indexable [r][c]) and
  // getOrigin() (indexable [r]); false on a bad id or a non-finite correction
  template <class Basis, class Origin>
  bool ApplyCorrection(int id, const Basis & basis, const Origin & origin)
  {
    if (id < 0 || id >= static_cast<int>(submaps_.size())) return false;
    double b[9], o[3];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) b[3 * r + c] = basis[r][c];
      o[r] = origin[r];
    }
    if (b200og_transform_scans(h_, submaps_[id].first, submaps_[id].count, b, o, nullptr) != B200_OK) {
      Fail();
      return false;
    }
    return true;
  }

  // kartoToROSOccupancyGrid's CreateFromScans over every submap's scans as they stand (caller deletes); NULL without
  // scans or when `resolution` is not the store's
  OccupancyGrid * Merge(kt_double resolution)
  {
    if (!h_ || b200og_num_scans(h_) == 0) return NULL;
    if (resolution != resolution_) {
      std::fprintf(stderr, "SubmapStore: resolution %g is not the store's %g\n", resolution, resolution_);
      return NULL;
    }
    return Build(0, b200og_num_scans(h_));
  }

  b200og * handle() const { return h_; }

private:
  struct Range { int32_t first, count; };

  // the grid of scans [first, first + count)
  OccupancyGrid * Build(int32_t first, int32_t count)
  {
    b200og_info info;
    if (b200og_build_range(h_, first, count, &info) != B200_OK) { Fail(); return NULL; }
    return detail::FetchGrid(h_, info, resolution_, "SubmapStore");
  }

  int Fail() const
  {
    std::fprintf(stderr, "SubmapStore (b200): %s\n", b200_last_error());
    return -1;
  }

  kt_double resolution_;
  b200og * h_ = nullptr;
  LaserRangeFinder * laser_ = nullptr;   // the first scan's: the handle's default limits only
  std::vector<Range> submaps_;
};

}  // namespace b200
}  // namespace karto
