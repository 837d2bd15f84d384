// TEST INFRASTRUCTURE: extern "C" driver of integration/merge_maps_b200.hpp (karto::b200::SubmapStore), linked by
// oracle/merge.mk with the unmodified reference karto_sdk, oracle/ref_driver.cpp and oracle/merge_ref_driver.cpp into
// oracle/_ref/libmerge_b200.so, so
// that one process holds both the reference's scans (kref_scan_create, kref_transform_scan, kref_occupancy_create) and
// the binding that builds the merged grid on the device from the same karto scans.
#include <cstring>

#include "merge_maps_b200.hpp"

using namespace karto;

extern "C" {

void * kmm_store_create(double resolution) { return new b200::SubmapStore(resolution); }
void kmm_store_destroy(void * s) { delete static_cast<b200::SubmapStore *>(s); }

// addSubmapCallback on n karto scans; info / offset / cells (cap bytes) receive the submap's own grid when not NULL
int kmm_add_submap(void * sp, void ** scans, int n, int info[3], double offset[2], unsigned char * cells, long cap)
{
  LocalizedRangeScanVector v;
  for (int i = 0; i < n; ++i) v.push_back(static_cast<LocalizedRangeScan *>(scans[i]));
  OccupancyGrid * g = nullptr;
  const int id = static_cast<b200::SubmapStore *>(sp)->AddSubmap(v, info ? &g : nullptr);
  if (g) {
    info[0] = g->GetWidth(); info[1] = g->GetHeight(); info[2] = g->GetWidthStep();
    offset[0] = g->GetCoordinateConverter()->GetOffset().GetX();
    offset[1] = g->GetCoordinateConverter()->GetOffset().GetY();
    if (cells && g->GetDataSize() <= cap) std::memcpy(cells, g->GetDataPointer(), g->GetDataSize());
    delete g;
  }
  return id;
}

// ApplyCorrection with a row-major basis and an origin, held the way tf2 indexes them
int kmm_apply(void * sp, int id, const double basis[9], const double origin[3])
{
  struct Rows { const double * b; const double * operator[](int r) const { return b + 3 * r; } } rows{basis};
  return static_cast<b200::SubmapStore *>(sp)->ApplyCorrection(id, rows, origin) ? 0 : -1;
}

// Merge: info = {width, height, width step}, cells = width step x height bytes (cap); -1 when no grid was made
int kmm_merge(void * sp, double resolution, int info[3], double offset[2], unsigned char * cells, long cap)
{
  OccupancyGrid * g = static_cast<b200::SubmapStore *>(sp)->Merge(resolution);
  if (!g) return -1;
  info[0] = g->GetWidth(); info[1] = g->GetHeight(); info[2] = g->GetWidthStep();
  offset[0] = g->GetCoordinateConverter()->GetOffset().GetX();
  offset[1] = g->GetCoordinateConverter()->GetOffset().GetY();
  if (cells && g->GetDataSize() <= cap) std::memcpy(cells, g->GetDataPointer(), g->GetDataSize());
  delete g;
  return 0;
}

}  // extern "C"
