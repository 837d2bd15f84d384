// ORACLE / TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// slam_toolbox's MergeMapsKinematic::transformScan (src/merge_maps_kinematic.cpp:195-248) restated with the UNMODIFIED
// reference karto_sdk's own setters, for the parts the occupancy grid reads: the unfiltered points, the stored bounding
// box (its four corners, each corrected, added in the tool's order), the corrected pose and IsDirty cleared, so that
// ComputeDimensions reads the stored box and AddScan the stored points.  The correction is tf2's basis (row-major 3x3)
// and origin; tf2::Transform applied to (x, y, 0) is the row dot product then + origin, evaluated here in that order
// (-ffp-contract=off).  The corrected heading (tf2::getYaw of a quaternion product in the tool) is not read by the grid;
// it is set to heading + atan2(b10, b00).
//
// oracle/merge.mk links this file with oracle/ref_driver.cpp, the reference's Karto / Mapper objects and
// integration/merge_maps_driver.cpp into oracle/_ref/libmerge_b200.so.  No reference source is copied here.
#include <cmath>

#include "karto_sdk/Mapper.h"

using namespace karto;

static Vector2<kt_double> kref_apply(const double b[9], const double o[3], const Vector2<kt_double> & p)
{
  const double x = p.GetX(), y = p.GetY();
  return Vector2<kt_double>(((b[0] * x + b[1] * y) + b[2] * 0.0) + o[0], ((b[3] * x + b[4] * y) + b[5] * 0.0) + o[1]);
}

extern "C" {

void kref_transform_scan(void * sp, const double basis[9], const double origin[3])
{
  LocalizedRangeScan * s = static_cast<LocalizedRangeScan *>(sp);
  BoundingBox2 bbox = s->GetBoundingBox();   // Update() first if the scan is dirty, as GetBarycenterPose does in the tool
  const Vector2<kt_double> mn = bbox.GetMinimum(), mx = bbox.GetMaximum();
  BoundingBox2 transformed;
  transformed.Add(kref_apply(basis, origin, mn));
  transformed.Add(kref_apply(basis, origin, mx));
  transformed.Add(kref_apply(basis, origin, Vector2<kt_double>(mx.GetX(), mn.GetY())));
  transformed.Add(kref_apply(basis, origin, Vector2<kt_double>(mn.GetX(), mx.GetY())));
  s->SetBoundingBox(transformed);
  PointVectorDouble pts = s->GetPointReadings();
  for (auto & p : pts) {
    const Vector2<kt_double> c = kref_apply(basis, origin, p);
    p.SetX(c.GetX());
    p.SetY(c.GetY());
  }
  s->SetPointReadings(pts);
  const Pose2 cp = s->GetCorrectedPose();
  const Vector2<kt_double> pos = kref_apply(basis, origin, cp.GetPosition());
  s->SetCorrectedPose(Pose2(pos.GetX(), pos.GetY(), math::NormalizeAngle(cp.GetHeading() + std::atan2(basis[3], basis[0]))));
  kt_bool dirty = false;
  s->SetIsDirty(dirty);
}

// the stored bounding box of a scan: {min x, min y, max x, max y}
void kref_scan_box(void * sp, double box[4])
{
  const BoundingBox2 & b = static_cast<LocalizedRangeScan *>(sp)->GetBoundingBox();
  box[0] = b.GetMinimum().GetX(); box[1] = b.GetMinimum().GetY();
  box[2] = b.GetMaximum().GetX(); box[3] = b.GetMaximum().GetY();
}

}  // extern "C"
