// ORACLE / TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// Scans of several lasers for the UNMODIFIED reference karto_sdk.  The reference looks a scan's laser up by its sensor
// name on every call (LocalizedRangeScan::GetLaserRangeFinder, Karto.h:5304-5306), and OccupancyGrid::AddScan /
// LocalizedRangeScan::Update take the range threshold, minimum and maximum range from that laser (Karto.h:6146-6151,
// :5646-5698).  These entry points register named lasers with the reference's SensorManager and create scans on a chosen
// one; oracle/ref_driver.cpp's kref_occupancy_* then run the unmodified OccupancyGrid::CreateFromScans over them.
//
// oracle/multilaser.mk links this file with oracle/ref_driver.cpp, oracle/merge_ref_driver.cpp and the reference's Karto /
// Mapper objects into oracle/_ref/libmultilaser_ref.so.  No reference source is copied here.
#include <map>
#include <string>

#include "karto_sdk/Mapper.h"

using namespace karto;

namespace {
std::map<std::string, LaserRangeFinder *> g_lasers;
}

extern "C" {

// Registers laser `name`, or sets the limits of the one already registered under it (the reference re-reads them on every
// AddScan; a scan's stored box keeps the limits of its last Update).  Returns the laser's number of range readings.
int kml_laser(const char * name, double min_angle, double max_angle, double ang_res, double min_range, double max_range,
              double range_threshold)
{
  auto it = g_lasers.find(name);
  LaserRangeFinder * l = nullptr;
  if (it == g_lasers.end()) {
    l = LaserRangeFinder::CreateLaserRangeFinder(LaserRangeFinder_Custom, Name(name));
    l->SetMinimumAngle(min_angle);
    l->SetMaximumAngle(max_angle);
    l->SetAngularResolution(ang_res);
    l->SetOffsetPose(Pose2(0.0, 0.0, 0.0));
  } else {
    l = it->second;
  }
  l->SetMinimumRange(min_range);
  l->SetMaximumRange(max_range);
  l->SetRangeThreshold(range_threshold);
  if (it == g_lasers.end()) {
    SensorManager::GetInstance()->RegisterSensor(l);
    g_lasers[name] = l;
  }
  return static_cast<int>(l->GetNumberOfRangeReadings());
}

// the limits laser `name` holds now: {range threshold, minimum range, maximum range} (SetRangeThreshold clips the threshold
// into [minimum, maximum]); zeros for an unknown name
void kml_laser_limits(const char * name, double out[3])
{
  auto it = g_lasers.find(name);
  out[0] = out[1] = out[2] = 0.0;
  if (it == g_lasers.end()) return;
  out[0] = it->second->GetRangeThreshold();
  out[1] = it->second->GetMinimumRange();
  out[2] = it->second->GetMaximumRange();
}

// A scan of laser `name` at pose (x, y, heading); Update() runs now, with that laser's current limits.
void * kml_scan_create(const char * name, const double * ranges, int n, const double pose[3], int unique_id)
{
  RangeReadingsVector r(ranges, ranges + n);
  LocalizedRangeScan * s = new LocalizedRangeScan(Name(name), r);
  Pose2 p(pose[0], pose[1], pose[2]);
  s->SetOdometricPose(p);
  s->SetCorrectedPose(p);
  s->SetUniqueId(unique_id);
  s->SetStateId(unique_id);
  s->SetTime(static_cast<double>(unique_id));
  (void)s->GetPointReadings();
  return s;
}

}  // extern "C"
