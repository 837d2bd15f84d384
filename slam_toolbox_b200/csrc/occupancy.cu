// Occupancy grid from scans: karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961), the
// map-publish step either side of the hot path (src/slam_mapper.cpp:63-69,
// src/slam_toolbox_common.cpp:630-654).  SURVEY.md 8(f) row 4.
//
// Data in HBM (all FP64 inputs are the reference's own values, nothing is re-derived):
//   ranges [B]      raw range readings of all stored scans, scan after scan
//   points [B][2]   their unfiltered world-frame point readings (LocalizedRangeScan::GetPointReadings(false))
//   sensor [S][2]   sensor position of every scan; start [S+1] = first beam of every scan
//   laser [S][3]    {range threshold, minimum range, maximum range} of every scan's own laser: AddScan and Update read
//                   pScan->GetLaserRangeFinder() per scan (Karto.h:6146-6151, :5646-5698), so one map may mix lasers
//   pass, hits [height][stride] uint32 counters; cells [height][stride] uint8 states
//
// Kernels of one build (b200og_build):
//   k_og_bbox    min / max over the sensor positions and the in-range points   (ComputeDimensions); one warp per scan,
//                so that every beam is tested against its own scan's limits
//   k_og_trace   a warp takes 32 adjacent beams of a scan, one per lane, and runs the reference's integer
//                Bresenham loop on them in lock step; equal cell indices of neighbouring lanes are merged
//                into one RED.ADD of the run length (no return value) -- integer sums commute, so the
//                result does not depend on the order and equals the reference's sequential loop
//   k_og_update  counters -> cell state (UpdateCell Karto.h:6241-6254), FP64 ratio test as the reference
// A build over a scan range [first, first + count) (b200og_build_range) runs the same kernels through the beam prefix.
//
// Map merge (slam_toolbox's merge_maps_kinematic, src/merge_maps_kinematic.cpp:195-310), on the resident store:
//   box [S][4]   per-scan bounding box {min x, min y, max x, max y}; filled lazily (k_og_scan_box, LocalizedRangeScan::
//                Update's box) on the first transform or box read-back, so add_scans and a plain build cost what they did
//   k_og_transform  one rigid correction (tf2 basis / origin) applied in place to the points, sensor positions and boxes
//                of a scan range, as transformScan does (:195-248); corrections compound across calls like the tool's
//   k_og_box_union  once any scan was transformed the stored boxes are authoritative (the tool clears IsDirty, so
//                ComputeDimensions reads them, Karto.h:6088-6112) and a build sizes the grid from their union
// Beam groups of DIFFERENT scans are interleaved over the warps so that the cells next to one sensor
// (which every beam of that scan crosses) are not hammered by the whole grid at the same time.
//
// Compiled with -fmad=false: the clipped end point sx + ratio * dx and (w - offset) * scale must
// round like the reference's x86-64 build.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "common.cuh"
#include "sm_math.cuh"

namespace b200 {

constexpr int kOgThreads = 256;
constexpr int kOgMaxCells = 1 << 24;   // longest line a beam may draw (cells); the reference has no limit but
                                       // a 16.7 M-cell beam is a corrupt pose, reported instead of traced

struct OgDev {
  const double * ranges;
  const double * points;
  const double * sensor;
  const int32_t * start;
  const double * laser;    // [nscans][3] range threshold, minimum range, maximum range of every scan
  int32_t nscans, maxbeams;
  int64_t beam0, nbeams;   // beams [beam0, nbeams) of the built scan range (absolute store indices)
  double scale, offx, offy;
  int32_t width, height, stride;
  uint32_t * pass;
  uint32_t * hits;
  uint8_t * cells;
  int32_t * flag;          // set when a beam was refused (kOgMaxCells)
};

// BoundingBox2 (Karto.h:2845-2910), stored as {min x, min y, max x, max y}.  It starts at +-999999999999999999.99999, and
// MakeFloor / MakeCeil compare strictly: NaN never wins, and of two equal values (-0.0 and +0.0) the first one added stays.
// So every caller keeps the order of additions it has: the order decides which zero a box, and a grid offset, holds.
struct OgBox {
  static constexpr double kEmpty = 999999999999999999.99999;
  double mnx = kEmpty, mny = kEmpty, mxx = -kEmpty, mxy = -kEmpty;

  __host__ __device__ static OgBox load(const double * b) { return OgBox{b[0], b[1], b[2], b[3]}; }
  __host__ __device__ void store(double * b) const { b[0] = mnx; b[1] = mny; b[2] = mxx; b[3] = mxy; }
  __host__ __device__ void add(const OgBox & b)     // BoundingBox2::Add(BoundingBox2), Karto.h:2906-2910
  {
    if (b.mnx < mnx) mnx = b.mnx;
    if (b.mny < mny) mny = b.mny;
    if (b.mxx > mxx) mxx = b.mxx;
    if (b.mxy > mxy) mxy = b.mxy;
  }
  __host__ __device__ void add(double x, double y) { add(OgBox{x, y, x, y}); }   // BoundingBox2::Add(Vector2), :2897-2901
  // every lane of the warp ends with the union of the warp's boxes
  __device__ void add_warp()
  {
    for (int o = 16; o; o >>= 1)
      add(OgBox{__shfl_xor_sync(0xffffffffu, mnx, o), __shfl_xor_sync(0xffffffffu, mny, o), __shfl_xor_sync(0xffffffffu, mxx, o),
                __shfl_xor_sync(0xffffffffu, mxy, o)});
  }
};

// partial[block][4] = the union of every thread's box b: over each warp, then over the block's warps in order
__device__ __forceinline__ void og_block_box(OgBox b, double * partial)
{
  __shared__ double sm[kOgThreads / 32][4];
  b.add_warp();
  if ((threadIdx.x & 31) == 0) b.store(sm[threadIdx.x >> 5]);
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kOgThreads / 32; ++k) b.add(OgBox::load(sm[k]));
    b.store(partial + 4 * (size_t)blockIdx.x);
  }
}

// adds to b the points of scan s that this lane reads (beams lane, lane + 32, ...) and that are in the scan's own range
// limits: math::InRange (Math.h:123) in LocalizedRangeScan::Update, Karto.h:5662
__device__ __forceinline__ void og_add_scan_points(const OgDev & d, int64_t s, int lane, OgBox & b)
{
  const double rt = d.laser[3 * s], minr = d.laser[3 * s + 1];
  for (int64_t i = d.start[s] + lane; i < d.start[s + 1]; i += 32) {
    const double r = d.ranges[i];
    if (r >= minr && r <= rt) b.add(d.points[2 * i], d.points[2 * i + 1]);
  }
}

// partial[block][4] = the box of the block's scans.  One warp per scan (grid-stride over the scans): its lanes walk the scan's
// beams with the scan's own range limits.  The result is a min / max, so it does not depend on which warp saw which scan.
__global__ void __launch_bounds__(kOgThreads) k_og_bbox(OgDev d, double * partial)
{
  OgBox b;
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (kOgThreads / 32);
  for (int64_t s = (int64_t)blockIdx.x * (kOgThreads / 32) + (threadIdx.x >> 5); s < d.nscans; s += nwarps) {
    og_add_scan_points(d, s, lane, b);
    if (lane == 0) b.add(d.sensor[2 * s], d.sensor[2 * s + 1]);   // m_BoundingBox.Add(scanPose.GetPosition()) Karto.h:5694
  }
  og_block_box(b, partial);
}

// LocalizedRangeScan::Update's box of every scan in [first, first + count) (Karto.h:5662-5698): one warp per scan, the
// in-range points and then the sensor position.  box[s] = {min x, min y, max x, max y}
__global__ void __launch_bounds__(kOgThreads) k_og_scan_box(OgDev d, int32_t first, int32_t count, double * box)
{
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (kOgThreads / 32);
  for (int64_t k = (int64_t)blockIdx.x * (kOgThreads / 32) + (threadIdx.x >> 5); k < count; k += nwarps) {
    const int32_t s = first + (int32_t)k;
    OgBox b;
    og_add_scan_points(d, s, lane, b);
    b.add_warp();
    if (lane == 0) {
      b.add(d.sensor[2 * s], d.sensor[2 * s + 1]);
      b.store(box + 4 * (size_t)s);
    }
  }
}

// One correction as tf2 holds it: rows 0 and 1 of basis[3][3], origin x, y.
struct OgTf {
  double b[2][3];
  double o[2];
};

// tf2::Transform::operator()(Vector3(x, y, 0)): the basis row dot product, then + origin, in this order and unfused
// (the unit is compiled with -fmad=false) -- MergeMapsKinematic::applyCorrection, src/merge_maps_kinematic.cpp:180-192
__device__ __forceinline__ void og_apply(const OgTf & t, double x, double y, double & ox, double & oy)
{
  ox = ((t.b[0][0] * x + t.b[0][1] * y) + t.b[0][2] * 0.0) + t.o[0];
  oy = ((t.b[1][0] * x + t.b[1][1] * y) + t.b[1][2] * 0.0) + t.o[1];
}

// transformScan (src/merge_maps_kinematic.cpp:195-248) on scans [first, first + count): every unfiltered point, the sensor
// position (when the host did not supply it) and the stored box, replaced by the box of its four corrected corners added
// in the tool's order: min, max, (max x, min y), (min x, max y) (:206-221).  Ranges are untouched.
__global__ void __launch_bounds__(kOgThreads) k_og_transform(OgDev d, int32_t first, int32_t count, OgTf t, int32_t do_sensor,
                                                             double * points, double * sensor, double * box)
{
  const int64_t step = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = d.beam0 + t0; i < d.nbeams; i += step) {
    double x, y;
    og_apply(t, points[2 * i], points[2 * i + 1], x, y);
    points[2 * i] = x; points[2 * i + 1] = y;
  }
  for (int64_t k = t0; k < count; k += step) {
    const int64_t s = first + k;
    if (do_sensor) {
      double x, y;
      og_apply(t, sensor[2 * s], sensor[2 * s + 1], x, y);
      sensor[2 * s] = x; sensor[2 * s + 1] = y;
    }
    double * bx = box + 4 * s;
    const double cx[4] = {bx[0], bx[2], bx[2], bx[0]}, cy[4] = {bx[1], bx[3], bx[1], bx[3]};
    OgBox b;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double x, y;
      og_apply(t, cx[c], cy[c], x, y);
      b.add(x, y);
    }
    b.store(bx);
  }
}

// ComputeDimensions over stored boxes (Karto.h:6097-6104): partial[block][4] like k_og_bbox, the union of
// box[first .. first + count)
__global__ void __launch_bounds__(kOgThreads) k_og_box_union(const double * box, int32_t first, int32_t count, double * partial)
{
  OgBox b;
  const int64_t step = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t k = t0; k < count; k += step) b.add(OgBox::load(box + 4 * (first + k)));
  og_block_box(b, partial);
}

// The scan store's arrays on the device (OgStore::dev): ranges [B], points [B][2], sensor [S][2], laser [S][3], box [S][4]
// (scans [0, nboxed) only), start [S + 1]
struct OgStoreDev {
  double * ranges;
  double * points;
  double * sensor;
  double * laser;
  double * box;
  int32_t * start;
};

// Store compaction (b200og_remove_scans): scan k0 + k of the compacted store `to` is scan src[k] of `from`.  One warp per
// surviving scan copies its beams from their offsets in `from` to their offsets in `to`, its sensor position, its laser
// limits, and its box while the old scan had one.  `from` and `to` are different allocations, so no thread can overwrite a
// value another one has not read yet.
struct OgCompact {
  const int32_t * src;
  int32_t k0, count, nboxed;
  OgStoreDev from, to;
};

__global__ void __launch_bounds__(kOgThreads) k_og_compact(OgCompact c)
{
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (kOgThreads / 32);
  for (int64_t k = (int64_t)blockIdx.x * (kOgThreads / 32) + (threadIdx.x >> 5); k < c.count; k += nwarps) {
    const int32_t s = c.src[k], t = c.k0 + (int32_t)k;
    const int32_t from = c.from.start[s], to = c.to.start[t], nb = c.from.start[s + 1] - from;
    for (int32_t b = lane; b < nb; b += 32) {
      c.to.ranges[to + b] = c.from.ranges[from + b];
      reinterpret_cast<double2 *>(c.to.points)[to + b] = reinterpret_cast<const double2 *>(c.from.points)[from + b];
    }
    if (lane == 0) reinterpret_cast<double2 *>(c.to.sensor)[t] = reinterpret_cast<const double2 *>(c.from.sensor)[s];
    if (lane < 4 && s < c.nboxed) c.to.box[4 * (size_t)t + lane] = c.from.box[4 * (size_t)s + lane];
    if (lane < 3) c.to.laser[3 * (size_t)t + lane] = c.from.laser[3 * (size_t)s + lane];
  }
}

// AddScan (Karto.h:6139-6182) + RayTrace (:6193-6229) + TraceLine (:4874-4927).
// A warp takes 32 ADJACENT beams of one scan: every lane prepares its beam (the FP64 part: skip / clip rules, the
// four world->grid conversions, the steep / direction swaps) and then runs the reference's own integer loop on it,
// all lanes in lock step.  Adjacent beams of a scan cross the same cells for most of their length (all 32 within
// ~7 cells of the sensor, still ~4 per cell at 55 cells), so before touching memory the warp merges runs of equal
// cell indices: one RED.ADD of the run length per distinct cell instead of one per lane.  Counter updates are the
// kernel's bound (REDG issues at ~1.3 cycles per LANE per SM, and equal addresses serialise in L2), so this is the
// main lever; sums of integers commute, so the counters still equal the reference's.
// key = cell index (< 2^31: b200og_build refuses larger grids), -1 when this lane has nothing to add
__device__ __forceinline__ void og_merged_add(uint32_t * __restrict__ base, int32_t key, bool valid, int lane, uint32_t * __restrict__ base2)
{
  const int32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool leader = valid && (lane == 0 || key != prev);
  const uint32_t bounds = __ballot_sync(0xffffffffu, leader || !valid);
  if (leader) {
    const uint32_t above = lane == 31 ? 0u : (bounds & (0xFFFFFFFEu << lane));
    const uint32_t count = (above ? (uint32_t)__ffs(above) - 1u : 32u) - (uint32_t)lane;
    atomicAdd(base + key, count);
    if (base2) atomicAdd(base2 + key, count);
  }
}

__global__ void __launch_bounds__(kOgThreads) k_og_trace(OgDev d)
{
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (kOgThreads / 32);
  const int32_t groups_per_scan = (d.maxbeams + 31) / 32;
  const int64_t total = (int64_t)d.nscans * groups_per_scan;
  // consecutive warps take groups of DIFFERENT scans, so that the cells around one sensor are not hit by the whole grid at once
  for (int64_t g = (int64_t)blockIdx.x * (kOgThreads / 32) + (threadIdx.x >> 5); g < total; g += nwarps) {
    const int32_t scan = (int32_t)(g % d.nscans), beam = (int32_t)(g / d.nscans) * 32 + lane;
    const int32_t b0 = d.start[scan];
    const double rt = d.laser[3 * scan], minr = d.laser[3 * scan + 1], maxr = d.laser[3 * scan + 2];   // warp-uniform
    int32_t x = 0, y = 0, dX = 0, dY = 0, ystep = 1, len = 0;
    bool steep = false, end_hit = false;
    int32_t end_key = -1;
    if (beam < d.start[scan + 1] - b0) {
      const int64_t i = (int64_t)b0 + beam;
      const double r = d.ranges[i];
      if (!(r <= minr || r >= maxr || r != r)) {                        // ignored readings, Karto.h:6160
        const bool valid_end = r < (rt - kTolerance);                   // Karto.h:6158
        const double sx = d.sensor[2 * scan], sy = d.sensor[2 * scan + 1];
        double px = d.points[2 * i], py = d.points[2 * i + 1];
        if (r >= rt) {                                                  // trace up to the range threshold, Karto.h:6164-6171
          const double ratio = rt / r;
          const double dx = px - sx, dy = py - sy;
          px = sx + ratio * dx;
          py = sy + ratio * dy;
        }
        const int32_t fx = world_to_grid(sx, d.offx, d.scale), fy = world_to_grid(sy, d.offy, d.scale);
        const int32_t tx = world_to_grid(px, d.offx, d.scale), ty = world_to_grid(py, d.offy, d.scale);
        int64_t a0 = fx, c0 = fy, a1 = tx, c1 = ty;
        steep = llabs(c1 - c0) > llabs(a1 - a0);                        // Karto.h:4876-4884
        if (steep) { int64_t t = a0; a0 = c0; c0 = t; t = a1; a1 = c1; c1 = t; }
        if (a0 > a1) { int64_t t = a0; a0 = a1; a1 = t; t = c0; c0 = c1; c1 = t; }
        if (a1 - a0 >= kOgMaxCells) {
          atomicExch(d.flag, 1);
        } else {
          x = (int32_t)a0; y = (int32_t)c0;
          dX = (int32_t)(a1 - a0); dY = (int32_t)llabs(c1 - c0);
          ystep = c0 < c1 ? 1 : -1;
          len = dX + 1;
          if (valid_end && is_up_to(tx, d.width) && is_up_to(ty, d.height)) {   // the end point, Karto.h:6212-6226
            end_hit = true;
            end_key = ty * d.stride + tx;
          }
        }
      }
    }
    int32_t maxlen = len;
    for (int o = 16; o; o >>= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, o));
    int32_t error = 0;
    for (int32_t step = 0; step < maxlen; ++step) {                     // TraceLine's loop, Karto.h:4900-4926
      const bool active = step < len;
      const int32_t cx = steep ? y : x, cy = steep ? x : y;
      const bool valid = active && is_up_to(cx, d.width) && is_up_to(cy, d.height);
      if (active) {
        error += dY;
        if (2 * error >= dX) { y += ystep; error -= dX; }
        ++x;
      }
      og_merged_add(d.pass, valid ? cy * d.stride + cx : -1, valid, lane, nullptr);
    }
    if (__any_sync(0xffffffffu, end_hit)) og_merged_add(d.pass, end_key, end_hit, lane, d.hits);
  }
}

// Update / UpdateCell (Karto.h:6241-6274): 4 cells per thread
__global__ void __launch_bounds__(kOgThreads) k_og_update(OgDev d, uint32_t min_pass, double threshold, size_t quads)
{
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (size_t)gridDim.x * blockDim.x) {
    const uint4 p = reinterpret_cast<const uint4 *>(d.pass)[q], h = reinterpret_cast<const uint4 *>(d.hits)[q];
    const uint32_t pp[4] = {p.x, p.y, p.z, p.w}, hh[4] = {h.x, h.y, h.z, h.w};
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t v = B200_CELL_UNKNOWN;
      if (pp[k] > min_pass) {
        const double ratio = static_cast<double>(hh[k]) / static_cast<double>(pp[k]);
        v = ratio > threshold ? B200_CELL_OCCUPIED : B200_CELL_FREE;
      }
      out |= v << (8 * k);
    }
    reinterpret_cast<uint32_t *>(d.cells)[q] = out;
  }
}

// vis_utils::toNavMap (include/slam_toolbox/visualization_utils.hpp:108-146): width x height, no padding
__global__ void __launch_bounds__(kOgThreads) k_og_nav(const uint8_t * cells, int32_t width, int32_t height, int32_t stride, int8_t * out)
{
  const size_t n = (size_t)width * height;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int32_t y = (int32_t)(i / width), x = (int32_t)(i - (size_t)y * width);
    const uint8_t v = cells[(size_t)y * stride + x];
    out[i] = v == B200_CELL_OCCUPIED ? 100 : (v == B200_CELL_FREE ? 0 : -1);
  }
}

// device buffer that keeps its contents when it grows (the scan store is appended to)
template <class T>
struct GrowBuf {
  T * p = nullptr;
  size_t cap = 0;
  ~GrowBuf() { if (p) cudaFree(p); }
  void ensure(size_t n, size_t keep, cudaStream_t st)
  {
    if (n <= cap) return;
    size_t want = std::max(n, cap + cap / 2) + 16;
    T * q = nullptr;
    B200_CUDA(cudaMalloc(reinterpret_cast<void **>(&q), want * sizeof(T)));
    if (keep && p) B200_CUDA(cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st));
    if (p) { B200_CUDA(cudaStreamSynchronize(st)); cudaFree(p); }
    p = q;
    cap = want;
  }
  void copy_from(const GrowBuf & o, size_t n, cudaStream_t st)   // the first n values of o
  {
    if (n) B200_CUDA(cudaMemcpyAsync(p, o.p, n * sizeof(T), cudaMemcpyDeviceToDevice, st));
  }
  void swap(GrowBuf & o) { std::swap(p, o.p); std::swap(cap, o.cap); }
};

// The scan store's device arrays (layout at OgStoreDev).  The box array is sized apart from the others: boxes are made
// lazily (ensure_boxes), and only scans [0, nboxed) have one.
struct OgStore {
  GrowBuf<double> ranges, points, sensor;
  GrowBuf<double> laser;   // every scan's own limits (the handle's params for scans added without a laser)
  GrowBuf<double> box;
  GrowBuf<int32_t> start;

  // room for `beams` beams and `scans` scans, keeping the first keep_beams beams and keep_scans scans (start: entries)
  void ensure(size_t beams, size_t scans, size_t keep_beams, size_t keep_scans, cudaStream_t st)
  {
    ranges.ensure(beams, keep_beams, st);
    points.ensure(2 * beams, 2 * keep_beams, st);
    sensor.ensure(2 * scans, 2 * keep_scans, st);
    laser.ensure(3 * scans, 3 * keep_scans, st);
    start.ensure(scans + 1, keep_scans, st);
  }
  // the first `beams` beams, `scans` scans and `boxes` boxes of o; start is not copied
  void copy_from(const OgStore & o, size_t beams, size_t scans, size_t boxes, cudaStream_t st)
  {
    ranges.copy_from(o.ranges, beams, st);
    points.copy_from(o.points, 2 * beams, st);
    sensor.copy_from(o.sensor, 2 * scans, st);
    laser.copy_from(o.laser, 3 * scans, st);
    box.copy_from(o.box, 4 * boxes, st);
  }
  void swap(OgStore & o, bool with_box)
  {
    ranges.swap(o.ranges); points.swap(o.points); sensor.swap(o.sensor); laser.swap(o.laser); start.swap(o.start);
    if (with_box) box.swap(o.box);
  }
  OgStoreDev dev() const { return OgStoreDev{ranges.p, points.p, sensor.p, laser.p, box.p, start.p}; }
};

}  // namespace b200

using namespace b200;

struct b200og {
  b200og_params p{};
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // scan store, and the compaction target (b200og_remove_scans) it is swapped with after each compaction
  OgStore store, spare;
  GrowBuf<int32_t> d_src;
  std::vector<int32_t> start{0};
  int32_t maxbeams = 0;
  // merge state: per-scan boxes of scans [0, nboxed), authoritative once a transform ran (boxes_auth)
  int32_t nboxed = 0;
  bool boxes_auth = false;
  // staging (two pinned halves, filled while the other one is in flight)
  double * stage[2] = {nullptr, nullptr};
  cudaEvent_t stage_done[2] = {nullptr, nullptr};
  // build state
  DevBuf<uint32_t> d_pass, d_hits;
  DevBuf<uint8_t> d_cells;
  DevBuf<int8_t> d_nav;
  DevBuf<double> d_partial;
  DevBuf<int32_t> d_flag;
  PinBuf<double> h_partial;
  PinBuf<int32_t> h_flag;
  b200og_info info{};
  bool built = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms = 0.f;
  int64_t launches = 0;
  int sms = 132;

  void ensure_stream()
  {
    if (!stream) { B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); own_stream = true; }
    if (!ev0) {
      B200_CUDA(cudaEventCreate(&ev0)); B200_CUDA(cudaEventCreate(&ev1));
      for (auto & e : stage_done) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      int dev = 0;
      B200_CUDA(cudaGetDevice(&dev));
      B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    }
  }
  int32_t nscans() const { return (int32_t)start.size() - 1; }
  // blocks of a one-warp-per-scan kernel over `count` scans: at most 8 per SM, grid-stride beyond that
  int scan_blocks(int64_t count) const
  {
    return (int)std::max<int64_t>(std::min<int64_t>((count + kOgThreads / 32 - 1) / (kOgThreads / 32), (int64_t)sms * 8), 1);
  }
  // after each launch: its error, and b200og_launch_count
  void launched()
  {
    B200_CUDA(cudaGetLastError());
    ++launches;
  }
  // b200og_kernel_ms = the device time between timer_start and timer_stop; timer_stop waits for the stream
  void timer_start() { B200_CUDA(cudaEventRecord(ev0, stream)); }
  void timer_stop()
  {
    B200_CUDA(cudaEventRecord(ev1, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaEventElapsedTime(&last_ms, ev0, ev1));
  }
};

namespace {

constexpr size_t kStageDoubles = (size_t)1 << 20;   // 8 MB per pinned half

// Pinned staging halves are kept for the life of the process (cudaMallocHost of 16 MB costs milliseconds, which the
// one-shot b200og_create_from_scans would pay on every map update). A handle borrows a pair and returns it.
struct StagePool {
  std::mutex m;
  std::vector<double *> free_list;
  double * take()
  {
    {
      std::lock_guard<std::mutex> g(m);
      if (!free_list.empty()) { double * p = free_list.back(); free_list.pop_back(); return p; }
    }
    double * p = nullptr;
    B200_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p), kStageDoubles * sizeof(double)));
    return p;
  }
  void give(double * p)
  {
    if (!p) return;
    std::lock_guard<std::mutex> g(m);
    if (free_list.size() < 4) { free_list.push_back(p); return; }
    cudaFreeHost(p);
  }
};
StagePool & stage_pool()
{
  static StagePool * pool = new StagePool();   // never destroyed: no cudaFreeHost after the runtime is gone
  return *pool;
}

bool params_ok(const b200og_params & p)
{
  if (!(p.resolution == p.resolution) || double_equal(p.resolution, 0.0)) {   // Karto.h:5916-5918 throws
    set_last_error("OccupancyGrid: resolution cannot be 0 (Karto.h:5916-5918)");
    return false;
  }
  if (!(p.range_threshold == p.range_threshold) || !(p.minimum_range == p.minimum_range) || !(p.maximum_range == p.maximum_range) ||
      !(p.occupancy_threshold == p.occupancy_threshold)) {
    set_last_error("b200og_params: NaN parameter");
    return false;
  }
  return true;
}

// Copies [src, src + n) doubles of every scan (selected by `pick`) to dst on the device through the pinned halves.
template <class Pick>
void upload_rows(b200og * h, const b200_scan * scans, int32_t n, double * dst, int per_beam, Pick pick)
{
  int half = 0;
  size_t fill = 0, sent = 0;
  bool pending[2] = {false, false};
  auto flush = [&]() {
    if (!fill) return;
    B200_CUDA(cudaMemcpyAsync(dst + sent, h->stage[half], fill * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    B200_CUDA(cudaEventRecord(h->stage_done[half], h->stream));
    pending[half] = true;
    sent += fill;
    fill = 0;
    half ^= 1;
    if (pending[half]) { B200_CUDA(cudaEventSynchronize(h->stage_done[half])); pending[half] = false; }
  };
  for (int32_t s = 0; s < n; ++s) {
    const double * src = pick(scans[s]);
    size_t left = (size_t)scans[s].n * per_beam;
    while (left) {
      const size_t take = std::min(left, kStageDoubles - fill);
      std::memcpy(h->stage[half] + fill, src, take * sizeof(double));
      fill += take; src += take; left -= take;
      if (fill == kStageDoubles) flush();
    }
  }
  flush();
  for (int k = 0; k < 2; ++k)
    if (pending[k]) B200_CUDA(cudaEventSynchronize(h->stage_done[k]));
}

// lasers == NULL: every scan takes the handle's params as its limits
int add_scans(b200og * h, const b200_scan * scans, int32_t n, const b200og_laser * lasers)
{
  if (n < 0 || (n > 0 && !scans)) { set_last_error("b200og_add_scans: bad argument"); return B200_ERR_INVALID_ARG; }
  size_t add = 0;
  for (int32_t s = 0; s < n; ++s) {
    if (scans[s].n < 0 || (scans[s].n > 0 && (!scans[s].ranges || !scans[s].points_xy))) {
      set_last_error("b200_scan: NULL pointer or negative size");
      return B200_ERR_INVALID_ARG;
    }
    if (lasers && !(std::isfinite(lasers[s].range_threshold) && std::isfinite(lasers[s].minimum_range) &&
                    std::isfinite(lasers[s].maximum_range))) {
      set_last_error("b200og_add_scans_lasers: non-finite laser limit");
      return B200_ERR_INVALID_ARG;
    }
    add += (size_t)scans[s].n;
  }
  const size_t old_beams = (size_t)h->start.back(), old_scans = (size_t)h->nscans();
  if (old_beams + add > (size_t)INT32_MAX) { set_last_error("b200og: more than 2^31-1 beams in the scan store"); return B200_ERR_UNSUPPORTED; }
  if (n == 0) return B200_OK;
  h->ensure_stream();
  for (auto & sp : h->stage)
    if (!sp) sp = stage_pool().take();
  OgStore & d = h->store;
  d.ensure(old_beams + add, old_scans + n, old_beams, old_scans, h->stream);   // start entry old_scans is rewritten below
  upload_rows(h, scans, n, d.ranges.p + old_beams, 1, [](const b200_scan & s) { return s.ranges; });
  upload_rows(h, scans, n, d.points.p + 2 * old_beams, 2, [](const b200_scan & s) { return s.points_xy; });
  // sensor positions, laser limits + prefix of beam counts: small, staged in the first pinned half
  double * sp = h->stage[0];
  std::vector<int32_t> st(n + 1);
  st[0] = (int32_t)old_beams;
  for (int32_t s = 0; s < n; ++s) {
    st[s + 1] = st[s] + scans[s].n;
    h->maxbeams = std::max(h->maxbeams, scans[s].n);
  }
  // (n sensor positions and limits fit the 8 MB half up to 209,715 scans per call; larger calls go in slices)
  constexpr int32_t kSlice = (int32_t)(kStageDoubles / 5);
  for (int32_t s0 = 0; s0 < n; s0 += kSlice) {
    const int32_t cnt = std::min<int32_t>(n - s0, kSlice);
    double * lp = sp + 2 * (size_t)cnt;
    for (int32_t s = 0; s < cnt; ++s) {
      sp[2 * s] = scans[s0 + s].sensor_pose[0]; sp[2 * s + 1] = scans[s0 + s].sensor_pose[1];
      const b200og_laser l = lasers ? lasers[s0 + s] : b200og_laser{h->p.range_threshold, h->p.minimum_range, h->p.maximum_range};
      lp[3 * s] = l.range_threshold; lp[3 * s + 1] = l.minimum_range; lp[3 * s + 2] = l.maximum_range;
    }
    B200_CUDA(cudaMemcpyAsync(d.sensor.p + 2 * (old_scans + s0), sp, 2 * (size_t)cnt * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    B200_CUDA(cudaMemcpyAsync(d.laser.p + 3 * (old_scans + s0), lp, 3 * (size_t)cnt * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  B200_CUDA(cudaMemcpyAsync(d.start.p + old_scans, st.data(), st.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  h->start.insert(h->start.end(), st.begin() + 1, st.end());
  h->built = false;
  return B200_OK;
}

// the store's view of scans [first, first + count): start / sensor shifted to the first scan, beams through the prefix
OgDev range_view(const b200og * h, int32_t first, int32_t count)
{
  OgDev d{};
  const OgStore & s = h->store;
  d.ranges = s.ranges.p; d.points = s.points.p; d.sensor = s.sensor.p + 2 * (size_t)first; d.start = s.start.p + first;
  d.laser = s.laser.p + 3 * (size_t)first;
  d.nscans = count;
  d.beam0 = h->start[first]; d.nbeams = h->start[first + count];
  if (first == 0 && count == h->nscans()) {
    d.maxbeams = h->maxbeams;
  } else {
    for (int32_t s = first; s < first + count; ++s) d.maxbeams = std::max(d.maxbeams, h->start[s + 1] - h->start[s]);
  }
  return d;
}

bool range_ok(const b200og * h, int32_t first, int32_t count, const char * who)
{
  if (first < 0 || count < 0 || (int64_t)first + count > h->nscans()) {
    set_last_error(std::string(who) + ": scan range outside the store");
    return false;
  }
  return true;
}

// Update's box for every scan that has none yet (scans appended since the last call included)
void ensure_boxes(b200og * h)
{
  const int32_t n = h->nscans();
  if (h->nboxed == n) return;
  h->ensure_stream();
  h->store.box.ensure(4 * (size_t)n, 4 * (size_t)h->nboxed, h->stream);
  const OgDev d = range_view(h, 0, n);
  const int32_t count = n - h->nboxed;
  k_og_scan_box<<<h->scan_blocks(count), kOgThreads, 0, h->stream>>>(d, h->nboxed, count, h->store.box.p);
  h->launched();
  h->nboxed = n;
}

int transform_scans(b200og * h, int32_t first, int32_t count, const double * basis, const double * origin, const double * sensor_poses)
{
  if (!basis || !origin) { set_last_error("b200og_transform_scans: NULL basis or origin"); return B200_ERR_INVALID_ARG; }
  if (!range_ok(h, first, count, "b200og_transform_scans")) return B200_ERR_INVALID_ARG;
  for (int k = 0; k < 9; ++k)
    if (!std::isfinite(basis[k])) { set_last_error("b200og_transform_scans: non-finite basis"); return B200_ERR_INVALID_ARG; }
  for (int k = 0; k < 3; ++k)
    if (!std::isfinite(origin[k])) { set_last_error("b200og_transform_scans: non-finite origin"); return B200_ERR_INVALID_ARG; }
  if (count == 0) return B200_OK;
  ensure_boxes(h);
  cudaStream_t st = h->stream;
  if (sensor_poses) {   // host-computed sensor poses (lasers with a mounting offset): positions only
    std::vector<double> xy(2 * (size_t)count);
    for (int32_t s = 0; s < count; ++s) { xy[2 * s] = sensor_poses[3 * s]; xy[2 * s + 1] = sensor_poses[3 * s + 1]; }
    B200_CUDA(cudaMemcpyAsync(h->store.sensor.p + 2 * (size_t)first, xy.data(), xy.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  OgTf t;
  for (int r = 0; r < 2; ++r) {
    for (int c = 0; c < 3; ++c) t.b[r][c] = basis[3 * r + c];
    t.o[r] = origin[r];
  }
  const OgDev d = range_view(h, first, count);
  const int64_t work = std::max<int64_t>(d.nbeams - d.beam0, count);
  const int nb = (int)std::min<int64_t>((work + kOgThreads - 1) / kOgThreads, (int64_t)h->sms * 8);
  h->timer_start();
  k_og_transform<<<std::max(nb, 1), kOgThreads, 0, st>>>(d, first, count, t, sensor_poses ? 0 : 1, h->store.points.p,
                                                         h->store.sensor.p, h->store.box.p);
  h->launched();
  h->timer_stop();   // the host staging of sensor_poses is released on return
  h->boxes_auth = true;
  h->built = false;
  return B200_OK;
}

int scan_boxes(b200og * h, int32_t first, int32_t count, double * boxes)
{
  if (!range_ok(h, first, count, "b200og_scan_boxes") || (count > 0 && !boxes)) {
    if (count > 0 && !boxes) set_last_error("b200og_scan_boxes: NULL output");
    return B200_ERR_INVALID_ARG;
  }
  if (count == 0) return B200_OK;
  ensure_boxes(h);
  B200_CUDA(cudaMemcpyAsync(boxes, h->store.box.p + 4 * (size_t)first, 4 * (size_t)count * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int remove_scans(b200og * h, const int32_t * idx, int32_t n)
{
  const int32_t S = h->nscans();
  if (n < 0 || (n > 0 && !idx)) { set_last_error("b200og_remove_scans: NULL indices or negative count"); return B200_ERR_INVALID_ARG; }
  for (int32_t k = 0; k < n; ++k) {
    if (idx[k] < 0 || idx[k] >= S) { set_last_error("b200og_remove_scans: index outside the store"); return B200_ERR_INVALID_ARG; }
    if (k > 0 && idx[k] <= idx[k - 1]) {
      set_last_error("b200og_remove_scans: indices not strictly increasing");
      return B200_ERR_INVALID_ARG;
    }
  }
  if (n == 0) return B200_OK;
  // the new beam prefix, and the old index of every surviving scan from the first removed one on (those are the ones that move)
  const int32_t k0 = idx[0], S2 = S - n;
  std::vector<int32_t> src;
  src.reserve((size_t)(S2 - k0));
  for (int32_t s = k0 + 1, r = 1; s < S; ++s) {
    if (r < n && idx[r] == s) { ++r; continue; }
    src.push_back(s);
  }
  std::vector<int32_t> start(h->start.begin(), h->start.begin() + k0 + 1);
  for (int32_t s : src) start.push_back(start.back() + (h->start[s + 1] - h->start[s]));
  int32_t maxbeams = 0;
  for (int32_t s = 0; s < S2; ++s) maxbeams = std::max(maxbeams, start[s + 1] - start[s]);
  const int32_t nboxed = h->nboxed <= k0 ? h->nboxed
                                         : k0 + (int32_t)(std::lower_bound(src.begin(), src.end(), h->nboxed) - src.begin());
  h->last_ms = 0.f;
  if (!src.empty()) {
    cudaStream_t st = h->stream;
    const size_t keep = (size_t)start[k0], nbeams = (size_t)start[S2], kbox = (size_t)std::min(k0, h->nboxed);
    const int32_t count = (int32_t)src.size();
    h->spare.ensure(nbeams, (size_t)S2, 0, 0, st);
    h->d_src.ensure((size_t)count, 0, st);
    if (h->nboxed) h->spare.box.ensure(4 * (size_t)nboxed, 0, st);
    // the scans before the first removed one keep their offsets: plain copies into the spare store
    h->spare.copy_from(h->store, keep, (size_t)k0, kbox, st);
    B200_CUDA(cudaMemcpyAsync(h->spare.start.p, start.data(), start.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(h->d_src.p, src.data(), src.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    const OgCompact c{h->d_src.p, k0, count, h->nboxed, h->store.dev(), h->spare.dev()};
    h->timer_start();
    k_og_compact<<<h->scan_blocks(count), kOgThreads, 0, st>>>(c);
    h->launched();
    h->timer_stop();   // start and src are released on return
    h->store.swap(h->spare, h->nboxed > 0);
  }
  // removing only trailing scans moves nothing: the device prefix up to the new end is unchanged
  h->start.swap(start);
  h->maxbeams = maxbeams;
  h->nboxed = nboxed;
  h->built = false;
  return B200_OK;
}

int build(b200og * h, int32_t first, int32_t count, b200og_info * info)
{
  if (info) std::memset(info, 0, sizeof(*info));
  h->built = false;
  if (count == 0) {
    set_last_error("OccupancyGrid::CreateFromScans: no scans (the reference returns NULL, Karto.h:5950-5952)");
    return B200_ERR_NOT_FOUND;
  }
  h->ensure_stream();
  cudaStream_t st = h->stream;
  OgDev d = range_view(h, first, count);
  const int blocks = h->sms * 8;
  h->d_partial.reserve(4 * (size_t)blocks);
  h->h_partial.reserve(4 * (size_t)blocks);
  h->d_flag.reserve(1);
  h->h_flag.reserve(1);
  h->timer_start();
  if (h->boxes_auth) {   // transformed store: the union of the stored boxes (ComputeDimensions reads them, IsDirty is clear)
    ensure_boxes(h);
    k_og_box_union<<<blocks, kOgThreads, 0, st>>>(h->store.box.p, first, count, h->d_partial.p);
  } else {
    k_og_bbox<<<blocks, kOgThreads, 0, st>>>(d, h->d_partial.p);
  }
  h->launched();
  B200_CUDA(cudaMemcpyAsync(h->h_partial.p, h->d_partial.p, 4 * (size_t)blocks * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  OgBox box;
  for (int b = 0; b < blocks; ++b) box.add(OgBox::load(h->h_partial.p + 4 * (size_t)b));
  // ComputeDimensions, Karto.h:6100-6106
  const double scale = 1.0 / h->p.resolution;
  const int32_t width = to_int32(round_half_away((box.mxx - box.mnx) * scale));
  const int32_t height = to_int32(round_half_away((box.mxy - box.mny) * scale));
  if (width < 0 || height < 0) { set_last_error("OccupancyGrid: bounding box of the scans is not finite"); return B200_ERR_UNSUPPORTED; }
  const int64_t stride = ((int64_t)width + 7) & ~(int64_t)7;   // Karto.h:4640
  const int64_t ncells = stride * height;
  if (stride > INT32_MAX || ncells > INT32_MAX) {
    set_last_error("OccupancyGrid: width step * height exceeds 2^31-1 cells");
    return B200_ERR_UNSUPPORTED;
  }
  h->info.width = width; h->info.height = height; h->info.stride = (int32_t)stride;
  h->info.offset[0] = box.mnx; h->info.offset[1] = box.mny;
  const size_t cells = (size_t)ncells;
  h->d_pass.reserve(cells + 4);
  h->d_hits.reserve(cells + 4);
  h->d_cells.reserve(cells + 4);
  d.scale = scale; d.offx = box.mnx; d.offy = box.mny;
  d.width = width; d.height = height; d.stride = (int32_t)stride;
  d.pass = h->d_pass.p; d.hits = h->d_hits.p; d.cells = h->d_cells.p; d.flag = h->d_flag.p;
  B200_CUDA(cudaMemsetAsync(h->d_flag.p, 0, sizeof(int32_t), st));
  if (cells) {
    B200_CUDA(cudaMemsetAsync(h->d_pass.p, 0, cells * sizeof(uint32_t), st));
    B200_CUDA(cudaMemsetAsync(h->d_hits.p, 0, cells * sizeof(uint32_t), st));
    k_og_trace<<<blocks, kOgThreads, 0, st>>>(d);
    h->launched();
    const size_t quads = cells / 4;   // stride is a multiple of 8
    const int ub = (int)std::min<size_t>((quads + kOgThreads - 1) / kOgThreads, (size_t)h->sms * 16);
    k_og_update<<<std::max(ub, 1), kOgThreads, 0, st>>>(d, h->p.min_pass_through, h->p.occupancy_threshold, quads);
    h->launched();
  }
  B200_CUDA(cudaMemcpyAsync(h->h_flag.p, h->d_flag.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  h->timer_stop();
  if (h->h_flag.p[0]) {
    set_last_error("OccupancyGrid: a beam spans more than 2^24 cells (corrupt pose or resolution)");
    return B200_ERR_UNSUPPORTED;
  }
  h->built = true;
  if (info) *info = h->info;
  return B200_OK;
}

}  // namespace

extern "C" {

void b200og_default_params(b200og_params * p)
{
  if (!p) return;
  p->resolution = 0.05;
  p->range_threshold = 12.0;
  p->minimum_range = 0.1;
  p->maximum_range = 30.0;
  p->min_pass_through = 2;        // Karto.h:5921
  p->occupancy_threshold = 0.1;   // Karto.h:5922
}

int b200og_create(const b200og_params * params, b200og ** out)
{
  B200_GUARD_BEGIN
  if (!params || !out) { set_last_error("b200og_create: NULL argument"); return B200_ERR_INVALID_ARG; }
  *out = nullptr;
  if (!params_ok(*params)) return B200_ERR_INVALID_ARG;
  require_device();
  std::unique_ptr<b200og> h(new b200og());
  h->p = *params;
  h->ensure_stream();
  *out = h.release();
  return B200_OK;
  B200_GUARD_END
}

void b200og_destroy(b200og * h)
{
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->ev0) { cudaEventDestroy(h->ev0); cudaEventDestroy(h->ev1); }
  for (auto & e : h->stage_done) if (e) cudaEventDestroy(e);
  for (auto & sp : h->stage) { stage_pool().give(sp); sp = nullptr; }
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

int b200og_set_stream(b200og * h, void * s)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  if (h->stream) B200_CUDA(cudaStreamSynchronize(h->stream));
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  h->stream = static_cast<cudaStream_t>(s);
  h->own_stream = false;
  h->ensure_stream();
  return B200_OK;
  B200_GUARD_END
}

int b200og_add_scans(b200og * h, const b200_scan * scans, int32_t n)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return add_scans(h, scans, n, nullptr);
  B200_GUARD_END
}

int b200og_add_scans_lasers(b200og * h, const b200_scan * scans, int32_t n, const b200og_laser * lasers)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return add_scans(h, scans, n, lasers);
  B200_GUARD_END
}

int b200og_clear_scans(b200og * h)
{
  if (!h) return B200_ERR_INVALID_ARG;
  h->start.assign(1, 0);
  h->maxbeams = 0;
  h->nboxed = 0;
  h->boxes_auth = false;
  h->built = false;
  return B200_OK;
}

int32_t b200og_num_scans(const b200og * h) { return h ? h->nscans() : 0; }

int b200og_build(b200og * h, b200og_info * info)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return build(h, 0, h->nscans(), info);
  B200_GUARD_END
}

int b200og_build_range(b200og * h, int32_t first, int32_t count, b200og_info * info)
{
  B200_GUARD_BEGIN
  if (info) std::memset(info, 0, sizeof(*info));
  if (!h) return B200_ERR_INVALID_ARG;
  if (!range_ok(h, first, count, "b200og_build_range")) return B200_ERR_INVALID_ARG;
  return build(h, first, count, info);
  B200_GUARD_END
}

int b200og_transform_scans(b200og * h, int32_t first, int32_t count, const double basis[9], const double origin[3],
                           const double * sensor_poses)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return transform_scans(h, first, count, basis, origin, sensor_poses);
  B200_GUARD_END
}

int b200og_scan_boxes(b200og * h, int32_t first, int32_t count, double * boxes)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return scan_boxes(h, first, count, boxes);
  B200_GUARD_END
}

int b200og_remove_scans(b200og * h, const int32_t * indices, int32_t n)
{
  B200_GUARD_BEGIN
  if (!h) { set_last_error("b200og_remove_scans: NULL handle"); return B200_ERR_INVALID_ARG; }
  return remove_scans(h, indices, n);
  B200_GUARD_END
}

int b200og_fetch(b200og * h, uint8_t * cells, uint32_t * pass, uint32_t * hits)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  if (!h->built) { set_last_error("b200og_fetch: no successful build"); return B200_ERR_NOT_FOUND; }
  const size_t n = (size_t)h->info.stride * h->info.height;
  if (n) {
    if (cells) B200_CUDA(cudaMemcpyAsync(cells, h->d_cells.p, n, cudaMemcpyDeviceToHost, h->stream));
    if (pass) B200_CUDA(cudaMemcpyAsync(pass, h->d_pass.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    if (hits) B200_CUDA(cudaMemcpyAsync(hits, h->d_hits.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B200_OK;
  B200_GUARD_END
}

int b200og_fetch_nav(b200og * h, int8_t * data)
{
  B200_GUARD_BEGIN
  if (!h || !data) return B200_ERR_INVALID_ARG;
  if (!h->built) { set_last_error("b200og_fetch_nav: no successful build"); return B200_ERR_NOT_FOUND; }
  const size_t n = (size_t)h->info.width * h->info.height;
  if (n) {
    h->d_nav.reserve(n);
    const int nb = (int)std::min<size_t>((n + kOgThreads - 1) / kOgThreads, (size_t)h->sms * 16);
    k_og_nav<<<nb, kOgThreads, 0, h->stream>>>(h->d_cells.p, h->info.width, h->info.height, h->info.stride, h->d_nav.p);
    h->launched();
    B200_CUDA(cudaMemcpyAsync(data, h->d_nav.p, n, cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B200_OK;
  B200_GUARD_END
}

int b200og_kernel_ms(b200og * h, float * ms)
{
  if (!h || !ms) return B200_ERR_INVALID_ARG;
  *ms = h->last_ms;
  return B200_OK;
}

int64_t b200og_launch_count(const b200og * h) { return h ? h->launches : 0; }

int b200og_create_from_scans(const b200og_params * params, const b200_scan * scans, int32_t n, b200og_info * info, b200og ** out)
{
  B200_GUARD_BEGIN
  if (!out) { set_last_error("b200og_create_from_scans: NULL argument"); return B200_ERR_INVALID_ARG; }
  *out = nullptr;
  if (info) std::memset(info, 0, sizeof(*info));
  b200og * raw = nullptr;
  int rc = b200og_create(params, &raw);
  if (rc != B200_OK) return rc;
  std::unique_ptr<b200og, void (*)(b200og *)> h(raw, b200og_destroy);
  rc = add_scans(h.get(), scans, n, nullptr);
  if (rc == B200_OK) rc = build(h.get(), 0, h->nscans(), info);
  if (rc != B200_OK) return rc;
  *out = h.release();
  return B200_OK;
  B200_GUARD_END
}

}  // extern "C"
