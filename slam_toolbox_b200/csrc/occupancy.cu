// Occupancy grid from scans: karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961), the
// map-publish step either side of the hot path (src/slam_mapper.cpp:63-69,
// src/slam_toolbox_common.cpp:630-654).  SURVEY.md 8(f) row 4.
//
// Data in HBM (all FP64 inputs are the reference's own values, nothing is re-derived):
//   ranges [B]      raw range readings of all stored scans, scan after scan
//   points [B][2]   their unfiltered world-frame point readings (LocalizedRangeScan::GetPointReadings(false))
//   sensor [S][2]   sensor position of every scan; start [S+1] = first beam of every scan
//   pass, hits [height][stride] uint32 counters; cells [height][stride] uint8 states
//
// Kernels of one build (b200og_build):
//   k_og_bbox    min / max over the sensor positions and the in-range points   (ComputeDimensions)
//   k_og_trace   a warp takes 32 adjacent beams of a scan, one per lane, and runs the reference's integer
//                Bresenham loop on them in lock step; equal cell indices of neighbouring lanes are merged
//                into one RED.ADD of the run length (no return value) -- integer sums commute, so the
//                result does not depend on the order and equals the reference's sequential loop
//   k_og_update  counters -> cell state (UpdateCell Karto.h:6241-6254), FP64 ratio test as the reference
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
  int32_t nscans, maxbeams;
  int64_t nbeams;
  double rt, minr, maxr;
  double scale, offx, offy;
  int32_t width, height, stride;
  uint32_t * pass;
  uint32_t * hits;
  uint8_t * cells;
  int32_t * flag;          // set when a beam was refused (kOgMaxCells)
};

__device__ __forceinline__ double warp_min(double v)
{
  for (int o = 16; o; o >>= 1) { double w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
  return v;
}
__device__ __forceinline__ double warp_max(double v)
{
  for (int o = 16; o; o >>= 1) { double w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
  return v;
}

// partial[block][4] = {min x, min y, max x, max y}; BoundingBox2 starts at +-999999999999999999.99999 (Karto.h:2845-2849)
__global__ void __launch_bounds__(kOgThreads) k_og_bbox(OgDev d, double * partial)
{
  __shared__ double sm[4][kOgThreads / 32];
  const double big = 999999999999999999.99999;
  double mnx = big, mny = big, mxx = -big, mxy = -big;
  const int64_t step = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = t0; i < d.nbeams; i += step) {
    const double r = d.ranges[i];
    if (r >= d.minr && r <= d.rt) {   // math::InRange (Math.h:123), LocalizedRangeScan::Update Karto.h:5662
      const double x = d.points[2 * i], y = d.points[2 * i + 1];
      if (x < mnx) mnx = x;   // MakeFloor / MakeCeil: strict comparisons, NaN never wins
      if (y < mny) mny = y;
      if (x > mxx) mxx = x;
      if (y > mxy) mxy = y;
    }
  }
  for (int64_t s = t0; s < d.nscans; s += step) {   // m_BoundingBox.Add(scanPose.GetPosition()) Karto.h:5694
    const double x = d.sensor[2 * s], y = d.sensor[2 * s + 1];
    if (x < mnx) mnx = x;
    if (y < mny) mny = y;
    if (x > mxx) mxx = x;
    if (y > mxy) mxy = y;
  }
  mnx = warp_min(mnx); mny = warp_min(mny); mxx = warp_max(mxx); mxy = warp_max(mxy);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sm[0][w] = mnx; sm[1][w] = mny; sm[2][w] = mxx; sm[3][w] = mxy; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kOgThreads / 32; ++k) {
      if (sm[0][k] < mnx) mnx = sm[0][k];
      if (sm[1][k] < mny) mny = sm[1][k];
      if (sm[2][k] > mxx) mxx = sm[2][k];
      if (sm[3][k] > mxy) mxy = sm[3][k];
    }
    double * o = partial + 4 * (size_t)blockIdx.x;
    o[0] = mnx; o[1] = mny; o[2] = mxx; o[3] = mxy;
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
    int32_t x = 0, y = 0, dX = 0, dY = 0, ystep = 1, len = 0;
    bool steep = false, end_hit = false;
    int32_t end_key = -1;
    if (beam < d.start[scan + 1] - b0) {
      const int64_t i = (int64_t)b0 + beam;
      const double r = d.ranges[i];
      if (!(r <= d.minr || r >= d.maxr || r != r)) {                    // ignored readings, Karto.h:6160
        const bool valid_end = r < (d.rt - kTolerance);                 // Karto.h:6158
        const double sx = d.sensor[2 * scan], sy = d.sensor[2 * scan + 1];
        double px = d.points[2 * i], py = d.points[2 * i + 1];
        if (r >= d.rt) {                                                // trace up to the range threshold, Karto.h:6164-6171
          const double ratio = d.rt / r;
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
};

}  // namespace b200

using namespace b200;

struct b200og {
  b200og_params p{};
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // scan store
  GrowBuf<double> d_ranges, d_points, d_sensor;
  GrowBuf<int32_t> d_start;
  std::vector<int32_t> start{0};
  int32_t maxbeams = 0;
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

int add_scans(b200og * h, const b200_scan * scans, int32_t n)
{
  if (n < 0 || (n > 0 && !scans)) { set_last_error("b200og_add_scans: bad argument"); return B200_ERR_INVALID_ARG; }
  size_t add = 0;
  for (int32_t s = 0; s < n; ++s) {
    if (scans[s].n < 0 || (scans[s].n > 0 && (!scans[s].ranges || !scans[s].points_xy))) {
      set_last_error("b200_scan: NULL pointer or negative size");
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
  h->d_ranges.ensure(old_beams + add, old_beams, h->stream);
  h->d_points.ensure(2 * (old_beams + add), 2 * old_beams, h->stream);
  h->d_sensor.ensure(2 * (old_scans + n), 2 * old_scans, h->stream);
  h->d_start.ensure(old_scans + n + 1, old_scans, h->stream);   // entry old_scans is rewritten below
  upload_rows(h, scans, n, h->d_ranges.p + old_beams, 1, [](const b200_scan & s) { return s.ranges; });
  upload_rows(h, scans, n, h->d_points.p + 2 * old_beams, 2, [](const b200_scan & s) { return s.points_xy; });
  // sensor positions + prefix of beam counts: small, staged in the first pinned half
  double * sp = h->stage[0];
  std::vector<int32_t> st(n + 1);
  st[0] = (int32_t)old_beams;
  for (int32_t s = 0; s < n; ++s) {
    st[s + 1] = st[s] + scans[s].n;
    h->maxbeams = std::max(h->maxbeams, scans[s].n);
  }
  // (n sensor positions fit the 8 MB half up to 524,288 scans per call; larger calls go in slices)
  for (int32_t s0 = 0; s0 < n; s0 += (int32_t)(kStageDoubles / 2)) {
    const int32_t cnt = std::min<int32_t>(n - s0, (int32_t)(kStageDoubles / 2));
    for (int32_t s = 0; s < cnt; ++s) { sp[2 * s] = scans[s0 + s].sensor_pose[0]; sp[2 * s + 1] = scans[s0 + s].sensor_pose[1]; }
    B200_CUDA(cudaMemcpyAsync(h->d_sensor.p + 2 * (old_scans + s0), sp, 2 * (size_t)cnt * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  B200_CUDA(cudaMemcpyAsync(h->d_start.p + old_scans, st.data(), st.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  h->start.insert(h->start.end(), st.begin() + 1, st.end());
  h->built = false;
  return B200_OK;
}

int build(b200og * h, b200og_info * info)
{
  if (info) std::memset(info, 0, sizeof(*info));
  h->built = false;
  if (h->nscans() == 0) {
    set_last_error("OccupancyGrid::CreateFromScans: no scans (the reference returns NULL, Karto.h:5950-5952)");
    return B200_ERR_NOT_FOUND;
  }
  h->ensure_stream();
  cudaStream_t st = h->stream;
  OgDev d{};
  d.ranges = h->d_ranges.p; d.points = h->d_points.p; d.sensor = h->d_sensor.p; d.start = h->d_start.p;
  d.nscans = h->nscans(); d.maxbeams = h->maxbeams; d.nbeams = h->start.back();
  d.rt = h->p.range_threshold; d.minr = h->p.minimum_range; d.maxr = h->p.maximum_range;
  const int blocks = h->sms * 8;
  h->d_partial.reserve(4 * (size_t)blocks);
  h->h_partial.reserve(4 * (size_t)blocks);
  h->d_flag.reserve(1);
  h->h_flag.reserve(1);
  B200_CUDA(cudaEventRecord(h->ev0, st));
  k_og_bbox<<<blocks, kOgThreads, 0, st>>>(d, h->d_partial.p);
  B200_CUDA(cudaGetLastError());
  ++h->launches;
  B200_CUDA(cudaMemcpyAsync(h->h_partial.p, h->d_partial.p, 4 * (size_t)blocks * sizeof(double), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  const double big = 999999999999999999.99999;
  double mnx = big, mny = big, mxx = -big, mxy = -big;
  for (int b = 0; b < blocks; ++b) {
    const double * o = h->h_partial.p + 4 * (size_t)b;
    if (o[0] < mnx) mnx = o[0];
    if (o[1] < mny) mny = o[1];
    if (o[2] > mxx) mxx = o[2];
    if (o[3] > mxy) mxy = o[3];
  }
  // ComputeDimensions, Karto.h:6100-6106
  const double scale = 1.0 / h->p.resolution;
  const int32_t width = to_int32(round_half_away((mxx - mnx) * scale));
  const int32_t height = to_int32(round_half_away((mxy - mny) * scale));
  if (width < 0 || height < 0) { set_last_error("OccupancyGrid: bounding box of the scans is not finite"); return B200_ERR_UNSUPPORTED; }
  const int64_t stride = ((int64_t)width + 7) & ~(int64_t)7;   // Karto.h:4640
  const int64_t ncells = stride * height;
  if (stride > INT32_MAX || ncells > INT32_MAX) {
    set_last_error("OccupancyGrid: width step * height exceeds 2^31-1 cells");
    return B200_ERR_UNSUPPORTED;
  }
  h->info.width = width; h->info.height = height; h->info.stride = (int32_t)stride;
  h->info.offset[0] = mnx; h->info.offset[1] = mny;
  const size_t cells = (size_t)ncells;
  h->d_pass.reserve(cells + 4);
  h->d_hits.reserve(cells + 4);
  h->d_cells.reserve(cells + 4);
  d.scale = scale; d.offx = mnx; d.offy = mny;
  d.width = width; d.height = height; d.stride = (int32_t)stride;
  d.pass = h->d_pass.p; d.hits = h->d_hits.p; d.cells = h->d_cells.p; d.flag = h->d_flag.p;
  B200_CUDA(cudaMemsetAsync(h->d_flag.p, 0, sizeof(int32_t), st));
  if (cells) {
    B200_CUDA(cudaMemsetAsync(h->d_pass.p, 0, cells * sizeof(uint32_t), st));
    B200_CUDA(cudaMemsetAsync(h->d_hits.p, 0, cells * sizeof(uint32_t), st));
    k_og_trace<<<blocks, kOgThreads, 0, st>>>(d);
    B200_CUDA(cudaGetLastError());
    const size_t quads = cells / 4;   // stride is a multiple of 8
    const int ub = (int)std::min<size_t>((quads + kOgThreads - 1) / kOgThreads, (size_t)h->sms * 16);
    k_og_update<<<std::max(ub, 1), kOgThreads, 0, st>>>(d, h->p.min_pass_through, h->p.occupancy_threshold, quads);
    B200_CUDA(cudaGetLastError());
    h->launches += 2;
  }
  B200_CUDA(cudaMemcpyAsync(h->h_flag.p, h->d_flag.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaEventRecord(h->ev1, st));
  B200_CUDA(cudaStreamSynchronize(st));
  B200_CUDA(cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
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
  return add_scans(h, scans, n);
  B200_GUARD_END
}

int b200og_clear_scans(b200og * h)
{
  if (!h) return B200_ERR_INVALID_ARG;
  h->start.assign(1, 0);
  h->maxbeams = 0;
  h->built = false;
  return B200_OK;
}

int32_t b200og_num_scans(const b200og * h) { return h ? h->nscans() : 0; }

int b200og_build(b200og * h, b200og_info * info)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return build(h, info);
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
    B200_CUDA(cudaGetLastError());
    ++h->launches;
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
  rc = add_scans(h.get(), scans, n);
  if (rc == B200_OK) rc = build(h.get(), info);
  if (rc != B200_OK) return rc;
  *out = h.release();
  return B200_OK;
  B200_GUARD_END
}

}  // extern "C"
