// b200slam scan matcher: Hopper-native implementation of karto::ScanMatcher::MatchScan
// (reference: lib/karto_sdk/src/Mapper.cpp:477-1208, "M.cpp" below; Karto.h = "K.h",
// Mapper.h = "M.h").  This file holds
//   * the host orchestration behind the C ABI in include/b200slam.h (grid geometry,
//     lookup-table construction -- the only place libm sin/cos is evaluated --, the FP64
//     epilogue in the reference's summation order), and
//   * the generic ("v1") CUDA kernels: raster (max-stamp of the smear kernel), the exhaustive
//     (x, y, theta) correlation, and the fused per-pair sweep kernel with its on-device
//     arg-max / tie / covariance reduction.
// The smem-tiled fast path for loop-closure sweeps lives in sm_sweep_fast.cu.
//
// Compile with -fmad=false (device) and -ffp-contract=off (host): every double expression
// below must round exactly like the reference's x86-64 build.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <functional>
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "sm_math.cuh"
#include "sm_types.cuh"
#include "sm_device.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
void set_last_error(const std::string & s) { g_last_error = s; }

void require_device()
{
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_last_error(std::string("no CUDA device available: ") + cudaGetErrorString(e) +
                   " -- b200slam has no CPU fallback");
    throw CudaFail{B200_ERR_CUDA};
  }
}

// ------------------------------------------------------------------------------------------
// host thread pool
// ------------------------------------------------------------------------------------------
namespace {
class HostPool {
 public:
  explicit HostPool(int workers)
  {
    for (int i = 0; i < workers; ++i) threads_.emplace_back([this] { loop(); });
  }
  ~HostPool()
  {
    { std::lock_guard<std::mutex> l(m_); stop_ = true; ++epoch_; epoch_a_.store(epoch_); }
    cv_.notify_all();
    for (auto & t : threads_) t.join();
  }
  int size() const { return (int)threads_.size() + 1; }
  void run(int n, const std::function<void(int)> & fn)
  {
    if (n <= 0) return;
    if (threads_.empty() || n == 1) { for (int i = 0; i < n; ++i) fn(i); return; }
    std::lock_guard<std::mutex> serial(run_m_);   // one parallel_for at a time (handles may be used from several threads)
    {
      std::lock_guard<std::mutex> l(m_);
      fn_ = &fn; n_ = n; next_.store(0); done_.store(0); ++epoch_;
      epoch_a_.store(epoch_, std::memory_order_release);
    }
    cv_.notify_all();
    work();
    // every index finished AND every worker out of work(): nobody can touch next_ / fn_ of this job any more
    while (done_.load(std::memory_order_acquire) < n) std::this_thread::yield();
    std::unique_lock<std::mutex> l(m_);
    idle_.wait(l, [&] { return active_ == 0; });
    fn_ = nullptr;
  }

 private:
  void work()
  {
    for (;;) {
      const int i = next_.fetch_add(1);
      if (i >= n_) break;
      (*fn_)(i);
      done_.fetch_add(1, std::memory_order_release);
    }
  }
  void loop()
  {
    uint64_t seen = 0;
    for (;;) {
      // a burst of parallel_for calls (one match = valid points, two lookup tables, two epilogues) arrives within a few hundred
      // microseconds: poll for that long before sleeping on the condition variable, whose wake-up costs 10-30 us per call
      const auto spin_until = std::chrono::steady_clock::now() + std::chrono::microseconds(300);
      while (epoch_a_.load(std::memory_order_acquire) == seen && std::chrono::steady_clock::now() < spin_until) {
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
      }
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return epoch_ != seen; });
        seen = epoch_;
        if (stop_) return;
        if (!fn_) continue;
        ++active_;
      }
      work();
      { std::lock_guard<std::mutex> l(m_); --active_; }
      idle_.notify_all();
    }
  }
  std::vector<std::thread> threads_;
  std::mutex m_, run_m_;
  std::condition_variable cv_, idle_;
  const std::function<void(int)> * fn_ = nullptr;
  int n_ = 0, active_ = 0;
  std::atomic<int> next_{0}, done_{0};
  std::atomic<uint64_t> epoch_a_{0};   // copy of epoch_ for the lock-free poll
  uint64_t epoch_ = 0;
  bool stop_ = false;
};

HostPool & pool()
{
  static HostPool p([] {
    int want = 0;
    if (const char * e = std::getenv("B200_HOST_THREADS")) want = std::atoi(e);
    if (want <= 0) {
      const int hw = (int)std::thread::hardware_concurrency();
      want = std::max(1, std::min(8, hw / 2));
    }
    return want - 1;
  }());
  return p;
}
}  // namespace

void host_parallel_for(int n, const std::function<void(int)> & fn) { pool().run(n, fn); }
int host_pool_threads() { return pool().size(); }

// ------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------

// CorrelationGrid::SmearPoint (M.h:1152-1183) for a list of occupied cells. One thread per (cell, kernel row):
// the row is applied word by word (4 cells at a time) with a byte-wise max and a 32-bit CAS, so a 41-tap row
// costs ~11 word updates instead of 41 byte updates. cells = packed ROI coordinates gx | gy << 16; negative = skipped.
__global__ void k_stamp(uint8_t * __restrict__ grid, int stride, int roi_x, int roi_y,
                        const int32_t * __restrict__ cells, int ncells,
                        const uint8_t * __restrict__ kern, int ksize)
{
  const int half = ksize / 2;
  const long long total = (long long)ncells * ksize;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int c = int(t / ksize), j = int(t % ksize);
    const int32_t cell = cells[c];
    if (cell < 0) continue;
    const int x0 = (cell & 0xFFFF) + roi_x - half;          // first column of the kernel row
    const int gy = (cell >> 16) + roi_y + j - half;
    const uint8_t * krow = kern + (size_t)j * ksize;
    uint8_t * rowp = grid + (size_t)gy * stride;
    for (int w0 = x0 & ~3; w0 < x0 + ksize; w0 += 4) {      // stride is a multiple of 8: words never straddle rows
      uint32_t kw = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int i = w0 + b - x0;
        if (i >= 0 && i < ksize) kw |= (uint32_t)krow[i] << (8 * b);
      }
      if (kw == 0) continue;
      uint32_t * wp = reinterpret_cast<uint32_t *>(rowp + w0);
      uint32_t old = *wp;
      uint32_t nw = __vmaxu4(old, kw);
      while (nw != old) {
        const uint32_t prev = atomicCAS(wp, old, nw);
        if (prev == old) break;
        old = prev;
        nw = __vmaxu4(old, kw);
      }
    }
  }
}

// ScanMatcher::GetResponse numerators (M.cpp:1172-1208) for every (pose, angle):
// sums[p * nA + a] = sum_i grid[pos[p] + off[a][i]], skipping invalid beams and indices outside [0, data_size).
// The grid (6.3 MB at the sequential matcher's 0.01 m) lives in global memory / L2, so a lookup costs an L2 round trip and the
// kernel is bound by how many of them are in flight, not by bandwidth: a block takes 32 consecutive poses of one angle (the
// lanes -- consecutive poses are 2 cells apart, so one warp load touches 1-2 sectors per grid row) and splits the beams over
// its kCorrWarps warps (interleaved), each lane keeping 8 loads in flight; the partial sums meet in shared memory.
// Round 1's kernel ran one thread per pose over all 1081 beams, at low occupancy and few loads in flight.
// gridDim.y is capped at 65,535 (kMaxGridY) while a window may have more angles (+-180 deg at 0.005 deg: 72,001): a block then
// takes angles blockIdx.y, blockIdx.y + gridDim.y, ...
constexpr int kCorrWarps = 8;
constexpr int kMaxGridY = 65535;
__global__ void __launch_bounds__(32 * kCorrWarps) k_correlate(const uint8_t * __restrict__ grid, int data_size,
                                                               const int32_t * __restrict__ offsets, const int32_t * __restrict__ pos,
                                                               int P, int nA, int n, int32_t * __restrict__ sums)
{
  extern __shared__ int32_t s_off[];
  __shared__ int s_part[kCorrWarps][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p = blockIdx.x * 32 + lane;
  const int base = p < P ? pos[p] : 0;
  for (int a = blockIdx.y; a < nA; a += gridDim.y) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) s_off[i] = offsets[(size_t)a * n + i];
    __syncthreads();
    int acc = 0;
    if (p < P) {
#pragma unroll 8
      for (int i = warp; i < n; i += kCorrWarps) {
        const int idx = base + s_off[i];
        if ((unsigned)idx < (unsigned)data_size) acc += __ldg(grid + idx);
      }
    }
    s_part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && p < P) {
      int t = 0;
#pragma unroll
      for (int w = 0; w < kCorrWarps; ++w) t += s_part[w][lane];
      sums[(size_t)p * nA + a] = t;
    }
    if (a + gridDim.y < nA) __syncthreads();   // every warp is done with this angle's s_off and s_part before the next is staged
  }
}

// The same numerators for a handful of poses (the fine pass: 3 x 3 poses x 11 angles): one warp per (pose, angle), the lanes
// split the beams.
__global__ void __launch_bounds__(256) k_correlate_few(const uint8_t * __restrict__ grid, int data_size,
                                                       const int32_t * __restrict__ offsets, const int32_t * __restrict__ pos,
                                                       int P, int nA, int n, int32_t * __restrict__ sums)
{
  const int lane = threadIdx.x & 31;
  const int item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (item >= P * nA) return;
  const int p = item / nA, a = item - p * nA;
  const int base = pos[p];
  const int32_t * off = offsets + (size_t)a * n;
  int acc = 0;
#pragma unroll 4
  for (int i = lane; i < n; i += 32) {
    const int idx = base + off[i];
    if ((unsigned)idx < (unsigned)data_size) acc += __ldg(grid + idx);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) sums[(size_t)p * nA + a] = acc;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------

static double normalize_angle(double angle)   // Math.h:182-205
{
  while (angle < -kPi) {
    if (angle < -k2Pi) angle += (uint32_t)(angle / -k2Pi) * k2Pi; else angle += k2Pi;
  }
  while (angle > kPi) {
    if (angle > k2Pi) angle -= (uint32_t)(angle / k2Pi) * k2Pi; else angle -= k2Pi;
  }
  return angle;
}
double normalize_angle_difference(double minuend, double subtrahend)   // Math.h:215-226
{
  while (minuend - subtrahend < -kPi) minuend += k2Pi;
  while (minuend - subtrahend > kPi) minuend -= k2Pi;
  return minuend;
}

}  // namespace b200

using namespace b200;

namespace b200 {

static int half_kernel(double smear, double resolution)   // M.h:1275-1280
{
  return (int)round_half_away(2.0 * smear / resolution);
}

// ScanMatcher::Create (M.cpp:477-522) + CorrelationGrid ctor / CalculateKernel (M.h:1194-1266)
static int build_geometry(const b200sm_params & p, GridGeom & g, int & probs_side)
{
  if (p.resolution <= 0 || p.search_size <= 0 || p.smear_deviation < 0 || p.range_threshold <= 0) {
    set_last_error("ScanMatcher::Create: invalid parameters (Mapper.cpp:481-493)");
    return B200_ERR_INVALID_ARG;
  }
  if (!(p.coarse_angle_resolution > 0) || !(p.coarse_search_angle_offset > 0) || !(p.fine_search_angle_offset > 0)) {
    set_last_error("angle offsets / resolutions must be positive (Karto.h:6803-6804)");
    return B200_ERR_INVALID_ARG;
  }
  uint32_t side = (uint32_t)(round_half_away(p.search_size / p.resolution) + 1);
  uint32_t margin = (uint32_t)ceil(p.range_threshold / p.resolution);
  int grid_size = (int)(side + 2 * margin);
  if (grid_size % 2 != 1) {
    set_last_error("ScanMatcher::Create: correlation grid size must be odd (assert, Mapper.cpp:508)");
    return B200_ERR_INVALID_ARG;
  }
  uint32_t border = (uint32_t)half_kernel(p.smear_deviation, p.resolution) + 1;
  g.width = (int)(grid_size + 2 * border);
  g.height = g.width;
  g.stride = (int)(((size_t)g.width + 7) & ~(size_t)7);
  g.roi_x = g.roi_y = (int)border;
  g.roi_w = g.roi_h = grid_size;
  g.data_size = g.stride * g.height;
  g.scale = 1.0 / p.resolution;
  if (g.roi_w >= 32768) {
    set_last_error("correlation grid too large for 16-bit packed cell coordinates");
    return B200_ERR_UNSUPPORTED;
  }
  // CalculateKernel
  double resolution = 1.0 / g.scale;   // GetResolution(), K.h:4518
  const double min_dev = 0.5 * resolution, max_dev = 10 * resolution;
  if (!(p.smear_deviation >= min_dev && p.smear_deviation <= max_dev)) {
    set_last_error("smear deviation must be within [0.5, 10] * resolution (Mapper.h:1226-1235)");
    return B200_ERR_INVALID_ARG;
  }
  g.ksize = 2 * half_kernel(p.smear_deviation, resolution) + 1;
  if ((int)border < g.ksize / 2 + 1) {
    set_last_error("grid border smaller than the smear kernel");
    return B200_ERR_UNSUPPORTED;
  }
  g.kernel.assign((size_t)g.ksize * g.ksize, 0);
  int half = g.ksize / 2;
  g.order_dependent = false;
  for (int i = -half; i <= half; i++) {
    for (int j = -half; j <= half; j++) {
      double d = hypot(i * resolution, j * resolution);
      double z = exp(-0.5 * pow(d / p.smear_deviation, 2));
      uint32_t kv = (uint32_t)round_half_away(z * kOccupied);
      g.kernel[(size_t)(i + half) + (size_t)g.ksize * (j + half)] = (uint8_t)kv;
      if (kv >= (uint32_t)kOccupied && !(i == 0 && j == 0)) g.order_dependent = true;
    }
  }
  probs_side = (int)side;
  return B200_OK;
}

// valid, in-ROI points of the base scans as packed ROI cells, in insertion order
// (AddScans/AddScan/FindValidPoints, M.cpp:1032-1164), with the order-dependent
// "already occupied" rule (M.cpp:1093-1096) resolved here when the kernel needs it.
static void host_cells(const GridGeom & g, CellScratch & sc, const b200_scan * query, const b200_scan * base, int nbase,
                       std::vector<int32_t> & cells)
{
  cells.clear();
  const double vx = query->sensor_pose[0], vy = query->sensor_pose[1];
  // FindValidPoints + WorldToGrid + ROI test are independent per base scan: one task each, concatenated in scan order
  std::vector<std::vector<int32_t>> per(nbase);
  auto one_scan = [&](int b) {
    const b200_scan & s = base[b];
    if (s.n <= 0 || s.points_xy == nullptr) return;   // NULL scans are skipped, M.cpp:1039
    std::vector<int32_t> & out = per[b];
    out.reserve((size_t)s.n);
    ValidPointState st;
    st.init();
    for (int i = 0; i < s.n; ++i) {
      int lo, hi;
      st.step(i, s.points_xy[2 * i], s.points_xy[2 * i + 1], vx, vy, lo, hi);
      for (int t = lo; t < hi; ++t) {
        int gx = world_to_grid(s.points_xy[2 * t], g.off_x, g.scale);
        int gy = world_to_grid(s.points_xy[2 * t + 1], g.off_y, g.scale);
        if (is_up_to(gx, g.roi_w) && is_up_to(gy, g.roi_h)) out.push_back(gx | (gy << 16));
      }
    }
  };
  if (nbase >= 2) host_parallel_for(nbase, one_scan); else for (int b = 0; b < nbase; ++b) one_scan(b);
  for (int b = 0; b < nbase; ++b) cells.insert(cells.end(), per[b].begin(), per[b].end());
  // AddScan's "cell already occupied" test (M.cpp:1093-1096): a point is dropped when its cell already holds 100,
  // i.e. lies in the 100-valued footprint of an earlier KEPT point (the centre only for most kernels; centre +
  // 4-neighbours for the shipped YAML smear). A bitmap over the full grid with lazy clearing replays it in O(points).
  // With a kernel whose only 100 is its centre the rule drops exact duplicates of earlier cells: the max-stamp raster is the
  // same with or without them, so the replay is skipped (it is most of this function's time).
  if (g.order_dependent) {
    const int half = g.ksize / 2;
    const size_t nbits = (size_t)g.width * g.height;
    if (sc.bits.size() * 64 < nbits) sc.bits.assign((nbits + 63) / 64, 0);
    if (sc.foot.empty()) {
      for (int j = -half; j <= half; ++j)
        for (int i = -half; i <= half; ++i)
          if (g.kernel[(size_t)(i + half) + (size_t)g.ksize * (j + half)] >= kOccupied) sc.foot.emplace_back(i, j);
    }
    size_t w = 0;
    for (size_t k = 0; k < cells.size(); ++k) {
      const int gx = (cells[k] & 0xFFFF) + g.roi_x, gy = (cells[k] >> 16) + g.roi_y;
      const size_t bit = (size_t)gy * g.width + gx;
      if (sc.bits[bit >> 6] >> (bit & 63) & 1) continue;
      for (auto & f : sc.foot) {
        const size_t b = (size_t)(gy + f.second) * g.width + (gx + f.first);
        if (sc.bits[b >> 6] == 0) sc.touched.push_back((uint32_t)(b >> 6));
        sc.bits[b >> 6] |= 1ull << (b & 63);
      }
      cells[w++] = cells[k];
    }
    cells.resize(w);
    for (uint32_t t : sc.touched) sc.bits[t] = 0;
    sc.touched.clear();
  }
}

void set_grid_offset(GridGeom & g, const b200_scan * query)   // M.cpp:560-569
{
  double res = 1.0 / g.scale;
  g.off_x = query->sensor_pose[0] - (0.5 * (g.roi_w - 1) * res);
  g.off_y = query->sensor_pose[1] - (0.5 * (g.roi_h - 1) * res);
}

// One CorrelateScan pass prepared on the host: GridIndexLookup::ComputeOffsets (K.h:6797-6894),
// the x / y / angle pose arrays (M.cpp:736-756, 641-668) and the search-space-probability cell map.
int build_plan(const GridGeom & g, int probs_side, const b200sm_params & prm, const b200_scan * q,
               const double center[3], const double sp_off[2], const double sp_res[2], double ang_off,
               double ang_res, bool fine, CorrPlan & pl)
{
  pl.fine = fine;
  for (int i = 0; i < 3; ++i) pl.center[i] = center[i];
  pl.sp_off[0] = sp_off[0]; pl.sp_off[1] = sp_off[1];
  pl.sp_res[0] = sp_res[0]; pl.sp_res[1] = sp_res[1];
  pl.ang_off = ang_off; pl.ang_res = ang_res;
  pl.n = q->n;
  pl.nA = (int)((uint32_t)(round_half_away(ang_off * 2.0 / ang_res) + 1));
  pl.nX = (int)((uint32_t)(round_half_away(sp_off[0] * 2.0 / sp_res[0]) + 1));
  pl.nY = (int)((uint32_t)(round_half_away(sp_off[1] * 2.0 / sp_res[1]) + 1));
  if (pl.nA <= 0 || pl.nX <= 0 || pl.nY <= 0 || (int64_t)pl.nA * pl.nX * pl.nY > (1 << 26)) {
    set_last_error("search space dimensions out of range");
    return B200_ERR_INVALID_ARG;
  }
  const int n = pl.n;
  // ---- lookup table ----
  pl.offsets.assign((size_t)pl.nA * n, kInvalidScan);
  pl.ogx.assign((size_t)pl.nA * n, 0);
  pl.ogy.assign((size_t)pl.nA * n, 0);
  double m00, m01, m02, m10, m11, m12, tx, ty, th;
  const double * sp = q->sensor_pose;
  if (sp[0] == 0.0 && sp[1] == 0.0 && sp[2] == 0.0) {   // Transform::SetTransform, K.h:3004-3009
    m00 = 1; m01 = 0; m02 = 0; m10 = 0; m11 = 1; m12 = 0; tx = 0; ty = 0; th = 0;
  } else {   // Matrix3::FromAxisAngle(0,0,1, 0 - heading), K.h:2482-2511 / 3013
    double radians = 0.0 - sp[2];
    double c = cos(radians), s = sin(radians), omc = 1.0 - c;
    double x = 0, y = 0, z = 1;
    double xyM = x * y * omc, xzM = x * z * omc, yzM = y * z * omc;
    double xS = x * s, yS = y * s, zS = z * s;
    m00 = x * x * omc + c; m01 = xyM - zS; m02 = xzM + yS;
    m10 = xyM + zS; m11 = y * y * omc + c; m12 = yzM - xS;
    tx = sp[0]; ty = sp[1]; th = sp[2] - 0.0;
  }
  std::vector<double> local((size_t)2 * (n > 0 ? n : 1));
  for (int i = 0; i < n; ++i) {   // Transform::InverseTransformPose(Pose2(point, 0)), K.h:2987-2994
    double dx = q->points_xy[2 * i] - tx, dy = q->points_xy[2 * i + 1] - ty, dh = 0.0 - th;
    local[2 * i] = m00 * dx + m01 * dy + m02 * dh;
    local[2 * i + 1] = m10 * dx + m11 * dy + m12 * dh;
  }
  pl.angle.resize(pl.nA); pl.heading.resize(pl.nA); pl.angpen.resize(pl.nA);
  double startAngle = center[2] - ang_off;
  auto one_angle = [&](int a) {
    double angle = startAngle + (uint32_t)a * ang_res;
    pl.angle[a] = angle;
    pl.heading[a] = normalize_angle(angle);
    pl.angpen[a] = angle_penalty(angle, center[2], prm.angle_variance_penalty, prm.minimum_angle_penalty);
    double cosine = cos(angle), sine = sin(angle);
    int32_t * out = pl.offsets.data() + (size_t)a * n;
    for (int i = 0; i < n; ++i) {
      double r = q->ranges[i];
      if (std::isnan(r) || std::isinf(r)) { out[i] = kInvalidScan; continue; }
      double ox = cosine * local[2 * i] - sine * local[2 * i + 1];
      double oy = sine * local[2 * i] + cosine * local[2 * i + 1];
      int gx = world_to_grid(ox + g.off_x, g.off_x, g.scale);   // WorldToGrid(offset + rGridOffset), K.h:6884
      int gy = world_to_grid(oy + g.off_y, g.off_y, g.scale);
      // Grid<T>::GridIndex(gridPoint, false) in 32-bit arithmetic like the reference (K.h:4692)
      out[i] = (int32_t)((uint32_t)gx + (uint32_t)gy * (uint32_t)g.stride);
      pl.ogx[(size_t)a * n + i] = gx;
      pl.ogy[(size_t)a * n + i] = gy;
    }
  };
  if ((size_t)pl.nA * n >= 4096) host_parallel_for(pl.nA, one_angle);   // one angle = one task (disjoint rows of the tables)
  else for (int a = 0; a < pl.nA; ++a) one_angle(a);
  // ---- pose arrays ----
  pl.xrel.resize(pl.nX); pl.newx.resize(pl.nX); pl.sqx.resize(pl.nX); pl.xs.resize(pl.nX); pl.px.resize(pl.nX);
  pl.yrel.resize(pl.nY); pl.newy.resize(pl.nY); pl.sqy.resize(pl.nY); pl.ys.resize(pl.nY); pl.py.resize(pl.nY);
  double startX = -sp_off[0], startY = -sp_off[1];
  double probs_off_x = center[0] - sp_off[0], probs_off_y = center[1] - sp_off[1];   // M.cpp:730
  for (int k = 0; k < pl.nX; ++k) {
    double x = startX + (uint32_t)k * sp_res[0];
    pl.xrel[k] = x; pl.newx[k] = center[0] + x; pl.sqx[k] = square(x);
    int gx = world_to_grid(pl.newx[k], g.off_x, g.scale);
    if (!is_up_to(gx + g.roi_x, g.width)) { set_last_error("search position outside the correlation grid (Karto.h:4684)"); return B200_ERR_INVALID_ARG; }
    pl.xs[k] = gx + g.roi_x;
    pl.px[k] = world_to_grid(pl.newx[k], probs_off_x, g.scale);
  }
  for (int k = 0; k < pl.nY; ++k) {
    double y = startY + (uint32_t)k * sp_res[1];
    pl.yrel[k] = y; pl.newy[k] = center[1] + y; pl.sqy[k] = square(y);
    int gy = world_to_grid(pl.newy[k], g.off_y, g.scale);
    if (!is_up_to(gy + g.roi_y, g.height)) { set_last_error("search position outside the correlation grid (Karto.h:4684)"); return B200_ERR_INVALID_ARG; }
    pl.ys[k] = gy + g.roi_y;
    pl.py[k] = world_to_grid(pl.newy[k], probs_off_y, g.scale);
  }
  if (!fine) {
    // the device reduction indexes m_pSearchSpaceProbs by (xIndex, yIndex); that equals the
    // reference's WorldToGrid cell map (M.cpp:783, 920-923) iff the map is injective and in range
    for (int k = 0; k < pl.nX; ++k)
      if (!is_up_to(pl.px[k], probs_side) || (k > 0 && pl.px[k] <= pl.px[k - 1])) {
        set_last_error("search-space probability grid cell map is not monotonic (Mapper.cpp:783-796 would alias or throw)");
        return B200_ERR_UNSUPPORTED;
      }
    for (int k = 0; k < pl.nY; ++k)
      if (!is_up_to(pl.py[k], probs_side) || (k > 0 && pl.py[k] <= pl.py[k - 1])) {
        set_last_error("search-space probability grid cell map is not monotonic (Mapper.cpp:783-796 would alias or throw)");
        return B200_ERR_UNSUPPORTED;
      }
  }
  return B200_OK;
}

// device form of a lookup entry: anything that can never index [0, data_size) for a position
// inside the grid becomes a sentinel that fails the unsigned range test without overflowing.
int32_t device_offset(int32_t off, int data_size)
{
  if (off == kInvalidScan || off <= -data_size || off >= data_size) return kDevInvalid;
  return off;
}

// ScanMatcher::CorrelateScan's reduction (M.cpp:775-862) + both covariance routines, in FP64 on the
// host, from the device's integer volume. sums index = (y*nX + x)*nA + a.
double host_epilogue(const b200sm_params & prm, const GridGeom & geom, int probs_side, const CorrPlan & pl,
                     const int32_t * sums, bool do_penalize, double mean[3], double cov[9],
                     const std::function<bool(int, int, int32_t *)> * extra_cell)
{
  const int nX = pl.nX, nY = pl.nY, nA = pl.nA;
  const size_t total = (size_t)nX * nY * nA;
  static thread_local std::vector<double> resp_scratch, probs_scratch;
  std::vector<double> & resp = resp_scratch;
  resp.resize(total);
  const double norm = (double)((uint32_t)pl.n * (uint32_t)kOccupied);
  const int side = probs_side;
  std::vector<double> & probs = probs_scratch;
  if (!pl.fine) probs.assign((size_t)side * side, 0.0);
  // responses (M.cpp:670-685), the per-cell maximum image (M.cpp:781-799) and the best response, one search row per task.
  // The distance penalty depends on (x, y) only: evaluated once per cell with the reference's expression -- same value.
  std::vector<double> row_best((size_t)nY, -1.0);
  auto one_row = [&](int y) {
    double rb = -1;
    for (int x = 0; x < nX; ++x) {
      const double dp = do_penalize ? distance_penalty(pl.sqx[x], pl.sqy[y], prm.distance_variance_penalty, prm.minimum_distance_penalty) : 0.0;
      double * cell = pl.fine ? nullptr : &probs[(size_t)pl.py[y] * side + pl.px[x]];
      for (int a = 0; a < nA; ++a) {
        const size_t k = ((size_t)y * nX + x) * nA + a;
        double r = 0.0;
        if (pl.n != 0) { r = (double)sums[k]; r /= norm; }
        if (do_penalize && !double_equal(r, 0.0)) r *= (dp * pl.angpen[a]);
        resp[k] = r;
        rb = maximum(rb, r);
        if (cell) *cell = maximum(r, *cell);
      }
    }
    row_best[y] = rb;
  };
  if (total >= 4096) host_parallel_for(nY, one_row); else for (int y = 0; y < nY; ++y) one_row(y);
  double best = -1;
  for (int y = 0; y < nY; ++y) best = maximum(best, row_best[y]);
  double ax = 0.0, ay = 0.0, thetaX = 0.0, thetaY = 0.0;
  int count = 0;
  for (size_t k = 0; k < total; ++k) {
    if (double_equal(resp[k], best)) {
      size_t xy = k / nA;
      ax += pl.newx[xy % nX]; ay += pl.newy[xy / nX];
      double heading = pl.heading[k % nA];
      thetaX += cos(heading); thetaY += sin(heading);
      count++;
    }
  }
  double avg[3] = {0, 0, 0};
  if (count > 0) {
    ax /= count; ay /= count; thetaX /= count; thetaY /= count;
    avg[0] = ax; avg[1] = ay; avg[2] = atan2(thetaY, thetaX);
  }
  if (!pl.fine) {
    // ComputePositionalCovariance, M.cpp:874-966
    for (int i = 0; i < 9; ++i) cov[i] = 0.0;
    cov[0] = cov[4] = cov[8] = 1.0;
    if (best < kTolerance) {
      cov[0] = kMaxVariance; cov[4] = kMaxVariance; cov[8] = 4 * square(pl.ang_res);
    } else {
      double aXX = 0, aXY = 0, aYY = 0, nrm = 0;
      double dx = avg[0] - pl.center[0], dy = avg[1] - pl.center[1];
      for (int y = 0; y < nY; ++y)
        for (int x = 0; x < nX; ++x) {
          double response = probs[(size_t)pl.py[y] * side + pl.px[x]];
          if (response >= (best - 0.1)) {
            nrm += response;
            aXX += (square(pl.xrel[x] - dx) * response);
            aXY += ((pl.xrel[x] - dx) * (pl.yrel[y] - dy) * response);
            aYY += (square(pl.yrel[y] - dy) * response);
          }
        }
      finish_positional_cov(nrm, aXX, aXY, aYY, best, pl.sp_res, pl.ang_res, cov);
    }
  } else {
    // ComputeAngularCovariance, M.cpp:977-1025
    double bestAngle = normalize_angle_difference(avg[2], pl.center[2]);
    int gx = world_to_grid(avg[0], geom.off_x, geom.scale) + geom.roi_x;
    int gy = world_to_grid(avg[1], geom.off_y, geom.scale) + geom.roi_y;
    int xi = -1, yi = -1;
    for (int x = 0; x < nX; ++x) if (pl.xs[x] == gx) xi = x;
    for (int y = 0; y < nY; ++y) if (pl.ys[y] == gy) yi = y;
    double nrm = 0.0, acc = 0.0;
    // the averaged best pose normally rounds to one of the searched cells; when the search centre sits on a half-cell boundary
    // it can round to a cell in between (the reference calls GetResponse on whatever cell WorldToGrid gives, M.cpp:1003-1011):
    // its nA sums are then computed on demand against the resident raster
    std::vector<int32_t> extra;
    const int32_t * col = nullptr;
    if (xi >= 0 && yi >= 0) {
      col = sums + ((size_t)yi * nX + xi) * nA;
    } else if (extra_cell) {
      extra.assign(nA, 0);
      if ((*extra_cell)(gx, gy, extra.data())) col = extra.data();
    }
    if (col) {
      for (int a = 0; a < nA; ++a) {
        double response = 0.0;
        if (pl.n != 0) { response = (double)col[a]; response /= norm; }
        if (response >= (best - 0.1)) {
          nrm += response;
          acc += (square(pl.angle[a] - bestAngle) * response);
        }
      }
    } else {
      set_last_error("fine-match best pose fell outside the searched cells");
      throw CudaFail{B200_ERR_UNSUPPORTED};
    }
    if (nrm > kTolerance) {
      if (acc < kTolerance) acc = square(pl.ang_res);
      acc /= nrm;
    } else {
      acc = 1000 * square(pl.ang_res);
    }
    cov[8] = acc;
  }
  mean[0] = avg[0]; mean[1] = avg[1]; mean[2] = avg[2];
  if (best > 1.0) best = 1.0;
  return best;
}

// host-side phase timer of the single-match path (b200sm_match_timing): 0 cells (FindValidPoints + occupancy replay), 1 raster
// upload + stamp, 2 plan build (lookup tables), 3 volume (H2D, kernel, D2H, wait), 4 epilogue, 5 matches
struct PhaseTimer {
  b200sm * h; int slot; std::chrono::steady_clock::time_point t0;
  PhaseTimer(b200sm * hh, int s) : h(hh), slot(s), t0(std::chrono::steady_clock::now()) {}
  ~PhaseTimer() { h->phase_ms[slot] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

static void upload_raster(b200sm * h, const std::vector<int32_t> & cells)
{
  PhaseTimer pt(h, 1);
  const GridGeom & g = h->g;
  h->ensure_stream();
  h->d_grid.reserve((size_t)g.data_size + 16);
  if (h->d_kernel.cap == 0) {
    h->d_kernel.reserve(g.kernel.size());
    B200_CUDA(cudaMemcpyAsync(h->d_kernel.p, g.kernel.data(), g.kernel.size(), cudaMemcpyHostToDevice, h->stream));
  }
  B200_CUDA(cudaMemsetAsync(h->d_grid.p, 0, (size_t)g.data_size, h->stream));   // Grid::Clear
  if (!cells.empty()) {
    h->d_cells.reserve(cells.size());
    h->h_stage_i.reserve(cells.size());
    std::memcpy(h->h_stage_i.p, cells.data(), cells.size() * sizeof(int32_t));
    B200_CUDA(cudaMemcpyAsync(h->d_cells.p, h->h_stage_i.p, cells.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    long long total = (long long)cells.size() * g.ksize;
    int blocks = (int)std::min<long long>((total + 255) / 256, 132 * 16);
    k_stamp<<<blocks, 256, 0, h->stream>>>(h->d_grid.p, g.stride, g.roi_x, g.roi_y, h->d_cells.p, (int)cells.size(),
                                          h->d_kernel.p, g.ksize);
    B200_CUDA(cudaGetLastError());
    h->launches++;
    // the staging buffer is reused by the next call
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  h->have_raster = true;
}

// integer volume of one plan against the current device grid -> host (pinned) buffer
static const int32_t * device_volume(b200sm * h, const CorrPlan & pl)
{
  const GridGeom & g = h->g;
  const int P = pl.nX * pl.nY;
  const size_t total = (size_t)P * pl.nA;
  h->ensure_stream();
  h->h_sums.reserve(total);
  if (pl.n == 0) { std::memset(h->h_sums.p, 0, total * sizeof(int32_t)); return h->h_sums.p; }
  if ((size_t)pl.n * sizeof(int32_t) > 200 * 1024) {
    set_last_error("scan has too many readings for the shared-memory lookup row");
    throw CudaFail{B200_ERR_UNSUPPORTED};
  }
  const size_t noff = (size_t)pl.nA * pl.n;
  h->h_stage_i.reserve(noff + P);
  for (size_t i = 0; i < noff; ++i) h->h_stage_i.p[i] = device_offset(pl.offsets[i], g.data_size);
  for (int y = 0; y < pl.nY; ++y)
    for (int x = 0; x < pl.nX; ++x) h->h_stage_i.p[noff + (size_t)y * pl.nX + x] = pl.xs[x] + pl.ys[y] * g.stride;
  h->d_offsets.reserve(noff + P);
  h->d_sums.reserve(total);
  B200_CUDA(cudaMemcpyAsync(h->d_offsets.p, h->h_stage_i.p, (noff + P) * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  if (P * pl.nA <= 2048) {
    const int items = P * pl.nA;
    k_correlate_few<<<(items + 7) / 8, 256, 0, h->stream>>>(h->d_grid.p, g.data_size, h->d_offsets.p, h->d_offsets.p + noff, P, pl.nA,
                                                           pl.n, h->d_sums.p);
  } else {
    dim3 grid((P + 31) / 32, std::min(pl.nA, kMaxGridY));
    size_t smem = (size_t)pl.n * sizeof(int32_t);
    if (smem > 40 * 1024) B200_CUDA(cudaFuncSetAttribute(k_correlate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_correlate<<<grid, 32 * kCorrWarps, smem, h->stream>>>(h->d_grid.p, g.data_size, h->d_offsets.p, h->d_offsets.p + noff, P,
                                                           pl.nA, pl.n, h->d_sums.p);
  }
  B200_CUDA(cudaGetLastError());
  h->launches++;
  B200_CUDA(cudaMemcpyAsync(h->h_sums.p, h->d_sums.p, total * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return h->h_sums.p;
}

static double correlate(b200sm * h, const b200_scan * q, const double center[3], const double sp_off[2],
                        const double sp_res[2], double ang_off, double ang_res, bool do_penalize, bool fine,
                        double mean[3], double cov[9], int32_t * sums_out, int32_t sums_cap, int32_t dims[3])
{
  CorrPlan pl;
  int rc;
  { PhaseTimer pt(h, 2); rc = build_plan(h->g, h->probs_side, h->p, q, center, sp_off, sp_res, ang_off, ang_res, fine, pl); }
  if (rc != B200_OK) throw CudaFail{rc};
  const int32_t * sums;
  { PhaseTimer pt(h, 3); sums = device_volume(h, pl); }
  if (dims) { dims[0] = pl.nX; dims[1] = pl.nY; dims[2] = pl.nA; }
  if (sums_out) {
    size_t total = (size_t)pl.nX * pl.nY * pl.nA;
    std::memcpy(sums_out, sums, std::min<size_t>(total, (size_t)std::max(0, sums_cap)) * sizeof(int32_t));
  }
  PhaseTimer pt(h, 4);
  const std::function<bool(int, int, int32_t *)> extra = [&](int gx, int gy, int32_t * out) {
    // one more pose against the raster and lookup table that are still on the device
    if (!is_up_to(gx, h->g.width) || !is_up_to(gy, h->g.height) || pl.n == 0) return false;
    const size_t noff = (size_t)pl.nA * pl.n;
    const int32_t posv = gx + gy * h->g.stride;
    h->d_extra.reserve((size_t)pl.nA + 1);
    B200_CUDA(cudaMemcpyAsync(h->d_extra.p + pl.nA, &posv, sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    k_correlate_few<<<(pl.nA + 7) / 8, 256, 0, h->stream>>>(h->d_grid.p, h->g.data_size, h->d_offsets.p, h->d_extra.p + pl.nA, 1, pl.nA, pl.n,
                                                           h->d_extra.p);
    B200_CUDA(cudaGetLastError());
    h->launches++;
    (void)noff;
    B200_CUDA(cudaMemcpyAsync(out, h->d_extra.p, (size_t)pl.nA * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
    return true;
  };
  return host_epilogue(h->p, h->g, h->probs_side, pl, sums, do_penalize, mean, cov, &extra);
}

static void check_scan(const b200_scan * s, bool need_ranges)
{
  if (!s || s->n < 0 || (s->n > 0 && (!s->points_xy || (need_ranges && !s->ranges)))) {
    set_last_error("b200_scan: NULL pointer or negative size");
    throw CudaFail{B200_ERR_INVALID_ARG};
  }
}

static void do_raster(b200sm * h, const b200_scan * query, const b200_scan * base, int nbase)
{
  set_grid_offset(h->g, query);
  std::vector<int32_t> cells;
  { PhaseTimer pt(h, 0); host_cells(h->g, h->cell_scratch, query, base, nbase, cells); }
  upload_raster(h, cells);
}

double do_match(b200sm * h, const b200_scan * query, const b200_scan * base, int nbase, bool pen, bool refine,
                       double mean[3], double cov[9])
{
  NvtxRange nvtx_("b200sm match");
  h->phase_ms[5] += 1.0;
  for (int i = 0; i < 9; ++i) cov[i] = 0.0;
  if (query->n == 0) {   // M.cpp:547-557
    mean[0] = query->sensor_pose[0]; mean[1] = query->sensor_pose[1]; mean[2] = query->sensor_pose[2];
    cov[0] = kMaxVariance; cov[4] = kMaxVariance; cov[8] = 4 * square(h->p.coarse_angle_resolution);
    return 0.0;
  }
  do_raster(h, query, base, nbase);
  double res = 1.0 / h->g.scale;
  double dim = (double)h->probs_side;
  double coarseOff[2] = {0.5 * (dim - 1) * res, 0.5 * (dim - 1) * res};
  double coarseRes[2] = {2 * res, 2 * res};
  double center[3] = {query->sensor_pose[0], query->sensor_pose[1], query->sensor_pose[2]};
  double best = correlate(h, query, center, coarseOff, coarseRes, h->p.coarse_search_angle_offset,
                          h->p.coarse_angle_resolution, pen, false, mean, cov, nullptr, 0, nullptr);
  if (h->p.use_response_expansion) {   // M.cpp:594-619
    if (double_equal(best, 0.0)) {
      double newOff = h->p.coarse_search_angle_offset;
      for (uint32_t i = 0; i < 3; i++) {
        newOff += 20 * kPi180;
        best = correlate(h, query, center, coarseOff, coarseRes, newOff, h->p.coarse_angle_resolution, pen, false,
                         mean, cov, nullptr, 0, nullptr);
        if (!double_equal(best, 0.0)) break;
      }
    }
  }
  if (refine) {   // M.cpp:621-629
    double fineOff[2] = {coarseRes[0] * 0.5, coarseRes[1] * 0.5};
    double fineRes[2] = {res, res};
    double c2[3] = {mean[0], mean[1], mean[2]};
    best = correlate(h, query, c2, fineOff, fineRes, 0.5 * h->p.coarse_angle_resolution, h->p.fine_search_angle_offset,
                     pen, true, mean, cov, nullptr, 0, nullptr);
  }
  return best;
}

}  // namespace b200

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

const char * b200_last_error(void) { return g_last_error.c_str(); }

int b200_set_device(int ordinal)
{
  B200_GUARD_BEGIN
  require_device();
  B200_CUDA(cudaSetDevice(ordinal));
  return B200_OK;
  B200_GUARD_END
}

int b200_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int b200_point_readings(const double * ranges, int32_t n, const double sensor_pose[3], double minimum_angle,
                        double angular_resolution, double * out_xy)
{
  if (!ranges || !sensor_pose || !out_xy || n < 0) return B200_ERR_INVALID_ARG;
  for (int32_t i = 0; i < n; ++i) {   // Karto.h:5660-5683 (both branches compute the same point)
    double angle = sensor_pose[2] + minimum_angle + (uint32_t)i * angular_resolution;
    out_xy[2 * i] = sensor_pose[0] + (ranges[i] * cos(angle));
    out_xy[2 * i + 1] = sensor_pose[1] + (ranges[i] * sin(angle));
  }
  return B200_OK;
}

int b200sm_create(const b200sm_params * params, b200sm ** out)
{
  B200_GUARD_BEGIN
  if (!params || !out) { set_last_error("b200sm_create: NULL argument"); return B200_ERR_INVALID_ARG; }
  *out = nullptr;
  std::unique_ptr<b200sm> h(new b200sm());
  h->p = *params;
  int rc = build_geometry(h->p, h->g, h->probs_side);
  if (rc != B200_OK) return rc;
  require_device();
  h->ensure_stream();
  *out = h.release();
  return B200_OK;
  B200_GUARD_END
}

void b200sm_destroy(b200sm * h)
{
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  h->sweep.release();
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

int b200sm_set_stream(b200sm * h, void * s)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  if (h->stream) B200_CUDA(cudaStreamSynchronize(h->stream));
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  h->stream = static_cast<cudaStream_t>(s);
  h->own_stream = false;
  if (!h->stream) h->ensure_stream();
  return B200_OK;
  B200_GUARD_END
}

int b200sm_match(b200sm * h, const b200_scan * query, const b200_scan * base, int32_t nbase, int32_t do_penalize,
                 int32_t do_refine, double mean[3], double cov[9], double * response)
{
  B200_GUARD_BEGIN
  if (!h || !mean || !cov || !response || nbase < 0 || (nbase > 0 && !base)) { set_last_error("b200sm_match: bad argument"); return B200_ERR_INVALID_ARG; }
  check_scan(query, true);
  for (int i = 0; i < nbase; ++i) check_scan(&base[i], false);
  *response = do_match(h, query, base, nbase, do_penalize != 0, do_refine != 0, mean, cov);
  return B200_OK;
  B200_GUARD_END
}

int b200sm_raster(b200sm * h, const b200_scan * query, const b200_scan * base, int32_t nbase)
{
  B200_GUARD_BEGIN
  if (!h || nbase < 0 || (nbase > 0 && !base)) return B200_ERR_INVALID_ARG;
  check_scan(query, false);
  for (int i = 0; i < nbase; ++i) check_scan(&base[i], false);
  do_raster(h, query, base, nbase);
  return B200_OK;
  B200_GUARD_END
}

int b200sm_correlate(b200sm * h, const b200_scan * query, const double center[3], const double sp_off[2],
                     const double sp_res[2], double ang_off, double ang_res, int32_t do_penalize, int32_t fine,
                     double mean[3], double cov[9], double * response, int32_t * sums, int32_t sums_cap, int32_t dims[3])
{
  B200_GUARD_BEGIN
  if (!h || !center || !sp_off || !sp_res || !mean || !cov || !response) return B200_ERR_INVALID_ARG;
  if (!h->have_raster) { set_last_error("b200sm_correlate: no raster yet"); return B200_ERR_INVALID_ARG; }
  if (!(ang_res != 0.0) || !(sp_res[0] > 0) || !(sp_res[1] > 0)) { set_last_error("b200sm_correlate: zero resolution"); return B200_ERR_INVALID_ARG; }
  check_scan(query, true);
  *response = correlate(h, query, center, sp_off, sp_res, ang_off, ang_res, do_penalize != 0, fine != 0, mean, cov, sums,
                        sums_cap, dims);
  return B200_OK;
  B200_GUARD_END
}

int b200sm_grid_info(b200sm * h, int32_t info[9], double offset[2])
{
  if (!h || !info || !offset) return B200_ERR_INVALID_ARG;
  const GridGeom & g = h->g;
  info[0] = g.width; info[1] = g.height; info[2] = g.stride; info[3] = g.roi_x; info[4] = g.roi_y;
  info[5] = g.roi_w; info[6] = g.roi_h; info[7] = g.data_size; info[8] = g.ksize;
  offset[0] = g.off_x; offset[1] = g.off_y;
  return B200_OK;
}

int b200sm_grid_copy(b200sm * h, uint8_t * out, int32_t cap)
{
  B200_GUARD_BEGIN
  if (!h || !out || cap < h->g.data_size) return B200_ERR_INVALID_ARG;
  if (!h->have_raster) { set_last_error("b200sm_grid_copy: no raster yet"); return B200_ERR_INVALID_ARG; }
  B200_CUDA(cudaMemcpyAsync(out, h->d_grid.p, (size_t)h->g.data_size, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
  B200_GUARD_END
}

int64_t b200sm_launch_count(const b200sm * h) { return h ? h->launches : 0; }

void b200_parallel_for(int32_t n, void (*fn)(int32_t, void *), void * ctx)
{
  if (!fn || n <= 0) return;
  host_parallel_for(n, [&](int i) { fn(i, ctx); });
}
int32_t b200_host_threads(void) { return host_pool_threads(); }

int b200sm_match_timing(b200sm * h, double out[6], int32_t reset)
{
  if (!h || !out) return B200_ERR_INVALID_ARG;
  for (int i = 0; i < 6; ++i) out[i] = h->phase_ms[i];
  if (reset) for (int i = 0; i < 6; ++i) h->phase_ms[i] = 0.0;
  return B200_OK;
}

int b200sm_set_option(b200sm * h, const char * name, int32_t value)
{
  if (!h || !name) return B200_ERR_INVALID_ARG;
  if (std::string(name) == "force_generic_sweep") { h->force_generic = value != 0; return B200_OK; }
  if (std::string(name) == "no_beam_dedup") { h->no_dedup = value != 0; return B200_OK; }
  if (std::string(name) == "sweep_kernel") { h->sweep_kernel = value; return B200_OK; }
  if (std::string(name) == "sweep_cluster") { h->tile_cluster = value; return B200_OK; }
  if (std::string(name) == "sweep_chunks") { h->tile_chunks = value; return B200_OK; }
  set_last_error(std::string("unknown option ") + name);
  return B200_ERR_INVALID_ARG;
}

}  // extern "C"
