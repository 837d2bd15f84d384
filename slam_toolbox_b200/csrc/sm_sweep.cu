// b200slam scan matcher, batched loop-closure sweep (generic path).
//
// Reference: MapperGraph::TryCloseLoop (lib/karto_sdk/src/Mapper.cpp:1500-1561) calls
// ScanMatcher::MatchScan once per candidate chain; here every (query, chain) pair of a sweep is
// rasterised, correlated and reduced on the device in one fused kernel launch.
//   k_find_valid     FindValidPoints + WorldToGrid + ROI test per (pair, scan)  (M.cpp:1073-1164)
//   k_sweep_generic  per pair: clear + smear raster, exhaustive correlation, arg-max / ties /
//                    positional-covariance accumulators                          (M.cpp:641-966)
//   k_sweep_fine     3x3xnA fine volumes for do_refine                           (M.cpp:621-629)
// Compile with -fmad=false / -ffp-contract=off (bit-exact FP64, see sm_math.cuh).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "sm_math.cuh"
#include "sm_types.cuh"
#include "sm_device.cuh"
#include "sm_sweep_dev.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------
// batch sweep, generic path
// ------------------------------------------------------------------------------------------

// ScanMatcher::FindValidPoints (M.cpp:1113-1164) + WorldToGrid + ROI test (M.cpp:1082-1088) for
// every (pair, scan of its chain).  One WARP per scan, the scan's points staged in shared memory.
// The reference walks the points one by one, but its state only changes at an ANCHOR: the first point
// farther than 10 cm from the previous anchor (M.cpp:1138-1139).  So the warp tests 32 points against
// the current anchor at once (the reference's own expression, evaluated per lane), a ballot finds the
// next anchor, and the side test + range bookkeeping (M.cpp:1145-1160) run once per anchor instead of
// once per point: ~4x fewer dependent steps at indoor point spacings.  Accepted index ranges set flags
// in shared memory; a second, parallel pass turns accepted points into grid cells and compacts the
// in-ROI ones in scan order.  cells[item * max_n + k] = gx | gy << 16 of the k-th point inside the ROI.
constexpr int kFvWarps = 4;
constexpr int kFvBytesPerPoint = 17;   // double2 + flag
__global__ void __launch_bounds__(kFvWarps * 32) k_find_valid(SweepDev d)
{
  extern __shared__ __align__(16) unsigned char s_fv[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int item = blockIdx.x * nw + warp;
  if (item >= d.nitems) return;
  double2 * P = reinterpret_cast<double2 *>(s_fv) + (size_t)warp * d.max_n;
  unsigned char * valid = s_fv + (size_t)nw * d.max_n * sizeof(double2) + (size_t)warp * d.max_n;
  const int pair = d.item_pair[item];
  const int scan = d.item_scan[item];
  const int q = d.pair_query[pair];
  const double vx = d.qgeom[q * 4 + 0], vy = d.qgeom[q * 4 + 1];
  const double ox = d.qgeom[q * 4 + 2], oy = d.qgeom[q * 4 + 3];
  const double2 * pts = reinterpret_cast<const double2 *>(d.points) + (size_t)d.scan_pt_start[scan];
  const int n = d.scan_pt_start[scan + 1] - d.scan_pt_start[scan];
  for (int i = lane; i < n; i += 32) { P[i] = pts[i]; valid[i] = 0; }
  __syncwarp();
  // the first point without a NaN coordinate becomes the first anchor (M.cpp:1130-1133); until then
  // firstPoint is (0, 0) and every distance test sees a NaN: nothing happens
  int i = n;
  for (int base = 0; base < n; base += 32) {
    const int t = base + lane;
    bool ok = false;
    if (t < n) { const double2 c = P[t]; ok = !(c.x != c.x) && !(c.y != c.y); }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (m) { i = base + __ffs(m) - 1; break; }
  }
  if (i < n) {
    double fx = P[i].x, fy = P[i].y;
    int trailing = 0;
    ++i;   // the anchor itself is at distance 0 (or NaN for an infinite point): no event
    while (i < n) {
      const int t = i + lane;
      bool far = false;
      if (t < n) {
        const double2 c = P[t];
        const double dx = fx - c.x, dy = fy - c.y;
        far = dx * dx + dy * dy > 0.1 * 0.1;                  // delta.SquaredLength() > minSquareDistance
      }
      const unsigned m = __ballot_sync(0xffffffffu, far);
      if (!m) { i += 32; continue; }
      const int idx = i + __ffs(m) - 1;
      const double2 c = P[idx];
      const double a = vy - fy;
      const double b = fx - vx;
      const double cc = fy * vx - fx * vy;
      const double ss = c.x * a + c.y * b + cc;
      fx = c.x; fy = c.y;
      if (!(ss < 0.0)) {
        for (int k = trailing + lane; k < idx; k += 32) valid[k] = 1;
      }
      trailing = idx;
      i = idx + 1;
    }
  }
  __syncwarp();
  int32_t * out = d.cells + (size_t)item * d.max_n;
  int total = 0;
  for (int base = 0; base < n; base += 32) {
    const int t = base + lane;
    bool keep = false;
    int cell = 0;
    if (t < n && valid[t]) {
      const int gx = world_to_grid(P[t].x, ox, d.scale);
      const int gy = world_to_grid(P[t].y, oy, d.scale);
      keep = is_up_to(gx, d.roi_w) && is_up_to(gy, d.roi_h);
      cell = gx | (gy << 16);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) out[total + __popc(m & ((1u << lane) - 1))] = cell;
    total += __popc(m);
  }
  if (lane == 0) d.cell_count[item] = total;
}

// The on-device part of CorrelateScan's reduction (M.cpp:775-829) and of
// ComputePositionalCovariance (M.cpp:893-933) for one pair whose integer volume is in `sums`
// (index (y*nX+x)*nA + a).  `probs` = P doubles of scratch.  Everything that needs libm
// (heading average) is finished on the host from the tie list.
struct SumsPoseMajor {   // generic path: volume index (y*nX + x)*nA + a in global memory
  const int32_t * v; int nA;
  __device__ __forceinline__ int operator()(int p, int a) const { return v[(size_t)p * nA + a]; }
};
struct SumsAngleMajor {  // fast path: accumulators [a][y*nX + x] in shared memory
  const int32_t * v; int P;
  __device__ __forceinline__ int operator()(int p, int a) const { return v[a * P + p]; }
};

template <class SumAt>
__device__ void pair_epilogue(const SweepDev & d, int pair, int q, const SumAt sums,
                              double * probs, double * s_dscratch, int * s_iscratch)
{
  const int P = d.nX * d.nY, nA = d.nA;
  PairOut & out = d.out[pair];
  // best response + per-cell max over angles (the m_pSearchSpaceProbs image, M.cpp:781-799)
  double lbest = -1.0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int x = p % d.nX, y = p / d.nX;
    double pm = 0.0;   // Grid<double>::Clear() initial value, M.cpp:727
    for (int a = 0; a < nA; ++a) {
      int s = sums(p, a);
      double r = pose_response(d, q, s, x, y, a);
      pm = r > pm ? r : pm;
      lbest = r > lbest ? r : lbest;
    }
    probs[p] = pm;
  }
  const double best = block_max(lbest, s_dscratch);

  // ordered tie list: poses with DoubleEqual(response, best) in array order (M.cpp:807-817)
  // each thread owns a contiguous run of cells so that ranks follow array order
  const int per = (P + blockDim.x - 1) / blockDim.x;
  const int p0 = min(P, (int)threadIdx.x * per), p1 = min(P, p0 + per);
  int cnt = 0;
  for (int p = p0; p < p1; ++p) {
    const int x = p % d.nX, y = p / d.nX;
    for (int a = 0; a < nA; ++a)
      if (double_equal(pose_response(d, q, sums(p, a), x, y, a), best)) ++cnt;
  }
  int total = 0;
  int rank = block_exclusive_scan(cnt, s_iscratch, total);
  for (int p = p0; p < p1 && rank < kMaxTies; ++p) {
    const int x = p % d.nX, y = p / d.nX;
    for (int a = 0; a < nA && rank < kMaxTies; ++a)
      if (double_equal(pose_response(d, q, sums(p, a), x, y, a), best)) {
        out.ties[rank++] = p * nA + a;
      }
  }
  __syncthreads();
  __shared__ double s_avg[2];
  if (threadIdx.x == 0) {
    out.best = best;
    out.best_sum = total > 0 ? sums(out.ties[0] / nA, out.ties[0] % nA) : 0;
    out.tie_count = total;
    double ax = 0.0, ay = 0.0;
    const int m = total < kMaxTies ? total : kMaxTies;
    for (int t = 0; t < m; ++t) {   // averagePosition += pose position, in order (M.cpp:809)
      int p = out.ties[t] / nA;
      ax += d.newx[q * d.nX + p % d.nX];
      ay += d.newy[q * d.nY + p / d.nX];
    }
    if (total > 0) { ax /= total; ay /= total; }
    s_avg[0] = ax; s_avg[1] = ay;
    out.avg_x = ax; out.avg_y = ay;
  }
  __syncthreads();
  // positional covariance accumulators (M.cpp:893-933): cells with response >= best - 0.1,
  // summed in (y, x) order. Terms are formed in parallel, compacted in order, then added
  // sequentially so the additions happen in the reference's order.
  const double dx = s_avg[0] - d.center[q * 3 + 0], dy = s_avg[1] - d.center[q * 3 + 1];
  int c2 = 0;
  for (int p = p0; p < p1; ++p) if (probs[p] >= (best - 0.1)) ++c2;
  int tot2 = 0;
  int r2 = block_exclusive_scan(c2, s_iscratch, tot2);
  double * terms = probs + P;   // 4 * P doubles of scratch after the probs image
  for (int p = p0; p < p1; ++p) {
    double resp = probs[p];
    if (resp >= (best - 0.1)) {
      double x = d.xrel[q * d.nX + p % d.nX], y = d.yrel[q * d.nY + p / d.nX];
      terms[4 * r2 + 0] = resp;
      terms[4 * r2 + 1] = (square(x - dx) * resp);
      terms[4 * r2 + 2] = ((x - dx) * (y - dy) * resp);
      terms[4 * r2 + 3] = (square(y - dy) * resp);
      ++r2;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double norm = 0, axx = 0, axy = 0, ayy = 0;
    for (int t = 0; t < tot2; ++t) {
      norm += terms[4 * t + 0];
      axx += terms[4 * t + 1];
      axy += terms[4 * t + 2];
      ayy += terms[4 * t + 3];
    }
    out.norm = norm; out.acc_xx = axx; out.acc_xy = axy; out.acc_yy = ayy;
  }
  __syncthreads();
}

// Generic fused sweep kernel: one CTA walks pairs p = blockIdx.x, blockIdx.x + gridDim.x, ...
// For each pair: clear its workspace grid (Grid::Clear, M.cpp:1034), max-stamp the smear kernel
// of every valid point (AddScan, M.cpp:1080-1104), correlate all (x, y, theta) poses against it
// (M.cpp:641-694 + 1172-1208) and reduce (pair_epilogue).  The grid lives in a per-CTA global
// workspace (L2 resident) and is read through L1.
// The query's nA x n lookup table is read from shared memory in ANGLE SLICES of slice_rows whole rows
// (generic_slice_rows).  When the whole table fits (slice_rows >= nA) it is staged once per query and
// kept across that query's pairs; otherwise every pair stages slice after slice.  The volume is written
// at sums[p * nA + a] either way and integer sums do not depend on order, so the epilogue is the same.
__global__ void __launch_bounds__(kSweepThreads) k_sweep_generic(SweepDev d, int slice_rows)
{
  extern __shared__ __align__(16) unsigned char s_raw[];
  int32_t * s_off = reinterpret_cast<int32_t *>(s_raw);   // slice_rows x n lookup rows of this pair's query
  __shared__ double s_dscratch[32];
  __shared__ int s_iscratch[32];

  uint8_t * grid = d.ws_grid + (size_t)blockIdx.x * d.ws_grid_pitch;
  int32_t * sums = d.ws_sums + (size_t)blockIdx.x * d.ws_sums_pitch;
  double * probs = d.ws_probs + (size_t)blockIdx.x * d.ws_probs_pitch;
  const int P = d.nX * d.nY, nA = d.nA, n = d.n;
  const int half = d.ksize / 2, taps = d.ksize * d.ksize;
  const bool whole = slice_rows >= nA;
  int last_q = -1;

  for (int pair = blockIdx.x; pair < d.npairs; pair += gridDim.x) {
    const int q = d.pair_query[pair];
    // (1) clear
    {
      uint4 * g4 = reinterpret_cast<uint4 *>(grid);
      const int n16 = d.data_size / 16;
      for (int i = threadIdx.x; i < n16; i += blockDim.x) g4[i] = make_uint4(0, 0, 0, 0);
      for (int i = n16 * 16 + threadIdx.x; i < d.data_size; i += blockDim.x) grid[i] = 0;
    }
    if (whole && q != last_q) {
      for (int i = threadIdx.x; i < nA * n; i += blockDim.x) s_off[i] = d.offsets[(size_t)q * nA * n + i];
      last_q = q;
    }
    __syncthreads();
    // (2) raster
    const int it0 = d.pair_item_start[pair], it1 = d.pair_item_start[pair + 1];
    if (d.order_dependent) {
      // AddScan's "already 100" test (M.cpp:1093-1096) makes the raster depend on insertion order
      // when the smear kernel has 100s off-centre: replay that greedy rule sequentially, stamping
      // only the 100-valued taps, and drop the points the reference would skip.
      if (threadIdx.x == 0) {
        for (int it = it0; it < it1; ++it) {
          int32_t * cl = d.cells + (size_t)it * d.max_n;
          const int cn = d.cell_count[it];
          for (int k = 0; k < cn; ++k) {
            if (cl[k] < 0) continue;
            int gx = (cl[k] & 0xFFFF) + d.roi_x, gy = (cl[k] >> 16) + d.roi_y;
            if (grid[(size_t)gy * d.stride + gx] == kOccupied) { cl[k] = -1; continue; }
            for (int t = 0; t < taps; ++t)
              if (d.kern[t] == kOccupied)
                grid[(size_t)(gy + t / d.ksize - half) * d.stride + gx + t % d.ksize - half] = kOccupied;
          }
        }
      }
      __syncthreads();
    }
    for (int it = it0; it < it1; ++it) {
      const int32_t * cl = d.cells + (size_t)it * d.max_n;
      const int total = d.cell_count[it] * taps;
      for (int t = threadIdx.x; t < total; t += blockDim.x) {
        int32_t cell = cl[t / taps];
        if (cell < 0) continue;
        const int k = t % taps;
        uint32_t kv = d.kern[k];
        if (kv == 0) continue;
        int gx = (cell & 0xFFFF) + d.roi_x + (k % d.ksize) - half;
        int gy = (cell >> 16) + d.roi_y + (k / d.ksize) - half;
        atomic_max_u8(grid + (size_t)gy * d.stride + gx, kv);
      }
    }
    __syncthreads();
    // (3) correlate: items = (angle, pose), angle-major so a warp shares one lookup row; one slice of angles at a time
    const int32_t * pos = d.posidx + (size_t)q * P;
    for (int a0 = 0; a0 < nA; a0 += slice_rows) {
      const int na = min(slice_rows, nA - a0);
      if (!whole) {
        const int32_t * src = d.offsets + ((size_t)q * nA + a0) * n;
        for (int i = threadIdx.x; i < na * n; i += blockDim.x) s_off[i] = src[i];
        __syncthreads();
      }
      for (int item = threadIdx.x; item < na * P; item += blockDim.x) {
        const int al = item / P, p = item - al * P;
        const int base = pos[p];
        const int32_t * off = s_off + al * n;
        int acc = 0;
#pragma unroll 8
        for (int i = 0; i < n; ++i) {
          int idx = base + off[i];
          if ((unsigned)idx < (unsigned)d.data_size) acc += grid[idx];
        }
        sums[(size_t)p * nA + a0 + al] = acc;
      }
      __syncthreads();
    }
    // (4) reduce
    pair_epilogue(d, pair, q, SumsPoseMajor{sums, nA}, probs, s_dscratch, s_iscratch);
  }
}

// fine pass of the batch: 3x3xnA volume per pair, lookup table per pair (the search centre is
// the pair's coarse mean). Re-rasterises the pair's grid, writes only the integer volume; the
// (tiny) reduction incl. ComputeAngularCovariance runs on the host.
__global__ void __launch_bounds__(kSweepThreads) k_sweep_fine(SweepDev d, FineDev f)
{
  uint8_t * grid = d.ws_grid + (size_t)blockIdx.x * d.ws_grid_pitch;
  const int half = d.ksize / 2, taps = d.ksize * d.ksize;
  for (int pair = blockIdx.x; pair < d.npairs; pair += gridDim.x) {
    {
      uint4 * g4 = reinterpret_cast<uint4 *>(grid);
      const int n16 = d.data_size / 16;
      for (int i = threadIdx.x; i < n16; i += blockDim.x) g4[i] = make_uint4(0, 0, 0, 0);
      for (int i = n16 * 16 + threadIdx.x; i < d.data_size; i += blockDim.x) grid[i] = 0;
    }
    __syncthreads();
    const int it0 = d.pair_item_start[pair], it1 = d.pair_item_start[pair + 1];
    // cells dropped by AddScan's occupancy test were marked < 0 by the coarse pass: plain max-stamp
    for (int it = it0; it < it1; ++it) {
      const int32_t * cl = d.cells + (size_t)it * d.max_n;
      const int total = d.cell_count[it] * taps;
      for (int t = threadIdx.x; t < total; t += blockDim.x) {
        int32_t cell = cl[t / taps];
        if (cell < 0) continue;
        const int k = t % taps;
        uint32_t kv = d.kern[k];
        if (kv == 0) continue;
        int gx = (cell & 0xFFFF) + d.roi_x + (k % d.ksize) - half;
        int gy = (cell >> 16) + d.roi_y + (k / d.ksize) - half;
        atomic_max_u8(grid + (size_t)gy * d.stride + gx, kv);
      }
    }
    __syncthreads();
    const int P = f.P, nA = f.nA, n = d.n;
    const int32_t * off = f.offsets + (size_t)pair * nA * n;
    const int32_t * pos = f.posidx + (size_t)pair * P;
    int32_t * sums = f.sums + (size_t)pair * P * nA;
    // one warp per (pose, angle): lanes split the beams
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int item = warp; item < P * nA; item += nw) {
      const int p = item / nA, a = item - p * nA;
      const int base = pos[p];
      int acc = 0;
      for (int i = lane; i < n; i += 32) {
        int idx = base + off[a * n + i];
        if ((unsigned)idx < (unsigned)d.data_size) acc += grid[idx];
      }
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) sums[item] = acc;
    }
    __syncthreads();
  }
}


// ------------------------------------------------------------------------------------------
// Fast sweep kernel (see FastDev in sm_types.cuh).  One CTA (1024 threads, ~224 KB smem) per pair.
//   smem: S = one parity sub-grid (bytes, row pitch 304 B) | A = int32 accumulators [a][y][x]
//   per phase (column parity p, row parity q):
//     raster the taps of every valid point that fall on (p, q) cells into S          (M.cpp:1080-1104)
//     warp-item = (angle, x-tile of 16 poses); lane = (row y_l = lane / 4, word j_l = lane % 4),
//       each thread owns rows y_l + 8 r (r < 6) x 4 consecutive x-poses of its word.
//     for every FAST beam of (angle, phase, alignment m): ONE 32-bit shared load per row gives the
//       4 poses' grid bytes; two beams' words are added bytewise first (values <= 100, so 2 fit a
//       byte), then split into 16-bit fields and accumulated; fields are flushed to A every <= 640
//       beams.  Integer sums are exact, so the volume equals M.cpp:1190-1201 bit for bit.
//     SLOW beams (window leaves the grid / wraps a row) take the reference's linear-index rule.
//   then the same reduction as the generic path (pair_epilogue).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t even_bytes(uint32_t w) { return __byte_perm(w, 0, 0x4240); }   // [b0, 0, b2, 0]
__device__ __forceinline__ uint32_t odd_bytes(uint32_t w) { return __byte_perm(w, 0, 0x4341); }    // [b1, 0, b3, 0]

__global__ void __launch_bounds__(kFastThreads, 1) k_sweep_fast(SweepDev d, FastDev f)
{
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ double s_dscratch[32];
  __shared__ int s_iscratch[32];
  const int sub_words = f.sub_rows * kSubPitchW;
  uint32_t * S = reinterpret_cast<uint32_t *>(s_raw);
  uint8_t * S8 = s_raw;
  int32_t * A = reinterpret_cast<int32_t *>(s_raw + (size_t)sub_words * 4);
  const int nX = d.nX, nY = d.nY, nA = d.nA, P = nX * nY;
  const int half = d.ksize / 2, taps = d.ksize * d.ksize;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int y_l = lane >> 2, j_l = lane & 3;
  constexpr int kPitchB = kSubPitchW * 4;

  for (int pair = blockIdx.x; pair < d.npairs; pair += gridDim.x) {
    const int q = d.pair_query[pair];
    for (int i = threadIdx.x; i < nA * P; i += blockDim.x) A[i] = 0;
    const int it0 = d.pair_item_start[pair], it1 = d.pair_item_start[pair + 1];

    for (int ph = 0; ph < 4; ++ph) {
      const int pp = ph & 1, pq = ph >> 1;
      __syncthreads();
      for (int i = threadIdx.x; i < sub_words; i += blockDim.x) S[i] = 0;
      __syncthreads();
      // ---- raster: taps landing on (pp, pq) cells ----
      for (int it = it0; it < it1; ++it) {
        const int32_t * cl = d.cells + (size_t)it * d.max_n;
        const int total = d.cell_count[it] * taps;
        for (int t = threadIdx.x; t < total; t += blockDim.x) {
          const int32_t cell = cl[t / taps];
          if (cell < 0) continue;
          const int k = t % taps;
          const uint32_t kv = d.kern[k];
          if (kv == 0) continue;
          const int gx = (cell & 0xFFFF) + d.roi_x + (k % d.ksize) - half;
          const int gy = (cell >> 16) + d.roi_y + (k / d.ksize) - half;
          if ((gx & 1) != pp || (gy & 1) != pq) continue;
          atomic_max_u8(S8 + (gy >> 1) * kPitchB + (gx >> 1), kv);
        }
      }
      __syncthreads();
      // ---- FAST beams ----
      for (int wi = warp; wi < nA * f.xtiles; wi += nwarps) {
        const int a = wi / f.xtiles, xt = wi - a * f.xtiles;
        const int32_t * cs = f.cls_start + ((size_t)q * nA + a) * 33 + ph * 8;
        const int32_t * es = f.edge_start + ((size_t)q * nA + a) * 17 + ph * 4;
        const uint32_t base = (uint32_t)((y_l * kSubPitchW + 4 * xt + j_l) * 4);
        int32_t * Arow = A + a * P;
        for (int m = 0; m < 4; ++m) {
          // group layout: [plain entries (one per beam) | multi entries (descriptor + multiplicity >= 3)]
          int b = cs[2 * m];
          const int mb = cs[2 * m + 1], me = cs[2 * m + 2];
          bool multi_done = (mb == me);
          const int x0 = 4 * (4 * xt + j_l) - m;
          // flush the 16-bit fields: pose x = x0 + t, t = 0..3 (most windows of a sparse grid are empty)
          auto flush = [&](const uint32_t (&T0)[kFastRowTiles], const uint32_t (&T1)[kFastRowTiles]) {
            uint32_t any = 0;
#pragma unroll
            for (int r = 0; r < kFastRowTiles; ++r) any |= T0[r] | T1[r];
            if (!__any_sync(0xffffffffu, any != 0)) return;
#pragma unroll
            for (int r = 0; r < kFastRowTiles; ++r) {
              const int y = y_l + 8 * r;
              if (y >= nY || (T0[r] | T1[r]) == 0) continue;
              int32_t * dst = Arow + y * nX + x0;
              const int v0 = T0[r] & 0xFFFF, v1 = T1[r] & 0xFFFF, v2 = T0[r] >> 16, v3 = T1[r] >> 16;
              if (v0 && (unsigned)(x0 + 0) < (unsigned)nX) atomicAdd(dst + 0, v0);
              if (v1 && (unsigned)(x0 + 1) < (unsigned)nX) atomicAdd(dst + 1, v1);
              if (v2 && (unsigned)(x0 + 2) < (unsigned)nX) atomicAdd(dst + 2, v2);
              if (v3 && (unsigned)(x0 + 3) < (unsigned)nX) atomicAdd(dst + 3, v3);
            }
          };
          do {
            const int ce = min(mb, b + kFastChunk);
            uint32_t T0[kFastRowTiles], T1[kFastRowTiles];
#pragma unroll
            for (int r = 0; r < kFastRowTiles; ++r) { T0[r] = 0; T1[r] = 0; }
            // descriptors are fetched 32 at a time (one per lane, coalesced) and broadcast by shuffle
            for (int b0 = b; b0 < ce; b0 += 32) {
              const int cnt = min(32, ce - b0);
              const uint32_t mine = (lane < cnt) ? 4u * f.beams[b0 + lane] : 0u;
              int k = 0;
              for (; k + 3 < cnt; k += 4) {   // 4 beams: two byte-wise pair sums, one 3-input add per field
                const uint32_t o0 = base + __shfl_sync(0xffffffffu, mine, k), o1 = base + __shfl_sync(0xffffffffu, mine, k + 1);
                const uint32_t o2 = base + __shfl_sync(0xffffffffu, mine, k + 2), o3 = base + __shfl_sync(0xffffffffu, mine, k + 3);
#pragma unroll
                for (int r = 0; r < kFastRowTiles; ++r) {
                  const uint32_t wa = *reinterpret_cast<const uint32_t *>(S8 + o0 + r * 8 * kPitchB) +
                                      *reinterpret_cast<const uint32_t *>(S8 + o1 + r * 8 * kPitchB);
                  const uint32_t wb = *reinterpret_cast<const uint32_t *>(S8 + o2 + r * 8 * kPitchB) +
                                      *reinterpret_cast<const uint32_t *>(S8 + o3 + r * 8 * kPitchB);
                  T0[r] = T0[r] + even_bytes(wa) + even_bytes(wb);
                  T1[r] = T1[r] + odd_bytes(wa) + odd_bytes(wb);
                }
              }
              for (; k + 1 < cnt; k += 2) {
                const uint32_t o0 = base + __shfl_sync(0xffffffffu, mine, k), o1 = base + __shfl_sync(0xffffffffu, mine, k + 1);
#pragma unroll
                for (int r = 0; r < kFastRowTiles; ++r) {
                  const uint32_t w = *reinterpret_cast<const uint32_t *>(S8 + o0 + r * 8 * kPitchB) +
                                     *reinterpret_cast<const uint32_t *>(S8 + o1 + r * 8 * kPitchB);
                  T0[r] += even_bytes(w);
                  T1[r] += odd_bytes(w);
                }
              }
              if (k < cnt) {
                const uint32_t o0 = base + __shfl_sync(0xffffffffu, mine, k);
#pragma unroll
                for (int r = 0; r < kFastRowTiles; ++r) {
                  const uint32_t w = *reinterpret_cast<const uint32_t *>(S8 + o0 + r * 8 * kPitchB);
                  T0[r] += even_bytes(w);
                  T1[r] += odd_bytes(w);
                }
              }
            }
            b = ce;
            if (b == mb && !multi_done) {
              // beams that share one grid cell (several per 5 cm cell at indoor ranges): one load, fields times k.
              // The host only builds multi entries when the whole group's weight fits one flush (<= kFastChunk).
              for (int b0 = mb; b0 < me; b0 += 32) {
                const int cnt = min(32, me - b0);
                const uint32_t mine = (lane < cnt) ? 4u * f.beams[b0 + lane] : 0u;
                const uint32_t myk = (lane < cnt) ? f.mult[b0 + lane] : 0u;
                for (int k = 0; k < cnt; ++k) {
                  const uint32_t o0 = base + __shfl_sync(0xffffffffu, mine, k);
                  const uint32_t kk = __shfl_sync(0xffffffffu, myk, k);
#pragma unroll
                  for (int r = 0; r < kFastRowTiles; ++r) {
                    const uint32_t w = *reinterpret_cast<const uint32_t *>(S8 + o0 + r * 8 * kPitchB);
                    T0[r] += even_bytes(w) * kk;
                    T1[r] += odd_bytes(w) * kk;
                  }
                }
              }
              multi_done = true;
            }
            flush(T0, T1);
          } while (b < mb || !multi_done);
          // EDGE beams of this group (window partly outside the grid): same word loads, but rows / words that fall
          // outside the sub-grid are skipped (they index outside [0, data_size) or wrap in the reference; the wrapped
          // part is added by the secondary list below). Rows / words inside the allocation but beyond the valid cells
          // are zero padding, so only the allocation bounds need checking.
          int eb = es[m];
          const int ee = es[m + 1];
          while (eb < ee) {
            const int ce = min(ee, eb + kFastChunk);
            uint32_t T0[kFastRowTiles], T1[kFastRowTiles];
#pragma unroll
            for (int r = 0; r < kFastRowTiles; ++r) { T0[r] = 0; T1[r] = 0; }
            for (int b0 = eb; b0 < ce; b0 += 32) {
              const int cnt = min(32, ce - b0);
              const int32_t mine = (lane < cnt) ? f.edge[b0 + lane] : 0;
              for (int k = 0; k < cnt; ++k) {
                const int32_t e = __shfl_sync(0xffffffffu, mine, k);
                const int row0 = (int)(int16_t)(e & 0xFFFF) + y_l, wq = (e >> 16) + 4 * xt + j_l;
                const bool cv = (unsigned)wq < (unsigned)kSubPitchW;
#pragma unroll
                for (int r = 0; r < kFastRowTiles; ++r) {
                  const int row = row0 + 8 * r;
                  const uint32_t w = (cv && (unsigned)row < (unsigned)f.sub_rows) ? S[row * kSubPitchW + wq] : 0u;
                  T0[r] += even_bytes(w);
                  T1[r] += odd_bytes(w);
                }
              }
            }
            eb = ce;
            flush(T0, T1);
          }
        }
      }
      // ---- EDGE beams: the window leaves the grid (readings close to / beyond the range threshold).
      //   primary list (this phase = the beam's own parity): poses whose column stays inside [0, stride); rows outside
      //     [0, height) index outside [0, data_size) in the reference and contribute 0;
      //   secondary list (row parity flipped): poses whose column left [0, stride) by less than one stride -- the
      //     reference's linear index (M.cpp:1192-1200) makes them read the neighbouring row at column -/+ stride.
      //   Every thread owns up to 3 fixed poses (coordinates in registers: no division in the loops) and walks the beams. ----
      {
        const bool has_wrap = f.wrap2_start[((size_t)q * nA + nA - 1) * 4 + 4] - f.wrap2_start[(size_t)q * nA * 4] > 0;
        if (has_wrap) {
          int ex[3], ey[3];
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int p = threadIdx.x + k * kFastThreads;
            ex[k] = p < P ? 2 * (p % nX) : -100000;   // poses beyond P never hit a valid column
            ey[k] = 2 * (p / nX);
          }
          if (has_wrap) {
            const int32_t * cl = f.wrap2_start + ((size_t)q * nA) * 4 + ph;
            for (int a = 0; a < nA; ++a) {
              int32_t * Aa = A + a * P + threadIdx.x;
              for (int bi = cl[4 * a]; bi < cl[4 * a + 1]; ++bi) {
                const int32_t e = f.wrap2[bi];
                const int Xb = (int)(int16_t)(e & 0xFFFF), Yb = e >> 16;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                  const int col = Xb + ex[k];
                  if ((unsigned)col < (unsigned)d.stride || ex[k] < 0) continue;
                  const int r2 = Yb + ey[k] + (col < 0 ? -1 : 1);
                  const int c2 = col + (col < 0 ? d.stride : -d.stride);
                  if ((unsigned)r2 >= (unsigned)d.height) continue;
                  const int v = S8[(r2 >> 1) * kPitchB + (c2 >> 1)];
                  if (v) atomicAdd(Aa + k * kFastThreads, v);
                }
              }
            }
          }
        }
      }
      // ---- FAR beams: column offsets of a stride or more (readings near the laser's maximum range at fine grids):
      //      pose by pose on the linear index with a division, every phase. Rare. ----
      {
        const int32_t * ss = f.slow_start + (size_t)q * (nA + 1);
        const int nslow = ss[nA] - ss[0];
        if (nslow > 0) {
          const int32_t * pos = d.posidx + (size_t)q * P;
          for (int a = 0; a < nA; ++a) {
            const int sb = ss[a], se = ss[a + 1];
            const int work = (se - sb) * P;
            for (int t = threadIdx.x; t < work; t += blockDim.x) {
              const int bi = t / P, p = t - bi * P;
              const int idx = pos[p] + f.slow[sb + bi];
              if ((unsigned)idx >= (unsigned)d.data_size) continue;
              const int row = idx / d.stride, col = idx - row * d.stride;
              if ((col & 1) != pp || (row & 1) != pq) continue;
              const int v = S8[(row >> 1) * kPitchB + (col >> 1)];
              if (v) atomicAdd(A + a * P + p, v);
            }
          }
        }
      }
    }
    __syncthreads();
    // S is free now: reuse it as the FP64 scratch of the reduction (5 P doubles)
    pair_epilogue(d, pair, q, SumsAngleMajor{A, P}, reinterpret_cast<double *>(s_raw), s_dscratch, s_iscratch);
  }
}

// Per-query best-response key for the multi-GPU sweep: key = best_sum << 32 | (0xFFFFFFFF - global
// candidate id), so that a max-reduction (here atomicMax, across GPUs ncclMax) picks the highest
// integer correlation sum and breaks ties towards the lowest candidate id, deterministically.
__global__ void k_best_keys(const PairOut * __restrict__ out, const int32_t * __restrict__ pair_query,
                            const int32_t * __restrict__ pair_chain, int npairs, long long id_offset,
                            unsigned long long * __restrict__ keys)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  const unsigned long long id = (unsigned long long)(id_offset + pair_chain[p]) & 0xFFFFFFFFull;
  const unsigned long long key = ((unsigned long long)(uint32_t)out[p].best_sum << 32) | (0xFFFFFFFFull - id);
  atomicMax(keys + pair_query[p], key);
}

// Winner records for the multi-GPU sweep (SURVEY.md 8e).  Per query: the pair with the highest best response, ties to the
// lowest global candidate id, and its raw device reduction (PairOut).  Three passes over the pairs: max of the response
// bit pattern (a non-negative double orders like its bits, so this also holds for penalised responses), min of the global
// id among the pairs that reach it, copy of that pair's PairOut.  The records of all ranks are exchanged with ONE
// all-gather (Q x 152 B per rank) and every rank selects and finishes the same winner locally.
struct WinRec {
  unsigned long long resp_bits;   // bit pattern of PairOut::best; 0 with gid < 0 = this rank has no pair for the query
  long long gid;                  // global candidate id (id_offset + chain index), -1 = none
  PairOut out;
};

__global__ void k_win_init(WinRec * __restrict__ rec, int nq)
{
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  rec[q].resp_bits = 0ull;
  rec[q].gid = 0x7FFFFFFFFFFFFFFFll;
}
__global__ void k_win_max(const PairOut * __restrict__ out, const int32_t * __restrict__ pair_query, int npairs, WinRec * __restrict__ rec)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  atomicMax(&rec[pair_query[p]].resp_bits, (unsigned long long)__double_as_longlong(out[p].best));
}
__global__ void k_win_id(const PairOut * __restrict__ out, const int32_t * __restrict__ pair_query, const int32_t * __restrict__ pair_chain,
                         int npairs, long long id_offset, WinRec * __restrict__ rec)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  WinRec & r = rec[pair_query[p]];
  if ((unsigned long long)__double_as_longlong(out[p].best) == r.resp_bits) atomicMin(&r.gid, id_offset + pair_chain[p]);
}
__global__ void k_win_copy(const PairOut * __restrict__ out, const int32_t * __restrict__ pair_query, const int32_t * __restrict__ pair_chain,
                           int npairs, long long id_offset, WinRec * __restrict__ rec, unsigned char * __restrict__ has_pair)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  WinRec & r = rec[pair_query[p]];
  if ((unsigned long long)__double_as_longlong(out[p].best) == r.resp_bits && id_offset + pair_chain[p] == r.gid) {
    r.out = out[p];   // (query, chain) pairs are unique, so exactly one thread copies
    has_pair[pair_query[p]] = 1;
  }
}
__global__ void k_win_fix(WinRec * __restrict__ rec, const unsigned char * __restrict__ has_pair, int nq)
{
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  if (!has_pair[q]) { rec[q].gid = -1; rec[q].resp_bits = 0ull; }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------

void SweepHost::release()
{
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  ev0 = ev1 = nullptr;
  uploaded = ran = false;
}

static thread_local int64_t * g_h2d_counter = nullptr;

// Host -> device copy of a small table through the sweep's pinned arena: the source may be reused or freed as soon as this
// returns and nothing blocks, so the host keeps building tables while the candidate points are still in flight.
static thread_local SweepHost * g_arena_owner = nullptr;
void sweep_stage_h2d(void * dst, const void * src, size_t bytes, cudaStream_t s)
{
  if (!bytes) return;
  SweepHost * S = g_arena_owner;
  const size_t need = (bytes + 63) & ~(size_t)63;
  if (S && S->arena_used + need <= S->arena.cap) {
    unsigned char * stage = S->arena.p + S->arena_used;
    S->arena_used += need;
    std::memcpy(stage, src, bytes);
    B200_CUDA(cudaMemcpyAsync(dst, stage, bytes, cudaMemcpyHostToDevice, s));
  } else {
    B200_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
    B200_CUDA(cudaStreamSynchronize(s));   // arena exhausted: plain copy, the source may go away after return
  }
  if (g_h2d_counter) *g_h2d_counter += (int64_t)bytes;
}

template <class T>
static void h2d(DevBuf<T> & dst, const T * src, size_t count, cudaStream_t s)
{
  dst.reserve(count);
  sweep_stage_h2d(dst.p, src, count * sizeof(T), s);
}

static GridGeom geom_for_query(const b200sm * h, const b200_scan * q)
{
  GridGeom g;
  g.width = h->g.width; g.height = h->g.height; g.stride = h->g.stride;
  g.roi_x = h->g.roi_x; g.roi_y = h->g.roi_y; g.roi_w = h->g.roi_w; g.roi_h = h->g.roi_h;
  g.data_size = h->g.data_size; g.ksize = h->g.ksize; g.order_dependent = h->g.order_dependent;
  g.scale = h->g.scale;
  set_grid_offset(g, q);
  return g;
}

static void coarse_search(const b200sm * h, double off[2], double res[2])
{
  double r = 1.0 / h->g.scale;
  double dim = (double)h->probs_side;
  off[0] = off[1] = 0.5 * (dim - 1) * r;   // M.cpp:579-581
  res[0] = res[1] = 2 * r;                 // M.cpp:584-585
}

static bool build_fast_tables(b200sm * h, SweepHost & S, cudaStream_t st);

// shared memory the generic kernel may fill with lookup rows; a query needs at least one row (n <= 51,200 readings)
constexpr size_t kGenericTableBytes = 200 * 1024;
// whole angle rows of the lookup table per slice of the generic kernel: all nA when the table fits (one slice, staged once
// per query), else as many as fit
static int generic_slice_rows(int nA, int n)
{
  const size_t row = (size_t)n * sizeof(int32_t);
  return (int)std::min<size_t>((size_t)nA, kGenericTableBytes / row);
}

static int sweep_upload(b200sm * h, const b200_scan * queries, int nq, const b200_scan * scans, int nscans,
                        const int32_t * chain_start, int nchains, const int32_t * pair_query,
                        const int32_t * pair_chain, int npairs, bool do_penalize)
{
  NvtxRange nvtx_("b200sm sweep upload");
  const auto t_enter = std::chrono::steady_clock::now();
  SweepHost & S = h->sweep;
  S.uploaded = S.ran = false;
  S.zero_done.clear(); S.zero_exp_done.clear();
  g_h2d_counter = &S.h2d_bytes;
  if (!queries || nq <= 0 || !scans || nscans <= 0 || !chain_start || nchains <= 0) {
    set_last_error("sweep: empty or NULL input");
    return B200_ERR_INVALID_ARG;
  }
  if ((pair_query == nullptr) != (pair_chain == nullptr)) { set_last_error("sweep: give both pair arrays or neither"); return B200_ERR_INVALID_ARG; }
  if (!pair_query) npairs = nq * nchains;
  if (npairs <= 0) { set_last_error("sweep: no pairs"); return B200_ERR_INVALID_ARG; }
  const int n = queries[0].n;
  for (int q = 0; q < nq; ++q) {
    if (queries[q].n != n || n <= 0 || !queries[q].ranges || !queries[q].points_xy) {
      set_last_error("sweep: every query needs the same, non-zero number of readings");
      return B200_ERR_INVALID_ARG;
    }
  }
  if (chain_start[0] != 0 || chain_start[nchains] != nscans) { set_last_error("sweep: chain_start must cover scans[0..nscans)"); return B200_ERR_INVALID_ARG; }
  for (int c = 0; c < nchains; ++c)
    if (chain_start[c + 1] < chain_start[c]) { set_last_error("sweep: chain_start must be non-decreasing"); return B200_ERR_INVALID_ARG; }
  h->ensure_stream();
  cudaStream_t st = h->stream;
  const GridGeom & g0 = h->g;
  B200_CUDA(cudaStreamSynchronize(st));   // copies of the previous upload are done: its staging arena can be reused
  g_arena_owner = &S;
  S.arena_used = S.arena.cap;             // nothing staged until the arena is sized (after the plans, below)

  // ---- candidate scans first: their 17 KB/scan copy runs while the host builds the per-query tables ----
  std::vector<int32_t> pt_start(nscans + 1, 0);
  int max_n = 0;
  bool contiguous = true;
  for (int s = 0; s < nscans; ++s) {
    if (scans[s].n < 0 || (scans[s].n > 0 && !scans[s].points_xy)) { set_last_error("sweep: candidate scan without points"); return B200_ERR_INVALID_ARG; }
    pt_start[s + 1] = pt_start[s] + scans[s].n;
    max_n = std::max(max_n, scans[s].n);
    if (s > 0 && scans[s].points_xy != scans[s - 1].points_xy + 2 * (size_t)scans[s - 1].n) contiguous = false;
  }
  const size_t npts = (size_t)pt_start[nscans];
  S.d_points.reserve(2 * npts + 2);
  if (contiguous) {
    // caller laid the scans out back to back (pinned or not): one copy straight from its buffer
    B200_CUDA(cudaMemcpyAsync(S.d_points.p, scans[0].points_xy, 2 * npts * sizeof(double), cudaMemcpyHostToDevice, st));
    S.h2d_bytes += (int64_t)(2 * npts * sizeof(double));
  } else {
    S.h_d.reserve(2 * npts);
    for (int s = 0; s < nscans; ++s)
      std::memcpy(S.h_d.p + 2 * (size_t)pt_start[s], scans[s].points_xy, 2 * (size_t)scans[s].n * sizeof(double));
    B200_CUDA(cudaMemcpyAsync(S.d_points.p, S.h_d.p, 2 * npts * sizeof(double), cudaMemcpyHostToDevice, st));
    S.h2d_bytes += (int64_t)(2 * npts * sizeof(double));
    B200_CUDA(cudaStreamSynchronize(st));   // h_d is reused for the per-query tables below
  }
  S.max_n = (std::max(max_n, 1) + 3) & ~3;   // multiple of 4: every scan's cell list starts 16-byte aligned (bulk-copy staging)

  // ---- coarse plans, one per query ----
  const auto t_plans0 = std::chrono::steady_clock::now();
  double off[2], res[2];
  coarse_search(h, off, res);
  S.plans.assign(nq, CorrPlan());
  for (int q = 0; q < nq; ++q) {
    GridGeom g = geom_for_query(h, &queries[q]);
    int rc = build_plan(g, h->probs_side, h->p, &queries[q], queries[q].sensor_pose, off, res,
                        h->p.coarse_search_angle_offset, h->p.coarse_angle_resolution, false, S.plans[q]);
    if (rc != B200_OK) return rc;
  }
  const auto t_plans1 = std::chrono::steady_clock::now();
  const CorrPlan & p0 = S.plans[0];
  const int nX = p0.nX, nY = p0.nY, nA = p0.nA, P = nX * nY;
  {
    // pinned staging arena for every table of this upload: per query the lookup table (int32), the descriptor lists of the
    // kernel that runs (16 bit + headers) and the pose arrays; per pair / item / scan the index arrays
    const size_t per_query = (size_t)nA * n * 4 * 3 + (size_t)P * 4 + (size_t)(nX + nY) * 48 + 16384;
    const size_t lists = (size_t)npairs * 16 + (size_t)nscans * 8 + (1u << 20);
    size_t items = 0;
    for (int c = 0; c < nchains; ++c) items = std::max<size_t>(items, (size_t)(chain_start[c + 1] - chain_start[c]));
    S.arena.reserve((size_t)nq * per_query + lists + (size_t)npairs * items * 8);
    S.arena_used = 0;
  }
  if ((size_t)n * sizeof(int32_t) > kGenericTableBytes) {
    set_last_error("sweep: one lookup row of the query does not fit shared memory (more than 51,200 readings per query)");
    return B200_ERR_UNSUPPORTED;
  }
  S.nq = nq; S.n = n; S.npairs = npairs; S.nscans = nscans; S.do_penalize = do_penalize;
  S.queries.assign(queries, queries + nq);
  S.scans.assign(scans, scans + nscans);
  S.chain_start.assign(chain_start, chain_start + nchains + 1);
  S.pair_query.resize(npairs); S.pair_chain.resize(npairs);
  for (int p = 0; p < npairs; ++p) {
    int q = pair_query ? pair_query[p] : p / nchains;
    int c = pair_chain ? pair_chain[p] : p % nchains;
    if (q < 0 || q >= nq || c < 0 || c >= nchains) { set_last_error("sweep: pair index out of range"); return B200_ERR_INVALID_ARG; }
    S.pair_query[p] = q; S.pair_chain[p] = c;
  }

  // ---- per-query tables ----
  {
    const size_t no = (size_t)nq * nA * n, np = (size_t)nq * P;
    S.h_i.reserve(no + np);
    for (int q = 0; q < nq; ++q) {
      const CorrPlan & pl = S.plans[q];
      for (size_t i = 0; i < (size_t)nA * n; ++i) S.h_i.p[(size_t)q * nA * n + i] = device_offset(pl.offsets[i], g0.data_size);
      for (int y = 0; y < nY; ++y)
        for (int x = 0; x < nX; ++x) S.h_i.p[no + (size_t)q * P + (size_t)y * nX + x] = pl.xs[x] + pl.ys[y] * g0.stride;
    }
    h2d(S.d_offsets, S.h_i.p, no, st);
    h2d(S.d_posidx, S.h_i.p + no, np, st);
    // doubles: qgeom[4], center[3], then 6 arrays of nX/nY, angpen
    const size_t per = 4 + 3 + 3 * (size_t)nX + 3 * (size_t)nY + nA;
    S.h_d.reserve(per * nq);
    double * qgeom = S.h_d.p, * center = qgeom + 4 * (size_t)nq, * xrel = center + 3 * (size_t)nq, * newx = xrel + (size_t)nq * nX,
           * sqx = newx + (size_t)nq * nX, * yrel = sqx + (size_t)nq * nX, * newy = yrel + (size_t)nq * nY,
           * sqy = newy + (size_t)nq * nY, * angpen = sqy + (size_t)nq * nY;
    for (int q = 0; q < nq; ++q) {
      const CorrPlan & pl = S.plans[q];
      GridGeom g = geom_for_query(h, &queries[q]);
      qgeom[4 * q + 0] = queries[q].sensor_pose[0]; qgeom[4 * q + 1] = queries[q].sensor_pose[1];   // view point, M.cpp:574
      qgeom[4 * q + 2] = g.off_x; qgeom[4 * q + 3] = g.off_y;
      for (int i = 0; i < 3; ++i) center[3 * q + i] = pl.center[i];
      for (int x = 0; x < nX; ++x) { xrel[(size_t)q * nX + x] = pl.xrel[x]; newx[(size_t)q * nX + x] = pl.newx[x]; sqx[(size_t)q * nX + x] = pl.sqx[x]; }
      for (int y = 0; y < nY; ++y) { yrel[(size_t)q * nY + y] = pl.yrel[y]; newy[(size_t)q * nY + y] = pl.newy[y]; sqy[(size_t)q * nY + y] = pl.sqy[y]; }
      for (int a = 0; a < nA; ++a) angpen[(size_t)q * nA + a] = pl.angpen[a];
    }
    h2d(S.d_qd, S.h_d.p, per * nq, st);
  }

  // ---- pairs and items ----
  std::vector<int32_t> pair_item_start(npairs + 1, 0);
  for (int p = 0; p < npairs; ++p) {
    int c = S.pair_chain[p];
    pair_item_start[p + 1] = pair_item_start[p] + (chain_start[c + 1] - chain_start[c]);
  }
  const int nitems = pair_item_start[npairs];
  S.nitems = nitems;
  {
    const size_t tot = (size_t)(nscans + 1) + npairs + (npairs + 1) + 2 * (size_t)nitems;
    S.h_i.reserve(tot);
    int32_t * a_pt = S.h_i.p, * a_pq = a_pt + nscans + 1, * a_pis = a_pq + npairs, * a_ip = a_pis + npairs + 1, * a_is = a_ip + nitems;
    std::memcpy(a_pt, pt_start.data(), (nscans + 1) * sizeof(int32_t));
    std::memcpy(a_pq, S.pair_query.data(), npairs * sizeof(int32_t));
    std::memcpy(a_pis, pair_item_start.data(), (npairs + 1) * sizeof(int32_t));
    for (int p = 0; p < npairs; ++p) {
      int c = S.pair_chain[p];
      for (int k = 0; k < chain_start[c + 1] - chain_start[c]; ++k) {
        a_ip[pair_item_start[p] + k] = p;
        a_is[pair_item_start[p] + k] = chain_start[c] + k;
      }
    }
    h2d(S.d_scan_pt_start, a_pt, nscans + 1, st);
    h2d(S.d_pair_query, a_pq, npairs, st);
    h2d(S.d_pair_chain, S.pair_chain.data(), npairs, st);
    h2d(S.d_pair_item_start, a_pis, npairs + 1, st);
    h2d(S.d_item_pair, a_ip, std::max(nitems, 1), st);
    h2d(S.d_item_scan, a_is, std::max(nitems, 1), st);
  }
  S.d_cells.reserve((size_t)std::max(nitems, 1) * S.max_n);
  S.d_cell_count.reserve(std::max(nitems, 1));
  if (S.d_kernel.cap == 0) h2d(S.d_kernel, g0.kernel.data(), g0.kernel.size(), st);

  // ---- workspaces: one per resident CTA ----
  int dev = 0, sms = 132;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const size_t smem = (size_t)generic_slice_rows(nA, n) * n * sizeof(int32_t);
  const int per_sm = smem <= 100 * 1024 ? 2 : 1;
  S.blocks = std::min(npairs, sms * per_sm);
  const size_t gpitch = ((size_t)g0.data_size + 255) & ~(size_t)255;
  const size_t spitch = ((size_t)P * nA + 63) & ~(size_t)63;
  const size_t ppitch = ((size_t)5 * P + 31) & ~(size_t)31;
  S.d_ws_grid.reserve(gpitch * S.blocks);
  S.d_ws_sums.reserve(spitch * S.blocks);
  S.d_ws_probs.reserve(ppitch * S.blocks);
  S.d_out.reserve(npairs);
  S.h_out.reserve(npairs);

  SweepDev & d = S.dev;
  d.stride = g0.stride; d.height = g0.height; d.roi_x = g0.roi_x; d.roi_y = g0.roi_y; d.roi_w = g0.roi_w; d.roi_h = g0.roi_h;
  d.data_size = g0.data_size; d.ksize = g0.ksize; d.order_dependent = g0.order_dependent ? 1 : 0;
  d.scale = g0.scale; d.kern = S.d_kernel.p;
  d.nX = nX; d.nY = nY; d.nA = nA; d.n = n;
  d.norm = (double)((uint32_t)n * (uint32_t)kOccupied);
  d.do_penalize = do_penalize ? 1 : 0;
  d.dist_var = h->p.distance_variance_penalty; d.min_dist_pen = h->p.minimum_distance_penalty;
  d.offsets = S.d_offsets.p; d.posidx = S.d_posidx.p;
  {
    double * base = S.d_qd.p;
    d.qgeom = base; d.center = base + 4 * (size_t)nq;
    d.xrel = d.center + 3 * (size_t)nq; d.newx = d.xrel + (size_t)nq * nX; d.sqx = d.newx + (size_t)nq * nX;
    d.yrel = d.sqx + (size_t)nq * nX; d.newy = d.yrel + (size_t)nq * nY; d.sqy = d.newy + (size_t)nq * nY;
    d.angpen = d.sqy + (size_t)nq * nY;
  }
  d.points = S.d_points.p; d.scan_pt_start = S.d_scan_pt_start.p;
  d.npairs = npairs; d.nitems = nitems; d.max_n = S.max_n;
  d.pair_query = S.d_pair_query.p; d.pair_item_start = S.d_pair_item_start.p;
  d.item_pair = S.d_item_pair.p; d.item_scan = S.d_item_scan.p;
  d.cells = S.d_cells.p; d.cell_count = S.d_cell_count.p;
  d.ws_grid = S.d_ws_grid.p; d.ws_grid_pitch = gpitch;
  d.ws_sums = S.d_ws_sums.p; d.ws_sums_pitch = spitch;
  d.ws_probs = S.d_ws_probs.p; d.ws_probs_pitch = ppitch;
  d.out = S.d_out.p;
  if (!S.ev0) { B200_CUDA(cudaEventCreate(&S.ev0)); B200_CUDA(cudaEventCreate(&S.ev1)); }
  // tables of the kernel that will run only (see sweep_kernel_choice).  The tiled cluster kernel is the default everywhere: with
  // the atomic-free levelled raster it is ahead of the single-CTA kernel on that kernel's own geometry too (on an H100, 400 W power
  // limit: 387 k vs 273 k matches/s at cfg2, bench.py); "sweep_kernel" = 1 still selects the single-CTA kernel.
  S.fast.enabled = 0; S.tile.enabled = 0;
  S.fast_info[0] = 0; S.tile_info[0] = 0;
  for (int i = 0; i < 4; ++i) S.tile_layout[i] = 0;
  const auto t_tab0 = std::chrono::steady_clock::now();
  bool have = false;
  if (!h->force_generic && h->sweep_kernel == 1) have = build_fast_tables(h, S, st);
  if (!h->force_generic && !have) have = build_tile_tables(h, S, st);
  if (!h->force_generic && !have && h->sweep_kernel != 1) build_fast_tables(h, S, st);
  const auto t_tab1 = std::chrono::steady_clock::now();
  auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  S.upload_ms[0] = ms(t_plans0, t_plans1); S.upload_ms[1] = ms(t_tab0, t_tab1); S.upload_ms[2] = ms(t_enter, t_tab1);
  S.uploaded = true;
  return B200_OK;
}

// Builds the per-query beam lists of the fast path; returns false when this sweep cannot use it.
static bool build_fast_tables(b200sm * h, SweepHost & S, cudaStream_t st)
{
  const GridGeom & g = h->g;
  const CorrPlan & p0 = S.plans[0];
  const int nX = p0.nX, nY = p0.nY, nA = p0.nA, n = p0.n, nq = S.nq;
  S.fast.enabled = 0;
  S.fast_info[0] = 0; S.fast_info[1] = S.fast_info[2] = S.fast_info[3] = 0;
  auto bail = [&](int why) { S.fast_info[4] = why; return false; };
  if (g.order_dependent) return bail(1);
  if (nY > 8 * kFastRowTiles || (g.stride & 1) || nX * nY > 3 * kFastThreads) return bail(2);
  if (g.stride / 2 > kSubPitchW * 4 - 16) return bail(3);   // sub-grid row + the 3-word overhang must fit the pitch
  const int xtiles = (nX + 3 + 15) / 16;
  int sub_rows = (g.height + 1) / 2 + 8;                     // + padding rows read by idle row tiles
  // the S region doubles as the FP64 scratch of the reduction (5 P doubles): small grids get extra rows for it
  sub_rows = std::max(sub_rows, (int)(((size_t)5 * nX * nY * sizeof(double) + kSubPitchW * 4 - 1) / (kSubPitchW * 4)));
  const size_t smem = (size_t)sub_rows * kSubPitchW * 4 + (size_t)nA * nX * nY * 4;
  if (smem > 227 * 1024 - 1024) return bail(4);
  if ((size_t)5 * nX * nY * sizeof(double) > (size_t)sub_rows * kSubPitchW * 4) return bail(5);   // epilogue scratch reuses S
  std::vector<int32_t> cls_start((size_t)nq * nA * 33), slow, slow_start((size_t)nq * (nA + 1));
  std::vector<uint16_t> beams, mult;
  std::vector<int32_t> wrap2, wrap2_start((size_t)nq * nA * 4 + 1);
  std::vector<int32_t> edge, edge_start((size_t)nq * nA * 17);
  int n_edge = 0;
  beams.reserve((size_t)nq * nA * n);
  mult.reserve((size_t)nq * nA * n);
  // one angle's lists, built independently (one host-pool task per angle), then concatenated in angle order
  struct AngleLists {
    std::vector<uint16_t> beams, mult;
    int32_t cs[33];                          // relative to the angle's first descriptor
    std::vector<int32_t> wgroup[4], egroup[16], slow;
    int n_edge = 0;
  };
  std::vector<AngleLists> al(nA);
  for (int q = 0; q < nq; ++q) {
    const CorrPlan & pl = S.plans[q];
    for (int k = 1; k < nX; ++k) if (pl.xs[k] != pl.xs[0] + 2 * k) return bail(6);   // coarse step must be exactly 2 cells
    for (int k = 1; k < nY; ++k) if (pl.ys[k] != pl.ys[0] + 2 * k) return bail(7);
    const int X0 = pl.xs[0], Y0 = pl.ys[0];
    auto one_angle = [&](int a) {
      AngleLists & L = al[a];
      std::vector<uint16_t> group[16];
      L.beams.clear(); L.mult.clear(); L.slow.clear(); L.n_edge = 0;
      for (auto & v : L.wgroup) v.clear();
      for (auto & v : L.egroup) v.clear();
      for (int i = 0; i < n; ++i) {
        const int32_t off = pl.offsets[(size_t)a * n + i];
        if (off == kInvalidScan) continue;
        const int gx = pl.ogx[(size_t)a * n + i], gy = pl.ogy[(size_t)a * n + i];
        const int Xb = X0 + gx, Yb = Y0 + gy;
        const bool inside = Xb >= 0 && Xb + 2 * (nX - 1) < g.stride && Yb >= 0 && Yb + 2 * (nY - 1) < g.height;
        if (inside) {
          const int pp = Xb & 1, pq = Yb & 1, c = Xb >> 1, r = Yb >> 1;
          const int wo = r * kSubPitchW + (c >> 2);
          group[(pq * 2 + pp) * 4 + (c & 3)].push_back((uint16_t)wo);
        } else if (Xb >= -g.stride && Xb + 2 * (nX - 1) < 2 * g.stride && Xb > -32768 && Xb < 32767 && Yb > -32768 && Yb < 32767) {
          // EDGE beam: at most one row wrap. Primary entry in the beam's own phase; if some column leaves
          // [0, stride), a secondary entry in the phase with the row parity flipped.
          const int32_t e = (int32_t)((uint32_t)(Xb & 0xFFFF) | ((uint32_t)Yb << 16));
          const bool rows_hit = Yb + 2 * (nY - 1) >= 0 && Yb < g.height;
          const bool cols_hit = Xb + 2 * (nX - 1) >= 0 && Xb < g.stride;
          if (rows_hit && cols_hit) {
            const int c = Xb >> 1, r = Yb >> 1;   // arithmetic shifts: floor for negative coordinates
            L.egroup[((Yb & 1) * 2 + (Xb & 1)) * 4 + (c & 3)].push_back((int32_t)((uint32_t)(r & 0xFFFF) | ((uint32_t)(c >> 2) << 16)));
            ++L.n_edge;
          }
          const bool wraps = Xb < 0 || Xb + 2 * (nX - 1) >= g.stride;
          if (wraps && Yb + 2 * (nY - 1) + 1 >= 0 && Yb - 1 < g.height) L.wgroup[((Yb & 1) ^ 1) * 2 + (Xb & 1)].push_back(e);
        } else {
          const int32_t dv = device_offset(off, g.data_size);
          if (dv != kDevInvalid) L.slow.push_back(dv);   // FAR: can still index [0, data_size) for some pose
        }
      }
      for (int k = 0; k < 16; ++k) {
        std::vector<uint16_t> & gk = group[k];
        std::sort(gk.begin(), gk.end());
        L.cs[2 * k] = (int32_t)L.beams.size();
        // run-length encode: beams that land in the same cell share a descriptor. Entries with multiplicity >= 3
        // go to the group's multi list (one load, fields multiplied), provided the whole group fits one flush.
        const bool dedup = !h->no_dedup && gk.size() <= (size_t)kFastChunk;
        std::vector<std::pair<uint16_t, uint16_t>> multi;
        for (size_t i = 0; i < gk.size();) {
          size_t j = i;
          while (j < gk.size() && gk[j] == gk[i]) ++j;
          const size_t cnt = j - i;
          if (dedup && cnt >= 3) {
            multi.emplace_back(gk[i], (uint16_t)cnt);
          } else {
            for (size_t t = 0; t < cnt; ++t) { L.beams.push_back(gk[i]); L.mult.push_back(1); }
          }
          i = j;
        }
        L.cs[2 * k + 1] = (int32_t)L.beams.size();
        for (auto & mk : multi) { L.beams.push_back(mk.first); L.mult.push_back(mk.second); }
      }
      L.cs[32] = (int32_t)L.beams.size();
    };
    host_parallel_for(nA, one_angle);
    for (int a = 0; a < nA; ++a) {
      const AngleLists & L = al[a];
      slow_start[(size_t)q * (nA + 1) + a] = (int32_t)slow.size();
      slow.insert(slow.end(), L.slow.begin(), L.slow.end());
      n_edge += L.n_edge;
      for (int k = 0; k < 4; ++k) {
        wrap2_start[((size_t)q * nA + a) * 4 + k] = (int32_t)wrap2.size();
        wrap2.insert(wrap2.end(), L.wgroup[k].begin(), L.wgroup[k].end());
      }
      for (int k = 0; k < 16; ++k) {
        edge_start[((size_t)q * nA + a) * 17 + k] = (int32_t)edge.size();
        edge.insert(edge.end(), L.egroup[k].begin(), L.egroup[k].end());
      }
      edge_start[((size_t)q * nA + a) * 17 + 16] = (int32_t)edge.size();
      int32_t * cs = &cls_start[((size_t)q * nA + a) * 33];
      const int32_t base = (int32_t)beams.size();
      for (int k = 0; k < 33; ++k) cs[k] = base + L.cs[k];
      beams.insert(beams.end(), L.beams.begin(), L.beams.end());
      mult.insert(mult.end(), L.mult.begin(), L.mult.end());
    }
    slow_start[(size_t)q * (nA + 1) + nA] = (int32_t)slow.size();
  }
  wrap2_start[(size_t)nq * nA * 4] = (int32_t)wrap2.size();
  // slow_start must be relative to one array: it is (single vector `slow`)
  h2d(S.d_fast_cls, cls_start.data(), cls_start.size(), st);
  S.d_fast_beams.reserve(std::max<size_t>(beams.size(), 1) + 8);
  sweep_stage_h2d(S.d_fast_beams.p, beams.data(), beams.size() * sizeof(uint16_t), st);
  S.d_fast_mult.reserve(std::max<size_t>(mult.size(), 1) + 8);
  sweep_stage_h2d(S.d_fast_mult.p, mult.data(), mult.size() * sizeof(uint16_t), st);
  slow.push_back(0);
  wrap2.push_back(0);
  edge.push_back(0);
  h2d(S.d_fast_edge, edge.data(), edge.size(), st);
  h2d(S.d_fast_edge_start, edge_start.data(), edge_start.size(), st);
  h2d(S.d_fast_wrap2, wrap2.data(), wrap2.size(), st);
  h2d(S.d_fast_wrap2_start, wrap2_start.data(), wrap2_start.size(), st);
  h2d(S.d_fast_slow, slow.data(), slow.size(), st);
  h2d(S.d_fast_slow_start, slow_start.data(), slow_start.size(), st);
  S.fast.enabled = 1;
  S.fast_info[0] = 1; S.fast_info[1] = (int32_t)beams.size(); S.fast_info[2] = n_edge; S.fast_info[3] = (int32_t)slow.size() - 1; S.fast_info[4] = 0;
  S.fast.sub_rows = sub_rows;
  S.fast.xtiles = xtiles;
  S.fast.beams = S.d_fast_beams.p;
  S.fast.mult = S.d_fast_mult.p;
  S.fast.cls_start = S.d_fast_cls.p;
  S.fast.slow = S.d_fast_slow.p;
  S.fast.edge = S.d_fast_edge.p;
  S.fast.edge_start = S.d_fast_edge_start.p;
  S.fast.wrap2 = S.d_fast_wrap2.p;
  S.fast.wrap2_start = S.d_fast_wrap2_start.p;
  S.fast.slow_start = S.d_fast_slow_start.p;
  S.fast_smem = smem;
  {
    int dev = 0, sms = 132;
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    S.fast_blocks = std::min(S.npairs, sms);
  }
  return true;
}

// which kernel an uploaded sweep runs on: 0 = generic (any geometry), 1 = single-CTA fast kernel (BASELINE's 4 m / 12 m
// geometry), 2 = tiled cluster kernel (any even-stride geometry whose raster is order independent)
static int sweep_kernel_choice(const b200sm * h, const SweepHost & S)
{
  if (h->force_generic) return 0;
  const bool fast = S.fast.enabled != 0, tile = S.tile.enabled != 0;
  if (h->sweep_kernel == 1 && fast) return 1;
  if (tile) return 2;
  return fast ? 1 : 0;
}

static int sweep_run(b200sm * h)
{
  NvtxRange nvtx_("b200sm sweep run");
  SweepHost & S = h->sweep;
  if (!S.uploaded) { set_last_error("sweep: nothing uploaded"); return B200_ERR_INVALID_ARG; }
  cudaStream_t st = h->stream;
  const SweepDev & d = S.dev;
  if (S.nitems > 0) {
    // warps (= scans) per CTA: as many as fit the shared-memory staging of their points, at most kFvWarps
    int fvw = (int)std::min<size_t>(kFvWarps, (size_t)200 * 1024 / ((size_t)kFvBytesPerPoint * std::max(S.max_n, 1)));
    if (fvw < 1) { set_last_error("sweep: scan has too many readings for the shared-memory staging of FindValidPoints"); return B200_ERR_UNSUPPORTED; }
    const size_t fv_smem = (size_t)fvw * S.max_n * kFvBytesPerPoint;
    B200_CUDA(cudaFuncSetAttribute(k_find_valid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(fv_smem, 48 * 1024)));
    k_find_valid<<<(S.nitems + fvw - 1) / fvw, fvw * 32, fv_smem, st>>>(d);
    B200_CUDA(cudaGetLastError());
    h->launches++;
  }
  B200_CUDA(cudaEventRecord(S.ev0, st));
  switch (sweep_kernel_choice(h, S)) {
    case 2:
      launch_sweep_tile(h, S, st);
      break;
    case 1:
      B200_CUDA(cudaFuncSetAttribute(k_sweep_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S.fast_smem));
      k_sweep_fast<<<S.fast_blocks, kFastThreads, S.fast_smem, st>>>(d, S.fast);
      break;
    default: {
      const int rows = generic_slice_rows(d.nA, d.n);
      const size_t smem = (size_t)rows * d.n * sizeof(int32_t);
      B200_CUDA(cudaFuncSetAttribute(k_sweep_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_sweep_generic<<<S.blocks, kSweepThreads, smem, st>>>(d, rows);
    }
  }
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaEventRecord(S.ev1, st));
  h->launches++;
  S.ran = true;
  return B200_OK;
}

// A pair whose whole correlation volume is zero (the candidate does not overlap the query's search window): every pose
// ties at response 0, so CorrelateScan averages ALL poses in array order (M.cpp:802-829) and the covariance is the
// "no response" one (M.cpp:886-891).  The result depends on the query's plan only: computed once per query, in the
// reference's summation order (cos / sin of the 21 headings evaluated once each -- same inputs, same libm results).
static void zero_volume_result(const CorrPlan & pl, double mean[3], double cov[9])
{
  std::vector<double> ch(pl.nA), shd(pl.nA);
  for (int a = 0; a < pl.nA; ++a) { ch[a] = cos(pl.heading[a]); shd[a] = sin(pl.heading[a]); }
  double ax = 0.0, ay = 0.0, thetaX = 0.0, thetaY = 0.0;
  for (int y = 0; y < pl.nY; ++y)
    for (int x = 0; x < pl.nX; ++x)
      for (int a = 0; a < pl.nA; ++a) {
        ax += pl.newx[x]; ay += pl.newy[y];
        thetaX += ch[a]; thetaY += shd[a];
      }
  const int icount = pl.nX * pl.nY * pl.nA;
  ax /= icount; ay /= icount; thetaX /= icount; thetaY /= icount;
  mean[0] = ax; mean[1] = ay; mean[2] = atan2(thetaY, thetaX);
  for (int i = 0; i < 9; ++i) cov[i] = 0.0;
  cov[0] = kMaxVariance; cov[4] = kMaxVariance; cov[8] = 4 * square(pl.ang_res);
}

// finish one pair on the host from the device reduction: heading average (libm) + covariance tail
// raster_empty: 1 = no valid point of the pair's chain fell inside the correlation grid (every lookup of every pass is 0),
// 0 = some did, -1 = unknown
static bool finish_query_pair(const b200sm * h, SweepHost & S, int q, const PairOut & o, double * response,
                              double * mean, double * cov, int raster_empty = -1)
{
  const CorrPlan & pl = S.plans[q];
  if (h->p.use_response_expansion && double_equal(o.best, 0.0)) {
    // M.cpp:594-619: up to three more coarse passes with the angle window widened by 20 degrees each.  With an EMPTY raster all
    // of them are zero too, so the result is the all-poses-tie average of the last (widest) pass: closed form, once per query.
    if (raster_empty != 1) return false;   // cells exist: a wider pass could hit them -> single-match path
    if ((int)S.zero_exp_done.size() != S.nq) { S.zero_exp_done.assign(S.nq, 0); S.zero_exp_mean.assign((size_t)3 * S.nq, 0.0); S.zero_exp_cov.assign((size_t)9 * S.nq, 0.0); }
    if (!S.zero_exp_done[q]) {
      double off[2], res[2];
      coarse_search(h, off, res);
      GridGeom g = geom_for_query(h, &S.queries[q]);
      double wide = h->p.coarse_search_angle_offset;
      for (int i = 0; i < 3; ++i) wide += 20 * kPi180;
      CorrPlan px;
      if (build_plan(g, h->probs_side, h->p, &S.queries[q], S.queries[q].sensor_pose, off, res, wide, h->p.coarse_angle_resolution, false, px) != B200_OK)
        return false;
      zero_volume_result(px, &S.zero_exp_mean[3 * (size_t)q], &S.zero_exp_cov[9 * (size_t)q]);
      S.zero_exp_done[q] = 1;
    }
    for (int i = 0; i < 3; ++i) mean[i] = S.zero_exp_mean[3 * (size_t)q + i];
    for (int i = 0; i < 9; ++i) cov[i] = S.zero_exp_cov[9 * (size_t)q + i];
    *response = 0.0;
    S.zero_pairs++;
    return true;
  }
  if (o.best == 0.0 && o.tie_count == pl.nX * pl.nY * pl.nA && o.tie_count > kMaxTies) {
    if ((int)S.zero_done.size() != S.nq) { S.zero_done.assign(S.nq, 0); S.zero_mean.assign((size_t)3 * S.nq, 0.0); S.zero_cov.assign((size_t)9 * S.nq, 0.0); }
    if (!S.zero_done[q]) { zero_volume_result(pl, &S.zero_mean[3 * (size_t)q], &S.zero_cov[9 * (size_t)q]); S.zero_done[q] = 1; }
    for (int i = 0; i < 3; ++i) mean[i] = S.zero_mean[3 * (size_t)q + i];
    for (int i = 0; i < 9; ++i) cov[i] = S.zero_cov[9 * (size_t)q + i];
    *response = 0.0;
    S.zero_pairs++;
    return true;
  }
  if (o.tie_count <= 0 || o.tie_count > kMaxTies) return false;
  double thetaX = 0.0, thetaY = 0.0;
  for (int t = 0; t < o.tie_count; ++t) {   // M.cpp:811-813
    double heading = pl.heading[o.ties[t] % pl.nA];
    thetaX += cos(heading); thetaY += sin(heading);
  }
  thetaX /= o.tie_count; thetaY /= o.tie_count;
  mean[0] = o.avg_x; mean[1] = o.avg_y; mean[2] = atan2(thetaY, thetaX);
  for (int i = 0; i < 9; ++i) cov[i] = 0.0;
  cov[0] = cov[4] = cov[8] = 1.0;   // SetToIdentity, M.cpp:882
  if (o.best < kTolerance) {
    cov[0] = kMaxVariance; cov[4] = kMaxVariance; cov[8] = 4 * square(pl.ang_res);
  } else {
    finish_positional_cov(o.norm, o.acc_xx, o.acc_xy, o.acc_yy, o.best, pl.sp_res, pl.ang_res, cov);
  }
  *response = o.best > 1.0 ? 1.0 : o.best;
  return true;
}

static bool finish_pair(const b200sm * h, SweepHost & S, int pair, const PairOut & o, double * response, double * mean, double * cov,
                        int raster_empty = -1)
{
  return finish_query_pair(h, S, S.pair_query[pair], o, response, mean, cov, raster_empty);
}

static void chain_of_pair(const SweepHost & S, int pair, const b200_scan *& base, int & nbase)
{
  int c = S.pair_chain[pair];
  base = S.scans.data() + S.chain_start[c];
  nbase = S.chain_start[c + 1] - S.chain_start[c];
}

static int sweep_fetch(b200sm * h, bool do_refine, double * response, double * mean, double * cov)
{
  NvtxRange nvtx_("b200sm sweep fetch");
  SweepHost & S = h->sweep;
  if (!S.ran) { set_last_error("sweep: run before fetch"); return B200_ERR_INVALID_ARG; }
  if (!response || !mean || !cov) return B200_ERR_INVALID_ARG;
  cudaStream_t st = h->stream;
  B200_CUDA(cudaMemcpyAsync(S.h_out.p, S.d_out.p, (size_t)S.npairs * sizeof(PairOut), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  S.d2h_bytes += (int64_t)((size_t)S.npairs * sizeof(PairOut));
  std::vector<char> done(S.npairs, 0);
  S.zero_pairs = S.fallback_pairs = 0;
  // response expansion: which zero-response pairs have an empty raster (then the wider passes are zero as well)
  std::vector<int32_t> cell_count;
  std::vector<int32_t> item_start;
  if (h->p.use_response_expansion && S.nitems > 0) {
    bool any_zero = false;
    for (int p = 0; p < S.npairs && !any_zero; ++p) any_zero = double_equal(S.h_out.p[p].best, 0.0);
    if (any_zero) {
      cell_count.resize(S.nitems);
      B200_CUDA(cudaMemcpyAsync(cell_count.data(), S.d_cell_count.p, (size_t)S.nitems * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      S.d2h_bytes += (int64_t)((size_t)S.nitems * sizeof(int32_t));
      item_start.assign(S.npairs + 1, 0);
      for (int p = 0; p < S.npairs; ++p) {
        const int c = S.pair_chain[p];
        item_start[p + 1] = item_start[p] + (S.chain_start[c + 1] - S.chain_start[c]);
      }
    }
  }
  for (int p = 0; p < S.npairs; ++p) {
    int raster_empty = -1;
    if (!cell_count.empty() || (h->p.use_response_expansion && S.nitems == 0)) {
      raster_empty = 1;
      if (!cell_count.empty())
        for (int it = item_start[p]; it < item_start[p + 1]; ++it) if (cell_count[it] > 0) { raster_empty = 0; break; }
    }
    if (!finish_pair(h, S, p, S.h_out.p[p], &response[p], &mean[3 * p], &cov[9 * p], raster_empty)) {
      // tie-list overflow / response expansion: this pair goes through the single-match path
      const b200_scan * base; int nbase;
      chain_of_pair(S, p, base, nbase);
      response[p] = do_match(h, &S.queries[S.pair_query[p]], base, nbase, S.do_penalize, do_refine, &mean[3 * p], &cov[9 * p]);
      done[p] = 1;
      S.fallback_pairs++;
    }
  }
  if (!do_refine) return B200_OK;

  // ---- fine pass (M.cpp:621-629): per-pair plan centred on the coarse mean ----
  const double r = 1.0 / h->g.scale;
  double coff[2], cres[2];
  coarse_search(h, coff, cres);
  double foff[2] = {cres[0] * 0.5, cres[1] * 0.5}, fres[2] = {r, r};
  std::vector<CorrPlan> fp(S.npairs);
  std::vector<GridGeom> fg(S.npairs);
  int P = 0, nA = 0;
  for (int p = 0; p < S.npairs; ++p) {
    const b200_scan * q = &S.queries[S.pair_query[p]];
    fg[p] = geom_for_query(h, q);
    double c2[3] = {mean[3 * p], mean[3 * p + 1], mean[3 * p + 2]};
    if (done[p]) { c2[0] = q->sensor_pose[0]; c2[1] = q->sensor_pose[1]; c2[2] = q->sensor_pose[2]; }   // placeholder plan, result unused
    int rc = build_plan(fg[p], h->probs_side, h->p, q, c2, foff, fres, 0.5 * h->p.coarse_angle_resolution,
                        h->p.fine_search_angle_offset, true, fp[p]);
    if (rc != B200_OK) return rc;
    // every pair's offsets, positions and sums are laid out with pair 0's plan size (the window and the angles are the same for
    // every pair, only the centre differs): a plan of another size would misplace its own and its neighbours' entries
    if (p == 0) {
      P = fp[0].nX * fp[0].nY; nA = fp[0].nA;
    } else if (fp[p].nX != fp[0].nX || fp[p].nY != fp[0].nY || fp[p].nA != nA) {
      set_last_error("sweep: fine plans of one batch differ in size");
      return B200_ERR_UNSUPPORTED;
    }
  }
  const int n = S.n;
  const size_t no = (size_t)S.npairs * nA * n, np = (size_t)S.npairs * P, ns = (size_t)S.npairs * P * nA;
  S.h_i.reserve(no + np + ns);
  for (int p = 0; p < S.npairs; ++p) {
    for (size_t i = 0; i < (size_t)nA * n; ++i) S.h_i.p[(size_t)p * nA * n + i] = device_offset(fp[p].offsets[i], h->g.data_size);
    for (int y = 0; y < fp[p].nY; ++y)
      for (int x = 0; x < fp[p].nX; ++x)
        S.h_i.p[no + (size_t)p * P + (size_t)y * fp[p].nX + x] = fp[p].xs[x] + fp[p].ys[y] * h->g.stride;
  }
  h2d(S.d_fine_off, S.h_i.p, no, st);
  h2d(S.d_fine_pos, S.h_i.p + no, np, st);
  S.d_fine_sums.reserve(ns);
  FineDev f{P, nA, S.d_fine_off.p, S.d_fine_pos.p, S.d_fine_sums.p};
  k_sweep_fine<<<S.blocks, kSweepThreads, 0, st>>>(S.dev, f);
  B200_CUDA(cudaGetLastError());
  h->launches++;
  int32_t * hs = S.h_i.p + no + np;
  B200_CUDA(cudaMemcpyAsync(hs, S.d_fine_sums.p, ns * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  S.d2h_bytes += (int64_t)(ns * sizeof(int32_t));
  B200_CUDA(cudaStreamSynchronize(st));
  for (int p = 0; p < S.npairs; ++p) {
    if (done[p]) continue;
    try {
      response[p] = host_epilogue(h->p, fg[p], h->probs_side, fp[p], hs + (size_t)p * P * nA, S.do_penalize, &mean[3 * p], &cov[9 * p]);
    } catch (const CudaFail & f) {
      if (f.code != B200_ERR_UNSUPPORTED) throw;
      // the averaged fine pose rounded to a cell outside the 3 x 3 searched ones: the single-match path evaluates that cell
      const b200_scan * base; int nbase;
      chain_of_pair(S, p, base, nbase);
      response[p] = do_match(h, &S.queries[S.pair_query[p]], base, nbase, S.do_penalize, true, &mean[3 * p], &cov[9 * p]);
      S.fallback_pairs++;
    }
  }
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200sm_batch_upload(b200sm * h, const b200_scan * queries, int32_t nq, const b200_scan * scans, int32_t nscans,
                        const int32_t * chain_start, int32_t nchains, const int32_t * pair_query,
                        const int32_t * pair_chain, int32_t npairs, int32_t do_penalize)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return sweep_upload(h, queries, nq, scans, nscans, chain_start, nchains, pair_query, pair_chain, npairs, do_penalize != 0);
  B200_GUARD_END
}

int b200sm_batch_run(b200sm * h)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return sweep_run(h);
  B200_GUARD_END
}

int b200sm_batch_fetch(b200sm * h, double * response, double * mean, double * cov)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return sweep_fetch(h, false, response, mean, cov);
  B200_GUARD_END
}

int b200sm_batch_kernel_ms(b200sm * h, float * ms)
{
  B200_GUARD_BEGIN
  if (!h || !ms || !h->sweep.ran) return B200_ERR_INVALID_ARG;
  B200_CUDA(cudaEventSynchronize(h->sweep.ev1));
  B200_CUDA(cudaEventElapsedTime(ms, h->sweep.ev0, h->sweep.ev1));
  return B200_OK;
  B200_GUARD_END
}

int b200sm_batch_best(b200sm * h, int32_t * best_sum, int32_t * best_index, int32_t * tie_count)
{
  B200_GUARD_BEGIN
  if (!h || !h->sweep.ran) return B200_ERR_INVALID_ARG;
  SweepHost & S = h->sweep;
  B200_CUDA(cudaMemcpyAsync(S.h_out.p, S.d_out.p, (size_t)S.npairs * sizeof(PairOut), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  for (int p = 0; p < S.npairs; ++p) {
    if (best_sum) best_sum[p] = S.h_out.p[p].best_sum;
    if (best_index) best_index[p] = S.h_out.p[p].tie_count > 0 ? S.h_out.p[p].ties[0] : -1;
    if (tie_count) tie_count[p] = S.h_out.p[p].tie_count;
  }
  return B200_OK;
  B200_GUARD_END
}

int b200sm_batch_reduce_keys(b200sm * h, void * device_keys, int64_t id_offset)
{
  B200_GUARD_BEGIN
  if (!h || !device_keys || !h->sweep.ran) return B200_ERR_INVALID_ARG;
  SweepHost & S = h->sweep;
  if (S.do_penalize) {
    set_last_error("batch_reduce_keys orders by the integer correlation sum, which is not the response order of a penalised sweep: "
                   "use b200sm_batch_winner_records / b200sm_batch_winners_select");
    return B200_ERR_UNSUPPORTED;
  }
  B200_CUDA(cudaMemsetAsync(device_keys, 0, (size_t)S.nq * sizeof(unsigned long long), h->stream));
  k_best_keys<<<(S.npairs + 255) / 256, 256, 0, h->stream>>>(S.d_out.p, S.d_pair_query.p, S.d_pair_chain.p, S.npairs,
                                                            (long long)id_offset, static_cast<unsigned long long *>(device_keys));
  B200_CUDA(cudaGetLastError());
  h->launches++;
  return B200_OK;
  B200_GUARD_END
}

int32_t b200sm_batch_winner_record_bytes(void) { return (int32_t)sizeof(WinRec); }

int b200sm_batch_winner_records(b200sm * h, void * device_records, int64_t id_offset)
{
  B200_GUARD_BEGIN
  if (!h || !device_records || !h->sweep.ran) return B200_ERR_INVALID_ARG;
  SweepHost & S = h->sweep;
  WinRec * rec = static_cast<WinRec *>(device_records);
  S.d_win_flag.reserve((size_t)S.nq);
  B200_CUDA(cudaMemsetAsync(S.d_win_flag.p, 0, (size_t)S.nq, h->stream));
  const int bq = (S.nq + 255) / 256, bp = (S.npairs + 255) / 256;
  k_win_init<<<bq, 256, 0, h->stream>>>(rec, S.nq);
  k_win_max<<<bp, 256, 0, h->stream>>>(S.d_out.p, S.d_pair_query.p, S.npairs, rec);
  k_win_id<<<bp, 256, 0, h->stream>>>(S.d_out.p, S.d_pair_query.p, S.d_pair_chain.p, S.npairs, (long long)id_offset, rec);
  k_win_copy<<<bp, 256, 0, h->stream>>>(S.d_out.p, S.d_pair_query.p, S.d_pair_chain.p, S.npairs, (long long)id_offset, rec, S.d_win_flag.p);
  k_win_fix<<<bq, 256, 0, h->stream>>>(rec, S.d_win_flag.p, S.nq);
  B200_CUDA(cudaGetLastError());
  h->launches += 5;
  return B200_OK;
  B200_GUARD_END
}

int b200sm_batch_winners_select(b200sm * h, const void * device_gathered, int32_t nranks, int64_t * winner_id, double * response,
                                double * mean, double * cov)
{
  B200_GUARD_BEGIN
  if (!h || !device_gathered || nranks <= 0 || !winner_id || !response || !mean || !cov || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  SweepHost & S = h->sweep;
  const size_t nrec = (size_t)nranks * S.nq;
  std::vector<WinRec> rec(nrec);
  B200_CUDA(cudaMemcpyAsync(rec.data(), device_gathered, nrec * sizeof(WinRec), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  S.d2h_bytes += (int64_t)(nrec * sizeof(WinRec));
  for (int q = 0; q < S.nq; ++q) {
    const WinRec * best = nullptr;
    for (int r = 0; r < nranks; ++r) {
      const WinRec & c = rec[(size_t)r * S.nq + q];
      if (c.gid < 0) continue;
      if (!best || c.resp_bits > best->resp_bits || (c.resp_bits == best->resp_bits && c.gid < best->gid)) best = &c;
    }
    if (!best) {   // no rank had a candidate for this query
      winner_id[q] = -1; response[q] = 0.0;
      for (int i = 0; i < 3; ++i) mean[3 * q + i] = 0.0;
      for (int i = 0; i < 9; ++i) cov[9 * q + i] = 0.0;
      continue;
    }
    winner_id[q] = best->gid;
    if (!finish_query_pair(h, S, q, best->out, &response[q], &mean[3 * q], &cov[9 * q])) {
      set_last_error("winners_select: the winning candidate's tie list overflowed (or needs response expansion); "
                     "fetch the per-candidate results on its owner instead");
      return B200_ERR_UNSUPPORTED;
    }
  }
  return B200_OK;
  B200_GUARD_END
}

int b200sm_batch_info(b200sm * h, int32_t info[8])
{
  if (!h || !info || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  const SweepHost & S = h->sweep;
  const int k = sweep_kernel_choice(h, S);
  for (int i = 0; i < 5; ++i) info[i] = S.fast_info[i];
  info[0] = k;
  if (k == 2) info[4] = 0; else if (k == 0 && S.tile_info[5]) info[4] = 100 + S.tile_info[5];
  info[5] = k == 2 ? S.tile_grid : (k == 1 ? S.fast_blocks : S.blocks);
  info[6] = S.npairs; info[7] = S.nitems;
  return B200_OK;
}

int b200sm_batch_tile_info(b200sm * h, int32_t info[8])
{
  if (!h || !info || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  for (int i = 0; i < 8; ++i) info[i] = h->sweep.tile_info[i];
  return B200_OK;
}

int b200sm_batch_tile_layout(b200sm * h, int32_t layout[4])
{
  if (!h || !layout || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  for (int i = 0; i < 4; ++i) layout[i] = h->sweep.tile_layout[i];
  return B200_OK;
}

int b200sm_batch_tile_stats(b200sm * h, int32_t stats[8])
{
  if (!h || !stats || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  for (int i = 0; i < 8; ++i) stats[i] = h->sweep.tile_stats[i];
  return B200_OK;
}

int b200sm_batch_fetch_stats(b200sm * h, int32_t stats[4])
{
  if (!h || !stats) return B200_ERR_INVALID_ARG;
  stats[0] = h->sweep.zero_pairs; stats[1] = h->sweep.fallback_pairs; stats[2] = h->sweep.npairs; stats[3] = 0;
  return B200_OK;
}

int b200sm_batch_upload_timing(b200sm * h, double out[3])
{
  if (!h || !out) return B200_ERR_INVALID_ARG;
  for (int i = 0; i < 3; ++i) out[i] = h->sweep.upload_ms[i];
  return B200_OK;
}

int b200sm_batch_transfer_bytes(b200sm * h, int64_t * h2d_bytes, int64_t * d2h_bytes, int32_t reset)
{
  if (!h) return B200_ERR_INVALID_ARG;
  if (h2d_bytes) *h2d_bytes = h->sweep.h2d_bytes;
  if (d2h_bytes) *d2h_bytes = h->sweep.d2h_bytes;
  if (reset) h->sweep.h2d_bytes = h->sweep.d2h_bytes = 0;
  return B200_OK;
}

int b200sm_match_batch(b200sm * h, const b200_scan * queries, int32_t nq, const b200_scan * scans, int32_t nscans,
                       const int32_t * chain_start, int32_t nchains, const int32_t * pair_query,
                       const int32_t * pair_chain, int32_t npairs, int32_t do_penalize, int32_t do_refine,
                       double * response, double * mean, double * cov)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  int rc = sweep_upload(h, queries, nq, scans, nscans, chain_start, nchains, pair_query, pair_chain, npairs, do_penalize != 0);
  if (rc != B200_OK) return rc;
  rc = sweep_run(h);
  if (rc != B200_OK) return rc;
  return sweep_fetch(h, do_refine != 0, response, mean, cov);
  B200_GUARD_END
}

}  // extern "C"
