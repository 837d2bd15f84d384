// b200slam scan matcher, batched loop-closure sweep: the generic kernel, the host side and the batch C ABI.
//
// Reference: MapperGraph::TryCloseLoop (lib/karto_sdk/src/Mapper.cpp:1500-1561) calls
// ScanMatcher::MatchScan once per candidate chain; here every (query, chain) pair of a sweep is
// rasterised, correlated and reduced on the device in one fused kernel launch.
//   k_find_valid     FindValidPoints + WorldToGrid + ROI test per (pair, scan)  (M.cpp:1073-1164)
//   k_sweep_generic  per pair: clear + smear raster, exhaustive correlation, arg-max / ties /
//                    positional-covariance accumulators                          (M.cpp:641-966)
//   k_sweep_fine     3x3xnA fine volumes for do_refine                           (M.cpp:621-629)
//   k_best_keys, k_win_*  per-query keys / winner records of the multi-GPU sweep
// The host side uploads a sweep, chooses its kernel once (the parity-sub-grid kernels live in sm_fast.cu and
// sm_tile.cu), runs it and finishes the pairs.
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
// batch sweep, generic kernel
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

// Grid::Clear (M.cpp:1034) of a CTA's workspace grid
__device__ __forceinline__ void clear_grid(const SweepDev & d, uint8_t * grid)
{
  uint4 * g4 = reinterpret_cast<uint4 *>(grid);
  const int n16 = d.data_size / 16;
  for (int i = threadIdx.x; i < n16; i += blockDim.x) g4[i] = make_uint4(0, 0, 0, 0);
  for (int i = n16 * 16 + threadIdx.x; i < d.data_size; i += blockDim.x) grid[i] = 0;
}

// AddScan's smear (M.cpp:1080-1104) of the valid points of items [it0, it1) into a workspace grid: every tap max-stamps its cell.
// Cells < 0 are points the order-dependent replay dropped.  half = ksize / 2 and taps = ksize^2 come from the caller, which
// computes them once per CTA.
__device__ __forceinline__ void stamp_cells(const SweepDev & d, uint8_t * grid, int it0, int it1, int half, int taps)
{
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
    clear_grid(d, grid);
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
    stamp_cells(d, grid, it0, it1, half, taps);
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
    clear_grid(d, grid);
    __syncthreads();
    const int it0 = d.pair_item_start[pair], it1 = d.pair_item_start[pair + 1];
    // cells dropped by AddScan's occupancy test were marked < 0 by the coarse pass: plain max-stamp
    stamp_cells(d, grid, it0, it1, half, taps);
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

// Host -> device copy of a small table through the sweep's pinned arena: the source may be reused or freed as soon as this
// returns and nothing blocks, so the host keeps building tables while the candidate points are still in flight.
void SweepHost::stage(void * dst, const void * src, size_t bytes, cudaStream_t s)
{
  if (!bytes) return;
  const size_t need = (bytes + 63) & ~(size_t)63;
  if (arena_used + need <= arena.cap) {
    unsigned char * slot = arena.p + arena_used;
    arena_used += need;
    std::memcpy(slot, src, bytes);
    B200_CUDA(cudaMemcpyAsync(dst, slot, bytes, cudaMemcpyHostToDevice, s));
  } else {
    B200_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
    B200_CUDA(cudaStreamSynchronize(s));   // arena exhausted: plain copy, the source may go away after return
  }
  h2d_bytes += (int64_t)bytes;
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

// whole angle rows of the lookup table per slice of the generic kernel: all nA when the table fits (one slice, staged once
// per query), else as many as fit
static int generic_slice_rows(int nA, int n)
{
  const size_t row = (size_t)n * sizeof(int32_t);
  return (int)std::min<size_t>((size_t)nA, kLookupSmemBytes / row);
}

static int sweep_upload(b200sm * h, const b200_scan * queries, int nq, const b200_scan * scans, int nscans,
                        const int32_t * chain_start, int nchains, const int32_t * pair_query,
                        const int32_t * pair_chain, int npairs, bool do_penalize)
{
  NvtxRange nvtx_("b200sm sweep upload");
  const auto t_enter = std::chrono::steady_clock::now();
  SweepHost & S = h->sweep;
  S.uploaded = S.ran = false;
  S.zero.done.clear(); S.zero_exp.done.clear();
  // readouts of the kernel choice: the builder that succeeds fills in its own.  The builders' refusal codes (tile_refusal,
  // fast_refusal) stay until that builder runs again.
  S.kernel = kSweepGeneric; S.refused_reason = 0;
  S.fast.enabled = 0; S.tile.enabled = 0;
  std::fill(S.beam_counts, S.beam_counts + 3, 0);
  S.tile_plan = TilePlan{}; S.tile_clusters = 0; S.tile_stats = TileStats{};
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
  if ((size_t)n * sizeof(int32_t) > kLookupSmemBytes) {
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
    for (int q = 0; q < nq; ++q) device_plan(S.plans[q], g0, S.h_i.p + (size_t)q * nA * n, S.h_i.p + no + (size_t)q * P);
    S.h2d(S.d_offsets, S.h_i.p, no, st);
    S.h2d(S.d_posidx, S.h_i.p + no, np, st);
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
    S.h2d(S.d_qd, S.h_d.p, per * nq, st);
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
    S.h2d(S.d_scan_pt_start, a_pt, nscans + 1, st);
    S.h2d(S.d_pair_query, a_pq, npairs, st);
    S.h2d(S.d_pair_chain, S.pair_chain.data(), npairs, st);
    S.h2d(S.d_pair_item_start, a_pis, npairs + 1, st);
    S.h2d(S.d_item_pair, a_ip, std::max(nitems, 1), st);
    S.h2d(S.d_item_scan, a_is, std::max(nitems, 1), st);
  }
  S.d_cells.reserve((size_t)std::max(nitems, 1) * S.max_n);
  S.d_cell_count.reserve(std::max(nitems, 1));
  if (S.d_kernel.cap == 0) S.h2d(S.d_kernel, g0.kernel.data(), g0.kernel.size(), st);

  // ---- workspaces: one per resident CTA ----
  const size_t smem = (size_t)generic_slice_rows(nA, n) * n * sizeof(int32_t);
  const int per_sm = smem <= 100 * 1024 ? 2 : 1;
  S.blocks = std::min(npairs, h->sms * per_sm);
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
  // The kernel is chosen here, once, and only its tables are built: the tiled cluster kernel (any geometry with an even stride and
  // an order-independent raster) is the default everywhere.  With the atomic-free levelled raster it is ahead of the single-CTA
  // kernel on that kernel's own geometry too (on an H100, 400 W power limit: 387 k vs 273 k matches/s at cfg2, bench.py); the
  // single-CTA kernel takes what the tiled planner refuses, and "sweep_kernel" = 1 selects it first.  Anything else runs on the
  // generic kernel.
  const auto t_tab0 = std::chrono::steady_clock::now();
  if (!h->force_generic) {
    if (h->sweep_kernel == 1 && build_fast_tables(h, S, st)) S.kernel = kSweepFast;
    else if (build_tile_tables(h, S, st)) S.kernel = kSweepTile;
    else if (h->sweep_kernel != 1 && build_fast_tables(h, S, st)) S.kernel = kSweepFast;
    else S.refused_reason = S.tile_refusal ? 100 + S.tile_refusal : S.fast_refusal;
  }
  const auto t_tab1 = std::chrono::steady_clock::now();
  auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  S.upload_ms[0] = ms(t_plans0, t_plans1); S.upload_ms[1] = ms(t_tab0, t_tab1); S.upload_ms[2] = ms(t_enter, t_tab1);
  S.uploaded = true;
  return B200_OK;
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
  // "force_generic_sweep" set after the upload still takes effect: the generic kernel needs no tables of its own
  switch (h->force_generic ? kSweepGeneric : S.kernel) {
    case kSweepTile:
      launch_sweep_tile(S, st);
      break;
    case kSweepFast:
      launch_sweep_fast(S, st);
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

// Copies query q's entry of the cache to mean / cov, evaluating it first with compute(mean, cov) (false: it cannot be evaluated)
template <class F>
static bool cached_zero_result(ZeroCache & c, int nq, int q, F compute, double * mean, double * cov)
{
  if ((int)c.done.size() != nq) { c.done.assign(nq, 0); c.mean.assign((size_t)3 * nq, 0.0); c.cov.assign((size_t)9 * nq, 0.0); }
  if (!c.done[q]) {
    if (!compute(&c.mean[3 * (size_t)q], &c.cov[9 * (size_t)q])) return false;
    c.done[q] = 1;
  }
  for (int i = 0; i < 3; ++i) mean[i] = c.mean[3 * (size_t)q + i];
  for (int i = 0; i < 9; ++i) cov[i] = c.cov[9 * (size_t)q + i];
  return true;
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
    auto widest = [&](double * m, double * c) {
      double off[2], res[2];
      coarse_search(h, off, res);
      GridGeom g = geom_for_query(h, &S.queries[q]);
      double wide = h->p.coarse_search_angle_offset;
      for (int i = 0; i < 3; ++i) wide += 20 * kPi180;
      CorrPlan px;
      if (build_plan(g, h->probs_side, h->p, &S.queries[q], S.queries[q].sensor_pose, off, res, wide, h->p.coarse_angle_resolution, false, px) != B200_OK)
        return false;
      zero_volume_result(px, m, c);
      return true;
    };
    if (!cached_zero_result(S.zero_exp, S.nq, q, widest, mean, cov)) return false;
    *response = 0.0;
    S.zero_pairs++;
    return true;
  }
  if (o.best == 0.0 && o.tie_count == pl.nX * pl.nY * pl.nA && o.tie_count > kMaxTies) {
    cached_zero_result(S.zero, S.nq, q, [&](double * m, double * c) { zero_volume_result(pl, m, c); return true; }, mean, cov);
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
    if (!finish_query_pair(h, S, S.pair_query[p], S.h_out.p[p], &response[p], &mean[3 * p], &cov[9 * p], raster_empty)) {
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
  for (int p = 0; p < S.npairs; ++p) device_plan(fp[p], h->g, S.h_i.p + (size_t)p * nA * n, S.h_i.p + no + (size_t)p * P);
  S.h2d(S.d_fine_off, S.h_i.p, no, st);
  S.h2d(S.d_fine_pos, S.h_i.p + no, np, st);
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
  info[0] = S.kernel;
  for (int i = 0; i < 3; ++i) info[1 + i] = S.beam_counts[i];
  info[4] = S.refused_reason;
  info[5] = S.kernel == kSweepTile ? S.tile_clusters * S.tile_plan.C : (S.kernel == kSweepFast ? S.fast_blocks : S.blocks);
  info[6] = S.npairs; info[7] = S.nitems;
  return B200_OK;
}

int b200sm_batch_tile_info(b200sm * h, int32_t info[8])
{
  if (!h || !info || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  const SweepHost & S = h->sweep;
  const TilePlan & p = S.tile_plan;
  info[0] = S.tile.enabled; info[1] = p.C; info[2] = p.V; info[3] = p.nbands; info[4] = p.band_rows; info[5] = S.tile_refusal;
  info[6] = S.tile_clusters; info[7] = (int32_t)(p.smem / 1024);
  return B200_OK;
}

int b200sm_batch_tile_layout(b200sm * h, int32_t layout[4])
{
  if (!h || !layout || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  const TilePlan & p = h->sweep.tile_plan;
  layout[0] = p.ytile_rows; layout[1] = p.ytiles; layout[2] = p.xtiles; layout[3] = p.tail;
  return B200_OK;
}

int b200sm_batch_tile_stats(b200sm * h, int32_t stats[8])
{
  if (!h || !stats || !h->sweep.uploaded) return B200_ERR_INVALID_ARG;
  static_assert(sizeof(TileStats) == 8 * sizeof(int32_t), "TileStats holds the 8 stats in their ABI order");
  std::memcpy(stats, &h->sweep.tile_stats, sizeof(TileStats));
  return B200_OK;
}

int b200sm_tile_plan(const int32_t in[13], int32_t out[7])
{
  if (!in || !out) return B200_ERR_INVALID_ARG;
  // the grid, window, beams, batch and SMs positive (max_n, do_penalize, cluster, chunks and tail may be 0); the window small
  // enough that the planner's byte counts stay in int
  for (int i = 0; i < 13; ++i)
    if (in[i] < (i == 6 || i == 7 || i >= 10 ? 0 : 1) || in[i] > (i == 2 || i == 3 ? 2048 : 1 << 20)) return B200_ERR_INVALID_ARG;
  const TilePlan p = plan_tile(TilePlanIn{in[0], in[1], in[2], in[3], in[4], in[5], in[6], in[7], in[8], in[9], in[10], in[11], in[12]});
  const int32_t v[7] = {p.refused, p.C, p.V, p.nbands, p.band_rows, (int32_t)p.smem, p.tail};
  std::copy(v, v + 7, out);
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
