// b200slam scan matcher, batched loop-closure sweep: the TILED CLUSTER kernel.
//
// Reference path: ScanMatcher::MatchScan -> CorrelateScan -> operator()(y) -> GetResponse
// (lib/karto_sdk/src/Mapper.cpp:534-1208, "M.cpp"), called once per candidate chain by
// MapperGraph::TryCloseLoop (M.cpp:1500-1561).
//
// k_sweep_fast (sm_fast.cu) keeps one parity sub-grid and the whole (x, y, theta) accumulator volume of
// a pair in ONE SM's shared memory, which only holds for BASELINE's 4 m / 12 m geometry.  This kernel lifts
// both limits so that the reference's shipped geometries (loop_search_space_dimension 8 m -> 81 x 81 x 21
// poses = 551 KB of accumulators; max_laser_range 20 m -> 881..965-cell grids) run on the same word-load
// scheme:
//   * the pose volume is cut into V angle CHUNKS; a thread-block CLUSTER of C CTAs shares one pair and CTA r
//     owns chunks r, r + C, ... (perfectly balanced: every angle has the same beams);
//   * the parity sub-grid is cut into row BANDS (band rows + a halo of one pose-window height), one band is
//     resident at a time, beams are grouped by (angle, parity phase, band, alignment);
//   * the beam-descriptor block of every (chunk, phase, band) STAGE is streamed into shared memory by
//     cp.async.bulk (TMA, 1-D) completing on an mbarrier, double buffered: the block of stage s + 1 lands
//     while stage s is being correlated; the hot loop reads descriptors with broadcast LDS.64;
//   * warp items (angle, x-tile, y-tile, alignment) come from a dynamic shared-memory queue;
//   * the reduction (CorrelateScan M.cpp:775-829, ComputePositionalCovariance M.cpp:893-933) is distributed:
//     every CTA reduces its chunks to (best, tie list, per-cell max image), the images and tie lists are
//     combined through DISTRIBUTED SHARED MEMORY by a leader CTA that rotates from pair to pair, and a split
//     cluster barrier (arrive ... wait) lets the other CTAs start the next pair while the leader runs the
//     order-preserving (sequential) covariance sums.
// Integer sums are exact in any order, the FP64 parts keep the reference's operation order: results are bit
// identical to the reference (tests/test_matcher_gpu.py).
// Compile with -fmad=false / -ffp-contract=off.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "sm_math.cuh"
#include "sm_types.cuh"
#include "sm_device.cuh"
#include "sm_sweep_dev.cuh"

namespace b200 {

constexpr int kRowTiles = 6;           // register pairs of 16-bit fields per thread: six row tiles of 8 rows (48-row y-tiles), or
                                       // five (40-row y-tiles) + the tail row nY - 1 (see k_sweep_tile)
constexpr int kChunkBeams = 640;       // beams accumulated in 16-bit fields before a flush (640 * 100 < 65536)
constexpr int kMaxSingles = 63;        // weighted singles of one item (6-bit field of the item record, sm_types.cuh)
constexpr int kMaxPairs = 255;         // weighted pairs of one item (8-bit field)
// guard words before / after the accumulator volume A: the flush adds zero to columns -3 .. 16 * xtiles - 1 <= nX + 17 of a row, so
// the first row reaches 3 words before A and the last row 18 words past it
constexpr int kAGuardLo = 4;
constexpr int kAGuardHi = 20;

// ------------------------------------------------------------------------------------------
// PTX helpers: mbarrier, bulk async copy (TMA 1-D), cluster barrier, distributed shared memory
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void * src, uint32_t bytes, uint32_t bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
  uint32_t done = 0;
  while (!done) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  }
}
__device__ __forceinline__ uint32_t cluster_rank()
{
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t dsmem_addr(const void * local, uint32_t rank)
{
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(local)), "r"(rank));
  return r;
}
__device__ __forceinline__ void dsmem_st_f64(uint32_t a, double v) { asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
__device__ __forceinline__ void dsmem_st_s32(uint32_t a, int v) { asm volatile("st.shared::cluster.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ int dsmem_ld_s32(uint32_t a)
{
  int v;
  asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ double dsmem_ld_f64(uint32_t a)
{
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
  return v;
}

// 32-bit shared-memory load from a shared-window byte address (keeps the window base folded into the per-lane base register)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a)
{
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}

// shared-memory reduction without a result.  The flush issues it unconditionally: ptxas wraps every lane-dependent shared atomic,
// predicated PTX included, in a BSSY / BRA / BSYNC region of its own
__device__ __forceinline__ void red_add(uint32_t a, uint32_t v)
{
  asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}

// Wrapped-word accumulation.  The item loops add every loaded word whole into Tw and only its odd bytes into To (uint32, mod
// 2^32).  Every word is w = even(w) + (odd(w) << 8) with even(w) = [b0, 0, b2, 0], and k * w = k * even(w) + ((k * odd(w)) << 8)
// mod 2^32, so Tw - (To << 8) is the sum of the even bytes mod 2^32 -- the even-field word E the loops would form by extracting
// both halves -- for any words and weights.  One byte extract per loaded word instead of two.  (That E and To hold their 16-bit
// fields without carries is the item's weight cap, kChunkBeams beams of cell values <= 100, as before.)
__device__ __forceinline__ uint32_t odd_bytes_t(uint32_t w) { return __byte_perm(w, 0, 0x4341); }    // [b1, 0, b3, 0]
__device__ __forceinline__ uint32_t even_fields(uint32_t tw, uint32_t to) { return tw - (to << 8); } // [sum b0 | sum b2]

// best / tie summary of a set of poses (one chunk, one CTA, or the whole pair)
struct TieRes {
  double L;        // best response
  double L2;       // highest chunk best strictly below L (ambiguity test: DoubleEqual(L2, L) -> the host decides)
  int cnt;         // number of poses with DoubleEqual(response, L)
  int sum0;        // integer sum of the first tie
  int ties[kMaxTies];
};

// folds b into a (both lists ascending in the flat pose index)
__device__ void tie_merge(TieRes & a, const double bL, const double bL2, const int bcnt, const int bsum0, const int * bties)
{
  if (bL == a.L) {
    int out[kMaxTies];
    const int na = a.cnt < kMaxTies ? a.cnt : kMaxTies, nb = bcnt < kMaxTies ? bcnt : kMaxTies;
    int i = 0, j = 0, k = 0;
    while (k < kMaxTies && (i < na || j < nb)) {
      if (j >= nb || (i < na && a.ties[i] < bties[j])) out[k++] = a.ties[i++];
      else out[k++] = bties[j++];
    }
    if (nb > 0 && (na == 0 || bties[0] < a.ties[0])) a.sum0 = bsum0;
    for (int t = 0; t < k; ++t) a.ties[t] = out[t];
    a.cnt += bcnt;
    a.L2 = bL2 > a.L2 ? bL2 : a.L2;
  } else if (bL > a.L) {
    double l2 = a.L > a.L2 ? a.L : a.L2;
    l2 = bL2 > l2 ? bL2 : l2;
    a.L = bL; a.L2 = l2; a.cnt = bcnt; a.sum0 = bsum0;
    const int nb = bcnt < kMaxTies ? bcnt : kMaxTies;
    for (int t = 0; t < nb; ++t) a.ties[t] = bties[t];
  } else {
    double l2 = bL > a.L2 ? bL : a.L2;
    a.L2 = bL2 > l2 ? bL2 : l2;
  }
}

struct TileShared {
  unsigned long long bar[4];       // [0..1] descriptor staging buffers, [2..3] cell-list staging buffers
  uint8_t kern[256];               // the smear kernel's taps (when ksize^2 <= 256)
  int ctr[2];
  double dscratch[32];
  int iscratch[32];
  TieRes chunk;                    // result of the chunk just reduced
  TieRes res;                      // this CTA's running result over its chunks
  // written by the other CTAs of the cluster when this CTA is the pair's leader
  double rankL[kTileMaxCluster], rankL2[kTileMaxCluster];
  int rankCnt[kTileMaxCluster], rankSum0[kTileMaxCluster];
  int rankTies[kTileMaxCluster][kMaxTies];
  double avg[2];
  double acc[4];
  int ok;
};
// The planner's shared-memory budget subtracts this size, and tests/tile_plan_rule.py restates the planner with it: a change here
// changes plans, so it has to be made in both places.
static_assert(sizeof(TileShared) == 1936, "TileShared changed size: update the planner restatement in tests/tile_plan_rule.py");

// ------------------------------------------------------------------------------------------
// section timers (build with -DB200_TILE_TIMERS, tools/tile_timers.py): lane 0 of every warp accumulates clock64() deltas
// per section and adds them to g_tile_timers at the end of the kernel.  Compiled out of the shipped library.
// ------------------------------------------------------------------------------------------
#ifdef B200_TILE_TIMERS
enum { kTmRaster, kTmDesc, kTmCorr, kTmFlush, kTmBarrier, kTmReduce, kTmPair, kTmTotal, kTmCount };
__device__ unsigned long long g_tile_timers[kTmCount];
#define TILE_TM_DECL                              \
  unsigned long long tm_acc[kTmCount] = {};       \
  long long tm_t = clock64();                     \
  const long long tm_start = tm_t;
#define TILE_TM(sec)                                                      \
  do {                                                                    \
    const long long tm_now = clock64();                                   \
    tm_acc[sec] += (unsigned long long)(tm_now - tm_t);                   \
    tm_t = tm_now;                                                        \
  } while (0)
#define TILE_TM_END                                                                 \
  do {                                                                              \
    TILE_TM(kTmPair);                                                               \
    tm_acc[kTmTotal] = (unsigned long long)(tm_t - tm_start);                       \
    if (lane == 0)                                                                  \
      for (int s = 0; s < kTmCount; ++s) atomicAdd(&g_tile_timers[s], tm_acc[s]);   \
  } while (0)
#else
#define TILE_TM_DECL
#define TILE_TM(sec) do {} while (0)
#define TILE_TM_END do {} while (0)
#endif
// loop-trip counters (build with -DB200_TILE_COUNTS, tools/tile_loop_account.py): lane 0 of every warp counts the items, the
// flushes that reduce something and the trips of each correlation loop (lane 0 is lane-row 0, which runs the most tail-row trips,
// so its count is the warp's).  Kept apart from the section timers: the counting itself costs correlation cycles.
#ifdef B200_TILE_COUNTS
enum { kCnItem, kCnFlush, kCnPlain4, kCnPlain2, kCnPlain1, kCnSingle, kCnPair, kCnTailPlain, kCnTailSingle, kCnTailPair, kCnEdge,
       kCnCount };
__device__ unsigned long long g_tile_counts[kCnCount];
#define TILE_CN_DECL unsigned long long cn_acc[kCnCount] = {};
#define TILE_CN(k) (++cn_acc[k])
#define TILE_CN_END                                                                \
  do {                                                                             \
    if (lane == 0)                                                                 \
      for (int s = 0; s < kCnCount; ++s) atomicAdd(&g_tile_counts[s], cn_acc[s]); \
  } while (0)
#else
#define TILE_CN_DECL
#define TILE_CN(k) do {} while (0)
#define TILE_CN_END do {} while (0)
#endif

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
// kPitchW = the sub-grid row pitch in words as a compile-time constant (0 = take it from TileDev): with a constant pitch the 24
// loads of a 4-beam step address as [descriptor register + immediate]; with a run-time pitch every load costs an extra IMAD
// (20 % of the beam loop).  The pitches of the four shipped geometry combinations are instantiated.
// kTail = the y-tile layout (TileDev.tail): false = 48-row y-tiles of six row tiles; true = 40-row y-tiles of five row tiles, and in
// the last y-tile the sixth register pair holds the tail row nY - 1, read lane-parallel over the entries (lane-row y_l takes every
// 8th entry from the y_l-th on) and summed over the lane-rows at the flush.  A 2k + 1-row window (41, 81) then loads 40 k rows + an
// eighth of a row per entry instead of 48 * ceil((2k + 1) / 48) rows.
// f is __grid_constant__: the raster indexes its tap masks by the level at run time, which then reads the parameter bank instead
// of a per-thread copy of TileDev.
template <int kPitchW, bool kTail>
__global__ void __launch_bounds__(kTileThreads, 1) k_sweep_tile(SweepDev d, const __grid_constant__ TileDev f)
{
  constexpr int kMain = kTail ? kRowTiles - 1 : kRowTiles;   // row tiles of 8 rows per y-tile
  constexpr int kYTile = 8 * kMain;
  extern __shared__ __align__(128) unsigned char s_raw[];
  __shared__ TileShared sh;
  uint32_t * S = reinterpret_cast<uint32_t *>(s_raw);
  uint8_t * S8 = s_raw;
  int32_t * A = reinterpret_cast<int32_t *>(s_raw + f.off_A);
  double * probs = reinterpret_cast<double *>(s_raw + f.off_probs);      // per-cell max response image (FP64 path) ...
  int32_t * iprobs = reinterpret_cast<int32_t *>(s_raw + f.off_probs);   // ... or per-cell max integer sum (integer path: half the bytes)
  const int C = f.C;
  const uint32_t rank = C > 1 ? cluster_rank() : 0u;
  const int cluster_id = blockIdx.x / C, nclusters = gridDim.x / C;
  const int nX = d.nX, nY = d.nY, nA = d.nA, P = nX * nY;
  const int half = d.ksize / 2, taps = d.ksize * d.ksize;
  const int tid = threadIdx.x, lane = tid & 31;
  const int y_l = lane >> 2, j_l = lane & 3;
  const int pitch_w = kPitchW ? kPitchW : f.pitch_w, pitchB = pitch_w * 4;
  const int sub_words = f.alloc_rows * pitch_w;
  const int nb = f.nbands;
  const uint32_t bar0 = smem_u32(&sh.bar[0]);
  const uint32_t stg0 = smem_u32(s_raw + f.off_stage);
  TILE_TM_DECL
  TILE_CN_DECL

  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    mbar_init(bar0 + 16, 1);
    mbar_init(bar0 + 24, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    sh.ctr[0] = 0; sh.ctr[1] = 0;
  }
  const bool kern_smem = taps <= 256;
  if (kern_smem && tid < taps) sh.kern[tid] = d.kern[tid];
  const uint8_t * kern = kern_smem ? sh.kern : d.kern;
  __syncthreads();
  if (C > 1) { cluster_arrive(); cluster_wait(); }   // every CTA of the cluster is running before any remote access

  uint32_t cnt = 0;          // descriptor blocks consumed so far (buffer = cnt & 1, mbarrier parity = (cnt >> 1) & 1)
  bool pending_wait = false; // a cluster barrier arrive without its wait yet (split barrier across pairs)
  auto issue = [&](const TileSeq * e, uint32_t buf) {
    mbar_expect_tx(bar0 + 8 * buf, (uint32_t)e->bytes);
    bulk_g2s(stg0 + buf * (uint32_t)f.stage_bytes, f.desc + e->off, (uint32_t)e->bytes, bar0 + 8 * buf);
  };
  // the valid-point cells of a pair's FIRST scan (what every stage's raster reads: 4.3 KB for 1081 beams) are staged in shared
  // memory by a bulk copy too, one pair ahead -- a stage then starts without a global-memory round trip
  const uint32_t cel0 = smem_u32(s_raw + f.off_cells);
  const uint32_t cell_bytes = (uint32_t)f.cell_cap * 4u;
  auto issue_cells = [&](int pr, uint32_t buf) {
    const int it = min(d.pair_item_start[pr], max(d.nitems - 1, 0));
    mbar_expect_tx(bar0 + 16 + 8 * buf, cell_bytes);
    bulk_g2s(cel0 + buf * cell_bytes, d.cells + (size_t)it * d.max_n, cell_bytes, bar0 + 16 + 8 * buf);
  };
  if (cluster_id < d.npairs && tid == 0) {
    const int q0 = d.pair_query[cluster_id];
    issue(f.seq + f.seq_start[q0 * C + rank], 0);
    if (f.cell_cap) issue_cells(cluster_id, 0);
  }

  int iter = 0;
  for (int pair = cluster_id; pair < d.npairs; pair += nclusters, ++iter) {
    const int q = d.pair_query[pair];
    const uint32_t leader = (uint32_t)(iter % C);
    const TileSeq * seq = f.seq + f.seq_start[q * C + rank];
    const int nseq = f.seq_start[q * C + rank + 1] - f.seq_start[q * C + rank];
    const int it0 = d.pair_item_start[pair], it1 = d.pair_item_start[pair + 1];
    bool first_chunk = true;
    const int32_t * cells0 = d.cells + (size_t)it0 * d.max_n;
    const int ncell0 = it0 < it1 ? d.cell_count[it0] : 0;   // read once per pair, not once per stage
    if (f.cell_cap) {
      if (tid == 0 && pair + nclusters < d.npairs) issue_cells(pair + nclusters, (uint32_t)((iter + 1) & 1));
      mbar_wait(bar0 + 16 + 8 * (iter & 1), (uint32_t)((iter >> 1) & 1));
      cells0 = reinterpret_cast<const int32_t *>(s_raw + f.off_cells + (size_t)(iter & 1) * cell_bytes);
    }
    TILE_TM(kTmPair);

    for (int si = 0; si < nseq; ++si) {
      const TileSeq e = seq[si];
      const int chunk_a0 = e.chunk * f.nAc;
      const int chunk_na = min(f.nAc, nA - chunk_a0);
      const int ph = e.stage / nb, band = e.stage - ph * nb;
      const int pp = ph & 1, pq = ph >> 1;
      const int band_r0 = band * f.band_rows;
      const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
      if (e.flags & kSeqNewChunk) {
        // A is 16-byte aligned (16 bytes behind the 16-byte aligned sub-grid); chunk_na * P need not be a multiple of 4
        const int na = chunk_na * P, na4 = na >> 2;
        uint4 * A4 = reinterpret_cast<uint4 *>(A);
        for (int i = tid; i < na4; i += kTileThreads) A4[i] = zero4;
        if (tid < (na & 3)) A[4 * na4 + tid] = 0;
      }
      if ((e.flags & (kSeqNewStage | kSeqKeepGrid)) == kSeqNewStage) {
        {
          uint4 * S4 = reinterpret_cast<uint4 *>(s_raw);
          for (int i = tid; i < (sub_words >> 2); i += kTileThreads) S4[i] = zero4;   // pitch_w is a multiple of 4
        }
        __syncthreads();
        // ---- raster: taps landing on (pp, pq) cells of this band (AddScan / SmearPoint, M.cpp:1080-1104, M.h:1152-1183) ----
        // Max-stamp without atomics when the kernel has few distinct values (3 x 3: {6, 25, 100}): one pass per value in ascending
        // order, plain byte stores (all writers of a pass store the same value, a later pass overwrites with a larger one), a
        // barrier between passes.  Neighbouring beams end in neighbouring cells, so a CAS loop on the shared 32-bit words
        // serialises up to 8 lanes per word; kernels with more values keep it.
        const int nlev = f.nlevels;
        if (f.tap_masks) {
          // one thread per valid point: the pass's four class masks are warp-uniform parameter loads, a point selects its class's
          // mask and stores one byte per set bit.  No table load and no compare per tap, and no tap is visited in a pass that
          // does not store it.  (On H100 a raster still takes about as long as with the per-tap loop below: DESIGN.md §3.3)
          for (int lv = 0; lv < nlev; ++lv) {
            const uint8_t want = (uint8_t)f.level[lv];
            const unsigned long long m0 = f.tap_mask[lv][0], m1 = f.tap_mask[lv][1], m2 = f.tap_mask[lv][2], m3 = f.tap_mask[lv][3];
            for (int it = it0; it < it1; ++it) {
              const int32_t * cl = it == it0 ? cells0 : d.cells + (size_t)it * d.max_n;
              const int ncell = it == it0 ? ncell0 : d.cell_count[it];
              for (int t = tid; t < ncell; t += kTileThreads) {
                const int32_t cell = cl[t];
                if (cell < 0) continue;
                const int cx = (cell & 0xFFFF) + d.roi_x - half, cy = (cell >> 16) + d.roi_y - half;
                const int ky0 = (cy ^ pq) & 1, kx0 = (cx ^ pp) & 1;
                unsigned long long m = ky0 ? (kx0 ? m3 : m2) : (kx0 ? m1 : m0);
                const int rel0 = ((cy + ky0) >> 1) - band_r0, col0 = (cx + kx0) >> 1;
                while (m) {
                  const int b = __ffsll((long long)m) - 1;
                  m &= m - 1;
                  const int rel = rel0 + (b >> 3);
                  if ((unsigned)rel < (unsigned)f.alloc_rows) S8[rel * pitchB + col0 + (b & 7)] = want;
                }
              }
            }
            if (lv + 1 < nlev) __syncthreads();
          }
        } else {
          // one thread per valid point, every kernel row / column of this phase's parity
          for (int lv = 0; lv < (nlev > 0 ? nlev : 1); ++lv) {
            const uint32_t want = nlev > 0 ? f.level[lv] : 0u;
            for (int it = it0; it < it1; ++it) {
              const int32_t * cl = it == it0 ? cells0 : d.cells + (size_t)it * d.max_n;
              const int ncell = it == it0 ? ncell0 : d.cell_count[it];
              for (int t = tid; t < ncell; t += kTileThreads) {
                const int32_t cell = cl[t];
                if (cell < 0) continue;
                const int cx = (cell & 0xFFFF) + d.roi_x - half, cy = (cell >> 16) + d.roi_y - half;
                for (int ky = (cy ^ pq) & 1; ky < d.ksize; ky += 2) {
                  const int rel = ((cy + ky) >> 1) - band_r0;
                  if ((unsigned)rel >= (unsigned)f.alloc_rows) continue;
                  for (int kx = (cx ^ pp) & 1; kx < d.ksize; kx += 2) {
                    const uint32_t kv = kern[ky * d.ksize + kx];
                    if (nlev > 0) { if (kv == want) S8[rel * pitchB + ((cx + kx) >> 1)] = (uint8_t)kv; }
                    else if (kv) atomic_max_u8(S8 + rel * pitchB + ((cx + kx) >> 1), kv);
                  }
                }
              }
            }
            if (lv + 1 < nlev) __syncthreads();
          }
        }
      }
      if (e.flags & (kSeqNewChunk | kSeqNewStage)) __syncthreads();
      TILE_TM(kTmRaster);
      // ---- prefetch the next descriptor block (this pair's, or the first of this cluster's next pair) ----
      if (tid == 0) {
        const TileSeq * nxt = nullptr;
        if (si + 1 < nseq) nxt = seq + si + 1;
        else if (pair + nclusters < d.npairs) nxt = f.seq + f.seq_start[d.pair_query[pair + nclusters] * C + rank];
        if (nxt) issue(nxt, (cnt + 1) & 1);
      }
      mbar_wait(bar0 + 8 * (cnt & 1), (cnt >> 1) & 1);
      TILE_TM(kTmDesc);
      const unsigned char * stg = s_raw + f.off_stage + (size_t)(cnt & 1) * f.stage_bytes;
      const uint2 * items = reinterpret_cast<const uint2 *>(stg);   // the host's item list, longest first (format: sm_types.cuh)
      const uint16_t * pay = reinterpret_cast<const uint16_t *>(stg + (((size_t)e.nitems * 8 + 15) & ~(size_t)15));
      // ---- FAST + EDGE beams: warp items from the shared queue ----
      for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(&sh.ctr[cnt & 1], 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= e.nitems) break;
        TILE_CN(kCnItem);
        const uint2 rec = items[item];
        const int b0 = (int)(rec.x & 0xFFFFu);
        int b = b0;
        // plain beams [b0, pe), weighted singles [pe, se) (offset, weight), weighted pairs [ps, pe2) (offset, offset, weight, 0)
        const int pe = b0 + (int)((rec.x >> 16) & 0x3FFu), se = pe + 2 * (int)(rec.x >> 26);
        const int ps = (se + 3) & ~3, pe2 = ps + 4 * (int)(rec.y & 0xFFu);
        const int al = (int)((rec.y >> 8) & 63u), m = (int)((rec.y >> 14) & 3u);
        const int xt = (int)((rec.y >> 16) & 63u), yt = (int)((rec.y >> 22) & 255u);
        const int a = e.a0 + al;
        int32_t * Arow = A + (size_t)(a - chunk_a0) * P;
        const int ybase = y_l + kYTile * yt;
        const int y_end = kTail ? nY - 1 : nY;          // rows of the main row tiles
        const bool tail = kTail && yt == f.ytiles - 1;  // this y-tile also holds the tail row (warp-uniform)
       {
        int eb = 0, ee = 0;
        if (rec.y >> 31) {
          const int32_t * es = f.edge_start + (((size_t)q * nA + a) * 4 * nb + e.stage) * 4 + m;
          eb = es[0]; ee = es[1];
        }
        uint32_t base = smem_u32(S8) + (uint32_t)(((y_l + kYTile * yt) * pitch_w + 4 * xt + j_l) * 4);   // shared-window address
        asm volatile("" : "+r"(base));   // one opaque register: every descriptor then costs PRMT + IMAD (no re-association of the sum)
        // Idle lanes of the last y-tile (rows beyond the last pose) read past the band's nY-row halo, at most 47 rows (48-row
        // y-tiles; 39 on the tail layout) into the accumulator region that follows S in shared memory: in bounds, and their sums
        // are dropped at the flush (y >= y_end) -- so a band needs a halo of nY rows, not of whole y-tiles, and the row offsets
        // stay warp-uniform (LDS [R + UR]).
        const int x0 = 4 * (4 * xt + j_l) - m;
        // The flush is straight-line code: every lane reduces all of its fields, and a field that is not a pose of this item adds
        // zero.  The lane's four x-range tests are fixed for the item and become masks of the two packed words (the even fields
        // hold x0 and x0 + 2, the odd fields x0 + 1 and x0 + 3); a row beyond the last pose row is masked to zero and its
        // address clamped to the last one.  Columns -3 .. nX + 17 of a row stay inside the angle's volume or the guard words
        // around A (kAGuardLo / kAGuardHi), so every address is one the item may add zero to.
        auto add4 = [&](uint32_t a, uint32_t te, uint32_t to) {
          red_add(a + 0, te & 0xFFFFu);
          red_add(a + 4, to & 0xFFFFu);
          red_add(a + 8, te >> 16);
          red_add(a + 12, to >> 16);
        };
        // Tw / To: wrapped whole-word and odd-byte sums of every row tile (even_fields above)
        auto flush = [&](const uint32_t (&Tw)[kRowTiles], const uint32_t (&To)[kRowTiles]) {
          TILE_TM(kTmCorr);
          uint32_t any = 0;   // Tw = To = 0 exactly when E = To = 0 (E = Tw - (To << 8))
#pragma unroll
          for (int r = 0; r < kRowTiles; ++r) any |= Tw[r] | To[r];
          if (!__any_sync(0xffffffffu, any != 0)) { TILE_TM(kTmFlush); return; }
          TILE_CN(kCnFlush);
          // the tail row's sums over the 8 lane-rows of a word column: three butterfly adds of Tw and To (E of a sum is the sum
          // of the Es; the item's whole weight fits 16 bits) ahead of the first reduction, so that no convergence check
          // splits the reductions.  Zero outside the last y-tile, so every item of the tail layout runs it unbranched.
          uint32_t tw = 0, to = 0;
          if (kTail) {
            tw = Tw[kRowTiles - 1]; to = To[kRowTiles - 1];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
              tw += __shfl_xor_sync(0xffffffffu, tw, o);
              to += __shfl_xor_sync(0xffffffffu, to, o);
            }
          }
          const uint32_t xm0 = ((unsigned)x0 < (unsigned)nX ? 0x0000FFFFu : 0u) | ((unsigned)(x0 + 2) < (unsigned)nX ? 0xFFFF0000u : 0u);
          const uint32_t xm1 = ((unsigned)(x0 + 1) < (unsigned)nX ? 0x0000FFFFu : 0u) | ((unsigned)(x0 + 3) < (unsigned)nX ? 0xFFFF0000u : 0u);
          const uint32_t ax = smem_u32(Arow) + 4u * (uint32_t)x0, rowB = 4u * (uint32_t)nX;   // x0 >= -3: modular, into the guard
          const int ylast = max(y_end - 1, 0);
#pragma unroll
          for (int r = 0; r < kMain; ++r) {
            const int y = ybase + 8 * r;
            const uint32_t rm = y < y_end ? ~0u : 0u;
            add4(ax + rowB * (uint32_t)min(y, ylast), even_fields(Tw[r], To[r]) & xm0 & rm, To[r] & xm1 & rm);
          }
          if (kTail) {
            // lane-row 0 (ybase == kYTile * yt) adds the tail row, the other lane-rows add zero to rows of their own (no
            // same-address atomics)
            const bool tv = tail && ybase == kYTile * yt;
            const uint32_t tm = tv ? ~0u : 0u;
            add4(ax + rowB * (uint32_t)(tv ? nY - 1 : min(ybase, ylast)), even_fields(tw, to) & xm0 & tm, to & xm1 & tm);
          }
          TILE_TM(kTmFlush);
        };
        // an item's plain and weighted beams weigh at most kChunkBeams (the host splits longer groups): one flush
        if (b < se || ps < pe2) {
          uint32_t Tw[kRowTiles], To[kRowTiles];
#pragma unroll
          for (int r = 0; r < kRowTiles; ++r) { Tw[r] = 0; To[r] = 0; }
          for (; b + 3 < pe; b += 4) {   // 4 beams: one broadcast LDS.64 of descriptors, two byte-wise pair sums, one 3-input add per sum
            TILE_CN(kCnPlain4);
            const uint2 dd = *reinterpret_cast<const uint2 *>(pay + b);
            // 16-bit word offsets -> byte addresses: one PRMT (half-word extract) + one shift-add each
            const uint32_t o0 = base + 4u * __byte_perm(dd.x, 0, 0x4410), o1 = base + 4u * __byte_perm(dd.x, 0, 0x4432);
            const uint32_t o2 = base + 4u * __byte_perm(dd.y, 0, 0x4410), o3 = base + 4u * __byte_perm(dd.y, 0, 0x4432);
#pragma unroll
            for (int r = 0; r < kMain; ++r) {
              const uint32_t wa = lds_u32(o0 + r * 8 * pitchB) +
                                  lds_u32(o1 + r * 8 * pitchB);
              const uint32_t wb = lds_u32(o2 + r * 8 * pitchB) +
                                  lds_u32(o3 + r * 8 * pitchB);
              Tw[r] = Tw[r] + wa + wb;
              To[r] = To[r] + odd_bytes_t(wa) + odd_bytes_t(wb);
            }
          }
          for (; b + 1 < pe; b += 2) {
            TILE_CN(kCnPlain2);
            const uint32_t dd = *reinterpret_cast<const uint32_t *>(pay + b);
            const uint32_t o0 = base + ((dd & 0xFFFFu) << 2), o1 = base + ((dd >> 16) << 2);
#pragma unroll
            for (int r = 0; r < kMain; ++r) {
              const uint32_t w = lds_u32(o0 + r * 8 * pitchB) +
                                 lds_u32(o1 + r * 8 * pitchB);
              Tw[r] += w;
              To[r] += odd_bytes_t(w);
            }
          }
          if (b < pe) {
            TILE_CN(kCnPlain1);
            const uint32_t o0 = base + ((uint32_t)pay[b] << 2);
#pragma unroll
            for (int r = 0; r < kMain; ++r) {
              const uint32_t w = lds_u32(o0 + r * 8 * pitchB);
              Tw[r] += w;
              To[r] += odd_bytes_t(w);
            }
            ++b;
          }
          // cells that k beams of the group share: one entry of weight k.  Two entries of equal weight are one pair: two loads
          // added byte-wise (cell values <= 100), then one multiply-add per sum; a weight without a partner is a single.
          // (The host only builds weighted entries when the whole group's weight fits one flush.)
          for (int k = pe; k < se; k += 2) {
            TILE_CN(kCnSingle);
            const uint32_t dm = *reinterpret_cast<const uint32_t *>(pay + k);
            const uint32_t o0 = base + ((dm & 0xFFFFu) << 2);
            const uint32_t kk = dm >> 16;
#pragma unroll
            for (int r = 0; r < kMain; ++r) {
              const uint32_t w = lds_u32(o0 + r * 8 * pitchB);
              Tw[r] += w * kk;
              To[r] += odd_bytes_t(w) * kk;
            }
          }
          for (int k = ps; k < pe2; k += 4) {
            TILE_CN(kCnPair);
            const uint2 dp = *reinterpret_cast<const uint2 *>(pay + k);
            const uint32_t o0 = base + 4u * __byte_perm(dp.x, 0, 0x4410), o1 = base + 4u * __byte_perm(dp.x, 0, 0x4432);
            const uint32_t kk = dp.y;
#pragma unroll
            for (int r = 0; r < kMain; ++r) {
              const uint32_t w = lds_u32(o0 + r * 8 * pitchB) +
                                 lds_u32(o1 + r * 8 * pitchB);
              Tw[r] += w * kk;
              To[r] += odd_bytes_t(w) * kk;
            }
          }
          if (tail) {
            // the tail row nY - 1, lane-parallel over the entries: lane-row y_l reads entry y_l, y_l + 8, ... (its descriptor
            // with one LDS.U16 / LDS.32 / LDS.64 from 8 neighbouring entries, then the tail word of its column)
            const uint32_t tb = smem_u32(S8) + (uint32_t)(((nY - 1) * pitch_w + 4 * xt + j_l) * 4);
            uint32_t tw = 0, to = 0;
            for (int k = b0 + y_l; k < pe; k += 8) {
              TILE_CN(kCnTailPlain);
              const uint32_t w = lds_u32(tb + ((uint32_t)pay[k] << 2));
              tw += w;
              to += odd_bytes_t(w);
            }
            for (int k = pe + 2 * y_l; k < se; k += 16) {
              TILE_CN(kCnTailSingle);
              const uint32_t dm = *reinterpret_cast<const uint32_t *>(pay + k);
              const uint32_t w = lds_u32(tb + ((dm & 0xFFFFu) << 2));
              tw += w * (dm >> 16);
              to += odd_bytes_t(w) * (dm >> 16);
            }
            for (int k = ps + 4 * y_l; k < pe2; k += 32) {
              TILE_CN(kCnTailPair);
              const uint2 dp = *reinterpret_cast<const uint2 *>(pay + k);
              const uint32_t w = lds_u32(tb + 4u * __byte_perm(dp.x, 0, 0x4410)) + lds_u32(tb + 4u * __byte_perm(dp.x, 0, 0x4432));
              tw += w * dp.y;
              to += odd_bytes_t(w) * dp.y;
            }
            Tw[kRowTiles - 1] = tw;
            To[kRowTiles - 1] = to;
          }
          flush(Tw, To);
        }
        // EDGE beams of this group (window partly outside the grid): the same word loads with rows / words outside the
        // band allocation masked (they index outside [0, data_size) or wrap in the reference; the wrapped part is added
        // from the wrap2 list below).  Rows / words inside the allocation but beyond the valid cells are zero padding.
        while (eb < ee) {
          const int ce = min(ee, eb + kChunkBeams);
          uint32_t Tw[kRowTiles], To[kRowTiles];
#pragma unroll
          for (int r = 0; r < kRowTiles; ++r) { Tw[r] = 0; To[r] = 0; }
          for (int b0 = eb; b0 < ce; b0 += 32) {
            const int cn = min(32, ce - b0);
            const int32_t mine = (lane < cn) ? f.edge[b0 + lane] : 0;
            for (int k = 0; k < cn; ++k) {
              TILE_CN(kCnEdge);
              const int32_t ev = __shfl_sync(0xffffffffu, mine, k);
              const int rowb = (int)(int16_t)(ev & 0xFFFF), wq = (ev >> 16) + 4 * xt + j_l;
              const int row0 = rowb + ybase;
              const bool cv = (unsigned)wq < (unsigned)pitch_w;
#pragma unroll
              for (int r = 0; r < kMain; ++r) {
                const int row = row0 + 8 * r;
                const uint32_t w = (cv && (unsigned)row < (unsigned)f.alloc_rows) ? S[row * pitch_w + wq] : 0u;
                Tw[r] += w;
                To[r] += odd_bytes_t(w);
              }
              if (tail) {   // the tail row in lane-row 0 only (the flush sums the lane-rows)
                const int row = rowb + nY - 1;
                const uint32_t w = (y_l == 0 && cv && (unsigned)row < (unsigned)f.alloc_rows) ? S[row * pitch_w + wq] : 0u;
                Tw[kRowTiles - 1] += w;
                To[kRowTiles - 1] += odd_bytes_t(w);
              }
            }
          }
          eb = ce;
          flush(Tw, To);
        }
       }
      }
      TILE_TM(kTmCorr);
      if (e.flags & kSeqNewStage) {
        // ---- wrapped part of EDGE beams (row parity flipped list): poses whose column left [0, stride) by less than a
        //      stride read the neighbouring row at column -/+ stride (linear index, M.cpp:1192-1200) ----
        const int32_t * ws = f.wrap2_start + ((size_t)q * nA + chunk_a0) * 4 * nb + e.stage;
        const bool has_wrap = (e.flags & kSeqHasWrap) != 0;
        if (has_wrap) {
          for (int p = tid; p < P; p += kTileThreads) {
            const int ex = 2 * (p % nX), ey = 2 * (p / nX);
            for (int al = 0; al < chunk_na; ++al) {
              int acc = 0;
              for (int bi = ws[(size_t)al * 4 * nb]; bi < ws[(size_t)al * 4 * nb + 1]; ++bi) {
                const int32_t ev = f.wrap2[bi];
                const int Xb = (int)(int16_t)(ev & 0xFFFF), Yb = ev >> 16;
                const int col = Xb + ex;
                if ((unsigned)col < (unsigned)d.stride) continue;
                const int r2 = Yb + ey + (col < 0 ? -1 : 1);
                const int c2 = col + (col < 0 ? d.stride : -d.stride);
                if ((unsigned)r2 >= (unsigned)d.height) continue;
                const int rel = (r2 >> 1) - band_r0;
                if ((unsigned)rel >= (unsigned)f.alloc_rows) continue;
                acc += S8[rel * pitchB + (c2 >> 1)];
              }
              if (acc) atomicAdd(A + (size_t)al * P + p, acc);
            }
          }
        }
        // ---- FAR beams (column offsets of a stride or more): pose by pose on the linear index; a row belongs to the band
        //      whose own rows contain it ----
        const int32_t * ss = f.slow_start + (size_t)q * (nA + 1);
        if (ss[nA] - ss[0] > 0) {
          const int32_t * pos = d.posidx + (size_t)q * P;
          const int own_hi = (band == nb - 1) ? 0x7FFFFFFF : f.band_rows;
          for (int al = 0; al < chunk_na; ++al) {
            const int sb = ss[chunk_a0 + al], se = ss[chunk_a0 + al + 1];
            const int work = (se - sb) * P;
            for (int t = tid; t < work; t += kTileThreads) {
              const int bi = t / P, p = t - bi * P;
              const int idx = pos[p] + f.slow[sb + bi];
              if ((unsigned)idx >= (unsigned)d.data_size) continue;
              const int row = idx / d.stride, col = idx - row * d.stride;
              if ((col & 1) != pp || (row & 1) != pq) continue;
              const int rel = (row >> 1) - band_r0;
              if (rel < 0 || rel >= own_hi || rel >= f.alloc_rows) continue;
              const int v = S8[rel * pitchB + (col >> 1)];
              if (v) atomicAdd(A + (size_t)al * P + p, v);
            }
          }
        }
      }
      if (tid == 0) sh.ctr[(cnt + 1) & 1] = 0;
      __syncthreads();
      ++cnt;
      TILE_TM(kTmBarrier);

      if (e.flags & kSeqEndChunk) {
        // ================= chunk reduction: per-cell max image, best response, ordered tie list =================
        if (pending_wait) { cluster_wait(); pending_wait = false; }   // the previous pair's leader has read our image
        double lbest = -1.0;
        int smax = -1;
        if (f.int_ties) {
          // responses are sum / norm: monotone in the sum and two different sums differ by more than the tie tolerance
          for (int p = tid; p < P; p += kTileThreads) {
            int sm = 0;
            for (int al = 0; al < chunk_na; ++al) { const int s = A[(size_t)al * P + p]; sm = s > sm ? s : sm; }
            smax = sm > smax ? sm : smax;                       // this chunk's best
            if (!first_chunk) { const int o = iprobs[p]; sm = o > sm ? o : sm; }
            iprobs[p] = sm;                                     // running per-cell maximum over the chunks so far
          }
          for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, smax, o); smax = t > smax ? t : smax; }
          __syncthreads();
          if (lane == 0) sh.iscratch[tid >> 5] = smax;
          __syncthreads();
          for (int i = 0; i < kTileThreads / 32; ++i) smax = sh.iscratch[i] > smax ? sh.iscratch[i] : smax;
          __syncthreads();
          lbest = (double)smax;
          lbest /= d.norm;
        } else {
          for (int p = tid; p < P; p += kTileThreads) {
            const int x = p % nX, y = p / nX;
            double pm = first_chunk ? 0.0 : probs[p];   // Grid<double>::Clear() initial value, M.cpp:727
            for (int al = 0; al < chunk_na; ++al) {
              const double r = pose_response(d, q, A[(size_t)al * P + p], x, y, chunk_a0 + al);
              pm = r > pm ? r : pm;
              lbest = r > lbest ? r : lbest;
            }
            probs[p] = pm;
          }
          lbest = block_max(lbest, sh.dscratch);
        }
        // ordered tie list: poses with DoubleEqual(response, best) in array order (M.cpp:807-817); every thread owns a
        // contiguous run of cells so that ranks follow array order
        const int per = (P + kTileThreads - 1) / kTileThreads;
        const int p0 = min(P, tid * per), p1 = min(P, p0 + per);
        int c = 0;
        for (int p = p0; p < p1; ++p) {
          const int x = p % nX, y = p / nX;
          for (int al = 0; al < chunk_na; ++al) {
            const int s = A[(size_t)al * P + p];
            const bool tie = f.int_ties ? (s == smax) : double_equal(pose_response(d, q, s, x, y, chunk_a0 + al), lbest);
            if (tie) ++c;
          }
        }
        int total = 0;
        int rk = block_exclusive_scan(c, sh.iscratch, total);
        if (c > 0 && rk < kMaxTies) {
          for (int p = p0; p < p1 && rk < kMaxTies; ++p) {
            const int x = p % nX, y = p / nX;
            for (int al = 0; al < chunk_na && rk < kMaxTies; ++al) {
              const int s = A[(size_t)al * P + p];
              const bool tie = f.int_ties ? (s == smax) : double_equal(pose_response(d, q, s, x, y, chunk_a0 + al), lbest);
              if (tie) {
                if (rk == 0) sh.chunk.sum0 = s;
                sh.chunk.ties[rk++] = p * nA + chunk_a0 + al;
              }
            }
          }
        }
        __syncthreads();
        if (tid == 0) {
          if (first_chunk) {
            sh.res.L = lbest; sh.res.L2 = -1e300; sh.res.cnt = total; sh.res.sum0 = sh.chunk.sum0;
            for (int t = 0; t < kMaxTies; ++t) sh.res.ties[t] = sh.chunk.ties[t];
          } else {
            tie_merge(sh.res, lbest, -1e300, total, sh.chunk.sum0, sh.chunk.ties);
          }
        }
        first_chunk = false;
        __syncthreads();
        TILE_TM(kTmReduce);
      }
    }

    // ================= pair reduction across the cluster =================
    if (C > 1) {
      if (tid < 32) {
        const uint32_t base = dsmem_addr(&sh, leader);
        const uint32_t off = smem_u32(&sh);
        if (tid == 0) {
          dsmem_st_f64(base + (smem_u32(&sh.rankL[rank]) - off), sh.res.L);
          dsmem_st_f64(base + (smem_u32(&sh.rankL2[rank]) - off), sh.res.L2);
          dsmem_st_s32(base + (smem_u32(&sh.rankCnt[rank]) - off), sh.res.cnt);
          dsmem_st_s32(base + (smem_u32(&sh.rankSum0[rank]) - off), sh.res.sum0);
        }
        if (tid < kMaxTies) dsmem_st_s32(base + (smem_u32(&sh.rankTies[rank][tid]) - off), sh.res.ties[tid]);
      }
      cluster_arrive();
      cluster_wait();
    }
    if (rank == leader) {
      PairOut & out = d.out[pair];
      if (tid == 0) {
        TieRes r = sh.res;
        if (C > 1) {
          r.L = sh.rankL[0]; r.L2 = sh.rankL2[0]; r.cnt = sh.rankCnt[0]; r.sum0 = sh.rankSum0[0];
          for (int t = 0; t < kMaxTies; ++t) r.ties[t] = sh.rankTies[0][t];
          for (int s = 1; s < C; ++s) tie_merge(r, sh.rankL[s], sh.rankL2[s], sh.rankCnt[s], sh.rankSum0[s], sh.rankTies[s]);
        }
        // a chunk best within the tie tolerance of (but not equal to) the pair's best could hold further ties: leave the
        // pair to the single-match path (tie_count -1).  Cannot happen on the integer path.
        const bool ambiguous = double_equal(r.L2, r.L);
        const int m = r.cnt < kMaxTies ? r.cnt : kMaxTies;
        out.best = r.L;
        out.best_sum = r.cnt > 0 ? r.sum0 : 0;
        out.tie_count = ambiguous ? -1 : r.cnt;
        for (int t = 0; t < m; ++t) out.ties[t] = r.ties[t];
        double ax = 0.0, ay = 0.0;
        for (int t = 0; t < m; ++t) {   // averagePosition += pose position, in order (M.cpp:809)
          const int p = r.ties[t] / nA;
          ax += d.newx[q * nX + p % nX];
          ay += d.newy[q * nY + p / nX];
        }
        if (r.cnt > 0) { ax /= r.cnt; ay /= r.cnt; }
        out.avg_x = ax; out.avg_y = ay;
        sh.avg[0] = ax; sh.avg[1] = ay;
        // the covariance sums are only used for an unambiguous, non-overflowing tie set with best >= tolerance (M.cpp:886-891)
        sh.ok = (!ambiguous && r.cnt > 0 && r.cnt <= kMaxTies && !(r.L < kTolerance)) ? 1 : 0;
        sh.acc[0] = sh.acc[1] = sh.acc[2] = sh.acc[3] = 0.0;
        sh.res.L = r.L;
      }
      __syncthreads();
      if (sh.ok && C > 1) {
        // per-cell max over the other CTAs' images, through distributed shared memory
        for (uint32_t s = 0; s < (uint32_t)C; ++s) {
          if (s == rank) continue;
          const uint32_t rp = dsmem_addr(probs, s);
          if (f.int_ties) {
            for (int p = tid; p < P; p += kTileThreads) {
              const int v = dsmem_ld_s32(rp + 4u * (uint32_t)p);
              if (v > iprobs[p]) iprobs[p] = v;
            }
          } else {
            for (int p = tid; p < P; p += kTileThreads) {
              const double v = dsmem_ld_f64(rp + 8u * (uint32_t)p);
              if (v > probs[p]) probs[p] = v;
            }
          }
        }
      }
    }
    if (C > 1) { cluster_arrive(); pending_wait = true; }   // the others may reuse their images once the leader has arrived
    if (rank == leader) {
      __syncthreads();
      PairOut & out = d.out[pair];
      if (sh.ok) {
        // positional covariance accumulators (M.cpp:893-933): cells with response >= best - 0.1, summed in (y, x) order.
        // Terms are formed in parallel, compacted in order, then added sequentially so the additions happen in the
        // reference's order.  The term buffer reuses S and A (free now), a sub-range of cells at a time.
        const double best = sh.res.L;
        const double dx = sh.avg[0] - d.center[q * 3 + 0], dy = sh.avg[1] - d.center[q * 3 + 1];
        double * terms = reinterpret_cast<double *>(s_raw);
        const int cap = (int)(f.off_probs / 32);
        for (int c0 = 0; c0 < P; c0 += cap) {
          const int c1 = min(P, c0 + cap), len = c1 - c0;
          const int per = (len + kTileThreads - 1) / kTileThreads;
          const int p0 = c0 + min(len, tid * per), p1 = min(c1, p0 + per);
          int c2 = 0;
          auto cell_max = [&](int p) -> double {   // the m_pSearchSpaceProbs value of cell p
            if (!f.int_ties) return probs[p];
            double v = (double)iprobs[p];
            v /= d.norm;
            return v;
          };
          for (int p = p0; p < p1; ++p) if (cell_max(p) >= (best - 0.1)) ++c2;
          int tot2 = 0;
          int r2 = block_exclusive_scan(c2, sh.iscratch, tot2);
          for (int p = p0; p < p1; ++p) {
            const double resp = cell_max(p);
            if (resp >= (best - 0.1)) {
              const double x = d.xrel[q * nX + p % nX], y = d.yrel[q * nY + p / nX];
              terms[4 * r2 + 0] = resp;
              terms[4 * r2 + 1] = (square(x - dx) * resp);
              terms[4 * r2 + 2] = ((x - dx) * (y - dy) * resp);
              terms[4 * r2 + 3] = (square(y - dy) * resp);
              ++r2;
            }
          }
          __syncthreads();
          if (tid == 0) {
            double norm = sh.acc[0], axx = sh.acc[1], axy = sh.acc[2], ayy = sh.acc[3];
            for (int t = 0; t < tot2; ++t) {
              norm += terms[4 * t + 0];
              axx += terms[4 * t + 1];
              axy += terms[4 * t + 2];
              ayy += terms[4 * t + 3];
            }
            sh.acc[0] = norm; sh.acc[1] = axx; sh.acc[2] = axy; sh.acc[3] = ayy;
          }
          __syncthreads();
        }
      }
      if (tid == 0) { out.norm = sh.acc[0]; out.acc_xx = sh.acc[1]; out.acc_xy = sh.acc[2]; out.acc_yy = sh.acc[3]; }
      __syncthreads();
    }
  }
  if (pending_wait) cluster_wait();   // nobody leaves while a leader may still read its shared memory
  TILE_TM_END;
  TILE_CN_END;
}

// ------------------------------------------------------------------------------------------
// host side: plan (chunks, bands, cluster size), descriptor blocks, launch
// ------------------------------------------------------------------------------------------
// the instantiation for a row pitch: 4 m / 12 m -> 76 words, 8 m / 12 m -> 92, 4 m / 20 m -> 116, 8 m / 20 m -> 132; anything else
// runs the run-time-pitch version; each in both y-tile layouts
template <bool kTail>
static const void * tile_kernel_for_layout(int pitch_w)
{
  switch (pitch_w) {
    case 76: return (const void *)k_sweep_tile<76, kTail>;
    case 92: return (const void *)k_sweep_tile<92, kTail>;
    case 116: return (const void *)k_sweep_tile<116, kTail>;
    case 132: return (const void *)k_sweep_tile<132, kTail>;
    default: return (const void *)k_sweep_tile<0, kTail>;
  }
}
static const void * tile_kernel_for(int pitch_w, bool tail)
{
  return tail ? tile_kernel_for_layout<true>(pitch_w) : tile_kernel_for_layout<false>(pitch_w);
}

static int env_int(const char * name, int dflt)
{
  const char * v = std::getenv(name);
  return (v && *v) ? std::atoi(v) : dflt;
}

// the first scan's cell list is staged when one list is small enough and its stride keeps the bulk copy 16-byte aligned
static inline bool d_max_n_ok(int max_n) { return max_n > 0 && (max_n & 3) == 0 && max_n <= 4096; }

static inline int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// Reorders a sorted descriptor list so that entries i, i + 1, ..., i + 7 (what the 8 lane-rows read at once for the tail row) come
// from 8 spread-out parts of the sorted order: neighbouring cells would put their 4-word runs on the same banks.  The sums are
// integers, so the order is free.
static void spread_rows(std::vector<uint16_t>::iterator b, std::vector<uint16_t>::iterator e)
{
  const size_t L = (size_t)(e - b), R = (L + 7) / 8;
  if (L < 9) return;
  const std::vector<uint16_t> src(b, e);
  size_t o = 0;
  for (size_t j = 0; j < R; ++j)
    for (size_t y = 0; y < 8; ++y)
      if (y * R + j < L) b[o++] = src[y * R + j];
}

// The warp items of one descriptor block, longest first (the shared queue then hands out long items first).  tbl holds (plain
// begin, singles begin, singles end, pairs end) per (angle, alignment) group (the pairs begin at the first 4-entry boundary from the
// singles' end), nedge the group's EDGE beams.  A group's plain list is cut into pieces of at most kChunkBeams beams (4-aligned
// starts: the 4-beam step reads descriptors with 64-bit loads), so that every item flushes its 16-bit fields once; the weighted
// singles and pairs and the EDGE beams go with the last piece.
// Returns false when a piece does not fit its record's fields (the encoder keeps them in range: a planner refusal, not a wrap).
static bool build_block_items(const std::vector<int32_t> & tbl, const std::vector<int> & nedge, int na, int xtiles, int ytiles,
                              std::vector<uint2> & out)
{
  struct Piece { int work; int pb, pe, nsingle, npair, al, m; bool edge; };
  std::vector<Piece> pieces;
  for (int g = 0; g < na * 4; ++g) {
    const int pb = tbl[4 * g], sb = tbl[4 * g + 1], se = tbl[4 * g + 2], pe2 = tbl[4 * g + 3];
    const int ns = (se - sb) / 2, np = pe2 > se ? (pe2 - ((se + 3) & ~3)) / 4 : 0;
    const int ne = nedge[g];
    if (sb == pb && ns == 0 && np == 0 && ne == 0) continue;
    for (int s = pb;; s += kChunkBeams) {
      Piece p{0, s, std::min(sb, s + kChunkBeams), 0, 0, g >> 2, g & 3, false};
      if (p.pe == sb) { p.nsingle = ns; p.npair = np; p.edge = ne > 0; }
      p.work = (p.pe - p.pb) + p.nsingle + 2 * p.npair + (p.edge ? ne : 0);   // entries loaded
      if (p.pb > 0xFFFF || p.pe - p.pb > 0x3FF || p.nsingle > kMaxSingles || p.npair > kMaxPairs) return false;
      pieces.push_back(p);
      if (p.pe == sb) break;
    }
  }
  std::stable_sort(pieces.begin(), pieces.end(), [](const Piece & x, const Piece & y) { return x.work > y.work; });
  out.clear();
  for (const Piece & p : pieces)
    for (int yt = 0; yt < ytiles; ++yt)
      for (int xt = 0; xt < xtiles; ++xt)
        out.push_back(make_uint2((uint32_t)p.pb | ((uint32_t)(p.pe - p.pb) << 16) | ((uint32_t)p.nsingle << 26),
                                 (uint32_t)p.npair | ((uint32_t)p.al << 8) | ((uint32_t)p.m << 14) | ((uint32_t)xt << 16) |
                                   ((uint32_t)yt << 22) | (p.edge ? 0x80000000u : 0u)));
  return true;
}

void classify_beams(const GridGeom & g, const CorrPlan & pl, int a, int pitch_w, int band_rows, int nbands, BeamClasses & c)
{
  const int nX = pl.nX, nY = pl.nY, n = pl.n, nstage = 4 * nbands, B = band_rows;
  const int X0 = pl.xs[0], Y0 = pl.ys[0];
  c.fast.resize((size_t)nstage * 4);
  c.edge.resize((size_t)nstage * 4);
  c.wrap2.resize(nstage);
  for (auto & v : c.fast) v.clear();
  for (auto & v : c.edge) v.clear();
  for (auto & v : c.wrap2) v.clear();
  c.far.clear();
  int nf = 0, ne = 0;
  for (int i = 0; i < n; ++i) {
    const int32_t off = pl.offsets[(size_t)a * n + i];
    if (off == kInvalidScan) continue;
    const int gx = pl.ogx[(size_t)a * n + i], gy = pl.ogy[(size_t)a * n + i];
    const int Xb = X0 + gx, Yb = Y0 + gy;
    const bool inside = Xb >= 0 && Xb + 2 * (nX - 1) < g.stride && Yb >= 0 && Yb + 2 * (nY - 1) < g.height;
    if (inside) {
      const int pp = Xb & 1, pq = Yb & 1, cx = Xb >> 1, r = Yb >> 1;
      const int band = std::min(r / B, nbands - 1);
      const int wo = (r - band * B) * pitch_w + (cx >> 2);
      c.fast[((pq * 2 + pp) * nbands + band) * 4 + (cx & 3)].push_back((uint16_t)wo);
      ++nf;
    } else if (Xb >= -g.stride && Xb + 2 * (nX - 1) < 2 * g.stride && Xb > -32768 && Xb < 32767 && Yb > -32768 && Yb < 32767) {
      // EDGE beam: at most one row wrap.  Primary entry in the beam's own phase; if some column leaves [0, stride), a
      // secondary entry in the phase with the row parity flipped.
      const bool rows_hit = Yb + 2 * (nY - 1) >= 0 && Yb < g.height;
      const bool cols_hit = Xb + 2 * (nX - 1) >= 0 && Xb < g.stride;
      if (rows_hit && cols_hit) {
        const int cx = Xb >> 1, r = Yb >> 1;   // arithmetic shifts: floor for negative coordinates
        const int band = std::min(std::max(floor_div(r, B), 0), nbands - 1);
        const int rr = r - band * B;
        if (rr > -32768 && rr < 32767) {
          c.edge[(((Yb & 1) * 2 + (Xb & 1)) * nbands + band) * 4 + (cx & 3)].push_back(
            (int32_t)((uint32_t)(rr & 0xFFFF) | ((uint32_t)(cx >> 2) << 16)));
          ++ne;
        }
      }
      const bool wraps = Xb < 0 || Xb + 2 * (nX - 1) >= g.stride;
      if (wraps && Yb + 2 * (nY - 1) + 1 >= 0 && Yb - 1 < g.height) {
        const int r = (Yb - 1) >> 1;
        const int band = std::min(std::max(floor_div(r, B), 0), nbands - 1);
        c.wrap2[(((Yb & 1) ^ 1) * 2 + (Xb & 1)) * nbands + band].push_back((int32_t)((uint32_t)(Xb & 0xFFFF) | ((uint32_t)Yb << 16)));
      }
    } else {
      const int32_t dv = device_offset(off, g.data_size);
      if (dv != kDevInvalid) c.far.push_back(dv);   // FAR: can still index [0, data_size) for some pose
    }
  }
  c.n_fast = nf; c.n_edge = ne;
}

void append_beam_lists(const std::vector<BeamClasses> & cls, int nstage, BeamLists & L)
{
  L.slow_start.push_back((int32_t)L.slow.size());
  for (const BeamClasses & c : cls) {
    L.slow.insert(L.slow.end(), c.far.begin(), c.far.end());
    L.slow_start.push_back((int32_t)L.slow.size());
    L.n_fast += c.n_fast; L.n_edge += c.n_edge;
    for (int sg = 0; sg < nstage; ++sg) {
      L.wrap2_start.push_back((int32_t)L.wrap2.size());
      L.wrap2.insert(L.wrap2.end(), c.wrap2[sg].begin(), c.wrap2[sg].end());
      for (int m = 0; m < 4; ++m) {
        L.edge_start.push_back((int32_t)L.edge.size());
        L.edge.insert(L.edge.end(), c.edge[sg * 4 + m].begin(), c.edge[sg * 4 + m].end());
      }
    }
  }
}

void upload_beam_lists(BeamLists & L, SweepHost & S, cudaStream_t st)
{
  L.edge_start.push_back((int32_t)L.edge.size());
  L.wrap2_start.push_back((int32_t)L.wrap2.size());
  S.beam_counts[0] = L.n_fast; S.beam_counts[1] = L.n_edge; S.beam_counts[2] = (int32_t)L.slow.size();
  L.edge.push_back(0); L.wrap2.push_back(0); L.slow.push_back(0);
  S.h2d(S.d_edge, L.edge.data(), L.edge.size(), st);
  S.h2d(S.d_edge_start, L.edge_start.data(), L.edge_start.size(), st);
  S.h2d(S.d_wrap2, L.wrap2.data(), L.wrap2.size(), st);
  S.h2d(S.d_wrap2_start, L.wrap2_start.data(), L.wrap2_start.size(), st);
  S.h2d(S.d_slow, L.slow.data(), L.slow.size(), st);
  S.h2d(S.d_slow_start, L.slow_start.data(), L.slow_start.size(), st);
}

void encode_runs(const std::vector<uint16_t> & group, int min_weight, bool merge, std::vector<uint16_t> & plain,
                 std::vector<std::pair<uint16_t, uint16_t>> & merged)
{
  for (size_t i = 0; i < group.size();) {
    size_t j = i;
    while (j < group.size() && group[j] == group[i]) ++j;
    if (merge && j - i >= (size_t)min_weight) merged.emplace_back(group[i], (uint16_t)(j - i));
    else plain.insert(plain.end(), j - i, group[i]);
    i = j;
  }
}

int parity_refusal(const GridGeom & g, const std::vector<CorrPlan> & plans)
{
  if (g.order_dependent) return 1;   // AddScan's occupancy test makes the raster sequential (generic kernel)
  for (const CorrPlan & pl : plans) {
    for (int k = 1; k < pl.nX; ++k) if (pl.xs[k] != pl.xs[0] + 2 * k) return 6;
    for (int k = 1; k < pl.nY; ++k) if (pl.ys[k] != pl.ys[0] + 2 * k) return 7;
  }
  return 0;
}

// Refusals (the sweep then runs on the generic kernel, which takes any n and nA): plan_tile's 2, 4, 9 (more x- / y-tiles than the
// item record holds) and 5 (the plan's shared memory exceeds 227 KB), schedule_query's 8 and 10 to 13.  Packed fields and bounds:
//   TileSeq.a0 / chunk (int16)   nA <= 4096                                                  -> 2
//   item al (6 bits)             nAc <= 63 angles per chunk (the V loop)                     -> 4 when no V fits
//   item plain count (10 bits)   pieces of <= kChunkBeams = 640 beams
//   item singles (6 bits)        weighted entries only in groups of <= kChunkBeams beams: one single per distinct weight
//                                k >= 2 (2 + 3 + ... + 36 = 665 > 640: <= 34 weights) + the odd plain beam: <= 35; without
//                                pairing (B200_TILE_PAIRS=0) the encoder returns singles beyond 62 to the plain list
//   item pairs (8 bits)          a pair weighs >= 4 beams: <= 640 / 4 = 160 per group
//   (all three, and pb, are checked per record by build_block_items)                        -> 13
//   one angle's block            payload <= n + 32 entries, records per the one_angle minimum  -> 8
//   TileSeq.nitems (int16)       records of one block                                        -> 10
//   item pb / pe (16 bits)       payload entries of one block                                -> 11
//   TileSeq.off (int32)          descriptor blob bytes                                       -> 12
//   cell-list staging            max_n > 4096: the raster reads the cells from global memory    (no refusal needed)
TilePlan plan_tile(const TilePlanIn & in)
{
  auto refuse = [](int why) { TilePlan r; r.refused = why; return r; };
  const int nX = in.nX, nY = in.nY, nA = in.nA, n = in.n, P = nX * nY;
  if ((in.stride & 1) || nA < 1 || nA > 4096) return refuse(2);
  // ---- geometry of one parity sub-grid ----
  int pitch_w = (in.stride / 2 + 16 + 3) / 4;            // sub-grid row + the 3-word overhang of the last x-tile
  while ((pitch_w & 7) != 4) ++pitch_w;                  // 8 rows x 4 words of a warp hit 32 distinct banks
  // y-tile layout, by the row-tile loads of one beam and x-tile (in eighths of a row tile): 48-row y-tiles of six row tiles, or
  // 40-row y-tiles of five + the tail row (one descriptor and one word load per 8 entries, i.e. 2 / 8).  41 rows: 42 vs 48; 81
  // rows: 82 vs 96; 45 rows: 82 vs 48 (stays on 48-row tiles)
  const int yt48 = (nY + 47) / 48, yt40 = std::max(1, (nY - 1 + 39) / 40);
  const bool tail = in.tail && 8 * 5 * yt40 + 2 < 8 * 6 * yt48;
  const int ytile_rows = tail ? 40 : 48;
  const int xtiles = (nX + 3 + 15) / 16, ytiles = tail ? yt40 : yt48;
  if (xtiles > kItemMaxXTiles || ytiles > kItemMaxYTiles) return refuse(9);
  const int rows_valid = (in.height + 1) / 2;
  const int halo = nY + 2;                               // rows a beam window reaches below its base row (idle row tiles are clamped) + the wrapped row
  const int base_rows = std::max(1, rows_valid - nY + 1);   // distinct base rows of beams whose window is inside the grid
  // ---- choose the number of angle chunks V and of bands ----
  int want_c = in.cluster;
  if (want_c <= 0) {
    // throughput mode (one CTA per pair) once the batch fills the GPU, otherwise spread a pair over a cluster
    want_c = 1;
    while (want_c < kTileMaxCluster && in.npairs * want_c * 2 <= in.sms) want_c *= 2;
  }
  int Cc = 1;
  while (Cc * 2 <= std::min(want_c, kTileMaxCluster)) Cc *= 2;
  Cc = std::min(Cc, nA);
  while (Cc & (Cc - 1)) --Cc;
  const int budget = 227 * 1024 - (int)sizeof(TileShared) - 256;
  const int int_ties = (!in.do_penalize && (double)n * kOccupied < 0.9e6) ? 1 : 0;
  const int probs_bytes = (P * (int_ties ? 4 : 8) + 15) & ~15;   // per-cell maximum image: integer sums or FP64 responses
  int bestV = 0, bestNb = 0, bestB = 0, bestStage = 0;
  long bestCost = -1;
  for (int V = Cc; V <= nA; ++V) {
    if (in.chunks > 0 && V < std::min(in.chunks, nA)) continue;   // "sweep_chunks" = at least this many chunks
    const int nAc = (nA + V - 1) / V;
    if ((nA + nAc - 1) / nAc != V || nAc > 63) continue;   // same chunk size as a smaller V; group ids are bytes
    const int a_bytes = (4 * (kAGuardLo + nAc * P + kAGuardHi) + 15) & ~15;
    // staging buffer: item list + 1.5 x the average descriptor bytes of a (chunk, phase) block, at least one angle's worst case:
    // one item record per (alignment, tile), plus one per tile for every further kChunkBeams-piece of a long group -- the
    // groups of one angle hold at most n beams, so they are cut at most (n - 1) / kChunkBeams more times
    // payload of one angle: <= 2 bytes per beam (a plain beam 2, a single of weight >= 2 4, a pair of weight >= 2 each 8) + per group
    // <= 6 bytes of 4-entry alignment before the plain list, 2 for the odd plain beam's single, 4 before the pairs; + 6 at the end
    const int one_angle = 8 * xtiles * ytiles * (4 + std::max(n - 1, 0) / kChunkBeams) + 2 * n + 4 * 12 + 6 + 10;
    int stage = 16 + nAc * 52 + (nAc * n * 2 * 3) / 8 + 64 * nAc;
    stage = std::max(stage, one_angle + 64);
    stage = (stage + 127) & ~127;
    const int s_avail = budget - a_bytes - probs_bytes - 2 * stage;
    if (s_avail <= 0) continue;
    int rows_avail = s_avail / (pitch_w * 4);
    if ((long)rows_avail * pitch_w > 65535) rows_avail = 65535 / pitch_w;   // descriptors are 16-bit word offsets
    int B = rows_avail - halo;
    if (B < 8) continue;
    B = std::min(B, base_rows);
    const int nbv = (base_rows + B - 1) / B;
    B = (base_rows + nbv - 1) / nbv;                     // even bands
    // cost of one pair on one CTA, in thread-instructions: rasters (4 phases per chunk and band) + the beam loop per angle
    // the accumulator flush of every (angle, stage, alignment, tile) item (32 warps) and the fixed cost of a stage (clear + raster +
    // three barriers) are what make extra bands expensive.  The flush is straight-line code: 124 warp instructions from the vote to
    // the last reduction on the tail layout, 112 on 48-row y-tiles (sm_90a SASS of k_sweep_tile)
    // the beam loop: ~2.3 thread-instructions per lane and row-tile load (6 per beam and 48-row y-tile; 5 + 2 / 8 with the tail)
    const double loads = tail ? 5.0 * ytiles + 0.25 : 6.0 * ytiles;
    const long flush_wi = tail ? 124 : 112;
    const long w_angle = (long)((double)n * xtiles * loads * 32 * 2.3 / kTileThreads) + 4L * nbv * (4L * xtiles * ytiles * flush_wi / 32);
    const long w_raster = 4 * (700 + 3L * std::min(B + halo, rows_valid + halo - nY) * pitch_w / kTileThreads);
    const long cost = (long)((V + Cc - 1) / Cc) * (nbv * w_raster + nAc * w_angle);
    if (bestCost < 0 || cost < bestCost) { bestCost = cost; bestV = V; bestNb = nbv; bestB = B; bestStage = stage; }
  }
  if (bestCost < 0) return refuse(4);
  TilePlan p;
  p.C = std::min(Cc, bestV); p.V = bestV; p.nAc = (nA + bestV - 1) / bestV; p.nbands = bestNb; p.band_rows = bestB;
  p.alloc_rows = std::max(std::min(bestB + halo, rows_valid + halo - nY), 1); p.pitch_w = pitch_w; p.xtiles = xtiles;
  p.ytiles = ytiles; p.ytile_rows = ytile_rows; p.tail = tail ? 1 : 0; p.stage_bytes = bestStage; p.int_ties = int_ties;
  const size_t s_bytes = ((size_t)p.alloc_rows * pitch_w * 4 + 15) & ~(size_t)15;
  const size_t a_bytes = (4 * ((size_t)kAGuardLo + (size_t)p.nAc * P + kAGuardHi) + 15) & ~(size_t)15;   // A and its guard words
  p.off_A = s_bytes + 4 * kAGuardLo; p.off_probs = s_bytes + a_bytes; p.off_stage = (p.off_probs + probs_bytes + 127) & ~(size_t)127;
  p.off_cells = p.off_stage + 2 * (size_t)p.stage_bytes;
  // cell-list staging only where the chosen plan leaves room for it (it must not cost a band or a chunk)
  int cell_cap = d_max_n_ok(in.max_n) ? in.max_n : 0;                   // entries per cell staging buffer (0 = read cells from global)
  if (p.off_cells + 2 * (size_t)cell_cap * 4 + sizeof(TileShared) + 64 > 227 * 1024) cell_cap = 0;
  p.cell_cap = cell_cap;
  size_t smem = p.off_cells + 2 * (size_t)cell_cap * 4;
  // idle lanes of the last y-tile read up to (ytile_rows * ytiles - nY) rows past the band (see the kernel): keep those reads inside
  // the allocation even when everything behind S is small (tiny search windows)
  const size_t overrun = (size_t)std::max(ytile_rows * ytiles - nY + 1, 1) * pitch_w * 4;
  if (smem - s_bytes < overrun) smem = s_bytes + overrun;
  if (smem + sizeof(TileShared) + 64 > 227 * 1024) return refuse(5);
  p.smem = smem;
  return p;
}

// The levelled raster's smear levels: the kernel's distinct non-zero values, ascending, when there are at most 4 (else none: the
// raster takes the atomic path), and their tap masks: for level l and class c = 2 ky0 + kx0 (the first kernel row / column of a
// point's phase parity), bit 8 dy + dx for the tap ky = ky0 + 2 dy, kx = kx0 + 2 dx of that value
static void raster_levels(const std::vector<uint8_t> & kernel, int ks, TileDev & T)
{
  std::vector<uint8_t> lv(kernel.begin(), kernel.end());
  std::sort(lv.begin(), lv.end());
  lv.erase(std::unique(lv.begin(), lv.end()), lv.end());
  if (!lv.empty() && lv[0] == 0) lv.erase(lv.begin());
  T.nlevels = (!lv.empty() && lv.size() <= 4) ? (int)lv.size() : 0;
  for (int i = 0; i < 4; ++i) T.level[i] = i < T.nlevels ? lv[i] : 0;
  T.tap_masks = (T.nlevels > 0 && ks <= kTileMaxMaskKsize) ? 1 : 0;
  if (T.tap_masks)
    for (int l = 0; l < T.nlevels; ++l)
      for (int c = 0; c < 4; ++c)
        for (int ky = c >> 1; ky < ks; ky += 2)
          for (int kx = c & 1; kx < ks; kx += 2)
            if (kernel[(size_t)ky * ks + kx] == T.level[l]) T.tap_mask[l][c] |= 1ull << (8 * (ky >> 1) + (kx >> 1));
}

// One angle's groups of one stage: table of (plain begin, singles begin, singles end, pairs end) per alignment, relative to the
// angle's own payload (whose start is 4-entry aligned in the block), and the payload
struct Encoded { int32_t tbl[16]; std::vector<uint16_t> pay; };

// Classifies the beams of angle a of plan pl into c, then sorts and run-length encodes its FAST groups stage by stage into
// enc[0 .. 4 nbands).  p.tail spreads the plain lists over the lane-rows of the tail row; pairs_on pairs entries of equal weight and
// merges runs of 2 (else of 3); no_dedup keeps one entry per beam.
static void encode_angle(const GridGeom & g, const CorrPlan & pl, int a, const TilePlan & p, bool pairs_on, bool no_dedup, BeamClasses & c,
                         Encoded * enc)
{
  classify_beams(g, pl, a, p.pitch_w, p.band_rows, p.nbands, c);
  for (int sg = 0; sg < 4 * p.nbands; ++sg) {
    Encoded & E = enc[sg];
    std::vector<uint16_t> & pay = E.pay;
    pay.clear();
    for (int m = 0; m < 4; ++m) {
      std::vector<uint16_t> & gk = c.fast[sg * 4 + m];
      std::sort(gk.begin(), gk.end());
      while (pay.size() & 3) pay.push_back(0);   // the plain list is read with 64-bit loads
      const int pb = (int)pay.size();
      // run-length encode: beams that land in the same cell share one entry of weight k (one load per row, fields times
      // k), provided the whole group fits one flush.  Entries of equal weight are then paired (two loads added byte-wise,
      // one multiply per field); weight-1 beams stay in the plain list.
      std::vector<std::pair<uint16_t, uint16_t>> multi;   // (offset, weight), by ascending weight
      encode_runs(gk, pairs_on ? 2 : 3, !no_dedup && gk.size() <= (size_t)kChunkBeams, pay, multi);
      std::stable_sort(multi.begin(), multi.end(),
                       [](const std::pair<uint16_t, uint16_t> & x, const std::pair<uint16_t, uint16_t> & y) { return x.second < y.second; });
      std::vector<std::pair<uint16_t, uint16_t>> single;   // (offset, weight)
      std::vector<uint16_t> pairs;                         // offset, offset, weight, 0
      for (size_t i = 0; i < multi.size();) {
        if (pairs_on && i + 1 < multi.size() && multi[i + 1].second == multi[i].second) {
          pairs.insert(pairs.end(), {multi[i].first, multi[i + 1].first, multi[i].second, (uint16_t)0});
          i += 2;
        } else {
          single.push_back(multi[i]);
          i += 1;
        }
      }
      // the item record counts the singles in 6 bits.  With pairing there are at most 35 (see the field bounds); without it
      // (B200_TILE_PAIRS=0) every merged cell is a single: those beyond kMaxSingles - 1 (one slot stays free for the odd plain
      // beam below) go back to the plain list as k plain beams each
      while (single.size() > (size_t)kMaxSingles - 1) {
        for (uint16_t t = 0; t < single.back().second; ++t) pay.push_back(single.back().first);
        single.pop_back();
      }
      // the tail row reads entries 8 apart in each lane-row: spread the plain list's neighbouring (sorted, so nearby)
      // word offsets over the lane-rows so that their 4-word runs rarely share banks (48-row y-tiles have no tail row)
      if (p.tail) spread_rows(pay.begin() + pb, pay.end());
      // the singles (offset, weight; read as 32-bit words) start where the plain list ends: keep that index even by
      // moving an odd plain list's last entry into the singles with weight 1
      if (((int)pay.size() - pb) & 1) {
        const uint16_t last = pay.back();
        pay.pop_back();
        single.emplace_back(last, (uint16_t)1);
      }
      const int sb = (int)pay.size();
      for (auto & s1 : single) { pay.push_back(s1.first); pay.push_back(s1.second); }
      const int se = (int)pay.size();
      if (!pairs.empty()) while (pay.size() & 3) pay.push_back(0);   // the pairs are read as 64-bit words
      pay.insert(pay.end(), pairs.begin(), pairs.end());
      E.tbl[4 * m + 0] = pb; E.tbl[4 * m + 1] = sb; E.tbl[4 * m + 2] = se; E.tbl[4 * m + 3] = (int)pay.size();
    }
    while (pay.size() & 3) pay.push_back(0);
  }
}

// The descriptor blocks of one query (its angles' classes cls and encodings enc, nstage per angle) and the schedule of each CTA r
// of its cluster: the chunks r, r + C, ..., each stage of a chunk cut into sub-blocks of as many angles as fit one staging buffer.
// Appends the blocks to blob, their records to seq and each CTA's first record to seq_start, adds to ts, and returns 0 or a
// refusal code (8, 10 to 13).
static int schedule_query(const TilePlan & p, int nA, const std::vector<BeamClasses> & cls, const std::vector<Encoded> & enc,
                          std::vector<uint8_t> & blob, std::vector<TileSeq> & seq, std::vector<int32_t> & seq_start, TileStats & ts)
{
  const int C = p.C, nAc = p.nAc, nstage = 4 * p.nbands, xtiles = p.xtiles, ytiles = p.ytiles;
  std::vector<uint16_t> pay;
  std::vector<int32_t> tbl;
  std::vector<int> nedge;
  std::vector<uint2> items;
  for (int r = 0; r < C; ++r) {
    seq_start.push_back((int32_t)seq.size());
    for (int v = r; v < p.V; v += C) {
      const int ca0 = v * nAc, cna = std::min(nAc, nA - ca0);
      // the CTA's chunks alternate the stage order (phase 0 -> 3, then 3 -> 0, ...): each chunk starts on the (phase, band) the
      // one before it ended on, whose sub-grid is still resident
      const bool backward = ((v - r) / C) & 1, keep = v != r;
      for (int si = 0; si < nstage; ++si) {
        const int sg = backward ? nstage - 1 - si : si;
        // sub-blocks: as many angles as fit one staging buffer
        int a = ca0;
        bool first_sub = true;
        do {
          tbl.clear(); pay.clear();
          int na = 0, npieces = 0;   // pieces of the block's groups so far (items = pieces x tiles)
          while (a + na < ca0 + cna) {
            const Encoded & E = enc[(size_t)(a + na) * nstage + sg];
            int ep = 0;
            for (int m = 0; m < 4; ++m) ep += std::max(1, (E.tbl[4 * m + 1] - E.tbl[4 * m] + kChunkBeams - 1) / kChunkBeams);
            const size_t hdr = (((size_t)(npieces + ep) * xtiles * ytiles * 8) + 15) & ~(size_t)15;
            const size_t bytes = (hdr + (pay.size() + E.pay.size()) * 2 + 15) & ~(size_t)15;
            const bool wide = pay.size() + E.pay.size() > 65535;   // item records hold 16-bit payload indices (pb, pe)
            if (bytes > (size_t)p.stage_bytes || wide) {
              if (na > 0) break;
              return wide ? 11 : 8;   // one angle does not fit the 16-bit indices / the staging buffer
            }
            const int shift = (int)pay.size();
            for (int k = 0; k < 16; ++k) tbl.push_back(E.tbl[k] + shift);
            pay.insert(pay.end(), E.pay.begin(), E.pay.end());
            npieces += ep;
            ++na;
          }
          nedge.assign((size_t)na * 4, 0);
          for (int g2 = 0; g2 < na * 4; ++g2) nedge[g2] = (int)cls[a + (g2 >> 2)].edge[sg * 4 + (g2 & 3)].size();
          if (!build_block_items(tbl, nedge, na, xtiles, ytiles, items)) return 13;
          if (items.size() > 32767) return 10;   // TileSeq.nitems is 16-bit
          ts.blocks += 1;
          ts.sub_blocks += first_sub ? 0 : 1;
          for (int g2 = 0; g2 < na * 4; ++g2) {
            const int pb = tbl[4 * g2], mb = tbl[4 * g2 + 1], se = tbl[4 * g2 + 2], pe2 = tbl[4 * g2 + 3];
            const int ps = pe2 > se ? ((se + 3) & ~3) : se;
            ts.max_edge_group = std::max(ts.max_edge_group, nedge[g2]);
            ts.split_groups += mb - pb > kChunkBeams ? 1 : 0;
            ts.multi_entries += (se - mb) / 2 + (pe2 - ps) / 2;   // weighted entries: singles + both entries of every pair
            for (int k = mb; k < se; k += 2) ts.max_multiplicity = std::max(ts.max_multiplicity, (int32_t)pay[k + 1]);
            for (int k = ps; k < pe2; k += 4) ts.max_multiplicity = std::max(ts.max_multiplicity, (int32_t)pay[k + 2]);
            ts.max_plain_group = std::max(ts.max_plain_group, mb - pb);
          }
          const size_t hdr = ((items.size() * 8) + 15) & ~(size_t)15;
          const size_t bytes = std::max<size_t>(16, (hdr + pay.size() * 2 + 15) & ~(size_t)15);
          if (blob.size() + bytes > 0x7FFFFFF0u) return 12;   // TileSeq.off is a 32-bit byte offset
          TileSeq e{};
          e.off = (int32_t)blob.size();
          e.bytes = (int32_t)bytes;
          e.chunk = (int16_t)v; e.stage = (int16_t)sg; e.a0 = (int16_t)a; e.nitems = (int16_t)items.size();
          e.flags = (first_sub ? kSeqNewStage : 0u) | ((first_sub && si == 0) ? kSeqNewChunk : 0u) |
                    ((first_sub && si == 0 && keep) ? kSeqKeepGrid : 0u);
          if (first_sub)
            for (int aa = ca0; aa < ca0 + cna; ++aa)
              if (!cls[aa].wrap2[sg].empty()) e.flags |= kSeqHasWrap;
          blob.resize(blob.size() + bytes, 0);
          if (!items.empty()) std::memcpy(blob.data() + e.off, items.data(), items.size() * 8);
          if (!pay.empty()) std::memcpy(blob.data() + e.off + hdr, pay.data(), pay.size() * 2);
          seq.push_back(e);
          a += na;
          first_sub = false;
        } while (a < ca0 + cna);
      }
      seq.back().flags |= kSeqEndChunk;
    }
  }
  return 0;
}

// The kernel of plan p with its dynamic shared memory raised to the plan's, and its launch on ctas CTAs in clusters of p.C on
// stream st (cfg, whose cluster attribute is at)
static const void * tile_launch_config(const TilePlan & p, int ctas, cudaStream_t st, cudaLaunchConfig_t & cfg, cudaLaunchAttribute & at)
{
  const void * kfn = tile_kernel_for(p.pitch_w, p.tail != 0);
  B200_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  cfg = cudaLaunchConfig_t{};
  cfg.gridDim = dim3((unsigned)ctas);
  cfg.blockDim = dim3(kTileThreads);
  cfg.dynamicSmemBytes = p.smem;
  cfg.stream = st;
  at.id = cudaLaunchAttributeClusterDimension;
  at.val.clusterDim.x = (unsigned)p.C; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
  cfg.attrs = &at; cfg.numAttrs = 1;
  return kfn;
}

bool build_tile_tables(b200sm * h, SweepHost & S, cudaStream_t st)
{
  const GridGeom & g = h->g;
  const CorrPlan & p0 = S.plans[0];
  const int nA = p0.nA, nq = S.nq;
  auto bail = [&](int why) { S.tile_refusal = why; return false; };
  if (const int why = parity_refusal(g, S.plans)) return bail(why);
  // B200_TILE_TAIL=0 / B200_TILE_PAIRS=0 switch the tail layout / the weight-2 entries and pairing off, to measure each part alone
  const TilePlan p = plan_tile({g.stride, g.height, p0.nX, p0.nY, nA, p0.n, S.max_n, S.do_penalize ? 1 : 0, S.npairs, h->sms,
                                h->tile_cluster > 0 ? h->tile_cluster : env_int("B200_SWEEP_CLUSTER", 0),
                                h->tile_chunks > 0 ? h->tile_chunks : env_int("B200_SWEEP_CHUNKS", 0),
                                env_int("B200_TILE_TAIL", 1) != 0 ? 1 : 0});
  if (p.refused) return bail(p.refused);
  const bool pairs_on = env_int("B200_TILE_PAIRS", 1) != 0;

  // ---- per-query descriptor blocks and schedules ----
  const int nstage = 4 * p.nbands;
  std::vector<uint8_t> blob;
  std::vector<TileSeq> seq;
  std::vector<int32_t> seq_start;
  TileStats ts;
  BeamLists lists;
  std::vector<BeamClasses> cls(nA);
  std::vector<Encoded> enc((size_t)nA * nstage);
  blob.reserve((size_t)nq * nA * p0.n * 2 + 4096);
  for (int q = 0; q < nq; ++q) {
    host_parallel_for(nA, [&](int a) { encode_angle(g, S.plans[q], a, p, pairs_on, h->no_dedup, cls[a], &enc[(size_t)a * nstage]); });
    append_beam_lists(cls, nstage, lists);
    if (const int why = schedule_query(p, nA, cls, enc, blob, seq, seq_start, ts)) return bail(why);
  }
  seq_start.push_back((int32_t)seq.size());
  ts.wrap2_entries = (int32_t)lists.wrap2.size();
  blob.resize(blob.size() + 16, 0);

  S.h2d(S.d_tile_desc, blob.data(), blob.size(), st);
  S.h2d(S.d_tile_seq, seq.data(), seq.size(), st);
  S.h2d(S.d_tile_seq_start, seq_start.data(), seq_start.size(), st);
  upload_beam_lists(lists, S, st);
  TileDev & T = S.tile;
  T = TileDev{};
  T.C = p.C; T.V = p.V; T.nAc = p.nAc; T.nbands = p.nbands; T.band_rows = p.band_rows; T.alloc_rows = p.alloc_rows;
  T.pitch_w = p.pitch_w; T.xtiles = p.xtiles; T.ytiles = p.ytiles; T.tail = p.tail; T.stage_bytes = p.stage_bytes;
  T.int_ties = p.int_ties; T.off_A = p.off_A; T.off_probs = p.off_probs; T.off_stage = p.off_stage; T.off_cells = p.off_cells;
  T.cell_cap = p.cell_cap;
  raster_levels(g.kernel, g.ksize, T);
  T.desc = S.d_tile_desc.p; T.seq = S.d_tile_seq.p; T.seq_start = S.d_tile_seq_start.p;
  T.edge = S.d_edge.p; T.edge_start = S.d_edge_start.p;
  T.wrap2 = S.d_wrap2.p; T.wrap2_start = S.d_wrap2_start.p;
  T.slow = S.d_slow.p; T.slow_start = S.d_slow_start.p;
  T.enabled = 1;

  // ---- grid: as many co-resident clusters as the device holds, one pair per cluster at a time ----
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at;
  const void * kfn = tile_launch_config(p, p.C * std::max(1, h->sms / p.C), nullptr, cfg, at);
  int max_clusters = h->sms / p.C, nc = 0;
  if (cudaOccupancyMaxActiveClusters(&nc, kfn, &cfg) == cudaSuccess && nc > 0) max_clusters = nc;
  else (void)cudaGetLastError();
  S.tile_plan = p;
  S.tile_clusters = std::max(1, std::min(S.npairs, max_clusters));
  S.tile_stats = ts;
  S.tile_refusal = 0;
  return true;
}

void launch_sweep_tile(SweepHost & S, cudaStream_t st)
{
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at;
  const void * kfn = tile_launch_config(S.tile_plan, S.tile_clusters * S.tile_plan.C, st, cfg, at);
  void * args[] = {(void *)&S.dev, (void *)&S.tile};
  B200_CUDA(cudaLaunchKernelExC(&cfg, kfn, args));
}

}  // namespace b200

#ifdef B200_TILE_TIMERS
// section totals of the instrumented build, in the order of the kTm* enum: copied to out (when non-null), then zeroed when
// reset != 0.  Returns the number of sections, or -1 on a CUDA error.
extern "C" int b200_tile_timers(unsigned long long * out, int reset)
{
  using namespace b200;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (out && cudaMemcpyFromSymbol(out, g_tile_timers, sizeof(g_tile_timers)) != cudaSuccess) return -1;
  if (reset) {
    const unsigned long long zero[kTmCount] = {};
    if (cudaMemcpyToSymbol(g_tile_timers, zero, sizeof(zero)) != cudaSuccess) return -1;
  }
  return kTmCount;
}
#endif

#ifdef B200_TILE_COUNTS
// loop-trip totals of the counting build, in the order of the kCn* enum: copied to out (when non-null), then zeroed when
// reset != 0.  Returns the number of counters, or -1 on a CUDA error.
extern "C" int b200_tile_counts(unsigned long long * out, int reset)
{
  using namespace b200;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (out && cudaMemcpyFromSymbol(out, g_tile_counts, sizeof(g_tile_counts)) != cudaSuccess) return -1;
  if (reset) {
    const unsigned long long zero[kCnCount] = {};
    if (cudaMemcpyToSymbol(g_tile_counts, zero, sizeof(zero)) != cudaSuccess) return -1;
  }
  return kCnCount;
}
#endif
