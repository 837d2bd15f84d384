// b200slam scan matcher, batched loop-closure sweep: round 1's SINGLE-CTA kernel (sweep_kernel = 1).
//
// k_sweep_fast keeps one parity sub-grid and the whole (x, y, theta) accumulator volume of a pair in one SM's shared memory,
// which holds for BASELINE's 4 m / 12 m geometry (search <= 48 x 48 poses, grid rows <= 576 cells).  In auto mode it runs the
// sweeps the tiled cluster kernel (sm_tile.cu) refuses.  Its beam lists stay in global memory, so it also takes queries with
// more readings than one of the tiled kernel's descriptor blocks can stage.
// Compile with -fmad=false / -ffp-contract=off (bit-exact FP64, see sm_math.cuh).
#include <algorithm>
#include <utility>
#include <vector>

#include "common.cuh"
#include "sm_math.cuh"
#include "sm_types.cuh"
#include "sm_device.cuh"
#include "sm_sweep_dev.cuh"

namespace b200 {

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
        const int32_t * es = f.edge_start + ((size_t)q * nA + a) * 16 + ph * 4;
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

// Builds the per-query beam lists of the fast path; returns false when this sweep cannot use it.
bool build_fast_tables(b200sm * h, SweepHost & S, cudaStream_t st)
{
  const GridGeom & g = h->g;
  const CorrPlan & p0 = S.plans[0];
  const int nX = p0.nX, nY = p0.nY, nA = p0.nA, n = p0.n, nq = S.nq;
  auto bail = [&](int why) { S.fast_refusal = why; return false; };
  if (const int why = parity_refusal(g, S.plans)) return bail(why);
  if (nY > 8 * kFastRowTiles || (g.stride & 1) || nX * nY > 3 * kFastThreads) return bail(2);
  if (g.stride / 2 > kSubPitchW * 4 - 16) return bail(3);   // sub-grid row + the 3-word overhang must fit the pitch
  const int xtiles = (nX + 3 + 15) / 16;
  int sub_rows = (g.height + 1) / 2 + 8;                     // + padding rows read by idle row tiles
  // the S region doubles as the FP64 scratch of the reduction (5 P doubles): small grids get extra rows for it
  sub_rows = std::max(sub_rows, (int)(((size_t)5 * nX * nY * sizeof(double) + kSubPitchW * 4 - 1) / (kSubPitchW * 4)));
  const size_t smem = (size_t)sub_rows * kSubPitchW * 4 + (size_t)nA * nX * nY * 4;
  if (smem > 227 * 1024 - 1024) return bail(4);
  if ((size_t)5 * nX * nY * sizeof(double) > (size_t)sub_rows * kSubPitchW * 4) return bail(5);   // epilogue scratch reuses S
  std::vector<int32_t> cls_start((size_t)nq * nA * 33);
  std::vector<uint16_t> beams, mult;
  BeamLists lists;
  beams.reserve((size_t)nq * nA * n);
  mult.reserve((size_t)nq * nA * n);
  // one angle's lists, built independently (one host-pool task per angle), then concatenated in angle order: its beam classes
  // (one band: stage = phase) and the FAST descriptors
  struct AngleLists {
    std::vector<uint16_t> beams, mult;
    int32_t cs[33];                          // relative to the angle's first descriptor
  };
  std::vector<BeamClasses> cls(nA);
  std::vector<AngleLists> al(nA);
  for (int q = 0; q < nq; ++q) {
    const CorrPlan & pl = S.plans[q];
    auto one_angle = [&](int a) {
      AngleLists & L = al[a];
      classify_beams(g, pl, a, kSubPitchW, sub_rows, 1, cls[a]);
      L.beams.clear(); L.mult.clear();
      for (int k = 0; k < 16; ++k) {
        std::vector<uint16_t> & gk = cls[a].fast[k];
        std::sort(gk.begin(), gk.end());
        L.cs[2 * k] = (int32_t)L.beams.size();
        // beams that land in the same cell share a descriptor: runs of >= 3 go to the group's multi list (one load, fields
        // multiplied), provided the whole group fits one flush
        std::vector<std::pair<uint16_t, uint16_t>> multi;
        encode_runs(gk, 3, !h->no_dedup && gk.size() <= (size_t)kFastChunk, L.beams, multi);
        L.mult.resize(L.beams.size(), 1);
        L.cs[2 * k + 1] = (int32_t)L.beams.size();
        for (auto & mk : multi) { L.beams.push_back(mk.first); L.mult.push_back(mk.second); }
      }
      L.cs[32] = (int32_t)L.beams.size();
    };
    host_parallel_for(nA, one_angle);
    append_beam_lists(cls, 4, lists);
    for (int a = 0; a < nA; ++a) {
      const AngleLists & L = al[a];
      int32_t * cs = &cls_start[((size_t)q * nA + a) * 33];
      const int32_t base = (int32_t)beams.size();
      for (int k = 0; k < 33; ++k) cs[k] = base + L.cs[k];
      beams.insert(beams.end(), L.beams.begin(), L.beams.end());
      mult.insert(mult.end(), L.mult.begin(), L.mult.end());
    }
  }
  S.h2d(S.d_fast_cls, cls_start.data(), cls_start.size(), st);
  S.d_fast_beams.reserve(std::max<size_t>(beams.size(), 1) + 8);
  S.stage(S.d_fast_beams.p, beams.data(), beams.size() * sizeof(uint16_t), st);
  S.d_fast_mult.reserve(std::max<size_t>(mult.size(), 1) + 8);
  S.stage(S.d_fast_mult.p, mult.data(), mult.size() * sizeof(uint16_t), st);
  upload_beam_lists(lists, S, st);
  S.beam_counts[0] = (int32_t)beams.size();   // this kernel counts FAST descriptors, not beams
  S.fast.enabled = 1;
  S.fast_refusal = 0;
  S.fast.sub_rows = sub_rows;
  S.fast.xtiles = xtiles;
  S.fast.beams = S.d_fast_beams.p;
  S.fast.mult = S.d_fast_mult.p;
  S.fast.cls_start = S.d_fast_cls.p;
  S.fast.slow = S.d_slow.p;
  S.fast.edge = S.d_edge.p;
  S.fast.edge_start = S.d_edge_start.p;
  S.fast.wrap2 = S.d_wrap2.p;
  S.fast.wrap2_start = S.d_wrap2_start.p;
  S.fast.slow_start = S.d_slow_start.p;
  S.fast_smem = smem;
  S.fast_blocks = std::min(S.npairs, h->sms);
  return true;
}

void launch_sweep_fast(SweepHost & S, cudaStream_t st)
{
  B200_CUDA(cudaFuncSetAttribute(k_sweep_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S.fast_smem));
  k_sweep_fast<<<S.fast_blocks, kFastThreads, S.fast_smem, st>>>(S.dev, S.fast);
}

}  // namespace b200
