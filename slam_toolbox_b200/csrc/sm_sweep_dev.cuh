// Block-level reductions, the response expression and the pair epilogue shared by the sweep kernels (sm_sweep.cu,
// sm_fast.cu, sm_tile.cu).
#pragma once
#include "sm_math.cuh"
#include "sm_types.cuh"

namespace b200 {

__device__ __forceinline__ double block_max(double v, double * scratch)
{
  for (int o = 16; o > 0; o >>= 1) {
    double other = __shfl_xor_sync(0xffffffffu, v, o);
    v = other > v ? other : v;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  double r = scratch[0];
  for (int i = 1; i < nw; ++i) r = scratch[i] > r ? scratch[i] : r;
  __syncthreads();
  return r;
}

// exclusive prefix sum of one int per thread over the block; returns the exclusive value and
// writes the block total
__device__ __forceinline__ int block_exclusive_scan(int v, int * scratch, int & total)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  int base = 0, tot = 0;
  for (int i = 0; i < nw; ++i) {
    if (i < warp) base += scratch[i];
    tot += scratch[i];
  }
  __syncthreads();
  total = tot;
  return base + inc - v;
}

// response of pose (xy, a) from its integer sum, exactly as ScanMatcher::operator() builds it
// (M.cpp:670-685)
__device__ __forceinline__ double pose_response(const SweepDev & d, int q, int sum, int x, int y, int a)
{
  double r = (double)sum;
  r /= d.norm;
  if (d.do_penalize && !double_equal(r, 0.0)) {
    double dp = distance_penalty(d.sqx[q * d.nX + x], d.sqy[q * d.nY + y], d.dist_var, d.min_dist_pen);
    double ap = d.angpen[q * d.nA + a];
    r *= (dp * ap);
  }
  return r;
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

}  // namespace b200
