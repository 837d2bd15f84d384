// b200slam SE(2) pose-graph solver: the karto::ScanSolver surface
// (lib/karto_sdk/include/karto_sdk/Mapper.h:954-1065) as solver_plugins::CeresSolver
// implements it (solvers/ceres_solver.cpp, solvers/ceres_utils.h), rebuilt for one H100:
//
//   * problem: nodes (x, y, theta), edges with relative-pose measurement z and sqrt-information
//     U = chol(cov^-1).matrixU() (ceres_solver.cpp:364-376); residual r = U [R(th_a)^T (p_b - p_a)
//     - t ; wrap(th_b - th_a - th_ab)] (ceres_utils.h:84-100); first node constant (:228-241).
//   * outer loop: Ceres' TrustRegionMinimizer (with TrustRegionStepEvaluator) and the reference's options
//     (ceres_solver.cpp:158-186), driven from the host with one small D2H of scalars per step, around one of two step
//     strategies: LevenbergMarquardtStrategy (the default) or DoglegStrategy, traditional or subspace (DESIGN.md §4).
//   * inner solve: instead of SPARSE_NORMAL_CHOLESKY, preconditioned CG on the 3x3-block normal equations inside ONE
//     persistent cooperative kernel per solve, planned from the graph's rows: two-level (block Jacobi plus 6 or 3 coarse modes
//     per aggregate, flag exchanges between CTAs; the default), the same two-level preconditioner on global-memory aggregates
//     with a dense coarse inverse (graphs too large for shared memory), block Jacobi with each CTA's rows in shared memory, or
//     block Jacobi from global memory. Reductions are summed in a fixed order.  Opt-in (linear_solver_type = 1): the exact solve
//     SPARSE_NORMAL_CHOLESKY does, a supernodal FP64 Cholesky in one persistent cooperative kernel per solve (k_pg_cholesky)
//     after a host symbolic analysis (cholesky_analyze).
//   * one fused kernel evaluates every edge's residual, both Jacobian blocks (analytic) and the
//     off-diagonal normal-equation block; a second gathers per-node diagonal blocks/gradients
//     through a CSR node->edge adjacency (no atomics: bit-reproducible results).
//
// Data layout (HBM, FP64): nodes AoS [N][3]; edges SoA-of-small-arrays: idx[E][2], z[E][3],
// U[E][6] (upper triangle), lin[E][30] = r(3) | A~(9) | B~(9) | M = A~^T B~ (9); node blocks
// Hd[N][6] (symmetric), g[N][3]. The whole 10k/40k problem is ~15 MB: L2 resident.
#include <cooperative_groups.h>

#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <complex>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b200 {

constexpr int kPgThreads = 256;
constexpr int kLin = 30;   // doubles per edge in the linearisation record
constexpr int kMaxPartials = 1024;

struct PgDev {
  int N, E;
  const int32_t * eidx;     // [E][2] node indices
  const double * z;         // [E][3]
  const double * U;         // [E][6] u00 u01 u02 u11 u12 u22
  const uint8_t * is_free;  // [N] 1 = optimised, 0 = constant / not in the problem
  const int32_t * adj_start;   // [N+1]
  const int32_t * adj;         // [2E] (edge << 1) | side   (side 0: node is a, 1: node is b)
  double * x;               // [N][3] current iterate
  double * xc;              // [N][3] candidate
  double * scale;           // [N][3] Jacobi column scaling
  double * lin;             // [E][30]
  double * Hd;              // [N][6] diag blocks of J~^T J~ (xx xy xt yy yt tt)
  double * g;               // [N][3] J~^T r
  double * diag;            // [N][3] LM diagonal (clamped squared column norms)
  double * y;               // [N][3] PCG solution of (H + D^2) y = g
  double * pr, * pz, * pp0, * pp1, * pq, * Minv;   // PCG work vectors [N][3], Minv [N][6]
  double * partial;         // [kMaxPartials * 4] per-CTA partial sums
  double * scalars;         // small result block
  int loss;                 // 0 none, 1 Huber, 2 Cauchy (ceres_solver.cpp:82-94)
  double loss_a;            // loss scale
};

__device__ __forceinline__ double wrap_angle(double a)   // ceres_utils.h:27-32
{
  const double two_pi = 2.0 * M_PI;
  return a - two_pi * floor((a + M_PI) / two_pi);
}

__device__ __forceinline__ double warp_sum(double v)
{
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v)
{
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// deterministic block reduction of up to 4 values; result valid in thread 0
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double * smem /* K*32 */)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
  __syncthreads();
  if (lane == 0)
    for (int k = 0; k < K; ++k) smem[k * 32 + warp] = v[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) {
      double s = 0;
      for (int w = 0; w < nw; ++w) s += smem[k * 32 + w];
      v[k] = s;
    }
  }
}

// residual of one edge at poses (pa, pb): PoseGraph2dErrorTerm::operator() (ceres_utils.h:84-100)
__device__ __forceinline__ void edge_residual(const double * pa, const double * pb, const double * z, const double * U,
                                              double & c, double & s, double & dx, double & dy, double r[3])
{
  sincos(pa[2], &s, &c);
  dx = pb[0] - pa[0]; dy = pb[1] - pa[1];
  const double e0 = c * dx + s * dy - z[0];
  const double e1 = -s * dx + c * dy - z[1];
  const double e2 = wrap_angle((pb[2] - pa[2]) - z[2]);
  r[0] = U[0] * e0 + U[1] * e1 + U[2] * e2;
  r[1] = U[3] * e1 + U[4] * e2;
  r[2] = U[5] * e2;
}

// ceres::LossFunction::Evaluate for the two losses the reference offers: rho(s) and rho'(s), s = ||r||^2.
// Both have rho'' <= 0, for which Ceres' Corrector reduces to scaling residual and Jacobian by sqrt(rho').
__device__ __forceinline__ void loss_eval(int loss, double a, double s, double & rho, double & rho1)
{
  const double b = a * a;
  if (loss == 1) {          // HuberLoss
    if (s > b) { const double r = sqrt(s); rho = 2.0 * a * r - b; rho1 = fmax(2.2250738585072014e-308, a / r); }
    else { rho = s; rho1 = 1.0; }
  } else if (loss == 2) {   // CauchyLoss
    const double sum = 1.0 + s / b;
    rho = b * log(sum); rho1 = fmax(2.2250738585072014e-308, 1.0 / sum);
  } else { rho = s; rho1 = 1.0; }
}

// Fused linearisation: residual, Jacobian blocks w.r.t. node a and b (analytic form of the
// reference's autodiff), Jacobi column scaling, off-diagonal normal block M = A~^T B~, cost partial.
// mode 0: full linearisation at d.x into d.lin ; mode 1: cost only at d.xc.
__global__ void __launch_bounds__(kPgThreads) k_pg_linearize(PgDev d, int mode)
{
  __shared__ double red[32];
  double cost[1] = {0.0};
  const double * X = mode == 0 ? d.x : d.xc;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < d.E; e += gridDim.x * blockDim.x) {
    const int a = d.eidx[2 * e], b = d.eidx[2 * e + 1];
    const double * pa = X + 3 * a, * pb = X + 3 * b;
    const double * U = d.U + 6 * e;
    double c, s, dx, dy, r[3];
    edge_residual(pa, pb, d.z + 3 * e, U, c, s, dx, dy, r);
    const double sq = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double w = 1.0;   // sqrt(rho'): Corrector::CorrectResiduals / CorrectJacobian for rho'' <= 0
    if (d.loss) {
      double rho, rho1;
      loss_eval(d.loss, d.loss_a, sq, rho, rho1);
      cost[0] += rho;
      w = sqrt(rho1);
    } else {
      cost[0] += sq;
    }
    if (mode == 1) continue;
    r[0] *= w; r[1] *= w; r[2] *= w;
    // de/d(xa,ya,tha) and de/d(xb,yb,thb)
    const double Ae[9] = {-c, -s, -s * dx + c * dy, s, -c, -c * dx - s * dy, 0.0, 0.0, -1.0};
    const double Be[9] = {c, s, 0.0, -s, c, 0.0, 0.0, 0.0, 1.0};
    double A[9], B[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      A[0 + j] = U[0] * Ae[0 + j] + U[1] * Ae[3 + j] + U[2] * Ae[6 + j];
      A[3 + j] = U[3] * Ae[3 + j] + U[4] * Ae[6 + j];
      A[6 + j] = U[5] * Ae[6 + j];
      B[0 + j] = U[0] * Be[0 + j] + U[1] * Be[3 + j] + U[2] * Be[6 + j];
      B[3 + j] = U[3] * Be[3 + j] + U[4] * Be[6 + j];
      B[6 + j] = U[5] * Be[6 + j];
    }
    const double fa = d.is_free[a] ? w : 0.0, fb = d.is_free[b] ? w : 0.0;
    const double * sa = d.scale + 3 * a, * sb = d.scale + 3 * b;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) { A[3 * i + j] *= fa * sa[j]; B[3 * i + j] *= fb * sb[j]; }
    double * L = d.lin + (size_t)kLin * e;
    L[0] = r[0]; L[1] = r[1]; L[2] = r[2];
#pragma unroll
    for (int k = 0; k < 9; ++k) { L[3 + k] = A[k]; L[12 + k] = B[k]; }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) L[21 + 3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
  }
  block_sum<1>(cost, red);
  if (threadIdx.x == 0) d.partial[blockIdx.x] = 0.5 * cost[0];
}

// Per node: diagonal block and gradient of the (scaled) normal equations gathered over incident
// edges in CSR order; squared column norms; ||x - Plus(x, -g_unscaled)||_inf partial (Ceres'
// gradient_max_norm); ||x||^2 partial over the free parameters.
__global__ void __launch_bounds__(kPgThreads) k_pg_assemble(PgDev d, int first /* compute Jacobi scaling */)
{
  __shared__ double red[64];
  double gmax = 0.0;
  double sums[1] = {0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.N; i += gridDim.x * blockDim.x) {
    double h[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    for (int k = d.adj_start[i]; k < d.adj_start[i + 1]; ++k) {
      const int e = d.adj[k] >> 1, side = d.adj[k] & 1;
      const double * L = d.lin + (size_t)kLin * e;
      const double * J = L + (side ? 12 : 3);
      h[0] += J[0] * J[0] + J[3] * J[3] + J[6] * J[6];
      h[1] += J[0] * J[1] + J[3] * J[4] + J[6] * J[7];
      h[2] += J[0] * J[2] + J[3] * J[5] + J[6] * J[8];
      h[3] += J[1] * J[1] + J[4] * J[4] + J[7] * J[7];
      h[4] += J[1] * J[2] + J[4] * J[5] + J[7] * J[8];
      h[5] += J[2] * J[2] + J[5] * J[5] + J[8] * J[8];
      g[0] += J[0] * L[0] + J[3] * L[1] + J[6] * L[2];
      g[1] += J[1] * L[0] + J[4] * L[1] + J[7] * L[2];
      g[2] += J[2] * L[0] + J[5] * L[1] + J[8] * L[2];
    }
    if (first) {
      // jacobian_scaling = 1 / (1 + sqrt(squared column norm)) from the UNSCALED Jacobian
      // (scale was all ones for this pass); the caller re-linearises with it afterwards
      d.scale[3 * i + 0] = 1.0 / (1.0 + sqrt(h[0]));
      d.scale[3 * i + 1] = 1.0 / (1.0 + sqrt(h[3]));
      d.scale[3 * i + 2] = 1.0 / (1.0 + sqrt(h[5]));
      continue;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) d.Hd[6 * i + k] = h[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) d.g[3 * i + k] = g[k];
    if (d.is_free[i]) {
      const double * x = d.x + 3 * i, * sc = d.scale + 3 * i;
      // unscaled gradient g / s ; Plus(x, -g): x,y plain, theta wrapped
      const double g0 = g[0] / sc[0], g1 = g[1] / sc[1], g2 = g[2] / sc[2];
      gmax = fmax(gmax, fabs(x[0] - (x[0] - g0)));
      gmax = fmax(gmax, fabs(x[1] - (x[1] - g1)));
      gmax = fmax(gmax, fabs(x[2] - wrap_angle(x[2] - g2)));
      sums[0] += x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    }
  }
  if (first) return;
  block_sum<1>(sums, red);
  gmax = warp_max(gmax);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[32 + (threadIdx.x >> 5)] = gmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, red[32 + w]);
    d.partial[blockIdx.x] = sums[0];
    d.partial[kMaxPartials + blockIdx.x] = m;
  }
}

// LM diagonal: clamp(squared column norms) (LevenbergMarquardtStrategy::ComputeStep)
__global__ void k_pg_diag(PgDev d, double min_diag, double max_diag)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.N; i += gridDim.x * blockDim.x) {
    d.diag[3 * i + 0] = fmin(fmax(d.Hd[6 * i + 0], min_diag), max_diag);
    d.diag[3 * i + 1] = fmin(fmax(d.Hd[6 * i + 3], min_diag), max_diag);
    d.diag[3 * i + 2] = fmin(fmax(d.Hd[6 * i + 5], min_diag), max_diag);
  }
}

// final reduction of per-CTA partials in fixed order (one warp)
__global__ void k_pg_reduce(PgDev d, int nparts, int slot_sum, int slot_max)
{
  if (threadIdx.x != 0) return;
  double s = 0, m = 0;
  for (int i = 0; i < nparts; ++i) { s += d.partial[i]; m = fmax(m, d.partial[kMaxPartials + i]); }
  if (slot_sum >= 0) d.scalars[slot_sum] = s;
  if (slot_max >= 0) d.scalars[slot_max] = m;
}

__device__ __forceinline__ double ld_cg(const double * p) { return __ldcg(p); }

// y_i = sum_j A_ij v_j for the scaled normal matrix plus damping: (Hd_i + D_i^2) v_i + sum_e M v_other.
// kL2: read v0 / v1 through L2 (ld.global.cg), for vectors other CTAs of the same launch write between flag exchanges.
template <bool kL2 = false>
__device__ __forceinline__ void spmv_row(const PgDev & d, int i, const double * __restrict__ v0,
                                         const double * __restrict__ v1, double beta, double inv_radius, double out[3],
                                         double vi[3])
{
  // effective vector v = v0 + beta * v1 (v1 may be null)
  auto ldv = [](const double * p) { return kL2 ? ld_cg(p) : *p; };
  auto ld = [&](int j, double w[3]) {
    w[0] = ldv(v0 + 3 * j); w[1] = ldv(v0 + 3 * j + 1); w[2] = ldv(v0 + 3 * j + 2);
    if (v1) { w[0] += beta * ldv(v1 + 3 * j); w[1] += beta * ldv(v1 + 3 * j + 1); w[2] += beta * ldv(v1 + 3 * j + 2); }
  };
  ld(i, vi);
  const double * h = d.Hd + 6 * i, * dg = d.diag + 3 * i;
  out[0] = (h[0] + dg[0] * inv_radius) * vi[0] + h[1] * vi[1] + h[2] * vi[2];
  out[1] = h[1] * vi[0] + (h[3] + dg[1] * inv_radius) * vi[1] + h[4] * vi[2];
  out[2] = h[2] * vi[0] + h[4] * vi[1] + (h[5] + dg[2] * inv_radius) * vi[2];
  for (int k = d.adj_start[i]; k < d.adj_start[i + 1]; ++k) {
    const int e = d.adj[k] >> 1, side = d.adj[k] & 1;
    const double * M = d.lin + (size_t)kLin * e + 21;
    const int other = d.eidx[2 * e + (side ? 0 : 1)];
    double w[3];
    ld(other, w);
    if (side == 0) {   // row block a: M w_b
      out[0] += M[0] * w[0] + M[1] * w[1] + M[2] * w[2];
      out[1] += M[3] * w[0] + M[4] * w[1] + M[5] * w[2];
      out[2] += M[6] * w[0] + M[7] * w[1] + M[8] * w[2];
    } else {           // row block b: M^T w_a
      out[0] += M[0] * w[0] + M[3] * w[1] + M[6] * w[2];
      out[1] += M[1] * w[0] + M[4] * w[1] + M[7] * w[2];
      out[2] += M[2] * w[0] + M[5] * w[1] + M[8] * w[2];
    }
  }
}

// Sum of the per-CTA partials of one slot. Warp 0 of every CTA adds them in the same fixed order,
// so every CTA obtains the identical value (deterministic, no atomics); broadcast through smem.
__device__ __forceinline__ double grid_total(const PgDev & d, int slot, int nblk, double * sh)
{
  if (threadIdx.x < 32) {
    const volatile double * p = d.partial + (size_t)slot * kMaxPartials;
    double s = 0;
    for (int i = threadIdx.x; i < nblk; i += 32) s += p[i];
    s = warp_sum(s);
    if (threadIdx.x == 0) sh[0] = s;
  }
  __syncthreads();
  const double r = sh[0];
  __syncthreads();
  return r;
}

// ---- steps the PCG kernels share ----
// Row r of the product of a symmetric 3x3 block stored as its upper triangle (xx xy xt yy yt tt) with v: H p and M^-1 r.
__device__ __forceinline__ double sym3_row(const double * m, int r, double v0, double v1, double v2)
{
  double q;
  if (r == 0) q = m[0] * v0 + m[1] * v1 + m[2] * v2;
  else if (r == 1) q = m[1] * v0 + m[3] * v1 + m[4] * v2;
  else q = m[2] * v0 + m[4] * v1 + m[5] * v2;
  return q;
}

// Block-Jacobi block a = Hd_i + D_i^2 / radius of node i (upper triangle) and its inverse mi by cofactors.
__device__ __forceinline__ void jacobi_block(const PgDev & d, int i, double inv_radius, double a[6], double mi[6])
{
  const double * h = d.Hd + 6 * i, * dg = d.diag + 3 * i;
  const double a00 = h[0] + dg[0] * inv_radius, a01 = h[1], a02 = h[2], a11 = h[3] + dg[1] * inv_radius, a12 = h[4],
               a22 = h[5] + dg[2] * inv_radius;
  a[0] = a00; a[1] = a01; a[2] = a02; a[3] = a11; a[4] = a12; a[5] = a22;
  const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
  const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
  const double id = 1.0 / (a00 * c00 + a01 * c01 + a02 * c02);
  mi[0] = c00 * id; mi[1] = c01 * id; mi[2] = c02 * id; mi[3] = c11 * id; mi[4] = c12 * id; mi[5] = c22 * id;
}

// The shared-memory kernels keep one CTA's rows [lo, hi) of the normal matrix: the off-diagonal blocks in CSR slot order
// (sB, oriented for the row's node), each slot's neighbour (sCol) and the rows' starts (sStart); the CTA's vectors are
// indexed by 3 * (node - lo) + component.

// load the CTA's off-diagonal row blocks: M of the edge for side a, M^T for side b
__device__ __forceinline__ void load_row_blocks(const PgDev & d, int s_lo, int nslots, double * sB, int * sCol)
{
  const int tid = threadIdx.x, T = blockDim.x;
  for (int s = tid; s < nslots; s += T) {
    const int a = d.adj[s_lo + s];
    const int e = a >> 1, side = a & 1;
    const double * M = d.lin + (size_t)kLin * e + 21;
    sCol[s] = d.eidx[2 * e + (side ? 0 : 1)];
    double * B = sB + 9 * s;
    if (side == 0) {
#pragma unroll
      for (int k = 0; k < 9; ++k) B[k] = M[k];
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) B[3 * i + j] = M[3 * j + i];
    }
  }
}

// sV[slot] = z + beta p of the slot's neighbour: from shared memory for an own node, else from the published gz / gpo
__device__ __forceinline__ void gather_neighbours(const int * sCol, int nslots, int lo, int hi, const double * sZ, const double * sP,
                                                  const double * gz, const double * gpo, double beta, double * sV)
{
  const int tid = threadIdx.x, T = blockDim.x;
  for (int s = tid; s < nslots; s += T) {
    const int j = sCol[s];
    double v0, v1, v2;
    if (j >= lo && j < hi) {
      const int n = j - lo;
      v0 = sZ[3 * n] + beta * sP[3 * n]; v1 = sZ[3 * n + 1] + beta * sP[3 * n + 1]; v2 = sZ[3 * n + 2] + beta * sP[3 * n + 2];
    } else {
      v0 = ld_cg(gz + 3 * j) + beta * ld_cg(gpo + 3 * j);
      v1 = ld_cg(gz + 3 * j + 1) + beta * ld_cg(gpo + 3 * j + 1);
      v2 = ld_cg(gz + 3 * j + 2) + beta * ld_cg(gpo + 3 * j + 2);
    }
    sV[3 * s] = v0; sV[3 * s + 1] = v1; sV[3 * s + 2] = v2;
  }
  __syncthreads();
}

// new search direction p = z + beta p of the own nodes (after the gather has read the old one), published to gpn;
// sQ is free until the SpMV and holds p meanwhile
__device__ __forceinline__ void new_direction(int n3, double beta, const double * sZ, double * sP, double * sQ, double * gpn)
{
  const int tid = threadIdx.x, T = blockDim.x;
  for (int k = tid; k < n3; k += T) sQ[k] = sZ[k] + beta * sP[k];
  __syncthreads();
  for (int k = tid; k < n3; k += T) { sP[k] = sQ[k]; gpn[k] = sQ[k]; }
  __syncthreads();
}

// component k = 3 n + r of q = A p for own node n: its diagonal block times p_n plus its row blocks times the gathered sV
__device__ __forceinline__ double own_row_spmv(int k, const double * sH, const double * sP, const double * sB, const double * sV,
                                               const int * sStart)
{
  const int n = k / 3, r = k - 3 * n;
  double q = sym3_row(sH + 6 * n, r, sP[3 * n], sP[3 * n + 1], sP[3 * n + 2]);
  for (int s = sStart[n]; s < sStart[n + 1]; ++s) {
    const double * B = sB + 9 * s + 3 * r, * v = sV + 3 * s;
    q += B[0] * v[0] + B[1] * v[1] + B[2] * v[2];
  }
  return q;
}

// Persistent cooperative PCG: solves (J~^T J~ + D^2/radius) y = J~^T r with the block-Jacobi
// preconditioner M_i = (Hd_i + D_i^2/radius)^-1.  Constant / unused nodes have zero Jacobian
// columns, so their rows reduce to D^2 y = 0.  scalars[8] = iterations, [9] = final relative residual.
__global__ void __launch_bounds__(kPgThreads) k_pg_pcg(PgDev d, double inv_radius, double tol, int max_iter)
{
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[4 * 32];
  __shared__ double bc[1];
  const int nblk = gridDim.x;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;

  // prologue: Minv, r = b, y = 0, z = Minv r, partials of b.b and r.z
  double acc[2] = {0, 0};
  for (int i = tid; i < d.N; i += nth) {
    double a[6], * mi = d.Minv + 6 * i;
    jacobi_block(d, i, inv_radius, a, mi);
    const double b0 = d.g[3 * i], b1 = d.g[3 * i + 1], b2 = d.g[3 * i + 2];
    d.pr[3 * i] = b0; d.pr[3 * i + 1] = b1; d.pr[3 * i + 2] = b2;
    d.y[3 * i] = 0; d.y[3 * i + 1] = 0; d.y[3 * i + 2] = 0;
    const double z0 = sym3_row(mi, 0, b0, b1, b2), z1 = sym3_row(mi, 1, b0, b1, b2), z2 = sym3_row(mi, 2, b0, b1, b2);
    d.pz[3 * i] = z0; d.pz[3 * i + 1] = z1; d.pz[3 * i + 2] = z2;
    d.pp0[3 * i] = 0; d.pp0[3 * i + 1] = 0; d.pp0[3 * i + 2] = 0;
    acc[0] += b0 * b0 + b1 * b1 + b2 * b2;
    acc[1] += b0 * z0 + b1 * z1 + b2 * z2;
  }
  block_sum<2>(acc, red);
  if (threadIdx.x == 0) { d.partial[blockIdx.x] = acc[0]; d.partial[kMaxPartials + blockIdx.x] = acc[1]; }
  grid.sync();
  const double bb = grid_total(d, 0, nblk, bc);
  double rz = grid_total(d, 1, nblk, bc);
  double rr = bb;
  const double stop = tol * tol * bb;
  int it = 0;
  double beta = 0.0;
  double * p_old = d.pp0, * p_new = d.pp1;
  if (bb > 0.0) {
    while (it < max_iter) {
      // phase A: p_new = z + beta p_old ; q = A p_new ; partial p.q
      double a1[1] = {0};
      for (int i = tid; i < d.N; i += nth) {
        double q[3], pi[3];
        spmv_row(d, i, d.pz, p_old, beta, inv_radius, q, pi);
        p_new[3 * i] = pi[0]; p_new[3 * i + 1] = pi[1]; p_new[3 * i + 2] = pi[2];
        d.pq[3 * i] = q[0]; d.pq[3 * i + 1] = q[1]; d.pq[3 * i + 2] = q[2];
        a1[0] += pi[0] * q[0] + pi[1] * q[1] + pi[2] * q[2];
      }
      block_sum<1>(a1, red);
      if (threadIdx.x == 0) d.partial[2 * kMaxPartials + blockIdx.x] = a1[0];
      grid.sync();
      const double pq = grid_total(d, 2, nblk, bc);
      const double alpha = rz / pq;
      // phase B: y += alpha p ; r -= alpha q ; z = Minv r ; partials r.z, r.r
      double a2[2] = {0, 0};
      for (int i = tid; i < d.N; i += nth) {
        double r0 = d.pr[3 * i] - alpha * d.pq[3 * i], r1 = d.pr[3 * i + 1] - alpha * d.pq[3 * i + 1],
               r2 = d.pr[3 * i + 2] - alpha * d.pq[3 * i + 2];
        d.y[3 * i] += alpha * p_new[3 * i]; d.y[3 * i + 1] += alpha * p_new[3 * i + 1]; d.y[3 * i + 2] += alpha * p_new[3 * i + 2];
        d.pr[3 * i] = r0; d.pr[3 * i + 1] = r1; d.pr[3 * i + 2] = r2;
        const double * mi = d.Minv + 6 * i;
        const double z0 = sym3_row(mi, 0, r0, r1, r2), z1 = sym3_row(mi, 1, r0, r1, r2), z2 = sym3_row(mi, 2, r0, r1, r2);
        d.pz[3 * i] = z0; d.pz[3 * i + 1] = z1; d.pz[3 * i + 2] = z2;
        a2[0] += r0 * z0 + r1 * z1 + r2 * z2;
        a2[1] += r0 * r0 + r1 * r1 + r2 * r2;
      }
      block_sum<2>(a2, red);
      // alternate partial slots so a fast CTA cannot overwrite values a slow one still reads
      const int s0 = 3 + 2 * (it & 1);
      if (threadIdx.x == 0) { d.partial[s0 * kMaxPartials + blockIdx.x] = a2[0]; d.partial[(s0 + 1) * kMaxPartials + blockIdx.x] = a2[1]; }
      grid.sync();
      const double rz_new = grid_total(d, s0, nblk, bc);
      rr = grid_total(d, s0 + 1, nblk, bc);
      ++it;
      if (!(rr > stop) || !(pq > 0.0)) break;
      beta = rz_new / rz;
      rz = rz_new;
      double * t = p_old; p_old = p_new; p_new = t;
    }
  }
  if (tid == 0) {
    d.scalars[8] = (double)it;
    d.scalars[9] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
  }
}

// ------------------------------------------------------------------------------------------
// k_pg_pcg_smem: the same PCG, restructured for graphs whose per-CTA share fits shared memory
// (cfg4: 68 nodes / ~550 off-diagonal blocks per CTA).  Each CTA owns a contiguous range of nodes and
// keeps THEIR rows of the block-sparse normal matrix (3x3 blocks, already oriented), the diagonal
// blocks, the preconditioner and all CG vectors of its nodes in shared memory for the whole solve.
// Per CG iteration the only global traffic is the neighbour gather of z and p (L2) and 2 light
// grid barriers (one atomic counter; partial dot products are summed by every CTA in the same fixed
// order, so the result is bit-reproducible).
// ------------------------------------------------------------------------------------------
struct PcgSmemCfg {
  int npc;          // nodes per CTA
  int max_slots;    // max off-diagonal blocks of one CTA
  double * gz;      // [N][3]
  double * gp;      // [2][N][3]
  unsigned int * bar;   // barrier counter (zeroed before launch)
};

__device__ __forceinline__ void grid_barrier(unsigned int * bar, unsigned int target)
{
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(512, 1) k_pg_pcg_smem(PgDev d, PcgSmemCfg c, double inv_radius, double tol, int max_iter)
{
  extern __shared__ __align__(16) unsigned char sm_raw[];
  __shared__ double red[4 * 32];
  __shared__ double bc[1];
  const int T = blockDim.x, tid = threadIdx.x, G = gridDim.x;
  const int lo = min(d.N, (int)blockIdx.x * c.npc), hi = min(d.N, lo + c.npc), nloc = hi - lo;
  const int s_lo = d.adj_start[lo], nslots = d.adj_start[hi] - s_lo;
  double * sB = reinterpret_cast<double *>(sm_raw);            // [max_slots][9]
  double * sV = sB + (size_t)c.max_slots * 9;                  // [max_slots][3]
  double * sH = sV + (size_t)c.max_slots * 3;                  // [npc][6]
  double * sMi = sH + (size_t)c.npc * 6;                       // [npc][6]
  double * sR = sMi + (size_t)c.npc * 6;                       // [npc][3] each below
  double * sZ = sR + (size_t)c.npc * 3;
  double * sP = sZ + (size_t)c.npc * 3;
  double * sQ = sP + (size_t)c.npc * 3;
  double * sY = sQ + (size_t)c.npc * 3;
  int * sCol = reinterpret_cast<int *>(sY + (size_t)c.npc * 3);   // [max_slots]
  int * sStart = sCol + c.max_slots;                              // [npc + 1]
  unsigned int bar_target = 0;

  // ---- prologue: load this CTA's rows ----
  for (int i = tid; i <= nloc; i += T) sStart[i] = d.adj_start[lo + i] - s_lo;
  load_row_blocks(d, s_lo, nslots, sB, sCol);
  double acc[2] = {0, 0};
  for (int n = tid; n < nloc; n += T) {
    const int i = lo + n;
    double * mi = sMi + 6 * n;
    jacobi_block(d, i, inv_radius, sH + 6 * n, mi);
    const double b0 = d.g[3 * i], b1 = d.g[3 * i + 1], b2 = d.g[3 * i + 2];
    const double z0 = sym3_row(mi, 0, b0, b1, b2), z1 = sym3_row(mi, 1, b0, b1, b2), z2 = sym3_row(mi, 2, b0, b1, b2);
    sR[3 * n] = b0; sR[3 * n + 1] = b1; sR[3 * n + 2] = b2;
    sZ[3 * n] = z0; sZ[3 * n + 1] = z1; sZ[3 * n + 2] = z2;
    sP[3 * n] = 0; sP[3 * n + 1] = 0; sP[3 * n + 2] = 0;
    sY[3 * n] = 0; sY[3 * n + 1] = 0; sY[3 * n + 2] = 0;
    c.gz[3 * i] = z0; c.gz[3 * i + 1] = z1; c.gz[3 * i + 2] = z2;
    c.gp[3 * i] = 0; c.gp[3 * i + 1] = 0; c.gp[3 * i + 2] = 0;
    acc[0] += b0 * b0 + b1 * b1 + b2 * b2;
    acc[1] += b0 * z0 + b1 * z1 + b2 * z2;
  }
  block_sum<2>(acc, red);
  if (tid == 0) { d.partial[blockIdx.x] = acc[0]; d.partial[kMaxPartials + blockIdx.x] = acc[1]; }
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  const double bb = grid_total(d, 0, G, bc);
  double rz = grid_total(d, 1, G, bc);
  double rr = bb;
  const double stop = tol * tol * bb;
  int it = 0;
  double beta = 0.0;
  int cur = 0;   // gp[cur] holds p_old
  if (bb > 0.0) {
    while (it < max_iter) {
      const double * gpo = c.gp + (size_t)cur * 3 * d.N;
      double * gpn = c.gp + (size_t)(cur ^ 1) * 3 * d.N;
      // ---- phase A: gather v_j = z_j + beta p_j ; p_new ; q = A p_new ; partial p.q ----
      gather_neighbours(sCol, nslots, lo, hi, sZ, sP, c.gz, gpo, beta, sV);
      new_direction(3 * nloc, beta, sZ, sP, sQ, gpn + 3 * lo);
      double a1[1] = {0};
      for (int k = tid; k < 3 * nloc; k += T) {
        const double q = own_row_spmv(k, sH, sP, sB, sV, sStart);
        sQ[k] = q;
        a1[0] += sP[k] * q;
      }
      block_sum<1>(a1, red);
      if (tid == 0) d.partial[2 * kMaxPartials + blockIdx.x] = a1[0];
      bar_target += G;
      grid_barrier(c.bar, bar_target);
      const double pq = grid_total(d, 2, G, bc);
      const double alpha = rz / pq;
      // ---- phase B: y += alpha p ; r -= alpha q ; z = Minv r ; partials r.z, r.r ----
      for (int k = tid; k < 3 * nloc; k += T) { sY[k] += alpha * sP[k]; sR[k] -= alpha * sQ[k]; }
      __syncthreads();
      double a2[2] = {0, 0};
      for (int k = tid; k < 3 * nloc; k += T) {
        const int n = k / 3, r = k - 3 * n;
        const double z = sym3_row(sMi + 6 * n, r, sR[3 * n], sR[3 * n + 1], sR[3 * n + 2]);
        sZ[k] = z;
        c.gz[3 * lo + k] = z;
        a2[0] += sR[k] * z;
        a2[1] += sR[k] * sR[k];
      }
      block_sum<2>(a2, red);
      const int s0 = 3 + 2 * (it & 1);
      if (tid == 0) { d.partial[s0 * kMaxPartials + blockIdx.x] = a2[0]; d.partial[(s0 + 1) * kMaxPartials + blockIdx.x] = a2[1]; }
      bar_target += G;
      grid_barrier(c.bar, bar_target);
      const double rz_new = grid_total(d, s0, G, bc);
      rr = grid_total(d, s0 + 1, G, bc);
      ++it;
      cur ^= 1;
      if (!(rr > stop) || !(pq > 0.0)) break;
      beta = rz_new / rz;
      rz = rz_new;
    }
  }
  for (int k = tid; k < 3 * nloc; k += T) d.y[3 * lo + k] = sY[k];
  if (blockIdx.x == 0 && tid == 0) {
    d.scalars[8] = (double)it;
    d.scalars[9] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
  }
}

// ------------------------------------------------------------------------------------------
// k_pg_pcg_2lvl: shared-memory-resident PCG (as k_pg_pcg_smem) with a TWO-LEVEL preconditioner
//     M^-1 = blockdiag(H_ii + D_i)^-1  +  P Ac^-1 P^T ,   Ac = P^T (H + D) P
// One aggregate per CTA (its contiguous node range); P holds CM coarse modes per aggregate, expressed
// in the Jacobi-scaled variables:
//   CM = 3  the aggregate's rigid-body modes (translation x, y, rotation about its centroid)
//   CM = 6  the same three modes once more, weighted by s in [-1, 1] = the node's position along the
//           aggregate (aggregates are stretches of the trajectory): the piecewise-LINEAR deformation
//           modes.  At cfg4 this costs 1.6x fewer CG iterations than CM = 3 (tools/precond_study.py:
//           359 vs 568 at LM step 2) for a coarse matrix of 888 instead of 444 rows.
// The low-frequency deformation modes that make block-Jacobi CG need thousands of iterations on a
// pose graph are removed by the coarse solve.
//   setup per solve: every CTA builds its CM rows of Ac, then a block Gauss-Jordan over the grid
//     (one CM-row pivot exchange per aggregate) leaves each CTA holding ITS CM rows of Ac^-1 in smem;
//   per CG iteration: 2 flag-based exchanges (no atomic barrier): {p.q, P^T q} and {r.z, r.r};
//     the coarse residual P^T r is carried by the recurrence rc -= alpha P^T q, identically in
//     every CTA, so the coarse correction needs no extra exchange.
// All reductions are summed in a fixed order: results are bit-reproducible.
// ------------------------------------------------------------------------------------------
struct Pcg2Cfg {
  int npc, max_slots;     // npc = MAX nodes of one aggregate (array sizing)
  int ex_doubles;         // size of the exchange scratch (>= (1 + CM) G and large enough for the set-up alias)
  const int32_t * agg_start;   // [G + 1] contiguous node ranges of equal node count
  const int32_t * agg_of;      // [N] aggregate of every node
  double * gz;            // [N][3]
  double * gp;            // [2][N][3]
  double * gPt;           // [N][10]  P~ base block of every node (rows: node comps, cols: rigid modes) + its s
  double * gRow;          // [G][CM][2 nc] published pivot rows of the block Gauss-Jordan
  double * grc;           // [G][CM]  initial coarse residual
  double * e1;            // [2][G] slots: {p.q partial, P^T q (CM)}
  double * e2;            // [2][G] slots: {r.z partial, r.r partial}
  unsigned int * gjflag;  // [G]
  unsigned int * bar;     // atomic barrier counter (set-up only)
};

__device__ __forceinline__ double pg_sentinel() { return __longlong_as_double(0x7FF8DEADBEEF0001LL); }
__device__ __forceinline__ bool pg_is_sentinel(double v) { return __double_as_longlong(v) == 0x7FF8DEADBEEF0001LL; }

// Exchange slots: one 256-byte line per (parity, CTA) so that the all-to-all polling spreads over
// every L2 slice instead of hammering a few sectors; a slot holds K <= 8 doubles, each self-flagged
// (a value is "published" when it is not the sentinel).  One thread per source CTA polls with
// 16-byte loads.
constexpr int kSlotStride = 32;   // doubles
__device__ __forceinline__ void ld_volatile2(const double * p, double & a, double & b)
{
  asm volatile("ld.volatile.global.v2.f64 {%0, %1}, [%2];" : "=d"(a), "=d"(b) : "l"(p) : "memory");
}
template <int K>
__device__ __forceinline__ void poll_slots(const double * slots, int G, double * s_out)
{
  constexpr int K2 = (K + 1) / 2;
  for (int t = threadIdx.x; t < G; t += blockDim.x) {
    const double * p = slots + (size_t)t * kSlotStride;
    double v[2 * K2];
    bool ok;
    do {
#pragma unroll
      for (int k = 0; k < K2; ++k) ld_volatile2(p + 2 * k, v[2 * k], v[2 * k + 1]);
      ok = true;
#pragma unroll
      for (int k = 0; k < K; ++k) ok = ok && !pg_is_sentinel(v[k]);
    } while (!ok);
#pragma unroll
    for (int k = 0; k < K; ++k) s_out[t * K + k] = v[k];
    __threadfence();
  }
  __syncthreads();
}
// fixed-order sum of s[i * stride + off], i < n, by warp 0; broadcast through bc
__device__ __forceinline__ double ordered_sum(const double * s, int n, int stride, int off, double * bc)
{
  if (threadIdx.x < 32) {
    double a = 0;
    for (int i = threadIdx.x; i < n; i += 32) a += s[i * stride + off];
    a = warp_sum(a);
    if (threadIdx.x == 0) bc[0] = a;
  }
  __syncthreads();
  const double r = bc[0];
  __syncthreads();
  return r;
}

template <int CM>
__global__ void __launch_bounds__(256, 2) k_pg_pcg_2lvl(PgDev d, Pcg2Cfg c, double inv_radius, double tol, int max_iter)
{
  static_assert(CM == 3 || CM == 6, "coarse modes per aggregate");
  constexpr int KE1 = 1 + CM;            // doubles of an E1 slot
  extern __shared__ __align__(16) unsigned char sm_raw[];
  __shared__ double red[KE1 * 32];
  __shared__ double bc[1];
  __shared__ double s_small[CM * CM + 4];
  __shared__ double s_y[8];
  const int T = blockDim.x, tid = threadIdx.x, G = gridDim.x, I = blockIdx.x;
  const int nc = CM * G;
  const int lo = c.agg_start[I], hi = c.agg_start[I + 1], nloc = hi - lo;
  const int s_lo = d.adj_start[lo], nslots = d.adj_start[hi] - s_lo;
  double * sB = reinterpret_cast<double *>(sm_raw);            // [max_slots][9]
  double * sV = sB + (size_t)c.max_slots * 9;                  // [max_slots][3]
  double * sEx = sV + (size_t)c.max_slots * 3;                 // [ex_doubles >= KE1 G] exchange scratch, right after sV
  double * sH = sEx + (size_t)c.ex_doubles;                    // [npc][6]
  double * sMi = sH + (size_t)c.npc * 6;                       // [npc][6]
  double * sR = sMi + (size_t)c.npc * 6;                       // [npc][3] each below
  double * sZ = sR + (size_t)c.npc * 3;
  double * sP = sZ + (size_t)c.npc * 3;
  double * sQ = sP + (size_t)c.npc * 3;
  double * sY = sQ + (size_t)c.npc * 3;
  double * sPt = sY + (size_t)c.npc * 3;                       // [npc][9]
  double * sS = sPt + (size_t)c.npc * 9;                       // [npc] position of the node along its aggregate, [-1, 1]
  double * sAr = sS + (size_t)c.npc;                           // [CM][nc] right half of [Ac | I] -> rows of Ac^-1
  double * sRc = sAr + (size_t)CM * nc;                        // [nc] coarse residual (identical in all CTAs)
  // the left half of [Ac | I] only lives during set-up: it aliases the CG-only scratch sV | sEx
  // (3 max_slots + ex_doubles >= CM nc is guaranteed by the host)
  double * sAl = sV;                                           // [CM][nc]
  int * sCol = reinterpret_cast<int *>(sRc + nc);              // [max_slots]
  int * sNode = sCol + c.max_slots;                            // [max_slots] local node of the slot
  int * sStart = sNode + c.max_slots;                          // [npc + 1]
  unsigned int bar_target = 0;
  const double SENT = pg_sentinel();
  unsigned long long t_start = 0, t_setup = 0, t_gj = 0;
  unsigned long long tA = 0, tB = 0, tC = 0, tD = 0, tE = 0, t0 = 0, t1 = 0;   // CG phase timers
#define PG_TICK(acc) do { if (I == 0 && tid == 0) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); acc += t1 - t0; t0 = t1; } } while (0)
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));

  // ---- load this CTA's rows (as k_pg_pcg_smem) ----
  for (int i = tid; i <= nloc; i += T) sStart[i] = d.adj_start[lo + i] - s_lo;
  __syncthreads();
  for (int n = tid; n < nloc; n += T)
    for (int s = sStart[n]; s < sStart[n + 1]; ++s) sNode[s] = n;
  load_row_blocks(d, s_lo, nslots, sB, sCol);
  // centroid of the aggregate's free nodes (fixed-order sum by thread 0: nloc is small)
  if (tid == 0) {
    double cx = 0, cy = 0; int cnt = 0;
    for (int n = 0; n < nloc; ++n)
      if (d.is_free[lo + n]) { cx += d.x[3 * (lo + n)]; cy += d.x[3 * (lo + n) + 1]; ++cnt; }
    s_small[0] = cnt ? cx / cnt : 0.0; s_small[1] = cnt ? cy / cnt : 0.0;
    s_small[2] = (double)cnt;
  }
  __syncthreads();
  for (int n = tid; n < nloc; n += T) {
    const int i = lo + n;
    jacobi_block(d, i, inv_radius, sH + 6 * n, sMi + 6 * n);
    // P~ base block: rigid-body modes of the aggregate in Jacobi-scaled variables (y~ = y / s); zero for constant nodes
    double * pt = sPt + 9 * n;
    const double f = d.is_free[i] ? 1.0 : 0.0;
    const double isx = f / d.scale[3 * i], isy = f / d.scale[3 * i + 1], ist = f / d.scale[3 * i + 2];
    pt[0] = isx; pt[1] = 0;   pt[2] = -(d.x[3 * i + 1] - s_small[1]) * isx;
    pt[3] = 0;   pt[4] = isy; pt[5] = (d.x[3 * i] - s_small[0]) * isy;
    pt[6] = 0;   pt[7] = 0;   pt[8] = ist;
    // the s-weighted modes need two free nodes to be independent of the rigid ones; otherwise they are switched off
    // (s = 0 gives zero rows and columns of Ac, which the Gauss-Jordan replaces by the identity)
    const double sn = (CM > 3 && nloc > 1 && s_small[2] >= 2.0) ? 2.0 * n / (double)(nloc - 1) - 1.0 : 0.0;
    sS[n] = sn;
#pragma unroll
    for (int k = 0; k < 9; ++k) c.gPt[10 * (size_t)i + k] = pt[k];
    c.gPt[10 * (size_t)i + 9] = sn;
  }
  // own exchange slots start empty
  if (tid < 2 * KE1) c.e1[((size_t)(tid / KE1) * G + I) * kSlotStride + (tid % KE1)] = SENT;
  if (tid < 4) c.e2[((size_t)(tid >> 1) * G + I) * kSlotStride + (tid & 1)] = SENT;
  bar_target += G;
  grid_barrier(c.bar, bar_target);   // gPt, empty slots visible everywhere

  // ---- coarse operator: this CTA's CM rows of Ac = P^T (H + D) P, then block Gauss-Jordan ----
  // With P_i = [pi | s_i pi], the (I, ct) block of Ac is [[W, Wj], [Wi, Wij]] with W = sum pi^T A_ij pj and the
  // sums weighted by s_j, s_i, s_i s_j.
  for (int k = tid; k < CM * nc; k += T) { sAl[k] = 0.0; sAr[k] = 0.0; }
  __syncthreads();
  for (int ct = tid; ct < G; ct += T) {   // a thread owns coarse column block ct; slots are visited in order: deterministic
    double acc[CM == 3 ? 9 : 36];
#pragma unroll
    for (int k = 0; k < (CM == 3 ? 9 : 36); ++k) acc[k] = 0.0;
    auto add_block = [&](const double (&w3)[9], double si, double sj) {   // w3 = pi^T A pj
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        acc[k] += w3[k];
        if constexpr (CM > 3) { acc[9 + k] += sj * w3[k]; acc[18 + k] += si * w3[k]; acc[27 + k] += si * sj * w3[k]; }
      }
    };
    for (int s = 0; s < nslots; ++s) {
      const int j = sCol[s];
      if (c.agg_of[j] != ct) continue;
      const double * B = sB + 9 * s, * pi = sPt + 9 * sNode[s];
      double pj[9], w[9], w3[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) pj[k] = ld_cg(c.gPt + 10 * (size_t)j + k);
      const double sj = ld_cg(c.gPt + 10 * (size_t)j + 9);
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q) w[3 * r + q] = B[3 * r] * pj[q] + B[3 * r + 1] * pj[3 + q] + B[3 * r + 2] * pj[6 + q];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q) w3[3 * r + q] = pi[r] * w[q] + pi[3 + r] * w[3 + q] + pi[6 + r] * w[6 + q];
      add_block(w3, sS[sNode[s]], sj);
    }
    if (ct == I) {   // diagonal blocks of own nodes
      for (int n = 0; n < nloc; ++n) {
        const double * H = sH + 6 * n, * pi = sPt + 9 * n;
        double w[9], w3[9];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          w[q] = H[0] * pi[q] + H[1] * pi[3 + q] + H[2] * pi[6 + q];
          w[3 + q] = H[1] * pi[q] + H[3] * pi[3 + q] + H[4] * pi[6 + q];
          w[6 + q] = H[2] * pi[q] + H[4] * pi[3 + q] + H[5] * pi[6 + q];
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int q = 0; q < 3; ++q) w3[3 * r + q] = pi[r] * w[q] + pi[3 + r] * w[3 + q] + pi[6 + r] * w[6 + q];
        add_block(w3, sS[n], sS[n]);
      }
    }
    // acc layout: [rb][cb][r][q] with rb / cb = 0 rigid, 1 s-weighted; Ac row = 3 rb + r, column = CM ct + 3 cb + q
#pragma unroll
    for (int rb = 0; rb < CM / 3; ++rb)
#pragma unroll
      for (int cb = 0; cb < CM / 3; ++cb)
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int q = 0; q < 3; ++q)
            sAl[(size_t)(3 * rb + r) * nc + CM * ct + 3 * cb + q] = acc[(CM == 3 ? 0 : 18 * rb + 9 * cb) + 3 * r + q];
  }
  if (tid < CM) sAr[(size_t)tid * nc + CM * I + tid] = 1.0;   // augmented identity
  __syncthreads();
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_setup));
  for (int k = 0; k < G; ++k) {
    double * row = c.gRow + (size_t)k * CM * 2 * nc;   // published pivot rows: [CM][2 nc] (left | right)
    auto elem = [&](int r, int j) -> double & { return j < nc ? sAl[(size_t)r * nc + j] : sAr[(size_t)r * nc + (j - nc)]; };
    // columns that can be non-zero in pivot rows k: the not yet reduced part of the left half, [CM k, nc), and the part of
    // the right half filled so far, [0, CM (k + 1)); everything else is 0 and stays 0
    const int nleft = nc - CM * k, nact = nleft + CM * (k + 1);
    if (I == k) {
      // inverse of the CM x CM pivot block by Gauss-Jordan without pivoting (the block is symmetric positive definite on
      // its non-degenerate modes); a mode with a zero diagonal (no free node, or the s-modes of a one-node aggregate) has
      // a zero row and column in all of Ac: it is replaced by the identity
      if (tid == 0) {
        double a[CM][2 * CM];
#pragma unroll
        for (int r = 0; r < CM; ++r)
#pragma unroll
          for (int q = 0; q < CM; ++q) { a[r][q] = elem(r, CM * k + q); a[r][CM + q] = (r == q) ? 1.0 : 0.0; }
        double d0[CM];
#pragma unroll
        for (int p = 0; p < CM; ++p) d0[p] = fabs(a[p][p]);
#pragma unroll
        for (int p = 0; p < CM; ++p) {
          if (!(fabs(a[p][p]) > 1e-12 * d0[p]) || !(d0[p] > 1e-300)) {   // zero or (numerically) dependent mode
#pragma unroll
            for (int q = 0; q < 2 * CM; ++q) a[p][q] = 0.0;
#pragma unroll
            for (int r = 0; r < CM; ++r) a[r][p] = 0.0;
            a[p][p] = 1.0; a[p][CM + p] = 1.0;
          }
          const double ip = 1.0 / a[p][p];
#pragma unroll
          for (int q = 0; q < 2 * CM; ++q) a[p][q] *= ip;
#pragma unroll
          for (int r = 0; r < CM; ++r) {
            if (r == p) continue;
            const double m = a[r][p];
#pragma unroll
            for (int q = 0; q < 2 * CM; ++q) a[r][q] -= m * a[p][q];
          }
        }
#pragma unroll
        for (int r = 0; r < CM; ++r)
#pragma unroll
          for (int q = 0; q < CM; ++q) s_small[CM * r + q] = a[r][CM + q];
      }
      __syncthreads();
      for (int t = tid; t < nact; t += T) {
        const int j = t < nleft ? CM * k + t : nc + (t - nleft);
        double v[CM], o[CM];
#pragma unroll
        for (int r = 0; r < CM; ++r) v[r] = elem(r, j);
#pragma unroll
        for (int r = 0; r < CM; ++r) {
          double a = 0;
#pragma unroll
          for (int q = 0; q < CM; ++q) a += s_small[CM * r + q] * v[q];
          o[r] = a;
        }
#pragma unroll
        for (int r = 0; r < CM; ++r) { elem(r, j) = o[r]; row[(size_t)r * 2 * nc + j] = o[r]; }
      }
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(c.gjflag + k), "r"(1u) : "memory");
      }
    } else {
      if (tid == 0) {
        unsigned int v;
        do {
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(c.gjflag + k) : "memory");
        } while (v == 0u);
      }
      if (tid < CM * CM) s_small[tid] = elem(tid / CM, CM * k + (tid % CM));   // my multipliers (read before they are eliminated)
      __syncthreads();
      for (int t = tid; t < nact; t += T) {
        const int j = t < nleft ? CM * k + t : nc + (t - nleft);
        double pr[CM];
#pragma unroll
        for (int q = 0; q < CM; ++q) pr[q] = ld_cg(row + (size_t)q * 2 * nc + j);
#pragma unroll
        for (int r = 0; r < CM; ++r) {
          double a = 0;
#pragma unroll
          for (int q = 0; q < CM; ++q) a += s_small[CM * r + q] * pr[q];
          elem(r, j) -= a;
        }
      }
      __syncthreads();
    }
  }
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_gj));
  // rows of Ac^-1 are now sAr[r * nc + j]
  __syncthreads();

  // ---- CG start: r = b, coarse residual, z = M^-1 r ----
  double accb[1] = {0};
  for (int k = tid; k < 3 * nloc; k += T) {
    const double b = d.g[3 * lo + k];
    sR[k] = b; sY[k] = 0.0; sP[k] = 0.0;
    c.gp[3 * lo + k] = 0.0;
    accb[0] += b * b;
  }
  __syncthreads();
  if (tid < CM) {   // P^T r of this aggregate, fixed order
    const int cb = tid / 3, q = tid % 3;
    double a = 0;
    for (int n = 0; n < nloc; ++n) {
      const double v = sPt[9 * n + q] * sR[3 * n] + sPt[9 * n + 3 + q] * sR[3 * n + 1] + sPt[9 * n + 6 + q] * sR[3 * n + 2];
      a += cb ? sS[n] * v : v;
    }
    c.grc[CM * I + tid] = a;
  }
  block_sum<1>(accb, red);
  if (tid == 0) d.partial[I] = accb[0];
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  const double bb = grid_total(d, 0, G, bc);
  for (int k = tid; k < nc; k += T) sRc[k] = ld_cg(c.grc + k);
  __syncthreads();

  // z = blockJacobi^-1 r + P Ac^-1 rc ; returns partial r.z and r.r through a2
  auto apply_precond = [&](double (&a2)[2]) {
    if (tid < 32 * CM) {   // CM warps: one row of Ac^-1 each
      const int w = tid >> 5, l = tid & 31;
      const double * Ai = sAr + (size_t)w * nc;
      double a = 0;
      for (int j = l; j < nc; j += 32) a += Ai[j] * sRc[j];
      a = warp_sum(a);
      if (l == 0) s_y[w] = a;
    }
    __syncthreads();
    a2[0] = 0; a2[1] = 0;
    for (int k = tid; k < 3 * nloc; k += T) {
      const int n = k / 3, r = k - 3 * n;
      const double * pt = sPt + 9 * n + 3 * r;
      double z = sym3_row(sMi + 6 * n, r, sR[3 * n], sR[3 * n + 1], sR[3 * n + 2]);
      double y0 = s_y[0], y1 = s_y[1], y2 = s_y[2];
      if constexpr (CM > 3) { const double sn = sS[n]; y0 += sn * s_y[3]; y1 += sn * s_y[4]; y2 += sn * s_y[5]; }
      z += pt[0] * y0 + pt[1] * y1 + pt[2] * y2;
      sZ[k] = z;
      c.gz[3 * lo + k] = z;
      a2[0] += sR[k] * z;
      a2[1] += sR[k] * sR[k];
    }
  };
  double a2[2];
  apply_precond(a2);
  block_sum<2>(a2, red);
  if (tid == 0) d.partial[kMaxPartials + I] = a2[0];
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  double rz = grid_total(d, 1, G, bc);
  double rr = bb;
  const double stop = tol * tol * bb;
  int it = 0;
  double beta = 0.0;
  int cur = 0;
  if (bb > 0.0) {
    while (it < max_iter) {
      const int par = it & 1;
      const double * gpo = c.gp + (size_t)cur * 3 * d.N;
      double * gpn = c.gp + (size_t)(cur ^ 1) * 3 * d.N;
      double * e1 = c.e1 + (size_t)par * G * kSlotStride, * e2 = c.e2 + (size_t)par * G * kSlotStride;
      // ---- phase A ----
      if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      gather_neighbours(sCol, nslots, lo, hi, sZ, sP, c.gz, gpo, beta, sV);
      PG_TICK(tA);
      new_direction(3 * nloc, beta, sZ, sP, sQ, gpn + 3 * lo);
      double a1[KE1];   // p.q and the CM components of P^T q of this aggregate
#pragma unroll
      for (int k = 0; k < KE1; ++k) a1[k] = 0.0;
      for (int k = tid; k < 3 * nloc; k += T) {
        const double q = own_row_spmv(k, sH, sP, sB, sV, sStart);
        sQ[k] = q;
        const int n = k / 3, r = k - 3 * n;
        const double * pt = sPt + 9 * n + 3 * r;
        a1[0] += sP[k] * q;
        const double u0 = pt[0] * q, u1 = pt[1] * q, u2 = pt[2] * q;
        a1[1] += u0; a1[2] += u1; a1[3] += u2;
        if constexpr (CM > 3) { const double sn = sS[n]; a1[4] += sn * u0; a1[5] += sn * u1; a1[6] += sn * u2; }
      }
      block_sum<KE1>(a1, red);
      PG_TICK(tB);
      if (tid == 0) {
        __threadfence();   // p_new of this CTA visible before the flagged values
        double * m = e1 + (size_t)I * kSlotStride;
#pragma unroll
        for (int k = 1; k < KE1; ++k) m[k] = a1[k];
        m[0] = a1[0];
      }
      poll_slots<KE1>(e1, G, sEx);
      PG_TICK(tC);
      // every CTA published E1(it) only after it finished reading E2(it-1): those slots can be recycled now
      if (it > 0 && tid < 2) c.e2[((size_t)(par ^ 1) * G + I) * kSlotStride + tid] = SENT;
      const double pq = ordered_sum(sEx, G, KE1, 0, bc);
      const double alpha = rz / pq;
      // ---- phase B ----
      for (int k = tid; k < nc; k += T) sRc[k] -= alpha * sEx[KE1 * (k / CM) + 1 + (k % CM)];
      for (int k = tid; k < 3 * nloc; k += T) { sY[k] += alpha * sP[k]; sR[k] -= alpha * sQ[k]; }
      __syncthreads();
      apply_precond(a2);
      block_sum<2>(a2, red);
      __syncthreads();
      PG_TICK(tD);
      if (tid == 0) {
        __threadfence();   // z of this CTA visible before the flagged values
        double * m = e2 + (size_t)I * kSlotStride;
        m[0] = a2[0]; m[1] = a2[1];
      }
      poll_slots<2>(e2, G, sEx);
      PG_TICK(tE);
      // every CTA published E2(it) only after it finished reading E1(it): recycle own E1(it) slots
      if (tid < KE1) c.e1[((size_t)par * G + I) * kSlotStride + tid] = SENT;
      if (tid < 32) {
        double u = 0, w = 0;
        for (int i = tid; i < G; i += 32) { u += sEx[2 * i]; w += sEx[2 * i + 1]; }
        u = warp_sum(u); w = warp_sum(w);
        if (tid == 0) { s_small[0] = u; s_small[1] = w; }
      }
      __syncthreads();
      const double rz_new = s_small[0];
      rr = s_small[1];
      ++it;
      cur ^= 1;
      if (!(rr > stop) || !(pq > 0.0)) break;
      beta = rz_new / rz;
      rz = rz_new;
    }
  }
  for (int k = tid; k < 3 * nloc; k += T) d.y[3 * lo + k] = sY[k];
  if (I == 0 && tid == 0) {
    unsigned long long t_end;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
    d.scalars[8] = (double)it;
    d.scalars[9] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
    d.scalars[10] = (double)(t_setup - t_start);   // ns: load rows + P~ + first barrier + Ac rows
    d.scalars[11] = (double)(t_gj - t_setup);      // ns: block Gauss-Jordan
    d.scalars[12] = (double)(t_end - t_gj);        // ns: CG iterations
    d.scalars[13] = (double)tA; d.scalars[14] = (double)tB; d.scalars[15] = (double)tC;
    d.scalars[6] = (double)tD; d.scalars[7] = (double)tE;
  }
#undef PG_TICK
}

// ------------------------------------------------------------------------------------------
// k_pg_pcg_2lvl_g: the preconditioner of k_pg_pcg_2lvl (same coarse modes, same flag exchanges, same coarse-residual
// recurrence) for graphs whose aggregates do not fit shared memory (DESIGN.md §4 "Large graphs").
//   * Aggregates are contiguous node ranges sized by the plan; CTA b owns aggregates [b apc, (b + 1) apc). The block rows,
//     the preconditioner blocks (d.Minv) and the CG vectors stay in global memory (L2 up to a few tens of MB, HBM beyond).
//   * Ac = P^T (H + D) P is assembled densely into global memory ([ld][ld], ld = CM na rounded up to kGjTile; the padding
//     is the identity) from the same block formulas, one warp per aggregate adding its slots in CSR order. A grid-wide
//     blocked Gauss-Jordan (kGjPanel columns per step, two grid barriers per step) inverts it in place once per solve.
//   * Per CG iteration each CTA applies its CM apc rows of Ac^-1 to the coarse residual (a dense mat-vec spread over the
//     grid), and P^T q travels through global memory (gPtq) ahead of the {p.q} flag, so the exchanges stay
//     {p.q, P^T q} and {r.z, r.r}.
// Every sum runs in a fixed order: results are bit-reproducible.
// ------------------------------------------------------------------------------------------
constexpr int kG2Threads = 512;
constexpr int kGjPanel = 32;   // columns one Gauss-Jordan step eliminates (one per lane of a warp)
constexpr int kGjTile = 64;    // the rank-kGjPanel update runs on kGjTile x kGjTile tiles
struct Pcg2GCfg {
  int na;                      // aggregates
  int apc;                     // aggregates per CTA
  int ld;                      // leading dimension of Ac: CM na rounded up to kGjTile
  const int32_t * agg_start;   // [na + 1] contiguous node ranges
  const int32_t * agg_of;      // [N]
  double * gz;                 // [N][3]
  double * gp;                 // [2][N][3]
  double * gPt;                // [N][10] P~ base block of every node + its s (as Pcg2Cfg::gPt)
  double * Ac;                 // [ld][ld] coarse matrix, then its inverse
  double * Cb, * Tb;           // [kGjPanel][ld] a Gauss-Jordan step's old column panel and new row panel
  double * gPtq;               // [ld] P^T q of the current iteration
  double * grc;                // [ld] initial coarse residual P^T b
  double * e1;                 // [2][G] slots: {p.q partial}
  double * e2;                 // [2][G] slots: {r.z partial, r.r partial}
  unsigned int * bar;          // atomic barrier counter (set-up only)
};

// In-place Gauss-Jordan inverse of a kGjPanel x kGjPanel block held by one warp, lane j holding column j (col[r] = D[r][j]).
// A pivot that is zero or (numerically) dependent on the earlier ones has its row and column replaced by the identity's, as
// in k_pg_pcg_2lvl's pivot blocks.
__device__ __forceinline__ void gj_invert_cols(double (&col)[kGjPanel], int lane)
{
  double dself = 0;
#pragma unroll
  for (int r = 0; r < kGjPanel; ++r)
    if (r == lane) dself = col[r];
#pragma unroll
  for (int p = 0; p < kGjPanel; ++p) {
    const double d0 = fabs(__shfl_sync(0xffffffffu, dself, p));
    double piv = __shfl_sync(0xffffffffu, col[p], p);
    if (!(fabs(piv) > 1e-12 * d0) || !(d0 > 1e-300)) {   // warp-uniform
      col[p] = 0.0;
      if (lane == p) {
#pragma unroll
        for (int r = 0; r < kGjPanel; ++r) col[r] = 0.0;
        col[p] = 1.0;
      }
      piv = 1.0;
    }
    const double inv = 1.0 / piv;
    col[p] = lane == p ? inv : col[p] * inv;   // row p
#pragma unroll
    for (int r = 0; r < kGjPanel; ++r) {
      if (r == p) continue;
      const double cr = __shfl_sync(0xffffffffu, col[r], p);   // a[r][p] before this step
      col[r] = lane == p ? -cr * inv : col[r] - cr * col[p];
    }
  }
}

template <int CM>
__global__ void __launch_bounds__(kG2Threads, 1) k_pg_pcg_2lvl_g(PgDev d, Pcg2GCfg c, double inv_radius, double tol, int max_iter)
{
  static_assert(CM == 3 || CM == 6, "coarse modes per aggregate");
  extern __shared__ __align__(16) unsigned char sm_raw[];
  __shared__ double red[CM * 32];
  __shared__ double bc[1];
  __shared__ double s_small[2];
  const int T = blockDim.x, tid = threadIdx.x, G = gridDim.x, I = blockIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = T >> 5;
  const int nc = CM * c.na, ld = c.ld;
  const int a_lo = min(c.na, I * c.apc), a_hi = min(c.na, a_lo + c.apc);
  const int lo = c.agg_start[a_lo], hi = c.agg_start[a_hi];
  double * sRc = reinterpret_cast<double *>(sm_raw);   // [ld] coarse residual (identical in all CTAs)
  double * sW = sRc + ld;   // scratch: assembly staging, then the Gauss-Jordan tiles, then the exchange and CM apc coarse values
  unsigned int bar_target = 0;
  const double SENT = pg_sentinel();
  unsigned long long t_start = 0, t_setup = 0, t_gj = 0;
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));

  // P^T v of every own aggregate into out[CM a + m]: the whole CTA on one aggregate at a time, threads over its nodes, then
  // a fixed-order block reduction (every thread calls it)
  auto aggregate_pt = [&](const double * v, double * out) {
    for (int a = a_lo; a < a_hi; ++a) {
      double u[CM];
#pragma unroll
      for (int m = 0; m < CM; ++m) u[m] = 0.0;
      for (int i = c.agg_start[a] + tid; i < c.agg_start[a + 1]; i += T) {
        const double * pt = c.gPt + 10 * (size_t)i;
        const double v0 = v[3 * i], v1 = v[3 * i + 1], v2 = v[3 * i + 2];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const double w = pt[q] * v0 + pt[3 + q] * v1 + pt[6 + q] * v2;
          u[q] += w;
          if constexpr (CM > 3) u[3 + q] += pt[9] * w;
        }
      }
      block_sum<CM>(u, red);
      if (tid == 0)
#pragma unroll
        for (int m = 0; m < CM; ++m) out[CM * a + m] = u[m];
    }
  };

  // ---- set-up 1: Ac = 0 (identity on the padding); per own node Minv, P~ and s, r = b, y = 0, p = 0; empty slots ----
  for (size_t k = (size_t)I * T + tid; k < (size_t)ld * ld; k += (size_t)G * T) {
    const size_t r = k / ld;
    c.Ac[k] = (r >= (size_t)nc && k == r * ld + r) ? 1.0 : 0.0;
  }
  for (int a = a_lo + warp; a < a_hi; a += nwarps) {
    const int alo = c.agg_start[a], nloc = c.agg_start[a + 1] - alo;
    double cx = 0, cy = 0, cnt = 0;   // centroid of the aggregate's free nodes
    for (int n = lane; n < nloc; n += 32)
      if (d.is_free[alo + n]) { cx += d.x[3 * (alo + n)]; cy += d.x[3 * (alo + n) + 1]; cnt += 1.0; }
    cx = warp_sum(cx); cy = warp_sum(cy); cnt = warp_sum(cnt);
    if (cnt > 0) { cx /= cnt; cy /= cnt; }
    for (int n = lane; n < nloc; n += 32) {
      const int i = alo + n;
      double hb[6];
      jacobi_block(d, i, inv_radius, hb, d.Minv + 6 * i);
      double * pt = c.gPt + 10 * (size_t)i;
      const double f = d.is_free[i] ? 1.0 : 0.0;
      const double isx = f / d.scale[3 * i], isy = f / d.scale[3 * i + 1], ist = f / d.scale[3 * i + 2];
      pt[0] = isx; pt[1] = 0;   pt[2] = -(d.x[3 * i + 1] - cy) * isx;
      pt[3] = 0;   pt[4] = isy; pt[5] = (d.x[3 * i] - cx) * isy;
      pt[6] = 0;   pt[7] = 0;   pt[8] = ist;
      pt[9] = (CM > 3 && nloc > 1 && cnt >= 2.0) ? 2.0 * n / (double)(nloc - 1) - 1.0 : 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        d.pr[3 * i + k] = d.g[3 * i + k]; d.y[3 * i + k] = 0.0; c.gp[3 * i + k] = 0.0;
      }
    }
  }
  if (tid < 2) c.e1[((size_t)tid * G + I) * kSlotStride] = SENT;
  if (tid < 4) c.e2[((size_t)(tid >> 1) * G + I) * kSlotStride + (tid & 1)] = SENT;
  bar_target += G;
  grid_barrier(c.bar, bar_target);   // gPt, zeroed Ac and empty slots visible everywhere

  // ---- set-up 2: rows CM a .. CM a + CM - 1 of Ac, a warp per own aggregate. Its items (the CSR slots of its nodes, then
  // the nodes' diagonal blocks) are staged 32 at a time; lane l owns entries l and l + 32 of the CM x CM block and adds
  // the staged items in order, flushing to Ac whenever the column block changes ----
  {
    double * stg = sW + (size_t)warp * 32 * 12;   // [32][12]: w3 = pi^T A_ij pj (9), s_i, s_j, column block
    for (int a = a_lo + warp; a < a_hi; a += nwarps) {
      const int alo = c.agg_start[a], ahi = c.agg_start[a + 1];
      const int s_lo = d.adj_start[alo], nslots = d.adj_start[ahi] - s_lo, nitems = nslots + (ahi - alo);
      double acc[2] = {0.0, 0.0};
      int cur = -1;
      auto flush = [&]() {
        if (cur >= 0)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int e = lane + 32 * h;
            if (e < CM * CM) c.Ac[(size_t)(CM * a + e / CM) * ld + CM * cur + e % CM] += acc[h];
          }
        acc[0] = 0.0; acc[1] = 0.0;
      };
      for (int t0 = 0; t0 < nitems; t0 += 32) {
        const int t = t0 + lane;
        if (t < nitems) {
          double B[9], pj[9], sj;
          int i, ct;
          if (t < nslots) {
            const int s = s_lo + t;
            int l = alo, u = ahi - 1;   // the slot's node: the last i with adj_start[i] <= s
            while (l < u) { const int m = (l + u + 1) >> 1; if (d.adj_start[m] <= s) l = m; else u = m - 1; }
            i = l;
            const int av = d.adj[s], e = av >> 1, side = av & 1;
            const double * M = d.lin + (size_t)kLin * e + 21;
            const int j = d.eidx[2 * e + (side ? 0 : 1)];
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
              for (int q = 0; q < 3; ++q) B[3 * r + q] = side == 0 ? M[3 * r + q] : M[3 * q + r];
#pragma unroll
            for (int k = 0; k < 9; ++k) pj[k] = ld_cg(c.gPt + 10 * (size_t)j + k);
            sj = ld_cg(c.gPt + 10 * (size_t)j + 9);
            ct = c.agg_of[j];
          } else {
            i = alo + (t - nslots);
            double hb[6], mi[6];
            jacobi_block(d, i, inv_radius, hb, mi);
            B[0] = hb[0]; B[1] = hb[1]; B[2] = hb[2]; B[3] = hb[1]; B[4] = hb[3]; B[5] = hb[4];
            B[6] = hb[2]; B[7] = hb[4]; B[8] = hb[5];
#pragma unroll
            for (int k = 0; k < 9; ++k) pj[k] = ld_cg(c.gPt + 10 * (size_t)i + k);
            sj = ld_cg(c.gPt + 10 * (size_t)i + 9);
            ct = a;
          }
          double pi[9], w[9];
#pragma unroll
          for (int k = 0; k < 9; ++k) pi[k] = ld_cg(c.gPt + 10 * (size_t)i + k);
          const double si = ld_cg(c.gPt + 10 * (size_t)i + 9);
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int q = 0; q < 3; ++q) w[3 * r + q] = B[3 * r] * pj[q] + B[3 * r + 1] * pj[3 + q] + B[3 * r + 2] * pj[6 + q];
          double * o = stg + 12 * lane;
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int q = 0; q < 3; ++q) o[3 * r + q] = pi[r] * w[q] + pi[3 + r] * w[3 + q] + pi[6 + r] * w[6 + q];
          o[9] = si; o[10] = sj; o[11] = (double)ct;
        }
        __syncwarp();
        const int nt = min(32, nitems - t0);
        for (int u = 0; u < nt; ++u) {
          const double * o = stg + 12 * u;
          const int ct = (int)o[11];
          if (ct != cur) { flush(); cur = ct; }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int e = lane + 32 * h;
            if (e < CM * CM) {
              const int R = e / CM, Q = e % CM;
              double v = o[3 * (R % 3) + Q % 3];
              if (R >= 3) v *= o[9];
              if (Q >= 3) v *= o[10];
              acc[h] += v;
            }
          }
        }
        __syncwarp();
      }
      flush();
      __syncwarp();
      // a mode without a free node (or the s-modes of an aggregate with fewer than two) has a zero row and column: identity
      if (lane < CM) {
        double * dg = c.Ac + (size_t)(CM * a + lane) * ld + CM * a + lane;
        if (*dg == 0.0) *dg = 1.0;
      }
    }
  }
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_setup));

  // ---- set-up 3: in-place blocked Gauss-Jordan. Step K (columns k0 .. k0 + 31): D = A(K, K);
  //   T = D^-1 [A(K, :) with the identity in columns K]   (the new rows K),
  //   C = A(:, K) with -I in rows K                        (the old columns K),
  //   A(i, j) <- [i, j outside K] A(i, j) - sum_k C(i, k) T(k, j)   for every (i, j),
  // which leaves D^-1, D^-1 A(K, :), -A(:, K) D^-1 and the Schur complement in place; after the last step A = Ac^-1 ----
  {
    double * sC = sW, * sT = sW + kGjPanel * kGjTile, * sD = sT + kGjPanel * kGjTile;   // [32][64], [32][64], [32][32]
    const int ntile = ld / kGjTile;
    for (int k0 = 0; k0 < ld; k0 += kGjPanel) {
      if (warp == 0) {   // every CTA inverts the pivot block the same way
        double col[kGjPanel];
#pragma unroll
        for (int r = 0; r < kGjPanel; ++r) col[r] = ld_cg(c.Ac + (size_t)(k0 + r) * ld + k0 + lane);
        gj_invert_cols(col, lane);
#pragma unroll
        for (int r = 0; r < kGjPanel; ++r) sD[r * kGjPanel + lane] = col[r];
      }
      __syncthreads();
      for (int j = I * T + tid; j < ld; j += G * T) {
        const bool piv = j >= k0 && j < k0 + kGjPanel;
        double v[kGjPanel];
#pragma unroll
        for (int m = 0; m < kGjPanel; ++m) v[m] = piv ? (j - k0 == m ? 1.0 : 0.0) : ld_cg(c.Ac + (size_t)(k0 + m) * ld + j);
#pragma unroll 4
        for (int k = 0; k < kGjPanel; ++k) {
          double t = 0;
#pragma unroll
          for (int m = 0; m < kGjPanel; ++m) t += sD[k * kGjPanel + m] * v[m];
          c.Tb[(size_t)k * ld + j] = t;
        }
#pragma unroll
        for (int k = 0; k < kGjPanel; ++k) c.Cb[(size_t)k * ld + j] = piv ? (j - k0 == k ? -1.0 : 0.0) : ld_cg(c.Ac + (size_t)j * ld + k0 + k);
      }
      bar_target += G;
      grid_barrier(c.bar, bar_target);
      for (int tl = I; tl < ntile * ntile; tl += G) {
        const int i0 = (tl / ntile) * kGjTile, j0 = (tl % ntile) * kGjTile;
        for (int k = tid; k < kGjPanel * kGjTile; k += T) {
          const int kk = k / kGjTile, x = k % kGjTile;
          sC[k] = ld_cg(c.Cb + (size_t)kk * ld + i0 + x);
          sT[k] = ld_cg(c.Tb + (size_t)kk * ld + j0 + x);
        }
        __syncthreads();
        const int r = tid >> 3, cl = tid & 7;   // row r of the tile, its columns cl + 8 m
        const int i = i0 + r;
        const bool rowK = i >= k0 && i < k0 + kGjPanel;
        double o[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) {
          const int j = j0 + cl + 8 * m;
          o[m] = (rowK || (j >= k0 && j < k0 + kGjPanel)) ? 0.0 : ld_cg(c.Ac + (size_t)i * ld + j);
        }
#pragma unroll 8
        for (int k = 0; k < kGjPanel; ++k) {
          const double cv = sC[k * kGjTile + r];
#pragma unroll
          for (int m = 0; m < 8; ++m) o[m] -= cv * sT[k * kGjTile + cl + 8 * m];
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) c.Ac[(size_t)i * ld + j0 + cl + 8 * m] = o[m];
        __syncthreads();
      }
      bar_target += G;
      grid_barrier(c.bar, bar_target);
    }
  }
  if (I == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_gj));

  // ---- CG start: coarse residual P^T b (every CTA keeps all of it), z = M^-1 r ----
  double * sEx = sW;                       // [2 G] polled exchange values
  double * sYc = sW + 2 * (size_t)G;       // [CM apc] Ac^-1 rc on the own aggregates
  double accb[1] = {0};
  for (int k = 3 * lo + tid; k < 3 * hi; k += T) accb[0] += d.g[k] * d.g[k];
  aggregate_pt(d.g, c.grc);
  block_sum<1>(accb, red);
  if (tid == 0) d.partial[I] = accb[0];
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  const double bb = grid_total(d, 0, G, bc);
  for (int k = tid; k < ld; k += T) sRc[k] = k < nc ? ld_cg(c.grc + k) : 0.0;
  __syncthreads();

  // z = blockJacobi^-1 r + P Ac^-1 rc on the own nodes (published to gz); partial r.z and r.r through a2
  auto apply_precond = [&](double (&a2)[2]) {
    for (int row = warp; row < CM * (a_hi - a_lo); row += nwarps) {   // a warp per row of Ac^-1
      const double * Ai = c.Ac + (size_t)(CM * a_lo + row) * ld;
      double a = 0;
      for (int j = lane; j < nc; j += 32) a += ld_cg(Ai + j) * sRc[j];
      a = warp_sum(a);
      if (lane == 0) sYc[row] = a;
    }
    __syncthreads();
    a2[0] = 0; a2[1] = 0;
    for (int k = 3 * lo + tid; k < 3 * hi; k += T) {
      const int i = k / 3, r = k - 3 * i;
      const double * pt = c.gPt + 10 * (size_t)i;
      const double * yc = sYc + CM * (c.agg_of[i] - a_lo);
      const double r0 = d.pr[3 * i], r1 = d.pr[3 * i + 1], r2 = d.pr[3 * i + 2];
      double z = sym3_row(d.Minv + 6 * i, r, r0, r1, r2);
      double y0 = yc[0], y1 = yc[1], y2 = yc[2];
      if constexpr (CM > 3) { const double sn = pt[9]; y0 += sn * yc[3]; y1 += sn * yc[4]; y2 += sn * yc[5]; }
      z += pt[3 * r] * y0 + pt[3 * r + 1] * y1 + pt[3 * r + 2] * y2;
      c.gz[k] = z;
      const double rk = d.pr[k];
      a2[0] += rk * z;
      a2[1] += rk * rk;
    }
  };
  double a2[2];
  apply_precond(a2);
  block_sum<2>(a2, red);
  if (tid == 0) d.partial[kMaxPartials + I] = a2[0];
  bar_target += G;
  grid_barrier(c.bar, bar_target);
  double rz = grid_total(d, 1, G, bc);
  double rr = bb;
  const double stop = tol * tol * bb;
  int it = 0;
  double beta = 0.0;
  int cur = 0;
  if (bb > 0.0) {
    while (it < max_iter) {
      const int par = it & 1;
      const double * gpo = c.gp + (size_t)cur * 3 * d.N;
      double * gpn = c.gp + (size_t)(cur ^ 1) * 3 * d.N;
      double * e1 = c.e1 + (size_t)par * G * kSlotStride, * e2 = c.e2 + (size_t)par * G * kSlotStride;
      // ---- phase A: p_new = z + beta p_old ; q = A p_new ; p.q ; P^T q of the own aggregates ----
      double a1[1] = {0};
      for (int i = lo + tid; i < hi; i += T) {
        double q[3], pv[3];
        spmv_row<true>(d, i, c.gz, gpo, beta, inv_radius, q, pv);
#pragma unroll
        for (int k = 0; k < 3; ++k) { gpn[3 * i + k] = pv[k]; d.pq[3 * i + k] = q[k]; }
        a1[0] += pv[0] * q[0] + pv[1] * q[1] + pv[2] * q[2];
      }
      block_sum<1>(a1, red);
      __syncthreads();
      aggregate_pt(d.pq, c.gPtq);
      __syncthreads();
      if (tid == 0) {
        __threadfence();   // p_new and P^T q of this CTA visible before the flagged value
        e1[(size_t)I * kSlotStride] = a1[0];
      }
      poll_slots<1>(e1, G, sEx);
      // every CTA published E1(it) only after it finished reading E2(it-1): those slots can be recycled now
      if (it > 0 && tid < 2) c.e2[((size_t)(par ^ 1) * G + I) * kSlotStride + tid] = SENT;
      const double pq = ordered_sum(sEx, G, 1, 0, bc);
      const double alpha = rz / pq;
      // ---- phase B: rc -= alpha P^T q ; y += alpha p ; r -= alpha q ; z = M^-1 r ----
      for (int k = tid; k < nc; k += T) sRc[k] -= alpha * ld_cg(c.gPtq + k);
      for (int k = 3 * lo + tid; k < 3 * hi; k += T) { d.y[k] += alpha * gpn[k]; d.pr[k] -= alpha * d.pq[k]; }
      __syncthreads();
      apply_precond(a2);
      block_sum<2>(a2, red);
      __syncthreads();
      if (tid == 0) {
        __threadfence();   // z of this CTA visible before the flagged values
        double * m = e2 + (size_t)I * kSlotStride;
        m[0] = a2[0]; m[1] = a2[1];
      }
      poll_slots<2>(e2, G, sEx);
      // every CTA published E2(it) only after it finished reading E1(it) and gPtq(it): recycle own E1(it) slot
      if (tid == 0) c.e1[((size_t)par * G + I) * kSlotStride] = SENT;
      if (tid < 32) {
        double u = 0, w = 0;
        for (int k = tid; k < G; k += 32) { u += sEx[2 * k]; w += sEx[2 * k + 1]; }
        u = warp_sum(u); w = warp_sum(w);
        if (tid == 0) { s_small[0] = u; s_small[1] = w; }
      }
      __syncthreads();
      const double rz_new = s_small[0];
      rr = s_small[1];
      ++it;
      cur ^= 1;
      if (!(rr > stop) || !(pq > 0.0)) break;
      beta = rz_new / rz;
      rz = rz_new;
    }
  }
  if (I == 0 && tid == 0) {
    unsigned long long t_end;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
    d.scalars[8] = (double)it;
    d.scalars[9] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
    d.scalars[10] = (double)(t_setup - t_start);   // ns: Minv, P~, Ac assembly
    d.scalars[11] = (double)(t_gj - t_setup);      // ns: blocked Gauss-Jordan
    d.scalars[12] = (double)(t_end - t_gj);        // ns: CG iterations
  }
}

// candidate point: delta = -(y * scale) ; xc = x (+) delta on free nodes; partial ||x - xc||^2
__global__ void __launch_bounds__(kPgThreads) k_pg_apply_step(PgDev d)
{
  __shared__ double red[32];
  double s[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.N; i += gridDim.x * blockDim.x) {
    const double * x = d.x + 3 * i;
    double c0 = x[0], c1 = x[1], c2 = x[2];
    if (d.is_free[i]) {
      const double d0 = -d.y[3 * i] * d.scale[3 * i], d1 = -d.y[3 * i + 1] * d.scale[3 * i + 1],
                   d2 = -d.y[3 * i + 2] * d.scale[3 * i + 2];
      c0 = x[0] + d0; c1 = x[1] + d1; c2 = wrap_angle(x[2] + d2);   // AngleLocalParameterization, ceres_utils.h:38-54
      s[0] += (x[0] - c0) * (x[0] - c0) + (x[1] - c1) * (x[1] - c1) + (x[2] - c2) * (x[2] - c2);
    }
    d.xc[3 * i] = c0; d.xc[3 * i + 1] = c1; d.xc[3 * i + 2] = c2;
  }
  block_sum<1>(s, red);
  if (threadIdx.x == 0) d.partial[blockIdx.x] = s[0];
}

// model_cost_change = -(J~ step)^T (r + J~ step / 2) with step = -y (TrustRegionMinimizer::ComputeTrustRegionStep)
__global__ void __launch_bounds__(kPgThreads) k_pg_model_change(PgDev d)
{
  __shared__ double red[32];
  double s[1] = {0};
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < d.E; e += gridDim.x * blockDim.x) {
    const int a = d.eidx[2 * e], b = d.eidx[2 * e + 1];
    const double * L = d.lin + (size_t)kLin * e;
    const double sa0 = -d.y[3 * a], sa1 = -d.y[3 * a + 1], sa2 = -d.y[3 * a + 2];
    const double sb0 = -d.y[3 * b], sb1 = -d.y[3 * b + 1], sb2 = -d.y[3 * b + 2];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double m = L[3 + 3 * i] * sa0 + L[4 + 3 * i] * sa1 + L[5 + 3 * i] * sa2 + L[12 + 3 * i] * sb0 +
                       L[13 + 3 * i] * sb1 + L[14 + 3 * i] * sb2;
      s[0] -= m * (L[i] + 0.5 * m);
    }
  }
  block_sum<1>(s, red);
  if (threadIdx.x == 0) d.partial[blockIdx.x] = s[0];
}

// ------------------------------------------------------------------------------------------
// Dogleg (DoglegStrategy, DESIGN.md §4).  In the scaled space of Ceres' dogleg, with D = sqrt(diag):
//   g_s = g / D,  gn_s = -D y_gn  (y_gn: PCG solution of (H + mu D^2) y = g),  J D^-1 g_s = J~ (g / D^2) = u,
//   J D^-1 gn_s = -J~ y_gn = -w.
// The host needs the six Gram scalars of {g_s, gn_s} and of their images {u, -w}; every step the strategy can take
// is a combination of g_s and gn_s, so the device only ever composes  y = cg (g / D^2) + cy y_gn  (k_pg_dogleg_compose)
// and k_pg_model_change / k_pg_apply_step run unchanged on it.
// ------------------------------------------------------------------------------------------

// per node: partials of ||g_s||^2 = sum g^2/D^2, ||gn_s||^2 = sum D^2 y^2, sum g.y (= -g_s.gn_s) -> partial slots 0..2
__global__ void __launch_bounds__(kPgThreads) k_pg_dogleg_nodes(PgDev d, const double * __restrict__ ygn)
{
  __shared__ double red[3 * 32];
  double s[3] = {0, 0, 0};
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 3 * d.N; k += gridDim.x * blockDim.x) {
    const double g = d.g[k], dg = d.diag[k], y = ygn[k];
    s[0] += g * g / dg;
    s[1] += dg * y * y;
    s[2] += g * y;
  }
  block_sum<3>(s, red);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) d.partial[k * kMaxPartials + blockIdx.x] = s[k];
}

// per edge: u = J~_e (g / D^2), w = J~_e y_gn from the linearisation record; partials of ||u||^2, ||w||^2, u.w -> slots 0..2
__global__ void __launch_bounds__(kPgThreads) k_pg_dogleg_edges(PgDev d, const double * __restrict__ ygn)
{
  __shared__ double red[3 * 32];
  double s[3] = {0, 0, 0};
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < d.E; e += gridDim.x * blockDim.x) {
    const int a = d.eidx[2 * e], b = d.eidx[2 * e + 1];
    const double * L = d.lin + (size_t)kLin * e;
    double va[3], vb[3], ya[3], yb[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      va[k] = d.g[3 * a + k] / d.diag[3 * a + k]; vb[k] = d.g[3 * b + k] / d.diag[3 * b + k];
      ya[k] = ygn[3 * a + k]; yb[k] = ygn[3 * b + k];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double * A = L + 3 + 3 * i, * B = L + 12 + 3 * i;
      const double u = A[0] * va[0] + A[1] * va[1] + A[2] * va[2] + B[0] * vb[0] + B[1] * vb[1] + B[2] * vb[2];
      const double w = A[0] * ya[0] + A[1] * ya[1] + A[2] * ya[2] + B[0] * yb[0] + B[1] * yb[1] + B[2] * yb[2];
      s[0] += u * u; s[1] += w * w; s[2] += u * w;
    }
  }
  block_sum<3>(s, red);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) d.partial[k * kMaxPartials + blockIdx.x] = s[k];
}

// the dogleg step in the y convention of k_pg_model_change / k_pg_apply_step (step = -y)
__global__ void k_pg_dogleg_compose(PgDev d, const double * __restrict__ ygn, double cg, double cy)
{
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 3 * d.N; k += gridDim.x * blockDim.x)
    d.y[k] = cg * (d.g[k] / d.diag[k]) + cy * ygn[k];
}

// fixed-order sums of partial slots 0..n-1 into scalars[slot0 + k] (k_pg_reduce for several sums)
__global__ void k_pg_reduce_n(PgDev d, int nparts, int n, int slot0)
{
  if (threadIdx.x >= n) return;
  double s = 0;
  for (int i = 0; i < nparts; ++i) s += d.partial[threadIdx.x * kMaxPartials + i];
  d.scalars[slot0 + threadIdx.x] = s;
}

__global__ void k_pg_fill(double * p, double v, int n)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}

// ------------------------------------------------------------------------------------------
// k_pg_cholesky: the exact linear solve (linear_solver_type = 1, DESIGN.md §4 "Cholesky"). One persistent cooperative
// kernel factors (H + shift D^2) over the free nodes with a left-looking supernodal FP64 Cholesky, runs the forward solve
// inside the factor and the backward solve after it, and writes y and the relative residual.  The symbolic analysis
// (ordering, supernodes, panel layout, update and assembly lists) comes from the host (cholesky_analyze).
//
// Schedule and progress.  Supernodes are numbered in a postorder of the supernodal elimination tree, so every descendant
// of J has a lower number than J.  A CTA takes the next number from an atomic ticket and, before it starts that
// supernode, waits for the completion flags of its children (the backward solve takes the numbers in reverse and waits for
// the parent).  Progress is guaranteed because
//   (1) a CTA waits only on supernodes whose tickets are lower than the one it holds (children precede their parent in
//       postorder; in the reverse order the parent precedes its children),
//   (2) every lower ticket has been taken by a CTA that is running: tickets are handed out in increasing order only to
//       CTAs that ask for one, and the cooperative launch makes all CTAs of the grid co-resident,
//   (3) a CTA never waits on a higher ticket,
// so by induction on the ticket every supernode completes.  Flags hold the epoch of the solve that completed them (one
// number per launch, never reused), so they need no reset between solves.
// Every sum runs in a fixed order (descendants in ascending order, products over the panel's columns in order), so a
// solve is bit-reproducible.  Panels are read with ld.global.cg: another CTA may have written them after this SM's L1
// saw the same line.
// ------------------------------------------------------------------------------------------
constexpr int kCholMaxWidth = 16;   // block columns of one supernode: its 48 x 48 diagonal block is factored in smem
// -DB200_CHOL_CHECKS compiles device asserts of the schedule's and the layout's invariants (tools/chol_checked.py)
#ifdef B200_CHOL_CHECKS
#define CHOL_CHECK(cond) assert(cond)
#else
#define CHOL_CHECK(cond) ((void)0)
#endif
constexpr int kCholThreads = 256;

struct CholDev {
  int ns;                      // supernodes, in postorder
  const int32_t * sn_col;      // [ns + 1] first block column of each supernode
  const int32_t * row_start;   // [ns + 1] into rows
  const int32_t * rows;        // block rows of each supernode: its own columns, then the rows below, ascending
  const int64_t * off;         // [ns] offset of the supernode's column-major panel (leading dimension 3 x its rows) in L
  const int32_t * upd_start, * upd;       // [ns + 1]: the descendants that update each supernode, ascending
  const int32_t * child_start, * child;   // [ns + 1]: children in the supernodal elimination tree
  const int32_t * parent;      // [ns], -1 for a root
  const int32_t * tgt_start;   // [ns + 1] into tgt_off: the 3x3 blocks of each panel that receive original entries
  const int64_t * tgt_off;     // element offset of such a block (its row 0, column 0) in L
  const int32_t * src_start;   // [blocks + 1] into src
  const int32_t * src;         // a block's contributors in a fixed order: -1 - node (diagonal block), (edge << 1) | transposed
  const int32_t * col_node;    // [columns] node of every block column
  double * L;
  double * z;                  // [columns][3]: forward, then backward solution, by column
  unsigned int * flag;         // [2 ns] epochs of completion: factor + forward, backward
  unsigned int * ctl;          // [0], [1] tickets of the two phases (zeroed before launch); [2] epoch of a failed pivot
  unsigned int epoch;
};

// host symbolic analysis of the factor (cholesky_analyze)
struct CholSymbolic {
  std::vector<int32_t> col_node;   // [n] node of each block column
  std::vector<int32_t> node_col;   // [N] block column of each node, -1 when the node is not a column
  std::vector<int32_t> sn_col, row_start, rows, upd_start, upd, child_start, child, parent, sn_of_col;
  std::vector<int64_t> off;        // [ns + 1]
  int64_t info[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int * p)
{
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int * p, unsigned int v)
{
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int lower_bound_i32(const int32_t * a, int n, int v)
{
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (__ldg(a + m) < v) lo = m + 1; else hi = m; }
  return lo;
}
// thread 0 draws the CTA's next ticket
__device__ __forceinline__ int chol_ticket(unsigned int * counter, int * s)
{
  __syncthreads();
  if (threadIdx.x == 0) *s = (int)atomicAdd(counter, 1u);
  __syncthreads();
  return *s;
}
// all threads return once every flag of list[0..n) holds the epoch
__device__ __forceinline__ void chol_wait(const unsigned int * flag, const int32_t * list, int n, unsigned int epoch)
{
  for (int k = threadIdx.x; k < n; k += blockDim.x)
    while (ld_acquire_u32(flag + list[k]) != epoch) __nanosleep(64);
  __syncthreads();
}
__device__ __forceinline__ void chol_publish(unsigned int * f, unsigned int epoch)
{
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); st_release_u32(f, epoch); }
}

// Supernode J: assemble its panel, apply its descendants' updates (and their forward-solve terms), factor the diagonal
// block, solve the rows below it, and finish the forward solve of its columns.
__device__ void chol_factor_supernode(const PgDev & d, const CholDev & c, double shift, int J, double * sD, double * sZ)
{
  const int T = blockDim.x, tid = threadIdx.x;
  const int c0 = c.sn_col[J], w = c.sn_col[J + 1] - c0, W = 3 * w;
  const int nr = c.row_start[J + 1] - c.row_start[J], ld = 3 * nr;
  const int32_t * R = c.rows + c.row_start[J];
  double * P = c.L + c.off[J];
  CHOL_CHECK(w >= 1 && w <= kCholMaxWidth && nr >= w && c.off[J + 1] - c.off[J] == (int64_t)ld * W);
  // 1. assembly: zeros, then every receiving block as the fixed-order sum of its contributors
  for (int k = tid; k < ld * W; k += T) P[k] = 0.0;
  if (tid < W) sZ[tid] = d.g[3 * c.col_node[c0 + tid / 3] + tid % 3];
  __syncthreads();
  for (int t = c.tgt_start[J] + tid; t < c.tgt_start[J + 1]; t += T) {
    double b[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = c.src_start[t]; s < c.src_start[t + 1]; ++s) {
      const int v = c.src[s];
      if (v < 0) {
        const double * h = d.Hd + 6 * (-1 - v), * dg = d.diag + 3 * (-1 - v);
        b[0] += h[0] + dg[0] * shift; b[1] += h[1]; b[2] += h[2];
        b[3] += h[1]; b[4] += h[3] + dg[1] * shift; b[5] += h[4];
        b[6] += h[2]; b[7] += h[4]; b[8] += h[5] + dg[2] * shift;
      } else {
        const double * M = d.lin + (size_t)kLin * (v >> 1) + 21;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
          for (int j = 0; j < 3; ++j) b[3 * i + j] += (v & 1) ? M[3 * j + i] : M[3 * i + j];
      }
    }
    CHOL_CHECK(c.tgt_off[t] >= c.off[J] && c.tgt_off[t] + 2 * ld + 3 <= c.off[J + 1]);
    double * B = c.L + c.tgt_off[t];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) B[j * ld + i] = b[3 * i + j];
  }
  __syncthreads();
  // 2. updates from the descendants, in ascending order: P -= L_K[rows >= c0] L_K[rows in J's columns]^T, z_J -= ...
  for (int u = c.upd_start[J]; u < c.upd_start[J + 1]; ++u) {
    const int K = c.upd[u];
    const int nk = c.row_start[K + 1] - c.row_start[K], ldk = 3 * nk, Wk = 3 * (c.sn_col[K + 1] - c.sn_col[K]);
    const int32_t * RK = c.rows + c.row_start[K];
    const int a = lower_bound_i32(RK, nk, c0), bnd = lower_bound_i32(RK, nk, c0 + w);
    const double * PK = c.L + c.off[K];
    const int mi = 3 * (nk - a), mj = 3 * (bnd - a);
    CHOL_CHECK(K < J && bnd > a);   // a descendant (a lower ticket) with at least one row in J's columns
    for (int e = tid; e < mi * mj; e += T) {
      const int i = e % mi, j = e / mi;
      if (i < j) continue;   // upper triangle of J's diagonal block: never read
      const int ri = 3 * a + i, rj = 3 * a + j;
      double s = 0.0;
      for (int k = 0; k < Wk; ++k) s += __ldcg(PK + (size_t)k * ldk + ri) * __ldcg(PK + (size_t)k * ldk + rj);
      const int pi = lower_bound_i32(R, nr, __ldg(RK + a + i / 3));
      const int q = __ldg(RK + a + j / 3) - c0;
      CHOL_CHECK(pi < nr && R[pi] == RK[a + i / 3] && q >= 0 && q < w);
      P[(size_t)(3 * q + j % 3) * ld + 3 * pi + i % 3] -= s;
    }
    if (tid < mj) {
      const int rj = 3 * a + tid, ck = c.sn_col[K];
      double s = 0.0;
      for (int k = 0; k < Wk; ++k) s += __ldcg(PK + (size_t)k * ldk + rj) * __ldcg(c.z + 3 * ck + k);
      sZ[3 * (__ldg(RK + a + tid / 3) - c0) + tid % 3] -= s;
    }
    __syncthreads();
  }
  // 3. dense Cholesky of the diagonal block in shared memory (column-major, lower triangle)
  for (int e = tid; e < W * W; e += T) {
    const int i = e % W, j = e / W;
    if (i >= j) sD[j * W + i] = P[(size_t)j * ld + i];
  }
  __syncthreads();
  for (int k = 0; k < W; ++k) {
    if (tid == 0) {
      double p = sD[k * W + k];
      if (!(p > 0.0) || !isfinite(p)) {   // not positive definite: the solve fails, the NaN runs through to the residual
        p = __longlong_as_double(0x7FF8000000000000LL);
        atomicExch(c.ctl + 2, c.epoch);
      }
      sD[k * W + k] = sqrt(p);
    }
    __syncthreads();
    for (int i = k + 1 + tid; i < W; i += T) sD[k * W + i] /= sD[k * W + k];
    __syncthreads();
    const int m = W - k - 1;
    for (int e = tid; e < m * m; e += T) {
      const int i = k + 1 + e % m, j = k + 1 + e / m;
      if (i >= j) sD[j * W + i] -= sD[k * W + i] * sD[k * W + j];
    }
    __syncthreads();
  }
  for (int e = tid; e < W * W; e += T) {
    const int i = e % W, j = e / W;
    if (i >= j) P[(size_t)j * ld + i] = sD[j * W + i];
  }
  CHOL_CHECK(c.row_start[J] + w <= c.row_start[J + 1] && R[0] == c0 && R[w - 1] == c0 + w - 1);
  // forward solve of J's columns: L_JJ z_J = rhs
  if (tid == 0) {
    for (int j = 0; j < W; ++j) {
      double s = sZ[j];
      for (int k = 0; k < j; ++k) s -= sD[k * W + j] * sZ[k];
      sZ[j] = s / sD[j * W + j];
    }
  }
  // 4. the rows below: X L_JJ^T = B, one thread per scalar row
  for (int i = W + tid; i < ld; i += T) {
    for (int j = 0; j < W; ++j) {
      double s = P[(size_t)j * ld + i];
      for (int k = 0; k < j; ++k) s -= P[(size_t)k * ld + i] * sD[k * W + j];
      P[(size_t)j * ld + i] = s / sD[j * W + j];
    }
  }
  __syncthreads();
  if (tid < W) c.z[3 * c0 + tid] = sZ[tid];
}

// backward solve of supernode J: L_JJ^T y_J = z_J - L_J,below^T y_below (the rows below are ancestors, already solved)
__device__ void chol_backward_supernode(const PgDev & d, const CholDev & c, int J, double * sZ)
{
  const int tid = threadIdx.x;
  const int c0 = c.sn_col[J], W = 3 * (c.sn_col[J + 1] - c0);
  const int nr = c.row_start[J + 1] - c.row_start[J], ld = 3 * nr;
  const int32_t * R = c.rows + c.row_start[J];
  const double * P = c.L + c.off[J];
  for (int j = tid; j < W; j += blockDim.x) {
    double s = __ldcg(c.z + 3 * c0 + j);
    for (int i = W; i < ld; ++i) s -= __ldcg(P + (size_t)j * ld + i) * __ldcg(c.z + 3 * __ldg(R + i / 3) + i % 3);
    sZ[j] = s;
  }
  __syncthreads();
  if (tid == 0) {
    for (int j = W - 1; j >= 0; --j) {
      double s = sZ[j];
      for (int k = j + 1; k < W; ++k) s -= __ldcg(P + (size_t)j * ld + k) * sZ[k];
      sZ[j] = s / __ldcg(P + (size_t)j * ld + j);
    }
  }
  __syncthreads();
  if (tid < W) {
    c.z[3 * c0 + tid] = sZ[tid];
    d.y[3 * c.col_node[c0 + tid / 3] + tid % 3] = sZ[tid];
  }
}

// (H + shift D^2) y = g on the free nodes; y = 0 elsewhere.  scalars[8] = 0 (no iterations), scalars[9] = the relative
// residual ||(H + shift D^2) y - g|| / ||g||, or NaN when a pivot was not positive and finite.  scalars[10..12] = ns of the
// factor + forward phase, the backward phase and the residual, as CTA 0 sees them (%globaltimer; printed under B200PG_DEBUG).
__global__ void __launch_bounds__(kCholThreads) k_pg_cholesky(PgDev d, CholDev c, double shift)
{
  cg::grid_group grid = cg::this_grid();
  __shared__ double sD[9 * kCholMaxWidth * kCholMaxWidth];
  __shared__ double sZ[3 * kCholMaxWidth];
  __shared__ double red[2 * 32];
  __shared__ double bc[1];
  __shared__ int s_ticket;
  const int tid = threadIdx.x;
  const bool timer = blockIdx.x == 0 && tid == 0;
  unsigned long long t0 = 0, t1 = 0, t2 = 0, t3 = 0;
  if (timer) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (int i = blockIdx.x * blockDim.x + tid; i < d.N; i += gridDim.x * blockDim.x)
    if (!d.is_free[i]) { d.y[3 * i] = 0.0; d.y[3 * i + 1] = 0.0; d.y[3 * i + 2] = 0.0; }
  // factor + forward, supernodes in postorder; a supernode waits for its children
  for (int J = chol_ticket(c.ctl, &s_ticket); J < c.ns; J = chol_ticket(c.ctl, &s_ticket)) {
    for (int k = c.child_start[J] + tid; k < c.child_start[J + 1]; k += blockDim.x) CHOL_CHECK(c.child[k] < J && c.parent[c.child[k]] == J);
    chol_wait(c.flag, c.child + c.child_start[J], c.child_start[J + 1] - c.child_start[J], c.epoch);
    chol_factor_supernode(d, c, shift, J, sD, sZ);
    chol_publish(c.flag + J, c.epoch);
  }
  grid.sync();
  if (timer) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
  // backward, supernodes in reverse postorder; a supernode waits for its parent
  for (int t = chol_ticket(c.ctl + 1, &s_ticket); t < c.ns; t = chol_ticket(c.ctl + 1, &s_ticket)) {
    const int J = c.ns - 1 - t;
    CHOL_CHECK(c.parent[J] < 0 || c.parent[J] > J);   // the parent holds a lower backward ticket
    if (c.parent[J] >= 0) chol_wait(c.flag + c.ns, c.parent + J, 1, c.epoch);
    chol_backward_supernode(d, c, J, sZ);
    chol_publish(c.flag + c.ns + J, c.epoch);
  }
  grid.sync();
  if (timer) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t2));
  // relative residual with the PCG kernels' row product
  double acc[2] = {0, 0};
  for (int i = blockIdx.x * blockDim.x + tid; i < d.N; i += gridDim.x * blockDim.x) {
    double q[3], yi[3];
    spmv_row(d, i, d.y, nullptr, 0.0, shift, q, yi);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double r = q[k] - d.g[3 * i + k];
      acc[0] += r * r;
      acc[1] += d.g[3 * i + k] * d.g[3 * i + k];
    }
  }
  block_sum<2>(acc, red);
  if (tid == 0) { d.partial[blockIdx.x] = acc[0]; d.partial[kMaxPartials + blockIdx.x] = acc[1]; }
  grid.sync();
  const double rr = grid_total(d, 0, gridDim.x, bc), gg = grid_total(d, 1, gridDim.x, bc);
  if (timer) {
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t3));
    d.scalars[10] = (double)(t1 - t0); d.scalars[11] = (double)(t2 - t1); d.scalars[12] = (double)(t3 - t2);
    d.scalars[8] = 0.0;
    d.scalars[9] = ld_acquire_u32(c.ctl + 2) == c.epoch ? __longlong_as_double(0x7FF8000000000000LL) : (gg > 0.0 ? sqrt(rr / gg) : 0.0);
  }
}

}  // namespace b200

using namespace b200;

// ------------------------------------------------------------------------------------------
// host side: graph store + LM driver
// ------------------------------------------------------------------------------------------
struct PgEdge {
  int32_t ida, idb;
  double z[3];
  double U[6];
};

struct b200pg {
  b200pg_opts o{};
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // graph store (mirrors CeresSolver's nodes_ / blocks_)
  std::vector<int32_t> node_ids;              // insertion order
  std::vector<double> node_pose;              // [n][3]
  std::unordered_map<int32_t, int32_t> index; // id -> position in node_ids
  std::vector<PgEdge> edges;
  int32_t first_node_id = 0;
  bool have_first = false;
  // flattened edge arrays (node positions, measurement, sqrt information), kept in step with `edges`: AddConstraint appends
  // (the mapper's normal traffic, Mapper.cpp:1634), removals / Reset mark them for a rebuild.  dev_edges of them are already
  // on the device, so a Compute after k new constraints uploads k edges, not the graph (SURVEY.md 8f-2).
  std::vector<int32_t> f_eidx;
  std::vector<double> f_z, f_U;
  bool flat_dirty = false;
  size_t dev_edges = 0;
  std::vector<int32_t> agg_start_h, agg_of_h;
  // corrections of the last solve
  std::vector<int32_t> corr_ids;
  std::vector<double> corr_pose;
  // device
  DevBuf<int32_t> d_eidx, d_adj_start, d_adj, d_agg_start, d_agg_of;
  DevBuf<uint8_t> d_free;
  DevBuf<double> d_gz, d_gp, d_gPt, d_gRow, d_grc, d_e1, d_e2;
  bool debug = false;
  int precond = 1;   // 1 = two-level (rigid-mode aggregation) + block Jacobi, 0 = block Jacobi only
  int coarse_modes = 6;   // two-level: coarse modes per aggregate (6 = rigid + linear deformation, 3 = rigid only)
  DevBuf<unsigned int> d_bar;
  bool force_global_pcg = false;
  bool force_2lvl_global = false;   // B200PG_FORCE_2LVL_GLOBAL: plan k_pg_pcg_2lvl_g at any size
  DevBuf<double> d_gAc, d_gCb, d_gTb, d_gPtq;   // k_pg_pcg_2lvl_g: dense coarse matrix / inverse and its step panels
  DevBuf<double> d_z, d_U, d_x, d_xc, d_scale, d_lin, d_Hd, d_g, d_diag, d_y, d_pr, d_pz, d_pp0, d_pp1, d_pq, d_Minv,
    d_partial, d_scalars;
  DevBuf<double> d_ygn;   // dogleg: the Gauss-Newton solution, kept for the iterations that reuse it
  // Cholesky linear solver (linear_solver_type = 1): the analysis in use and what it was made for (free nodes, adjacent
  // pairs); chol_stale forces a new one after a removal or Reset
  std::vector<uint8_t> free_h;   // is_free of the last upload
  b200::CholSymbolic chol;
  std::vector<uint8_t> chol_free;
  std::vector<int64_t> chol_pairs;
  bool chol_stale = true, chol_valid = false;
  int64_t chol_asm_edges = -1;   // edges the device's assembly lists were built from; -1 = none for the current analysis
  int64_t chol_analyses = 0;
  int64_t chol_info[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // the analysis the last Cholesky solve used
  unsigned int chol_epoch = 0;
  DevBuf<int32_t> d_ch_sn_col, d_ch_row_start, d_ch_rows, d_ch_upd_start, d_ch_upd, d_ch_child_start, d_ch_child, d_ch_parent,
    d_ch_tgt_start, d_ch_src_start, d_ch_src, d_ch_col_node;
  DevBuf<int64_t> d_ch_off, d_ch_tgt_off;
  DevBuf<double> d_ch_L, d_ch_z;
  DevBuf<unsigned int> d_ch_flag, d_ch_ctl;
  PinBuf<double> h_scalars;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int64_t launches = 0;
};

namespace b200 {

void b200pg_defaults(b200pg_opts * o)
{
  o->max_num_iterations = 50;
  o->function_tolerance = 1e-3;
  o->gradient_tolerance = 1e-6;
  o->parameter_tolerance = 1e-3;
  o->min_relative_decrease = 1e-3;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e8;
  o->min_trust_region_radius = 1e-16;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->jacobi_scaling = 1;
  o->use_nonmonotonic_steps = 1;
  o->max_consecutive_nonmonotonic_steps = 3;
  o->max_num_consecutive_invalid_steps = 3;
  o->pcg_tolerance = 1e-9;    // loosest tolerance that keeps cfg4 (0.05 m / 0.02 rad) within 5e-6 m of the exact-solve LM (tools/pcg_tolerance_study.py)
  o->pcg_max_iterations = 20000;
  o->loss_function = 0;
  o->loss_scale = 0.7;
  o->trust_region_strategy = 0;
  o->dogleg_type = 0;
  o->linear_solver_type = 0;
}

// karto::Matrix3::Inverse by cofactors (Karto.h:2533-2577) then Eigen's llt().matrixU()
// of the matrix rebuilt from its upper triangle (ceres_solver.cpp:364-376)
static bool sqrt_information(const double cov[9], double U[6])
{
  const double * m = cov;
  double inv[9];
  inv[0] = m[4] * m[8] - m[5] * m[7];
  inv[1] = m[2] * m[7] - m[1] * m[8];
  inv[2] = m[1] * m[5] - m[2] * m[4];
  inv[3] = m[5] * m[6] - m[3] * m[8];
  inv[4] = m[0] * m[8] - m[2] * m[6];
  inv[5] = m[2] * m[3] - m[0] * m[5];
  inv[6] = m[3] * m[7] - m[4] * m[6];
  inv[7] = m[1] * m[6] - m[0] * m[7];
  inv[8] = m[0] * m[4] - m[1] * m[3];
  double det = m[0] * inv[0] + m[1] * inv[3] + m[2] * inv[6];
  if (!(fabs(det) > 1e-14)) return false;   // Matrix3::Inverse asserts
  double id = 1.0 / det;
  for (int i = 0; i < 9; ++i) inv[i] *= id;
  const double a00 = inv[0], a01 = inv[1], a02 = inv[2], a11 = inv[4], a12 = inv[5], a22 = inv[8];
  if (!(a00 > 0)) return false;
  const double l00 = sqrt(a00), l10 = a01 / l00, l20 = a02 / l00;
  const double t11 = a11 - l10 * l10;
  if (!(t11 > 0)) return false;
  const double l11 = sqrt(t11), l21 = (a12 - l20 * l10) / l11;
  const double t22 = a22 - l20 * l20 - l21 * l21;
  if (!(t22 > 0)) return false;
  const double l22 = sqrt(t22);
  U[0] = l00; U[1] = l10; U[2] = l20; U[3] = l11; U[4] = l21; U[5] = l22;
  return true;
}

template <class T>
static void up(DevBuf<T> & dst, const std::vector<T> & src, cudaStream_t s)
{
  dst.reserve(std::max<size_t>(src.size(), 1));
  if (!src.empty()) B200_CUDA(cudaMemcpyAsync(dst.p, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice, s));
}

// grow a device buffer to n elements keeping its first `keep` ones
template <class T>
static void grow_keep(DevBuf<T> & b, size_t n, size_t keep, cudaStream_t s)
{
  if (n <= b.cap) return;
  if (keep == 0 || !b.p) { b.reserve(n); return; }
  DevBuf<T> nb;
  nb.reserve(n + n / 2);
  B200_CUDA(cudaMemcpyAsync(nb.p, b.p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s));
  B200_CUDA(cudaStreamSynchronize(s));
  std::swap(b.p, nb.p); std::swap(b.cap, nb.cap);
}

// ---- dogleg strategy: host FP64 algebra on six Gram scalars (DESIGN.md §4) ----
// Every step the strategy takes is s_s = ca g_s + cb gn_s in the scaled space; the device composes it from (ca, cb).
constexpr double kDlMinMu = 1e-8, kDlMaxMu = 1.0, kDlMuIncrease = 10.0, kDlKktCosine = 0.99;
// The Gauss-Newton solve runs 10x tighter than pcg_tolerance: its nearly undamped step (mu ~ 1e-8) carries the PCG error
// into the iterate in full, and at 1e-9 the final cost of cfg4 (0.05 m / 0.02 rad) is 1.2e-8 away from the exact-solve
// oracle's, at 1e-10 4.4e-10 (tools/dogleg_study.py on an H100, DESIGN.md §4).
constexpr double kDlPcgTolFactor = 0.1;

struct DoglegModel {
  double G[2][2];    // Gram matrix of (g_s, gn_s)
  double GJ[2][2];   // Gram matrix of their images J D^-1 g_s, J D^-1 gn_s
  double alpha;      // Cauchy factor ||g_s||^2 / ||J D^-1 g_s||^2
  bool rank1;
  double C[2][2];    // orthonormal basis of span{g_s, gn_s}: column k = C[0][k] g_s + C[1][k] gn_s
  double g2[2], B2[2][2];   // the 2-D model in that basis

  // from k_pg_dogleg_nodes / k_pg_dogleg_edges: sum g^2/D^2, sum D^2 y^2, sum g.y, ||u||^2, ||w||^2, u.w
  void set(const double * s)
  {
    G[0][0] = s[0]; G[1][1] = s[1]; G[0][1] = G[1][0] = -s[2];
    GJ[0][0] = s[3]; GJ[1][1] = s[4]; GJ[0][1] = GJ[1][0] = -s[5];
    alpha = G[0][0] / GJ[0][0];
  }
  // column-pivoted QR of [g_s gn_s] carried out on the Gram matrix; rank 1 when |R22| <= 2 eps |R11|
  void subspace()
  {
    const int p = G[1][1] > G[0][0] ? 1 : 0, q = 1 - p;
    const double r11 = sqrt(G[p][p]), r12 = G[p][q] / r11, r22 = sqrt(std::max(0.0, G[q][q] - r12 * r12));
    rank1 = !(r22 > 2.0 * 2.220446049250313e-16 * r11);
    C[p][0] = 1.0 / r11; C[q][0] = 0.0;
    C[p][1] = rank1 ? 0.0 : -r12 / (r11 * r22); C[q][1] = rank1 ? 0.0 : 1.0 / r22;
    for (int k = 0; k < 2; ++k) g2[k] = C[0][k] * G[0][0] + C[1][k] * G[1][0];
    for (int k = 0; k < 2; ++k)
      for (int l = 0; l < 2; ++l) {
        double s = 0;
        for (int i = 0; i < 2; ++i)
          for (int j = 0; j < 2; ++j) s += C[i][k] * GJ[i][j] * C[j][l];
        B2[k][l] = s;
      }
  }
  double norm(double ca, double cb) const
  {
    return sqrt(std::max(0.0, ca * ca * G[0][0] + 2.0 * ca * cb * G[0][1] + cb * cb * G[1][1]));
  }
};

// the four complex roots of c[0] y^4 + ... + c[4] (Aberth-Ehrlich iteration; no LAPACK in this library)
static void quartic_roots(const double c[5], std::complex<double> z[4])
{
  using cd = std::complex<double>;
  double a[5], rad = 0.0;
  for (int k = 0; k < 5; ++k) a[k] = c[k] / c[0];
  for (int k = 1; k < 5; ++k) rad = std::max(rad, pow(fabs(a[k]), 1.0 / k));
  if (!(rad > 0.0)) rad = 1.0;
  for (int k = 0; k < 4; ++k) z[k] = std::polar(rad, 0.7 + 2.0 * M_PI * k / 4.0);
  for (int iter = 0; iter < 500; ++iter) {
    bool moved = false;
    for (int i = 0; i < 4; ++i) {
      cd p = a[0], dp = 0.0;
      for (int k = 1; k < 5; ++k) { dp = dp * z[i] + p; p = p * z[i] + a[k]; }
      if (p == 0.0) continue;
      cd s = 0.0;
      for (int j = 0; j < 4; ++j)
        if (j != i) s += 1.0 / (z[i] - z[j]);
      const cd ratio = p / dp, w = ratio / (1.0 - ratio * s);
      if (!std::isfinite(w.real()) || !std::isfinite(w.imag())) continue;
      if (std::abs(w) > 1e-16 * std::abs(z[i])) moved = true;
      z[i] -= w;
    }
    if (!moved) break;
  }
}

// minimum of 1/2 x^T B x + g^T x on ||x|| = r over the stationary points (B + y I) x = -g, y a root of the quartic;
// false when no root gives a usable point or the first-order (KKT) check fails
static bool boundary_minimum(const double g[2], const double B[2][2], double r, double x[2])
{
  const double tr = B[0][0] + B[1][1], det = B[0][0] * B[1][1] - B[0][1] * B[1][0];
  const double ag0 = B[1][1] * g[0] - B[0][1] * g[1], ag1 = -B[1][0] * g[0] + B[0][0] * g[1];
  const double r2 = r * r;
  const double poly[5] = {r2, 2.0 * r2 * tr, r2 * (tr * tr + 2.0 * det) - (g[0] * g[0] + g[1] * g[1]),
                          -2.0 * ((g[0] * ag0 + g[1] * ag1) - r2 * det * tr), r2 * det * det - (ag0 * ag0 + ag1 * ag1)};
  std::complex<double> z[4];
  quartic_roots(poly, z);
  bool found = false;
  double best_f = INFINITY;
  for (int k = 0; k < 4; ++k) {
    const double y = z[k].real();
    const double m00 = B[0][0] + y, m01 = B[0][1], m10 = B[1][0], m11 = B[1][1] + y;
    const double dm = m00 * m11 - m01 * m10;
    if (dm == 0.0) continue;
    double x0 = -(m11 * g[0] - m01 * g[1]) / dm, x1 = -(-m10 * g[0] + m00 * g[1]) / dm;
    const double n = sqrt(x0 * x0 + x1 * x1);
    if (!std::isfinite(n) || !(n > 0.0)) continue;
    x0 *= r / n; x1 *= r / n;
    const double f = 0.5 * (x0 * (B[0][0] * x0 + B[0][1] * x1) + x1 * (B[1][0] * x0 + B[1][1] * x1)) + g[0] * x0 + g[1] * x1;
    if (f < best_f) { best_f = f; x[0] = x0; x[1] = x1; found = true; }
  }
  if (!found) return false;
  const double q0 = B[0][0] * x[0] + B[0][1] * x[1] + g[0], q1 = B[1][0] * x[0] + B[1][1] * x[1] + g[1];
  const double cosine = -(x[0] * q0 + x[1] * q1) / (sqrt(x[0] * x[0] + x[1] * x[1]) * sqrt(q0 * q0 + q1 * q1));
  return !(cosine < kDlKktCosine);
}

// ComputeTraditionalDoglegStep / ComputeSubspaceDoglegStep: coefficients of s_s = ca g_s + cb gn_s and ||s_s||
static void traditional_step(const DoglegModel & m, double radius, double & ca, double & cb, double & step_norm)
{
  const double gn_norm = sqrt(m.G[1][1]), g_norm = sqrt(m.G[0][0]);
  if (gn_norm <= radius) { ca = 0.0; cb = 1.0; step_norm = gn_norm; return; }
  if (m.alpha * g_norm >= radius) { ca = -radius / g_norm; cb = 0.0; step_norm = radius; return; }
  // the point where the segment a = -alpha g_s -> b = gn_s crosses ||.|| = radius, in Ceres' cancellation-safe form
  const double b_dot_a = -m.alpha * m.G[0][1], a_sq = m.alpha * m.alpha * m.G[0][0];
  const double bma_sq = a_sq - 2.0 * b_dot_a + m.G[1][1];
  const double c = b_dot_a - a_sq;
  const double dd = sqrt(c * c + bma_sq * (radius * radius - a_sq));
  const double beta = c <= 0 ? (dd - c) / bma_sq : (radius * radius - a_sq) / (dd + c);
  ca = -(1.0 - beta) * m.alpha; cb = beta;
  step_norm = m.norm(ca, cb);
}

static void subspace_step(const DoglegModel & m, double radius, double & ca, double & cb, double & step_norm)
{
  const double gn_norm = sqrt(m.G[1][1]);
  if (gn_norm <= radius) { ca = 0.0; cb = 1.0; step_norm = gn_norm; return; }
  if (m.rank1) { ca = -radius / sqrt(m.G[0][0]); cb = 0.0; step_norm = radius; return; }
  double x[2];
  if (!boundary_minimum(m.g2, m.B2, radius, x)) { traditional_step(m, radius, ca, cb, step_norm); return; }
  ca = m.C[0][0] * x[0] + m.C[0][1] * x[1];
  cb = m.C[1][0] * x[0] + m.C[1][1] * x[1];
  step_norm = radius;
}

// The linear-solve kernel of a solve and how it is launched. kernel is the b200pg_summary.linear_solver code: 0 global
// block-Jacobi, 1 shared-memory block-Jacobi, 3 / 6 two-level with that many coarse modes per aggregate (PCG), 13 / 16 the
// same two-level preconditioner with global-memory aggregates and a dense coarse inverse (k_pg_pcg_2lvl_g), 8 Cholesky.
constexpr int kLinearSolverCholesky = 8;
struct PcgPlan {
  int kernel = 0;
  int blocks = 0;           // cooperative grid
  size_t smem_bytes = 0;    // dynamic shared memory
  PcgSmemCfg smem{};        // kernel 1
  Pcg2Cfg two_level{};      // kernels 3 and 6
  Pcg2GCfg two_level_g{};   // kernels 13 and 16
};

constexpr int kMin2lvlGlobalNodes = 8192;
constexpr int kMaxCoarse2lvlGlobal = 4096;

// Algorithmic bytes of one CG iteration's fine level (SpMV, block-Jacobi, vector updates) on a graph of N nodes and `slots`
// CSR slots (2 E): per node Hd, D, Minv and the ten vector streams (30 doubles), per slot its 3x3 block, the neighbour's
// z and p and the slot's index words.
static double pcg_fine_bytes(double N, double slots) { return 240.0 * N + 128.0 * slots; }

// The coarse size of k_pg_pcg_2lvl_g: nc = CM x aggregates, with the dense Ac^-1 mat-vec (8 nc^2 bytes per iteration) held
// to a quarter of the fine level's bytes, nc <= sqrt(fine / 32), at most kMaxCoarse2lvlGlobal (the inverse costs 2 nc^3 flops
// and 16 nc^2 bytes per kGjPanel columns once per solve) and aggregates of at least 16 nodes.
static int coarse_aggregates_2lvl_global(int N, int slots, int cm)
{
  const int nc = std::min(kMaxCoarse2lvlGlobal, (int)std::sqrt(pcg_fine_bytes(N, slots) / 32.0));
  return std::max(1, std::min((N + 15) / 16, nc / cm));
}

// Plans k_pg_pcg_2lvl_g into P (kernel 13 or 16) when its dense coarse inverse fits the free device memory; otherwise
// leaves P as it is (B200PG_DEBUG says why).
static void plan_pcg_2lvl_global(b200pg * h, const std::vector<int32_t> & adj_start, int sms, cudaStream_t st, PcgPlan & P)
{
  const int N = (int)adj_start.size() - 1;
  const int cm = h->coarse_modes >= 6 ? 6 : 3;
  const int want = coarse_aggregates_2lvl_global(N, adj_start[N], cm);
  std::vector<int32_t> agg_start, agg_of(N, 0);
  const int per = (N + want - 1) / want;
  for (int i = 0; i < N; i += per) agg_start.push_back(i);
  agg_start.push_back(N);
  const int na = (int)agg_start.size() - 1;
  for (int a = 0; a < na; ++a)
    for (int i = agg_start[a]; i < agg_start[a + 1]; ++i) agg_of[i] = a;
  const int nc = cm * na, ld = (nc + kGjTile - 1) / kGjTile * kGjTile;
  const void * fn = cm == 6 ? (const void *)k_pg_pcg_2lvl_g<6> : (const void *)k_pg_pcg_2lvl_g<3>;
  // shared memory: the coarse residual, then the largest scratch of the three stages (assembly staging, Gauss-Jordan
  // tiles, exchange + coarse values; the last is at most 2 G + cm na doubles, G <= 2 sms)
  const size_t scratch = std::max<size_t>({(size_t)(kG2Threads / 32) * 32 * 12, 2 * kGjPanel * kGjTile + kGjPanel * kGjPanel,
                                           4 * (size_t)sms + (size_t)nc});
  const size_t bytes = ((size_t)ld + scratch) * sizeof(double);
  int occ = 0;
  if (bytes <= 220 * 1024) {
    B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kG2Threads, bytes));
    occ = std::min(occ, 2);
  }
  if (occ < 1) {
    if (h->debug) fprintf(stderr, "[b200pg] two-level global plan: %zu B of shared memory for nc = %d do not fit; kernel 0\n", bytes, nc);
    return;
  }
  const int apc = (na + std::min(na, occ * sms) - 1) / std::min(na, occ * sms);
  const int G = (na + apc - 1) / apc;
  // device memory the plan adds: Ac, the two step panels, P^T q and the initial coarse residual, P~, p and z, slots, indices
  auto grow = [](const DevBuf<double> & b, size_t n) { return n > b.cap ? (n + n / 4 + 16) * sizeof(double) : (size_t)0; };
  const size_t n3 = 3 * (size_t)N;
  const size_t need = grow(h->d_gAc, (size_t)ld * ld) + grow(h->d_gCb, (size_t)kGjPanel * ld) + grow(h->d_gTb, (size_t)kGjPanel * ld) +
                      grow(h->d_gPtq, ld) + grow(h->d_grc, ld) + grow(h->d_gPt, 10 * (size_t)N) + grow(h->d_gz, n3) + grow(h->d_gp, 2 * n3) +
                      (size_t)(2 * N + na) * sizeof(int32_t) + 4 * (size_t)G * kSlotStride * sizeof(double);
  size_t free_b = 0, total_b = 0;
  B200_CUDA(cudaMemGetInfo(&free_b, &total_b));
  if (need + (size_t)64 * 1024 * 1024 > free_b) {
    if (h->debug) fprintf(stderr, "[b200pg] two-level global plan: the dense coarse inverse (nc = %d, %zu MB) needs %zu MB, %zu MB free; kernel 0\n", nc, (size_t)ld * ld * 8 >> 20, need >> 20, free_b >> 20);
    return;
  }
  if (h->debug) fprintf(stderr, "[b200pg] two-level global plan: %d aggregates x %d modes (nc = %d, ld = %d), %d nodes each, %d CTAs x %d aggregates, %zu B smem\n", na, cm, nc, ld, per, G, apc, bytes);
  h->d_gAc.reserve((size_t)ld * ld); h->d_gCb.reserve((size_t)kGjPanel * ld); h->d_gTb.reserve((size_t)kGjPanel * ld);
  h->d_gPtq.reserve(ld); h->d_grc.reserve(ld); h->d_gPt.reserve(10 * (size_t)N); h->d_gz.reserve(n3); h->d_gp.reserve(2 * n3);
  h->d_bar.reserve(4096); h->d_e1.reserve((size_t)2 * G * kSlotStride); h->d_e2.reserve((size_t)2 * G * kSlotStride);
  h->agg_start_h.swap(agg_start); h->agg_of_h.swap(agg_of);   // the vectors live in the handle
  up(h->d_agg_start, h->agg_start_h, st); up(h->d_agg_of, h->agg_of_h, st);
  P = PcgPlan{};
  P.kernel = 10 + cm; P.blocks = G; P.smem_bytes = bytes;
  Pcg2GCfg & c = P.two_level_g;
  c.na = na; c.apc = apc; c.ld = ld; c.agg_start = h->d_agg_start.p; c.agg_of = h->d_agg_of.p;
  c.gz = h->d_gz.p; c.gp = h->d_gp.p; c.gPt = h->d_gPt.p; c.Ac = h->d_gAc.p; c.Cb = h->d_gCb.p; c.Tb = h->d_gTb.p;
  c.gPtq = h->d_gPtq.p; c.grc = h->d_grc.p; c.e1 = h->d_e1.p; c.e2 = h->d_e2.p; c.bar = h->d_bar.p;
}

// Picks the PCG kernel from the graph's CSR rows: shared-memory block-Jacobi where every CTA's rows fit, then the two-level
// kernel where its aggregates fit (B200PG_PRECOND, B200PG_COARSE_MODES and B200PG_FORCE_GLOBAL_PCG narrow the choice).
// Allocates the work buffers of the kernels it considers.
static PcgPlan plan_pcg(b200pg * h, const std::vector<int32_t> & adj_start, cudaStream_t st)
{
  const int N = (int)adj_start.size() - 1;
  const size_t n3 = 3 * (size_t)N;
  PcgPlan P;
  int dev = 0, sms = 132, per_sm = 1;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pg_pcg, kPgThreads, 0));
  P.blocks = std::max(1, std::min({kMaxPartials, sms * std::max(per_sm, 1), (N + kPgThreads - 1) / kPgThreads}));

  {
    // shared-memory-resident PCG when every CTA's rows fit (one CTA per SM, 512 threads)
    const int G = std::min(sms, std::max(1, (N + 31) / 32));
    const int npc = (N + G - 1) / G;
    const int Gu = (N + npc - 1) / npc;
    int max_slots = 0;
    for (int c = 0; c < Gu; ++c) {
      const int lo = c * npc, hi = std::min(N, lo + npc);
      max_slots = std::max(max_slots, adj_start[hi] - adj_start[lo]);
    }
    max_slots = std::max(max_slots, 1);
    const size_t bytes = ((size_t)max_slots * 12 + (size_t)npc * 27) * sizeof(double) + ((size_t)max_slots + npc + 1) * sizeof(int) + 16;
    if (bytes <= 200 * 1024 && !h->force_global_pcg) {
      P.kernel = 1; P.blocks = Gu; P.smem_bytes = bytes;
      h->d_gz.reserve(n3); h->d_gp.reserve(2 * n3); h->d_bar.reserve(4096);
      P.smem.npc = npc; P.smem.max_slots = max_slots; P.smem.gz = h->d_gz.p; P.smem.gp = h->d_gp.p; P.smem.bar = h->d_bar.p;
      B200_CUDA(cudaFuncSetAttribute(k_pg_pcg_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    }
  }
  if (h->precond == 1 && !h->force_global_pcg) {
    // two-level preconditioner: one aggregate per 256-thread CTA. One CTA per SM is preferred: with two per SM
    // CG needs fewer iterations, but the all-to-all exchanges and the Gauss-Jordan, whose cost grows with the number of
    // aggregates, get slower per iteration and the solve as a whole slower. Two per SM is the
    // fallback when one aggregate per SM does not fit shared memory.
    for (int per_sm = 1; per_sm <= 2 && P.kernel < 3; ++per_sm) {
      const int G2 = std::min(per_sm * sms, std::max(1, (N + 15) / 16));
      // contiguous node ranges of equal node count: compact aggregates give the best coarse space (balancing by
      // block count was tried: it merges sparse chain stretches into large aggregates and costs more iterations)
      std::vector<int32_t> & agg_start = h->agg_start_h;
      std::vector<int32_t> & agg_of = h->agg_of_h;
      agg_start.clear(); agg_of.assign(N, 0);
      {
        const int per = (N + G2 - 1) / G2;
        for (int i = 0; i < N; i += per) agg_start.push_back(i);
        agg_start.push_back(N);
        for (int a = 0; a + 1 < (int)agg_start.size(); ++a)
          for (int i = agg_start[a]; i < agg_start[a + 1]; ++i) agg_of[i] = a;
      }
      const int Gu = (int)agg_start.size() - 1;
      int max_slots = 1, npc = 1;
      for (int c = 0; c < Gu; ++c) {
        max_slots = std::max(max_slots, adj_start[agg_start[c + 1]] - adj_start[agg_start[c]]);
        npc = std::max(npc, agg_start[c + 1] - agg_start[c]);
      }
      // coarse modes per aggregate: 6 (rigid + piecewise-linear deformation) when it fits shared memory, else 3
      int cm = 0, nc = 0, ex_doubles = 0;
      size_t bytes2 = 0;
      for (int try_cm : {6, 3}) {
        if (try_cm > h->coarse_modes) continue;
        nc = try_cm * Gu;
        ex_doubles = std::max((1 + try_cm) * Gu, try_cm * nc - 3 * max_slots);
        bytes2 = ((size_t)max_slots * 12 + (size_t)npc * 37 + (size_t)(try_cm + 1) * nc + (size_t)ex_doubles) * sizeof(double) +
                 ((size_t)2 * max_slots + npc + 1) * sizeof(int) + 16;
        if (bytes2 > 220 * 1024) continue;
        int occ = 0;
        const void * fn = try_cm == 6 ? (const void *)k_pg_pcg_2lvl<6> : (const void *)k_pg_pcg_2lvl<3>;
        B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes2));
        B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, 256, bytes2));
        if (h->debug) fprintf(stderr, "[b200pg] two-level plan: %d aggregates x %d modes, <= %d nodes and <= %d blocks each, %zu B smem, occupancy %d/SM\n", Gu, try_cm, npc, max_slots, bytes2, occ);
        if (occ * sms < Gu) continue;
        cm = try_cm;
        break;
      }
      if (!cm) continue;
      P.kernel = cm; P.blocks = Gu; P.smem_bytes = bytes2;
      h->d_gz.reserve(n3); h->d_gp.reserve(2 * n3);
      h->d_bar.reserve(std::max<size_t>(4096, (size_t)Gu + 4));
      h->d_gPt.reserve(10 * (size_t)N); h->d_gRow.reserve((size_t)Gu * cm * 2 * nc); h->d_grc.reserve(nc);
      h->d_e1.reserve((size_t)2 * Gu * kSlotStride); h->d_e2.reserve((size_t)2 * Gu * kSlotStride);
      up(h->d_agg_start, agg_start, st); up(h->d_agg_of, agg_of, st);   // the vectors live in the handle
      Pcg2Cfg & c2 = P.two_level;
      c2.npc = npc; c2.max_slots = max_slots; c2.ex_doubles = ex_doubles; c2.agg_start = h->d_agg_start.p; c2.agg_of = h->d_agg_of.p;
      c2.gz = h->d_gz.p; c2.gp = h->d_gp.p; c2.gPt = h->d_gPt.p; c2.gRow = h->d_gRow.p;
      c2.grc = h->d_grc.p; c2.e1 = h->d_e1.p; c2.e2 = h->d_e2.p; c2.bar = h->d_bar.p; c2.gjflag = h->d_bar.p + 1;
    }
  }
  // Past the shared-memory kernels' reach, the two-level preconditioner with global-memory aggregates instead of kernel 0.
  // Below kMin2lvlGlobalNodes a plan ends on kernel 0 only when one row (a hub node) is too long for shared memory. Those
  // graphs keep kernel 0 so that the plan of every graph of that size stays what it was before this kernel existed; which
  // of the two kernels is faster there has not been measured. B200PG_FORCE_2LVL_GLOBAL plans it at any size.
  if (h->precond == 1 && !h->force_global_pcg && (h->force_2lvl_global || (P.kernel == 0 && N >= kMin2lvlGlobalNodes)))
    plan_pcg_2lvl_global(h, adj_start, sms, st, P);
  return P;
}

// ---- Cholesky linear solver: host symbolic analysis (DESIGN.md §4 "Cholesky") ----

// The adjacent pairs of free nodes as sorted, unique keys lo * N + hi (lo < hi node positions): the pattern of the block
// normal matrix, whatever the edges' multiplicity and order.
static std::vector<int64_t> free_pairs(int N, const int32_t * eidx, int E, const std::vector<uint8_t> & is_free)
{
  std::vector<int64_t> p;
  p.reserve(E);
  for (int e = 0; e < E; ++e) {
    const int a = eidx[2 * e], b = eidx[2 * e + 1];
    if (a != b && is_free[a] && is_free[b]) p.push_back((int64_t)std::min(a, b) * N + std::max(a, b));
  }
  std::sort(p.begin(), p.end());
  p.erase(std::unique(p.begin(), p.end()), p.end());
  return p;
}

// Ordering and symbolic factorisation of the free nodes' block matrix:
//   * minimum degree (Tinney-Walker / Rose) on the explicit elimination graph, ties to the lowest node position; the
//     structure of column v of L is v's neighbour set at its elimination, so the elimination gives the fill as well;
//   * the elimination tree, postordered (children in ascending order): an equivalent ordering with the same fill whose
//     subtrees are contiguous column ranges;
//   * fundamental supernodes (a column joins its only child when their structures nest), split at kCholMaxWidth, then
//     relaxed amalgamation of a supernode into its parent when they are adjacent in the postorder and the merged panel
//     is at most kCholMaxWidth wide and either at most 4 wide or at most 10% explicit zeros;
//   * panel layout, the supernodal tree and every supernode's updating descendants in ascending order.
// info = {block columns, nonzero blocks of L, supernodes, supernodal critical path, widest supernode (block columns),
// tallest panel (block rows), factor flops (sum over scalar columns of the squared column count), 0}.

static void cholesky_analyze(int N, const std::vector<uint8_t> & is_free, const std::vector<int64_t> & pairs, CholSymbolic & S)
{
  std::vector<int32_t> loc(N, -1), node;
  for (int i = 0; i < N; ++i)
    if (is_free[i]) { loc[i] = (int32_t)node.size(); node.push_back(i); }
  const int n = (int)node.size();
  std::vector<std::vector<int32_t>> adj(n), st(n);
  for (int64_t p : pairs) {
    const int a = loc[p / N], b = loc[p % N];
    adj[a].push_back(b); adj[b].push_back(a);
  }
  for (auto & a : adj) std::sort(a.begin(), a.end());
  // minimum degree
  std::set<std::pair<int32_t, int32_t>> q;
  for (int v = 0; v < n; ++v) q.insert({(int32_t)adj[v].size(), v});
  std::vector<int32_t> elim, merged;
  elim.reserve(n);
  while (!q.empty()) {
    const int v = q.begin()->second;
    q.erase(q.begin());
    elim.push_back(v);
    const std::vector<int32_t> & nv = adj[v];
    for (int u : nv) {
      q.erase({(int32_t)adj[u].size(), u});
      merged.clear();
      std::set_union(adj[u].begin(), adj[u].end(), nv.begin(), nv.end(), std::back_inserter(merged));
      merged.erase(std::remove_if(merged.begin(), merged.end(), [&](int x) { return x == u || x == v; }), merged.end());
      adj[u].swap(merged);
      q.insert({(int32_t)adj[u].size(), u});
    }
    st[v] = std::move(adj[v]);
  }
  // elimination tree in elimination positions, then its postorder
  std::vector<int32_t> pos(n), et(n, -1);
  for (int k = 0; k < n; ++k) pos[elim[k]] = k;
  for (int k = 0; k < n; ++k) {
    int m = n;
    for (int u : st[elim[k]]) m = std::min(m, pos[u]);
    if (m < n) et[k] = m;
  }
  std::vector<int32_t> head(n, -1), next(n, -1), post;
  for (int k = n - 1; k >= 0; --k)
    if (et[k] >= 0) { next[k] = head[et[k]]; head[et[k]] = k; }   // children lists in ascending order
  post.reserve(n);
  {
    std::vector<int32_t> stack;
    for (int r = 0; r < n; ++r) {
      if (et[r] >= 0) continue;
      stack.push_back(r);
      while (!stack.empty()) {
        const int k = stack.back();
        if (head[k] >= 0) { const int ch = head[k]; head[k] = next[ch]; stack.push_back(ch); }
        else { post.push_back(k); stack.pop_back(); }
      }
    }
  }
  // columns in postorder: their nodes, structures (below the diagonal), counts and parents
  std::vector<int32_t> colpos(n);   // elimination position -> column
  for (int c = 0; c < n; ++c) colpos[post[c]] = c;
  S.col_node.resize(n);
  S.node_col.assign(N, -1);
  std::vector<std::vector<int32_t>> cs(n);
  std::vector<int32_t> cnt(n), par(n, -1), nchild(n, 0);
  for (int c = 0; c < n; ++c) {
    const int v = elim[post[c]];
    S.col_node[c] = node[v];
    S.node_col[node[v]] = c;
    for (int u : st[v]) cs[c].push_back(colpos[pos[u]]);
    std::sort(cs[c].begin(), cs[c].end());
    cnt[c] = 1 + (int)cs[c].size();
    if (!cs[c].empty()) { par[c] = cs[c][0]; nchild[par[c]]++; }
  }
  // fundamental supernodes, split at the width cap
  std::vector<int32_t> fs;   // first column of each
  for (int c = 0; c < n; ++c) {
    const bool join = c > 0 && par[c - 1] == c && nchild[c] == 1 && cnt[c - 1] == cnt[c] + 1 && c - fs.back() < kCholMaxWidth;
    if (!join) fs.push_back(c);
  }
  const int nf = (int)fs.size();
  fs.push_back(n);
  // relaxed amalgamation: group g = [gfirst, last column of fundamental supernode f]; f merges into f + 1 when that is its
  // parent and starts right after it
  std::vector<int32_t> fsn(n);
  for (int f = 0; f < nf; ++f)
    for (int c = fs[f]; c < fs[f + 1]; ++c) fsn[c] = f;
  std::vector<int32_t> gfirst(nf);
  std::vector<int64_t> greal(nf);
  std::vector<char> absorbed(nf, 0);
  for (int f = 0; f < nf; ++f) {
    int64_t real = 0;
    for (int c = fs[f]; c < fs[f + 1]; ++c) real += cnt[c];
    if (f == 0 || !absorbed[f - 1]) { gfirst[f] = fs[f]; greal[f] = real; }
    else { greal[f] += real; }
    const int last = fs[f + 1] - 1;
    if (par[last] >= 0 && f + 1 < nf && par[last] == fs[f + 1]) {
      const int64_t wc = last - gfirst[f] + 1, wp = fs[f + 2] - fs[f + 1], rp = cnt[fs[f + 1]];
      const int64_t w = wc + wp, r = wc + rp, stored = w * r - w * (w - 1) / 2;
      int64_t realp = 0;
      for (int c = fs[f + 1]; c < fs[f + 2]; ++c) realp += cnt[c];
      const int64_t zeros = stored - (greal[f] + realp);
      if (w <= kCholMaxWidth && (w <= 4 || zeros * 10 <= stored)) {
        absorbed[f] = 1;
        gfirst[f + 1] = gfirst[f];
        greal[f + 1] = greal[f];
      }
    }
  }
  // supernodes: the groups that were not absorbed, in column order
  S.sn_col.clear();
  for (int f = 0; f < nf; ++f)
    if (!absorbed[f]) S.sn_col.push_back(gfirst[f]);
  const int ns = (int)S.sn_col.size();
  S.sn_col.push_back(n);
  S.sn_of_col.resize(n);
  for (int s = 0; s < ns; ++s)
    for (int c = S.sn_col[s]; c < S.sn_col[s + 1]; ++c) S.sn_of_col[c] = s;
  // rows: the columns, then the union of the columns' structures below the supernode
  S.row_start.assign(1, 0);
  S.rows.clear();
  S.off.assign(1, 0);
  S.parent.assign(ns, -1);
  std::vector<int32_t> below;
  int64_t max_w = 0, max_r = 0;
  for (int s = 0; s < ns; ++s) {
    const int c0 = S.sn_col[s], c1 = S.sn_col[s + 1];
    below.clear();
    for (int c = c0; c < c1; ++c)
      for (int r : cs[c])
        if (r >= c1) below.push_back(r);
    std::sort(below.begin(), below.end());
    below.erase(std::unique(below.begin(), below.end()), below.end());
    for (int c = c0; c < c1; ++c) S.rows.push_back(c);
    S.rows.insert(S.rows.end(), below.begin(), below.end());
    const int64_t nr = (int64_t)(c1 - c0) + (int64_t)below.size();
    S.row_start.push_back((int32_t)S.rows.size());
    S.off.push_back(S.off.back() + 9 * nr * (c1 - c0));
    if (par[c1 - 1] >= 0) S.parent[s] = S.sn_of_col[par[c1 - 1]];
    max_w = std::max<int64_t>(max_w, c1 - c0);
    max_r = std::max(max_r, nr);
  }
  // children and updating descendants, both ascending
  std::vector<std::vector<int32_t>> ch(ns), up(ns);
  for (int s = 0; s < ns; ++s) {
    if (S.parent[s] >= 0) ch[S.parent[s]].push_back(s);
    int lastJ = -1;
    for (int k = S.row_start[s] + (S.sn_col[s + 1] - S.sn_col[s]); k < S.row_start[s + 1]; ++k) {
      const int J = S.sn_of_col[S.rows[k]];
      if (J != lastJ) { up[J].push_back(s); lastJ = J; }
    }
  }
  auto csr = [](const std::vector<std::vector<int32_t>> & l, std::vector<int32_t> & start, std::vector<int32_t> & v) {
    start.assign(1, 0);
    v.clear();
    for (const auto & x : l) { v.insert(v.end(), x.begin(), x.end()); start.push_back((int32_t)v.size()); }
  };
  csr(ch, S.child_start, S.child);
  csr(up, S.upd_start, S.upd);
  // statistics
  std::vector<int32_t> depth(ns, 1);
  int64_t crit = 0, nnz = 0, flops = 0;
  for (int s = 0; s < ns; ++s) {
    for (int k = S.child_start[s]; k < S.child_start[s + 1]; ++k) depth[s] = std::max(depth[s], depth[S.child[k]] + 1);
    crit = std::max<int64_t>(crit, depth[s]);
  }
  for (int c = 0; c < n; ++c) {
    nnz += cnt[c];
    for (int k = 0; k < 3; ++k) flops += (int64_t)(3 * cnt[c] - k) * (3 * cnt[c] - k);
  }
  const int64_t info[8] = {n, nnz, ns, crit, max_w, max_r, flops, 0};
  std::copy(info, info + 8, S.info);
}

// The Cholesky plan of a solve: the analysis (kept while the free nodes and their adjacent pairs stay the same), its
// device copy, the assembly lists of the current edges and the cooperative grid. B200_ERR_UNSUPPORTED when the factor does
// not fit the device memory that is free.
static int plan_cholesky(b200pg * h, const std::vector<uint8_t> & is_free, cudaStream_t st, PcgPlan & P);

// Puts the problem on the device: the flattened edges (kept incrementally, see b200pg::f_eidx: only the edges appended
// since the last solve are copied), the free nodes, the CSR node->edge adjacency and the start point, and sizes the work
// buffers. Returns false, uploading nothing, when there is nothing to optimise (no edge or no free node).
static bool upload_problem(b200pg * h, std::vector<int32_t> & adj_start, int32_t & uploaded_edges)
{
  cudaStream_t st = h->stream;
  const int N = (int)h->node_ids.size(), E = (int)h->edges.size();
  if (h->flat_dirty || h->f_eidx.size() != 2 * (size_t)E) {
    h->f_eidx.resize(2 * (size_t)E); h->f_z.resize(3 * (size_t)E); h->f_U.resize(6 * (size_t)E);
    for (int e = 0; e < E; ++e) {
      const PgEdge & ed = h->edges[e];
      h->f_eidx[2 * e] = h->index.at(ed.ida); h->f_eidx[2 * e + 1] = h->index.at(ed.idb);
      for (int k = 0; k < 3; ++k) h->f_z[3 * e + k] = ed.z[k];
      for (int k = 0; k < 6; ++k) h->f_U[6 * e + k] = ed.U[k];
    }
    h->flat_dirty = false;
    h->dev_edges = 0;
  }
  const std::vector<int32_t> & eidx = h->f_eidx;
  std::vector<uint8_t> is_free(N, 0);
  std::vector<int32_t> deg(N + 1, 0);
  for (int e = 0; e < E; ++e) {
    const int a = eidx[2 * e], b = eidx[2 * e + 1];
    is_free[a] = 1; is_free[b] = 1;   // only nodes that appear in a residual block are Ceres parameter blocks
    deg[a + 1]++; deg[b + 1]++;
  }
  // first node constant, if it is part of the problem (ceres_solver.cpp:228-241)
  if (h->have_first) {
    auto it = h->index.find(h->first_node_id);
    if (it != h->index.end()) is_free[it->second] = 0;
  }
  int nfree = 0;
  for (int i = 0; i < N; ++i) nfree += is_free[i];
  if (E == 0 || nfree == 0) return false;
  adj_start.assign(N + 1, 0);
  std::vector<int32_t> adj(2 * (size_t)E);
  for (int i = 0; i < N; ++i) adj_start[i + 1] = adj_start[i] + deg[i + 1];
  {
    std::vector<int32_t> fill(adj_start.begin(), adj_start.end() - 1);
    for (int e = 0; e < E; ++e) {
      adj[fill[eidx[2 * e]]++] = (e << 1) | 0;
      adj[fill[eidx[2 * e + 1]]++] = (e << 1) | 1;
    }
  }
  {
    // edges: only the ones appended since the last solve travel (the buffers grow with their contents kept)
    if (h->dev_edges > (size_t)E) h->dev_edges = 0;
    const size_t e0 = h->dev_edges, ne = (size_t)E - e0;
    grow_keep(h->d_eidx, 2 * (size_t)E, 2 * e0, st); grow_keep(h->d_z, 3 * (size_t)E, 3 * e0, st); grow_keep(h->d_U, 6 * (size_t)E, 6 * e0, st);
    if (ne) {
      B200_CUDA(cudaMemcpyAsync(h->d_eidx.p + 2 * e0, h->f_eidx.data() + 2 * e0, 2 * ne * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      B200_CUDA(cudaMemcpyAsync(h->d_z.p + 3 * e0, h->f_z.data() + 3 * e0, 3 * ne * sizeof(double), cudaMemcpyHostToDevice, st));
      B200_CUDA(cudaMemcpyAsync(h->d_U.p + 6 * e0, h->f_U.data() + 6 * e0, 6 * ne * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    uploaded_edges = (int32_t)ne;
    h->dev_edges = (size_t)E;
  }
  up(h->d_free, is_free, st);
  h->free_h = is_free;
  up(h->d_adj_start, adj_start, st); up(h->d_adj, adj, st); up(h->d_x, h->node_pose, st);
  const size_t n3 = 3 * (size_t)N;
  h->d_xc.reserve(n3); h->d_scale.reserve(n3); h->d_lin.reserve((size_t)kLin * E); h->d_Hd.reserve(6 * (size_t)N);
  h->d_g.reserve(n3); h->d_diag.reserve(n3); h->d_y.reserve(n3); h->d_pr.reserve(n3); h->d_pz.reserve(n3);
  h->d_pp0.reserve(n3); h->d_pp1.reserve(n3); h->d_pq.reserve(n3); h->d_Minv.reserve(6 * (size_t)N);
  h->d_partial.reserve((size_t)kMaxPartials * 8); h->d_scalars.reserve(32); h->h_scalars.reserve(32);
  return true;
}

static int plan_cholesky(b200pg * h, const std::vector<uint8_t> & is_free, cudaStream_t st, PcgPlan & P)
{
  const int N = (int)h->node_ids.size(), E = (int)h->edges.size();
  const int32_t * eidx = h->f_eidx.data();
  std::vector<int64_t> pairs = free_pairs(N, eidx, E, is_free);
  CholSymbolic & S = h->chol;
  const bool fresh = h->chol_stale || !h->chol_valid || is_free != h->chol_free || pairs != h->chol_pairs;
  if (fresh) {
    h->chol_valid = false;
    cholesky_analyze(N, is_free, pairs, S);
    h->chol_analyses++;
    h->chol_free = is_free;
    h->chol_pairs.swap(pairs);
    h->chol_stale = false;
  }
  const int ns = (int)S.sn_col.size() - 1, n = (int)S.col_node.size();
  const size_t l_doubles = (size_t)S.off[ns];
  if (l_doubles > h->d_ch_L.cap) {
    size_t free_b = 0, total_b = 0;
    B200_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t want = (l_doubles + l_doubles / 4 + 16) * sizeof(double);   // DevBuf::reserve, after the old buffer is freed
    if (want > free_b + h->d_ch_L.cap * sizeof(double)) {
      set_last_error("b200pg_solve: the Cholesky factor needs " + std::to_string(l_doubles * sizeof(double) >> 20) +
                     " MB of device memory, more than is free (" + std::to_string(free_b >> 20) + " MB); linear_solver_type = 0 solves it by PCG");
      return B200_ERR_UNSUPPORTED;
    }
  }
  if (fresh) {
    up(h->d_ch_sn_col, S.sn_col, st); up(h->d_ch_row_start, S.row_start, st); up(h->d_ch_rows, S.rows, st);
    up(h->d_ch_upd_start, S.upd_start, st); up(h->d_ch_upd, S.upd, st); up(h->d_ch_child_start, S.child_start, st);
    up(h->d_ch_child, S.child, st); up(h->d_ch_parent, S.parent, st); up(h->d_ch_col_node, S.col_node, st);
    up(h->d_ch_off, S.off, st);
    h->d_ch_L.reserve(l_doubles); h->d_ch_z.reserve(3 * (size_t)n);
    h->d_ch_flag.reserve(2 * (size_t)ns); h->d_ch_ctl.reserve(4);
    B200_CUDA(cudaMemsetAsync(h->d_ch_flag.p, 0, h->d_ch_flag.cap * sizeof(unsigned int), st));
    B200_CUDA(cudaMemsetAsync(h->d_ch_ctl.p, 0, h->d_ch_ctl.cap * sizeof(unsigned int), st));
    h->chol_valid = true;
    h->chol_asm_edges = -1;
  }
  // the assembly lists depend on the analysis and the edges; edges are only appended while the analysis is kept (a removal
  // or Reset forces a new analysis), so an unchanged edge count means unchanged lists
  if (h->chol_asm_edges != E) {
    // assembly lists of the current edges: every receiving block of L (supernode, column within it, row position) with its
    // contributors, the diagonal block first, the edges in edge order
    struct Contrib { int32_t sn, q, p, src; };
    std::vector<Contrib> cb;
    cb.reserve((size_t)n + E);
    for (int k = 0; k < n; ++k) {
      const int J = S.sn_of_col[k];
      cb.push_back({J, k - S.sn_col[J], k - S.sn_col[J], -1 - S.col_node[k]});
    }
    for (int e = 0; e < E; ++e) {
      const int a = eidx[2 * e], b = eidx[2 * e + 1];
      if (!is_free[a] || !is_free[b]) continue;
      const int ca = S.node_col[a], cb_ = S.node_col[b];
      const int row = std::max(ca, cb_), col = std::min(ca, cb_);   // A[a][b] = M_e: transposed when the row is b
      const int J = S.sn_of_col[col];
      const int32_t * R = S.rows.data() + S.row_start[J];
      const int p = (int)(std::lower_bound(R, R + (S.row_start[J + 1] - S.row_start[J]), row) - R);
      cb.push_back({J, col - S.sn_col[J], p, (e << 1) | (row == cb_ ? 1 : 0)});
    }
    std::stable_sort(cb.begin(), cb.end(), [](const Contrib & x, const Contrib & y) {
      return x.sn != y.sn ? x.sn < y.sn : (x.q != y.q ? x.q < y.q : x.p < y.p);
    });
    std::vector<int32_t> tgt_start(ns + 1, 0), src_start(1, 0), src;
    std::vector<int64_t> tgt_off;
    src.reserve(cb.size());
    for (size_t i = 0; i < cb.size(); ++i) {
      const Contrib & x = cb[i];
      if (i == 0 || x.sn != cb[i - 1].sn || x.q != cb[i - 1].q || x.p != cb[i - 1].p) {
        if (i > 0) src_start.push_back((int32_t)src.size());
        const int64_t ld = 3 * (int64_t)(S.row_start[x.sn + 1] - S.row_start[x.sn]);
        tgt_off.push_back(S.off[x.sn] + 3 * (int64_t)x.q * ld + 3 * (int64_t)x.p);
        tgt_start[x.sn + 1]++;
      }
      src.push_back(x.src);
    }
    src_start.push_back((int32_t)src.size());
    for (int s = 0; s < ns; ++s) tgt_start[s + 1] += tgt_start[s];
    up(h->d_ch_tgt_start, tgt_start, st); up(h->d_ch_tgt_off, tgt_off, st); up(h->d_ch_src_start, src_start, st);
    up(h->d_ch_src, src, st);
    h->chol_asm_edges = E;
  }
  std::copy(S.info, S.info + 8, h->chol_info);

  int dev = 0, sms = 132, per_sm = 1;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pg_cholesky, kCholThreads, 0));
  P = PcgPlan{};
  P.kernel = kLinearSolverCholesky;
  P.blocks = std::max(1, std::min({kMaxPartials, sms * std::max(per_sm, 1), ns}));
  return B200_OK;
}

// What a solve launches with: the device view of the problem, the grids of the per-node and per-edge kernels, the PCG plan
// and the stream; counts the launches.
struct Launcher {
  b200pg * h;
  PgDev d;
  int blocksN, blocksE;
  PcgPlan plan;
  cudaStream_t st;

  void fetch(int n = 16)
  {
    B200_CUDA(cudaMemcpyAsync(h->h_scalars.p, h->d_scalars.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  // one linear solve of (H + shift * diag) y = g on the planned kernel; scalars[8] = iterations, [9] = relative residual.
  // tol and max_iter bound the PCG kernels; the Cholesky kernel solves exactly and ignores them.
  void linear_solve(double shift, double tol, int max_iter)
  {
    if (plan.kernel == kLinearSolverCholesky) {
      if (++h->chol_epoch == 0) {   // the epochs wrapped: restart them from clean flags
        B200_CUDA(cudaMemsetAsync(h->d_ch_flag.p, 0, h->d_ch_flag.cap * sizeof(unsigned int), st));
        B200_CUDA(cudaMemsetAsync(h->d_ch_ctl.p + 2, 0, sizeof(unsigned int), st));
        h->chol_epoch = 1;
      }
      B200_CUDA(cudaMemsetAsync(h->d_ch_ctl.p, 0, 2 * sizeof(unsigned int), st));
      CholDev c;
      c.ns = (int)h->chol.sn_col.size() - 1;
      c.sn_col = h->d_ch_sn_col.p; c.row_start = h->d_ch_row_start.p; c.rows = h->d_ch_rows.p; c.off = h->d_ch_off.p;
      c.upd_start = h->d_ch_upd_start.p; c.upd = h->d_ch_upd.p; c.child_start = h->d_ch_child_start.p; c.child = h->d_ch_child.p;
      c.parent = h->d_ch_parent.p; c.tgt_start = h->d_ch_tgt_start.p; c.tgt_off = h->d_ch_tgt_off.p;
      c.src_start = h->d_ch_src_start.p; c.src = h->d_ch_src.p; c.col_node = h->d_ch_col_node.p;
      c.L = h->d_ch_L.p; c.z = h->d_ch_z.p; c.flag = h->d_ch_flag.p; c.ctl = h->d_ch_ctl.p; c.epoch = h->chol_epoch;
      void * args[] = {&d, &c, &shift};
      B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_cholesky, dim3(plan.blocks), dim3(kCholThreads), args, 0, st));
    } else if (plan.kernel == 13 || plan.kernel == 16) {
      B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, sizeof(unsigned int), st));
      void * args[] = {&d, &plan.two_level_g, &shift, &tol, &max_iter};
      B200_CUDA(cudaLaunchCooperativeKernel(plan.kernel == 16 ? (void *)k_pg_pcg_2lvl_g<6> : (void *)k_pg_pcg_2lvl_g<3>, dim3(plan.blocks), dim3(kG2Threads), args, plan.smem_bytes, st));
    } else if (plan.kernel >= 3) {
      B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, (size_t)(plan.blocks + 1) * sizeof(unsigned int), st));
      void * args[] = {&d, &plan.two_level, &shift, &tol, &max_iter};
      B200_CUDA(cudaLaunchCooperativeKernel(plan.kernel == 6 ? (void *)k_pg_pcg_2lvl<6> : (void *)k_pg_pcg_2lvl<3>, dim3(plan.blocks), dim3(256), args, plan.smem_bytes, st));
    } else if (plan.kernel == 1) {
      B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, sizeof(unsigned int), st));
      void * args[] = {&d, &plan.smem, &shift, &tol, &max_iter};
      B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_pcg_smem, dim3(plan.blocks), dim3(512), args, plan.smem_bytes, st));
    } else {
      void * args[] = {&d, &shift, &tol, &max_iter};
      B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_pcg, dim3(plan.blocks), dim3(kPgThreads), args, 0, st));
    }
    h->launches++;
  }
  void launched() { B200_CUDA(cudaGetLastError()); h->launches++; }

  // cost at x (mode 0, also linearises) or at xc (mode 1) -> scalars[slot]
  void linearize(int mode, int slot)
  {
    k_pg_linearize<<<blocksE, kPgThreads, 0, st>>>(d, mode); launched();
    k_pg_reduce<<<1, 32, 0, st>>>(d, blocksE, slot, -1); launched();
  }
  // Hd, g, gradient max norm (scalars[2]) and ||x||^2 (scalars[3])
  void assemble()
  {
    k_pg_assemble<<<blocksN, kPgThreads, 0, st>>>(d, 0); launched();
    k_pg_reduce<<<1, 32, 0, st>>>(d, blocksN, 3, 2); launched();
  }
};

// The two trust-region strategies. Each computes a step into d.y (the step is -y) and reacts to the outcome of the step:
// accepted (with its quality), rejected, or invalid. compute_step returns false when the linear solve failed, which the
// minimiser treats as an invalid step.

// LevenbergMarquardtStrategy: (H + D^2 / radius) y = g, D^2 the clamped squared column norms, reused after a rejected step
struct LmStrategy {
  static constexpr const char * kIterationRange = "b200pg LM iteration";
  Launcher & L;
  const b200pg_opts & o;
  double radius, decrease_factor = 2.0;
  bool reuse_diagonal = false;

  bool compute_step(b200pg_summary & S)
  {
    if (!reuse_diagonal) { k_pg_diag<<<L.blocksN, kPgThreads, 0, L.st>>>(L.d, o.min_lm_diagonal, o.max_lm_diagonal); L.launched(); }
    L.linear_solve(1.0 / radius, o.pcg_tolerance, o.pcg_max_iterations);
    S.linear_solves++;
    reuse_diagonal = true;
    return true;
  }
  // the step's scalars have been fetched: its PCG iterations, and the two-level kernel's timers under B200PG_DEBUG
  void fetched(const double * sc, int it, b200pg_summary & S)
  {
    S.pcg_iterations += (int)sc[8];
    if (L.h->debug && L.plan.kernel == kLinearSolverCholesky)
      fprintf(stderr, "[b200pg] lm %d: cholesky factor+forward %.1f us, backward %.1f us, residual %.1f us\n", it, sc[10] * 1e-3,
              sc[11] * 1e-3, sc[12] * 1e-3);
    if (L.h->debug && (L.plan.kernel == 13 || L.plan.kernel == 16))
      fprintf(stderr, "[b200pg] lm %d: pcg %d it, setup %.1f us, gauss-jordan %.1f us, cg %.1f us (%.2f us/it)\n", it, (int)sc[8],
              sc[10] * 1e-3, sc[11] * 1e-3, sc[12] * 1e-3, sc[12] * 1e-3 / std::max(1.0, sc[8]));
    if (L.h->debug && (L.plan.kernel == 3 || L.plan.kernel == 6))
      fprintf(stderr, "[b200pg] lm %d: pcg %d it, setup %.1f us, gauss-jordan %.1f us, cg %.1f us (%.2f us/it: gather %.2f spmv+reduce %.2f exch1 %.2f precond %.2f exch2 %.2f)\n", it, (int)sc[8],
              sc[10] * 1e-3, sc[11] * 1e-3, sc[12] * 1e-3, sc[12] * 1e-3 / std::max(1.0, sc[8]), sc[13] * 1e-3 / std::max(1.0, sc[8]),
              sc[14] * 1e-3 / std::max(1.0, sc[8]), sc[15] * 1e-3 / std::max(1.0, sc[8]), sc[6] * 1e-3 / std::max(1.0, sc[8]), sc[7] * 1e-3 / std::max(1.0, sc[8]));
  }
  void accepted(double quality)
  {
    radius = std::min(o.max_trust_region_radius, radius / std::max(1.0 / 3.0, 1.0 - pow(2.0 * quality - 1.0, 3)));
    decrease_factor = 2.0; reuse_diagonal = false;
  }
  void rejected() { radius /= decrease_factor; decrease_factor *= 2.0; reuse_diagonal = true; }
  void invalid() { radius /= decrease_factor; decrease_factor *= 2.0; }
};

// DoglegStrategy (DESIGN.md §4): the Gauss-Newton step of (H + mu D^2) y = g and its DoglegModel, reused after a rejected step
struct DoglegStrategy {
  static constexpr const char * kIterationRange = "b200pg dogleg iteration";
  Launcher & L;
  const b200pg_opts & o;
  double radius, mu = kDlMinMu, step_norm = 0.0;
  bool reuse = false;
  DoglegModel model{};

  bool compute_step(b200pg_summary & S)
  {
    b200pg * h = L.h;
    const bool subspace = o.dogleg_type == 1;
    const double gn_tol = kDlPcgTolFactor * o.pcg_tolerance;   // the Gauss-Newton solve's PCG tolerance
    if (!reuse) {
      h->d_ygn.reserve(3 * (size_t)L.d.N);
      k_pg_diag<<<L.blocksN, kPgThreads, 0, L.st>>>(L.d, o.min_lm_diagonal, o.max_lm_diagonal); L.launched();
      bool solved = false;
      while (mu < kDlMaxMu) {   // Gauss-Newton step: (H + mu D^2) y = g, mu grows while the solve fails
        L.linear_solve(mu, gn_tol, o.pcg_max_iterations);
        S.linear_solves++;
        B200_CUDA(cudaMemcpyAsync(h->d_ygn.p, L.d.y, 3 * (size_t)L.d.N * sizeof(double), cudaMemcpyDeviceToDevice, L.st));
        k_pg_dogleg_nodes<<<L.blocksN, kPgThreads, 0, L.st>>>(L.d, h->d_ygn.p); L.launched();
        k_pg_reduce_n<<<1, 32, 0, L.st>>>(L.d, L.blocksN, 3, 16); L.launched();
        k_pg_dogleg_edges<<<L.blocksE, kPgThreads, 0, L.st>>>(L.d, h->d_ygn.p); L.launched();
        k_pg_reduce_n<<<1, 32, 0, L.st>>>(L.d, L.blocksE, 3, 19); L.launched();
        L.fetch(22);
        const double * sc = h->h_scalars.p;
        S.pcg_iterations += (int)sc[8];
        solved = sc[9] <= gn_tol;
        for (int k = 16; k < 22; ++k) solved = solved && std::isfinite(sc[k]);
        if (solved) { model.set(sc + 16); break; }
        mu *= kDlMuIncrease;
      }
      if (!solved) return false;   // linear solver failure: DoglegStrategy::StepIsInvalid
      if (subspace) model.subspace();
      reuse = true;
    }
    double ca, cb;
    if (subspace) subspace_step(model, radius, ca, cb, step_norm);
    else traditional_step(model, radius, ca, cb, step_norm);
    k_pg_dogleg_compose<<<L.blocksN, kPgThreads, 0, L.st>>>(L.d, h->d_ygn.p, -ca, cb); L.launched();
    return true;
  }
  void fetched(const double *, int, b200pg_summary &) {}   // the PCG iterations were counted per solve
  void accepted(double quality)   // StepAccepted (no clamp to max_trust_region_radius, DESIGN.md §4)
  {
    if (quality < 0.25) radius *= 0.5;
    if (quality > 0.75) radius = std::max(radius, 3.0 * step_norm);
    mu = std::max(kDlMinMu, mu / 5.0);
    reuse = false;
  }
  void rejected() { radius *= 0.5; reuse = true; }          // StepRejected: shrink the region, keep the Gauss-Newton step
  void invalid() { mu *= kDlMuIncrease; reuse = false; }   // StepIsInvalid: radius unchanged
};

// Ceres' TrustRegionMinimizer with the non-monotonic TrustRegionStepEvaluator, driven from the host with one small D2H of
// scalars per step. The solution is the minimum-cost iterate; it is left in h->node_pose when usable.
template <class Strategy>
static void minimize(Launcher & L, Strategy & strategy, b200pg_summary & S)
{
  b200pg * h = L.h;
  const b200pg_opts & o = h->o;
  PgDev & d = L.d;
  cudaStream_t st = L.st;
  const size_t n3 = 3 * (size_t)d.N;
  // ---- iteration 0: evaluate, Jacobi scaling from the unscaled Jacobian ----
  k_pg_fill<<<64, 256, 0, st>>>(d.scale, 1.0, 3 * d.N); L.launched();
  if (o.jacobi_scaling) {
    L.linearize(0, 0);
    k_pg_assemble<<<L.blocksN, kPgThreads, 0, st>>>(d, 1); L.launched();
  }
  L.linearize(0, 0);   // scalars[0] = cost(x)
  L.assemble();        // scalars[2] = gradient max norm, scalars[3] = ||x||^2
  L.fetch();
  double cost = h->h_scalars.p[0], gmax = h->h_scalars.p[2], x_norm = sqrt(h->h_scalars.p[3]);
  S.initial_cost = cost;
  double minimum_cost = cost;
  std::vector<double> best_x;   // empty = the start point
  bool have_best_on_device_x = true;

  const int max_nonmono = o.use_nonmonotonic_steps ? o.max_consecutive_nonmonotonic_steps : 0;
  double ev_min = cost, ev_cur = cost, ev_ref = cost, ev_cand = cost, acc_ref = 0.0, acc_cand = 0.0;
  int n_nonmono = 0, invalid_steps = 0, it = 0;
  bool step_successful = false;
  // HandleInvalidStep: true when there were too many in a row
  auto invalid_step = [&]() {
    if (++invalid_steps >= o.max_num_consecutive_invalid_steps) { S.termination = 5; S.usable = 0; return true; }
    strategy.invalid();
    return false;
  };
  S.termination = 3;
  // TrustRegionMinimizer::IterationZero: an already-converged start returns CONVERGENCE before any step is computed
  const bool converged_at_start = gmax <= o.gradient_tolerance;
  if (converged_at_start) S.termination = 1;
  while (!converged_at_start) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue
    if (it >= o.max_num_iterations) { S.termination = 3; break; }
    if (step_successful && gmax <= o.gradient_tolerance) { S.termination = 1; break; }
    if (strategy.radius <= o.min_trust_region_radius) { S.termination = 4; break; }
    ++it;
    NvtxRange nvtx_it(Strategy::kIterationRange);
    step_successful = false;
    if (!strategy.compute_step(S)) {
      if (invalid_step()) break;
      continue;
    }
    k_pg_model_change<<<L.blocksE, kPgThreads, 0, st>>>(d); L.launched();
    k_pg_reduce<<<1, 32, 0, st>>>(d, L.blocksE, 4, -1); L.launched();
    k_pg_apply_step<<<L.blocksN, kPgThreads, 0, st>>>(d); L.launched();
    k_pg_reduce<<<1, 32, 0, st>>>(d, L.blocksN, 5, -1); L.launched();
    L.linearize(1, 1);   // scalars[1] = cost(xc)
    L.fetch();
    const double * sc = h->h_scalars.p;
    strategy.fetched(sc, it, S);
    const double model_cost_change = sc[4], step_norm = sqrt(sc[5]), cand_cost = sc[1];
    const bool finite = std::isfinite(model_cost_change) && std::isfinite(cand_cost) && std::isfinite(sc[9]);
    if (!finite || !(model_cost_change > 0.0)) {
      if (invalid_step()) break;
      continue;
    }
    invalid_steps = 0;
    if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) { S.termination = 2; break; }
    const double cost_change = cost - cand_cost;
    if (fabs(cost_change) <= o.function_tolerance * cost) { S.termination = 0; break; }
    const double rel = (ev_cur - cand_cost) / model_cost_change;
    const double hist = (ev_ref - cand_cost) / (acc_ref + model_cost_change);
    const double quality = std::max(rel, hist);
    if (!(quality > o.min_relative_decrease)) {
      strategy.rejected();
      continue;
    }
    // HandleSuccessfulStep
    std::swap(d.x, d.xc);
    cost = cand_cost;
    L.linearize(0, 0);
    L.assemble();
    L.fetch();
    gmax = h->h_scalars.p[2]; x_norm = sqrt(h->h_scalars.p[3]);
    step_successful = true;
    S.successful_steps++;
    strategy.accepted(quality);
    ev_cur = cost; acc_cand += model_cost_change; acc_ref += model_cost_change;
    if (ev_cur < ev_min) { ev_min = ev_cur; n_nonmono = 0; ev_cand = ev_cur; acc_cand = 0.0; }
    else { ++n_nonmono; if (ev_cur > ev_cand) { ev_cand = ev_cur; acc_cand = 0.0; } }
    if (n_nonmono == max_nonmono) { ev_ref = ev_cand; acc_ref = acc_cand; }
    if (cost < minimum_cost) {   // the solution Ceres returns is the minimum-cost iterate
      minimum_cost = cost;
      have_best_on_device_x = true;
    } else if (have_best_on_device_x) {
      // x moved away from the best iterate (non-monotonic step): keep a host copy of the best one,
      // which is the previous x, now in d.xc
      best_x.resize(n3);
      B200_CUDA(cudaMemcpyAsync(best_x.data(), d.xc, n3 * sizeof(double), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      have_best_on_device_x = false;
    }
  }
  B200_CUDA(cudaEventRecord(h->ev1, st));
  S.iterations = it;
  S.final_cost = minimum_cost;
  if (S.usable) {
    if (have_best_on_device_x) {
      B200_CUDA(cudaMemcpyAsync(h->node_pose.data(), d.x, n3 * sizeof(double), cudaMemcpyDeviceToHost, st));
    } else {
      std::memcpy(h->node_pose.data(), best_x.data(), n3 * sizeof(double));
    }
  }
}

static int solve(b200pg * h, b200pg_summary * sum)
{
  const auto t_enter = std::chrono::steady_clock::now();
  NvtxRange nvtx_solve("b200pg solve");
  b200pg_summary S{};
  S.usable = 1;
  S.linear_solver = -1;
  const int N = (int)h->node_ids.size();
  if (N == 0) {   // "Ceres was called when there are no nodes" (ceres_solver.cpp:219-225)
    set_last_error("b200pg_solve: no nodes");
    if (sum) *sum = S;
    return B200_ERR_INVALID_ARG;
  }
  require_device();
  if (!h->stream) { B200_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
  cudaStream_t st = h->stream;
  if (!h->ev0) { B200_CUDA(cudaEventCreate(&h->ev0)); B200_CUDA(cudaEventCreate(&h->ev1)); }
  const int64_t launches0 = h->launches;
  auto store_corrections = [&]() {
    h->corr_ids = h->node_ids;
    h->corr_pose = h->node_pose;
  };
  std::vector<int32_t> adj_start;
  if (!upload_problem(h, adj_start, S.uploaded_edges)) {   // nothing to optimise: Ceres returns CONVERGENCE immediately
    store_corrections();
    S.termination = 0;
    if (sum) *sum = S;
    return B200_OK;
  }
  const int E = (int)h->edges.size();
  Launcher L;
  L.h = h; L.st = st;
  PgDev & d = L.d;
  d.N = N; d.E = E; d.eidx = h->d_eidx.p; d.z = h->d_z.p; d.U = h->d_U.p; d.is_free = h->d_free.p;
  d.adj_start = h->d_adj_start.p; d.adj = h->d_adj.p; d.x = h->d_x.p; d.xc = h->d_xc.p; d.scale = h->d_scale.p;
  d.lin = h->d_lin.p; d.Hd = h->d_Hd.p; d.g = h->d_g.p; d.diag = h->d_diag.p; d.y = h->d_y.p; d.pr = h->d_pr.p;
  d.pz = h->d_pz.p; d.pp0 = h->d_pp0.p; d.pp1 = h->d_pp1.p; d.pq = h->d_pq.p; d.Minv = h->d_Minv.p;
  d.partial = h->d_partial.p; d.scalars = h->d_scalars.p;
  d.loss = h->o.loss_function; d.loss_a = h->o.loss_scale;
  L.blocksN = std::min(kMaxPartials, std::max(1, (N + kPgThreads - 1) / kPgThreads));
  L.blocksE = std::min(kMaxPartials, std::max(1, (E + kPgThreads - 1) / kPgThreads));
  if (h->o.linear_solver_type == 1) {
    const int rc = plan_cholesky(h, h->free_h, st, L.plan);
    if (rc != B200_OK) {
      if (sum) *sum = S;
      return rc;
    }
  } else {
    L.plan = plan_pcg(h, adj_start, st);
  }
  S.linear_solver = L.plan.kernel;
  S.setup_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_enter).count();
  B200_CUDA(cudaEventRecord(h->ev0, st));
  if (h->o.trust_region_strategy == 1) {
    DoglegStrategy strategy{L, h->o, h->o.initial_trust_region_radius};
    minimize(L, strategy, S);
  } else {
    LmStrategy strategy{L, h->o, h->o.initial_trust_region_radius};
    minimize(L, strategy, S);
  }
  B200_CUDA(cudaStreamSynchronize(st));
  B200_CUDA(cudaEventElapsedTime(&S.solve_ms, h->ev0, h->ev1));
  S.kernel_launches = h->launches - launches0;
  S.wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_enter).count();
  if (sum) *sum = S;
  if (!S.usable) {
    set_last_error("pose-graph solve produced no usable solution (too many invalid steps)");
    return B200_ERR_NUMERIC;
  }
  store_corrections();
  return B200_OK;
}

}  // namespace b200

#define B200_GUARD_BEGIN try {
#define B200_GUARD_END                                                     \
  }                                                                        \
  catch (const b200::CudaFail & f) { return f.code; }                      \
  catch (const std::bad_alloc &) { b200::set_last_error("out of host memory"); return B200_ERR_CUDA; } \
  catch (const std::exception & e) { b200::set_last_error(e.what()); return B200_ERR_CUDA; }

extern "C" {

void b200pg_default_opts(b200pg_opts * o) { if (o) b200pg_defaults(o); }

int b200pg_create(const b200pg_opts * opts, b200pg ** out)
{
  B200_GUARD_BEGIN
  if (!out) return B200_ERR_INVALID_ARG;
  *out = nullptr;
  std::unique_ptr<b200pg> h(new b200pg());
  if (opts) h->o = *opts; else b200pg_defaults(&h->o);
  if (h->o.max_num_iterations < 0 || !(h->o.pcg_tolerance > 0) || h->o.pcg_max_iterations <= 0 ||
      !(h->o.initial_trust_region_radius > 0) || h->o.loss_function < 0 || h->o.loss_function > 2 ||
      (h->o.loss_function != 0 && !(h->o.loss_scale > 0)) || h->o.trust_region_strategy < 0 || h->o.trust_region_strategy > 1 ||
      h->o.dogleg_type < 0 || h->o.dogleg_type > 1 || h->o.linear_solver_type < 0 || h->o.linear_solver_type > 1) {
    set_last_error("b200pg_create: invalid options");
    return B200_ERR_INVALID_ARG;
  }
  require_device();
  if (const char * e = getenv("B200PG_FORCE_GLOBAL_PCG")) h->force_global_pcg = atoi(e) != 0;
  if (const char * e = getenv("B200PG_FORCE_2LVL_GLOBAL")) h->force_2lvl_global = atoi(e) != 0;
  if (const char * e = getenv("B200PG_DEBUG")) h->debug = atoi(e) != 0;
  if (const char * e = getenv("B200PG_PRECOND")) h->precond = std::string(e) == "jacobi" ? 0 : 1;
  if (const char * e = getenv("B200PG_COARSE_MODES")) h->coarse_modes = atoi(e) >= 6 ? 6 : 3;
  *out = h.release();
  return B200_OK;
  B200_GUARD_END
}

void b200pg_destroy(b200pg * h)
{
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

static bool valid_opts(const b200pg_opts & o)
{
  return !(o.max_num_iterations < 0 || !(o.pcg_tolerance > 0) || o.pcg_max_iterations <= 0 || !(o.initial_trust_region_radius > 0) ||
           o.loss_function < 0 || o.loss_function > 2 || (o.loss_function != 0 && !(o.loss_scale > 0)) ||
           o.trust_region_strategy < 0 || o.trust_region_strategy > 1 || o.dogleg_type < 0 || o.dogleg_type > 1 ||
           o.linear_solver_type < 0 || o.linear_solver_type > 1);
}

int b200pg_set_opts(b200pg * h, const b200pg_opts * opts)
{
  if (!h || !opts) return B200_ERR_INVALID_ARG;
  if (!valid_opts(*opts)) { set_last_error("b200pg_set_opts: invalid options"); return B200_ERR_INVALID_ARG; }
  h->o = *opts;
  return B200_OK;
}

int b200pg_get_opts(const b200pg * h, b200pg_opts * opts)
{
  if (!h || !opts) return B200_ERR_INVALID_ARG;
  *opts = h->o;
  return B200_OK;
}

int b200pg_set_stream(b200pg * h, void * s)
{
  if (!h) return B200_ERR_INVALID_ARG;
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  h->stream = static_cast<cudaStream_t>(s);
  h->own_stream = false;
  return B200_OK;
}

int b200pg_reset(b200pg * h)
{
  if (!h) return B200_ERR_INVALID_ARG;
  h->node_ids.clear(); h->node_pose.clear(); h->index.clear(); h->edges.clear();
  h->corr_ids.clear(); h->corr_pose.clear();
  h->have_first = false;
  h->f_eidx.clear(); h->f_z.clear(); h->f_U.clear(); h->flat_dirty = false; h->dev_edges = 0;
  h->chol_stale = true;
  return B200_OK;
}

int b200pg_clear(b200pg * h)
{
  if (!h) return B200_ERR_INVALID_ARG;
  h->corr_ids.clear(); h->corr_pose.clear();
  return B200_OK;
}

int b200pg_add_node(b200pg * h, int32_t id, const double pose[3])
{
  if (!h || !pose) return B200_ERR_INVALID_ARG;
  if (h->index.count(id)) return B200_OK;   // unordered_map::insert keeps the existing entry (ceres_solver.cpp:331)
  h->index[id] = (int32_t)h->node_ids.size();
  h->node_ids.push_back(id);
  h->node_pose.insert(h->node_pose.end(), pose, pose + 3);
  if (h->node_ids.size() == 1) { h->first_node_id = id; h->have_first = true; }   // :333-335
  return B200_OK;
}

int b200pg_add_edge(b200pg * h, int32_t ida, int32_t idb, const double z[3], const double cov[9])
{
  if (!h || !z || !cov) return B200_ERR_INVALID_ARG;
  if (!h->index.count(ida) || !h->index.count(idb) || ida == idb) {
    set_last_error("b200pg_add_edge: could not find nodes (CeresSolver warns and ignores, ceres_solver.cpp:351-358)");
    return B200_ERR_NOT_FOUND;
  }
  PgEdge e;
  e.ida = ida; e.idb = idb;
  e.z[0] = z[0]; e.z[1] = z[1]; e.z[2] = z[2];
  if (!sqrt_information(cov, e.U)) {
    set_last_error("b200pg_add_edge: covariance is singular or its inverse is not positive definite");
    return B200_ERR_NUMERIC;
  }
  h->edges.push_back(e);
  if (!h->flat_dirty) {
    h->f_eidx.push_back(h->index[ida]); h->f_eidx.push_back(h->index[idb]);
    h->f_z.insert(h->f_z.end(), e.z, e.z + 3);
    h->f_U.insert(h->f_U.end(), e.U, e.U + 6);
  }
  return B200_OK;
}

int b200pg_remove_node(b200pg * h, int32_t id)
{
  if (!h) return B200_ERR_INVALID_ARG;
  auto it = h->index.find(id);
  if (it == h->index.end()) { set_last_error("RemoveNode: failed to find node"); return B200_ERR_NOT_FOUND; }
  // RemoveParameterBlock also removes every residual block that uses it (ceres_solver.cpp:405-407)
  h->edges.erase(std::remove_if(h->edges.begin(), h->edges.end(), [&](const PgEdge & e) { return e.ida == id || e.idb == id; }),
                 h->edges.end());
  const int pos = it->second, last = (int)h->node_ids.size() - 1;
  h->flat_dirty = true;   // node positions move and edges go: the flattened arrays are rebuilt by the next solve
  h->chol_stale = true;
  h->index.erase(it);
  if (pos != last) {
    h->node_ids[pos] = h->node_ids[last];
    for (int k = 0; k < 3; ++k) h->node_pose[3 * pos + k] = h->node_pose[3 * last + k];
    h->index[h->node_ids[pos]] = pos;
  }
  h->node_ids.pop_back();
  h->node_pose.resize(3 * h->node_ids.size());
  return B200_OK;
}

int b200pg_remove_edge(b200pg * h, int32_t ida, int32_t idb)
{
  if (!h) return B200_ERR_INVALID_ARG;
  // the block stored under (source,target) first, else (target,source) (ceres_solver.cpp:432-447)
  for (int pass = 0; pass < 2; ++pass) {
    for (size_t k = 0; k < h->edges.size(); ++k) {
      const PgEdge & e = h->edges[k];
      if ((pass == 0 && e.ida == ida && e.idb == idb) || (pass == 1 && e.ida == idb && e.idb == ida)) {
        h->edges.erase(h->edges.begin() + k);
        h->flat_dirty = true;
        h->chol_stale = true;
        return B200_OK;
      }
    }
  }
  set_last_error("RemoveConstraint: failed to find residual block");
  return B200_ERR_NOT_FOUND;
}

int b200pg_modify_node(b200pg * h, int32_t id, const double pose[3])
{
  if (!h || !pose) return B200_ERR_INVALID_ARG;
  auto it = h->index.find(id);
  if (it == h->index.end()) return B200_ERR_NOT_FOUND;
  double * p = &h->node_pose[3 * it->second];
  const double yaw_init = p[2];
  p[0] = pose[0]; p[1] = pose[1]; p[2] = pose[2];
  p[2] += yaw_init;   // ceres_solver.cpp:457-459
  return B200_OK;
}

int b200pg_get_node(const b200pg * h, int32_t id, double pose[3])
{
  if (!h || !pose) return B200_ERR_INVALID_ARG;
  auto it = h->index.find(id);
  if (it == h->index.end()) return B200_ERR_NOT_FOUND;
  for (int k = 0; k < 3; ++k) pose[k] = h->node_pose[3 * it->second + k];
  return B200_OK;
}

int32_t b200pg_num_nodes(const b200pg * h) { return h ? (int32_t)h->node_ids.size() : 0; }
int32_t b200pg_num_edges(const b200pg * h) { return h ? (int32_t)h->edges.size() : 0; }

int b200pg_solve(b200pg * h, b200pg_summary * summary)
{
  B200_GUARD_BEGIN
  if (!h) return B200_ERR_INVALID_ARG;
  return solve(h, summary);
  B200_GUARD_END
}

int b200pg_cholesky_analyze(int32_t n, int32_t e, const int32_t * edge_nodes, int32_t fixed, int64_t info[8], int32_t * order,
                            int32_t cap)
{
  B200_GUARD_BEGIN
  if (n < 0 || e < 0 || (e > 0 && !edge_nodes) || !info || fixed < -1 || fixed >= n) {
    set_last_error("b200pg_cholesky_analyze: invalid arguments");
    return B200_ERR_INVALID_ARG;
  }
  std::vector<uint8_t> is_free(n, 0);
  for (int k = 0; k < e; ++k) {
    const int a = edge_nodes[2 * k], b = edge_nodes[2 * k + 1];
    if (a < 0 || a >= n || b < 0 || b >= n || a == b) {
      set_last_error("b200pg_cholesky_analyze: edge " + std::to_string(k) + " does not join two distinct nodes in [0, n)");
      return B200_ERR_INVALID_ARG;
    }
    is_free[a] = 1; is_free[b] = 1;
  }
  if (fixed >= 0) is_free[fixed] = 0;
  CholSymbolic S;
  cholesky_analyze(n, is_free, free_pairs(n, edge_nodes, e, is_free), S);
  std::copy(S.info, S.info + 8, info);
  if (order) {
    if (cap < (int32_t)S.col_node.size()) {
      set_last_error("b200pg_cholesky_analyze: order holds fewer entries than there are free nodes");
      return B200_ERR_INVALID_ARG;
    }
    std::copy(S.col_node.begin(), S.col_node.end(), order);
  }
  return B200_OK;
  B200_GUARD_END
}

int b200pg_factor_info(const b200pg * h, int64_t info[8])
{
  if (!h || !info) return B200_ERR_INVALID_ARG;
  std::copy(h->chol_info, h->chol_info + 8, info);
  info[7] = h->chol_analyses;
  return B200_OK;
}

int32_t b200pg_get_corrections(const b200pg * h, int32_t * ids, double * poses, int32_t cap)
{
  if (!h || !ids || !poses) return 0;
  int32_t n = (int32_t)std::min<size_t>(h->corr_ids.size(), (size_t)std::max(cap, 0));
  for (int32_t i = 0; i < n; ++i) {
    ids[i] = h->corr_ids[i];
    for (int k = 0; k < 3; ++k) poses[3 * i + k] = h->corr_pose[3 * i + k];
  }
  return n;
}

}  // extern "C"
