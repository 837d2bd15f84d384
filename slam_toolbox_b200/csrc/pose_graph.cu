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
//     persistent cooperative kernel per solve, planned from the graph's rows (pg_pcg.cu).  Opt-in (linear_solver_type = 1):
//     the exact solve SPARSE_NORMAL_CHOLESKY does, a supernodal FP64 Cholesky (pg_cholesky.cu).
//   * one fused kernel evaluates every edge's residual, both Jacobian blocks (analytic) and the
//     off-diagonal normal-equation block; a second gathers per-node diagonal blocks/gradients
//     through a CSR node->edge adjacency (no atomics: bit-reproducible results).
//
// Data layout (HBM, FP64): nodes AoS [N][3]; edges SoA-of-small-arrays: idx[E][2], z[E][3],
// U[E][6] (upper triangle), lin[E][30] = r(3) | A~(9) | B~(9) | M = A~^T B~ (9); node blocks
// Hd[N][6] (symmetric), g[N][3]. The whole 10k/40k problem is ~15 MB: L2 resident.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <complex>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pg_common.cuh"

namespace b200 {

__device__ __forceinline__ double wrap_angle(double a)   // ceres_utils.h:27-32
{
  const double two_pi = 2.0 * M_PI;
  return a - two_pi * floor((a + M_PI) / two_pi);
}

__device__ __forceinline__ double warp_max(double v)
{
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
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
// host side: LM driver
// ------------------------------------------------------------------------------------------

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
    if (plan.kernel == kLinearSolverCholesky) cholesky_solve(h, d, plan.blocks, shift, st);
    else pcg_solve(h, d, plan, shift, tol, max_iter, st);
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
    if (L.h->debug && is_two_level_global(L.plan.kernel))
      fprintf(stderr, "[b200pg] lm %d: pcg %d it, setup %.1f us, gauss-jordan %.1f us, cg %.1f us (%.2f us/it)\n", it, (int)sc[8],
              sc[10] * 1e-3, sc[11] * 1e-3, sc[12] * 1e-3, sc[12] * 1e-3 / std::max(1.0, sc[8]));
    if (L.h->debug && is_two_level(L.plan.kernel))
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

using namespace b200;

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

