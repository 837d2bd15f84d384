// b200slam pose-graph solver: the PCG linear solvers (DESIGN.md §4), their plan and their launch. Each runs one persistent
// cooperative kernel per solve; every reduction is summed in a fixed order.
#include <cooperative_groups.h>

#include <cstdio>

#include "pg_common.cuh"

namespace cg = cooperative_groups;

namespace b200 {

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

// the result of a solve: scalars[8] = iterations, [9] = final relative residual ||r|| / ||b||
__device__ __forceinline__ void pcg_result(const PgDev & d, int it, double rr, double bb)
{
  d.scalars[8] = (double)it;
  d.scalars[9] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
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
  if (tid == 0) pcg_result(d, it, rr, bb);
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
__device__ __forceinline__ void grid_barrier(unsigned int * bar, unsigned int target)
{
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    while (ld_acquire_u32(bar) < target) {}
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
  if (blockIdx.x == 0 && tid == 0) pcg_result(d, it, rr, bb);
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

// ---- steps the two-level kernels share ----
// P~ base block of node i, the n-th of the nloc nodes of its aggregate: the aggregate's rigid-body modes in Jacobi-scaled
// variables (y~ = y / s) about the centroid (cx, cy) of its nfree free nodes; zero for a constant node. Returns the node's
// weight s of the s-weighted modes.
template <int CM>
__device__ __forceinline__ double rigid_modes(const PgDev & d, int i, int n, int nloc, double cx, double cy, double nfree,
                                              double * pt)
{
  const double f = d.is_free[i] ? 1.0 : 0.0;
  const double isx = f / d.scale[3 * i], isy = f / d.scale[3 * i + 1], ist = f / d.scale[3 * i + 2];
  pt[0] = isx; pt[1] = 0;   pt[2] = -(d.x[3 * i + 1] - cy) * isx;
  pt[3] = 0;   pt[4] = isy; pt[5] = (d.x[3 * i] - cx) * isy;
  pt[6] = 0;   pt[7] = 0;   pt[8] = ist;
  // the s-weighted modes need two free nodes to be independent of the rigid ones; otherwise they are switched off
  // (s = 0 gives zero rows and columns of Ac, which are replaced by the identity's)
  return (CM > 3 && nloc > 1 && nfree >= 2.0) ? 2.0 * n / (double)(nloc - 1) - 1.0 : 0.0;
}

// w3 = pi^T B pj: the 3x3 block B (row-major) of H + D between nodes i and j, projected on their P~ base blocks
__device__ __forceinline__ void coarse_block(const double * B, const double * pi, const double * pj, double * w3)
{
  double w[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int q = 0; q < 3; ++q) w[3 * r + q] = B[3 * r] * pj[q] + B[3 * r + 1] * pj[3 + q] + B[3 * r + 2] * pj[6 + q];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int q = 0; q < 3; ++q) w3[3 * r + q] = pi[r] * w[q] + pi[3 + r] * w[3 + q] + pi[6 + r] * w[6 + q];
}

// fixed-order sums of the G polled {r.z, r.r} pairs s by warp 0; broadcast through out[0], out[1]
__device__ __forceinline__ void ordered_sum_pairs(const double * s, int G, double * out)
{
  if (threadIdx.x < 32) {
    double u = 0, w = 0;
    for (int i = threadIdx.x; i < G; i += 32) { u += s[2 * i]; w += s[2 * i + 1]; }
    u = warp_sum(u); w = warp_sum(w);
    if (threadIdx.x == 0) { out[0] = u; out[1] = w; }
  }
  __syncthreads();
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
  unsigned long long tA = 0, tB = 0, tC = 0, tD = 0, tE = 0, t0 = 0;   // CG phase timers
  auto tick = [&](unsigned long long & acc) {
    if (I == 0 && tid == 0) { const unsigned long long t1 = globaltimer(); acc += t1 - t0; t0 = t1; }
  };
  if (I == 0 && tid == 0) t_start = globaltimer();

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
    double * pt = sPt + 9 * n;
    const double sn = rigid_modes<CM>(d, i, n, nloc, s_small[0], s_small[1], s_small[2], pt);
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
      double pj[9], w3[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) pj[k] = ld_cg(c.gPt + 10 * (size_t)j + k);
      const double sj = ld_cg(c.gPt + 10 * (size_t)j + 9);
      coarse_block(sB + 9 * s, sPt + 9 * sNode[s], pj, w3);
      add_block(w3, sS[sNode[s]], sj);
    }
    if (ct == I) {   // diagonal blocks of own nodes
      for (int n = 0; n < nloc; ++n) {
        const double * H = sH + 6 * n, * pi = sPt + 9 * n;
        const double B[9] = {H[0], H[1], H[2], H[1], H[3], H[4], H[2], H[4], H[5]};
        double w3[9];
        coarse_block(B, pi, pi, w3);
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
  if (I == 0 && tid == 0) t_setup = globaltimer();
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
        st_release_u32(c.gjflag + k, 1u);
      }
    } else {
      if (tid == 0)
        while (ld_acquire_u32(c.gjflag + k) == 0u) {}
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
  if (I == 0 && tid == 0) t_gj = globaltimer();
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
      if (I == 0 && tid == 0) t0 = globaltimer();
      gather_neighbours(sCol, nslots, lo, hi, sZ, sP, c.gz, gpo, beta, sV);
      tick(tA);
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
      tick(tB);
      if (tid == 0) {
        __threadfence();   // p_new of this CTA visible before the flagged values
        double * m = e1 + (size_t)I * kSlotStride;
#pragma unroll
        for (int k = 1; k < KE1; ++k) m[k] = a1[k];
        m[0] = a1[0];
      }
      poll_slots<KE1>(e1, G, sEx);
      tick(tC);
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
      tick(tD);
      if (tid == 0) {
        __threadfence();   // z of this CTA visible before the flagged values
        double * m = e2 + (size_t)I * kSlotStride;
        m[0] = a2[0]; m[1] = a2[1];
      }
      poll_slots<2>(e2, G, sEx);
      tick(tE);
      // every CTA published E2(it) only after it finished reading E1(it): recycle own E1(it) slots
      if (tid < KE1) c.e1[((size_t)par * G + I) * kSlotStride + tid] = SENT;
      ordered_sum_pairs(sEx, G, s_small);
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
    const unsigned long long t_end = globaltimer();
    pcg_result(d, it, rr, bb);
    d.scalars[10] = (double)(t_setup - t_start);   // ns: load rows + P~ + first barrier + Ac rows
    d.scalars[11] = (double)(t_gj - t_setup);      // ns: block Gauss-Jordan
    d.scalars[12] = (double)(t_end - t_gj);        // ns: CG iterations
    d.scalars[13] = (double)tA; d.scalars[14] = (double)tB; d.scalars[15] = (double)tC;
    d.scalars[6] = (double)tD; d.scalars[7] = (double)tE;
  }
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
  if (I == 0 && tid == 0) t_start = globaltimer();

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
      pt[9] = rigid_modes<CM>(d, i, n, nloc, cx, cy, cnt, pt);
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
          double pi[9];
#pragma unroll
          for (int k = 0; k < 9; ++k) pi[k] = ld_cg(c.gPt + 10 * (size_t)i + k);
          const double si = ld_cg(c.gPt + 10 * (size_t)i + 9);
          double * o = stg + 12 * lane;
          coarse_block(B, pi, pj, o);
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
  if (I == 0 && tid == 0) t_setup = globaltimer();

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
  if (I == 0 && tid == 0) t_gj = globaltimer();

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
      ordered_sum_pairs(sEx, G, s_small);
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
    const unsigned long long t_end = globaltimer();
    pcg_result(d, it, rr, bb);
    d.scalars[10] = (double)(t_setup - t_start);   // ns: Minv, P~, Ac assembly
    d.scalars[11] = (double)(t_gj - t_setup);      // ns: blocked Gauss-Jordan
    d.scalars[12] = (double)(t_end - t_gj);        // ns: CG iterations
  }
}

constexpr int kMin2lvlGlobalNodes = 8192;
constexpr int kMaxCoarse2lvlGlobal = 4096;

// Cuts the N nodes into contiguous aggregates of `per` nodes (the last one may be shorter): agg_start [aggregates + 1],
// agg_of [N] the aggregate of every node.
static void contiguous_aggregates(int N, int per, std::vector<int32_t> & agg_start, std::vector<int32_t> & agg_of)
{
  agg_start.clear(); agg_of.assign(N, 0);
  for (int i = 0; i < N; i += per) agg_start.push_back(i);
  agg_start.push_back(N);
  for (int a = 0; a + 1 < (int)agg_start.size(); ++a)
    for (int i = agg_start[a]; i < agg_start[a + 1]; ++i) agg_of[i] = a;
}

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

// Plans k_pg_pcg_2lvl_g into P (kLinearSolverTwoLevelGlobal3 / 6) when its dense coarse inverse fits the free device
// memory; otherwise leaves P as it is (B200PG_DEBUG says why).
static void plan_pcg_2lvl_global(b200pg * h, const std::vector<int32_t> & adj_start, int sms, cudaStream_t st, PcgPlan & P)
{
  const int N = (int)adj_start.size() - 1;
  const int cm = h->coarse_modes >= 6 ? 6 : 3;
  const int want = coarse_aggregates_2lvl_global(N, adj_start[N], cm);
  std::vector<int32_t> agg_start, agg_of;
  const int per = (N + want - 1) / want;
  contiguous_aggregates(N, per, agg_start, agg_of);
  const int na = (int)agg_start.size() - 1;
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
  P.kernel = cm == 6 ? kLinearSolverTwoLevelGlobal6 : kLinearSolverTwoLevelGlobal3; P.blocks = G; P.smem_bytes = bytes;
  Pcg2GCfg & c = P.two_level_g;
  c.na = na; c.apc = apc; c.ld = ld; c.agg_start = h->d_agg_start.p; c.agg_of = h->d_agg_of.p;
  c.gz = h->d_gz.p; c.gp = h->d_gp.p; c.gPt = h->d_gPt.p; c.Ac = h->d_gAc.p; c.Cb = h->d_gCb.p; c.Tb = h->d_gTb.p;
  c.gPtq = h->d_gPtq.p; c.grc = h->d_grc.p; c.e1 = h->d_e1.p; c.e2 = h->d_e2.p; c.bar = h->d_bar.p;
}

// Picks the PCG kernel from the graph's CSR rows: shared-memory block-Jacobi where every CTA's rows fit, then the two-level
// kernel where its aggregates fit (B200PG_PRECOND, B200PG_COARSE_MODES and B200PG_FORCE_GLOBAL_PCG narrow the choice).
// Allocates the work buffers of the kernels it considers.
PcgPlan plan_pcg(b200pg * h, const std::vector<int32_t> & adj_start, cudaStream_t st)
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
      P.kernel = kLinearSolverJacobiSmem; P.blocks = Gu; P.smem_bytes = bytes;
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
    for (int per_sm = 1; per_sm <= 2 && !is_two_level(P.kernel); ++per_sm) {
      const int G2 = std::min(per_sm * sms, std::max(1, (N + 15) / 16));
      // contiguous node ranges of equal node count: compact aggregates give the best coarse space (balancing by
      // block count was tried: it merges sparse chain stretches into large aggregates and costs more iterations)
      std::vector<int32_t> & agg_start = h->agg_start_h;
      std::vector<int32_t> & agg_of = h->agg_of_h;
      contiguous_aggregates(N, (N + G2 - 1) / G2, agg_start, agg_of);
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
      P.kernel = cm == 6 ? kLinearSolverTwoLevel6 : kLinearSolverTwoLevel3; P.blocks = Gu; P.smem_bytes = bytes2;
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
  if (h->precond == 1 && !h->force_global_pcg && (h->force_2lvl_global || (P.kernel == kLinearSolverJacobi && N >= kMin2lvlGlobalNodes)))
    plan_pcg_2lvl_global(h, adj_start, sms, st, P);
  return P;
}

// The PCG branches of a linear solve: zero the barrier counter, launch the planned kernel cooperatively.
void pcg_solve(b200pg * h, PgDev d, PcgPlan & plan, double shift, double tol, int max_iter, cudaStream_t st)
{
  if (is_two_level_global(plan.kernel)) {
    B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, sizeof(unsigned int), st));
    void * args[] = {&d, &plan.two_level_g, &shift, &tol, &max_iter};
    B200_CUDA(cudaLaunchCooperativeKernel(plan.kernel == kLinearSolverTwoLevelGlobal6 ? (void *)k_pg_pcg_2lvl_g<6> : (void *)k_pg_pcg_2lvl_g<3>, dim3(plan.blocks), dim3(kG2Threads), args, plan.smem_bytes, st));
  } else if (is_two_level(plan.kernel)) {
    B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, (size_t)(plan.blocks + 1) * sizeof(unsigned int), st));
    void * args[] = {&d, &plan.two_level, &shift, &tol, &max_iter};
    B200_CUDA(cudaLaunchCooperativeKernel(plan.kernel == kLinearSolverTwoLevel6 ? (void *)k_pg_pcg_2lvl<6> : (void *)k_pg_pcg_2lvl<3>, dim3(plan.blocks), dim3(256), args, plan.smem_bytes, st));
  } else if (plan.kernel == kLinearSolverJacobiSmem) {
    B200_CUDA(cudaMemsetAsync(h->d_bar.p, 0, sizeof(unsigned int), st));
    void * args[] = {&d, &plan.smem, &shift, &tol, &max_iter};
    B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_pcg_smem, dim3(plan.blocks), dim3(512), args, plan.smem_bytes, st));
  } else {
    void * args[] = {&d, &shift, &tol, &max_iter};
    B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_pcg, dim3(plan.blocks), dim3(kPgThreads), args, 0, st));
  }
}

}  // namespace b200
