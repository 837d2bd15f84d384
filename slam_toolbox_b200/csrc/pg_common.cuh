// What the pose-graph solver's units share: pose_graph.cu (driver, graph store, C ABI), pg_pcg.cu and pg_cholesky.cu (the
// linear solvers). Each unit plans, launches and instantiates its own kernels.
#pragma once
#include <algorithm>
#include <cmath>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

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

__device__ __forceinline__ double warp_sum(double v)
{
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
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

__device__ __forceinline__ double ld_cg(const double * p) { return __ldcg(p); }

// flags other CTAs of the same launch wait on
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

// ns since an arbitrary epoch (%globaltimer): the kernels' phase timers, printed under B200PG_DEBUG
__device__ __forceinline__ unsigned long long globaltimer()
{
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

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

// ---- launch configurations of the PCG kernels (pg_pcg.cu) ----
struct PcgSmemCfg {
  int npc;          // nodes per CTA
  int max_slots;    // max off-diagonal blocks of one CTA
  double * gz;      // [N][3]
  double * gp;      // [2][N][3]
  unsigned int * bar;   // barrier counter (zeroed before launch)
};

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

// host symbolic analysis of the factor (cholesky_analyze, pg_cholesky.cu)
struct CholSymbolic {
  std::vector<int32_t> col_node;   // [n] node of each block column
  std::vector<int32_t> node_col;   // [N] block column of each node, -1 when the node is not a column
  std::vector<int32_t> sn_col, row_start, rows, upd_start, upd, child_start, child, parent, sn_of_col;
  std::vector<int64_t> off;        // [ns + 1]
  int64_t info[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

}  // namespace b200

// ------------------------------------------------------------------------------------------
// host side: the graph store and the solver's device buffers (the b200pg handle of the C ABI)
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
  b200::DevBuf<int32_t> d_eidx, d_adj_start, d_adj, d_agg_start, d_agg_of;
  b200::DevBuf<uint8_t> d_free;
  b200::DevBuf<double> d_gz, d_gp, d_gPt, d_gRow, d_grc, d_e1, d_e2;
  bool debug = false;
  int precond = 1;   // 1 = two-level (rigid-mode aggregation) + block Jacobi, 0 = block Jacobi only
  int coarse_modes = 6;   // two-level: coarse modes per aggregate (6 = rigid + linear deformation, 3 = rigid only)
  b200::DevBuf<unsigned int> d_bar;
  bool force_global_pcg = false;
  bool force_2lvl_global = false;   // B200PG_FORCE_2LVL_GLOBAL: plan k_pg_pcg_2lvl_g at any size
  b200::DevBuf<double> d_gAc, d_gCb, d_gTb, d_gPtq;   // k_pg_pcg_2lvl_g: dense coarse matrix / inverse and its step panels
  b200::DevBuf<double> d_z, d_U, d_x, d_xc, d_scale, d_lin, d_Hd, d_g, d_diag, d_y, d_pr, d_pz, d_pp0, d_pp1, d_pq, d_Minv,
    d_partial, d_scalars;
  b200::DevBuf<double> d_ygn;   // dogleg: the Gauss-Newton solution, kept for the iterations that reuse it
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
  b200::DevBuf<int32_t> d_ch_sn_col, d_ch_row_start, d_ch_rows, d_ch_upd_start, d_ch_upd, d_ch_child_start, d_ch_child, d_ch_parent,
    d_ch_tgt_start, d_ch_src_start, d_ch_src, d_ch_col_node;
  b200::DevBuf<int64_t> d_ch_off, d_ch_tgt_off;
  b200::DevBuf<double> d_ch_L, d_ch_z;
  b200::DevBuf<unsigned int> d_ch_flag, d_ch_ctl;
  b200::PinBuf<double> h_scalars;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int64_t launches = 0;
};

namespace b200 {

template <class T>
void up(DevBuf<T> & dst, const std::vector<T> & src, cudaStream_t s)
{
  dst.reserve(std::max<size_t>(src.size(), 1));
  if (!src.empty()) B200_CUDA(cudaMemcpyAsync(dst.p, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice, s));
}

// The linear-solve kernel of a solve, as b200pg_summary.linear_solver reports it: k_pg_pcg (block-Jacobi PCG from global
// memory), k_pg_pcg_smem (block-Jacobi, each CTA's rows in shared memory), k_pg_pcg_2lvl<3 | 6> (two-level PCG with 3 or 6
// coarse modes per aggregate), k_pg_pcg_2lvl_g<3 | 6> (the same with global-memory aggregates), k_pg_cholesky.
constexpr int kLinearSolverJacobi = 0, kLinearSolverJacobiSmem = 1, kLinearSolverTwoLevel3 = 3, kLinearSolverTwoLevel6 = 6,
              kLinearSolverTwoLevelGlobal3 = 13, kLinearSolverTwoLevelGlobal6 = 16, kLinearSolverCholesky = 8;
constexpr bool is_two_level(int k) { return k == kLinearSolverTwoLevel3 || k == kLinearSolverTwoLevel6; }
constexpr bool is_two_level_global(int k) { return k == kLinearSolverTwoLevelGlobal3 || k == kLinearSolverTwoLevelGlobal6; }

// The linear-solve kernel of a solve and how it is launched.
struct PcgPlan {
  int kernel = kLinearSolverJacobi;
  int blocks = 0;           // cooperative grid
  size_t smem_bytes = 0;    // dynamic shared memory
  PcgSmemCfg smem{};        // kLinearSolverJacobiSmem
  Pcg2Cfg two_level{};      // kLinearSolverTwoLevel3 / 6
  Pcg2GCfg two_level_g{};   // kLinearSolverTwoLevelGlobal3 / 6
};

// pg_pcg.cu: picks the PCG kernel from the graph's CSR rows and allocates its work buffers; one linear solve
// (H + shift D^2) y = g on it, scalars[8] = iterations, [9] = relative residual
PcgPlan plan_pcg(b200pg * h, const std::vector<int32_t> & adj_start, cudaStream_t st);
void pcg_solve(b200pg * h, PgDev d, PcgPlan & plan, double shift, double tol, int max_iter, cudaStream_t st);

// pg_cholesky.cu: the Cholesky plan of a solve (B200_ERR_UNSUPPORTED when the factor does not fit the free device memory);
// one exact linear solve (H + shift D^2) y = g, scalars[8] = 0, [9] = relative residual
int plan_cholesky(b200pg * h, const std::vector<uint8_t> & is_free, cudaStream_t st, PcgPlan & P);
void cholesky_solve(b200pg * h, PgDev d, int blocks, double shift, cudaStream_t st);

}  // namespace b200
