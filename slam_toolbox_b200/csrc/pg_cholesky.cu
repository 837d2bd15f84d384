// b200slam pose-graph solver: the exact linear solve (linear_solver_type = 1), the one SPARSE_NORMAL_CHOLESKY does: a
// supernodal FP64 Cholesky in one persistent cooperative kernel per solve (k_pg_cholesky) after a host symbolic analysis
// (cholesky_analyze), and the ABI entries that report the analysis.
#include <cooperative_groups.h>

#include <cassert>
#include <iterator>
#include <set>

#include "pg_common.cuh"

namespace cg = cooperative_groups;

namespace b200 {

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
  if (timer) t0 = globaltimer();
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
  if (timer) t1 = globaltimer();
  // backward, supernodes in reverse postorder; a supernode waits for its parent
  for (int t = chol_ticket(c.ctl + 1, &s_ticket); t < c.ns; t = chol_ticket(c.ctl + 1, &s_ticket)) {
    const int J = c.ns - 1 - t;
    CHOL_CHECK(c.parent[J] < 0 || c.parent[J] > J);   // the parent holds a lower backward ticket
    if (c.parent[J] >= 0) chol_wait(c.flag + c.ns, c.parent + J, 1, c.epoch);
    chol_backward_supernode(d, c, J, sZ);
    chol_publish(c.flag + c.ns + J, c.epoch);
  }
  grid.sync();
  if (timer) t2 = globaltimer();
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
    t3 = globaltimer();
    d.scalars[10] = (double)(t1 - t0); d.scalars[11] = (double)(t2 - t1); d.scalars[12] = (double)(t3 - t2);
    d.scalars[8] = 0.0;
    d.scalars[9] = ld_acquire_u32(c.ctl + 2) == c.epoch ? __longlong_as_double(0x7FF8000000000000LL) : (gg > 0.0 ? sqrt(rr / gg) : 0.0);
  }
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
int plan_cholesky(b200pg * h, const std::vector<uint8_t> & is_free, cudaStream_t st, PcgPlan & P)
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

// The Cholesky branch of a linear solve: a new epoch for the completion flags, fresh tickets, the cooperative launch.
void cholesky_solve(b200pg * h, PgDev d, int blocks, double shift, cudaStream_t st)
{
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
  B200_CUDA(cudaLaunchCooperativeKernel((void *)k_pg_cholesky, dim3(blocks), dim3(kCholThreads), args, 0, st));
}

}  // namespace b200

using namespace b200;

extern "C" {

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

}  // extern "C"
