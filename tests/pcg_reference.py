"""Plain FP64 restatement of the pose-graph solver's PCG linear solve (pg_pcg.cu: k_pg_pcg, k_pg_pcg_smem, k_pg_pcg_2lvl and
k_pg_pcg_2lvl_g), written from the kernels, for tests that compare the solver iterate by iterate.

The system is the LM step's Jacobi-scaled normal equations over all N nodes in insertion order,
    A = J~^T J~ + D^2 / radius,   b = J~^T r,   J~ = J diag(s),   s = 1 / (1 + ||J col||),   D^2 = clamp(colnorm^2(J~)),
built from oracle.posegraph.Problem at the start point (robust-loss corrector included).  Fixed and isolated nodes have zero
Jacobian columns, s = 1 and D^2 = min_lm_diagonal: their rows reduce to D^2 y / radius = 0.

Under LM the solver accepts the linear solve whatever its residual, so a solve capped at k PCG iterations returns the k-th
iterate y_k and the step x1 = x0 (+) (-s * y_k).  y_k depends on the preconditioner at O(1) for small k, so comparing it
with the restated iterate checks every piece of the preconditioner, which the converged outcome of an LM solve cannot see.

Preconditioners, as each kernel applies them:
  * kernels 0 / 1: block Jacobi, (Hd_i + D_i^2 / radius)^-1 per node;
  * kernels 3 / 6 and 13 / 16: M^-1 = blockdiag^-1 + P~ Ac^-1 P~^T with Ac = P~^T A P~.  P~ holds CM (3 or 6) modes per
    aggregate: the rigid modes about the centroid of the aggregate's free nodes, divided by the Jacobi scale, and (CM = 6) the
    same modes weighted by s = 2 n / (nloc - 1) - 1 over the node's index n in the aggregate; s = 0 for an aggregate of one node
    or with fewer than two free nodes.  Ac^-1 comes from each kernel's own Gauss-Jordan: CM x CM block pivots for 3 / 6,
    32-column panels over Ac padded with the identity to a multiple of 64 for 13 / 16.  Both replace a pivot that is zero
    or dependent (|pivot| <= 1e-12 |its diagonal when its block / panel step began|) by the identity's row and column;
    13 / 16 also put 1 on the zero diagonal of a mode without support when they assemble Ac.  The coarse residual P~^T r is
    carried by the recurrence rc -= alpha P~^T q, as in the kernels.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

from oracle import posegraph as PG

H100_SMS = 132
GJ_PANEL, GJ_TILE = 32, 64
MIN_2LVL_GLOBAL_NODES, MAX_COARSE_2LVL_GLOBAL = 8192, 4096


# ---- the linear system of the first LM step ----

class System:
    """A, b, the Jacobi scale s and the damping of the first LM step at x0, over all N nodes in insertion order."""

    def __init__(self, x0, ia, ib, z, cov, anchor=0, loss="none", loss_scale=0.7, radius=1e4, min_diag=1e-6,
                 max_diag=1e32):
        x0 = np.asarray(x0, dtype=np.float64)
        N = len(x0)
        U = np.stack([PG.sqrt_information(c) for c in cov])
        pb = PG.Problem(x0, ia, ib, z, U, anchor, loss, loss_scale)
        J = pb.jacobian(x0)
        r = pb.residuals(x0)
        sf = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(axis=0)).reshape(-1)))
        Js = (J @ sp.diags(sf)).tocsr()
        Df = np.clip(np.asarray(Js.multiply(Js).sum(axis=0)).reshape(-1), min_diag, max_diag)
        cols = (3 * pb.free[:, None] + np.arange(3)[None, :]).reshape(-1)
        emb = sp.csr_matrix((np.ones(len(cols)), (cols, np.arange(len(cols)))), shape=(3 * N, len(cols)))
        self.N, self.x0, self.pb, self.radius, self.cols = N, x0, pb, radius, cols
        self.free = np.zeros(N, dtype=bool)
        self.free[pb.free] = True
        self.s = np.ones(3 * N)
        self.s[cols] = sf
        D = np.full(3 * N, float(np.clip(0.0, min_diag, max_diag)))
        D[cols] = Df
        self.D = D
        self.Js, self.r = Js, r
        self.H = (emb @ (Js.T @ Js) @ emb.T).tocsr()
        self.A = (self.H + sp.diags(D / radius)).tocsr()
        self.b = emb @ (Js.T @ r)
        # the diagonal 3 x 3 blocks of A (Hd_i + D_i^2 / radius)
        coo = self.A.tocoo()
        m = coo.row // 3 == coo.col // 3
        self.blocks = np.zeros((N, 3, 3))
        np.add.at(self.blocks, (coo.row[m] // 3, coo.row[m] % 3, coo.col[m] % 3), coo.data[m])
        deg = np.bincount(np.concatenate([np.asarray(ia), np.asarray(ib)]), minlength=N)
        self.slots = deg   # CSR slots of every node's row: its incident edge ends

    def step(self, y):
        """x0 (+) (-s * y) on the free nodes (AngleLocalParameterization on theta), k_pg_apply_step."""
        d = (-self.s * y)[self.cols]
        return self.pb.plus(self.x0, d)

    def step_quality(self, y):
        """(cost at x0, candidate cost, model cost change, step norm) of the LM step -y, as the minimiser evaluates them."""
        mr = self.Js @ (-y[self.cols])
        model = -float(mr @ (self.r + mr / 2.0))
        x1 = self.step(y)
        return self.pb.cost(self.x0), self.pb.cost(x1), model, float(np.linalg.norm((x1 - self.x0)[self.free]))


# ---- aggregate layouts ----

def plan_two_level(deg, sms=H100_SMS, coarse_modes=6):
    """plan_pcg()'s shared-memory two-level branch (kernels 3 / 6) restated from the node degrees in insertion order:
    G2 = min(per_sm * sms, ceil(N / 16)) contiguous aggregates of equal node count, one CTA per SM first, then two, and 6
    coarse modes before 3 where the CTA's bytes fit. Returns (CM, aggregate starts) or None when no layout fits."""
    deg = np.asarray(deg)
    N = len(deg)
    start = np.concatenate([[0], np.cumsum(deg)])
    for per_sm in (1, 2):
        G2 = min(per_sm * sms, max(1, (N + 15) // 16))
        per = -(-N // G2)
        lo = list(range(0, N, per))
        hi = lo[1:] + [N]
        Gu = len(lo)
        ms2 = max(1, max(int(start[h] - start[l]) for l, h in zip(lo, hi)))
        npc2 = max(1, max(h - l for l, h in zip(lo, hi)))
        for cm in (6, 3):
            if cm > coarse_modes:
                continue
            nc = cm * Gu
            ex = max((1 + cm) * Gu, cm * nc - 3 * ms2)
            b2 = (ms2 * 12 + npc2 * 37 + (cm + 1) * nc + ex) * 8 + (2 * ms2 + npc2 + 1) * 4 + 16
            if b2 > 220 * 1024:
                continue
            static = (1 + cm) * 32 * 8 + 8 + (cm * cm + 4) * 8 + 64
            occ = min(2, (228 * 1024) // (b2 + static + 1024))
            if occ * sms < Gu:
                continue
            return cm, np.array(lo + [N])
    return None


def plan_two_level_global(N, slots, cm):
    """coarse_aggregates_2lvl_global() and plan_pcg_2lvl_global()'s layout (kernels 13 / 16): nc <= sqrt(fine bytes per
    iteration / 32), at most 4096, aggregates of at least 16 nodes. Returns (aggregate starts, ld)."""
    fine = 240.0 * N + 128.0 * slots
    nc = min(MAX_COARSE_2LVL_GLOBAL, int(math.sqrt(fine / 32.0)))
    want = max(1, min((N + 15) // 16, nc // cm))
    per = -(-N // want)
    starts = np.array(list(range(0, N, per)) + [N])
    ncoarse = cm * (len(starts) - 1)
    return starts, -(-ncoarse // GJ_TILE) * GJ_TILE


# ---- the coarse space ----

def prolongation(sy: System, agg_start, cm, centroid=True, s_sign=1.0, s_one_free=False):
    """P~ (3N x CM na, sparse): rows 3 i + component, columns CM a + mode.  The keyword arguments change the kernels' rule
    (for tests that show a changed rule moves the iterates): centroid=False puts the rotation mode about the origin,
    s_sign=-1 reverses s, s_one_free=True keeps the s-modes of an aggregate with one free node."""
    x, free, sc = sy.x0, sy.free, sy.s
    rows, cols, vals = [], [], []
    for a in range(len(agg_start) - 1):
        lo, hi = int(agg_start[a]), int(agg_start[a + 1])
        nloc = hi - lo
        fm = free[lo:hi]
        cnt = int(fm.sum())
        cx = x[lo:hi, 0][fm].mean() if cnt and centroid else 0.0
        cy = x[lo:hi, 1][fm].mean() if cnt and centroid else 0.0
        on = cm > 3 and nloc > 1 and (cnt >= 2 or (s_one_free and cnt >= 1))
        for n in range(nloc):
            i = lo + n
            if not free[i]:
                continue
            isx, isy, ist = 1.0 / sc[3 * i], 1.0 / sc[3 * i + 1], 1.0 / sc[3 * i + 2]
            pt = np.array([[isx, 0.0, -(x[i, 1] - cy) * isx], [0.0, isy, (x[i, 0] - cx) * isy], [0.0, 0.0, ist]])
            sn = s_sign * (2.0 * n / (nloc - 1) - 1.0) if on else 0.0
            for r in range(3):
                for q in range(3):
                    rows.append(3 * i + r); cols.append(cm * a + q); vals.append(pt[r, q])
                    if cm > 3:
                        rows.append(3 * i + r); cols.append(cm * a + 3 + q); vals.append(sn * pt[r, q])
    nc = cm * (len(agg_start) - 1)
    return sp.csr_matrix((vals, (rows, cols)), shape=(3 * sy.N, nc))


def coarse_matrix(sy: System, P):
    """Ac = P~^T A P~ (dense)."""
    return np.asarray((P.T @ (sy.A @ P)).todense())


def _dependent(piv, d0):
    return not (abs(piv) > 1e-12 * d0) or not (d0 > 1e-300)


def gj_small(D):
    """k_pg_pcg_2lvl's inverse of one CM x CM pivot block: Gauss-Jordan on [D | I] without pivoting; a zero or dependent pivot
    has its row (both halves) and its column (left half) zeroed and a 1 on both diagonals."""
    m = D.shape[0]
    a = np.hstack([D.astype(np.float64), np.eye(m)])
    d0 = np.abs(np.diag(D)).copy()
    for p in range(m):
        if _dependent(a[p, p], d0[p]):
            a[p, :] = 0.0
            a[:m, p] = 0.0
            a[p, p] = 1.0
            a[p, m + p] = 1.0
        a[p, :] *= 1.0 / a[p, p]
        for r in range(m):
            if r != p:
                a[r, :] -= a[r, p] * a[p, :]
    return a[:, m:]


def gj_block(Ac, cm):
    """k_pg_pcg_2lvl's block Gauss-Jordan on [Ac | I], one CM-row pivot block per aggregate; returns Ac^-1."""
    nc = Ac.shape[0]
    M = np.hstack([Ac.astype(np.float64), np.eye(nc)])
    for k in range(nc // cm):
        ks = slice(cm * k, cm * k + cm)
        M[ks, :] = gj_small(M[ks, ks]) @ M[ks, :]
        other = np.r_[0:cm * k, cm * k + cm:nc]
        mult = M[other, ks].copy()
        M[other, :] -= mult @ M[ks, :]
    return M[:, nc:]


def gj_invert_cols(D):
    """gj_invert_cols: in-place Gauss-Jordan inverse of one 32 x 32 block; d0 is the diagonal when the panel step began."""
    a = D.astype(np.float64).copy()
    n = a.shape[0]
    d0 = np.abs(np.diag(a)).copy()
    for p in range(n):
        piv = a[p, p]
        if _dependent(piv, d0[p]):
            a[p, :] = 0.0
            a[:, p] = 0.0
            a[p, p] = 1.0
            piv = 1.0
        inv = 1.0 / piv
        rowp = a[p, :] * inv
        rowp[p] = inv
        cp = a[:, p].copy()
        a -= np.outer(cp, rowp)
        a[:, p] = -cp * inv
        a[p, :] = rowp
    return a


def gj_panel(Ac, ld=None):
    """k_pg_pcg_2lvl_g's set-up: a zero diagonal becomes 1, Ac is padded with the identity to ld (a multiple of 64), and
    the blocked in-place Gauss-Jordan steps 32 columns at a time. Returns the nc x nc block of the inverse."""
    nc = Ac.shape[0]
    ld = ld or -(-nc // GJ_TILE) * GJ_TILE
    A = np.eye(ld)
    A[:nc, :nc] = Ac
    d = np.arange(nc)
    A[d, d] = np.where(A[d, d] == 0.0, 1.0, A[d, d])
    for k0 in range(0, ld, GJ_PANEL):
        K = slice(k0, k0 + GJ_PANEL)
        Dinv = gj_invert_cols(A[K, K])
        V = A[K, :].copy()
        V[:, K] = np.eye(GJ_PANEL)
        T = Dinv @ V
        C = A[:, K].copy()
        C[K, :] = -np.eye(GJ_PANEL)
        A[K, :] = 0.0
        A[:, K] = 0.0
        A -= C @ T
    return A[:nc, :nc]


# ---- preconditioners and PCG ----

class Preconditioner:
    """M^-1 = blockdiag^-1 (+ P~ Ac^-1 P~^T)."""

    def __init__(self, sy: System, P=None, Aci=None):
        self.Binv = np.linalg.inv(sy.blocks)
        self.P, self.Aci = P, Aci
        self.PT = None if P is None else P.T.tocsr()

    def fine(self, r):
        return np.einsum("nij,nj->ni", self.Binv, r.reshape(-1, 3)).reshape(-1)

    def apply(self, r, rc=None):
        z = self.fine(r)
        if self.P is not None:
            z = z + self.P @ (self.Aci @ rc)
        return z

    def dense(self):
        """M^-1 as a dense matrix (small systems)."""
        n = len(self.Binv)
        M = np.zeros((3 * n, 3 * n))
        for i in range(n):
            M[3 * i:3 * i + 3, 3 * i:3 * i + 3] = self.Binv[i]
        if self.P is not None:
            Pd = self.P.toarray()
            M += Pd @ self.Aci @ Pd.T
        return M


def jacobi(sy: System):
    return Preconditioner(sy)


def two_level(sy: System, agg_start, cm, gj="block", coarse=True, **mutation):
    """The two-level preconditioner of kernels 3 / 6 (gj='block') or 13 / 16 (gj='panel'); coarse=False drops the coarse term."""
    if not coarse:
        return Preconditioner(sy)
    P = prolongation(sy, agg_start, cm, **mutation)
    Ac = coarse_matrix(sy, P)
    Aci = gj_block(Ac, cm) if gj == "block" else gj_panel(Ac)
    pc = Preconditioner(sy, P, Aci)
    pc.Ac = Ac
    return pc


def pcg(sy: System, pc: Preconditioner, tol=1e-30, max_iter=10, keep=None):
    """k_pg_pcg's recurrences from y0 = 0: r0 = b, z = M^-1 r; p = z + beta p, alpha = rz / pq; stop when rr <= tol^2 bb or
    pq <= 0 (tested after the update).  Returns (iterates y_1 .. y_keep, final y, iterations)."""
    A, b = sy.A, sy.b
    two = pc.P is not None
    y = np.zeros_like(b)
    r = b.copy()
    rc = pc.PT @ b if two else None
    z = pc.apply(r, rc)
    bb = float(b @ b)
    rz = float(r @ z)
    stop = tol * tol * bb
    p = np.zeros_like(b)
    beta, it, out = 0.0, 0, []
    keep = max_iter if keep is None else keep
    if bb > 0.0:
        while it < max_iter:
            p = z + beta * p
            q = A @ p
            pq = float(p @ q)
            alpha = rz / pq
            if two:
                rc = rc - alpha * (pc.PT @ q)
            y = y + alpha * p
            r = r - alpha * q
            z = pc.apply(r, rc)
            rz_new, rr = float(r @ z), float(r @ r)
            it += 1
            if len(out) < keep:
                out.append(y.copy())
            if not (rr > stop) or not (pq > 0.0):
                break
            beta = rz_new / rz
            rz = rz_new
    return out, y, it


# ---- the kernels and their layouts ----

KERNELS = (0, 1, 3, 6, 13, 16)
KERNEL_ENV = {0: {"B200PG_FORCE_GLOBAL_PCG": "1"}, 1: {"B200PG_PRECOND": "jacobi"}, 3: {"B200PG_COARSE_MODES": "3"}, 6: {},
              13: {"B200PG_FORCE_2LVL_GLOBAL": "1", "B200PG_COARSE_MODES": "3"}, 16: {"B200PG_FORCE_2LVL_GLOBAL": "1"}}


def layout(sy: System, kernel, sms=H100_SMS):
    """(CM, aggregate starts) of a two-level kernel on this graph, as its plan lays them out."""
    if kernel in (3, 6):
        plan = plan_two_level(sy.slots, sms, coarse_modes=kernel)
        assert plan is not None and plan[0] == kernel, (kernel, plan)
        return plan
    cm = kernel - 10
    return cm, plan_two_level_global(sy.N, int(sy.slots.sum()), cm)[0]


def preconditioner(sy: System, kernel, sms=H100_SMS):
    if kernel in (0, 1):
        return jacobi(sy)
    cm, starts = layout(sy, kernel, sms)
    return two_level(sy, starts, cm, gj="block" if kernel < 10 else "panel")


# ---- the case graphs ----

def interleave_isolated(g, after, run):
    """g with `run` isolated nodes inserted after each insertion position in `after`: aggregates that cover such a stretch
    hold one free node or none."""
    N = len(g["init"])
    rng = np.random.default_rng(5)
    seq, iso = [], 0
    for p in range(N):
        seq.append(p)
        if p in after:
            seq += [-1] * run
    newpos = {p: k for k, p in enumerate(seq) if p >= 0}
    init = np.array([g["init"][p] if p >= 0 else [rng.uniform(-20, 20), rng.uniform(-20, 20), rng.uniform(-3, 3)]
                     for p in seq])
    comp = np.array([g["component"][p] if p >= 0 else -1 for p in seq])
    M = len(seq)
    ids = np.arange(M, dtype=np.int32)
    ia = np.array([newpos[p] for p in g["ia"]])
    ib = np.array([newpos[p] for p in g["ib"]])
    return dict(g, ids=ids, init=init, truth=init, ia=ia, ib=ib, edge_a=ids[ia], edge_b=ids[ib], component=comp, anchor=0)


def with_outliers(g, frac, sigma, seed):
    """g with the loop closures of a fraction `frac` of its edges' xy measurements moved by N(0, sigma)."""
    rng = np.random.default_rng(seed)
    z = g["z"].copy()
    bad = rng.choice(len(z), size=max(4, int(frac * len(z))), replace=False)
    z[bad, :2] += rng.normal(0.0, sigma, (len(bad), 2))
    return dict(g, z=z)


def case_graph(name):
    """The graphs the iterate tests run on, each pushing the kernels into one case (see CASES)."""
    from slam_toolbox_b200 import synth
    fam = synth.make_pose_graph_family
    if name == "lattice_321":
        return fam(70, 321, 640, cov_model="karto", lattice=12, min_gap=20)
    if name == "karto_shuffled":
        return fam(31, 1500, 3000, cov_model="karto", reversed_frac=0.3, duplicate_frac=0.05, order="shuffled", ids="sparse",
                   world_rotation=0.7, isolated_runs=((0.3, 40), (0.7, 48)), detached_nodes=120)
    if name == "iso_far":
        return fam(33, 800, 1600, cov_model="iso", order="chain", ids="sparse", world_rotation=0.7,
                   world_translation=(1e4, -3e4))
    if name == "one_free":
        g = fam(71, 500, 1000, cov_model="karto", lattice=14, min_gap=20)
        return interleave_isolated(g, after=set(range(150, 170)) | set(range(300, 304)), run=40)
    if name == "hub":
        return fam(72, 1000, 2000, cov_model="karto", reversed_frac=0.2, lattice=30, hub_degree=300)
    if name == "huber":
        return with_outliers(fam(73, 900, 1800, cov_model="karto", reversed_frac=0.3, lattice=18), 0.02, 2.0, 74)
    raise KeyError(name)


# graph -> (kernels, loss)
CASES = {
    "lattice_321": (KERNELS, "none"),       # ~300-node lattice walk near the origin; 3 / 6: a last aggregate of one node
    "karto_shuffled": (KERNELS, "none"),    # sparse ids, shuffled order, reversed / parallel edges, isolated runs, no anchor
    "iso_far": (KERNELS, "none"),           # centroids at (1e4, -3e4)
    "one_free": (KERNELS, "none"),          # isolated nodes interleaved: aggregates with exactly one free node
    "hub": ((0, 1), "none"),                # a node of degree ~300
    "huber": ((6,), "huber"),               # HuberLoss with outliers
}


def case_system(name):
    g = case_graph(name)
    return g, System(g["init"], g["ia"], g["ib"], g["z"], g["cov"], anchor=g.get("anchor", 0), loss=CASES[name][1])
