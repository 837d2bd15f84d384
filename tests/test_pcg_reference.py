"""The FP64 restatement of the pose-graph PCG (tests/pcg_reference.py) checked on its own, without a GPU: converged PCG is
the direct solve, Ac is P~^T A P~, both Gauss-Jordan restatements invert Ac, M^-1 is symmetric positive definite, the
restated steps of the GPU test are accepted steps, the layouts match the plan's restatement in tools/, and the iterates the
GPU test compares move far more than its tolerance when the preconditioner is changed the way a bug would change it."""
import functools
import importlib.util
import os

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import pcg_reference as R

TAU = 1e-9   # the GPU test's relative tolerance on y_k
EPS = np.finfo(np.float64).eps
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def case(name):
    return R.case_system(name)


@functools.lru_cache(maxsize=None)
def free_spectrum(name):
    _, sy = case(name)
    Af = sy.A[sy.cols][:, sy.cols].toarray()
    return np.linalg.eigvalsh(Af)


def moved(a, b, s):
    """max |s (a - b)| / max |s b|: the change of the pose step; a non-finite change counts as moved"""
    d = np.abs(s * (a - b)).max() / np.abs(s * b).max()
    return d if np.isfinite(d) else np.inf


# ---- PCG to convergence is the direct solve ----

@pytest.mark.parametrize("kernel", R.KERNELS)
@pytest.mark.parametrize("name", ["lattice_321", "one_free", "iso_far"])
def test_converged_pcg_is_the_direct_solve(name, kernel):
    """As the bound of test_lm_trajectory_and_one_step_bound: ||y - y*|| <= (tol ||b|| + k eps ||A|| ||y*||) / lambda_min,
    over the free rows (the others are D^2 y / radius = 0 on both sides)."""
    _, sy = case(name)
    tol = 1e-12
    _, y, its = R.pcg(sy, R.preconditioner(sy, kernel), tol=tol, max_iter=20000, keep=0)
    ystar = spla.spsolve(sy.A.tocsc(), sy.b)
    lam = free_spectrum(name)
    bound = (tol * np.linalg.norm(sy.b) + its * EPS * lam[-1] * np.linalg.norm(ystar)) / lam[0]
    assert np.linalg.norm(y - ystar) <= bound, (np.linalg.norm(y - ystar), bound)
    assert not np.any(y[~np.isin(np.arange(3 * sy.N), sy.cols)])


# ---- the coarse operator ----

def coarse_by_blocks(sy, starts, cm):
    """Ac as the kernels assemble it: per block (i, j) of A with W = pi^T A_ij pj, the coarse block [[W, s_j W], [s_i W,
    s_i s_j W]] added at (aggregate of i, aggregate of j)."""
    P = R.prolongation(sy, starts, cm).toarray()
    agg = np.repeat(np.arange(len(starts) - 1), np.diff(starts))
    pt = np.zeros((sy.N, 3, 3))
    sn = np.zeros(sy.N)
    for i in range(sy.N):
        a = agg[i]
        pt[i] = P[3 * i:3 * i + 3, cm * a:cm * a + 3]
        if cm > 3 and np.any(pt[i]):
            k = np.nonzero(pt[i])
            sn[i] = P[3 * i:3 * i + 3, cm * a + 3:cm * a + 6][k][0] / pt[i][k][0]
    Ac = np.zeros((cm * (len(starts) - 1),) * 2)
    A = sy.A.tocsr()
    for i in range(sy.N):
        for j in set(A.indices[A.indptr[3 * i]:A.indptr[3 * i + 3]] // 3):
            W = pt[i].T @ A[3 * i:3 * i + 3, 3 * j:3 * j + 3].toarray() @ pt[j]
            blk = W if cm == 3 else np.block([[W, sn[j] * W], [sn[i] * W, sn[i] * sn[j] * W]])
            Ac[cm * agg[i]:cm * agg[i] + cm, cm * agg[j]:cm * agg[j] + cm] += blk
    return Ac


@pytest.mark.parametrize("kernel", [3, 6, 13, 16])
def test_coarse_matrix_is_the_dense_product(kernel):
    _, sy = case("lattice_321")
    cm, starts = R.layout(sy, kernel)
    P = R.prolongation(sy, starts, cm)
    Ac = R.coarse_matrix(sy, P)
    Pd = P.toarray()
    dense = Pd.T @ sy.A.toarray() @ Pd
    scale = np.abs(dense).max()
    assert np.abs(Ac - dense).max() <= 1e-12 * scale
    assert np.abs(coarse_by_blocks(sy, starts, cm) - dense).max() <= 1e-12 * scale


def spd(n, seed, cond=1e4):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    return (Q * np.geomspace(1.0, cond, n)) @ Q.T


@pytest.mark.parametrize("cm", [3, 6])
def test_gauss_jordan_restatements_invert(cm):
    """nc = 138 / 141: not a multiple of 32, so the panel restatement uses the identity padding."""
    n = cm * (23 if cm == 6 else 47)
    Ac = spd(n, cm)
    inv = np.linalg.inv(Ac)
    for got in (R.gj_block(Ac, cm), R.gj_panel(Ac)):
        assert np.abs(got - inv).max() <= 1e-12 * np.abs(inv).max() * 1e4   # 1e-12 relative at cond 1e4
    assert np.linalg.norm(R.gj_panel(Ac) - inv) / np.linalg.norm(inv) <= 1e-12
    assert np.linalg.norm(R.gj_block(Ac, cm) - inv) / np.linalg.norm(inv) <= 1e-12


@pytest.mark.parametrize("cm", [3, 6])
def test_gauss_jordan_zero_modes_become_the_identity(cm):
    n = cm * 23
    Ac = spd(n, 10 + cm)
    zero = np.array([1, cm + 2, 5 * cm, 5 * cm + 1, n - 1])
    Ac[zero, :] = 0.0
    Ac[:, zero] = 0.0
    keep = np.setdiff1d(np.arange(n), zero)
    inv = np.linalg.inv(Ac[np.ix_(keep, keep)])
    for got in (R.gj_block(Ac, cm), R.gj_panel(Ac)):
        assert np.linalg.norm(got[np.ix_(keep, keep)] - inv) / np.linalg.norm(inv) <= 1e-12
        assert np.array_equal(got[np.ix_(zero, zero)], np.eye(len(zero)))
        assert not np.any(got[np.ix_(zero, keep)]) and not np.any(got[np.ix_(keep, zero)])


def test_pivot_rules_differ_only_on_coupled_dependent_modes():
    """The CM-block rule (3 / 6) and the 32-panel rule (13 / 16) agree on every case graph's Ac, which is nonsingular on its
    supported modes; they differ where a mode depends on earlier ones and still couples to later ones: a mode that equals
    a combination of two others of the same 32-column panel."""
    for name in ("karto_shuffled", "one_free"):
        _, sy = case(name)
        cm, starts = R.layout(sy, 16)
        Ac = R.coarse_matrix(sy, R.prolongation(sy, starts, cm))
        a, b = R.gj_block(Ac, cm), R.gj_panel(Ac)
        assert np.abs(a - b).max() <= 1e-9 * np.abs(b).max(), name
    n, cm = 96, 6
    B = np.random.default_rng(3).normal(size=(n, n + 8))
    B[10] = B[3] + 0.5 * B[7]   # mode 10 depends on modes 3 and 7
    Ac = B @ B.T
    a, b = R.gj_block(Ac, cm), R.gj_panel(Ac)
    assert np.all(np.isfinite(b))
    assert not np.allclose(a, b, rtol=1e-6, atol=0.0)


# ---- the preconditioner ----

@pytest.mark.parametrize("name,kernel", [(n, k) for n, (ks, _) in R.CASES.items() for k in ks])
def test_preconditioner_is_symmetric_positive_definite(name, kernel):
    """M^-1 = blockdiag^-1 + P~ Ac^-1 P~^T: SPD when every Jacobi block is and the symmetric part of Ac^-1 is positive
    semi-definite, with Ac^-1 symmetric to rounding."""
    _, sy = case(name)
    pc = R.preconditioner(sy, kernel)
    assert np.abs(pc.Binv - pc.Binv.transpose(0, 2, 1)).max() <= 1e-12 * np.abs(pc.Binv).max(axis=(1, 2)).max()
    assert np.linalg.eigvalsh(0.5 * (pc.Binv + pc.Binv.transpose(0, 2, 1))).min() > 0.0
    if pc.P is None:
        return
    X = pc.Aci
    assert np.abs(X - X.T).max() <= 1e-9 * np.abs(X).max()
    lam = np.linalg.eigvalsh(0.5 * (X + X.T))
    assert lam.min() > -1e-12 * lam.max(), (lam.min(), lam.max())
    if sy.N <= 400:   # and once densely
        M = pc.dense()
        assert np.abs(M - M.T).max() <= 1e-9 * np.abs(M).max()
        assert np.linalg.eigvalsh(0.5 * (M + M.T)).min() > 0.0


# ---- mutations: a changed preconditioner moves y_1 and y_3 far beyond the GPU tolerance ----

def iterates(sy, pc):
    its = R.pcg(sy, pc, max_iter=3)[0]
    return its[0], its[2] if len(its) > 2 else np.full_like(its[0], np.nan)


MUTATIONS = {
    "no_coarse_term": dict(coarse=False),
    "3_modes": dict(cm=3),
    "boundary_moved": dict(boundary=1),
    "centroid_at_origin": dict(centroid=False),
    "s_modes_on_one_free_node": dict(s_one_free=True),
}
# where a mutation changes the operator M^-1: the centroid only far from the origin (near it, rotating about the origin is
# a change of basis of the same coarse space), the s-modes only where an aggregate has one free node and more nodes
WHERE = {"centroid_at_origin": ("iso_far",), "s_modes_on_one_free_node": ("one_free",)}
GRAPHS = ["lattice_321", "karto_shuffled", "iso_far", "one_free", "huber"]


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
@pytest.mark.parametrize("kernel", [6, 16])
def test_mutations_move_the_iterates(kernel, mutation):
    m = dict(MUTATIONS[mutation])
    for name in WHERE.get(mutation, GRAPHS):
        _, sy = case(name)
        cm, starts = R.layout(sy, kernel)
        gj = "block" if kernel < 10 else "panel"
        base = iterates(sy, R.two_level(sy, starts, cm, gj=gj))
        if m.pop("boundary", 0):
            # a boundary in the middle whose first node is free (moving one between isolated nodes changes nothing)
            b = next(b for b in range(len(starts) // 2, len(starts) - 1) if sy.free[starts[b]])
            starts = starts.copy()
            starts[b] += 1
        cm = m.pop("cm", cm)
        with np.errstate(all="ignore"):   # the s-modes of one free node make Ac singular: the block rule overflows
            mut = iterates(sy, R.two_level(sy, starts, cm, gj=gj, **m))
        m = dict(MUTATIONS[mutation])
        for a, b in zip(mut, base):
            assert moved(a, b, sy.s) >= 1e3 * TAU, (name, moved(a, b, sy.s))


@pytest.mark.parametrize("kernel", [6, 16])
def test_basis_changes_leave_the_iterates(kernel):
    """Reversing s or rotating about another point changes P~ by an invertible map of each aggregate's modes, which leaves
    P~ Ac^-1 P~^T, and so every iterate, as it is: those are not preconditioner bugs, and no iterate test can see them."""
    _, sy = case("lattice_321")
    cm, starts = R.layout(sy, kernel)
    gj = "block" if kernel < 10 else "panel"
    base = iterates(sy, R.two_level(sy, starts, cm, gj=gj))
    for kw in (dict(s_sign=-1.0), dict(centroid=False)):
        for a, b in zip(iterates(sy, R.two_level(sy, starts, cm, gj=gj, **kw)), base):
            assert moved(a, b, sy.s) <= 1e-10, kw


def test_case_graphs_reach_their_cases():
    """The layouts put each case where the GPU test needs it."""
    _, sy = case("lattice_321")
    for k in (3, 6):
        assert np.diff(R.layout(sy, k)[1])[-1] == 1   # a last aggregate of one node
    _, sy = case("one_free")
    for k in (3, 6, 13, 16):
        starts = R.layout(sy, k)[1]
        free = np.add.reduceat(sy.free.astype(int), starts[:-1])
        assert np.any((free == 1) & (np.diff(starts) > 1)), k
    for name in ("karto_shuffled", "iso_far", "one_free"):
        _, sy = case(name)
        for k in (13, 16):
            cm, starts = R.layout(sy, k)
            nc = cm * (len(starts) - 1)
            assert nc > 64 and nc % 32, (name, k, nc)
    g, sy = case("hub")
    assert np.max(sy.slots) >= 300


# ---- the restated steps of the GPU test are accepted steps ----

@pytest.mark.parametrize("name,kernel", [(n, k) for n, (ks, _) in R.CASES.items() for k in ks])
def test_restated_steps_are_accepted(name, kernel):
    """With max_num_iterations = 1 and the tight tolerances, the solver returns x0 (+) (-s y_k) only if that step is accepted:
    cost falls, quality far above min_relative_decrease (1e-3) and neither the parameter nor the function tolerance ends
    the solve first."""
    _, sy = case(name)
    its = R.pcg(sy, R.preconditioner(sy, kernel), max_iter=10)[0]
    assert len(its) == 10
    x_norm = np.linalg.norm(sy.x0[sy.free])
    for k in (1, 2, 3, 5, 10):
        c0, c1, model, step = sy.step_quality(its[k - 1])
        assert model > 0 and c1 < c0
        assert (c0 - c1) / model > 0.1, (k, (c0 - c1) / model)
        assert step > 1e-12 * (x_norm + 1e-12) and abs(c0 - c1) > 1e-10 * c0


# ---- the global layout against the study's restatement ----

def test_global_layout_matches_the_study():
    from slam_toolbox_b200 import synth
    spec = importlib.util.spec_from_file_location("large_graph_study", os.path.join(ROOT, "tools", "large_graph_study.py"))
    study = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(study)
    for n, e, lat in ((15000, 60000, 122), (60000, 73200, 245)):   # the LARGE graphs of test_posegraph_large_gpu.py
        g = synth.make_pose_graph(7, n, e, lattice=lat, sigma_xy=0.03, sigma_th=0.01)
        E = len(g["edge_a"])
        for cm in (3, 6):
            starts, ld = R.plan_two_level_global(n, 2 * E, cm)
            want = study.coarse_plan(n, E, cm)
            assert (len(starts) - 1, int(starts[1] - starts[0]), cm * (len(starts) - 1)) == \
                (want["aggregates"], want["nodes_per_aggregate"], want["nc"])
            assert ld % R.GJ_TILE == 0 and ld - want["nc"] < R.GJ_TILE
