"""The CUDA pose-graph solver against the restated-Ceres oracle on graphs of the shapes a mapper produces
(synth.make_pose_graph_family): correlated covariances (full sqrt-information), reversed and parallel edges, shuffled
insertion order with the anchor in the middle of the walk, sparse / negative / extreme int32 ids, a rotated and
translated world, runs of isolated nodes, a component without the anchor and hub nodes.  Every case runs under each
of the four PCG kernels the solver plans between and asserts which one ran (b200pg_summary.linear_solver)."""
import math

import numpy as np
import pytest

from oracle import posegraph as PG
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
TOL_XY, TOL_TH = 1e-4, 1e-5
TERMINATION = {"CONVERGENCE (function tolerance)": 0, "CONVERGENCE (nothing to optimise)": 0,
               "CONVERGENCE (gradient tolerance)": 1, "CONVERGENCE (parameter tolerance)": 2,
               "NO_CONVERGENCE (max iterations)": 3, "CONVERGENCE (min trust region radius)": 4,
               "FAILURE (too many invalid steps)": 5}
KERNEL_ENV = {6: {}, 3: {"B200PG_COARSE_MODES": "3"}, 1: {"B200PG_PRECOND": "jacobi"}, 0: {"B200PG_FORCE_GLOBAL_PCG": "1"}}

FAMILIES = {
    # correlated xy covariances, reversed and parallel edges, shuffled order, sparse ids, a detached walk and isolated runs
    "karto_shuffled": dict(seed=31, n_nodes=1500, n_loops=3000, cov_model="karto", reversed_frac=0.3, duplicate_frac=0.05,
                           order="shuffled", ids="sparse", world_rotation=0.7, isolated_runs=((0.3, 40), (0.7, 48)),
                           detached_nodes=120),
    # xy-theta correlations, half the edges reversed, the anchor at the end of the walk
    "full_reversed": dict(seed=32, n_nodes=1200, n_loops=2400, cov_model="full", reversed_frac=0.5, duplicate_frac=0.02,
                          order="reversed", world_rotation=-2.0, isolated_runs=((0.5, 40),)),
    # far from the origin: Ceres' relative parameter tolerance ends the solve early, on both sides
    "iso_far": dict(seed=33, n_nodes=800, n_loops=1600, cov_model="iso", order="chain", ids="sparse", world_rotation=0.7,
                    world_translation=(1e4, -3e4)),
}


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def family(name):
    kw = dict(FAMILIES[name])
    return synth.make_pose_graph_family(kw.pop("seed"), **kw)


def build(g, init=None, **opts):
    s = api.ScanSolver(**opts)
    for nid, p in zip(g["ids"], g["init"] if init is None else init):
        s.AddNode(int(nid), p)
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
        assert s.AddConstraint(int(a), int(b), z, c)
    return s


def oracle(g, init=None, **opts):
    x0 = g["init"] if init is None else init
    return PG.solve(x0, g["ia"], g["ib"], g["z"], cov=g["cov"], fixed=g["anchor"], opts=PG.Options(**opts))


def degrees(n, ia, ib):
    return np.bincount(np.concatenate([ia, ib]), minlength=n)


def planned_kernel(deg, sms, coarse_modes=6, precond=1, force_global=False):
    """The host plan of pg_pcg.cu (plan_pcg(): shared-memory Jacobi bytes, then the two-level aggregates and their
    bytes for 6 and 3 coarse modes) restated from the node degrees in insertion order."""
    N = len(deg)
    start = np.concatenate([[0], np.cumsum(deg)])
    G = min(sms, max(1, (N + 31) // 32))
    npc = -(-N // G)
    ms = max(1, max(int(start[min(N, lo + npc)] - start[lo]) for lo in range(0, N, npc)))
    use_smem = ((ms * 12 + npc * 27) * 8 + (ms + npc + 1) * 4 + 16) <= 200 * 1024 and not force_global
    if precond == 1 and not force_global:
        for per_sm in (1, 2):
            G2 = min(per_sm * sms, max(1, (N + 15) // 16))
            per = -(-N // G2)
            lo = list(range(0, N, per))
            hi = lo[1:] + [N]
            Gu = len(lo)
            ms2 = max(1, max(int(start[h] - start[l]) for l, h in zip(lo, hi)))
            npc2 = max(h - l for l, h in zip(lo, hi))
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
                return cm
    return 1 if use_smem else 0


def diff(x, y):
    d = x - y
    d[:, 2] = synth.wrap(d[:, 2])
    return np.abs(d[:, :2]).max(), np.abs(d[:, 2]).max()


def check_solve(g, s, xo, so, kernel, x0):
    """Parity with the oracle plus the invariants every solve must keep."""
    sm = s.summary
    assert sm.linear_solver == kernel, (sm.linear_solver, kernel)
    ids, xg = s.GetCorrections()
    assert np.array_equal(ids, g["ids"])
    dxy, dth = diff(xg, xo)
    assert dxy < TOL_XY and dth < TOL_TH, (dxy, dth)
    assert (sm.iterations, sm.successful_steps) == (so.iterations, so.successful_steps), \
        ((sm.iterations, sm.successful_steps), (so.iterations, so.successful_steps))
    assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (sm.final_cost, so.final_cost)
    assert sm.termination == TERMINATION[so.termination], (sm.termination, so.termination)
    # nodes outside the problem (the anchor, isolated nodes) come back bit-identical, whatever their yaw
    fixed = np.zeros(len(xg), dtype=bool)
    fixed[g["anchor"]] = True
    fixed[g["component"] < 0] = True
    assert np.array_equal(xg[fixed], x0[fixed])
    # every optimised node's yaw was wrapped to [-pi, pi) by the step (AngleLocalParameterization)
    assert np.all(xg[~fixed, 2] >= -math.pi) and np.all(xg[~fixed, 2] < math.pi)
    return xg


_ORACLE = {}


def family_oracle(name, g, x0):
    if name not in _ORACLE:
        _ORACLE[name] = oracle(g, x0)
    return _ORACLE[name]


def push_yaws(g, s):
    """ModifyNode adds the stored yaw (ceres_solver.cpp:457-459): push the anchor's and an isolated node's yaw outside
    [-pi, pi). Returns the initial poses as the solver now holds them."""
    x0 = g["init"].copy()
    for p in [g["anchor"]] + list(np.nonzero(g["component"] < 0)[0][:1]):
        s.ModifyNode(int(g["ids"][p]), [x0[p, 0], x0[p, 1], 7.0])
        x0[p] = s.get_node(int(g["ids"][p]))
        assert x0[p, 2] > math.pi
    return x0


@pytest.mark.parametrize("kernel", [6, 3, 1, 0])
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_family_matches_oracle_under_each_kernel(name, kernel, monkeypatch):
    for k, v in KERNEL_ENV[kernel].items():
        monkeypatch.setenv(k, v)
    g = family(name)
    s = build(g)
    x0 = push_yaws(g, s)
    xo, so = family_oracle(name, g, x0)
    assert s.Compute()
    xg = check_solve(g, s, xo, so, kernel, x0)
    # a second solve of the same input is bit-identical
    s2 = build(g)
    push_yaws(g, s2)
    assert s2.Compute()
    assert np.array_equal(s2.GetCorrections()[1], xg)
    assert (s2.summary.iterations, s2.summary.pcg_iterations) == (s.summary.iterations, s.summary.pcg_iterations)


def test_karto_covariances_at_cfg4_size():
    """One cfg4-sized graph (10,000 nodes, 40,000 loop closures) with karto covariances, shuffled insertion order and sparse ids
    on the default kernel."""
    g = synth.make_pose_graph_family(34, 10000, 40000, cov_model="karto", reversed_frac=0.3, order="shuffled", ids="sparse",
                                     lattice=100, min_gap=50)
    s = build(g)
    xo, so = oracle(g)
    assert s.Compute()
    check_solve(g, s, xo, so, planned_kernel(degrees(len(g["ids"]), g["ia"], g["ib"]), sm_count()), g["init"])


@pytest.mark.parametrize("model", ["iso", "karto", "full"])
@pytest.mark.parametrize("loss,code", [("none", 0), ("huber", 1), ("cauchy", 2)])
def test_cost_kernel_alone(model, loss, code):
    """max_num_iterations = 0: the solve evaluates the cost at the start point and stops. The initial cost is a sum of
    positive terms, so the GPU's summation order can only move it by a few ulps per term."""
    g = synth.make_pose_graph_family(40, 600, 1200, cov_model=model, reversed_frac=0.4, duplicate_frac=0.05, order="shuffled",
                                     ids="sparse", world_rotation=0.7, world_translation=(1e4, -3e4))
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["init"], g["ia"], g["ib"], g["z"], U, g["anchor"], loss, 0.7)
    s = build(g, max_num_iterations=0, loss_function=code, loss_scale=0.7)
    assert s.Compute()
    want = pb.cost(g["init"])
    assert abs(s.summary.initial_cost - want) <= 1e-12 * want, (s.summary.initial_cost, want)
    assert s.summary.iterations == 0 and s.summary.final_cost == s.summary.initial_cost
    assert np.array_equal(s.GetCorrections()[1], g["init"])


# tight, but stopping before candidate costs differ only by rounding (where accepting a step is a coin toss on any solver)
TIGHT = dict(function_tolerance=1e-10, parameter_tolerance=1e-12, gradient_tolerance=1e-12)


@pytest.mark.parametrize("model", ["karto", "full"])
def test_lm_trajectory_and_one_step_bound(model):
    """The LM trajectory step by step: the solve stopped after k iterations (k = 1..8) has the oracle's accepted-step count
    and minimum cost over the first k iterations of its trace.

    After one accepted step the poses differ from the oracle's exact (SuperLU) step only by the PCG error.  PCG stops when
    its recurrence residual r_k satisfies ||r_k||_2 <= tol ||b||_2 for the Jacobi-scaled system A y = b,
    A = J~^T J~ + D / radius.  The true residual b - A y_k differs from r_k by rounding that accumulates over the k PCG
    iterations, at most about k eps ||A||_2 max_j ||y_j||_2, and the CG iterates' norms grow monotonically towards ||y*||_2.
    So ||y - y*||_2 <= ||b - A y||_2 / lambda_min(A) <= (tol ||b||_2 + k eps ||A||_2 ||y*||_2) / lambda_min(A).  The pose
    step is delta = -s * y with the Jacobi scaling s, so no coordinate moves more than max(s) times that from the oracle's.
    The bound is computed from A at the start point and must be 1000x tighter than the 1e-4 m parity bound.  Measured on
    an H100 (pcg_tolerance 1e-14, 100 nodes, ~500 PCG iterations): the largest one-step difference was 2.8e-14 (karto)
    and 6.9e-14 (full) against bounds of 2.8e-8 and 2.4e-8."""
    g = synth.make_pose_graph_family(41, 100, 200, cov_model=model, reversed_frac=0.3, duplicate_frac=0.05, order="shuffled",
                                     ids="sparse", world_rotation=0.7)
    K, tol = 8, 1e-14
    _, so = oracle(g, max_num_iterations=K, **TIGHT)
    trace = so.trace
    for k in range(1, K + 1):
        s = build(g, max_num_iterations=k, pcg_tolerance=tol, **TIGHT)
        assert s.Compute()
        pre = [t for t in trace if t[0] <= k]
        want_cost = min(t[1] for t in pre)
        want_steps = sum(1 for t in pre[1:] if t[2])
        assert s.summary.successful_steps == want_steps, (k, s.summary.successful_steps, want_steps)
        assert abs(s.summary.final_cost - want_cost) <= 1e-9 * want_cost, (k, s.summary.final_cost, want_cost)
        if k == 1:
            x1, pcg_its = s.GetCorrections()[1], s.summary.pcg_iterations
    assert trace[1][2], "the first LM step of this graph is accepted"
    xo1, so1 = oracle(g, max_num_iterations=1, **TIGHT)
    # the bound, from the scaled normal equations at the start point
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["init"], g["ia"], g["ib"], g["z"], U, g["anchor"])
    J = pb.jacobian(g["init"])
    r = pb.residuals(g["init"])
    sc = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(axis=0)).reshape(-1)))
    Js = J.multiply(sc[None, :]).tocsc()
    D = np.clip(np.asarray(Js.multiply(Js).sum(axis=0)).reshape(-1), 1e-6, 1e32)
    A = (Js.T @ Js).toarray() + np.diag(D / 1e4)
    b = Js.T @ r
    lam = np.linalg.eigvalsh(A)
    ystar = np.linalg.solve(A, b)
    eps = np.finfo(np.float64).eps
    bound = sc.max() * (tol * np.linalg.norm(b) + pcg_its * eps * lam[-1] * np.linalg.norm(ystar)) / lam[0]
    assert bound <= 1e-7, bound
    dxy, dth = diff(x1, xo1)
    assert max(dxy, dth) <= bound, (dxy, dth, bound)


def boundary_sizes():
    n = 16 * sm_count()
    return [2, 15, 16, 17, 33, n - 1, n, n + 1]


@pytest.mark.parametrize("i", range(8))
def test_plan_boundaries_through_the_node_count(i):
    """Node counts at the edges of the plan: one aggregate, the 16-node aggregate size, and one aggregate per SM."""
    n = boundary_sizes()[i]
    small = n < 64   # a 3 x 3 lattice: small walks revisit sites, so they have loop closures
    g = synth.make_pose_graph_family(50 + i, n, 2 * n, cov_model="karto", reversed_frac=0.3, duplicate_frac=0.3, order="shuffled",
                                     ids="sparse", min_gap=1 if small else 20, lattice=3 if small else 60)
    want = planned_kernel(degrees(n, g["ia"], g["ib"]), sm_count())
    s = build(g)
    x0 = push_yaws(g, s)
    xo, so = oracle(g, x0)
    assert s.Compute()
    check_solve(g, s, xo, so, want, x0)


def hub_degrees(n, base_deg, hub, sms):
    """Hub degrees that push the plan from 6 coarse modes to 3, to shared-memory Jacobi and to global Jacobi: the middle of
    each degree window of planned_kernel (the byte formulas of the plan) with the hub's edges added to its row."""
    windows = {}
    for d in range(0, 4000, 4):
        deg = base_deg.copy()
        deg[hub] += d
        windows.setdefault(planned_kernel(deg, sms), []).append(d)
    return {k: v[len(v) // 2] for k, v in windows.items()}


@pytest.mark.parametrize("kernel", [6, 3, 1, 0])
def test_plan_fallbacks_through_a_hub_node(kernel):
    n = 5000
    kw = dict(n_nodes=n, n_loops=2 * n, cov_model="karto", reversed_frac=0.2, order="chain", lattice=70)
    g0 = synth.make_pose_graph_family(60, **kw)
    sms = sm_count()
    d = hub_degrees(n, degrees(n, g0["ia"], g0["ib"]), n // 2, sms)
    assert kernel in d, d
    g = synth.make_pose_graph_family(60, hub_degree=d[kernel], **kw)
    assert degrees(n, g["ia"], g["ib"])[n // 2] >= d[kernel]
    assert planned_kernel(degrees(n, g["ia"], g["ib"]), sms) == kernel
    s = build(g)
    xo, so = oracle(g)
    assert s.Compute()
    check_solve(g, s, xo, so, kernel, g["init"])


def test_remove_node_in_the_middle_then_solve():
    """RemoveNode moves the last inserted node into the freed slot; the solve must still match the oracle on the remaining
    graph (and keep the anchor, the first node ever added)."""
    g = family("karto_shuffled")
    s = build(g)
    N = len(g["ids"])
    p = next(q for q in range(N // 2, N) if g["component"][q] == 0)
    assert s.RemoveNode(int(g["ids"][p]))
    keep = np.ones(N, dtype=bool)
    keep[p] = False
    ek = (g["ia"] != p) & (g["ib"] != p)
    newpos = np.cumsum(keep) - 1
    g2 = dict(g, ids=g["ids"][keep], init=g["init"][keep], component=g["component"][keep], ia=newpos[g["ia"][ek]],
              ib=newpos[g["ib"][ek]], edge_a=g["edge_a"][ek], edge_b=g["edge_b"][ek], z=g["z"][ek], cov=g["cov"][ek])
    xo, so = oracle(g2)
    assert s.Compute()
    ids, xg = s.GetCorrections()
    order = np.argsort(g2["ids"])
    back = order[np.searchsorted(g2["ids"], ids, sorter=order)]
    assert np.array_equal(g2["ids"][back], ids)
    dxy, dth = diff(xg, xo[back])
    assert dxy < TOL_XY and dth < TOL_TH, (dxy, dth)
    assert (s.summary.iterations, s.summary.successful_steps) == (so.iterations, so.successful_steps)
    assert abs(s.summary.final_cost - so.final_cost) <= 1e-8 * so.final_cost
    assert np.array_equal(xg[list(ids).index(g["ids"][0])], g["init"][0])
