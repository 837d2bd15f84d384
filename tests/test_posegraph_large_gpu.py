"""The two-level PCG with global-memory aggregates (k_pg_pcg_2lvl_g, b200pg_summary.linear_solver 13 / 16) on pose graphs
too large for the shared-memory kernels, and forced (B200PG_FORCE_2LVL_GLOBAL=1) on the small graphs of the other suites:
which kernel the plan picks, P1 parity with the exact-solve oracles under LM, both dogleg types and HuberLoss,
bit-reproducibility and an incremental solve."""
import math

import numpy as np
import pytest

import posegraph_dogleg as DL
from oracle import posegraph as PG
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
TOL_XY, TOL_TH = 1e-4, 1e-5
FORCE = "B200PG_FORCE_2LVL_GLOBAL"
SIGMAS = [(0.03, 0.01), (0.05, 0.02)]
# cfg4 density (4 edges per node) past the shared-memory kernels' reach, lattice side scaled with sqrt(N); and the density of
# a recorded mapping run (1.22 edges per node)
LARGE = {"cfg4_15k": (15000, 60000, 122), "recorded_60k": (60000, 73200, 245)}


def large_graph(name, sigma=SIGMAS[0]):
    n, e, lat = LARGE[name]
    return synth.make_pose_graph(7, n, e, lattice=lat, sigma_xy=sigma[0], sigma_th=sigma[1])


def build(g, init=None, **opts):
    s = api.ScanSolver(**opts)
    for nid, p in zip(g["ids"], g["init"] if init is None else init):
        s.AddNode(int(nid), p)
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
        assert s.AddConstraint(int(a), int(b), z, c)
    return s


def diff(x, y):
    d = x - y
    d[:, 2] = synth.wrap(d[:, 2])
    return np.abs(d[:, :2]).max(), np.abs(d[:, 2]).max()


def check_p1(s, so, xo, kernel, linear_solves=False):
    sm = s.summary
    assert sm.linear_solver == kernel, (sm.linear_solver, kernel)
    got, want = (sm.iterations, sm.successful_steps), (so.iterations, so.successful_steps)
    if linear_solves:
        got, want = got + (sm.linear_solves,), want + (so.linear_solves,)
    assert got == want, (got, want)
    assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (sm.final_cost, so.final_cost)
    dxy, dth = diff(s.GetCorrections()[1], xo)
    assert dxy < TOL_XY and dth < TOL_TH, (dxy, dth)


def planned(g, **opts):
    s = build(g, max_num_iterations=1, **opts)
    assert s.Compute()
    return s.summary.linear_solver


def test_plan_choice(monkeypatch):
    """cfg4 keeps the shared-memory two-level kernel; both graphs past its reach plan the global one, and
    B200PG_FORCE_GLOBAL_PCG still plans block-Jacobi from global memory there."""
    assert planned(synth.make_pose_graph(0, 10000, 40000, sigma_xy=0.05, sigma_th=0.02)) == 6
    graphs = [large_graph(name) for name in sorted(LARGE)]
    assert [planned(g) for g in graphs] == [16, 16]
    monkeypatch.setenv("B200PG_COARSE_MODES", "3")
    assert planned(graphs[0]) == 13
    monkeypatch.delenv("B200PG_COARSE_MODES")
    monkeypatch.setenv("B200PG_FORCE_GLOBAL_PCG", "1")
    assert [planned(g) for g in graphs] == [0, 0]


# At 0.05 m / 0.02 rad the recorded-density graph's dead-reckoned start is so far off that the exact-solve oracle itself stops at
# max_num_iterations (50) with the cost still falling, where a final-cost tolerance says nothing about the linear solver
@pytest.mark.parametrize("name,sigma", [("cfg4_15k", SIGMAS[0]), ("cfg4_15k", SIGMAS[1]), ("recorded_60k", SIGMAS[0])])
def test_p1_past_the_cliff(name, sigma):
    """P1 of the parity protocol (as test_cfg4_full_size) against the exact-solve LM oracle."""
    g = large_graph(name, sigma)
    xo, so = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"])
    s = build(g)
    assert s.Compute()
    check_p1(s, so, xo, 16)
    assert np.array_equal(s.GetCorrections()[1][0], g["init"][0])


@pytest.mark.parametrize("t", ["traditional", "subspace"])
def test_dogleg_past_the_cliff(t):
    g = large_graph("cfg4_15k", SIGMAS[1])
    o = DL.Options(trust_region_strategy="dogleg", dogleg_type=t)
    xo, so = DL.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], fixed=0, opts=o)
    s = build(g, trust_region_strategy=1, dogleg_type={"traditional": 0, "subspace": 1}[t])
    assert s.Compute()
    check_p1(s, so, xo, 16, linear_solves=True)


def test_huber_past_the_cliff():
    g = large_graph("cfg4_15k", SIGMAS[1])
    xo, so = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=PG.Options(loss_function="huber"))
    s = build(g, loss_function=1, loss_scale=0.7)
    assert s.Compute()
    check_p1(s, so, xo, 16)
    assert s.summary.linear_solves == so.iterations


# the families of test_posegraph_shapes_gpu.py, rebuilt here: correlated covariances, reversed and parallel edges, shuffled and
# reversed insertion order (the anchor in the middle / at the end of the walk), sparse ids, runs of isolated nodes and a
# component without the anchor
FAMILIES = {
    "karto_shuffled": dict(seed=31, n_nodes=1500, n_loops=3000, cov_model="karto", reversed_frac=0.3, duplicate_frac=0.05,
                           order="shuffled", ids="sparse", world_rotation=0.7, isolated_runs=((0.3, 40), (0.7, 48)),
                           detached_nodes=120),
    "full_reversed": dict(seed=32, n_nodes=1200, n_loops=2400, cov_model="full", reversed_frac=0.5, duplicate_frac=0.02,
                          order="reversed", world_rotation=-2.0, isolated_runs=((0.5, 40),)),
    "iso_far": dict(seed=33, n_nodes=800, n_loops=1600, cov_model="iso", order="chain", ids="sparse", world_rotation=0.7,
                    world_translation=(1e4, -3e4)),
}
TERMINATION = {"CONVERGENCE (function tolerance)": 0, "CONVERGENCE (nothing to optimise)": 0,
               "CONVERGENCE (gradient tolerance)": 1, "CONVERGENCE (parameter tolerance)": 2,
               "NO_CONVERGENCE (max iterations)": 3, "CONVERGENCE (min trust region radius)": 4,
               "FAILURE (too many invalid steps)": 5}


@pytest.mark.parametrize("modes,kernel", [("6", 16), ("3", 13)])
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_forced_on_families(name, modes, kernel, monkeypatch):
    monkeypatch.setenv(FORCE, "1")
    monkeypatch.setenv("B200PG_COARSE_MODES", modes)
    kw = dict(FAMILIES[name])
    g = synth.make_pose_graph_family(kw.pop("seed"), **kw)
    xo, so = PG.solve(g["init"], g["ia"], g["ib"], g["z"], cov=g["cov"], fixed=g["anchor"])
    s = build(g)
    assert s.Compute()
    check_p1(s, so, xo, kernel)
    assert s.summary.termination == TERMINATION[so.termination]
    ids, xg = s.GetCorrections()
    assert np.array_equal(ids, g["ids"])
    fixed = np.zeros(len(xg), dtype=bool)
    fixed[g["anchor"]] = True
    fixed[g["component"] < 0] = True
    assert np.array_equal(xg[fixed], g["init"][fixed])   # the anchor and isolated nodes stay where they were
    assert np.all(xg[~fixed, 2] >= -math.pi) and np.all(xg[~fixed, 2] < math.pi)


@pytest.mark.parametrize("sigma", SIGMAS)
def test_forced_on_cfg4(sigma, monkeypatch):
    monkeypatch.setenv(FORCE, "1")
    g = synth.make_pose_graph(0, 10000, 40000, sigma_xy=sigma[0], sigma_th=sigma[1])
    xo, so = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"])
    s = build(g)
    assert s.Compute()
    check_p1(s, so, xo, 16)


def test_reproducible_on_fresh_handles_and_a_callers_stream():
    import torch
    g = large_graph("cfg4_15k")
    runs = []
    for stream in (None, torch.cuda.Stream()):
        s = build(g)
        if stream is not None:
            s.set_stream(stream.cuda_stream)
        assert s.Compute()
        runs.append((s.GetCorrections()[1], s.summary.pcg_iterations, s.summary.linear_solver))
    assert runs[0][2] == runs[1][2] == 16
    assert np.array_equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]


def test_incremental_constraint_on_the_solved_graph():
    g = large_graph("cfg4_15k")
    s = build(g)
    assert s.Compute() and s.summary.linear_solver == 16
    x = s.GetCorrections()[1]
    a, b = 100, 9000   # a new loop closure consistent with the solution
    ca, sa = math.cos(x[a, 2]), math.sin(x[a, 2])
    dx, dy = x[b, 0] - x[a, 0], x[b, 1] - x[a, 1]
    z = [ca * dx + sa * dy, -sa * dx + ca * dy, synth.wrap(np.array([x[b, 2] - x[a, 2]]))[0]]
    assert s.AddConstraint(int(g["ids"][a]), int(g["ids"][b]), z, np.diag([0.03 ** 2, 0.03 ** 2, 0.01 ** 2]).ravel())
    assert s.Compute()
    sm = s.summary
    assert (sm.uploaded_edges, sm.linear_solver) == (1, 16) and sm.iterations <= 2


def test_coarse_space_cuts_cg_iterations(monkeypatch):
    """Any SPD preconditioner lets CG reach pcg_tolerance, so parity alone would not notice a broken coarse space: on the
    15,000-node graph the two-level kernel must need under a third of block-Jacobi's CG iterations (5.7x fewer when
    measured on an H100)."""
    g = large_graph("cfg4_15k", SIGMAS[1])
    s = build(g)
    assert s.Compute() and s.summary.linear_solver == 16
    monkeypatch.setenv("B200PG_FORCE_GLOBAL_PCG", "1")
    s0 = build(g)
    assert s0.Compute() and s0.summary.linear_solver == 0
    assert s.summary.iterations == s0.summary.iterations
    assert 3 * s.summary.pcg_iterations < s0.summary.pcg_iterations, (s.summary.pcg_iterations, s0.summary.pcg_iterations)


@pytest.mark.parametrize("name", sorted(LARGE))
def test_plan_prints_the_coarse_size_of_the_study(name, monkeypatch, capfd):
    """tools/large_graph_study.py restates the plan's coarse-size rule to report it: it must equal what the plan prints."""
    import importlib.util
    import os
    import re
    spec = importlib.util.spec_from_file_location(
        "large_graph_study", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "large_graph_study.py"))
    study = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(study)
    monkeypatch.setenv("B200PG_DEBUG", "1")
    g = large_graph(name)
    assert planned(g) == 16
    m = re.search(r"two-level global plan: (\d+) aggregates x 6 modes \(nc = (\d+), ld = \d+\), (\d+) nodes each", capfd.readouterr().err)
    assert m, "no plan line"
    want = study.coarse_plan(*LARGE[name][:2])
    assert [int(x) for x in m.groups()] == [want["aggregates"], want["nc"], want["nodes_per_aggregate"]]
