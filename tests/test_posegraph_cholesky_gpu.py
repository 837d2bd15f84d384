"""The exact linear solver of the CUDA pose-graph solver (linear_solver_type = 1, block-sparse supernodal Cholesky) against
the exact-solve oracles (oracle/posegraph.py for LM, tests/posegraph_dogleg.py for both dogleg types): the same
iterations, accepted steps and linear solves, final cost and poses, robust losses, tiny and singular graphs,
bit-reproducibility, switching solvers on a live handle and the reuse of the host analysis."""
import json

import numpy as np
import pytest

import posegraph_dogleg as DL
from slam_toolbox_b200 import api, synth
from test_posegraph_dogleg_gpu import build, diff
from test_posegraph_shapes_gpu import family

pytestmark = pytest.mark.gpu
TOL_XY, TOL_TH = 1e-4, 1e-5
STRATEGIES = {"lm": dict(trust_region_strategy=0), "traditional": dict(trust_region_strategy=1, dogleg_type=0),
              "subspace": dict(trust_region_strategy=1, dogleg_type=1)}
CHOL = dict(linear_solver_type=1)


def oracle(g, t, ia="edge_a", ib="edge_b", fixed=0, init=None, **opts):
    o = DL.Options(trust_region_strategy="lm", **opts) if t == "lm" else \
        DL.Options(trust_region_strategy="dogleg", dogleg_type=t, **opts)
    return DL.solve(g["init"] if init is None else init, g[ia], g[ib], g["z"], cov=g["cov"], fixed=fixed, opts=o)


def check_p1(s, so, xg, xo):
    sm = s.summary
    assert (sm.linear_solver, sm.pcg_iterations) == (8, 0)
    assert (sm.iterations, sm.successful_steps, sm.linear_solves) == (so.iterations, so.successful_steps, so.linear_solves), \
        ((sm.iterations, sm.successful_steps, sm.linear_solves), (so.iterations, so.successful_steps, so.linear_solves))
    assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (sm.final_cost, so.final_cost)
    dxy, dth = diff(xg, xo)
    assert dxy < TOL_XY and dth < TOL_TH, (dxy, dth)
    return dxy, dth


@pytest.mark.parametrize("t", sorted(STRATEGIES))
@pytest.mark.parametrize("n,e,seed", [(60, 120, 0), (500, 1400, 1), (3000, 9000, 2)])
def test_p1_matches_oracle(n, e, seed, t):
    g = synth.make_pose_graph(seed, n, e, sigma_xy=0.03, sigma_th=0.01)
    xo, so = oracle(g, t)
    s = build(g, **STRATEGIES[t], **CHOL)
    assert s.Compute()
    ids, xg = s.GetCorrections()
    assert np.array_equal(ids, g["ids"])
    check_p1(s, so, xg, xo)
    assert np.array_equal(xg[0], g["init"][0])   # the anchor is untouched
    info = s.factor_info()
    assert info["columns"] == n - 1 and info["analyses"] == 1


@pytest.mark.parametrize("t", sorted(STRATEGIES))
@pytest.mark.parametrize("sigma", [(0.03, 0.01), (0.05, 0.02)])
def test_p1_cfg4(sigma, t):
    g = synth.make_pose_graph(0, 10000, 40000, sigma_xy=sigma[0], sigma_th=sigma[1])
    xo, so = oracle(g, t)
    s = build(g, **STRATEGIES[t], **CHOL)
    assert s.Compute()
    xg = s.GetCorrections()[1]
    dxy, dth = check_p1(s, so, xg, xo)
    print(f"cfg4 sigma {sigma} {t}: {dxy:.2e} m / {dth:.2e} rad, cost rel "
          f"{abs(s.summary.final_cost - so.final_cost) / so.final_cost:.2e}")
    assert np.array_equal(xg[0], g["init"][0])


@pytest.mark.parametrize("t", ["traditional", "subspace"])
def test_karto_shuffled_dogleg(t):
    """The graph on which block-Jacobi PCG ends 4.1e-4 m from the exact-solve oracle under dogleg."""
    g = family("karto_shuffled")
    xo, so = oracle(g, t, ia="ia", ib="ib", fixed=g["anchor"])
    s = build(g, **STRATEGIES[t], **CHOL)
    assert s.Compute()
    xg = s.GetCorrections()[1]
    check_p1(s, so, xg, xo)
    isolated = g["component"] < 0
    assert np.array_equal(xg[isolated], g["init"][isolated])
    assert np.array_equal(xg[g["anchor"]], g["init"][g["anchor"]])


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_p2_tight_tolerances(t):
    g = synth.make_pose_graph(5, 400, 1100, sigma_xy=0.03, sigma_th=0.01)
    kw = dict(function_tolerance=1e-14, parameter_tolerance=1e-13, gradient_tolerance=1e-13, max_num_iterations=100)
    xo, so = oracle(g, t, **kw)
    s = build(g, **STRATEGIES[t], **CHOL, **kw)
    assert s.Compute()
    dxy, dth = diff(s.GetCorrections()[1], xo)
    print(f"P2 {t}: {dxy:.2e} m / {dth:.2e} rad")
    assert dxy < 1e-8 and dth < 1e-8, (dxy, dth)


@pytest.mark.parametrize("t", sorted(STRATEGIES))
@pytest.mark.parametrize("loss,code", [("huber", 1), ("cauchy", 2)])
def test_robust_losses_with_outliers(loss, code, t):
    g = synth.make_pose_graph(21, 2500, 9000, sigma_xy=0.03, sigma_th=0.01)
    rng = np.random.default_rng(0)
    z = g["z"].copy()
    loops = np.arange(2499, len(z))
    bad = rng.choice(loops, size=max(4, len(loops) // 50), replace=False)
    z[bad, :2] += rng.normal(0, 2.0, (len(bad), 2))
    g = dict(g, z=z)
    xo, so = oracle(g, t, loss_function=loss)
    s = build(g, **STRATEGIES[t], **CHOL, loss_function=code, loss_scale=0.7)
    assert s.Compute()
    check_p1(s, so, s.GetCorrections()[1], xo)


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_tiny_and_degenerate_graphs(t):
    cov = np.diag([0.01, 0.01, 0.001])
    # one edge; a triangle; two components (the second without the anchor) with isolated nodes between them
    cases = [(2, [(0, 1)], []), (3, [(0, 1), (1, 2), (0, 2)], []), (7, [(0, 1), (1, 2), (4, 5), (5, 6), (4, 6)], [3])]
    for n, edges, isolated in cases:
        poses = np.array([[0, 0, 0], [1.05, 0.1, 0.05], [2.1, -0.05, -0.02], [9.0, 9.0, 0.3], [4.0, 0.0, 0.1],
                          [5.1, 0.2, 0.15], [6.0, -0.1, 0.05]])[:n]
        ea, eb = np.array([a for a, _ in edges]), np.array([b for _, b in edges])
        z = np.array([[float(b - a), 0.0, 0.0] for a, b in edges])
        g = dict(init=poses, edge_a=ea, edge_b=eb, z=z, cov=np.repeat(cov[None], len(edges), axis=0), ids=np.arange(n))
        xo, so = oracle(g, t)
        s = build(g, **STRATEGIES[t], **CHOL)
        assert s.Compute()
        assert (s.summary.iterations, s.summary.linear_solves) == (so.iterations, so.linear_solves), n
        x = s.GetCorrections()[1]
        dxy, dth = diff(x, xo)
        assert dxy < TOL_XY and dth < TOL_TH, (n, dxy, dth)
        assert np.array_equal(x[0], poses[0]) and np.array_equal(x[isolated], poses[isolated])
    # no free node: no edge at all, then an edge whose free end is removed again
    s = api.ScanSolver(**STRATEGIES[t], **CHOL)
    s.AddNode(0, np.zeros(3))
    s.AddNode(1, np.array([1.0, 0.0, 0.0]))
    assert s.Compute() and s.summary.iterations == 0
    assert s.AddConstraint(0, 1, np.array([1.0, 0.1, 0.0]), cov)
    assert s.RemoveNode(1)
    assert s.Compute() and s.summary.iterations == 0
    assert np.array_equal(s.GetCorrections()[1], np.zeros((1, 3)))


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_singular_system_ends_cleanly(t):
    """A component without the anchor and no LM diagonal: (H + shift D^2) is singular. The solve must end without a fault,
    either usable with finite poses or B200_ERR_NUMERIC with the node store untouched, never with NaN poses."""
    g = synth.make_pose_graph(3, 200, 500, sigma_xy=0.03, sigma_th=0.01)
    h = synth.make_pose_graph(4, 100, 220, sigma_xy=0.03, sigma_th=0.01)
    init = np.concatenate([g["init"], h["init"] + np.array([50.0, 0.0, 0.0])])
    ea = np.concatenate([g["edge_a"], h["edge_a"] + 200])
    eb = np.concatenate([g["edge_b"], h["edge_b"] + 200])
    gg = dict(init=init, ids=np.arange(300), edge_a=ea, edge_b=eb, z=np.concatenate([g["z"], h["z"]]),
              cov=np.concatenate([g["cov"], h["cov"]]))
    s = build(gg, **STRATEGIES[t], **CHOL, min_lm_diagonal=0.0, max_lm_diagonal=0.0)
    ok = s.Compute()
    x = np.array([s.get_node(i) for i in range(300)])
    assert np.all(np.isfinite(x))
    if not ok:
        assert np.array_equal(x, init)
    assert s.summary.linear_solver == 8


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_two_solves_are_bit_identical(t):
    import torch
    g = synth.make_pose_graph(11, 1500, 4500, sigma_xy=0.05, sigma_th=0.02)
    s1 = build(g, **STRATEGIES[t], **CHOL)
    s2 = build(g, **STRATEGIES[t], **CHOL)
    stream = torch.cuda.Stream()
    s2.set_stream(stream.cuda_stream)
    assert s1.Compute() and s2.Compute()
    assert np.array_equal(s1.GetCorrections()[1], s2.GetCorrections()[1])
    a, b = s1.summary, s2.summary
    assert (a.iterations, a.successful_steps, a.linear_solves, a.final_cost) == \
        (b.iterations, b.successful_steps, b.linear_solves, b.final_cost)


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_zero_pivot_is_a_failed_linear_solve(t):
    """A component without the anchor whose block matrix is exactly singular: one edge with identity information between
    poses on the x axis, no Jacobi scaling, no LM diagonal. Every product is exact, so the last pivot is exactly zero. LM
    counts each step invalid, dogleg retries at 10x mu until mu reaches 1, and both end as the oracles do (whose SuperLU
    raises): no usable solution, B200_ERR_NUMERIC, the node store untouched."""
    poses = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [5.0, 0.0, 0.0], [6.0, 0.0, 0.0]])
    z = np.array([[0.9, 0.1, 0.05], [0.9, 0.1, 0.05]])
    g = dict(init=poses, ids=np.arange(4), edge_a=np.array([0, 2]), edge_b=np.array([1, 3]), z=z,
             cov=np.repeat(np.eye(3)[None], 2, axis=0))
    kw = dict(min_lm_diagonal=0.0, max_lm_diagonal=0.0)
    xo, so = oracle(g, t, jacobi_scaling=False, **kw)
    assert not so.usable
    s = build(g, **STRATEGIES[t], **CHOL, jacobi_scaling=0, **kw)
    assert not s.Compute()
    sm = s.summary
    assert (sm.linear_solver, sm.usable, sm.termination) == (8, 0, 5)
    assert (sm.iterations, sm.successful_steps, sm.linear_solves) == (so.iterations, so.successful_steps, so.linear_solves), \
        ((sm.iterations, sm.successful_steps, sm.linear_solves), (so.iterations, so.successful_steps, so.linear_solves))
    assert np.array_equal(np.array([s.get_node(i) for i in range(4)]), poses)


def test_set_opts_refuses_other_linear_solvers_on_a_live_handle():
    L = api.lib()
    s = api.ScanSolver(**CHOL)
    for value in (2, -1):
        bad = api.PgOpts()
        assert L.b200pg_get_opts(s._h, api.C.byref(bad)) == 0
        bad.linear_solver_type = value
        assert L.b200pg_set_opts(s._h, api.C.byref(bad)) == api.ERR_INVALID_ARG
    o = api.PgOpts()
    assert L.b200pg_get_opts(s._h, api.C.byref(o)) == 0 and o.linear_solver_type == 1


def test_binding_key_selects_the_linear_solver():
    """integration/b200_solver.hpp: b200_linear_solver = PCG / SPARSE_NORMAL_CHOLESKY sets linear_solver_type; an unknown value
    is reported and leaves it; ceres_linear_solver keeps its meaning (accepted, no change of solver)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "integration"))
    import replay
    if not replay.available():
        pytest.skip("oracle/_ref/libreplay_*.so not built")
    code = f"""
import ctypes as C, json, math
L = C.CDLL({replay.library("b200")!r})
L.krep_create.restype = C.c_void_p
L.krep_create.argtypes = [C.c_int]
L.krep_init_laser.argtypes = [C.c_double] * 6
L.krep_solver_configure.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
L.krep_solver_linear_solver_type.argtypes = [C.c_void_p]
L.krep_destroy.argtypes = [C.c_void_p]
L.krep_init_laser(math.radians(-135), math.radians(135), math.radians(0.25), 0.1, 30.0, 12.0)
h = L.krep_create(1)
out = [L.krep_solver_linear_solver_type(h)]
for k, v in (("b200_linear_solver", "SPARSE_NORMAL_CHOLESKY"), ("b200_linear_solver", "Bogus"), ("ceres_linear_solver", "CGNR"),
             ("b200_linear_solver", "PCG"), ("ceres_linear_solver", "SPARSE_NORMAL_CHOLESKY")):
    out.append([L.krep_solver_configure(h, k.encode(), v.encode()), L.krep_solver_linear_solver_type(h)])
L.krep_destroy(h)
print(json.dumps(out))
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "unknown b200_linear_solver 'Bogus'" in r.stderr
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out == [0, [1, 1], [0, 1], [1, 1], [1, 0], [1, 0]], out


def test_switching_solvers_on_a_live_handle():
    L = api.lib()
    g = synth.make_pose_graph(8, 1500, 4200, sigma_xy=0.03, sigma_th=0.01)
    s = build(g)
    o = api.PgOpts()
    assert L.b200pg_get_opts(s._h, api.C.byref(o)) == 0
    o.linear_solver_type = 1
    assert L.b200pg_set_opts(s._h, api.C.byref(o)) == 0
    o.linear_solver_type = 0
    assert L.b200pg_set_opts(s._h, api.C.byref(o)) == 0
    assert s.Compute()
    never = build(g)
    assert never.Compute()
    assert np.array_equal(s.GetCorrections()[1], never.GetCorrections()[1])
    assert s.summary.linear_solver != 8 and s.summary.pcg_iterations == never.summary.pcg_iterations
    # then Cholesky on the same handle (which now holds PCG's solution) matches a fresh Cholesky handle on that state
    state = s.GetCorrections()[1].copy()
    o.linear_solver_type = 1
    assert L.b200pg_set_opts(s._h, api.C.byref(o)) == 0
    assert s.Compute() and s.summary.linear_solver == 8
    f = build(dict(g, init=state), **CHOL)
    assert f.Compute()
    assert np.array_equal(s.GetCorrections()[1], f.GetCorrections()[1])
    assert (s.summary.iterations, s.summary.linear_solves) == (f.summary.iterations, f.summary.linear_solves)


def test_analysis_reuse():
    g = synth.make_pose_graph(9, 1200, 3300, sigma_xy=0.03, sigma_th=0.01)
    s = build(g, **CHOL)
    assert s.factor_info()["analyses"] == 0 and s.factor_info()["columns"] == 0
    assert s.Compute()
    first = s.factor_info()
    assert first["analyses"] == 1 and first["columns"] == 1199
    assert s.Compute()                                            # nothing changed
    assert s.factor_info() == first
    a, b = int(g["edge_a"][-1]), int(g["edge_b"][-1])             # a second constraint between adjacent nodes
    assert s.AddConstraint(a, b, g["z"][-1], g["cov"][-1])
    state = s.GetCorrections()[1].copy()
    assert s.Compute()
    assert s.factor_info()["analyses"] == 1
    # bit-identical to a fresh handle given the nodes at their solved poses and the same constraints in the same order
    f = api.ScanSolver(**CHOL)
    for nid, p in zip(g["ids"], state):
        f.AddNode(int(nid), p)
    for k in range(len(g["z"])):
        assert f.AddConstraint(int(g["edge_a"][k]), int(g["edge_b"][k]), g["z"][k], g["cov"][k])
    assert f.AddConstraint(a, b, g["z"][-1], g["cov"][-1])
    assert f.Compute()
    assert np.array_equal(s.GetCorrections()[1], f.GetCorrections()[1])
    assert f.factor_info()["nnz_blocks"] == first["nnz_blocks"]
    # a constraint joining a new pair
    assert s.AddConstraint(5, 900, np.array([0.0, 0.0, 0.0]), np.diag([1.0, 1.0, 0.1]))
    assert s.Compute() and s.factor_info()["analyses"] == 2
    # a removal
    assert s.RemoveNode(1100)
    assert s.Compute() and s.factor_info()["analyses"] == 3
    assert s.factor_info()["columns"] == 1198
    # Reset, then the same graph again
    s.Reset()
    for nid, p in zip(g["ids"], g["init"]):
        s.AddNode(int(nid), p)
    for k in range(len(g["z"])):
        assert s.AddConstraint(int(g["edge_a"][k]), int(g["edge_b"][k]), g["z"][k], g["cov"][k])
    assert s.Compute() and s.factor_info()["analyses"] == 4
    assert {k: v for k, v in s.factor_info().items() if k != "analyses"} == \
        {k: v for k, v in first.items() if k != "analyses"}
