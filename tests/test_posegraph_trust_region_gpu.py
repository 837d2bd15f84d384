"""The CUDA pose-graph minimiser against the restated-Ceres oracles under the trust-region knobs of
posegraph_trust_region.py: non-monotonic steps and the minimum-cost iterate, the monotonic evaluator, the LM radius
clamp, the minimum radius, the diagonal clamp, Jacobi scaling off under each PCG kernel and both dogleg types, and a
singular system ending in FAILURE; a failed solve leaving the handle as it was; options changed on a live handle; and
two solves of each case bit-identical."""
import numpy as np
import pytest

import posegraph_trust_region as TR
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
TOL_XY, TOL_TH = 1e-4, 1e-5
TERMINATION = {"CONVERGENCE (function tolerance)": 0, "CONVERGENCE (gradient tolerance)": 1,
               "CONVERGENCE (parameter tolerance)": 2, "NO_CONVERGENCE (max iterations)": 3,
               "CONVERGENCE (min trust region radius)": 4, "FAILURE (too many invalid steps)": 5}


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


def check(s, run, g):
    """Same iterations, accepted steps and termination as the oracle, final cost at P1's relative tolerance, poses within
    the pose-graph suites' tolerances.  For a case that fails: the same iterations, accepted steps and linear solves, and
    nothing published."""
    sm, so = s.summary, run.summary
    assert (sm.iterations, sm.successful_steps, sm.termination) == (so.iterations, so.successful_steps, TERMINATION[so.termination]), \
        ((sm.iterations, sm.successful_steps, sm.termination), (so.iterations, so.successful_steps, so.termination))
    if not so.usable:
        assert sm.usable == 0 and sm.linear_solves == so.linear_solves, (sm.linear_solves, so.linear_solves)
        return None
    assert sm.usable == 1
    assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (sm.final_cost, so.final_cost)
    ids, xg = s.GetCorrections()
    assert np.array_equal(ids, g["ids"])
    dxy, dth = diff(xg, run.x)
    assert dxy < TOL_XY and dth < TOL_TH, (dxy, dth)
    return xg


@pytest.mark.parametrize("name", sorted(TR.CASES))
def test_case_matches_oracle(name, monkeypatch):
    case = TR.CASES[name]
    if case.kernel is not None:
        for k, v in TR.KERNEL_ENV[case.kernel].items():
            monkeypatch.setenv(k, v)
    g = TR.graph(case.graph)
    run = TR.oracle(case)
    s1 = build(g, **case.opts)
    assert s1.Compute() == run.summary.usable
    if case.kernel is not None:
        assert s1.summary.linear_solver == case.kernel
    if case.opts.get("linear_solver_type") == 1:
        assert s1.summary.linear_solver == 8
    check(s1, run, g)
    x1 = s1.GetCorrections()[1]
    # a second solve of the same case on a fresh handle is bit-identical (fixed-order sums, no atomics)
    s2 = build(g, **case.opts)
    assert s2.Compute() == run.summary.usable
    assert np.array_equal(s2.GetCorrections()[1], x1)
    a, b = s1.summary, s2.summary
    assert (a.iterations, a.successful_steps, a.termination, a.pcg_iterations, a.linear_solves, a.final_cost) == \
        (b.iterations, b.successful_steps, b.termination, b.pcg_iterations, b.linear_solves, b.final_cost)


def test_truncated_solve_returns_the_minimum_cost_iterate():
    """The solve stops right after a non-monotonic step: the poses returned are the oracle's minimum-cost iterate (the
    one before that step), which lies measurably away from the iterate the minimiser stopped at."""
    case = TR.CASES["nonmono-truncated-lm"]
    g = TR.graph(case.graph)
    run = TR.oracle(case)
    s = build(g, **case.opts)
    assert s.Compute()
    xg = check(s, run, g)
    dxy, _ = diff(xg, run.x_exit)
    assert dxy > 100 * TOL_XY, dxy
    assert s.summary.final_cost < run.summary.trace[-1][1]


@pytest.mark.parametrize("name", ["min-radius-lm", "min-radius-dogleg-traditional", "min-radius-dogleg-subspace"])
def test_min_radius_is_usable(name):
    """Termination 4 is a convergence: Compute succeeds and publishes the minimum-cost iterate (here the start)."""
    case = TR.CASES[name]
    g = TR.graph(case.graph)
    s = build(g, **case.opts)
    assert s.Compute() and s.summary.termination == 4 and s.summary.usable == 1
    ids, xg = s.GetCorrections()
    assert np.array_equal(xg, g["init"])


@pytest.mark.parametrize("name", [n for n in TR.CASES if n.startswith("invalid")])
def test_failed_solve_leaves_the_handle_as_it_was(name):
    """b200pg_solve's FAILURE contract on a live handle: the anchored component is solved at the defaults, the anchorless
    one is added, and the case's options make every linear solve meet a zero pivot.  Compute returns False with
    termination 5 and usable 0 after max_num_consecutive_invalid_steps invalid steps, as the oracle from the same state
    ends; the corrections and the node store are bit-identical to what they were before the call; back at the defaults
    the same handle solves."""
    case = TR.CASES[name]
    g = TR.graph(case.graph)
    s = api.ScanSolver()
    for i in (0, 1):
        s.AddNode(i, g["init"][i])
    assert s.AddConstraint(0, 1, g["z"][0], g["cov"][0])
    assert s.Compute()
    for i in (2, 3):
        s.AddNode(i, g["init"][i])
    assert s.AddConstraint(2, 3, g["z"][1], g["cov"][1])
    ids0, corr0 = (a.copy() for a in s.GetCorrections())
    graph0 = s.getGraph()
    assert len(ids0) == 2 and sorted(graph0) == [0, 1, 2, 3]
    state = np.array([graph0[i] for i in range(4)])
    run = TR.solve(g, case.opts, init=state)
    assert run.summary.termination == "FAILURE (too many invalid steps)"
    s.SetOptions(**case.opts)
    assert not s.Compute()
    sm = s.summary
    assert (sm.termination, sm.usable, sm.linear_solver) == (5, 0, 8)
    assert (sm.iterations, sm.successful_steps, sm.linear_solves) == \
        (run.summary.iterations, run.summary.successful_steps, run.summary.linear_solves)
    ids1, corr1 = s.GetCorrections()
    assert np.array_equal(ids1, ids0) and np.array_equal(corr1, corr0)
    graph1 = s.getGraph()
    assert sorted(graph1) == sorted(graph0) and all(np.array_equal(graph1[i], graph0[i]) for i in graph0)
    s.SetOptions()
    assert s.Compute() and s.summary.termination != 5 and s.summary.usable == 1
    ids2, corr2 = s.GetCorrections()
    assert sorted(ids2) == [0, 1, 2, 3] and np.all(np.isfinite(corr2))


def test_options_round_trip():
    """SetOptions takes the constructor's keywords over the defaults, and b200pg_get_opts gives them back; an unknown
    key raises KeyError and an invalid value raises the library's INVALID_ARG, both leaving the options as they were."""
    s = api.ScanSolver()
    want = dict(max_num_iterations=7, max_trust_region_radius=3.0, min_trust_region_radius=1e-9, min_lm_diagonal=0.5,
                max_lm_diagonal=2.0, jacobi_scaling=0, use_nonmonotonic_steps=0, max_consecutive_nonmonotonic_steps=9,
                max_num_consecutive_invalid_steps=1, trust_region_strategy=1, dogleg_type=1)
    s.SetOptions(**want)
    got = s.GetOptions()
    for k, v in want.items():
        assert getattr(got, k) == v, k
    default = api.PgOpts()
    api.lib().b200pg_default_opts(api.C.byref(default))
    assert got.function_tolerance == default.function_tolerance   # keys not given are the defaults
    with pytest.raises(KeyError):
        s.SetOptions(no_such_option=1)
    with pytest.raises(api.B200Error) as e:
        s.SetOptions(trust_region_strategy=2)
    assert e.value.code == api.ERR_INVALID_ARG
    after = s.GetOptions()
    assert all(getattr(after, k) == getattr(got, k) for k, _ in api.PgOpts._fields_)
    s.SetOptions()
    back = s.GetOptions()
    assert all(getattr(back, k) == getattr(default, k) for k, _ in api.PgOpts._fields_)


@pytest.mark.parametrize("name", ["diag-clamp-lm", "monotonic-lm", "radius-above-max-dogleg-subspace"])
def test_knobs_set_on_a_live_handle(name):
    """Solve at the defaults, set the case's options on the same handle and solve again: the second solve is the oracle's
    under those options from the first solve's output, and no constraint travels again."""
    case = TR.CASES[name]
    g = TR.graph(case.graph)
    s = build(g)
    assert s.Compute()
    first = s.GetCorrections()[1].copy()
    s.SetOptions(**case.opts)
    assert s.Compute() and s.summary.uploaded_edges == 0
    run = TR.solve(g, case.opts, init=first)
    check(s, run, g)


def test_get_graph_follows_the_node_store():
    """getGraph gives every stored node's pose by id: a repeated AddNode keeps the first pose, RemoveNode and Reset
    take nodes out."""
    s = api.ScanSolver()
    assert s.getGraph() == {}
    s.AddNode(7, [1.0, 2.0, 0.5])
    s.AddNode(-3, [0.0, 0.0, 0.0])
    s.AddNode(7, [9.0, 9.0, 9.0])
    s.AddNode(12, [4.0, 5.0, -0.25])
    gr = s.getGraph()
    assert sorted(gr) == [-3, 7, 12] and np.array_equal(gr[7], [1.0, 2.0, 0.5]) and np.array_equal(gr[12], [4.0, 5.0, -0.25])
    assert s.RemoveNode(-3) and not s.RemoveNode(-3)
    assert sorted(s.getGraph()) == [7, 12]
    s.Reset()
    assert s.getGraph() == {}
