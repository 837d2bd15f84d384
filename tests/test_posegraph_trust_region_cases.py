"""The trust-region cases of posegraph_trust_region.py show the events they are named for on the restated-Ceres
oracles, and each knob changes the oracle's outcome the way its case claims, so that the GPU comparison in
test_posegraph_trust_region_gpu.py would see a minimiser that ignored it.  No GPU."""
import numpy as np
import pytest

import posegraph_trust_region as TR
from oracle import posegraph as PG
from slam_toolbox_b200 import synth

TOL_XY = 1e-4   # the GPU tests' pose tolerance: a knob must move the poses by far more than this


def far_apart(x, y, factor=100.0):
    d = x - y
    d[:, 2] = synth.wrap(d[:, 2])
    return np.abs(d[:, :2]).max() > factor * TOL_XY


def trajectory(run):
    s = run.summary
    return s.trace, s.iterations, s.successful_steps, s.termination


@pytest.mark.parametrize("name", ["nonmono-lm", "nonmono-dogleg-traditional", "nonmono-dogleg-subspace"])
def test_nonmonotonic_steps_are_accepted(name):
    """nonmono-*: at least one accepted step leaves the cost at or above the minimum so far."""
    run = TR.oracle(TR.CASES[name])
    assert TR.nonmonotonic_steps(run.summary), run.summary.trace
    assert run.summary.usable


def test_truncated_solve_returns_an_earlier_iterate():
    """nonmono-truncated-lm: the last step is non-monotonic, so the returned poses are the iterate before it and the
    minimiser stands elsewhere when it stops."""
    assert TR.nonmonotonic_steps(TR.oracle(TR.CASES["nonmono-lm"]).summary)[0] == TR.TRUNCATE_AT
    run = TR.oracle(TR.CASES["nonmono-truncated-lm"])
    s = run.summary
    assert s.termination == "NO_CONVERGENCE (max iterations)" and s.iterations == TR.TRUNCATE_AT
    assert TR.nonmonotonic_steps(s)[-1] == TR.TRUNCATE_AT and s.trace[-1][2]
    assert s.final_cost < s.trace[-1][1]
    assert far_apart(run.x, run.x_exit)
    # the returned poses are the minimum-cost iterate: the solve stopped one iteration earlier
    prev = TR.solve(TR.graph("noisy"), dict(max_num_iterations=TR.TRUNCATE_AT - 1))
    assert np.array_equal(run.x, prev.x_exit) and prev.summary.final_cost == s.final_cost


def test_nonmonotonic_knobs_change_the_trajectory():
    """monotonic-lm, nonmono-window-*: with the evaluator monotonic or another window the trajectory differs from the
    default's (window 3), so a minimiser that held the window at 3 would be seen."""
    default = trajectory(TR.oracle(TR.CASES["nonmono-lm"]))
    runs = {n: TR.oracle(TR.CASES[n]) for n in ("monotonic-lm", "nonmono-window-1-lm", "nonmono-window-10-lm")}
    assert any(trajectory(r) != default for r in runs.values())
    assert trajectory(runs["monotonic-lm"]) != default
    for r in runs.values():
        assert r.summary.usable


@pytest.mark.parametrize("t", ["traditional", "subspace"])
def test_monotonic_evaluator_changes_the_dogleg_trajectory(t):
    """monotonic-dogleg-*: the step evaluator is shared by both strategies; under dogleg too the monotonic one takes
    another path and ends elsewhere."""
    run = TR.oracle(TR.CASES[f"monotonic-dogleg-{t}"])
    default = TR.oracle(TR.CASES[f"nonmono-dogleg-{t}"])
    assert trajectory(run) != trajectory(default) and far_apart(run.x, default.x)
    assert run.summary.usable


@pytest.mark.parametrize("name", ["radius-clamp-lm", "radius-above-max-lm"])
def test_lm_radius_clamp_binds(name):
    """radius-clamp-lm, radius-above-max-lm: an accepted step would grow the radius past max_trust_region_radius, so the
    radius after it is the maximum, and the poses differ from those of the same solve without the clamp."""
    case = TR.CASES[name]
    run = TR.oracle(case)
    cap = case.opts["max_trust_region_radius"]
    radii = [t[3] for t in run.summary.trace[1:] if t[2]]
    assert radii and all(r <= cap for r in radii) and cap in radii
    free = {k: v for k, v in case.opts.items() if k != "max_trust_region_radius"}
    unclamped = TR.solve(TR.graph(case.graph), free)
    assert max(t[3] for t in unclamped.summary.trace) > cap
    assert far_apart(run.x, unclamped.x)
    if name == "radius-above-max-lm":
        assert case.opts.get("initial_trust_region_radius", PG.Options.initial_trust_region_radius) > cap


@pytest.mark.parametrize("t", ["traditional", "subspace"])
def test_dogleg_ignores_the_radius_clamp(t):
    """radius-above-max-dogleg-*: dogleg does not clamp its radius (DESIGN.md §4), so max_trust_region_radius leaves its
    trajectory and poses unchanged, while the radius does pass the maximum."""
    case = TR.CASES[f"radius-above-max-dogleg-{t}"]
    run = TR.oracle(case)
    free = {k: v for k, v in case.opts.items() if k != "max_trust_region_radius"}
    unclamped = TR.solve(TR.graph(case.graph), free)
    assert trajectory(run) == trajectory(unclamped)
    assert np.array_equal(run.x, unclamped.x)
    assert max(tr[3] for tr in run.summary.trace) > case.opts["max_trust_region_radius"]


def test_two_dogleg_types_agree_where_they_should():
    """On the clean graph the Gauss-Newton step fits the region at every iteration, so both dogleg types take it."""
    a = TR.oracle(TR.CASES["radius-above-max-dogleg-traditional"])
    b = TR.oracle(TR.CASES["radius-above-max-dogleg-subspace"])
    assert trajectory(a) == trajectory(b)
    assert np.array_equal(a.x, b.x)


@pytest.mark.parametrize("name", ["min-radius-lm", "min-radius-dogleg-traditional", "min-radius-dogleg-subspace"])
def test_min_radius_ends_the_solve_usable(name):
    """min-radius-*: the first steps are rejected with a rising candidate cost, the radius falls to the minimum or below
    and the solve ends with CONVERGENCE (min trust region radius), usable; without the knob the same steps are taken and
    the solve goes on until another test ends it."""
    case = TR.CASES[name]
    run = TR.oracle(case)
    s = run.summary
    assert s.termination == "CONVERGENCE (min trust region radius)" and s.usable
    assert s.successful_steps == 0 and s.iterations >= 2
    assert all(not t[2] for t in s.trace[1:])
    assert all(c > s.initial_cost for c in run.cand_costs)
    assert s.trace[-1][3] <= case.opts["min_trust_region_radius"]
    free = TR.solve(TR.graph(case.graph), {k: v for k, v in case.opts.items() if k != "min_trust_region_radius"})
    assert free.summary.iterations > s.iterations and free.summary.termination != s.termination
    assert free.summary.trace[:s.iterations + 1] == s.trace


@pytest.mark.parametrize("name", [n for n in TR.CASES if n.startswith("diag-clamp")])
def test_diagonal_clamp_binds(name):
    """diag-clamp-*: min_lm_diagonal is above and max_lm_diagonal below some squared column norms of the (scaled or
    unscaled) Jacobian at the start; the clamp moves the poses, and so does a clamp with its bounds swapped (every
    column at the lower bound)."""
    case = TR.CASES[name]
    g = TR.graph(case.graph)
    unscaled, jacobi = TR.lm_diagonal(g)
    d = jacobi if case.opts.get("jacobi_scaling", 1) else unscaled
    lo, hi = case.opts["min_lm_diagonal"], case.opts["max_lm_diagonal"]
    assert (d < lo).any() and (d > hi).any() and ((d > lo) & (d < hi)).any()
    run = TR.oracle(case)
    assert run.summary.usable and run.summary.successful_steps > 0
    base = {k: v for k, v in case.opts.items() if k not in ("min_lm_diagonal", "max_lm_diagonal")}
    assert far_apart(run.x, TR.solve(g, base).x, factor=10.0)
    assert far_apart(run.x, TR.solve(g, dict(base, min_lm_diagonal=lo, max_lm_diagonal=lo)).x, factor=10.0)


@pytest.mark.parametrize("name", [n for n in TR.CASES if n.startswith("jacobi-off")])
def test_jacobi_off_changes_the_trajectory(name):
    """jacobi-off-*: without Jacobi scaling the LM diagonal and the dogleg metric are the unscaled column norms, so the
    poses differ from the scaled solve's."""
    case = TR.CASES[name]
    run = TR.oracle(case)
    assert run.summary.usable
    scaled = TR.solve(TR.graph(case.graph), {k: v for k, v in case.opts.items() if k != "jacobi_scaling"})
    assert trajectory(run) != trajectory(scaled) or far_apart(run.x, scaled.x, factor=1.0)


@pytest.mark.parametrize("name", [n for n in TR.CASES if n.startswith("invalid")])
def test_singular_system_ends_in_failure(name):
    """invalid-*: every linear solve meets the zero pivot, so every step is invalid and the solve ends with FAILURE after
    max_num_consecutive_invalid_steps of them (dogleg retries each solve at 10x mu until mu reaches 1), not usable,
    returning the start.  With the default options the same graph solves."""
    case = TR.CASES[name]
    run = TR.oracle(case)
    s = run.summary
    k = case.opts["max_num_consecutive_invalid_steps"]
    assert s.termination == "FAILURE (too many invalid steps)" and not s.usable
    assert (s.iterations, s.successful_steps) == (k, 0) and run.cand_costs == []
    assert np.array_equal(run.x, TR.graph(case.graph)["init"])
    assert s.linear_solves == (k if name.endswith("-lm") else 8)
    assert TR.solve(TR.graph(case.graph), {}).summary.usable


@pytest.mark.parametrize("name", ["invalid-1-lm", "invalid-3-dogleg-subspace"])
def test_singular_system_fails_after_a_solve(name):
    """The GPU's failed-solve contract test starts from a solved graph: its anchored component solved at the defaults,
    then the anchorless one added on the x axis.  From there the zero pivot stays exact, so the case still fails, and
    the default options still solve it."""
    case = TR.CASES[name]
    g = TR.graph(case.graph)
    head, _ = PG.solve(g["init"][:2], g["ia"][:1], g["ib"][:1], g["z"][:1], cov=g["cov"][:1])
    state = np.concatenate([head, g["init"][2:]])
    run = TR.solve(g, case.opts, init=state)
    assert run.summary.termination == "FAILURE (too many invalid steps)" and not run.summary.usable
    assert run.summary.iterations == case.opts["max_num_consecutive_invalid_steps"]
    assert TR.solve(g, {}, init=state).summary.usable


def test_zero_tolerances_converge_before_three_invalid_steps():
    """The rounding route to an invalid step (a model cost change that is not positive) does not end these solves: with
    all three tolerances at 0 the oracle ends at the exact function or parameter tolerance, never with non-positive model
    changes in a row."""
    zero = dict(function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0, max_num_iterations=300)
    for seed, n, e in ((0, 60, 120), (1, 200, 500), (2, 500, 1400)):
        g = synth.make_pose_graph(seed, n, e, sigma_xy=0.03, sigma_th=0.01)
        for invalid in (1, 3):
            _, s = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"],
                            opts=PG.Options(max_num_consecutive_invalid_steps=invalid, **zero))
            assert s.usable and s.termination in ("CONVERGENCE (function tolerance)", "CONVERGENCE (parameter tolerance)")
            assert s.iterations < 300


def test_overflowing_costs_need_covariances_the_solver_refuses():
    """Scaling every U by one factor s scales every cost by s^2 and keeps the LM trajectory.  On the swung chain an
    overflowing candidate from a finite start needs s^2 above 1e302; the covariance of such an edge has a determinant far
    below 1e-14, which AddConstraint refuses (Matrix3::Inverse), so no uniform scaling of this graph reaches a non-finite
    candidate cost through the public API.  (A determinant bound does not bound single entries: an anisotropic
    covariance can still carry a very large information entry.)"""
    g = TR.graph("swung")
    run = TR.solve(g, {})
    need = np.finfo(np.float64).max / (2.0 * max(run.cand_costs))
    assert need > 1e302
    cov = g["cov"][0] / need
    with pytest.raises(np.linalg.LinAlgError):
        PG.sqrt_information(cov)
    # the largest uniform scale AddConstraint accepts leaves every cost many decades below overflow
    s2 = min((np.linalg.det(c) / 1e-14) ** (1.0 / 3.0) for c in g["cov"])
    assert s2 * max(run.cand_costs) < 1e20
