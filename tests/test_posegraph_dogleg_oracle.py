"""Checks of the dogleg oracle (tests/posegraph_dogleg.py; PARITY UNPINNED like oracle/posegraph.py): the traditional
step in each of its cases, the subspace boundary minimiser against brute force, its rank-1 and fallback branches, both
dogleg types reaching the scipy.optimize.least_squares minimiser, the LM default unchanged, and the new option fields
through the C ABI."""
import ctypes as C

import numpy as np
import pytest
from scipy.optimize import least_squares

import posegraph_dogleg as DL
from oracle import posegraph as PG
from slam_toolbox_b200 import api, synth
from test_posegraph_oracle import shaped_graph


def dense_problem(seed, m=30, n=8):
    """A small dense least-squares model: scaled gradient, Gauss-Newton step and Cauchy factor as DoglegStrategy forms them."""
    rng = np.random.default_rng(seed)
    J = rng.normal(size=(m, n)) * np.exp(rng.normal(size=n))
    r = rng.normal(size=m)
    D = np.sqrt(np.clip((J * J).sum(axis=0), 1e-6, 1e32))
    g_s = (J.T @ r) / D
    Jg = J @ (g_s / D)
    alpha = (g_s @ g_s) / (Jg @ Jg)
    y = np.linalg.solve(J.T @ J + 1e-8 * np.diag(D * D), J.T @ r)
    return J, r, D, g_s, -D * y, alpha


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_traditional_step_cases(seed):
    J, r, D, g_s, gn_s, alpha = dense_problem(seed)
    gn_norm, g_norm = np.linalg.norm(gn_s), np.linalg.norm(g_s)
    cauchy = alpha * g_norm
    assert cauchy < gn_norm      # the Cauchy point lies inside the Gauss-Newton step's sphere
    # 1. Gauss-Newton step inside the region: returned as it is
    s, n = DL.traditional_step(g_s, gn_s, alpha, 1.5 * gn_norm)
    assert np.array_equal(s, gn_s) and n == gn_norm
    # 2. the Cauchy point outside: the scaled steepest-descent step on the boundary
    radius = 0.5 * cauchy
    s, n = DL.traditional_step(g_s, gn_s, alpha, radius)
    assert abs(np.linalg.norm(s) - radius) <= 1e-12 * radius and n == radius
    assert np.allclose(s / np.linalg.norm(s), -g_s / g_norm, rtol=0, atol=1e-14)
    # 3. between: the dogleg segment from -alpha g_s to gn_s meets the boundary
    for radius in (1.01 * cauchy, 0.5 * (cauchy + gn_norm), 0.99 * gn_norm):
        s, n = DL.traditional_step(g_s, gn_s, alpha, radius)
        assert abs(np.linalg.norm(s) - radius) <= 1e-12 * radius and abs(n - radius) <= 1e-12 * radius
        a = -alpha * g_s
        beta = (s - a) @ (gn_s - a) / ((gn_s - a) @ (gn_s - a))
        assert 0.0 < beta < 1.0
        assert np.allclose(s, a + beta * (gn_s - a), rtol=0, atol=1e-12 * radius)
    # the model decreases along the way: the dogleg step beats the Cauchy step of the same length
    def model(step_s):
        step = step_s / D
        return 0.5 * (J @ step) @ (J @ step) + (J.T @ r) @ step
    radius = 0.5 * (cauchy + gn_norm)
    assert model(DL.traditional_step(g_s, gn_s, alpha, radius)[0]) < model(-(radius / g_norm) * g_s)


def test_boundary_minimum_against_brute_force():
    rng = np.random.default_rng(3)
    th = np.linspace(0.0, 2.0 * np.pi, 200001)
    circle = np.stack([np.cos(th), np.sin(th)], 1)
    checked = 0
    while checked < 200:
        A = rng.normal(size=(2, 2))
        B = A @ A.T * 10 ** rng.uniform(-2, 2)           # random PSD model
        g = rng.normal(size=2) * 10 ** rng.uniform(-2, 2)
        r = 10 ** rng.uniform(-2, 1)
        if np.linalg.norm(np.linalg.solve(B, g)) <= r:   # the unconstrained minimum is inside: not a boundary problem
            continue
        x = DL.boundary_minimum(g, B, r)
        assert x is not None
        assert abs(np.linalg.norm(x) - r) <= 1e-12 * r
        P = r * circle
        f = 0.5 * np.einsum("ni,ij,nj->n", P, B, P) + P @ g
        fx = 0.5 * x @ B @ x + g @ x
        assert fx <= f.min() + 1e-12 * np.abs(f).max()
        assert np.linalg.norm(x - P[np.argmin(f)]) <= 1e-4 * r
        checked += 1


def test_subspace_rank_one_branch():
    g_s = np.array([3.0, 4.0, 0.0, 0.0])
    gn_s = -2.5 * g_s                                    # parallel to the gradient: the subspace is one-dimensional
    basis, rank1 = DL.subspace_basis(g_s, gn_s)
    assert rank1 and basis.shape == (4, 1)
    radius = 2.0
    s, n = DL.subspace_step(g_s, gn_s, 0.3, radius, basis, rank1, None, None)
    assert np.allclose(s, -(radius / 5.0) * g_s, rtol=0, atol=1e-15) and n == radius
    # inside the region the Gauss-Newton step is taken whatever the rank
    s, n = DL.subspace_step(g_s, gn_s, 0.3, 20.0, basis, rank1, None, None)
    assert np.array_equal(s, gn_s)


def test_subspace_step_on_the_boundary_and_its_fallback():
    J, r, D, g_s, gn_s, alpha = dense_problem(4)
    basis, rank1 = DL.subspace_basis(g_s, gn_s)
    assert not rank1 and np.allclose(basis.T @ basis, np.eye(2), atol=1e-14)
    JB = J @ (basis / D[:, None])
    g2, B2 = basis.T @ g_s, JB.T @ JB
    radius = 0.5 * (alpha * np.linalg.norm(g_s) + np.linalg.norm(gn_s))
    s, n = DL.subspace_step(g_s, gn_s, alpha, radius, basis, rank1, g2, B2)
    assert abs(np.linalg.norm(s) - radius) <= 1e-12 * radius and n == radius
    # the subspace minimiser is at least as good as the traditional dogleg point, which lies in the same plane
    def model(step_s):
        step = step_s / D
        return 0.5 * (J @ step) @ (J @ step) + (J.T @ r) @ step
    t, _ = DL.traditional_step(g_s, gn_s, alpha, radius)
    assert model(s) <= model(t) + 1e-12 * abs(model(t))
    # a root that is not a stationary point fails the first-order check: the traditional step is taken instead
    bad_roots = lambda poly: np.array([-1e3 * np.abs(B2).max()])   # noqa: E731
    assert DL.boundary_minimum(g2, B2, radius, roots=bad_roots) is None
    s_fb, n_fb = DL.subspace_step(g_s, gn_s, alpha, radius, basis, rank1, g2, B2, roots=bad_roots)
    assert np.array_equal(s_fb, t) and n_fb == DL.traditional_step(g_s, gn_s, alpha, radius)[1]
    # no usable root at all: the same fallback
    s_fb, _ = DL.subspace_step(g_s, gn_s, alpha, radius, basis, rank1, g2, B2, roots=lambda poly: np.array([]))
    assert np.array_equal(s_fb, t)


def check_least_squares_minimiser(g, dogleg_type):
    tight = DL.Options(function_tolerance=1e-15, parameter_tolerance=1e-14, gradient_tolerance=1e-14, max_num_iterations=200,
                       trust_region_strategy="dogleg", dogleg_type=dogleg_type)
    x, sm = DL.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=tight)
    assert sm.usable and 0 < sm.linear_solves <= sm.iterations
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["init"], g["edge_a"], g["edge_b"], g["z"], U, 0)

    def fun(p):
        xx = x.copy()
        xx[pb.free] = p.reshape(-1, 3)
        return pb.residuals(xx)

    ref = least_squares(fun, x[pb.free].reshape(-1), method="trf", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    xr = x.copy()
    xr[pb.free] = ref.x.reshape(-1, 3)
    d = xr - x
    d[:, 2] = synth.wrap(d[:, 2])
    assert np.abs(d).max() < 1e-6
    assert abs(0.5 * float(ref.fun @ ref.fun) - sm.final_cost) < 1e-9 * max(1.0, sm.final_cost)
    assert np.array_equal(x[0], g["init"][0]) and sm.final_cost < sm.initial_cost


@pytest.mark.parametrize("dogleg_type", ["traditional", "subspace"])
@pytest.mark.parametrize("seed", [0, 1])
def test_dogleg_reaches_the_least_squares_minimiser(seed, dogleg_type):
    check_least_squares_minimiser(synth.make_pose_graph(seed, 150, 400, sigma_xy=0.03, sigma_th=0.01), dogleg_type)


@pytest.mark.parametrize("dogleg_type", ["traditional", "subspace"])
@pytest.mark.parametrize("model,seed", [("karto", 0), ("full", 1)])
def test_dogleg_reaches_the_least_squares_minimiser_on_correlated_covariances(model, seed, dogleg_type):
    check_least_squares_minimiser(shaped_graph(model, seed, 150, 251), dogleg_type)


def test_rejected_steps_reuse_the_gauss_newton_step():
    """A rejected step shrinks the region and reuses the Gauss-Newton step: fewer linear solves than iterations."""
    g = synth.make_pose_graph(0, 500, 1500, sigma_xy=0.3, sigma_th=0.2)
    for t in ("traditional", "subspace"):
        _, sm = DL.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"],
                         opts=DL.Options(trust_region_strategy="dogleg", dogleg_type=t))
        rejected = sum(1 for tr in sm.trace[1:] if not tr[2])
        assert rejected > 0 and sm.linear_solves == sm.iterations - rejected, (t, sm.trace, sm.linear_solves)


def test_explicit_lm_is_the_default_bit_for_bit():
    g = synth.make_pose_graph(3, 300, 800, sigma_xy=0.05, sigma_th=0.02)
    args = (g["init"], g["edge_a"], g["edge_b"], g["z"])
    x0, s0 = PG.solve(*args, cov=g["cov"])
    x1, s1 = DL.solve(*args, cov=g["cov"])
    x2, s2 = DL.solve(*args, cov=g["cov"], opts=DL.Options(trust_region_strategy="lm", dogleg_type="subspace"))
    assert np.array_equal(x0, x1) and np.array_equal(x0, x2)
    for s in (s1, s2):
        assert (s.iterations, s.successful_steps, s.final_cost, s.trace) == (s0.iterations, s0.successful_steps, s0.final_cost, s0.trace)
        assert s.linear_solves == s.iterations
    with pytest.raises(ValueError):
        DL.solve(*args, cov=g["cov"], opts=DL.Options(trust_region_strategy="dogleg", dogleg_type="double"))


def test_default_opts_through_the_abi():
    L = api.lib()
    o = api.PgOpts()
    L.b200pg_default_opts(C.byref(o))
    assert (o.trust_region_strategy, o.dogleg_type) == (0, 0)
    assert (o.loss_function, o.loss_scale, o.pcg_max_iterations) == (0, 0.7, 20000)   # the fields before them are in place
    assert [f for f, _ in api.PgSummary._fields_][-1] == "linear_solves"
    # values outside {0, 1} are refused before any device is needed
    h = C.c_void_p()
    for field, value in (("trust_region_strategy", 2), ("trust_region_strategy", -1), ("dogleg_type", 2)):
        bad = api.PgOpts()
        L.b200pg_default_opts(C.byref(bad))
        setattr(bad, field, value)
        assert L.b200pg_create(C.byref(bad), C.byref(h)) == api.ERR_INVALID_ARG
        assert L.b200pg_set_opts(None, C.byref(bad)) == api.ERR_INVALID_ARG
