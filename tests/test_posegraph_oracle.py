"""Checks of the restated pose-graph oracle (oracle/posegraph.py; PARITY UNPINNED -- Ceres is not in
the container): its building blocks against what the reference's own karto code computes where that exists
(LinkInfo, Matrix3::Inverse: tests/golden/reference_golden.npz) and its minimiser against scipy.optimize.least_squares."""
import hashlib

import numpy as np
import pytest
from scipy.optimize import least_squares

import helpers as H
from golden import make_reference_golden as G
from oracle import posegraph as PG
from slam_toolbox_b200 import synth


def test_normalize_angle_range():
    a = np.linspace(-20, 20, 1001)
    w = PG.normalize_angle(a)
    assert np.all(w >= -np.pi) and np.all(w < np.pi)
    assert np.allclose(np.sin(w), np.sin(a)) and np.allclose(np.cos(w), np.cos(a))
    assert PG.normalize_angle(np.array([np.pi]))[0] == -np.pi


def test_link_info_and_inverse_match_karto():
    ref = H.reference_golden()
    for i, (p1, p2, cov) in enumerate(G.link_info_inputs()):
        d_ref, c_ref = ref["link_info/delta"][i], ref["link_info/cov"][i]
        d, c = PG.link_info(p1, p2, cov)
        assert np.allclose(d[:2], d_ref[:2], atol=1e-12)
        assert abs(np.sin(d[2] - d_ref[2])) < 1e-12 and np.cos(d[2] - d_ref[2]) > 0
        assert np.allclose(c, c_ref, atol=1e-12)
        assert np.allclose(PG.matrix3_inverse(cov), ref["link_info/inverse"][i], rtol=1e-13, atol=0)


def test_sqrt_information_is_upper_cholesky_of_the_information():
    rng = np.random.default_rng(1)
    A = rng.normal(size=(3, 3))
    cov = A @ A.T + 0.5 * np.eye(3)
    U = PG.sqrt_information(cov)
    assert np.allclose(np.tril(U, -1), 0)
    assert np.allclose(U.T @ U, np.linalg.inv(cov), rtol=1e-10)


def shaped_graph(model, seed, n, loops):
    """A graph of synth.make_pose_graph_family with edges as insertion positions (what the oracle indexes)."""
    g = synth.make_pose_graph_family(seed, n, loops, cov_model=model, reversed_frac=0.3, duplicate_frac=0.05, order="shuffled",
                                     ids="sparse", world_rotation=0.7)
    return dict(g, edge_a=g["ia"], edge_b=g["ib"])


def check_jacobian(g):
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["init"], g["edge_a"], g["edge_b"], g["z"], U, 0)
    x = g["init"].copy()
    J = pb.jacobian(x).toarray()
    r0 = pb.residuals(x)
    eps = 1e-6
    for k in range(0, J.shape[1], 7):
        d = np.zeros(J.shape[1]); d[k] = eps
        num = (pb.residuals(pb.plus(x, d)) - r0) / eps
        assert np.allclose(num, J[:, k], atol=2e-4 * (1 + np.abs(J[:, k]).max()))


def test_jacobian_matches_finite_differences():
    check_jacobian(synth.make_pose_graph(2, 40, 70, sigma_xy=0.03, sigma_th=0.01))


@pytest.mark.parametrize("model", ["karto", "full"])
def test_jacobian_matches_finite_differences_on_correlated_covariances(model):
    g = shaped_graph(model, 2, 40, 30)
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    # every off-diagonal sqrt-information term is in use; (0, 2) and (1, 2) come from xy-theta terms ("full", or a reversed edge)
    for i, j in ((0, 1), (0, 2), (1, 2)):
        assert np.abs(U[:, i, j]).max() > 0.1 * np.abs(U[:, i, i]).max(), (i, j)
    check_jacobian(g)


def check_least_squares_minimiser(g):
    tight = PG.Options(function_tolerance=1e-15, parameter_tolerance=1e-14, gradient_tolerance=1e-14, max_num_iterations=200)
    x, sm = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=tight)
    assert sm.usable
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
    # anchor untouched; cost decreased
    assert np.array_equal(x[0], g["init"][0]) and sm.final_cost < sm.initial_cost


@pytest.mark.parametrize("seed", [0, 1])
def test_lm_reaches_the_least_squares_minimiser(seed):
    check_least_squares_minimiser(synth.make_pose_graph(seed, 150, 400, sigma_xy=0.03, sigma_th=0.01))


@pytest.mark.parametrize("model,seed", [("karto", 0), ("full", 1)])
def test_lm_reaches_the_least_squares_minimiser_on_correlated_covariances(model, seed):
    check_least_squares_minimiser(shaped_graph(model, seed, 150, 251))


def test_reference_tolerances_stop_early_but_near_the_minimum():
    g = synth.make_pose_graph(3, 300, 800, sigma_xy=0.03, sigma_th=0.01)
    x, sm = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"])
    assert sm.usable and sm.iterations <= 50 and "CONVERGENCE" in sm.termination
    tight = PG.Options(function_tolerance=1e-15, parameter_tolerance=1e-14, gradient_tolerance=1e-14, max_num_iterations=200)
    _, st = PG.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=tight)
    # function_tolerance 1e-3 stops close to the minimum cost, never below it
    assert st.final_cost <= sm.final_cost <= 1.25 * st.final_cost


def test_nodes_without_edges_and_missing_anchor_edges():
    g = synth.make_pose_graph(4, 30, 40, sigma_xy=0.03, sigma_th=0.01)
    init = np.vstack([g["init"], [[100.0, 100.0, 1.0]]])   # an isolated node: not a Ceres parameter block
    x, sm = PG.solve(init, g["edge_a"], g["edge_b"], g["z"], cov=g["cov"])
    assert np.array_equal(x[-1], init[-1]) and sm.usable


def graph_digest(g):
    h = hashlib.sha256()
    for k in ("ids", "init", "truth", "edge_a", "edge_b", "z", "cov"):
        a = np.ascontiguousarray(g[k])
        h.update(k.encode() + str(a.dtype).encode() + str(a.shape).encode() + a.tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("args,digest", [
    ((0, 10000, 40000, 0.05, 0.02), "23841374cad805cbe05a54b0b4cff877928a608601ebcb80bcb37393c58e3f3a"),
    ((0, 10000, 40000, 0.03, 0.01), "f9ac0b6d416bf0563d370ee12f733456fee4e5c38ed5add2d0741625da6a1f89"),
    ((1, 300, 700, 0.03, 0.01), "0815a20f9cc5caa96826d6293a45421bae6dd7bfd439feea60628e568a5e56fc"),
])
def test_make_pose_graph_is_unchanged(args, digest):
    """bench.py's cfg4 graphs (both noise levels) and smoke()'s graph are what they always were."""
    seed, n, e, sxy, sth = args
    assert graph_digest(synth.make_pose_graph(seed, n, e, sigma_xy=sxy, sigma_th=sth)) == digest


def test_graph_family_shapes():
    """make_pose_graph_family builds what its options ask for."""
    g = synth.make_pose_graph_family(3, 400, 800, cov_model="full", reversed_frac=0.4, duplicate_frac=0.1, order="shuffled",
                                     ids="sparse", world_rotation=0.7, world_translation=(1e4, -3e4), isolated_runs=((0.5, 40),),
                                     detached_nodes=60, hub_degree=30)
    N, E = len(g["ids"]), len(g["z"])
    assert N == 400 + 60 + 40 and len(np.unique(g["ids"])) == N and g["ids"].dtype == np.int32
    assert g["ids"].min() == np.iinfo(np.int32).min and g["ids"].max() == np.iinfo(np.int32).max and (g["ids"] < 0).sum() > N // 4
    assert np.array_equal(g["edge_a"], g["ids"][g["ia"]]) and np.array_equal(g["edge_b"], g["ids"][g["ib"]])
    assert 0.3 < (g["ia"] > g["ib"]).mean() < 0.7          # shuffled order and reversed edges
    pairs = np.sort(np.stack([g["ia"], g["ib"]], 1), axis=1)
    assert len(np.unique(pairs, axis=0)) < E                 # parallel edges
    iso = np.nonzero(g["component"] < 0)[0]
    assert len(iso) == 40 and np.all(np.diff(iso) == 1) and iso[0] > 0
    assert not np.isin(iso, np.concatenate([g["ia"], g["ib"]])).any()
    det = g["component"] == 1
    assert det.sum() == 60 and not np.any(det[g["ia"]] != det[g["ib"]])
    assert np.bincount(np.concatenate([g["ia"], g["ib"]]), minlength=N).max() >= 30
    assert np.all(np.linalg.eigvalsh(g["cov"]) > 0) and np.allclose(g["cov"], np.transpose(g["cov"], (0, 2, 1)))
    main = g["component"] == 0
    assert np.abs(g["truth"][main, 0].mean() - 1e4) < 200 and np.abs(g["truth"][main, 1].mean() + 3e4) < 200
    # headings are off the lattice directions
    assert np.abs(np.sin(2 * g["truth"][main, 2])).max() > 0.1
    # measurements are the truth's relative poses up to noise of the stated covariance: whitened residuals ~ N(0, I)
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["truth"], g["ia"], g["ib"], g["z"], U, 0)
    w = pb.raw_residuals(g["truth"])
    assert 0.85 < w.var() < 1.15 and abs(w.mean()) < 0.1
