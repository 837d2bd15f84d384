"""Cases for the pose-graph minimiser's trust-region control (minimize(), LmStrategy and DoglegStrategy in
slam_toolbox_b200/csrc/pose_graph.cu) away from the default options: non-monotonic steps and the minimum-cost iterate,
the monotonic evaluator, the LM radius clamp, the minimum radius, the diagonal clamp, Jacobi scaling off, and invalid
steps ending the solve in FAILURE.

Each case is a fixed graph plus a b200pg_opts override (ScanSolver keyword form), selected so that the restated-Ceres
oracles (oracle/posegraph.py for LM, posegraph_dogleg.py for dogleg) show the event the case is named for; the CPU test
test_posegraph_trust_region_cases.py pins each case to its event and the GPU test compares the solver with the oracle.

Invalid steps.  A step is invalid when the linear solve fails (a residual that is not finite; under dogleg also a
Gauss-Newton solve that stays above its tolerance until mu reaches 1) or when the model cost change is not positive.
The invalid-* cases take the first route the plain way: a component without the anchor, no Jacobi scaling and both LM
diagonal bounds at 0 make the normal matrix exactly singular, so the Cholesky solve meets a zero pivot (the graph of
test_posegraph_cholesky_gpu.py's zero-pivot test).  The second route has no case: with the function, gradient and
parameter tolerances at 0 the oracle ends at the exact function or parameter tolerance before three model changes in a
row come out non-positive.

A non-finite candidate cost has no case either.  Scaling every U by one factor s keeps the LM trajectory and
multiplies every cost by s^2, so an overflowing candidate from a finite start needs s^2 near 1e303 on the swung chain
below; AddConstraint refuses the covariance of such an edge (determinant at most 1e-14, Karto's Matrix3::Inverse).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from unittest import mock

import numpy as np

import posegraph_dogleg as DL
from oracle import posegraph as PG
from pcg_reference import KERNEL_ENV
from slam_toolbox_b200 import synth

# ScanSolver options -> oracle options: the strategy enums become names, the PCG and solver-type knobs have no oracle twin
_ENUMS = {"trust_region_strategy": {0: "lm", 1: "dogleg"}, "dogleg_type": {0: "traditional", 1: "subspace"}}
_GPU_ONLY = ("pcg_tolerance", "pcg_max_iterations", "linear_solver_type")


def oracle_options(opts: dict) -> DL.Options:
    o = {}
    for k, v in opts.items():
        if k in _GPU_ONLY:
            continue
        if k in _ENUMS:
            v = _ENUMS[k][v]
        elif k in ("jacobi_scaling", "use_nonmonotonic_steps"):
            v = bool(v)
        o[k] = v
    return DL.Options(**o)


def swung(g, phi, pivot=1):
    """g's dead-reckoned start with every node from `pivot` on turned rigidly by phi about node `pivot`: only the edges
    into the pivot see it, so the start cost is one large heading residual whose Gauss-Newton step is a linearised
    rotation of the whole tail, which overshoots."""
    x = g["init"].copy()
    c, s = math.cos(phi), math.sin(phi)
    d = x[pivot:, :2] - x[pivot, :2]
    x[pivot:, 0] = x[pivot, 0] + c * d[:, 0] - s * d[:, 1]
    x[pivot:, 1] = x[pivot, 1] + s * d[:, 0] + c * d[:, 1]
    x[pivot:, 2] = synth.wrap(x[pivot:, 2] + phi)
    return dict(g, init=x)


def _plain(g):
    return dict(g, ia=g["edge_a"], ib=g["edge_b"], anchor=0)


def _family(name):
    from test_posegraph_shapes_gpu import FAMILIES
    kw = dict(FAMILIES[name])
    return synth.make_pose_graph_family(kw.pop("seed"), **kw)


_GRAPHS = {
    # very noisy odometry: steps overshoot, and several accepted steps raise the cost (non-monotonic)
    "noisy": lambda: _plain(synth.make_pose_graph(0, 500, 1500, sigma_xy=0.3, sigma_th=0.2)),
    # the P1 graphs' noise level
    "clean": lambda: _plain(synth.make_pose_graph(1, 500, 1400, sigma_xy=0.03, sigma_th=0.01)),
    # an odometry chain whose tail is turned by 2.5 rad at node 1: the first four LM steps are rejected
    "swung": lambda: _plain(swung(synth.make_pose_graph(0, 100, 99, sigma_xy=0.03, sigma_th=0.1, min_gap=5), 2.5)),
    # correlated covariances, reversed and parallel edges, shuffled order, sparse ids, isolated runs
    "karto_shuffled": lambda: _family("karto_shuffled"),
    # two one-edge components on the x axis, the second without the anchor, identity information
    "zero_pivot": lambda: dict(init=ZERO_PIVOT_POSES, ids=np.arange(4), edge_a=np.array([0, 2]), edge_b=np.array([1, 3]),
                               ia=np.array([0, 2]), ib=np.array([1, 3]), anchor=0, z=np.array([[0.9, 0.1, 0.05]] * 2),
                               cov=np.repeat(np.eye(3)[None], 2, axis=0)),
}
ZERO_PIVOT_POSES = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [5.0, 0.0, 0.0], [6.0, 0.0, 0.0]])
_GRAPH_CACHE = {}


def graph(name):
    if name not in _GRAPH_CACHE:
        _GRAPH_CACHE[name] = _GRAPHS[name]()
    return _GRAPH_CACHE[name]


@dataclass(frozen=True)
class Case:
    name: str
    graph: str
    opts: dict = field(default_factory=dict)   # ScanSolver keywords
    kernel: int | None = None                    # PCG kernel forced through KERNEL_ENV (None: the planned one)


def _lm_and_dogleg(name, g, **opts):
    return [Case(f"{name}-lm", g, dict(opts))] + [
        Case(f"{name}-dogleg-{t}", g, dict(opts, trust_region_strategy=1, dogleg_type=k)) for t, k in (("traditional", 0), ("subspace", 1))]


# diagonal clamp bounds between the quartiles of the start's squared column norms (see test_diagonal_clamp_binds), of
# the Jacobi-scaled and of the unscaled Jacobian
DIAG_SCALED = dict(min_lm_diagonal=0.97, max_lm_diagonal=0.99)          # "clean"
DIAG_UNSCALED = dict(min_lm_diagonal=5e3, max_lm_diagonal=5e4)
DIAG_NOISY_SCALED = dict(min_lm_diagonal=0.7, max_lm_diagonal=0.79)     # "noisy"
DIAG_NOISY_UNSCALED = dict(min_lm_diagonal=25.0, max_lm_diagonal=60.0)
# a singular normal matrix: Cholesky, no Jacobi scaling, no diagonal
SINGULAR = dict(linear_solver_type=1, jacobi_scaling=0, min_lm_diagonal=0.0, max_lm_diagonal=0.0)
TRUNCATE_AT = 5   # the first non-monotonic accepted step of "noisy"

CASES = {c.name: c for c in [
    # non-monotonic steps: accepted steps with cost >= the minimum so far
    *_lm_and_dogleg("nonmono", "noisy"),
    # stopped right after the first such step: the minimum-cost iterate is the one before the last
    Case("nonmono-truncated-lm", "noisy", dict(max_num_iterations=TRUNCATE_AT)),
    # the monotonic evaluator and other windows of the non-monotonic one
    *_lm_and_dogleg("monotonic", "noisy", use_nonmonotonic_steps=0),
    Case("nonmono-window-1-lm", "noisy", dict(max_consecutive_nonmonotonic_steps=1)),
    Case("nonmono-window-10-lm", "noisy", dict(max_consecutive_nonmonotonic_steps=10)),
    # LM radius growth clamped to max_trust_region_radius, from below it and from above it
    Case("radius-clamp-lm", "clean", dict(initial_trust_region_radius=1.0, max_trust_region_radius=3.0)),
    *_lm_and_dogleg("radius-above-max", "clean", max_trust_region_radius=1e2),
    # four rejected steps take the radius from 1e4 below 1e2 (LM) or 1e3 (dogleg): termination 4, usable
    Case("min-radius-lm", "swung", dict(min_trust_region_radius=1e2)),
    *_lm_and_dogleg("min-radius", "swung", min_trust_region_radius=1e3)[1:],
    # both sides of the LM diagonal clamp bind, with and without Jacobi scaling (a small radius makes the diagonal matter)
    Case("diag-clamp-lm", "clean", dict(initial_trust_region_radius=1.0, **DIAG_SCALED)),
    Case("diag-clamp-nojacobi-lm", "clean", dict(initial_trust_region_radius=1.0, jacobi_scaling=0, **DIAG_UNSCALED)),
    # dogleg's metric is the clamped diagonal too; on the noisy graph its steps end inside the region, where it matters
    *_lm_and_dogleg("diag-clamp", "noisy", **DIAG_NOISY_SCALED)[1:],
    *_lm_and_dogleg("diag-clamp-nojacobi", "noisy", jacobi_scaling=0, **DIAG_NOISY_UNSCALED)[1:],
    # Jacobi scaling off under each PCG kernel and both dogleg types
    *[Case(f"jacobi-off-kernel{k}-lm", "karto_shuffled", dict(jacobi_scaling=0), kernel=k) for k in (6, 3, 1, 0, 13, 16)],
    *_lm_and_dogleg("jacobi-off", "karto_shuffled", jacobi_scaling=0)[1:],
    # every step invalid (a zero pivot): FAILURE after max_num_consecutive_invalid_steps of them
    *[c for k in (1, 3) for c in _lm_and_dogleg(f"invalid-{k}", "zero_pivot", max_num_consecutive_invalid_steps=k, **SINGULAR)],
]}


@dataclass
class Run:
    x: np.ndarray          # the returned poses (the minimum-cost iterate)
    summary: object        # DL.Summary
    x_exit: np.ndarray     # the iterate the minimiser stood at when it stopped
    cand_costs: list       # the cost of every candidate point, in order


def solve(g, opts: dict, init=None) -> Run:
    """The oracle of `opts`' strategy on graph g, with the iterate at exit and the candidate costs recorded: the
    oracles linearise every accepted iterate (and only those) and evaluate each candidate once."""
    lin, costs = [], []

    class Recording(PG.Problem):
        def jacobian(self, x):
            lin.append(x.copy())
            return super().jacobian(x)

        def cost(self, x):
            c = super().cost(x)
            costs.append(c)
            return c

    x0 = g["init"] if init is None else init
    with mock.patch.object(PG, "Problem", Recording):
        x, s = DL.solve(x0, g["ia"], g["ib"], g["z"], cov=g["cov"], fixed=g["anchor"], opts=oracle_options(opts))
    return Run(x, s, lin[-1], costs[1:])


_RUNS = {}


def oracle(case: Case) -> Run:
    if case.name not in _RUNS:
        _RUNS[case.name] = solve(graph(case.graph), case.opts)
    return _RUNS[case.name]


def nonmonotonic_steps(summary):
    """Iterations whose step was accepted with a cost at or above the minimum of the iterates before it."""
    out, best = [], summary.trace[0][1]
    for it, cost, accepted, _ in summary.trace[1:]:
        if accepted:
            if cost >= best:
                out.append(it)
            best = min(best, cost)
    return out


def lm_diagonal(g):
    """Squared column norms of the Jacobian at the start, unscaled and Jacobi-scaled (the LM diagonal before its clamp)."""
    U = np.stack([PG.sqrt_information(c) for c in g["cov"]])
    pb = PG.Problem(g["init"], g["ia"], g["ib"], g["z"], U, g["anchor"])
    J = pb.jacobian(g["init"])
    d = np.asarray(J.multiply(J).sum(axis=0)).ravel()
    return d, d / (1.0 + np.sqrt(d)) ** 2
