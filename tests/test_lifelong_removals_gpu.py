"""The pose-graph solver under slam_toolbox's lifelong-mode removal traffic (tests/lifelong_removals.py): interior nodes leave
as Mapper::RemoveNodeFromGraph retires them, which cuts the trajectory into pieces with no anchor (only the LM diagonal, or
dogleg's mu, holds them), leaves nodes without an edge, moves the last slot's node into the freed slot (so the slot ranges
the two-level kernels aggregate stop following the trajectory) and marks the problem for a full upload and, on the Cholesky
path, a new analysis.  After every Compute the result must match the exact-solve oracle (oracle.posegraph for LM,
tests/posegraph_dogleg.py for dogleg) on the problem rebuilt from the solver's own state in its slot order, at P1: equal
iterations, accepted steps and linear solves, final cost within 1e-8 relative, poses within 1e-4 m / 1e-5 rad, corrections in
slot order, and the anchor and isolated nodes returned bit for bit.  Every run asserts the linear solver that ran."""
import numpy as np
import pytest

import lifelong_removals as LR
import posegraph_dogleg as DL
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
TOL_XY, TOL_TH = 1e-4, 1e-5

# name: (solver options, environment read when the handle is created (pose_graph.cu:953-957), linear solver that must run,
# oracle strategy).  Kernel numbers as b200pg_summary.linear_solver: 0 / 1 block-Jacobi (global / shared memory), 3 / 6
# two-level with shared-memory aggregates, 13 / 16 two-level with global-memory aggregates, 8 Cholesky.
LM, TRAD, SUB = dict(), dict(trust_region_strategy=1, dogleg_type=0), dict(trust_region_strategy=1, dogleg_type=1)
CONFIGS = {
    "lm-k0": (LM, {"B200PG_FORCE_GLOBAL_PCG": "1"}, 0, "lm"),
    "lm-k1": (LM, {"B200PG_PRECOND": "jacobi"}, 1, "lm"),
    "lm-k3": (LM, {"B200PG_COARSE_MODES": "3"}, 3, "lm"),
    "lm-k6": (LM, {}, 6, "lm"),
    "lm-k13": (LM, {"B200PG_FORCE_2LVL_GLOBAL": "1", "B200PG_COARSE_MODES": "3"}, 13, "lm"),
    "lm-k16": (LM, {"B200PG_FORCE_2LVL_GLOBAL": "1"}, 16, "lm"),
    "lm-cholesky": (dict(linear_solver_type=1), {}, 8, "lm"),
    "traditional-k6": (TRAD, {}, 6, "traditional"),
    "traditional-k3": (TRAD, {"B200PG_COARSE_MODES": "3"}, 3, "traditional"),
    "traditional-cholesky": (dict(TRAD, linear_solver_type=1), {}, 8, "traditional"),
    "subspace-k6": (SUB, {}, 6, "subspace"),
    "subspace-k3": (SUB, {"B200PG_COARSE_MODES": "3"}, 3, "subspace"),
    "subspace-cholesky": (dict(SUB, linear_solver_type=1), {}, 8, "subspace"),
    "huber-k6": (dict(loss_function=1, loss_scale=0.7), {}, 6, "huber"),
}


def oracle(strategy, init, ea, eb, z, cov, fixed):
    kw = dict(trust_region_strategy="dogleg", dogleg_type=strategy) if strategy in ("traditional", "subspace") else {}
    if strategy == "huber":
        kw["loss_function"] = "huber"
    return DL.solve(init, ea, eb, z, cov=cov, fixed=fixed, opts=DL.Options(**kw))


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("case", LR.CASES)
def test_lifelong_removals_match_oracle(case, config, monkeypatch):
    opts, env, kernel, strategy = CONFIGS[config]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = LR.scenario(case)
    g = sc["graph"]
    s = api.ScanSolver(**opts)
    book = LR._base(g)
    for nid, p in zip(g["ids"], g["init"]):
        s.AddNode(int(nid), p)
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
        assert s.AddConstraint(int(a), int(b), z, c)
    assert s.Compute() and s.summary.linear_solver == kernel, (s.summary.linear_solver, kernel)
    analyses = s.factor_info()["analyses"]
    worst = np.zeros(2)
    for k, ops in enumerate(sc["steps"][1:], 1):
        removed = appended = 0
        for op in ops:
            if op[0] == "remove":
                calls, _ = book.remove(op[1])
                for a, b in calls:
                    assert s.RemoveConstraint(a, b), (k, op, a, b)
                assert s.RemoveNode(op[1])
                removed += 1
            elif op[0] == "edge":
                assert s.AddConstraint(*op[1:])
                book.add_edge(*op[1:])
                appended += 1
            else:
                p = s.get_node(op[1])
                s.ModifyNode(op[1], [p[0], p[1], op[2]])
        init, ea, eb, z, cov, fixed = book.problem({n: s.get_node(n) for n in book.order})
        _, isolated = book.components()
        xo, so = oracle(strategy, init, ea, eb, z, cov, fixed)
        assert s.Compute()
        sm = s.summary
        assert sm.linear_solver == kernel, (k, sm.linear_solver, kernel)
        # a removal marks the problem for a full upload; constraints appended after a solve travel alone
        assert sm.uploaded_edges == (len(ea) if removed else appended), (k, sm.uploaded_edges, len(ea), appended)
        assert s.num_edges() == len(ea) and s.num_nodes() == len(book.order)
        if kernel == 8:
            info = s.factor_info()
            if removed:
                assert info["analyses"] == analyses + 1, (k, info, analyses)
            elif case == "append" and k == len(sc["steps"]) - 1:
                assert info["analyses"] == analyses, (k, info, analyses)   # a parallel edge keeps the pattern
            analyses = info["analyses"]
            assert info["columns"] == len(book.order) - len(isolated) - (fixed is not None)
        ids, xg = s.GetCorrections()
        assert np.array_equal(ids, book.order)
        assert (sm.iterations, sm.successful_steps, sm.linear_solves) == (so.iterations, so.successful_steps, so.linear_solves), \
            (k, (sm.iterations, sm.successful_steps, sm.linear_solves), (so.iterations, so.successful_steps, so.linear_solves))
        assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (k, sm.final_cost, so.final_cost)
        d = xg - xo
        d[:, 2] = synth.wrap(d[:, 2])
        gap = np.array([np.abs(d[:, :2]).max(), np.abs(d[:, 2]).max()])
        worst = np.maximum(worst, gap)
        assert gap[0] < TOL_XY and gap[1] < TOL_TH, (k, gap)
        # the anchor (while it is there) and every node without an edge are outside the problem: returned as they went in
        held = [book.order.index(n) for n in isolated] + ([fixed] if fixed is not None else [])
        assert np.array_equal(xg[held], init[held])
        if case == "isolated":
            assert len(isolated) == 1 and init[book.order.index(isolated[0]), 2] > np.pi
        if case == "anchor" and k >= 1:
            assert fixed is None
    print(f"{case} {config}: kernel {kernel}, worst gap {worst[0]:.2e} m / {worst[1]:.2e} rad")
