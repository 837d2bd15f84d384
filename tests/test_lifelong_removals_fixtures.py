"""The removal plans of test_lifelong_removals_gpu.py have the shapes their cases claim (anchorless components, isolated nodes,
swapping and non-swapping removals, lifelong's guards), and the oracle tells apart the rules those tests must separate: the
anchor held by id or by slot 0, and a node without an edge held or taken as a parameter block.  No GPU."""
import numpy as np
import pytest

import lifelong_removals as LR
import posegraph_dogleg as DL
from oracle import posegraph as PG

SCENARIOS = {}


def scenario(name):
    if name not in SCENARIOS:
        SCENARIOS[name] = LR.scenario(name)
    return SCENARIOS[name]


def final_book(sc, upto=None):
    book = LR._base(sc["graph"])
    for ops in sc["steps"][:upto]:
        for op in ops:
            if op[0] == "remove":
                book.remove(op[1])
            elif op[0] == "edge":
                book.add_edge(*op[1:])
    return book


@pytest.mark.parametrize("case", LR.CASES)
def test_removals_meet_lifelong_guards(case):
    """Every removal but the deliberate ones of 'slots' (the newest node) and 'anchor' (id 0) is one lifelong mode may make:
    not ids 0 and 1, at least scan_buffer_size ids older than the newest, two or more edges when it goes."""
    sc = scenario(case)
    assert sc["steps"][0] == []
    assert all(s["guarded"] for s in sc["shapes"])
    removed = [op[1] for ops in sc["steps"] for op in ops if op[0] == "remove"]
    assert len(removed) == len(set(removed)) and removed
    if case not in ("slots", "anchor"):
        assert not {0, 1} & set(removed)
        assert max(removed) <= len(sc["graph"]["ids"]) - 1 - LR.BUFFER


def test_batches_shape():
    sc = scenario("batches")
    assert len(sc["graph"]["ids"]) == 600 and len(sc["steps"]) == 5
    assert [sum(op[0] == "remove" for op in ops) for ops in sc["steps"][1:]] == [12, 12, 12, 12]
    frags = [s["fragments"] for s in sc["shapes"]]
    assert frags[0] == 0 and frags[-1] >= 2 and frags == sorted(frags)


@pytest.mark.parametrize("n", [1, 2, 8])
def test_fragments_shape(n):
    """Each removal cuts off one more component without the anchor, and leaves no node without an edge."""
    sc = scenario(f"fragments_{n}")
    assert [s["fragments"] for s in sc["shapes"]] == list(range(n + 1))
    assert all(not s["isolated"] for s in sc["shapes"])
    assert all(s["swaps"] == 1 for s in sc["shapes"][1:])


def test_isolated_shape():
    sc = scenario("isolated")
    iso = sc["shapes"][1]["isolated"]
    assert len(iso) == 1 and sc["shapes"][2]["isolated"] == iso
    assert ("yaw", iso[0], 7.0) in sc["steps"][1]
    # its two neighbours left in that step, and nothing else touches it afterwards
    assert {op[1] for op in sc["steps"][1] if op[0] == "remove"} == {iso[0] - 1, iso[0] + 1}


def test_slot_moves_happen_both_ways():
    """'slots' removes the node in the last slot (no swap), then one whose slot receives the last node; across the suite
    both kinds occur."""
    sh = scenario("slots")["shapes"]
    assert (sh[1]["plain"], sh[1]["swaps"]) == (1, 0) and (sh[2]["plain"], sh[2]["swaps"]) == (0, 1)
    assert sum(s["swaps"] for c in LR.CASES for s in scenario(c)["shapes"]) > 50


def test_anchor_shape():
    sc = scenario("anchor")
    assert sc["steps"][1] == [("remove", 0)]
    # without the anchor the whole graph is one component that nothing holds
    assert sc["shapes"][1]["fragments"] == 1
    book = final_book(sc, 2)
    assert book.anchor == 0 and 0 not in book.order and book.problem(dict(zip(sc["graph"]["ids"].tolist(), sc["graph"]["init"])))[5] is None


def test_append_shape():
    sc = scenario("append")
    assert [op[0] for op in sc["steps"][1]] == ["remove"]
    assert [op[0] for op in sc["steps"][2]] == ["edge"] * 5
    book = final_book(sc, 3)
    pairs = {tuple(sorted(e[:2])) for e in book.live()}
    a, b = sc["steps"][3][0][1:3]
    assert tuple(sorted((a, b))) in pairs      # a parallel edge: the same Cholesky pattern
    assert all(tuple(sorted(op[1:3])) not in {tuple(sorted(e[:2])) for e in final_book(sc, 2).live()} for op in sc["steps"][2])


def _solve(book, poses, fixed, strategy="lm"):
    init, ea, eb, z, cov, _ = book.problem(poses)
    kw = dict(trust_region_strategy="dogleg", dogleg_type=strategy) if strategy != "lm" else {}
    return init, DL.solve(init, ea, eb, z, cov=cov, fixed=fixed, opts=DL.Options(**kw))


@pytest.mark.parametrize("strategy", ["lm", "traditional"])
def test_anchor_by_id_differs_from_slot_zero(strategy):
    """After the anchor leaves, slot 0 holds the node that was last: fixing it (the mistake) gives another answer than
    fixing nothing (CeresSolver)."""
    sc = scenario("anchor")
    book = final_book(sc, 2)
    poses = dict(zip(sc["graph"]["ids"].tolist(), sc["graph"]["init"]))
    _, (x_id, s_id) = _solve(book, poses, None, strategy)
    init, (x_s0, s_s0) = _solve(book, poses, 0, strategy)
    assert np.array_equal(x_s0[0], init[0]) and not np.array_equal(x_id[0], init[0])
    d = np.abs(x_id - x_s0)[:, :2].max()
    assert d > 100 * 1e-4 or (s_id.iterations, s_id.final_cost) != (s_s0.iterations, s_s0.final_cost), d


def test_isolated_node_free_differs_from_held(monkeypatch):
    """A node without an edge is no parameter block.  Taken as one, the step's AngleLocalParameterization would wrap its
    yaw (pushed outside [-pi, pi) by the case) and its coordinates would enter the parameter tolerance."""
    sc = scenario("isolated")
    book = final_book(sc, 2)
    v = sc["shapes"][1]["isolated"][0]
    poses = {int(n): p.copy() for n, p in zip(sc["graph"]["ids"], sc["graph"]["init"])}
    poses[v][2] += 7.0
    init, (x_held, _) = _solve(book, poses, 0)
    slot = book.order.index(v)
    assert np.array_equal(x_held[slot], init[slot])
    real_init = PG.Problem.__init__

    def free_isolated(self, *a, **k):
        real_init(self, *a, **k)
        self.free = np.union1d(self.free, [slot])
        self.col = -np.ones(self.N, dtype=np.int64)
        self.col[self.free] = np.arange(len(self.free))
    monkeypatch.setattr(PG.Problem, "__init__", free_isolated)
    _, (x_free, _) = _solve(book, poses, 0)
    assert x_free[slot, 2] != x_held[slot, 2] and -np.pi <= x_free[slot, 2] < np.pi
