"""slam_toolbox's localization mode (src/slam_toolbox_localization.cpp:176-237) on a map built in the same process: the
reference's own Mapper::ProcessLocalization / ProcessAgainstNodesNearBy / ClearLocalizationBuffer, once with the reference
CPU ScanMatcher and once with every MatchScan on the GPU, both with the GPU ScanSolver adapter.  The rolling buffer retires
scans through ScanSolver::RemoveConstraint / RemoveNode, which the mapping replays never reach.  Last, the solver alone
under that removal traffic against the restated-Ceres oracles."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import replay  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not replay.available(), reason="oracle/_ref/libreplay_*.so not built")]

N_MAP, N_LOC, SEED = 120, 80, 4
BUFFER = replay.LOCALIZATION_PARAMS["scan_buffer_size"]
SMEARS = {"order_free": 0.03, "shipped": 0.1}


def trajectories():
    mr, mo, _ = replay.make_trajectory(SEED, N_MAP)
    lr, lo, lt = replay.make_localization_trajectory(SEED, N_LOC, map_scans=N_MAP)
    return mr, mo, lr, lo, lt


def params(smear):
    return dict(replay.YAML_PARAMS, correlation_search_space_smear_deviation=smear, loop_search_space_dimension=4.0)


def start_events(lo):
    # the robot starts on the map from a pose estimate: its odometric pose, a few centimetres off the truth
    return [(0, "process_near", lo[0])]


_RUNS = {}


def localize(tag):
    """(reference CPU matcher run, GPU matcher run) at SMEARS[tag], cached for the tests that share them."""
    if tag not in _RUNS:
        mr, mo, lr, lo, _ = trajectories()
        ev = start_events(lo)
        a = replay.run_localization("ref", mr, mo, lr, lo, params(SMEARS[tag]), events=ev)
        b = replay.run_localization("b200", mr, mo, lr, lo, params(SMEARS[tag]), events=ev, map_resolution=0.05)
        _RUNS[tag] = (a, b)
    return _RUNS[tag]


def assert_identical(a, b):
    assert np.array_equal(a["flags"], b["flags"])
    assert np.array_equal(a["poses"], b["poses"], equal_nan=True)
    assert np.array_equal(a["covs"], b["covs"], equal_nan=True)
    assert np.array_equal(a["step_counts"], b["step_counts"]) and np.array_equal(a["clear_counts"], b["clear_counts"])
    assert np.array_equal(a["scan_ids"], b["scan_ids"]) and np.array_equal(a["scan_poses"], b["scan_poses"])
    for k in ("edge_src", "edge_dst", "edge_diff", "edge_cov"):
        assert np.array_equal(a[k], b[k]), k
    assert a["graph_nodes"] == b["graph_nodes"]
    assert np.array_equal(a["graph_ids"], b["graph_ids"]) and np.array_equal(a["graph_poses"], b["graph_poses"])
    assert np.array_equal(a["compute_uploaded"], b["compute_uploaded"])


@pytest.mark.parametrize("tag", sorted(SMEARS))
def test_localization_is_identical_with_the_gpu_matcher(tag):
    """Smear 0.03 m: the sequential raster does not depend on scan order; 0.1 m @ 0.01 m (the shipped YAML): it does."""
    a, b = localize(tag)
    assert_identical(a, b)
    assert b["flags"].sum() > N_LOC // 2 and b["loc_match_calls"] >= b["flags"].sum() - 1
    # localization corrected the odometry's offset and drift
    _, _, _, lo, lt = trajectories()
    done = b["flags"] == 1
    assert np.abs(b["poses"][done, :2] - lt[done, :2]).max() < np.abs(lo[done, :2] - lt[done, :2]).max()
    if tag == "order_free":
        # the map publish over the scans left after the removals: b200og == OccupancyGrid::CreateFromScans
        assert b["map_cpu_seconds"] >= 0 and b["map_gpu_seconds"] >= 0
        assert np.array_equal(b["map_cpu_dims"], b["map_gpu_dims"]) and np.array_equal(b["map_cpu_offset"], b["map_gpu_offset"])
        assert np.array_equal(b["map_cpu_cells"], b["map_gpu_cells"]) and (b["map_gpu_cells"] == 100).sum() > 100


@pytest.mark.parametrize("which", ["ref", "b200"])
def test_rolling_buffer_reaches_the_solver(which):
    r = localize("order_free")[0 if which == "ref" else 1]
    c = r["step_counts"]                      # mapper vertices, mapper edges, solver nodes, solver edges after every step
    n_map = int(r["map_counts"][0])
    assert np.array_equal(c[:, 2], c[:, 0]) and np.array_equal(c[:, 3], c[:, 1])
    assert (c[:, 0] >= n_map).all() and (c[:, 0] <= n_map + BUFFER).all()
    assert c[-1, 0] == n_map + BUFFER
    removals = int(r["flags"].sum()) - (int(c[-1, 0]) - n_map)
    loc_computes = len(r["compute_ms"]) - r["map_computes"]
    assert removals > 0 and loc_computes > 0, (removals, loc_computes)
    # the graph the solver holds is exactly the mapper's processed set, the last BUFFER localization scans included
    assert r["graph_nodes"] == len(r["scan_ids"]) and np.array_equal(r["graph_ids"], np.sort(r["scan_ids"]))
    assert np.isfinite(r["graph_poses"]).all()
    # no edge of the mapper's graph still names a retired scan
    assert len(r["edge_src"]) == c[-1, 1]
    assert set(r["edge_src"].tolist()) | set(r["edge_dst"].tolist()) <= set(r["scan_ids"].tolist())
    # a removal marks the problem for a full rebuild: a compute after one uploads every constraint
    assert r["compute_uploaded"][r["map_computes"]:].max() >= r["map_counts"][1]


def test_relocalisation_and_buffer_clear():
    """A pose estimate mid-run (PROCESS_NEAR_REGION at a pose a few decimetres off the truth), then the node's localizePose
    flow: ClearLocalizationBuffer, the next scan near a new estimate, then ProcessLocalization to the end."""
    mr, mo, lr, lo, lt = trajectories()
    ev = start_events(lo) + [(25, "process_near", lt[25] + [0.2, -0.15, 0.03]),
                             (50, "clear_localization_buffer", None), (50, "process_near", lt[50] + [-0.12, 0.18, -0.02])]
    a = replay.run_localization("ref", mr, mo, lr, lo, params(SMEARS["order_free"]), events=ev)
    b = replay.run_localization("b200", mr, mo, lr, lo, params(SMEARS["order_free"]), events=ev)
    assert_identical(a, b)
    assert b["flags"][25] == 1 and b["flags"][50] == 1
    assert np.abs(b["poses"][25, :2] - lt[25, :2]).max() < 0.1 and np.abs(b["poses"][50, :2] - lt[50, :2]).max() < 0.1
    # the clear took every buffered scan out of the mapper's graph and out of the solver: back to the map alone
    assert len(b["clear_counts"]) == 1 and b["clear_counts"][0, 0] == 50
    assert np.array_equal(b["clear_counts"][0, 1:], b["map_counts"])
    c = b["step_counts"]
    assert np.array_equal(c[:, 2], c[:, 0]) and np.array_equal(c[:, 3], c[:, 1])
    assert b["graph_nodes"] == len(b["scan_ids"]) and np.array_equal(b["graph_ids"], np.sort(b["scan_ids"]))


def test_without_a_solver_the_localization_calls_refuse():
    """ProcessLocalization dereferences the scan solver on every removal (Mapper.cpp:2977, 3003): the driver refuses instead."""
    import subprocess
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); import replay\n"
            "L = replay._bind('b200'); h = replay._create(L, replay.DEFAULT_LASER, replay.YAML_PARAMS, False)\n"
            "import numpy as np; r = np.full(1081, 5.0); o = np.zeros(3); p = np.zeros(3); c = np.zeros(9)\n"
            "D = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))\n"
            "print(L.krep_process_localization(h, D(r), 1081, D(o), 0, D(p), D(c)), L.krep_process_near(h, D(r), 1081, D(o), 0, D(o), D(p), D(c)),"
            " L.krep_clear_localization_buffer(h))") % os.path.join(ROOT, "integration")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split()[-3:] == ["-1", "-1", "-1"]


# --- the solver alone under the rolling buffer's removal traffic ------------------------------------------------------------

STRATEGIES = {"lm": dict(), "traditional": dict(trust_region_strategy=1, dogleg_type=0),
              "subspace": dict(trust_region_strategy=1, dogleg_type=1), "huber": dict(loss_function=1, loss_scale=0.7),
              "cholesky": dict(linear_solver_type=1)}


def _oracle(t, init, ea, eb, z, cov):
    import posegraph_dogleg as DL
    kw = dict(trust_region_strategy="dogleg", dogleg_type=t) if t in ("traditional", "subspace") else dict(trust_region_strategy="lm")
    if t == "huber":
        kw["loss_function"] = "huber"
    return DL.solve(init, ea, eb, z, cov=cov, fixed=0, opts=DL.Options(**kw))


@pytest.mark.parametrize("t", sorted(STRATEGIES))
def test_solver_under_rolling_buffer_removals_matches_oracle(t):
    """A map graph, then rolling nodes each with a sequential edge and a link to the map; the oldest leaves as
    Mapper::RemoveNodeFromGraph (Mapper.cpp:2964-3021) retires it: RemoveConstraint(source, target) for each of its
    neighbours' edges that touch it, neighbours in the retired vertex's edge order, then RemoveNode.  After every retirement
    Compute must match the oracle on the remaining graph (P1: iterations, accepted steps, linear solves, final cost, poses),
    with the node order the removals left (the last node moves into the freed slot)."""
    from slam_toolbox_b200 import api, synth
    g = synth.make_pose_graph(3, 300, 700, sigma_xy=0.03, sigma_th=0.01)
    rng = np.random.default_rng(17)
    cov = np.diag([0.03 ** 2, 0.03 ** 2, 0.01 ** 2])
    s = api.ScanSolver(**STRATEGIES[t])
    order = []                                 # node ids in slot order, as the solver keeps them
    edges = []                                 # (source, target, z, cov) in insertion order
    vedges = {}                                # Vertex::GetEdges of every node: indices into edges

    def add_node(nid, p):
        s.AddNode(nid, p)
        order.append(nid)
        vedges[nid] = []

    def add_edge(a, b, z, c):
        assert s.AddConstraint(a, b, z, c)
        edges.append((a, b, np.asarray(z, dtype=np.float64), c))
        vedges[a].append(len(edges) - 1)
        vedges[b].append(len(edges) - 1)

    def rel(pa, pb):
        return synth._pose_rel(pa[None], pb[None])[0]

    for nid, p in zip(g["ids"], g["init"]):
        add_node(int(nid), p)
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
        add_edge(int(a), int(b), z, c)
    assert s.Compute()
    truth = g["truth"]
    roll, live = [], []
    checked = 0
    for k in range(12):
        m = 60 + 9 * k
        tk = truth[m] + np.array([0.3, -0.2, 0.05])
        nid = 10000 + k
        add_node(nid, tk + rng.normal(0, [0.05, 0.05, 0.02]))
        if live:
            add_edge(live[-1], nid, rel(roll[-1], tk) + rng.normal(0, [0.03, 0.03, 0.01]), cov)
        add_edge(m, nid, rel(truth[m], tk) + rng.normal(0, [0.03, 0.03, 0.01]), cov)
        roll.append(tk)
        live.append(nid)
        if len(live) <= BUFFER:
            continue
        old = live.pop(0)
        adj = [edges[j][0] if edges[j][1] == old else edges[j][1] for j in vedges[old]]
        for v in adj:
            for j in list(vedges[v]):
                if old in edges[j][:2]:
                    vedges[v].remove(j)
                    assert s.RemoveConstraint(edges[j][0], edges[j][1])
                    edges[j] = (None, None) + edges[j][2:]
        assert s.RemoveNode(old)
        del vedges[old]
        slot = order.index(old)
        order[slot] = order[-1]
        order.pop()
        # the oracle from the solver's state before this solve, in the solver's slot order
        init = np.array([s.get_node(i) for i in order])
        pos = {nid_: i for i, nid_ in enumerate(order)}
        rem = [e for e in edges if e[0] is not None]
        ea = np.array([pos[e[0]] for e in rem])
        eb = np.array([pos[e[1]] for e in rem])
        xo, so = _oracle(t, init, ea, eb, np.array([e[2] for e in rem]), np.array([e[3] for e in rem]))
        assert s.Compute()
        sm = s.summary
        assert sm.uploaded_edges == len(rem) == s.num_edges() and s.num_nodes() == len(order)
        ids, xg = s.GetCorrections()
        assert np.array_equal(ids, order)
        assert (sm.iterations, sm.successful_steps, sm.linear_solves) == (so.iterations, so.successful_steps, so.linear_solves), \
            (k, (sm.iterations, sm.successful_steps, sm.linear_solves), (so.iterations, so.successful_steps, so.linear_solves))
        assert abs(sm.final_cost - so.final_cost) <= 1e-8 * so.final_cost + 1e-18, (k, sm.final_cost, so.final_cost)
        d = xg - xo
        d[:, 2] = synth.wrap(d[:, 2])
        assert np.abs(d[:, :2]).max() < 1e-4 and np.abs(d[:, 2]).max() < 1e-5, (k, np.abs(d).max(0))
        assert np.array_equal(xg[0], init[0])     # the map's first node stays the anchor
        checked += 1
    assert checked == 12 - BUFFER
