"""slam_toolbox's lifelong mode removing scans from a mapping run, through the reference's own mapper: about 15 interior scans
leave as LifelongSlamToolbox::removeFromSlamGraph retires them (krep_remove_node: Mapper::RemoveNodeFromGraph, the sensor
manager's RemoveScan, then the vertex and the scan are freed), each picked from the mapper's edges by lifelong's guards
(replay.lifelong_candidates).  Around every removal the map is published through the resident b200og store and through the
reference's CreateFromScans; the publish right after a removal, before the next scan, takes the store's in-place removal
rather than the reload that follows a CorrectPoses.  Once with the reference CPU matcher and once with the GPU matcher, both
with the GPU solver."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import replay  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not replay.available(), reason="oracle/_ref/libreplay_*.so not built")]

N_SCANS, SEED = 160, 5
REMOVAL_STEPS = list(range(40, N_SCANS, 8))
PARAMS = dict(replay.YAML_PARAMS, correlation_search_space_smear_deviation=0.03, loop_search_space_dimension=4.0)
BUFFER = PARAMS["scan_buffer_size"]
# removals rows of replay._remove_node
STEP, ID, DEG, POS, STORED, RC, MV, ME, SN, SE, SAME = range(11)
# publishes rows of replay._publish_pair
P_STEP, P_EQUAL, P_REMOVED, P_APPENDED, P_RELOADED = range(5)

_RUNS = {}


def runs():
    if not _RUNS:
        ranges, odom, _ = replay.make_trajectory(SEED, N_SCANS)
        ev = [e for s in REMOVAL_STEPS for e in ((s, "publish"), (s, "remove_node", -1), (s, "publish"))]
        for which in ("ref", "b200"):
            _RUNS[which] = replay.run(which, ranges, odom, PARAMS, map_resolution=0.05, events=ev)
    return _RUNS["ref"], _RUNS["b200"]


def test_gpu_matcher_is_identical_under_removals():
    a, b = runs()
    assert np.array_equal(a["removals"], b["removals"])
    assert np.array_equal(a["poses"], b["poses"]) and np.array_equal(a["scan_ids"], b["scan_ids"])
    for k in ("edge_src", "edge_dst", "edge_diff", "edge_cov"):
        assert np.array_equal(a[k], b[k]), k
    assert a["graph_nodes"] == b["graph_nodes"]
    assert np.array_equal(a["graph_ids"], b["graph_ids"]) and np.array_equal(a["graph_poses"], b["graph_poses"])
    # loop closures ran the solver, and the final graph is what the removals left
    assert b["solver_computes"] > 0 and len(b["edge_src"]) > len(b["scan_ids"])
    assert np.array_equal(b["graph_ids"], np.sort(b["scan_ids"]))
    assert not set(b["removals"][:, ID].tolist()) & set(b["scan_ids"].tolist())


@pytest.mark.parametrize("which", ["ref", "b200"])
def test_removals_meet_the_guards_and_reach_the_solver(which):
    r = runs()[0 if which == "ref" else 1]
    rm = r["removals"]
    assert len(rm) == len(REMOVAL_STEPS) and (rm[:, RC] == 0).all()
    # lifelong's guards held when each scan went: not 0 or 1, scan_buffer_size older than the newest, two or more edges
    assert (rm[:, ID] > 1).all() and (rm[:, DEG] >= 2).all()
    assert (rm[:, POS] > 0).all() and (rm[:, POS] < rm[:, STORED] - 1).all()
    assert (rm[:, POS] <= rm[:, STORED] - 1 - BUFFER).all()
    # after every removal the solver holds the mapper's node set and as many edges as the mapper's graph
    assert (rm[:, MV] == rm[:, SN]).all() and (rm[:, ME] == rm[:, SE]).all() and (rm[:, SAME] == 1).all()
    assert (rm[:, MV] == rm[:, STORED] - 1).all()


@pytest.mark.parametrize("which", ["ref", "b200"])
def test_every_publish_equals_the_reference(which):
    p = runs()[0 if which == "ref" else 1]["publishes"]
    assert len(p) == 2 * len(REMOVAL_STEPS)
    assert (p[:, P_EQUAL] == 1).all(), p[p[:, P_EQUAL] != 1]


def test_publishes_after_removals_compact_in_place():
    """With the GPU matcher the driver counts CorrectPoses: the publish after a removal (no scan, no correction in between)
    removes exactly that scan from the store, interior ones included."""
    b = runs()[1]
    p, rm = b["publishes"], b["removals"]
    after = p[1::2]
    assert np.array_equal(after[:, P_STEP], rm[:, STEP])
    in_place = (after[:, P_REMOVED] == 1) & (after[:, P_RELOADED] == 0) & (after[:, P_APPENDED] == 0)
    assert in_place.sum() >= 5, after
    # an in-place removal of a scan that was neither the first nor the last stored one
    assert (in_place & (rm[:, POS] > 0) & (rm[:, POS] < rm[:, STORED] - 1)).any()
    # the publish before each removal left the store current: nothing was removed in place there
    assert (p[0::2, P_REMOVED] == 0).all()
