"""Two lasers through the reference's own mapper and the reference-side bindings.  Scans alternate between two named lasers in
blocks of six (replay.make_two_laser_trajectory), so karto's multi-sensor path runs: AddEdges links the first scan of the
new sensor to the other sensor's scans.  The second laser has a shorter threshold, a larger minimum range and a shorter
maximum range (replay.TWO_LASER).  The map is published every fifth step through the resident store
(karto::b200::ResidentOccupancyMap) and through the reference's CreateFromScans, and once more at the end through
CreateOccupancyGridFromScans.  Halfway, the second laser's maximum range changes, which must reload the resident store
exactly once.  The map-merge binding (karto::b200::SubmapStore) merges two submaps on different lasers.  Once with the
reference CPU matcher and once with the GPU matcher, both with the GPU solver."""
import os
import sys

import numpy as np
import pytest

import multilaser as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import replay  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not replay.available(), reason="oracle/_ref/libreplay_*.so not built")]

N_SCANS, SEED, EVERY = 90, 7, 5
CHANGE_STEP = 47                                   # (CHANGE_STEP + 1) % EVERY != 0: its publishes are the change's own
CHANGE = {"max_range": 14.0}                       # traces change, Update's boxes do not (they read the threshold and minimum)
PARAMS = dict(replay.YAML_PARAMS, correlation_search_space_smear_deviation=0.03, loop_search_space_dimension=4.0)
P_STEP, P_EQUAL, P_REMOVED, P_APPENDED, P_RELOADED = range(5)

_RUNS = {}


def runs():
    if not _RUNS:
        ranges, odom, _, sensors = replay.make_two_laser_trajectory(SEED, N_SCANS)
        for which in ("ref", "b200"):
            _RUNS[which] = replay.run(which, ranges, odom, PARAMS, map_resolution=0.05, publish_every=EVERY, sensors=sensors,
                                      laser2=replay.TWO_LASER, laser2_changes=[(CHANGE_STEP, CHANGE)])
        _RUNS["sensors"] = sensors
    return _RUNS["ref"], _RUNS["b200"]


def test_both_lasers_reach_the_map():
    a, b = runs()
    kept = b["kept"]
    assert (_RUNS["sensors"][kept] == 0).any() and (_RUNS["sensors"][kept] == 1).any()
    assert b["edges"] > len(kept) - 1   # loop or cross-sensor links beyond the chain


def test_gpu_matcher_equals_cpu_matcher():
    a, b = runs()
    assert np.array_equal(a["kept"], b["kept"])
    assert np.array_equal(a["poses"], b["poses"])
    assert np.array_equal(a["graph_ids"], b["graph_ids"]) and np.array_equal(a["graph_poses"], b["graph_poses"])
    assert a["edges"] == b["edges"]


@pytest.mark.parametrize("which", ["ref", "b200"])
def test_every_resident_publish_equals_the_reference(which):
    p = runs()[0 if which == "ref" else 1]["publishes"]
    assert len(p) == N_SCANS // EVERY + 3
    assert (p[:, P_EQUAL] == 1).all(), p[p[:, P_EQUAL] != 1]


@pytest.mark.parametrize("which", ["ref", "b200"])
def test_create_from_scans_binding_equals_the_reference(which):
    r = runs()[0 if which == "ref" else 1]
    for k in ("dims", "offset", "cells"):
        assert np.array_equal(r[f"map_gpu_{k}"], r[f"map_cpu_{k}"]), k


def test_a_changed_limit_reloads_exactly_once():
    """with the GPU matcher the driver counts CorrectPoses: of the two publishes after the change, with no scan in between,
    the first reloads and the second does not; the publish before the change left the store current"""
    p = runs()[1]["publishes"]
    at = p[p[:, P_STEP] == CHANGE_STEP]
    assert len(at) == 3
    assert at[1, P_RELOADED] == 1 and at[1, P_REMOVED] == 0
    assert at[2, P_RELOADED] == 0 and at[2, P_APPENDED] == 0 and at[2, P_REMOVED] == 0
    # the two lasers alone never reload the store: publishes of steps without a correction keep it
    assert (p[:, P_RELOADED] == 0).sum() >= 5


def test_submap_store_with_per_submap_lasers_equals_reference():
    name = "merge_rot"
    z = np.load(M.GOLDEN)
    c = {k: z[f"{name}/{k}"] for k in ("ranges", "poses", "laser_id", "laser_table")} | {"res": float(z[f"{name}/res"][0])}
    scans = M.ref_scans(c, "submap_store_")
    dims, off, cells = M.binding_merge(scans, z[f"{name}/submap"], z[f"{name}/corr"], c["res"])
    e = M.golden_grid(z, f"{name}/merged")
    assert list(dims) == e["dims"] and np.array_equal(off, e["offset"]) and np.array_equal(cells, e["cells"])
