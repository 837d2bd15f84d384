"""GPU parity of the occupancy grid (b200og_*, include/b200slam.h) with the oracle and the reference-generated
fixtures: dimensions, offset, cell bytes and both counters must be identical (integer work: bit-exact)."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
from oracle import karto_port as P
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "occupancy_golden.npz")
CASES = ["coarse_strict", "default", "one_scan", "short_threshold"]


def as_dict(g: api.OccupancyGrid):
    cells, ps, ht = g.GetData(counters=True)
    return dict(width=g.GetWidth(), height=g.GetHeight(), stride=g.GetWidthStep(), offset=g.GetOffset(), cells=cells,
                passes=ps, hits=ht)


def oracle_grid(ranges, poses, res, rt=12.0, mp=2, th=0.1):
    return P.occupancy(H.port_scans(ranges, poses), res, rt, H.LASER["min_range"], H.LASER["max_range"], mp, th)


def assert_same(a, b):
    assert (a["width"], a["height"], a["stride"]) == (b["width"], b["height"], b["stride"])
    assert np.array_equal(a["offset"], b["offset"])
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("name", CASES)
def test_matches_reference_golden(name):
    z = np.load(GOLDEN)
    res, rt, mp, th = z[f"{name}/params"]
    blk = H.gpu_block(z[f"{name}/ranges"], z[f"{name}/poses"], range_threshold=rt)
    g = api.OccupancyGrid.CreateFromScans(blk, res, 2 if mp < 0 else int(mp), 0.1 if th < 0 else th)
    H.assert_occupancy_equals_golden(as_dict(g), z, name)
    assert g.launch_count() >= 3


@pytest.mark.parametrize("seed,n,res,mp,th", [(0, 40, 0.05, 2, 0.1), (1, 25, 0.1, 4, 0.25), (2, 12, 0.02, 0, 0.05), (3, 60, 0.03, 2, 0.1)])
def test_matches_oracle(seed, n, res, mp, th):
    run = synth.make_mapping_run(seed, n, inf_frac=0.03)
    g = api.OccupancyGrid.CreateFromScans(H.gpu_block(run["ranges"], run["poses"]), res, mp, th)
    assert_same(as_dict(g), oracle_grid(run["ranges"], run["poses"], res, 12.0, mp, th))


def test_nav_map_and_incremental_store():
    run = synth.make_mapping_run(5, 30)
    exp = oracle_grid(run["ranges"], run["poses"], 0.05)
    g = api.OccupancyGrid(0.05, H.gpu_block(run["ranges"][:1], run["poses"][:1]).laser)
    for lo, hi in ((0, 7), (7, 8), (8, 30)):       # scans arrive as the mapper processes them
        g.AddScans(H.gpu_block(run["ranges"][lo:hi], run["poses"][lo:hi]))
    assert g.NumScans() == 30
    g.Build()
    assert_same(as_dict(g), exp)
    nav = g.toNavMap()                              # vis_utils::toNavMap
    cells = exp["cells"][:, :exp["width"]]
    assert nav.shape == (exp["height"], exp["width"])
    assert np.array_equal(nav == 100, cells == 100) and np.array_equal(nav == 0, cells == 255) and np.array_equal(nav == -1, cells == 0)
    # a second build over the same store gives the same bytes (counters are re-zeroed)
    g.Build()
    assert_same(as_dict(g), exp)
    # poses moved by a loop closure: clear + reload
    g.ClearScans()
    assert g.NumScans() == 0
    moved = run["poses"] + np.array([0.31, -0.17, 0.02])
    g.AddScans(H.gpu_block(run["ranges"], moved))
    g.Build()
    assert_same(as_dict(g), oracle_grid(run["ranges"], moved, 0.05))


def test_empty_and_rejected_inputs():
    assert api.OccupancyGrid.CreateFromScans(None, 0.05) is None            # reference: NULL (Karto.h:5950-5952)
    g = api.OccupancyGrid(0.05)
    with pytest.raises(api.B200Error) as e:
        g.Build()
    assert e.value.code == api.ERR_NOT_FOUND
    with pytest.raises(api.B200Error) as e:
        api.OccupancyGrid(0.0)                                               # "Resolution cannot be 0" (Karto.h:5916-5918)
    assert e.value.code == api.ERR_INVALID_ARG
    h = C.c_void_p()
    info = api.OgInfo()
    p = api.OgParams()
    api.lib().b200og_default_params(C.byref(p))
    assert (p.min_pass_through, p.occupancy_threshold) == (2, 0.1)
    assert api.lib().b200og_create_from_scans(C.byref(p), None, 0, C.byref(info), C.byref(h)) == api.ERR_NOT_FOUND and not h.value


def test_ragged_scans_and_all_readings_ignored():
    """scans with different beam counts (two lasers) and a scan whose readings are all out of range"""
    run = synth.make_mapping_run(8, 6)
    full = H.gpu_block(run["ranges"], run["poses"])
    # every second scan keeps only its first 400 beams; the last scan has nothing usable
    rr = [run["ranges"][s][:400] if s % 2 else run["ranges"][s] for s in range(6)]
    rr[5] = np.full(1081, np.inf)
    pts = [api.point_readings(rr[s] if len(rr[s]) == 1081 else np.pad(rr[s], (0, 681)), run["poses"][s], full.laser)[0][:len(rr[s])] for s in range(6)]
    arr = (api.CScan * 6)()
    keep = []
    for s in range(6):
        r = np.ascontiguousarray(rr[s]); p = np.ascontiguousarray(pts[s])
        keep += [r, p]
        arr[s].n = len(r)
        arr[s].ranges = r.ctypes.data_as(C.POINTER(C.c_double))
        arr[s].points_xy = p.ctypes.data_as(C.POINTER(C.c_double))
        arr[s].sensor_pose = (C.c_double * 3)(*run["poses"][s])
    g = api.OccupancyGrid(0.05, full.laser)
    assert api.lib().b200og_add_scans(g._h, arr, 6) == api.OK
    g.Build()
    parr = (P.KpScan * 6)()
    for s in range(6):
        parr[s] = P.KpScan(len(rr[s]), keep[2 * s].ctypes.data_as(C.POINTER(C.c_double)), keep[2 * s + 1].ctypes.data_as(C.POINTER(C.c_double)),
                           (C.c_double * 3)(*run["poses"][s]))
    exp = P.occupancy_array(parr, 6, 0.05, 12.0, 0.1, 30.0, 2, 0.1)
    got = as_dict(g)
    assert (got["width"], got["height"], got["stride"]) == (exp["width"], exp["height"], exp["stride"])
    assert np.array_equal(got["offset"], exp["offset"])
    assert np.array_equal(got["passes"], exp["passes"]) and np.array_equal(got["cells"], exp["cells"])


def test_full_size_map_properties():
    """cfg3-sized input (5,000 scans): identical to the oracle, and the size-independent invariants hold"""
    world = synth.make_world(3, size=60.0)
    run = synth.make_mapping_run(3, 5000, world=world, odd_readings=False)
    blk = H.gpu_block(run["ranges"], run["poses"])
    g = api.OccupancyGrid.CreateFromScans(blk, 0.05)
    got = as_dict(g)
    ps, ht = got["passes"].astype(np.int64), got["hits"].astype(np.int64)
    assert (ht <= ps).all() and not got["cells"][:, got["width"]:].any()
    r = run["ranges"]
    traced = (r > 0.1) & (r < 30.0)
    ends = traced & (r < 12.0 - 1e-6)
    assert ht.sum() <= ends.sum() and ht.sum() >= 0.99 * ends.sum()          # a hit per valid end point inside the grid
    assert ps.sum() >= ht.sum() + traced.sum()                                # >= 1 traced cell per beam + its end point
    exp = oracle_grid(run["ranges"], run["poses"], 0.05)
    assert_same(got, exp)
