"""The multi-laser occupancy fixtures (tests/golden/make_multilaser_golden.py, from the reference) without a GPU: the host
oracle of tests/multilaser.py reproduces every case bit for bit, and each case depends on its scans' own lasers."""
from __future__ import annotations

import numpy as np
import pytest

import multilaser as M
from oracle import karto_port as P
from slam_toolbox_b200 import synth

Z = np.load(M.GOLDEN)
NAMES = ["thr_only", "minr_only", "maxr_only", "tolerance", "box_long", "interleaved", "no_inrange", "merge_rot"]


def case(name):
    return {k: Z[f"{name}/{k}"] for k in ("ranges", "poses", "lasers", "laser_id", "laser_table")} | {"res": float(Z[f"{name}/res"][0])}


def port_points(ranges, poses):
    return np.stack([P.point_readings(np.ascontiguousarray(r), np.ascontiguousarray(p), synth.ANGLE_MIN, synth.ANGLE_INC)
                     for r, p in zip(ranges, poses)])


def test_cases_match_the_generator():
    for name, c in M.cases().items():
        for k in ("ranges", "poses", "lasers", "laser_id", "laser_table"):
            assert np.array_equal(c[k], Z[f"{name}/{k}"], equal_nan=True), (name, k)
    assert sorted(M.cases()) == sorted(NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_host_oracle_equals_reference(name):
    c = case(name)
    pts = port_points(c["ranges"], c["poses"])
    assert M.sha(pts) == Z[f"{name}/points_sha"][0]
    M.assert_equals_golden(M.host_occupancy(c["ranges"], pts, c["poses"], c["lasers"], c["res"]), Z, name)


# what each case changes when every scan takes the first scan's laser: the limit the case is named for
ONE_LASER_DIFFERS = {
    "thr_only": "hits",       # the shorter threshold clips readings the longer one hits
    "minr_only": "passes",    # readings between the two minimum ranges are traced by one laser only
    "maxr_only": "passes",    # readings between the two maximum ranges are traced by one laser only
    "tolerance": "hits",      # the second laser's readings are below the first laser's tolerance band: 4 hits, not 2
    "box_long": "dims",       # the long laser's far points would size the grid from every scan
    "interleaved": "passes",
    "no_inrange": "dims",     # the second laser's scans would add their points to the box
    "merge_rot": "passes",
}


@pytest.mark.parametrize("name", NAMES)
def test_one_laser_for_the_map_differs(name):
    """the grid the map would get with the first scan's laser for every scan differs from the reference's in what the case
    was built for"""
    c = case(name)
    pts = port_points(c["ranges"], c["poses"])
    one = np.repeat(c["lasers"][:1], len(c["lasers"]), axis=0)
    g = M.host_occupancy(c["ranges"], pts, c["poses"], one, c["res"])
    e = M.golden_grid(Z, name)
    what = ONE_LASER_DIFFERS[name]
    if what == "dims":
        assert [g["width"], g["height"], g["stride"]] != e["dims"] or not np.array_equal(g["offset"], e["offset"])
    elif what == "hits":
        assert int(g["hits"].sum()) != e["sums"][1]
    else:
        assert int(g["passes"].sum()) != e["sums"][0]
    if name == "tolerance":
        assert int(g["hits"].sum()) == 4


def test_tolerance_hits_only_below_the_band():
    """per laser: threshold - KT_TOLERANCE - 1 ulp hits its end cell, threshold - KT_TOLERANCE and above do not"""
    assert M.golden_grid(Z, "tolerance")["sums"][1] == 2
    c = case("tolerance")
    for lid, lim in enumerate(c["laser_table"]):
        t = lim[0] - M.KT_TOLERANCE
        own = c["ranges"][c["laser_id"] == lid]
        finite = own[np.isfinite(own)]
        assert sorted(finite.tolist()) == sorted([float(np.nextafter(t, 0.0)), t, float(np.nextafter(t, np.inf))])


def test_no_inrange_laser_has_no_inrange_reading():
    c = case("no_inrange")
    rt, minr, _ = c["laser_table"][1]
    r = c["ranges"][c["laser_id"] == 1]
    assert len(r) and not np.any((r >= minr) & (r <= rt))


def test_box_long_is_set_by_the_long_laser():
    """with the long laser's scans left out of the box, the grid would be smaller"""
    c = case("box_long")
    pts = port_points(c["ranges"], c["poses"])
    boxes = [M.scan_box(c["ranges"][s], pts[s], c["poses"][s], c["lasers"][s]) for s in range(len(pts))]
    short = [M.scan_box(c["ranges"][s], pts[s], c["poses"][s], c["laser_table"][1]) for s in range(len(pts))]
    assert M.union(boxes) != M.union(short)
