"""GPU occupancy grid (b200og_*) on the crafted reference fixtures (tests/golden/make_occupancy_edge_golden.py) and, at shapes
the reference cannot take (one laser per process), against the C port: ragged stores, stores that cross the pinned staging
halves, very fine and very coarse grids; handle semantics (streams, two handles, clear + reload, fetch without a build) and
the refusals.  Every grid must be bit-exact: dimensions, offset, cell bytes, both counters and toNavMap."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
from golden import make_occupancy_edge_golden as E
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "occupancy_edge_golden.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]


def as_dict(g: api.OccupancyGrid):
    cells, ps, ht = g.GetData(counters=True)
    return dict(width=g.GetWidth(), height=g.GetHeight(), stride=g.GetWidthStep(), offset=g.GetOffset(), cells=cells,
                passes=ps, hits=ht)


def assert_same(a, b):
    assert (a["width"], a["height"], a["stride"]) == (b["width"], b["height"], b["stride"])
    assert np.array_equal(a["offset"], b["offset"])
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


def assert_nav(g: api.OccupancyGrid, cells):
    nav = g.toNavMap()
    c = cells[:, :g.GetWidth()]
    assert nav.shape == (g.GetHeight(), g.GetWidth())
    assert np.array_equal(nav, np.where(c == 100, 100, np.where(c == 255, 0, -1)).astype(np.int8))


def laser(rt=12.0):
    return api.LaserRangeFinder(range_threshold=rt)


@pytest.mark.parametrize("name", NAMES)
def test_matches_edge_golden(name):
    """the stored reference points go in (the GPU host's libm stays out of the comparison), except for far_*, whose points
    are recomputed here and must first equal the reference's"""
    res, rt, mp, th = H.occupancy_params(Z[f"{name}/params"])
    if name.startswith("far_"):
        ranges, poses = E.far_inputs(name)
        pts = api.point_readings(ranges, poses, laser(rt))
        assert H.digest(pts) == Z[f"{name}/points_digest"][0], "host libm differs from the reference's: far_* points"
    else:
        ranges, poses, pts = Z[f"{name}/ranges"], Z[f"{name}/poses"], Z[f"{name}/points"]
    g = api.OccupancyGrid.CreateFromScans(api.ScanBlock(ranges, poses, laser(rt), points=pts), res, mp, th)
    got = as_dict(g)
    H.assert_occupancy_equals_golden(got, Z, name)
    assert_nav(g, got["cells"])


# ---------------------------------------------------------------------------------------------------------------------------
# against the port
# ---------------------------------------------------------------------------------------------------------------------------
class Store:
    """flat ranges / points of a ragged set of scans and their scan records (shared by the GPU and the port)"""

    def __init__(self, ranges_list, points_list, poses, counts=None):
        self.ranges = np.ascontiguousarray(np.concatenate(ranges_list), dtype=np.float64)
        self.points = np.ascontiguousarray(np.concatenate(points_list), dtype=np.float64).reshape(-1, 2)
        self.poses = np.asarray(poses, dtype=np.float64).reshape(-1, 3)
        counts = [len(r) for r in ranges_list] if counts is None else counts
        self.rec = H.scan_records(self.ranges, self.points, counts, self.poses)

    def ptr(self, lo=0, hi=None):
        return C.cast(self.rec[lo:hi].ctypes.data, C.POINTER(api.CScan))

    def __len__(self):
        return len(self.rec)


def fan(n, pose, rng, amin=synth.ANGLE_MIN, inc=synth.ANGLE_INC, lo=0.05, hi=35.0):
    """n readings of one scan (a few inf / NaN, some beyond the range threshold) and their points"""
    r = rng.uniform(lo, hi, n)
    r[rng.random(n) < 0.03] = np.inf
    r[rng.random(n) < 0.01] = np.nan
    a = pose[2] + amin + np.arange(n) * inc
    return r, np.column_stack([pose[0] + r * np.cos(a), pose[1] + r * np.sin(a)])


def gpu_grid(store, res, rt=12.0, mp=2, th=0.1, lo=0, hi=None):
    g = api.OccupancyGrid(res, laser(rt), mp, th)
    n = len(store) if hi is None else hi - lo
    assert api.lib().b200og_add_scans(g._h, store.ptr(lo, hi), n) == api.OK
    return g.Build()


def check_vs_port(store, res, rt=12.0, mp=2, th=0.1):
    g = gpu_grid(store, res, rt, mp, th)
    exp = H.port_occupancy(store.rec, res, rt, mp, th)
    got = as_dict(g)
    assert_same(got, exp)
    assert_nav(g, got["cells"])
    return got


def test_ragged_store_with_crafted_scans():
    """scans of 1, 31, 32, 33 and 8192 beams (other lasers) in one store with the crafted exact-axis scans"""
    rng = np.random.default_rng(3)
    rr, pp, poses = [], [], []
    for n in (1, 31, 32, 33, 8192, 33, 1, 32):
        pose = np.array([rng.uniform(2, 18), rng.uniform(2, 14), rng.uniform(-3, 3)])
        r, p = fan(n, pose, rng, inc=(synth.ANGLE_MAX - synth.ANGLE_MIN) / max(n - 1, 1), hi=14.0)
        rr.append(r); pp.append(p); poses.append(pose)
    for name in ("half_sensor_r1", "fma_clip_r005", "merge_lane31"):
        for s in range(len(Z[f"{name}/ranges"])):
            rr.append(Z[f"{name}/ranges"][s]); pp.append(Z[f"{name}/points"][s]); poses.append(Z[f"{name}/poses"][s])
    st = Store(rr, pp, poses)
    for res in (0.05, 1.0):
        got = check_vs_port(st, res)
        assert got["hits"].sum() > 0


def test_many_one_beam_scans_in_one_call():
    """600,000 one-beam scans: the readings cross a 2^20-double staging half and the sensors the 524,288-scan slice"""
    rng = np.random.default_rng(4)
    S = 600_000
    poses = np.column_stack([rng.uniform(0, 30, S), rng.uniform(0, 20, S), rng.uniform(-3, 3, S)])
    r = rng.uniform(0.05, 20.0, S)
    r[rng.random(S) < 0.02] = np.inf
    pts = poses[:, :2] + r[:, None] * np.column_stack([np.cos(poses[:, 2]), np.sin(poses[:, 2])])
    st = Store([r], [pts], poses, counts=np.ones(S, dtype=np.int64))
    got = check_vs_port(st, 0.1)
    assert got["passes"].sum() > S


def test_one_scan_longer_than_a_staging_half():
    """one scan of 600,000 beams: its 1.2 M point doubles cross a pinned half in the middle of the scan"""
    rng = np.random.default_rng(5)
    pose = np.array([10.0, 8.0, 0.3])
    r, p = fan(600_000, pose, rng, amin=-np.pi, inc=2 * np.pi / 600_000, hi=15.0)
    check_vs_port(Store([r], [p], [pose]), 0.05)


def test_fine_grid_over_a_large_world():
    """0.01 m cells over a 60 m world (millions of cells, lines of 1,000+ cells)"""
    world = synth.make_world(9, size=60.0)
    run = synth.make_mapping_run(9, 50, world=world)
    pts = api.point_readings(run["ranges"], run["poses"], laser())
    st = Store(list(run["ranges"]), list(pts), run["poses"])
    got = check_vs_port(st, 0.01)
    assert got["width"] * got["height"] > 5_000_000


def test_coarse_grid_over_the_full_run():
    """2 m cells over the 5,000-scan run: whole warps share cells (runs of 32 lanes) and counters grow large"""
    world = synth.make_world(3, size=60.0)
    run = synth.make_mapping_run(3, 5000, world=world, odd_readings=False)
    pts = api.point_readings(run["ranges"], run["poses"], laser())
    st = Store(list(run["ranges"]), list(pts), run["poses"])
    got = check_vs_port(st, 2.0)
    assert got["passes"].max() > 100_000


# ---------------------------------------------------------------------------------------------------------------------------
# handle semantics
# ---------------------------------------------------------------------------------------------------------------------------
def fixture_store(*names):
    rr, pp, poses = [], [], []
    for name in names:
        for s in range(len(Z[f"{name}/ranges"])):
            rr.append(Z[f"{name}/ranges"][s]); pp.append(Z[f"{name}/points"][s]); poses.append(Z[f"{name}/poses"][s])
    return Store(rr, pp, poses)


def test_set_stream_and_back():
    import torch
    st = fixture_store("merge_r1", "merge_alt_inf")
    exp = H.port_occupancy(st.rec, 0.05, 12.0)
    g = api.OccupancyGrid(0.05, laser())
    s = torch.cuda.Stream()
    g.set_stream(s.cuda_stream)
    assert api.lib().b200og_add_scans(g._h, st.ptr(), len(st)) == api.OK
    g.Build()
    assert_same(as_dict(g), exp)
    g.set_stream(0)
    g.Build()
    assert_same(as_dict(g), exp)
    assert_nav(g, exp["cells"])


def test_two_handles_interleaved_on_two_streams():
    """add / build alternate between two handles on two torch streams; the stores grow over several calls (buffer
    regrowth keeps what was uploaded)"""
    import torch
    a, b = fixture_store("merge_r1", "merge_near_far", "half_end_r005"), fixture_store("merge_alt_inf", "fma_clip_r1")
    ga, gb = api.OccupancyGrid(0.05, laser()), api.OccupancyGrid(0.1, laser())
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ga.set_stream(sa.cuda_stream)
    gb.set_stream(sb.cuda_stream)
    cuts_a, cuts_b = np.linspace(0, len(a), 5).astype(int), np.linspace(0, len(b), 4).astype(int)
    for k in range(4):
        if k < len(cuts_a) - 1:
            assert api.lib().b200og_add_scans(ga._h, a.ptr(cuts_a[k], cuts_a[k + 1]), int(cuts_a[k + 1] - cuts_a[k])) == api.OK
            ga.Build()
        if k < len(cuts_b) - 1:
            assert api.lib().b200og_add_scans(gb._h, b.ptr(cuts_b[k], cuts_b[k + 1]), int(cuts_b[k + 1] - cuts_b[k])) == api.OK
            gb.Build()
    assert (ga.NumScans(), gb.NumScans()) == (len(a), len(b))
    assert_same(as_dict(ga), H.port_occupancy(a.rec, 0.05, 12.0))
    assert_same(as_dict(gb), H.port_occupancy(b.rec, 0.1, 12.0))


def test_clear_and_reload_smaller_store():
    """a smaller grid after a bigger one: no counters of the first build survive"""
    big, small = fixture_store("merge_alt_inf", "merge_r1"), fixture_store("update_default")
    g = gpu_grid(big, 1.0)
    assert_same(as_dict(g), H.port_occupancy(big.rec, 1.0, 12.0))
    g.ClearScans()
    assert api.lib().b200og_add_scans(g._h, small.ptr(), len(small)) == api.OK
    g.Build()
    assert_same(as_dict(g), H.port_occupancy(small.rec, 1.0, 12.0))


def test_fetch_after_add_without_build():
    st = fixture_store("update_default")
    g = gpu_grid(st, 1.0)
    assert api.lib().b200og_add_scans(g._h, st.ptr(), len(st)) == api.OK
    cells = np.zeros(g.GetHeight() * g.GetWidthStep(), dtype=np.uint8)
    assert api.lib().b200og_fetch(g._h, cells.ctypes.data_as(C.POINTER(C.c_uint8)), None, None) == api.ERR_NOT_FOUND
    nav = np.zeros(g.GetHeight() * g.GetWidth(), dtype=np.int8)
    assert api.lib().b200og_fetch_nav(g._h, nav.ctypes.data_as(C.POINTER(C.c_int8))) == api.ERR_NOT_FOUND
    g.Build()
    assert g.NumScans() == 2 * len(st)
    cells, ps, ht = g.GetData(counters=True)
    exp = H.port_occupancy(st.rec, 1.0, 12.0)
    assert np.array_equal(ps, 2 * exp["passes"]) and np.array_equal(ht, 2 * exp["hits"])


# ---------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------
def build_raw(store, res, rt=12.0):
    g = api.OccupancyGrid(res, laser(rt))
    assert api.lib().b200og_add_scans(g._h, store.ptr(), len(store)) == api.OK
    info = api.OgInfo(7, 7, 7, (C.c_double * 2)(7.0, 7.0))
    rc = api.lib().b200og_build(g._h, C.byref(info))
    return rc, info, g


def test_refuses_more_than_2_31_cells():
    inf = np.full(4, np.inf)
    st = Store([inf, inf], [np.zeros((4, 2)), np.zeros((4, 2))], [[0.0, 0.0, 0.0], [60.0, 40.0, 0.0]])
    rc, info, g = build_raw(st, 0.001)                       # 60,000 x 40,000 cells
    assert rc == api.ERR_UNSUPPORTED
    assert (info.width, info.height, info.stride, info.offset[0], info.offset[1]) == (0, 0, 0, 0.0, 0.0)
    cells = np.zeros(8, dtype=np.uint8)
    assert api.lib().b200og_fetch(g._h, cells.ctypes.data_as(C.POINTER(C.c_uint8)), None, None) == api.ERR_NOT_FOUND


def test_refuses_a_nan_sensor_position():
    r = np.array([5.0, np.inf])
    st = Store([r], [np.full((2, 2), np.nan)], [[np.nan, 1.0, 0.0]])
    rc, info, _ = build_raw(st, 0.05)
    assert rc == api.ERR_UNSUPPORTED and (info.width, info.height, info.stride) == (0, 0, 0)


def test_refuses_a_beam_longer_than_2_24_cells():
    """res 1.5e-6 m, range threshold 29 m: a 29.5 m reading is traced over 1.9e7 cells.  The reference would trace it; the
    kernel reports it instead (a corrupt pose or resolution).  1e-6 m itself is a zero resolution to the reference
    (DoubleEqual with KT_TOLERANCE, Karto.h:5916-5918)"""
    with pytest.raises(api.B200Error) as e:
        api.OccupancyGrid(1e-6)
    assert e.value.code == api.ERR_INVALID_ARG
    st = Store([np.array([29.5]), np.array([np.inf])], [np.array([[29.5, 0.0]]), np.array([[np.inf, 0.0]])],
               [[0.0, 0.0, 0.0], [29.0, 1.5e-6, 0.0]])
    rc, info, _ = build_raw(st, 1.5e-6, rt=29.0)
    assert rc == api.ERR_UNSUPPORTED and (info.width, info.height, info.stride) == (0, 0, 0)
