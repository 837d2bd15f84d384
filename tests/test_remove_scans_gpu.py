"""In-place scan removal from the resident map store (b200og_remove_scans, OccupancyGrid.RemoveScans): after any removal the
store must build exactly what a fresh handle loaded with the surviving scans builds (their transformed values after a
transform): dimensions, offset, cell bytes, both counters, stored boxes, for whole-store and range builds.  Ragged stores,
stores that cross the pinned staging halves, transformed stores with authoritative boxes, streams and two handles, and
refusals that must leave the store unchanged."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from slam_toolbox_b200 import api, merge_maps, synth

pytestmark = pytest.mark.gpu
LASER = api.LaserRangeFinder()


class Store:
    """flat ranges / points of a ragged set of scans and their scan records; the records of any subset load a fresh handle"""

    def __init__(self, counts, seed):
        rng = np.random.default_rng(seed)
        world = synth.make_world(seed)
        poses = synth.chain_poses(world, synth.free_pose(world, rng), len(counts), rng, step=0.4)
        rr, pp = [], []
        for n, p in zip(counts, poses):
            r = rng.uniform(0.05, 35.0, n)
            r[rng.random(n) < 0.03] = np.inf
            r[rng.random(n) < 0.01] = np.nan
            a = p[2] + synth.ANGLE_MIN + np.arange(n) * (2 * np.pi / max(n, 1))
            rr.append(r)
            pp.append(np.column_stack([p[0] + r * np.cos(a), p[1] + r * np.sin(a)]))
        self.ranges = np.ascontiguousarray(np.concatenate(rr))
        self.points = np.ascontiguousarray(np.concatenate(pp)).reshape(-1, 2)
        self.rec = H.scan_records(self.ranges, self.points, list(counts), poses)

    def load(self, g, idx=None):
        rec = self.rec if idx is None else np.ascontiguousarray(self.rec[np.asarray(idx, dtype=np.int64)])
        if len(rec):
            assert api.lib().b200og_add_scans(g._h, C.cast(rec.ctypes.data, C.POINTER(api.CScan)), len(rec)) == api.OK
        return g

    def __len__(self):
        return len(self.rec)


def as_dict(g):
    cells, ps, ht = g.GetData(counters=True)
    return dict(width=g.GetWidth(), height=g.GetHeight(), stride=g.GetWidthStep(), offset=g.GetOffset(), cells=cells,
                passes=ps, hits=ht)


def assert_same(a, b):
    assert (a["width"], a["height"], a["stride"]) == (b["width"], b["height"], b["stride"])
    assert np.asarray(a["offset"]).tobytes() == np.asarray(b["offset"]).tobytes()
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


def assert_same_store(g, fresh, ranges=()):
    """whole-store build, range builds and the stored boxes of g equal those of fresh"""
    assert g.NumScans() == fresh.NumScans()
    if fresh.NumScans() == 0:
        with pytest.raises(api.B200Error) as e:
            g.Build()
        assert e.value.code == api.ERR_NOT_FOUND
        return
    assert_same(as_dict(g.Build()), as_dict(fresh.Build()))
    for first, count in ranges:
        assert_same(as_dict(g.Build(first, count)), as_dict(fresh.Build(first, count)))
    assert np.array_equal(g.ScanBoxes(), fresh.ScanBoxes())


def remove(g, alive, idx):
    """RemoveScans on g; alive (original scan numbers in store order) follows"""
    g.RemoveScans(idx)
    keep = np.ones(len(alive), dtype=bool)
    keep[np.asarray(idx, dtype=np.int64)] = False
    return [a for a, k in zip(alive, keep) if k]


RAGGED = [1081, 1, 31, 32, 33, 0, 2000, 1081, 64, 1081, 7, 1081, 8192, 1081, 1081, 33, 1, 1081, 500, 1081] * 3


@pytest.mark.parametrize("res", [0.05, 0.1])
def test_random_removals_on_a_ragged_store_equal_a_fresh_handle(res):
    """removal rounds (random sets, the first scan, the last scan, a middle run) interleaved with appends; after each round
    the store equals a fresh handle loaded with the survivors, whole-store and range builds and boxes alike"""
    rng = np.random.default_rng(11)
    st = Store(RAGGED, 5)
    g = api.OccupancyGrid(res, LASER)
    st.load(g, range(40))
    alive = list(range(40))
    nxt = 40
    rounds = [None, [0], "last", "run", None, None]
    for k, kind in enumerate(rounds):
        n = g.NumScans()
        if kind is None:
            idx = np.sort(rng.choice(n, size=int(rng.integers(1, max(2, n // 3))), replace=False))
        elif kind == "last":
            idx = [n - 1]
        elif kind == "run":
            idx = list(range(n // 3, n // 3 + 5))
        else:
            idx = kind
        alive = remove(g, alive, idx)
        fresh = st.load(api.OccupancyGrid(res, LASER), alive)
        m = len(alive)
        assert_same_store(g, fresh, [(0, 1), (m // 2, m - m // 2), (1, m - 2)])
        if nxt < len(st):
            add = list(range(nxt, min(nxt + 4, len(st))))
            st.load(g, add)
            alive += add
            nxt += len(add)


def test_store_across_the_staging_halves():
    """1,200 scans of 1,081 beams (the points cross both 8 MB pinned halves twice); remove a random quarter, then the rest"""
    rng = np.random.default_rng(12)
    st = Store([1081] * 1200, 6)
    g = st.load(api.OccupancyGrid(0.05, LASER))
    idx = np.sort(rng.choice(1200, 300, replace=False))
    alive = remove(g, list(range(1200)), idx)
    assert_same_store(g, st.load(api.OccupancyGrid(0.05, LASER), alive), [(100, 700)])
    alive = remove(g, alive, np.arange(len(alive)))
    assert alive == [] and g.NumScans() == 0
    assert_same_store(g, api.OccupancyGrid(0.05, LASER))
    st.load(g, range(10))   # an emptied store fills again like a new one
    assert_same_store(g, st.load(api.OccupancyGrid(0.05, LASER), range(10)))


def submaps(n):
    """three submaps of n scans each, apart in the world"""
    out = []
    for k, seed in enumerate((31, 32, 33)):
        run = synth.make_mapping_run(seed, n)
        p = run["poses"].copy()
        p[:, 0] += 40.0 * k
        out.append(api.ScanBlock(run["ranges"], p, LASER))
    return out


def transforms(rng, k):
    return [merge_maps.Transform.from_quaternion(merge_maps.quaternion_yaw(rng.uniform(-3, 3)), [rng.uniform(-5, 5), rng.uniform(-5, 5), 0.0])
            for _ in range(k)]


def test_removal_after_transform_keeps_authoritative_boxes():
    """after transforms the stored boxes (corner boxes, not the points' box) size every build; a removal must carry them
    with their scans.  Survivors of each submap are loaded into a fresh handle and given the same corrections.  Scans
    appended after the transform (no stored box yet) are in the store too."""
    rng = np.random.default_rng(13)
    blocks = submaps(60)
    extra = api.ScanBlock(synth.make_mapping_run(34, 10)["ranges"], synth.make_mapping_run(34, 10)["poses"], LASER)
    g = api.OccupancyGrid(0.05, LASER)
    for b in blocks:
        g.AddScans(b)
    ts = transforms(rng, 4)
    g.TransformScans(0, 60, ts[0].basis, ts[0].origin)
    g.TransformScans(60, 60, ts[1].basis, ts[1].origin)
    g.TransformScans(60, 60, ts[2].basis, ts[2].origin)   # compounded
    g.AddScans(extra)
    idx = np.sort(np.concatenate([rng.choice(60, 12, replace=False), 60 + rng.choice(60, 20, replace=False),
                                  120 + rng.choice(60, 5, replace=False), [183, 185]]))
    g.RemoveScans(idx)
    keep = [np.setdiff1d(np.arange(60), idx[(idx >= 60 * i) & (idx < 60 * (i + 1))] - 60 * i) for i in range(3)]
    keep_extra = np.setdiff1d(np.arange(10), idx[idx >= 180] - 180)
    fresh = api.OccupancyGrid(0.05, LASER)
    subs = [api.ScanBlock(b.ranges[k], b.poses[k], LASER) for b, k in zip(blocks, keep)]
    for b in subs:
        fresh.AddScans(b)
    n0, n1 = len(keep[0]), len(keep[1])
    fresh.TransformScans(0, n0, ts[0].basis, ts[0].origin)
    fresh.TransformScans(n0, n1, ts[1].basis, ts[1].origin)
    fresh.TransformScans(n0, n1, ts[2].basis, ts[2].origin)
    fresh.AddScans(api.ScanBlock(extra.ranges[keep_extra], extra.poses[keep_extra], LASER))
    assert_same_store(g, fresh, [(0, n0), (n0, n1), (n0 + n1, len(keep[2]))])
    # a later correction still compounds on the compacted store
    g.TransformScans(n0, n1, ts[3].basis, ts[3].origin)
    fresh.TransformScans(n0, n1, ts[3].basis, ts[3].origin)
    assert_same_store(g, fresh)


def test_trailing_removal_moves_nothing_and_others_launch_one_kernel():
    st = Store(RAGGED[:20], 7)
    g = st.load(api.OccupancyGrid(0.05, LASER))
    n0 = g.launch_count()
    alive = remove(g, list(range(20)), [17, 18, 19])
    assert g.launch_count() == n0 and g.kernel_ms() == 0.0
    assert_same_store(g, st.load(api.OccupancyGrid(0.05, LASER), alive))
    n0 = g.launch_count()
    alive = remove(g, alive, [3, 9])
    assert g.launch_count() == n0 + 1 and g.kernel_ms() > 0.0
    assert_same_store(g, st.load(api.OccupancyGrid(0.05, LASER), alive))


def test_caller_stream_and_two_handles():
    import torch
    st = Store(RAGGED, 8)
    rng = np.random.default_rng(14)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ga, gb = api.OccupancyGrid(0.05, LASER), api.OccupancyGrid(0.1, LASER)
    ga.set_stream(sa.cuda_stream)
    gb.set_stream(sb.cuda_stream)
    st.load(ga)
    st.load(gb)
    alive_a, alive_b = list(range(len(st))), list(range(len(st)))
    for _ in range(3):
        ia = np.sort(rng.choice(len(alive_a), 5, replace=False))
        ib = np.sort(rng.choice(len(alive_b), 7, replace=False))
        alive_a = remove(ga, alive_a, ia)
        alive_b = remove(gb, alive_b, ib)
        ga.Build()
        gb.Build()
    assert_same(as_dict(ga), as_dict(st.load(api.OccupancyGrid(0.05, LASER), alive_a).Build()))
    assert_same(as_dict(gb), as_dict(st.load(api.OccupancyGrid(0.1, LASER), alive_b).Build()))
    ga.set_stream(0)
    alive_a = remove(ga, alive_a, [0])
    assert_same_store(ga, st.load(api.OccupancyGrid(0.05, LASER), alive_a))


def test_refusals_leave_the_store_unchanged():
    rng = np.random.default_rng(15)
    st = Store(RAGGED[:20], 9)
    g = st.load(api.OccupancyGrid(0.05, LASER))
    t = transforms(rng, 1)[0]
    g.TransformScans(5, 10, t.basis, t.origin)
    before = as_dict(g.Build())
    boxes = g.ScanBoxes()
    L = api.lib()
    for bad in ([3, 3], [4, 2], [-1, 2], [2, 20], [0, 5, 5, 7], [19, 20]):
        with pytest.raises(api.B200Error) as e:
            g.RemoveScans(bad)
        assert e.value.code == api.ERR_INVALID_ARG
    assert L.b200og_remove_scans(g._h, None, 2) == api.ERR_INVALID_ARG
    assert L.b200og_remove_scans(g._h, None, -1) == api.ERR_INVALID_ARG
    one = (C.c_int32 * 1)(0)
    assert L.b200og_remove_scans(None, one, 1) == api.ERR_INVALID_ARG
    g.RemoveScans([])   # n = 0 is a no-op
    assert L.b200og_remove_scans(g._h, None, 0) == api.OK
    assert g.NumScans() == 20
    assert_same(as_dict(g.Build()), before)
    assert np.array_equal(g.ScanBoxes(), boxes)
