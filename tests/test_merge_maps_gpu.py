"""Map merge on the GPU (b200og_transform_scans / b200og_build_range / b200og_scan_boxes, slam_toolbox_b200.merge_maps):
bit-exact against the reference's goldens (tests/golden/make_merge_golden.py), against the host restatement with the C
port's build (tests/merge_port.py) on larger submaps under random corrections and repeated moves, handle semantics and refusals, and the reference-side binding
(integration/merge_maps_b200.hpp) against the reference itself where oracle/_ref holds it."""
import math
import os

import numpy as np
import pytest

import helpers as H
import merge_port as MP
import merge_ref
from slam_toolbox_b200 import api, merge_maps, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "merge_golden.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]
LASER = api.LaserRangeFinder()
RT, MINR, MAXR = LASER.range_threshold, LASER.minimum_range, LASER.maximum_range


def as_dict(g):
    cells, ps, ht = g.GetData(counters=True)
    return dict(width=g.GetWidth(), height=g.GetHeight(), stride=g.GetWidthStep(), offset=g.GetOffset(), cells=cells,
                passes=ps, hits=ht)


def assert_same(a, b):
    assert (a["width"], a["height"], a["stride"]) == (b["width"], b["height"], b["stride"])
    assert np.asarray(a["offset"], dtype=np.float64).tobytes() == np.asarray(b["offset"], dtype=np.float64).tobytes()
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


def golden_store(name, res):
    g = api.OccupancyGrid(res, LASER)
    bounds = [0]
    for i in range(int(Z[f"{name}/nsub"][0])):
        p = f"{name}/sub{i}"
        g.AddScans(api.ScanBlock(Z[f"{p}/ranges"], Z[f"{p}/sensor"], LASER, points=Z[f"{p}/points"]))
        bounds.append(g.NumScans())
    return g, bounds


@pytest.mark.parametrize("name", NAMES)
def test_matches_merge_golden(name):
    res = float(Z[f"{name}/res"][0])
    g, bounds = golden_store(name, res)
    for m, corr in enumerate(Z[f"{name}/corr"]):
        for i, c in enumerate(corr):
            g.TransformScans(bounds[i], bounds[i + 1] - bounds[i], c[:9].reshape(3, 3), c[9:])
        g.Build()
        H.assert_occupancy_equals_golden(as_dict(g), Z, f"{name}/m{m}")
        assert np.array_equal(g.ScanBoxes(), Z[f"{name}/m{m}/boxes"])


def test_corner_order_signed_zero_box():
    """the tool's corner order keeps -0 for a box whose corrected corners are -0 and +0"""
    g = api.OccupancyGrid(1.0, LASER)
    pts = np.array([[-1.0, 0.0], [1.0, 0.0]])
    g.AddScans(api.ScanBlock(np.array([[1.0, 1.0]]), np.array([[0.5, 0.0, 0.0]]), LASER, points=pts))
    assert np.array_equal(g.ScanBoxes(), [[-1.0, 0.0, 1.0, 0.0]])
    g.TransformScans(0, 1, [[0.0, -1.0, -0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]], [-0.0, 0.0, 0.0])
    box = g.ScanBoxes()[0]
    assert np.signbit(box[0]) and np.signbit(box[2]) and box[0] == 0.0 and box[2] == 0.0


# ---------------------------------------------------------------------------------------------------------------------------
# against the C port
# ---------------------------------------------------------------------------------------------------------------------------
def submaps(seeds, n):
    out = []
    for k, seed in enumerate(seeds):
        run = synth.make_mapping_run(seed, n)
        t = math.radians(25.0 * k)
        c, s = math.cos(t), math.sin(t)
        p = run["poses"].copy()
        p[:, 0], p[:, 1] = c * run["poses"][:, 0] - s * run["poses"][:, 1] + 40.0 * k, s * run["poses"][:, 0] + c * run["poses"][:, 1]
        p[:, 2] = synth.wrap(p[:, 2] + t)
        out.append(api.ScanBlock(run["ranges"], p, LASER))
    return out


def port_of(blocks):
    ranges = np.concatenate([b.ranges.ravel() for b in blocks])
    points = np.concatenate([b.points.reshape(-1, 2) for b in blocks])
    counts = [b.ranges.shape[1] for b in blocks for _ in range(len(b))]
    sensor = np.concatenate([b.poses[:, :2] for b in blocks])
    return MP.MergeStore(ranges, points, counts, sensor, RT, MINR, MAXR)


def random_correction(rng):
    t = rng.uniform(-math.pi, math.pi)
    return merge_maps.Transform.from_quaternion(merge_maps.quaternion_yaw(t), [rng.uniform(-5, 5), rng.uniform(-5, 5), 0.0])


def test_random_corrections_equal_port():
    """3 x 2,000-scan submaps, random corrections, three merges in a row (each compounding), plus a submap's own grid"""
    rng = np.random.default_rng(7)
    blocks = submaps((91, 92, 93), 2000)
    g = api.OccupancyGrid(0.05, LASER)
    for b in blocks:
        g.AddScans(b)
    port = port_of(blocks)
    bounds = [0, 2000, 4000, 6000]
    for _ in range(3):
        for i in range(3):
            t = random_correction(rng)
            g.TransformScans(bounds[i], 2000, t.basis, t.origin)
            port.transform(bounds[i], 2000, t.basis, t.origin)
        g.Build()
        assert_same(as_dict(g), port.build(0.05))
    g.Build(2000, 2000)
    assert_same(as_dict(g), port.build(0.05, 2000, 2000))


def test_merge_maps_kinematic_moves_equal_port():
    """MergeMapsKinematic: add three submaps, move markers, merge after each move; the port applies the same corrections"""
    blocks = submaps((94, 95, 96), 300)
    mm = merge_maps.MergeMapsKinematic(0.05, LASER)
    port = port_of(blocks)
    for k, b in enumerate(blocks):
        sid, nav, (cx, cy) = mm.AddSubmap(b)
        own = port_of([b]).build(0.05)
        assert sid == k + 1 and nav.shape == (own["height"], own["width"])
        assert cx == own["offset"][0] + own["width"] * 0.05 / 2.0 and cy == own["offset"][1] + own["height"] * 0.05 / 2.0
    for sid, x, y, yaw in ((2, 3.0, -1.0, 0.4), (3, -2.0, 4.0, -1.1), (2, 1.0, 1.0, 0.25)):
        mm.MoveSubmap(sid, x, y, yaw)
        grid = mm.Merge()
        for j, (first, count) in mm.ranges.items():
            t = mm.corrections[j]
            port.transform(first, count, t.basis, t.origin)
        assert_same(as_dict(grid), port.build(0.05))


def test_identity_equals_plain_build():
    blocks = submaps((97,), 40)
    a = api.OccupancyGrid(0.05, LASER)
    a.AddScans(blocks[0])
    a.Build()
    b = api.OccupancyGrid(0.05, LASER)
    b.AddScans(blocks[0])
    b.TransformScans(0, len(blocks[0]), np.eye(3), np.zeros(3))
    b.Build()
    assert_same(as_dict(a), as_dict(b))


def test_untransformed_box_union_equals_bbox_and_same_launches():
    """on a store never transformed: the per-scan boxes' union is today's bounding box, and b200og_build launches what it did"""
    for name in ("rot30", "three"):
        res = float(Z[f"{name}/res"][0])
        g, _ = golden_store(name, res)
        n0 = g.launch_count()
        g.Build()
        assert g.launch_count() - n0 == 3
        boxes = g.ScanBoxes()
        assert np.array_equal(boxes[:, :2].min(0), g.GetOffset())
        w = synth.grid_cell(boxes[:, 2].max(), boxes[:, 0].min(), 1.0 / res)
        h = synth.grid_cell(boxes[:, 3].max(), boxes[:, 1].min(), 1.0 / res)
        assert (w, h) == (g.GetWidth(), g.GetHeight())
        n1 = g.launch_count()
        g.Build()
        assert g.launch_count() - n1 == 3


def test_build_range_equals_separate_handle():
    blocks = submaps((98, 99), 50)
    g = api.OccupancyGrid(0.05, LASER)
    for b in blocks:
        g.AddScans(b)
    for k, (first, count) in enumerate(((0, 50), (50, 50))):
        one = api.OccupancyGrid.CreateFromScans(blocks[k], 0.05)
        g.Build(first, count)
        assert_same(as_dict(g), as_dict(one))
    t = merge_maps.Transform.from_quaternion(merge_maps.quaternion_yaw(0.7), [1.0, 2.0, 0.0])
    g.TransformScans(50, 50, t.basis, t.origin)
    one = api.OccupancyGrid(0.05, LASER)
    one.AddScans(blocks[1])
    one.TransformScans(0, 50, t.basis, t.origin)
    g.Build(50, 50)
    assert_same(as_dict(g), as_dict(one.Build()))


def test_clear_after_transform_is_fresh():
    blocks = submaps((100,), 30)
    g = api.OccupancyGrid(0.05, LASER)
    g.AddScans(blocks[0])
    g.TransformScans(0, 30, merge_maps.Transform.from_quaternion(merge_maps.quaternion_yaw(1.0), [0, 0, 0]).basis, np.zeros(3))
    g.ClearScans()
    g.AddScans(blocks[0])
    n0 = g.launch_count()
    g.Build()
    assert g.launch_count() - n0 == 3
    assert_same(as_dict(g), as_dict(api.OccupancyGrid.CreateFromScans(blocks[0], 0.05)))


def test_refusals():
    blocks = submaps((101,), 5)
    g = api.OccupancyGrid(0.05, LASER)
    g.AddScans(blocks[0])
    for first, count in ((-1, 2), (3, 3), (0, -1), (6, 0)):
        with pytest.raises(api.B200Error) as e:
            g.TransformScans(first, count, np.eye(3), np.zeros(3))
        assert e.value.code == api.ERR_INVALID_ARG
        with pytest.raises(api.B200Error) as e:
            g.Build(first, count)
        assert e.value.code == api.ERR_INVALID_ARG
    for bad in (np.nan, np.inf):
        b = np.eye(3)
        b[1, 0] = bad
        with pytest.raises(api.B200Error) as e:
            g.TransformScans(0, 5, b, np.zeros(3))
        assert e.value.code == api.ERR_INVALID_ARG
        with pytest.raises(api.B200Error) as e:
            g.TransformScans(0, 5, np.eye(3), [0.0, 0.0, bad])
        assert e.value.code == api.ERR_INVALID_ARG
    with pytest.raises(api.B200Error) as e:
        g.Build(2, 0)
    assert e.value.code == api.ERR_NOT_FOUND
    g.TransformScans(2, 0, np.eye(3), np.zeros(3))   # an empty range is a no-op
    g.Build()
    assert_same(as_dict(g), as_dict(api.OccupancyGrid.CreateFromScans(blocks[0], 0.05)))


def test_caller_stream_and_two_handles():
    import torch
    blocks = submaps((102, 103), 200)
    t = merge_maps.Transform.from_quaternion(merge_maps.quaternion_yaw(-0.6), [2.0, -3.0, 0.0])

    def run(stream=None):
        g = api.OccupancyGrid(0.05, LASER)
        if stream is not None:
            g.set_stream(stream)
        for b in blocks:
            g.AddScans(b)
        g.TransformScans(200, 200, t.basis, t.origin)
        return g
    base = as_dict(run().Build())
    s = torch.cuda.Stream()
    assert_same(as_dict(run(s.cuda_stream).Build()), base)
    a, b = run(), run()
    a.TransformScans(0, 200, t.basis, t.origin)
    b.TransformScans(0, 200, t.basis, t.origin)
    a.Build()
    b.Build()
    assert_same(as_dict(a), as_dict(b))
    assert not (a.GetWidth() == base["width"] and np.array_equal(a.GetOffset(), base["offset"]))


# ---------------------------------------------------------------------------------------------------------------------------
# the reference-side binding against the reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not merge_ref.available(), reason="oracle/_ref/libmerge_b200.so not built (no reference sources)")
@pytest.mark.parametrize("name", ["rot30", "compound", "three"])
def test_binding_equals_reference(name):
    """SubmapStore::Merge on the karto scans vs the reference's CreateFromScans on kref_transform_scan-ed copies"""
    res = float(Z[f"{name}/res"][0])
    store = merge_ref.SubmapStore(res)
    ref_scans = []
    for i in range(int(Z[f"{name}/nsub"][0])):
        ranges, poses = Z[f"{name}/sub{i}/ranges"], Z[f"{name}/sub{i}/poses"]
        mine = merge_ref.scans(ranges, poses, uid0=1000 * i)
        assert store.add_submap(mine) == i
        ref_scans.append(merge_ref.scans(ranges, poses, uid0=1000 * i))
    for corr in Z[f"{name}/corr"]:
        for i, c in enumerate(corr):
            assert store.apply(i, c[:9], c[9:]) == 0
            for s in ref_scans[i]:
                s.transform(c[:9], c[9:])
        ref = merge_ref.occupancy([s for sub in ref_scans for s in sub], res, counters=False)
        got = store.merge(res, ref["cells"].size + 8)
        assert got is not None
        info, off, cells = got
        assert info == [ref["width"], ref["height"], ref["stride"]]
        assert off.tobytes() == ref["offset"].tobytes()
        assert np.array_equal(cells[:ref["cells"].size], ref["cells"].ravel())
    store.close()
