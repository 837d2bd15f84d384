"""The map-merge fixtures (tests/golden/make_merge_golden.py) without a GPU: each crafted case detects the defect it was made
for (exact rational arithmetic for the fused multiply-add and half-cell cases), and the host restatement of the transform
with the C port's build over the stored boxes (tests/merge_port.py) equals the reference on every case, merge after merge."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import helpers as H
from golden import make_merge_golden as G
import merge_port as MP
from slam_toolbox_b200 import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "merge_golden.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]
RT, MINR, MAXR = H.LASER["range_threshold"], H.LASER["min_range"], H.LASER["max_range"]


def subs(name):
    return [dict(ranges=Z[f"{name}/sub{i}/ranges"], points=Z[f"{name}/sub{i}/points"], sensor=Z[f"{name}/sub{i}/sensor"])
            for i in range(int(Z[f"{name}/nsub"][0]))]


def port_store(name):
    ss = subs(name)
    ranges = np.concatenate([s["ranges"].ravel() for s in ss])
    points = np.concatenate([s["points"].reshape(-1, 2) for s in ss])
    counts = [s["ranges"].shape[1] for s in ss for _ in range(s["ranges"].shape[0])]
    sensor = np.concatenate([s["sensor"][:, :2] for s in ss])
    bounds = np.cumsum([0] + [s["ranges"].shape[0] for s in ss])
    return MP.MergeStore(ranges, points, counts, sensor, RT, MINR, MAXR), bounds


def merge(store, bounds, corr):
    for i, c in enumerate(corr):
        store.transform(int(bounds[i]), int(bounds[i + 1] - bounds[i]), c[:9].reshape(3, 3), c[9:])


def golden(name, m):
    return name + f"/m{m}"


@pytest.mark.parametrize("name", NAMES)
def test_port_equals_golden(name):
    store, bounds = port_store(name)
    res = float(Z[f"{name}/res"][0])
    for m, corr in enumerate(Z[f"{name}/corr"]):
        merge(store, bounds, corr)
        H.assert_occupancy_equals_golden(store.build(res), Z, golden(name, m))
        assert np.array_equal(store.boxes, Z[f"{golden(name, m)}/boxes"])


def test_rot30_point_box_gives_other_dims():
    """the shipped rule (box from the corrected points and sensors) differs from the corrected-corner boxes"""
    store, bounds = port_store("rot30")
    merge(store, bounds, Z["rot30/corr"][0])
    store.transformed = False   # the port's own box: the point-box rule
    g = store.build(float(Z["rot30/res"][0]))
    ref = Z["rot30/m0/dims"]
    assert [g["width"], g["height"]] != list(ref[:2])
    assert not np.array_equal(g["offset"], Z["rot30/m0/offset"])


def _fused_x(b, o, x, y, which):
    return G.apply_x_fused(b, o, x, y, which)


def test_fma_point_fused_lands_in_another_cell():
    """every crafted beam end: the unfused correction and both fused forms (exact rationals, rounded once) fall in
    different cells; the reference's cell is the unfused one"""
    c = Z["fma_point/corr"][0][0]
    b, o = c[:9].reshape(3, 3).tolist(), c[9:].tolist()
    off = float(Z["fma_point/m0/offset"][0])
    ranges, pts = Z["fma_point/sub0/ranges"], Z["fma_point/sub0/points"]
    n = 0
    for s in range(2, len(ranges)):
        k = int(np.flatnonzero(np.isfinite(ranges[s]))[0])
        x, y = float(pts[s, k, 0]), float(pts[s, k, 1])
        u = G.apply_x(b, o, x, y)
        cu = synth.grid_cell(u, off, 1.0)
        v = (Fraction(u) - Fraction(off))
        assert abs(v - (math.floor(v) + Fraction(1, 2))) < Fraction(1, 1 << 40)   # within a few ulps of a half cell
        assert all(synth.grid_cell(_fused_x(b, o, x, y, w), off, 1.0) != cu for w in (0, 1)), s
        n += 1
    assert n >= 6


def test_fma_corner_fused_width_differs():
    """the far anchor's corrected x sets the width: fused, Round(width) is another integer"""
    c = Z["fma_corner/corr"][0][0]
    b, o = c[:9].reshape(3, 3).tolist(), c[9:].tolist()
    sen = Z["fma_corner/sub0/sensor"][1]
    off = float(Z["fma_corner/m0/offset"][0])
    w = int(Z["fma_corner/m0/dims"][0])
    assert synth.grid_cell(G.apply_x(b, o, float(sen[0]), float(sen[1])), off, 1.0) == w
    assert all(synth.grid_cell(_fused_x(b, o, float(sen[0]), float(sen[1]), k), off, 1.0) != w for k in (0, 1))


def test_round_half_width():
    """the corrected box is exactly k + 0.5 cells wide with k even: Round gives k + 1, rint and truncation give k"""
    box = Z["round_half/m0/boxes"]
    size = (box[:, 2].max() - box[:, 0].min()) * 1.0
    assert size == math.floor(size) + 0.5 and int(math.floor(size)) % 2 == 0
    w = int(Z["round_half/m0/dims"][0])
    assert w == int(math.floor(size)) + 1
    assert int(np.rint(size)) != w and int(size) != w


def test_compound_needs_the_second_application():
    """merge 1 corrects merge 0's scans again: correcting the original scans once gives another grid"""
    store, bounds = port_store("compound")
    merge(store, bounds, Z["compound/corr"][1])
    g = store.build(float(Z["compound/res"][0]))
    assert [g["width"], g["height"]] != list(Z["compound/m1/dims"][:2]) or not np.array_equal(g["offset"], Z["compound/m1/offset"])
    store2, _ = port_store("compound")
    merge(store2, bounds, Z["compound/corr"][0])
    merge(store2, bounds, Z["compound/corr"][1])
    H.assert_occupancy_equals_golden(store2.build(float(Z["compound/res"][0])), Z, "compound/m1")


def test_empty_submap_boxes_are_sensor_positions():
    """a submap without in-range readings: each box is its corrected sensor position alone"""
    n0 = Z["empty/sub0/ranges"].shape[0]
    boxes = Z["empty/m0/boxes"][n0:]
    assert np.array_equal(boxes[:, :2], boxes[:, 2:])
    store, bounds = port_store("empty")
    merge(store, bounds, Z["empty/corr"][0])
    assert np.array_equal(store.sensor[n0:], boxes[:, :2])


def test_three_submaps_identity_keeps_update_boxes():
    """the identity-corrected submap keeps LocalizedRangeScan::Update's boxes; the translated one moves them exactly"""
    store, bounds = port_store("three")
    before = store.boxes.copy()
    merge(store, bounds, Z["three/corr"][0])
    a, b = int(bounds[1]), int(bounds[2])
    assert np.array_equal(store.boxes[:a], before[:a])
    assert np.array_equal(store.boxes[a:b], before[a:b] + np.array([3.1, -1.7, 3.1, -1.7]))


def corner_order_box(order):
    """the box of four corners of {-1, 0, 1, 0} under a 90 degree basis with -0 entries, corners added in `order`"""
    b, o = [[0.0, -1.0, -0.0], [1.0, 0.0, 0.0]], [-0.0, 0.0]
    corners = {"min": (-1.0, 0.0), "max": (1.0, 0.0), "maxmin": (1.0, 0.0), "minmax": (-1.0, 0.0)}
    big = 999999999999999999.99999
    mnx, mny, mxx, mxy = big, big, -big, -big
    for k in order:
        x, y = corners[k]
        cx = ((b[0][0] * x + b[0][1] * y) + b[0][2] * 0.0) + o[0]
        cy = ((b[1][0] * x + b[1][1] * y) + b[1][2] * 0.0) + o[1]
        mnx, mny = (cx if cx < mnx else mnx), (cy if cy < mny else mny)
        mxx, mxy = (cx if cx > mxx else mxx), (cy if cy > mxy else mxy)
    return np.array([mnx, mny, mxx, mxy])


def test_corner_order_decides_signed_zero():
    """the corners' order is visible in the sign of a zero bound: the tool's order keeps -0, max-first would keep +0; the
    host restatement follows the tool"""
    tool = corner_order_box(["min", "max", "maxmin", "minmax"])
    other = corner_order_box(["max", "min", "maxmin", "minmax"])
    assert np.signbit(tool[0]) and np.signbit(tool[2])
    assert not np.signbit(other[0])
    box = MP.corner_boxes([[-1.0, 0.0, 1.0, 0.0]], [[0.0, -1.0, -0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]], [-0.0, 0.0, 0.0])
    assert box[0].tobytes() == tool.tobytes()
