"""The crafted occupancy-grid fixtures (tests/golden/make_occupancy_edge_golden.py): the generators reproduce the stored
inputs, the crafted beams are what they claim to be (checked on the reference's own stored points with exact arithmetic),
each case can detect the defect it was built for, and the C port (kp_occupancy_create) equals the reference on every case."""
import functools
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import helpers as H
from golden import make_occupancy_edge_golden as E
from oracle import karto_port as P
from slam_toolbox_b200 import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "occupancy_edge_golden.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]
CRAFTED = [n for n in NAMES if not n.startswith("far_")]
HALF = [n for n in NAMES if n.startswith("half_")]
FMA = [n for n in NAMES if n.startswith("fma_clip_")]


@functools.lru_cache(maxsize=1)
def crafted_inputs():
    return E.crafted_cases()


def half_away(v):
    """math::Round (Math.h:87-90)"""
    return math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5)


def c_round(v):
    """C round(): the exact value rounded half away from zero (no v + 0.5 rounding step)"""
    a = abs(v)
    k = math.floor(a)
    k += 1 if a - k >= 0.5 else 0
    return math.copysign(k, v)


def bresenham(x0, y0, x1, y1, width, height):
    """Grid::TraceLine (Karto.h:4874-4927): the in-grid cells of a line, in order"""
    steep = abs(y1 - y0) > abs(x1 - x0)
    if steep:
        x0, y0, x1, y1 = y0, x0, y1, x1
    if x0 > x1:
        x0, x1, y0, y1 = x1, x0, y1, y0
    dx, dy, err, y = x1 - x0, abs(y1 - y0), 0, y0
    ystep = 1 if y0 < y1 else -1
    out = []
    for x in range(x0, x1 + 1):
        px, py = (y, x) if steep else (x, y)
        err += dy
        if 2 * err >= dx:
            y += ystep
            err -= dx
        if 0 <= px < width and 0 <= py < height:
            out.append((px, py))
    return out


def beams(name):
    """(scan, beam, range, sensor xy, point xy) of every finite reading of a crafted case, on the stored reference data"""
    r, pts, sensor = Z[f"{name}/ranges"], Z[f"{name}/points"], Z[f"{name}/sensor"]
    for s, k in zip(*np.nonzero(np.isfinite(r))):
        yield int(s), int(k), float(r[s, k]), sensor[s, :2], pts[s, k]


def grid_geometry(name):
    res = float(Z[f"{name}/params"][0])
    w, h, _ = (int(v) for v in Z[f"{name}/dims"])
    return Z[f"{name}/offset"], 1.0 / res, w, h


def port_case(name):
    res, rt, mp, th = H.occupancy_params(Z[f"{name}/params"])
    if name.startswith("far_"):
        ranges, poses = E.far_inputs(name)
        pts = np.stack([P.point_readings(r, p, synth.ANGLE_MIN, synth.ANGLE_INC) for r, p in zip(ranges, poses)])
        assert H.digest(pts) == Z[f"{name}/points_digest"][0], "this host's libm differs from the reference's: far_* points"
    else:
        ranges, poses, pts = Z[f"{name}/ranges"], Z[f"{name}/poses"], Z[f"{name}/points"]
    ranges, pts = np.ascontiguousarray(ranges, dtype=np.float64), np.ascontiguousarray(pts, dtype=np.float64)
    rec = H.scan_records(ranges.reshape(-1), pts.reshape(-1, 2), [ranges.shape[1]] * len(ranges), poses)
    return H.port_occupancy(rec, res, rt, mp, th)


def test_fixture_is_small_and_complete():
    assert os.path.getsize(GOLDEN) < 1_000_000
    fams = {n.split("_")[0] for n in NAMES}
    assert fams == {"half", "fma", "merge", "dims", "far", "update"}
    assert len(FMA) >= 3 and all(np.isfinite(Z[f"{n}/ranges"]).sum(axis=1).max() <= 1 for n in FMA)


@pytest.mark.parametrize("name", NAMES)
def test_generators_are_deterministic(name):
    if name.startswith("far_"):
        ranges, poses = E.far_inputs(name)
        assert H.digest(np.concatenate([ranges.ravel(), poses.ravel()])) == Z[f"{name}/inputs"][0]
        return
    c = crafted_inputs()[name]
    for k in ("ranges", "poses", "params"):
        assert np.array_equal(c[k], Z[f"{name}/{k}"], equal_nan=True), k


@pytest.mark.parametrize("name", CRAFTED)
def test_sensor_is_the_pose_position(name):
    """the reference's sensor pose is the scan pose (the laser has no offset): the GPU store takes poses as sensor poses"""
    assert np.array_equal(Z[f"{name}/sensor"][:, :2], Z[f"{name}/poses"][:, :2])


def test_exact_axis_beams_are_exact():
    """Every reading whose angle (heading + angle_min) + k * inc is exactly 0, pi or +-pi/2 has a point exactly sensor +- r on
    that axis in the reference's own output (no libm involved: cos(0) = 1, sin(0) = 0, cos(pi) = -1, sin(pi/2) = 1)."""
    n = 0
    for name in CRAFTED:
        if name.startswith("merge_"):
            continue
        poses = Z[f"{name}/poses"]
        for s, k, r, sxy, p in beams(name):
            ang = (poses[s, 2] + synth.ANGLE_MIN) + k * synth.ANGLE_INC
            if ang == 0.0:
                assert p[0] == sxy[0] + r and p[1] == sxy[1], (name, s, k)
            elif ang == math.pi:
                assert p[0] == sxy[0] - r, (name, s, k)
            elif ang == math.pi / 2:
                assert p[1] == sxy[1] + r, (name, s, k)
            elif ang == -math.pi / 2:
                assert p[1] == sxy[1] - r, (name, s, k)
            else:
                continue
            n += 1
    assert n > 300


def half_coordinates(name):
    """(v, label) of every crafted coordinate of a half_* case: sensor cells, in-range end points and clipped ends of
    over-range beams, v = (w - offset) * scale as the kernel computes it"""
    off, scale, _, _ = grid_geometry(name)
    rt = float(Z[f"{name}/params"][1])
    out = []
    for s, k, r, sxy, p in beams(name):
        for a in range(2):
            out.append(((sxy[a] - off[a]) * scale, "sensor"))
        if not (0.1 < r < 30.0):
            continue
        e = p if r < rt else [synth.clipped_end(sxy[a], p[a], r, rt) for a in range(2)]
        for a in range(2):
            out.append(((e[a] - off[a]) * scale, "end" if r < rt else "clipped"))
    return out


@pytest.mark.parametrize("name", HALF)
def test_half_cells_are_half_cells(name):
    """the crafted coordinates sit on or within a few ulps of half cells, and some of them round to another cell under
    round-half-even (rint) or C round() than under the reference's floor(v + 0.5) / ceil(v - 0.5)"""
    near, rint_diff, round_diff, kinds = 0, 0, 0, set()
    for v, kind in half_coordinates(name):
        frac = v - math.floor(v)
        if abs(frac - 0.5) > 8 * math.ulp(max(abs(v), 1.0)):
            continue
        near += 1
        kinds.add(kind)
        rint_diff += half_away(v) != round(v)          # Python round() is round-half-even
        round_diff += half_away(v) != c_round(v)
    assert near >= 2 and rint_diff >= 1, (near, rint_diff)
    if name in ("half_sensor_r1", "half_low_tiny"):
        assert round_diff >= 1                          # v = +-0.49999999999999994
    if name.startswith(("half_clip", "half_low")):
        assert "clipped" in kinds
    if name == "half_low_r1" or name == "half_low_tiny":
        assert any(v < 0 and kind == "clipped" for v, kind in half_coordinates(name))


@pytest.mark.parametrize("name", FMA)
def test_fma_beams_change_the_grid_when_fused(name):
    """every over-range beam's clipped end lands in another cell when s + ratio * dx is fused (exact rational arithmetic,
    rounded once), and that moves at least one in-grid pass counter (Bresenham on both ends)"""
    off, scale, w, h = grid_geometry(name)
    rt = float(Z[f"{name}/params"][1])
    n = 0
    for s, k, r, sxy, p in beams(name):
        assert rt < r < 30.0
        ratio, dx = rt / r, p[0] - sxy[0]
        e = sxy[0] + ratio * dx
        f = float(Fraction(sxy[0]) + Fraction(ratio) * Fraction(dx))
        assert e == synth.clipped_end(sxy[0], p[0], r, rt) and f == synth.clipped_end_fused(sxy[0], p[0], r, rt)
        ce, cf = half_away((e - off[0]) * scale), half_away((f - off[0]) * scale)
        assert ce != cf and 0 <= min(ce, cf) and max(ce, cf) < w
        fx, fy = half_away((sxy[0] - off[0]) * scale), half_away((sxy[1] - off[1]) * scale)
        ty = half_away((sxy[1] + ratio * (p[1] - sxy[1]) - off[1]) * scale)
        assert sorted(bresenham(fx, fy, ce, ty, w, h)) != sorted(bresenham(fx, fy, cf, ty, w, h))
        n += 1
    assert n >= 20


def test_update_fixtures_hold_the_boundaries():
    """cells with hits / pass exactly at 0.1 (and pass > 2), cells with pass == min_pass_through (2 and 50); the cell states
    follow UpdateCell (Karto.h:6242-6253) from the port's counters, which equal the reference's (test_port_equals_reference)"""
    for name in ("update_default", "update_mp0_th0", "update_th1", "update_mp50"):
        g = port_case(name)
        H.assert_occupancy_equals_golden(g, Z, name)
        _, _, mp, th = H.occupancy_params(Z[f"{name}/params"])
        ps, ht = g["passes"].astype(np.int64), g["hits"].astype(np.int64)
        known = ps > mp
        ratio = np.divide(ht, ps, out=np.zeros(ps.shape), where=ps > 0)
        exp = np.where(known, np.where(ratio > th, 100, 255), 0).astype(np.uint8)
        assert np.array_equal(exp, Z[f"{name}/cells"])
        assert ((ps > 2) & (ht * 10 == ps) & (ht > 0)).any()          # hits / pass == 0.1 exactly
        assert ((ps == 2) & (ht > 0)).any() and (ps == 50).any()      # pass == 2 and pass == 50
        if th == 0.0:
            assert (known & (ht == 0)).any() and (known & (ht > 0)).any()


DIMS = {"dims_half_box": (11, 7, 16), "dims_w16": (16, 8, 16), "dims_w17": (17, 8, 24), "dims_sensor_max": (10, 5, 16),
        "dims_zero": (0, 0, 0), "dims_n_by_0": (7, 0, 8), "dims_0_by_n": (0, 9, 0), "dims_all_inf": (3, 2, 8),
        "dims_range_edges": (242, 42, 248)}


@pytest.mark.parametrize("name", sorted(DIMS))
def test_dims_cases_have_the_intended_shape(name):
    assert tuple(Z[f"{name}/dims"]) == DIMS[name]
    off, scale, w, h = grid_geometry(name)
    if name == "dims_sensor_max":
        fx = [half_away((sxy[0] - off[0]) * scale) for _, _, _, sxy, _ in beams(name)]
        assert fx and all(x == w for x in fx)                                 # every trace starts at fx == width
    if name == "dims_half_box":
        assert (10.5 * scale, 6.5 * scale) == (10.5, 6.5)
    if name == "dims_range_edges":
        pts = [(r, p) for _, _, r, _, p in beams(name)]
        at_rt = [p for r, p in pts if r == 12.0]
        at_min = [p for r, p in pts if r == 0.1]
        assert len(at_rt) == 1 and len(at_min) == 2
        assert off[0] == min(p[0] for p in at_min) and off[0] + w / scale == pytest.approx(at_rt[0][0], abs=1e-9)
    if w == 0 or h == 0:
        assert Z[f"{name}/sums"].tolist() == [0, 0]
        assert any(12.0 < r < 30.0 for _, _, r, _, _ in beams(name))        # over-range beams were traced


@pytest.mark.parametrize("name", NAMES)
def test_port_equals_reference(name):
    """kp_occupancy_create fed the reference's points: dims, offset, cells and both counters"""
    H.assert_occupancy_equals_golden(port_case(name), Z, name)
