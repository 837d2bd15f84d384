"""Occupancy grids over scans of several lasers: the cases, a host oracle and the binding of the reference's own run.

The reference takes every scan's range threshold, minimum and maximum range from that scan's own laser
(OccupancyGrid::AddScan, Karto.h:6146-6151; LocalizedRangeScan::Update's box, :5646-5698).

host_occupancy is the host oracle for large random stores.  Integer counters commute, so a grid of several lasers is the
sum of one single-laser grid per laser, each traced by the C port (oracle/karto_port.c) with that laser's limits over the
same box.  Two zero-beam anchor scans at the corners of the union of every scan's own box make each single-laser grid take
that box (an anchor adds its sensor position and traces nothing).  The cell states are then Update's rule on the summed
counters.  test_multilaser_fixtures.py pins this oracle to the reference's fixtures.

The reference binding (oracle/_ref/libmultilaser_ref.so, oracle/multilaser.mk) registers named lasers with the reference's
SensorManager and runs the unmodified OccupancyGrid::CreateFromScans on scans made on them."""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

from slam_toolbox_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libmultilaser_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "multilaser_golden.npz")
KT_TOLERANCE = 1e-6
BIG = 999999999999999999.99999

_DP = C.POINTER(C.c_double)
_lib = None


# ---- cases ------------------------------------------------------------------------------------------------------------
# a laser = (range_threshold, minimum_range, maximum_range); every laser has the standard angular geometry
STD = (12.0, 0.1, 30.0)


def _run(seed, n, size=24.0):
    run = synth.make_mapping_run(seed, n, world=synth.make_world(seed, size=size))
    return run["ranges"], run["poses"]


def _axis_scans(sensor, readings):
    """scans along +x from `sensor`: one beam per reading on the exact +x beam, every other reading inf"""
    out = []
    for r in readings:
        rr, pose = synth.axis_scan(sensor, "+x", [float(r)])
        out.append((rr, pose))
    return out


def _stack(scans):
    return np.stack([s[0] for s in scans]), np.stack([s[1] for s in scans])


def cases():
    """name -> dict(ranges (S, N), poses (S, 3), lasers (S, 3), laser_id (S,), res, [submap (S,), corr (k, 12)])"""
    out = {}

    def put(name, ranges, poses, lasers, ids, res=0.05, **extra):
        out[name] = dict(ranges=np.ascontiguousarray(ranges, dtype=np.float64), poses=np.ascontiguousarray(poses, dtype=np.float64),
                         lasers=np.array([lasers[i] for i in ids], dtype=np.float64), laser_id=np.asarray(ids, dtype=np.int32),
                         res=float(res), laser_table=np.array(lasers, dtype=np.float64), **extra)

    # the lasers differ in one limit each; scans alternate between them
    r, p = _run(41, 16)
    put("thr_only", r, p, [STD, (6.0, 0.1, 30.0)], [i % 2 for i in range(16)])
    r, p = _run(42, 16)
    put("minr_only", r, p, [STD, (12.0, 1.5, 30.0)], [i % 2 for i in range(16)])
    r, p = _run(43, 16)
    put("maxr_only", r, p, [STD, (12.0, 0.1, 14.0)], [i % 2 for i in range(16)])
    # readings at each laser's threshold - KT_TOLERANCE and one ulp either side: the end cell is hit below it only
    la, lb = (12.0, 0.1, 30.0), (5.0, 0.1, 30.0)
    sc, ids = [], []
    for k, (lid, l) in enumerate(((0, la), (1, lb))):
        t = l[0] - KT_TOLERANCE
        for j, v in enumerate((float(np.nextafter(t, 0.0)), t, float(np.nextafter(t, np.inf)))):
            sc += _axis_scans((0.3 + 0.7 * j, 0.2 + 1.3 * k + 0.4 * j), [v])
            ids.append(lid)
    # anchors that keep every end cell inside the grid
    sc += [(np.full(synth.N_BEAMS, np.inf), np.array([-1.0, -1.0, 0.0])), (np.full(synth.N_BEAMS, np.inf), np.array([15.0, 5.0, 0.0]))]
    ids += [0, 1]
    r, p = _stack(sc)
    put("tolerance", r, p, [la, lb], ids, res=0.05)
    # the longer-threshold laser's far readings set the grid box; the other laser would clip them out of the box
    r, p = _run(44, 12, size=40.0)
    put("box_long", r, p, [(20.0, 0.1, 30.0), (4.0, 0.1, 30.0)], [0, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1])
    # A / B / A in blocks, so that a store keyed on the first laser or the last laser differs
    r, p = _run(49, 18)   # (headings within [-pi, pi]: the reference's points of a wrapped heading differ in the last bits)
    put("interleaved", r, p, [STD, (8.0, 0.5, 10.0)], [0] * 6 + [1] * 6 + [0] * 6)
    # laser B has no in-range reading: every reading is below its minimum range or beyond its 0.12 m threshold, so its
    # scans add only their sensor positions to the box, and their beams are traced up to 0.12 m without a hit
    r, p = _run(46, 12)
    put("no_inrange", r, p, [STD, (0.12, 0.11, 30.0)], [int(i % 3 == 1) for i in range(12)])
    # two submaps on different lasers, the second one merged under a rotated correction
    r1, p1 = _run(51, 10)
    r2, p2 = _run(48, 10)
    b, o = _rot(23.0, (1.5, -0.7, 0.0))
    corr = np.stack([np.concatenate([np.eye(3).ravel(), np.zeros(3)]), np.concatenate([b.ravel(), o])])
    put("merge_rot", np.concatenate([r1, r2]), np.concatenate([p1, p2]), [STD, (7.0, 0.3, 9.0)], [0] * 10 + [1] * 10,
        submap=np.array([0] * 10 + [1] * 10, dtype=np.int32), corr=corr)
    return out


def _rot(deg, origin):
    t = math.radians(deg)
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]), np.array(origin, dtype=np.float64)


def random_store(seed, n_scans, n_lasers=3, res=0.05, n_beams=None):
    """a mapping run whose scans draw their laser at random from n_lasers random lasers"""
    rng = np.random.default_rng(seed)
    r, p = _run(seed, n_scans, size=30.0)
    if n_beams is not None:
        r = r[:, :n_beams]
    lasers = [STD]
    for _ in range(n_lasers - 1):
        rt = float(rng.uniform(3.0, 15.0))
        lasers.append((rt, float(rng.uniform(0.05, 2.0)), float(rng.uniform(rt, 30.0))))
    ids = rng.integers(0, n_lasers, n_scans)
    return dict(ranges=r, poses=p, lasers=np.array([lasers[i] for i in ids]), laser_id=ids.astype(np.int32), res=res,
                laser_table=np.array(lasers))


# ---- host oracle ------------------------------------------------------------------------------------------------------
def scan_box(ranges, points, pose, laser):
    """LocalizedRangeScan::Update's box: the sensor position and the points whose range is in [minimum range, threshold]"""
    rt, minr = float(laser[0]), float(laser[1])
    box = [float(pose[0]), float(pose[1]), float(pose[0]), float(pose[1])]
    for k in range(len(ranges)):
        v = float(ranges[k])
        if v >= minr and v <= rt:
            x, y = float(points[k][0]), float(points[k][1])
            if x < box[0]:
                box[0] = x
            if y < box[1]:
                box[1] = y
            if x > box[2]:
                box[2] = x
            if y > box[3]:
                box[3] = y
    return box


def union(boxes):
    u = [BIG, BIG, -BIG, -BIG]
    for b in boxes:
        if b[0] < u[0]:
            u[0] = b[0]
        if b[1] < u[1]:
            u[1] = b[1]
        if b[2] > u[2]:
            u[2] = b[2]
        if b[3] > u[3]:
            u[3] = b[3]
    return u


def host_occupancy(ranges, points, poses, lasers, res, min_pass_through=2, occupancy_threshold=0.1):
    """CreateFromScans over scans whose limits are lasers[s] = (range threshold, minimum range, maximum range).  ranges
    (S, N), points (S, N, 2), poses (S, 3).  Same dict as oracle.karto_port.occupancy."""
    from oracle import karto_port as P
    ranges = np.ascontiguousarray(ranges, dtype=np.float64)
    points = np.ascontiguousarray(points, dtype=np.float64)
    poses = np.ascontiguousarray(poses, dtype=np.float64)
    lasers = np.asarray(lasers, dtype=np.float64)
    S = len(ranges)
    if S == 0:
        return None
    boxes = [scan_box(ranges[s], points[s], poses[s], lasers[s]) for s in range(S)]
    u = union(boxes)
    anchors = [P.KpScan(0, None, None, (C.c_double * 3)(u[0], u[1], 0.0)), P.KpScan(0, None, None, (C.c_double * 3)(u[2], u[3], 0.0))]
    total = None
    for lim in sorted({tuple(v) for v in lasers.tolist()}):
        members = [s for s in range(S) if tuple(lasers[s].tolist()) == lim]
        arr = (P.KpScan * (len(members) + 2))()
        for i, s in enumerate(members):
            arr[i] = P.KpScan(ranges.shape[1], ranges[s].ctypes.data_as(_DP), points[s].ctypes.data_as(_DP), (C.c_double * 3)(*poses[s]))
        arr[len(members)], arr[len(members) + 1] = anchors
        g = P.occupancy_array(arr, len(members) + 2, res, lim[0], lim[1], lim[2], min_pass_through, occupancy_threshold)
        if total is None:
            total = g
        else:
            assert (g["width"], g["height"], g["stride"]) == (total["width"], total["height"], total["stride"])
            assert np.array_equal(g["offset"], total["offset"])
            total["passes"] += g["passes"]
            total["hits"] += g["hits"]
    ps, ht = total["passes"], total["hits"]
    cells = np.zeros(ps.shape, dtype=np.uint8)
    seen = ps > min_pass_through
    ratio = np.zeros(ps.shape)
    ratio[seen] = ht[seen].astype(np.float64) / ps[seen].astype(np.float64)
    cells[seen & (ratio > occupancy_threshold)] = 100
    cells[seen & ~(ratio > occupancy_threshold)] = 255
    total["cells"] = cells
    return total


# ---- the reference ----------------------------------------------------------------------------------------------------
def ref_available() -> bool:
    return os.path.exists(REF_PATH)


def ref_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(REF_PATH)
        L.kml_laser.restype = C.c_int
        L.kml_laser.argtypes = [C.c_char_p] + [C.c_double] * 6
        L.kml_laser_limits.argtypes = [C.c_char_p, _DP]
        L.kml_scan_create.restype = C.c_void_p
        L.kml_scan_create.argtypes = [C.c_char_p, _DP, C.c_int, _DP, C.c_int]
        L.kref_scan_destroy.argtypes = [C.c_void_p]
        L.kref_scan_points.restype = C.c_int
        L.kref_scan_points.argtypes = [C.c_void_p, _DP, C.c_int]
        L.kref_transform_scan.argtypes = [C.c_void_p, _DP, _DP]
        L.kref_scan_box.argtypes = [C.c_void_p, _DP]
        L.kref_occupancy_create.restype = C.c_void_p
        L.kref_occupancy_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_double, C.c_int, C.c_double]
        L.kref_occupancy_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), _DP]
        L.kref_occupancy_copy.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.kref_occupancy_destroy.argtypes = [C.c_void_p]
        L.kmm_store_create.restype = C.c_void_p
        L.kmm_store_create.argtypes = [C.c_double]
        L.kmm_store_destroy.argtypes = [C.c_void_p]
        L.kmm_add_submap.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
        L.kmm_apply.argtypes = [C.c_void_p, C.c_int, _DP, _DP]
        L.kmm_merge.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_int), _DP, C.POINTER(C.c_uint8), C.c_long]
        _lib = L
    return _lib


def ref_laser(name: str, laser) -> int:
    """registers laser `name` with limits (range threshold, minimum range, maximum range), or sets them"""
    rt, minr, maxr = (float(v) for v in laser)
    n = ref_lib().kml_laser(name.encode(), synth.ANGLE_MIN, synth.ANGLE_MAX, synth.ANGLE_INC, minr, maxr, rt)
    held = np.zeros(3)
    ref_lib().kml_laser_limits(name.encode(), held.ctypes.data_as(_DP))
    assert held.tolist() == [rt, minr, maxr], (name, held, laser)   # the reference did not clip the threshold
    return n


class RefScan:
    def __init__(self, laser_name: str, ranges, pose, uid=0):
        r = np.ascontiguousarray(ranges, dtype=np.float64)
        p = np.ascontiguousarray(pose, dtype=np.float64)
        self.n = len(r)
        self.h = ref_lib().kml_scan_create(laser_name.encode(), r.ctypes.data_as(_DP), len(r), p.ctypes.data_as(_DP), uid)

    def points(self):
        out = np.empty((self.n, 2))
        n = ref_lib().kref_scan_points(self.h, out.ctypes.data_as(_DP), self.n)
        return out[:n]

    def transform(self, basis, origin):
        b = np.ascontiguousarray(basis, dtype=np.float64).reshape(9)
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        ref_lib().kref_transform_scan(self.h, b.ctypes.data_as(_DP), o.ctypes.data_as(_DP))

    def box(self):
        out = np.zeros(4)
        ref_lib().kref_scan_box(self.h, out.ctypes.data_as(_DP))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            ref_lib().kref_scan_destroy(self.h)
            self.h = None


def ref_occupancy(scans, res):
    """the reference's static OccupancyGrid::CreateFromScans over RefScans"""
    arr = (C.c_void_p * max(1, len(scans)))(*[s.h for s in scans])
    h = ref_lib().kref_occupancy_create(arr, len(scans), float(res), -1, -1.0)
    if not h:
        return None
    info = (C.c_int * 3)()
    off = np.zeros(2)
    ref_lib().kref_occupancy_info(h, info, off.ctypes.data_as(_DP))
    w, hh, st = info[0], info[1], info[2]
    cells = np.zeros((hh, st), dtype=np.uint8)
    ps = np.zeros((hh, st), dtype=np.uint32)
    ht = np.zeros((hh, st), dtype=np.uint32)
    ref_lib().kref_occupancy_copy(h, cells.ctypes.data_as(C.POINTER(C.c_uint8)), ps.ctypes.data_as(C.POINTER(C.c_uint32)),
                                  ht.ctypes.data_as(C.POINTER(C.c_uint32)))
    ref_lib().kref_occupancy_destroy(h)
    return dict(width=w, height=hh, stride=st, offset=off, cells=cells, passes=ps, hits=ht)


def ref_scans(case, prefix):
    """RefScans of a case, scan s on laser f"{prefix}{laser_id[s]}" (registered with the case's limits)"""
    for i, lim in enumerate(case["laser_table"]):
        ref_laser(f"{prefix}{i}", lim)
    return [RefScan(f"{prefix}{int(case['laser_id'][s])}", case["ranges"][s], case["poses"][s], s) for s in range(len(case["ranges"]))]


def binding_merge(scans, submap, corr, res):
    """the map-merge binding (karto::b200::SubmapStore, integration/merge_maps_b200.hpp) on RefScans: one submap per value of
    submap, each corrected by corr[k] (basis 9 + origin 3), merged.  Returns (width, height, stride), offset, cells."""
    L = ref_lib()
    h = L.kmm_store_create(float(res))
    try:
        for k in range(len(corr)):
            mine = [s.h for s, m in zip(scans, submap) if m == k]
            arr = (C.c_void_p * max(1, len(mine)))(*mine)
            assert L.kmm_add_submap(h, arr, len(mine), None, None, None, 0) == k
        for k in range(len(corr)):
            b = np.ascontiguousarray(corr[k][:9])
            o = np.ascontiguousarray(corr[k][9:])
            assert L.kmm_apply(h, k, b.ctypes.data_as(_DP), o.ctypes.data_as(_DP)) == 0
        info, off = (C.c_int * 3)(), np.zeros(2)
        assert L.kmm_merge(h, float(res), info, off.ctypes.data_as(_DP), None, 0) == 0
        cells = np.zeros((info[1], info[2]), dtype=np.uint8)
        assert L.kmm_merge(h, float(res), info, off.ctypes.data_as(_DP), cells.ctypes.data_as(C.POINTER(C.c_uint8)), cells.size) == 0
        return tuple(info), off, cells
    finally:
        L.kmm_store_destroy(h)


# ---- comparisons ------------------------------------------------------------------------------------------------------
def sha(a) -> str:
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def assert_grid_equal(g, e):
    assert (g["width"], g["height"], g["stride"]) == (e["width"], e["height"], e["stride"])
    assert np.array_equal(g["offset"], e["offset"])
    assert np.array_equal(g["cells"], e["cells"])
    assert np.array_equal(g["passes"], e["passes"])
    assert np.array_equal(g["hits"], e["hits"])


def golden_grid(z, name):
    """the fixture's grid of case `name` (counters as digests and sums)"""
    return dict(dims=list(z[f"{name}/dims"]), offset=z[f"{name}/offset"], cells=z[f"{name}/cells"], sums=list(z[f"{name}/sums"]),
                pass_sha=str(z[f"{name}/pass_sha"][0]), hits_sha=str(z[f"{name}/hits_sha"][0]))


def assert_equals_golden(g, z, name):
    e = golden_grid(z, name)
    assert [g["width"], g["height"], g["stride"]] == e["dims"]
    assert np.array_equal(g["offset"], e["offset"])
    assert np.array_equal(g["cells"], e["cells"])
    assert [int(g["passes"].sum()), int(g["hits"].sum())] == e["sums"]
    assert sha(np.asarray(g["passes"], dtype=np.uint32)) == e["pass_sha"]
    assert sha(np.asarray(g["hits"], dtype=np.uint32)) == e["hits_sha"]
