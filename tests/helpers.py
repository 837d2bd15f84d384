"""Shared fixtures for the parity tests: the parameter sets of BASELINE.json's configs and
constructors for the three implementations (reference .so, C port oracle, CUDA product)."""
from __future__ import annotations

import math
import os

import numpy as np

from slam_toolbox_b200 import synth

LASER = dict(min_angle=synth.ANGLE_MIN, max_angle=synth.ANGLE_MAX, ang_res=synth.ANGLE_INC, min_range=0.1, max_range=30.0,
             range_threshold=12.0)

# toolbox-style parameter values (before the setters square the variance penalties)
MAPPER_SEQ = dict(coarse_search_angle_offset=math.radians(5.0), coarse_angle_resolution=math.radians(2.0),
                  fine_search_angle_offset=math.radians(0.2), distance_variance_penalty=0.5, angle_variance_penalty=1.0,
                  minimum_distance_penalty=0.5, minimum_angle_penalty=0.9, use_response_expansion=1)
MAPPER_LOOP = dict(MAPPER_SEQ, coarse_search_angle_offset=math.radians(20.0))

# ScanMatcher::Create arguments: (searchSize, resolution, smearDeviation, rangeThreshold)
GRID_SEQ = (1.0, 0.01, 0.03, 12.0)       # cfg1, Karto smear
GRID_SEQ_YAML = (1.0, 0.01, 0.1, 12.0)   # cfg1, shipped YAML smear (order-dependent raster)
GRID_LOOP = (4.0, 0.05, 0.03, 12.0)      # cfg2 / cfg5
GRID_SMALL = (0.5, 0.05, 0.03, 6.0)      # small fast case for unit tests


def ref_matcher(mapper_kw, grid):
    from oracle import karto_ref as R
    R.init_laser(**LASER)
    return R.RefMatcher(R.RefMapper(**mapper_kw), *grid)


def port_matcher(mapper_kw, grid):
    from oracle import karto_port as P
    return P.PortMatcher(search_size=grid[0], resolution=grid[1], smear_deviation=grid[2], range_threshold=grid[3],
                         coarse_search_angle_offset=mapper_kw["coarse_search_angle_offset"],
                         coarse_angle_resolution=mapper_kw["coarse_angle_resolution"],
                         fine_search_angle_offset=mapper_kw["fine_search_angle_offset"],
                         distance_variance_penalty=mapper_kw["distance_variance_penalty"] ** 2,
                         angle_variance_penalty=mapper_kw["angle_variance_penalty"] ** 2,
                         minimum_distance_penalty=mapper_kw["minimum_distance_penalty"],
                         minimum_angle_penalty=mapper_kw["minimum_angle_penalty"],
                         use_response_expansion=int(mapper_kw["use_response_expansion"]))


def gpu_matcher(mapper_kw, grid):
    from slam_toolbox_b200 import api
    mp = api.MapperParams(**{k: (bool(v) if k == "use_response_expansion" else v) for k, v in mapper_kw.items()})
    return api.ScanMatcher.Create(mp, *grid)


def port_scans(ranges, poses):
    from oracle import karto_port as P
    return [P.PortScan(r, p, synth.ANGLE_MIN, synth.ANGLE_INC) for r, p in zip(np.atleast_2d(ranges), np.atleast_2d(poses))]


def ref_scans(ranges, poses, uid0=0):
    from oracle import karto_ref as R
    R.init_laser(**LASER)
    return [R.RefScan(r, p, uid0 + i) for i, (r, p) in enumerate(zip(np.atleast_2d(ranges), np.atleast_2d(poses)))]


def coarse_search(grid):
    """(searchSpaceOffset, searchSpaceResolution) of MatchScan's coarse pass (Mapper.cpp:577-585)."""
    side = math.floor(grid[0] / grid[1] + 0.5) + 1
    res = 1.0 / (1.0 / grid[1])
    off = 0.5 * (side - 1) * res
    return (off, off), (2 * res, 2 * res)


def gpu_block(ranges, poses, range_threshold=None):
    from slam_toolbox_b200 import api
    laser = api.LaserRangeFinder(minimum_angle=LASER["min_angle"], maximum_angle=LASER["max_angle"], angular_resolution=LASER["ang_res"],
                                 minimum_range=LASER["min_range"], maximum_range=LASER["max_range"],
                                 range_threshold=LASER["range_threshold"] if range_threshold is None else range_threshold)
    return api.ScanBlock(ranges, poses, laser)


def digest(a) -> str:
    """sha256 of shape + bytes, with NaN payloads and signed zeros folded so that equal digests mean
    np.array_equal(..., equal_nan=True)"""
    import hashlib
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = np.ascontiguousarray(np.where(np.isnan(a), np.nan, a + 0.0))
    return hashlib.sha256(str(a.shape).encode() + a.tobytes()).hexdigest()


REFERENCE_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.npz")


def reference_golden():
    """what the unmodified reference computed for the cases of tests/golden/make_reference_golden.py"""
    return np.load(REFERENCE_GOLDEN)


def assert_occupancy_equals_golden(g, z, name):
    """g = dict(width, height, stride, offset, cells, passes, hits) vs tests/golden/occupancy_golden.npz case `name`"""
    import hashlib
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()   # noqa: E731
    assert [g["width"], g["height"], g["stride"]] == list(z[f"{name}/dims"])
    assert np.array_equal(g["offset"], z[f"{name}/offset"])
    assert np.array_equal(g["cells"], z[f"{name}/cells"])
    assert [int(g["passes"].sum()), int(g["hits"].sum())] == list(z[f"{name}/sums"])
    assert sha(g["passes"].astype(np.uint32)) == z[f"{name}/pass_sha"][0]
    assert sha(g["hits"].astype(np.uint32)) == z[f"{name}/hits_sha"][0]


# b200_scan (include/b200slam.h) and kp_scan (oracle/karto_port.h) share this layout: int32 n, two pointers, double[3] pose
SCAN_DTYPE = np.dtype([("n", "<i4"), ("pad", "<i4"), ("ranges", "<u8"), ("points_xy", "<u8"), ("sensor_pose", "<f8", (3,))])


def scan_records(ranges, points, counts, poses):
    """One scan record per scan over flat buffers (ragged stores): scan s is the counts[s] readings that start at
    sum(counts[:s]) of ranges (B,) and points (B, 2).  The caller keeps the buffers alive."""
    counts = np.asarray(counts, dtype=np.int64)
    start = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint64)
    assert ranges.flags.c_contiguous and points.flags.c_contiguous and ranges.dtype == points.dtype == np.float64
    assert len(ranges) == counts.sum() and points.shape == (len(ranges), 2)
    rec = np.zeros(max(len(counts), 1), dtype=SCAN_DTYPE)[:len(counts)]
    rec["n"] = counts
    rec["ranges"] = np.uint64(ranges.ctypes.data) + np.uint64(8) * start
    rec["points_xy"] = np.uint64(points.ctypes.data) + np.uint64(16) * start
    rec["sensor_pose"] = np.asarray(poses, dtype=np.float64).reshape(len(counts), 3)
    return rec


def port_occupancy(rec, res, rt, mp=2, th=0.1):
    """kp_occupancy_create (the C port) on scan_records: dict(width, height, stride, offset, cells, passes, hits)"""
    import ctypes as C
    from oracle import karto_port as P
    assert C.sizeof(P.KpScan) == SCAN_DTYPE.itemsize
    return P.occupancy_array(rec.ctypes.data_as(C.POINTER(P.KpScan)), len(rec), res, rt, LASER["min_range"], LASER["max_range"],
                             int(mp), th)


def occupancy_params(params):
    """(resolution, range threshold, min_pass_through, occupancy_threshold) of a fixture's params row; negative = the
    reference's defaults (2, 0.1)"""
    res, rt, mp, th = (float(v) for v in params)
    return res, rt, 2 if mp < 0 else int(mp), 0.1 if th < 0 else th
