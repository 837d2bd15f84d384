"""The single-match inputs of tests/test_single_match_gpu.py checked against the oracle alone: every parameter set is accepted and has
the intended grid and smear kernel, every case has a real answer, the long queries straddle the shared-memory limits of the
correlation kernel, the explicit windows fall on the intended side of the two kernels' boundary (and of the 65,535-block grid
limit), and the fine-pass centres reach the covariance fallback (the averaged best pose rounds to a cell that was not searched).

The configurations are defined here and imported by the GPU test."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H

# slam_toolbox's config/mapper_params_online_sync.yaml: angles in radians
MAPPER_YAML = dict(coarse_search_angle_offset=0.349, coarse_angle_resolution=0.0349, fine_search_angle_offset=0.00349,
                   distance_variance_penalty=0.5, angle_variance_penalty=1.0, minimum_distance_penalty=0.5,
                   minimum_angle_penalty=0.9, use_response_expansion=1)

# name: (mapper, (searchSize, resolution, smearDeviation, rangeThreshold), (grid width, stride, smear kernel size))
GEOMETRIES = {
    "seq_shipped": (MAPPER_YAML, (0.5, 0.01, 0.1, 20.0), (4093, 4096, 41)),
    "loop_shipped": (MAPPER_YAML, (8.0, 0.05, 0.03, 20.0), (965, 968, 3)),
    "seq_20m": (H.MAPPER_SEQ, (1.0, 0.01, 0.03, 20.0), (4115, 4120, 13)),
    "loop_20m": (H.MAPPER_LOOP, (4.0, 0.05, 0.03, 20.0), (885, 888, 3)),
    "smear_half": (H.MAPPER_LOOP, (4.0, 0.05, 0.025, 12.0), (565, 568, 3)),
    "smear_10x": (H.MAPPER_LOOP, (4.0, 0.05, 0.5, 12.0), (603, 608, 41)),
    "res_10cm": (H.MAPPER_LOOP, (2.0, 0.1, 0.1, 12.0), (267, 272, 5)),
}
QUERIES = ("match", "partial", "far")

# reported query poses the synthetic trajectories never produce: the origin (Transform::SetTransform's identity branch), headings
# whose coarse window crosses +-pi, a heading beyond 2 pi (normalize_angle's multi-wrap branch), large negative coordinates
POSES = {"origin": (0.0, 0.0, 0.0), "heading_pi": (3.0, -2.0, math.pi - 0.01), "heading_minus_pi": (-3.0, 2.0, -math.pi + 0.01),
         "multi_wrap": (1.5, 2.5, 7 * math.pi + 0.3), "far_negative": (-1.0e4 + 0.37, -1.0e4 - 0.61, 0.8)}

# limits of the single-match correlation kernel (one lookup row of n int32 in dynamic shared memory)
SMEM_ATTR_BYTES = 40 * 1024      # above this the kernel's dynamic shared-memory attribute is raised before the launch
SMEM_DEFAULT_BYTES = 48 * 1024   # the per-block limit without that attribute
ROW_BYTES_MAX = 200 * 1024       # longest row accepted: 51,200 readings
LONG_BEAMS = (10240, 10241, 12288, 12289, 30000, 51200)
REFUSED_BEAMS = 51201

FEW_ITEMS = 2048                 # P * nAngles up to this runs the warp-per-(pose, angle) kernel, above it the block kernel
MAX_GRID_Y = 65535               # CUDA's limit on gridDim.y, the block kernel's angle axis

# explicit CorrelateScan windows on the GRID_LOOP raster: (searchSpaceOffset, searchSpaceResolution, angle offset, angle
# resolution) and the expected (nX, nY, nAngles)
WINDOWS = {
    "few_2048": ((0.175, 0.175), (0.05, 0.05), math.radians(15.5), math.radians(1.0), (8, 8, 32)),
    "block_2112": ((0.175, 0.175), (0.05, 0.05), math.radians(16.0), math.radians(1.0), (8, 8, 33)),
    "one_pose_few": ((0.0, 0.0), (0.05, 0.05), math.radians(10.0), math.radians(1.0), (1, 1, 21)),
    "one_pose_block": ((0.0, 0.0), (0.05, 0.05), math.radians(10.24), math.radians(0.01), (1, 1, 2049)),
    "rect_few": ((0.3, 0.1), (0.05, 0.05), math.radians(10.0), math.radians(1.0), (13, 5, 21)),
    "rect_block": ((0.3, 0.1), (0.05, 0.05), math.radians(20.0), math.radians(1.0), (13, 5, 41)),
    "odd_block": ((0.55, 0.45), (0.05, 0.05), math.radians(2.0), math.radians(1.0), (23, 19, 5)),
}
# +-180 deg at 0.005 deg on the GRID_SMALL coarse window: more angles than the block kernel's grid can hold in y
WIDE = dict(grid=H.GRID_SMALL, mapper=dict(H.MAPPER_LOOP, coarse_search_angle_offset=math.pi,
                                           coarse_angle_resolution=math.radians(0.005), fine_search_angle_offset=math.radians(0.001)),
            beams=90, dims=(6, 6, 72001))

# fine-pass centres at half-cell boundaries on the shipped-smear sequential raster (GRID_SEQ_YAML), few-beam queries
FALLBACK_READINGS = (3, 7, 9)
FALLBACK_CELLS = 20              # centres in the 2 * 20 cells around the query, each +-2 ulps


def port_case(case: synth.SingleMatchCase):
    """(query, base scans) of a case as oracle scans"""
    q = P.PortScan(case.query_ranges, case.query_pose, *case.query_laser)
    return q, [P.PortScan(r, p, *case.base_laser) for r, p in zip(case.base_ranges, case.base_poses)]


def n_angles(offset: float, resolution: float) -> int:
    return int(math.floor(offset * 2.0 / resolution + 0.5)) + 1


def world_to_grid(w: float, offset: float, resolution: float) -> int:
    """sm_math.cuh world_to_grid (Karto.h WorldToGrid with round-half-away)"""
    v = (w - offset) * (1.0 / resolution)
    return int(math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5))


def geometry_case(name: str, query: str) -> synth.SingleMatchCase:
    grid = GEOMETRIES[name][1]
    return synth.make_single_match_case(10 + list(GEOMETRIES).index(name), query=query, search_size=grid[0])


def pose_case(name: str) -> synth.SingleMatchCase:
    return synth.make_single_match_case(40 + list(POSES).index(name), pose=POSES[name])


def long_case(n: int) -> synth.SingleMatchCase:
    return synth.make_single_match_case(n % 997, n_beams=n, fov_deg=360.0)


def window_case() -> synth.SingleMatchCase:
    return synth.make_single_match_case(61)


def wide_case() -> synth.SingleMatchCase:
    return synth.make_single_match_case(62, n_beams=WIDE["beams"], fov_deg=360.0)


def fallback_case(n_readings: int) -> synth.SingleMatchCase:
    """a sequential case reported at its true pose, the query cut down to n_readings"""
    c = synth.make_sequential_case(3, buffer_len=4)
    return synth.make_few_beam_query(synth.SingleMatchCase(c["query_ranges"], c["query_true"], c["base_ranges"], c["base_poses"]),
                                     n_readings)


def fine_window(mapper, grid):
    """(searchSpaceOffset, searchSpaceResolution, angle offset, angle resolution) of MatchScan's fine pass (Mapper.cpp:621-629)"""
    res = 1.0 / (1.0 / grid[1])
    return (res, res), (res, res), 0.5 * mapper["coarse_angle_resolution"], mapper["fine_search_angle_offset"]


def fallback_centres(n_readings: int, do_penalize: bool):
    """Fine-pass centres for fallback_case(n_readings) with the oracle's answer at each: a list of (centre, flagged, (response,
    mean, cov)), flagged when the averaged best pose rounds to a cell outside the 3 x 3 searched cells"""
    mapper, grid = H.MAPPER_SEQ, H.GRID_SEQ_YAML
    case = fallback_case(n_readings)
    q, base = port_case(case)
    pm = H.port_matcher(mapper, grid)
    pm.raster(q, base)
    offx, offy = pm.grid()["offset"]
    so, sr, ao, ar = fine_window(mapper, grid)
    k0 = world_to_grid(case.query_pose[0], offx, grid[1])
    out = []
    for cx in synth.half_cell_centres(offx, grid[1], range(k0 - FALLBACK_CELLS, k0 + FALLBACK_CELLS)):
        c = np.array([cx, case.query_pose[1], case.query_pose[2]])
        r, mean, cov, _ = pm.correlate(q, c, so, sr, ao, ar, do_penalize, True)
        xs = {world_to_grid(c[0] + (-so[0] + k * sr[0]), offx, grid[1]) for k in range(3)}
        ys = {world_to_grid(c[1] + (-so[1] + k * sr[1]), offy, grid[1]) for k in range(3)}
        flagged = world_to_grid(mean[0], offx, grid[1]) not in xs or world_to_grid(mean[1], offy, grid[1]) not in ys
        out.append((c, flagged, (r, mean, cov)))
    return out


def assert_real_answer(vol):
    assert vol.max() > 0
    assert (vol == vol.max()).sum() < vol.size   # not every pose ties


# --------------------------------------------------------------------------------------------------------------------------------
def test_generators_are_deterministic():
    for make in (lambda: geometry_case("loop_20m", "far"), lambda: pose_case("origin"), lambda: long_case(10241),
                 lambda: fallback_case(9)):
        a, b = make(), make()
        for f in ("query_ranges", "query_pose", "base_ranges", "base_poses", "query_laser", "base_laser"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert np.array_equal(synth.make_dense_base((3.0, 4.0, 0.0), 0.05)[0][1], synth.make_dense_base((3.0, 4.0, 0.0), 0.05)[0][1])


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_geometry_is_accepted_and_every_query_kind_has_its_answer(name):
    mapper, grid, (width, stride, ksize) = GEOMETRIES[name]
    pm = H.port_matcher(mapper, grid)   # ScanMatcher::Create accepts the parameter set
    so, sr = H.coarse_search(grid)
    for kind in QUERIES:
        case = geometry_case(name, kind)
        q, base = port_case(case)
        pm.raster(q, base)
        g = pm.grid()
        assert (g["width"], g["stride"], g["kernel_size"]) == (width, stride, ksize)
        assert g["data"].max() == 100                # a non-empty raster
        r, _, _, vol = pm.correlate(q, case.query_pose, so, sr, mapper["coarse_search_angle_offset"],
                                    mapper["coarse_angle_resolution"], False, False)
        side = int(round(2 * so[0] / sr[0])) + 1
        assert vol.shape == (side, side, n_angles(mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"]))
        if kind == "far":
            assert r == 0.0 and vol.max() == 0        # MatchScan then runs the response-expansion passes
        else:
            assert_real_answer(vol)
    if name == "seq_shipped":
        assert stride * width > 16_000_000            # the 16.8 MB grid of the shipped sequential matcher at 20 m


@pytest.mark.parametrize("name", list(POSES))
def test_pose_cases_sit_where_intended_and_match(name):
    case = pose_case(name)
    assert np.array_equal(case.query_pose, np.array(POSES[name]))
    if name == "origin":
        assert case.query_pose[0] == 0.0 and case.query_pose[1] == 0.0 and case.query_pose[2] == 0.0
    off = H.MAPPER_SEQ["coarse_search_angle_offset"]
    if name.startswith("heading"):
        assert abs(case.query_pose[2]) + off > math.pi      # the coarse window crosses the wrap
    if name == "multi_wrap":
        assert case.query_pose[2] > 2 * math.pi
    q, base = port_case(case)
    pm = H.port_matcher(H.MAPPER_SEQ, H.GRID_SEQ)
    pm.raster(q, base)
    so, sr = H.coarse_search(H.GRID_SEQ)
    assert_real_answer(pm.correlate(q, case.query_pose, so, sr, off, H.MAPPER_SEQ["coarse_angle_resolution"], False, False)[3])


def test_long_queries_straddle_the_shared_memory_limits():
    rows = {n: 4 * n for n in LONG_BEAMS}
    for limit in (SMEM_ATTR_BYTES, SMEM_DEFAULT_BYTES):
        assert limit in rows.values() and limit + 4 in rows.values()   # at the limit and one reading above
    assert max(rows.values()) == ROW_BYTES_MAX and 4 * REFUSED_BEAMS > ROW_BYTES_MAX
    assert any(SMEM_DEFAULT_BYTES < b < ROW_BYTES_MAX for b in rows.values())


@pytest.mark.parametrize("n", LONG_BEAMS)
def test_long_query_has_a_real_answer(n):
    case = long_case(n)
    assert case.query_ranges.shape == (n,) and np.isfinite(case.query_ranges).sum() > n // 2
    q, base = port_case(case)
    pm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    pm.raster(q, base)
    so, sr = H.coarse_search(H.GRID_LOOP)
    vol = pm.correlate(q, case.query_pose, so, sr, H.MAPPER_LOOP["coarse_search_angle_offset"],
                       H.MAPPER_LOOP["coarse_angle_resolution"], False, False)[3]
    assert vol.shape[0] * vol.shape[1] * vol.shape[2] > FEW_ITEMS    # the coarse pass runs the block kernel
    assert_real_answer(vol)


def test_windows_fall_on_the_intended_side_of_each_kernel_limit():
    case = window_case()
    q, base = port_case(case)
    pm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    pm.raster(q, base)
    sides = {}
    for name, (so, sr, ao, ar, dims) in WINDOWS.items():
        r, _, _, vol = pm.correlate(q, case.query_pose, so, sr, ao, ar, False, False)
        nx, ny, na = dims
        assert vol.shape == (ny, nx, na), name
        assert r > 0, name
        sides[name] = nx * ny * na <= FEW_ITEMS
        assert sides[name] == name.startswith(("few", "one_pose_few", "rect_few")), name
    assert WINDOWS["few_2048"][4][0] * WINDOWS["few_2048"][4][1] * WINDOWS["few_2048"][4][2] == FEW_ITEMS
    assert any(d[0] != d[1] for *_, d in WINDOWS.values())
    assert any((d[0] * d[1]) % 32 and d[0] * d[1] > 32 and d[0] * d[1] * d[2] > FEW_ITEMS for *_, d in WINDOWS.values())


def test_wide_window_exceeds_the_grid_limit():
    mapper, grid = WIDE["mapper"], WIDE["grid"]
    case = wide_case()
    q, base = port_case(case)
    pm = H.port_matcher(mapper, grid)
    pm.raster(q, base)
    so, sr = H.coarse_search(grid)
    r, _, _, vol = pm.correlate(q, case.query_pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"],
                                False, False)
    nx, ny, na = WIDE["dims"]
    assert vol.shape == (ny, nx, na) and na == n_angles(mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"])
    assert na > MAX_GRID_Y and nx * ny * na > FEW_ITEMS
    assert r > 0
    assert_real_answer(vol)


def test_fallback_centres_reach_the_extra_column():
    ar = H.MAPPER_SEQ["fine_search_angle_offset"]
    flagged = [(n, pen, res) for n in FALLBACK_READINGS for pen in (False, True)
               for _, f, res in fallback_centres(n, pen) if f]
    assert any(res[0] > 0 for _, _, res in flagged)
    # the extra column is not all zeros: its angular variance is not the all-zero value
    assert any(res[2][2, 2] != 1000 * ar * ar for _, _, res in flagged)
    # most centres round into the searched cells
    assert len(flagged) < len(FALLBACK_READINGS) * 2 * 2 * FALLBACK_CELLS * 5 // 4
