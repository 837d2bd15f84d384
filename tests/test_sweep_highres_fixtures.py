"""The high-resolution sweep inputs of synth.make_highres_sweep checked against the oracle alone: the generator is deterministic,
every configuration the GPU tests run has a coarse lookup table larger than the 200 KB the generic kernel stages at once (so it
runs in angle slices), and the oracle's answers are not degenerate (a positive best response that not every pose shares).

The configurations are defined here and imported by tests/test_sweep_highres_gpu.py."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H

MAPPER = dict(H.MAPPER_LOOP, use_response_expansion=0)                         # +-20 deg / 2 deg: 21 angles
MAPPER_1DEG = dict(MAPPER, coarse_angle_resolution=math.radians(1.0))          # +-20 deg / 1 deg: 41 angles
MAPPER_WIDE = dict(MAPPER, coarse_search_angle_offset=math.radians(90.0))      # +-90 deg / 2 deg: 91 angles
MAPPERS = {21: MAPPER, 41: MAPPER_1DEG, 91: MAPPER_WIDE}
GRIDS = {"4m12": H.GRID_LOOP, "8m12": (8.0, 0.05, 0.03, 12.0), "4m20": (4.0, 0.05, 0.03, 20.0), "yaml": H.GRID_SEQ_YAML}
FOV = {1081: 270.0, 2701: 270.0, 3600: 360.0, 8192: 360.0}   # 0.25 deg, 0.1 deg over 270 / 360 deg, a flattened 3-D lidar
TABLE_BYTES = 200 * 1024   # lookup rows the generic kernel stages in shared memory at once

# (beams, grid, angles): 0.1 deg lidars on the three shipped geometries at both windows, the +-90 deg window on the standard
# laser, more than 4096 beams (the tiled kernel reads candidate cell lists from global memory), and the order-dependent raster
CONFIGS = [(n, g, a) for n in (2701, 3600) for g in ("4m12", "8m12", "4m20") for a in (21, 41)] + \
          [(1081, "4m12", 91), (8192, "4m12", 21), (2701, "yaml", 21)]


def config_id(c):
    return f"{c[0]}-{c[1]}-{c[2]}"


def sweep(n: int, n_chains: int = 2) -> synth.AdversarialSweep:
    return synth.make_highres_sweep(n, FOV[n], n_chains=n_chains)


def n_angles(mapper) -> int:
    """angles of the coarse pass (Mapper.cpp:755-756: nAngles = Round(2 * offset / resolution) + 1)"""
    return int(math.floor(2 * mapper["coarse_search_angle_offset"] / mapper["coarse_angle_resolution"] + 0.5)) + 1


def port_scans(ranges, poses, laser):
    return [P.PortScan(r, p, laser[0], laser[1]) for r, p in zip(np.atleast_2d(ranges), np.atleast_2d(poses))]


def test_generator_is_deterministic_and_shaped_like_the_laser():
    for n in (2701, 3600):
        a, b = sweep(n), sweep(n)
        for f in ("query_ranges", "query_poses", "cand_ranges", "cand_poses", "chain_start"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
        assert a.query_ranges.shape == (1, n) and a.cand_ranges.shape == (2, n)
        assert a.query_laser == a.cand_laser
        assert abs(math.degrees(a.query_laser[1]) - 0.1) < 1e-12          # 0.1 deg between readings
        assert np.isfinite(a.query_ranges).all() and (a.query_ranges > 0).all()
    assert synth.highres_laser(1081, 270.0) == (synth.ANGLE_MIN, (synth.ANGLE_MAX - synth.ANGLE_MIN) / 1080)


@pytest.mark.parametrize("config", CONFIGS, ids=config_id)
def test_configuration_needs_angle_slices_and_has_a_real_answer(config):
    n, g, na = config
    mapper, grid = MAPPERS[na], GRIDS[g]
    assert n_angles(mapper) == na
    # the whole table no longer fits: the generic kernel needs at least two slices
    assert na * n * 4 > TABLE_BYTES
    rows = TABLE_BYTES // (4 * n)
    assert -(-na // rows) >= 2
    if n == 8192:
        assert n > 4096   # candidate scans of more than 4096 readings: no shared-memory staging of the cell lists
    sw = sweep(n)
    pm = H.port_matcher(mapper, grid)
    q = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)[0]
    assert len(pm.offsets(q, q.pose[2], mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"])) == na
    cs = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
    off, res = H.coarse_search(grid)
    for c in range(len(sw.chain_start) - 1):
        base = cs[sw.chain_start[c]:sw.chain_start[c + 1]]
        pm.raster(q, base)
        vol = pm.correlate(q, q.pose, off, res, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], False,
                           False)[3]
        assert vol.shape[2] == na
        assert vol.max() > 0, (config, c)
        assert (vol == vol.max()).sum() < vol.size, (config, c)   # not every pose ties
