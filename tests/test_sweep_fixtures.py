"""The adversarial sweep inputs of synth.py (make_dense_sweep, make_tie_sweep, make_long_query_sweep) checked against the oracle
alone, so that a generator that drifts away from the case it was built for fails on any machine: how many beams share one cell
per search angle, how many poses tie for the best, and the s / s - 1 near tie of the long query."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H

MAPPER = dict(H.MAPPER_LOOP, use_response_expansion=0)
MAPPER_NARROW = dict(MAPPER, coarse_search_angle_offset=math.radians(2.0))   # 3 angles: lookup tables of 10 000 beams fit
GRID_DIM8 = (8.0, 0.05, 0.03, 12.0)
GRID_SMEAR5 = (4.0, 0.05, 0.05, 12.0)   # 5 x 5 smear kernel


def port_scans(ranges, poses, laser):
    return [P.PortScan(r, p, laser[0], laser[1]) for r, p in zip(np.atleast_2d(ranges), np.atleast_2d(poses))]


def oracle_volume(pm, mapper, grid, q, base):
    """integer sums [nY, nX, nA] of the coarse pass of MatchScan(q, base)"""
    pm.raster(q, base)
    off, res = H.coarse_search(grid)
    return pm.correlate(q, q.pose, off, res, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], False,
                        False)[3]


def same_cell_counts(pm, mapper, q):
    """per search angle: the largest number of the query's beams that look up one grid cell"""
    offs = pm.offsets(q, q.pose[2], mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"])
    return [int(np.unique(o[o != np.iinfo(np.int32).max], return_counts=True)[1].max()) for o in offs]


@pytest.mark.parametrize("clusters,edge", [((639,), False), ((640,), False), ((641,), False), ((1280,), False),
                                           ((1281, 639), False), ((1920,), False), ((1281,), True)])
def test_dense_query_piles_each_cluster_into_one_cell(clusters, edge):
    sw = synth.make_dense_sweep(clusters, edge=edge)
    assert sw.query_ranges.shape == (1, sum(clusters))
    for grid in (H.GRID_LOOP, GRID_DIM8):
        pm = H.port_matcher(MAPPER, grid)
        q = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)[0]
        pm.raster(q, port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser))   # sets the grid origin the offsets refer to
        assert same_cell_counts(pm, MAPPER, q) == [max(clusters)] * 21, grid
        # the ring chain puts the whole cluster on occupied cells: the best pose scores 100 per beam of the largest cluster
        cs = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        vol = oracle_volume(pm, MAPPER, grid, q, cs[sw.chain_start[-2]:sw.chain_start[-1]])
        assert vol.max() >= 100 * max(clusters), grid


@pytest.mark.parametrize("k", sorted(synth.TIE_BEAMS))
def test_tie_query_has_exactly_k_best_poses(k):
    sw = synth.make_tie_sweep((k,))
    pm = H.port_matcher(MAPPER, H.GRID_LOOP)
    q = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)[0]
    base = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
    vol = oracle_volume(pm, MAPPER, H.GRID_LOOP, q, base)
    assert int((pm.grid()["data"] == 100).sum()) == 1    # one occupied cell
    assert vol.max() == 100 and int((vol == 100).sum()) == k
    if k > 1:
        assert len(np.unique(np.nonzero(vol == 100)[2])) > 1   # the ties sit at several angles (several angle chunks)


def test_long_queries_straddle_the_integer_tie_rule():
    pm = H.port_matcher(MAPPER_NARROW, GRID_SMEAR5)
    for n, int_rule in ((8990, True), (10240, False)):
        sw = synth.make_long_query_sweep(n)
        assert sw.query_ranges.shape == (1, n)
        assert (n * 100 < 0.9e6) == int_rule   # the integer tie rule (sum equality) is only used below 9000 beams
        q = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)[0]
        base = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        vol = oracle_volume(pm, MAPPER_NARROW, GRID_SMEAR5, q, base[1:2])
        assert vol.shape == (41, 41, 3)
        s = np.unique(vol)
        if n == 10240:
            assert (s[-1], s[-2]) == (6705, 6704) and (vol == s[-1]).sum() == 1 and (vol == s[-2]).sum() == 1
            best, second = s[-1] / float(n * 100), s[-2] / float(n * 100)
            assert best - second <= 1e-6      # DoubleEqual: the reference counts both poses as ties of the best
