"""The long-range sweep inputs of synth.make_long_range_sweep and the planner restatement of tile_plan_rule.py, checked without a
GPU: the restatement gives the plans DESIGN.md section 3.3 documents, every configuration lands in the regime it is chosen for
(its band count or its refusal code), the oracle's answers are not degenerate, and the query's readings reach the first and last
row bands of the plan, and where intended beyond the correlation grid.

The configurations are defined here and imported by tests/test_sweep_long_range_gpu.py."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H
import tile_plan_rule as T

MAPPER = dict(H.MAPPER_LOOP, use_response_expansion=0)     # +-20 deg at 2 deg: 21 angles
N_BEAMS, BATCH_PAIRS, SMS = 1081, 1000, 132                 # the regimes below are those of a 1000-pair batch on 132 SMs


def _grid(window, res, rt):
    return (window, res, 0.03, rt)


# name -> (grid, readings beyond the threshold, (plain, penalised) at one CTA per pair: the band count, or the refusal as "r4")
CONFIGS = {
    "8m-25m": (_grid(8.0, 0.05, 25.0), True, (5, 5)),           # slam_toolbox's code default max_laser_range, a 125 m lidar
    "8m-40m": (_grid(8.0, 0.05, 40.0), False, (11, 17)),
    "8m-60m": (_grid(8.0, 0.05, 60.0), True, (27, 47)),
    "8m-80m": (_grid(8.0, 0.05, 80.0), False, (95, "r4")),       # tiled when plain, generic when penalised
    "8m-100m": (_grid(8.0, 0.05, 100.0), True, ("r4", "r4")),
    "4m-150m": (_grid(4.0, 0.05, 150.0), False, (167, 167)),
    "11m-20m": (_grid(11.0, 0.05, 20.0), True, (4, 19)),
    "12m-20m": (_grid(12.0, 0.05, 20.0), False, (7, "r4")),
    "8m-0.025-20m": (_grid(8.0, 0.025, 20.0), True, ("r4", "r4")),   # 161 x 161 poses
    "4m-0.025-20m": (_grid(4.0, 0.025, 20.0), False, (11, 17)),      # 5 x 5 smear kernel
}
NAMES = list(CONFIGS)


def sweep(name: str) -> synth.AdversarialSweep:
    grid, beyond, _ = CONFIGS[name]
    return synth.make_long_range_sweep(grid[3], beyond=beyond)


def geometry(name: str) -> T.Geometry:
    return T.geometry(CONFIGS[name][0], MAPPER["coarse_search_angle_offset"], MAPPER["coarse_angle_resolution"])


def expected_regime(plan: T.Plan):
    return f"r{plan.refused}" if plan.refused else plan.bands


def beam_classes(sw, name: str, band_rows: int, nbands: int):
    """the first query's beams at the central search angle (its own heading), classified like classify_beams: inside the grid
    for every pose (FAST), leaving it by less than a grid width in x (EDGE), or by more (FAR); and the number of FAST beams
    per row band of a plan with nbands bands of band_rows rows"""
    g = geometry(name)
    res = CONFIGS[name][0][1]
    border = g.ksize // 2 + 1
    roi = g.width - 2 * border
    r, s = sw.query_ranges[0], sw.query_poses[0]
    a = s[2] + sw.query_laser[0] + np.arange(len(r)) * sw.query_laser[1]
    ok = np.isfinite(r)
    cx = border + (roi - 1) // 2 + np.floor(r * np.cos(a) / res + 0.5).astype(np.int64)
    cy = border + (roi - 1) // 2 + np.floor(r * np.sin(a) / res + 0.5).astype(np.int64)
    xb, yb = cx - (g.nX - 1), cy - (g.nY - 1)   # cell of the window's first pose
    inside = ok & (xb >= 0) & (xb + 2 * (g.nX - 1) < g.stride) & (yb >= 0) & (yb + 2 * (g.nY - 1) < g.height)
    far = ok & ((xb < -g.stride) | (xb + 2 * (g.nX - 1) >= 2 * g.stride))
    edge = ok & ~inside & ~far
    bands = np.bincount(np.clip((yb[inside] >> 1) // band_rows, 0, nbands - 1), minlength=nbands)
    return int(inside.sum()), int(edge.sum()), int(far.sum()), bands


def test_restatement_reproduces_the_documented_plans():
    """DESIGN.md 3.3: 4 m/12 m -> V 2, 1 band; 8 m/12 m -> V 11, 1; 4 m/20 m -> V 2, 2; 8 m/20 m -> V 7, 3 (1000 pairs)"""
    for (window, rt), (v, nb) in {(4.0, 12.0): (2, 1), (8.0, 12.0): (11, 1), (4.0, 20.0): (2, 2), (8.0, 20.0): (7, 3)}.items():
        g = T.geometry(_grid(window, 0.05, rt), MAPPER["coarse_search_angle_offset"], MAPPER["coarse_angle_resolution"])
        p = T.plan(g, N_BEAMS, False, BATCH_PAIRS, SMS)
        assert (p.refused, p.chunks, p.bands, p.cluster) == (0, v, nb, 1), (window, rt, p)
        assert T.plan(g, N_BEAMS, False, 2, SMS).cluster == 8   # a small batch spreads each pair over a cluster
    assert T.TILE_SHARED_BYTES % 8 == 0


@pytest.mark.parametrize("name", NAMES)
def test_configuration_lands_in_its_regime(name):
    grid, beyond, regimes = CONFIGS[name]
    g = geometry(name)
    # the restated geometry is the oracle's correlation grid
    pm = H.port_matcher(MAPPER, grid)
    sw = sweep(name)
    q = P.PortScan(sw.query_ranges[0], sw.query_poses[0], *sw.query_laser)
    pm.raster(q, [P.PortScan(sw.cand_ranges[0], sw.cand_poses[0], *sw.cand_laser)])
    og = pm.grid()
    assert (og["width"], og["height"], og["stride"], og["kernel_size"]) == (g.width, g.height, g.stride, g.ksize)
    assert len(pm.offsets(q, q.pose[2], MAPPER["coarse_search_angle_offset"], MAPPER["coarse_angle_resolution"])) == g.nA
    plans = [T.plan(g, N_BEAMS, pen, BATCH_PAIRS, SMS) for pen in (False, True)]
    assert tuple(expected_regime(p) for p in plans) == regimes, (name, plans)
    for p in plans:
        if not p.refused:
            assert p.cluster == 1 and p.band_rows >= 8 and p.smem + T.TILE_SHARED_BYTES + 64 <= T.SMEM_LIMIT, p
    if name == "8m-25m":
        assert plans[0].bands >= 5
    if name == "8m-80m":   # about 8,000 (chunk, phase, band) stages per pair
        assert plans[0].bands > 50 and T.stages_per_pair(plans[0]) > 7500, plans[0]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_answer_is_not_degenerate(name):
    grid = CONFIGS[name][0]
    sw = sweep(name)
    pm = H.port_matcher(MAPPER, grid)
    q = P.PortScan(sw.query_ranges[0], sw.query_poses[0], *sw.query_laser)
    off, res = H.coarse_search(grid)
    for c in range(len(sw.chain_start) - 1):
        pm.raster(q, [P.PortScan(sw.cand_ranges[c], sw.cand_poses[c], *sw.cand_laser)])
        vol = pm.correlate(q, q.pose, off, res, MAPPER["coarse_search_angle_offset"], MAPPER["coarse_angle_resolution"], False,
                           False)[3]
        assert vol.max() > 0, (name, c)
        assert (vol == vol.max()).sum() < vol.size, (name, c)


@pytest.mark.parametrize("name", NAMES)
def test_query_readings_reach_the_outer_bands(name):
    grid, beyond, _ = CONFIGS[name]
    sw = sweep(name)
    assert sw.query_ranges.shape == (1, N_BEAMS) and np.isfinite(sw.query_ranges).all()
    rt = grid[3]
    if beyond:
        assert sw.query_ranges.max() > 2 * rt
    else:
        assert sw.query_ranges.max() <= rt and (sw.query_ranges > rt - 0.1).sum() > 50
    for pen in (False, True):
        p = T.plan(geometry(name), N_BEAMS, pen, BATCH_PAIRS, SMS)
        nb, rows = (p.bands, p.band_rows) if not p.refused else (1, 1 << 20)
        inside, edge, far, bands = beam_classes(sw, name, rows, nb)
        assert inside > 50, (name, inside)
        if nb > 1:   # FAST beams in the first and the last (shorter) band
            assert bands[0] > 0 and bands[-1] > 0, (name, pen, bands)
            assert (bands > 0).sum() >= nb // 2, (name, pen, bands)
        if beyond:
            assert edge > 100 and far > 0, (name, edge, far)
        else:
            assert edge == 0 and far == 0, (name, edge, far)


def test_noise_keeps_the_shipped_range_max():
    """noisy()'s range_max defaults to RANGE_MAX: the generators that do not pass it are unchanged"""
    rng_a, rng_b = np.random.default_rng(3), np.random.default_rng(3)
    r = np.linspace(0.0, 60.0, 101)
    assert np.array_equal(synth.noisy(r, rng_a), synth.noisy(r, rng_b, range_max=synth.RANGE_MAX))
    assert synth.noisy(r, np.random.default_rng(3)).max() == synth.RANGE_MAX
    a, b = synth.make_long_range_sweep(25.0, beyond=True), synth.make_long_range_sweep(25.0, beyond=True)
    assert all(np.array_equal(getattr(a, f), getattr(b, f)) for f in ("query_ranges", "query_poses", "cand_ranges", "cand_poses"))
    assert math.isclose(a.query_poses[0, 2], 0.0, abs_tol=0.5)
