"""The tiled sweep kernel's weighted entries and tail row (csrc/sm_tile.cu): cells that k >= 2 beams of a descriptor group share
are one entry of weight k, entries of equal weight are loaded as pairs, and 2k + 1-row search windows run on 40-row y-tiles plus
a tail row read lane-parallel over the entries.  synth.make_weighted_sweep builds groups of chosen weights; every run is bit-exact
against the oracle, with and without beam dedup, on several cluster sizes and chunkings, and on windows of 41, 45 (48-row
y-tiles), 81 and 6 rows.  The *_fixture tests check on the CPU, with the oracle's lookup table, that each case holds the group it
is meant to exercise."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H
from test_sweep_adversarial_gpu import Case, MAPPER

GRID_DIM8 = (8.0, 0.05, 0.03, 12.0)
GRID_DIM44 = (4.4, 0.05, 0.03, 12.0)   # 45-row window: 48-row y-tiles load less than 2 x 40 rows + the tail
SMALL_MAPPER = dict(MAPPER, coarse_search_angle_offset=math.radians(4.0))

# cell weights of the query (see synth.make_weighted_sweep): at the central angle all cells are in one group
WEIGHTS = {
    "pairs_only": [2] * 100,                                   # weight-2 cells only: 50 pairs
    "mixed_odd": [2, 2, 2, 3, 3, 4, 5, 5, 5, 7, 1, 1, 1] * 7,   # equal weights paired, odd leftovers as singles, odd plain list
    "w639": [2] * 319 + [1],                                   # 319 weight-2 entries + 1 plain beam: one flush
    "w640": [2] * 320,                                         # 320 merged entries (> 213), 160 pairs
    "w641": [2] * 320 + [1],                                   # above one flush: dedup off, 641 plain beams
    "w3x100": [3] * 100,                                       # 100 weight-3 cells: with pairing off, more singles than the
}                                                              # item record's 6-bit count holds (the rest go back to plain beams)
TAIL_ROWS = {41: True, 81: True, 45: False, 6: True}   # window rows -> the planner takes 40-row y-tiles + the tail row


def weighted_sweep(name):
    return synth.make_weighted_sweep(WEIGHTS[name])


def lookup_groups(sw, mapper, grid):
    """per search angle: {(column mod 8, row mod 2): sorted cell weights} of the query's beams (one band: the descriptor groups)"""
    pm = H.port_matcher(mapper, grid)
    q = P.PortScan(sw.query_ranges[0], sw.query_poses[0], *sw.query_laser)
    pm.raster(q, [P.PortScan(sw.cand_ranges[0], sw.cand_poses[0], *sw.cand_laser)])
    stride = pm.grid()["stride"]
    offs = pm.offsets(q, q.pose[2], mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"])
    out = []
    for o in offs:
        o = o[o != np.iinfo(np.int32).max].astype(np.int64)
        gy = np.rint(o / stride).astype(np.int64)
        key = ((o - gy * stride) % 8) * 2 + gy % 2
        out.append({int(k): np.sort(np.unique(o[key == k], return_counts=True)[1]) for k in np.unique(key)})
    return out


def central_group(sw, mapper=MAPPER, grid=H.GRID_LOOP):
    gs = lookup_groups(sw, mapper, grid)
    g = gs[len(gs) // 2]
    return max(g.values(), key=lambda w: w.sum())


@pytest.mark.parametrize("name", sorted(WEIGHTS))
def test_weighted_groups_fixture(name):
    w = central_group(weighted_sweep(name))
    want = np.sort(np.array(WEIGHTS[name]))
    assert np.array_equal(w, want), (name, np.unique(w, return_counts=True))
    if name == "pairs_only":
        assert set(w) == {2}
    if name == "mixed_odd":
        vals, cnt = np.unique(w[w >= 2], return_counts=True)
        assert (cnt % 2 == 1).any() and (cnt % 2 == 0).any() and (w == 1).sum() % 2 == 1, (vals, cnt)
    if name.startswith("w6"):
        assert w.sum() == int(name[1:]) and (w >= 2).sum() > 213
    if name == "w3x100":
        assert set(w) == {3} and len(w) > 63


def test_tail_layout_windows_fixture():
    """window rows of the geometries below: 41 and 81 (= 40 k + 1), 45, 6 (tiny); the GPU tests check the planner's layout"""
    for grid, rows in ((H.GRID_LOOP, 41), (GRID_DIM8, 81), (GRID_DIM44, 45), (H.GRID_SMALL, 6)):
        off, res = H.coarse_search(grid)
        assert int(round(2 * off[1] / res[1])) + 1 == rows, grid


def test_edge_beams_reach_the_tail_row_fixture():
    """make_dense_sweep(edge=True): clusters whose pose windows leave the grid through its left side, with every row of the
    window (the tail row too) inside the grid"""
    sw = synth.make_dense_sweep((1281,), edge=True)
    pm = H.port_matcher(MAPPER, H.GRID_LOOP)
    q = P.PortScan(sw.query_ranges[0], sw.query_poses[0], *sw.query_laser)
    pm.raster(q, [P.PortScan(r, p, *sw.cand_laser) for r, p in zip(sw.cand_ranges, sw.cand_poses)])
    g = pm.grid()
    off, res = H.coarse_search(H.GRID_LOOP)
    half = int(round(off[1] / (res[1] / 2)))   # window half-height in cells
    o = pm.offsets(q, q.pose[2], MAPPER["coarse_search_angle_offset"], MAPPER["coarse_angle_resolution"])[10]
    o = o[o != np.iinfo(np.int32).max].astype(np.int64)
    gy = np.rint(o / g["stride"]).astype(np.int64)
    gx = o - gy * g["stride"]
    cx, cy = g["width"] // 2 + gx, g["height"] // 2 + gy
    assert (cx - half < 0).all()                                      # windows leave the grid on the left: EDGE beams
    assert ((cy - half >= 0) & (cy + half < g["height"])).all()       # all rows, the last (tail) row too, are in the grid


def window_rows(grid):
    off, res = H.coarse_search(grid)
    return int(round(2 * off[1] / res[1])) + 1


def _check(case, opts, expect_tile=True):
    gm = case.matcher()
    for o in opts:
        info, plan, st, fs, best = case.run(gm, o)
        case.check_best(best, o)
        if expect_tile:
            assert info["kernel"] == "tile" and plan["available"], (o, info, plan)
            rows = window_rows(case.grid)
            assert plan["tail"] == TAIL_ROWS[rows] and plan["ytile_rows"] == (40 if plan["tail"] else 48), (rows, plan)
    return gm


def _opts(clusters=(1, 2, 8), chunks=(0, 21), dedup=(0, 1)):
    return [dict(force_generic_sweep=0, sweep_kernel=2, sweep_cluster=cl, sweep_chunks=ch, no_beam_dedup=d)
            for cl in clusters for ch in chunks for d in dedup]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WEIGHTS))
def test_weighted_groups_vs_oracle(name):
    case = Case(weighted_sweep(name), MAPPER, H.GRID_LOOP)
    gm = _check(case, _opts())
    gm.set_option("no_beam_dedup", 0)
    gm.set_option("sweep_cluster", 1)
    gm.set_option("sweep_chunks", 0)
    case.run(gm, {})
    st = gm.batch_tile_stats()
    if name == "w641":
        assert st["max_multiplicity"] <= 2, st    # the central group is not merged (other angles' smaller groups are)
    else:
        assert st["max_multiplicity"] >= 2 and st["multi_entries"] > 0, st
    if name in ("w639", "w640"):
        assert st["multi_entries"] >= 319, st


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w3x100", "mixed_odd", "w640"])
@pytest.mark.parametrize("pairs,tail", [(0, 1), (1, 0), (0, 0)])
def test_each_part_switched_off_vs_oracle(monkeypatch, name, pairs, tail):
    """B200_TILE_PAIRS=0 (cells of weight >= 3 as singles, no pairing: 100 weight-3 cells are more singles than one record
    holds) and B200_TILE_TAIL=0 (48-row y-tiles at 41 rows): the same bits"""
    monkeypatch.setenv("B200_TILE_PAIRS", str(pairs))
    monkeypatch.setenv("B200_TILE_TAIL", str(tail))
    case = Case(weighted_sweep(name), MAPPER, H.GRID_LOOP)
    gm = case.matcher()
    for o in _opts(clusters=(1, 2), chunks=(0, 21), dedup=(0, 1)):
        info, plan, st, fs, best = case.run(gm, o)
        case.check_best(best, o)
        assert info["kernel"] == "tile" and plan["available"] and plan["tail"] == bool(tail), (o, info, plan)
        if o["no_beam_dedup"]:
            continue
        if not pairs and name == "w640":
            assert st["max_multiplicity"] <= 1, st      # weight-2 cells stay plain beams without pairing
        else:
            assert st["max_multiplicity"] >= (2 if name == "w640" else 3), st


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [GRID_DIM8, GRID_DIM44, H.GRID_SMALL])
def test_weighted_groups_on_other_windows(grid):
    """81-row (tail layout, two y-tiles), 45-row (48-row y-tiles) and 6-row windows"""
    mapper = SMALL_MAPPER if grid == GRID_DIM8 else MAPPER
    case = Case(weighted_sweep("mixed_odd"), mapper, grid)
    _check(case, _opts(clusters=(1, 8), chunks=(0, 3)))


@pytest.mark.gpu
def test_room_scans_on_tail_and_48_row_windows():
    """room scans (make_loop_sweep: weight-1, -2 and -3+ cells mixed) on 41-, 45- and 81-row windows"""
    sw = synth.make_loop_sweep(91, n_queries=2, n_chains=4, chain_len=2, inf_frac=0.02)
    asw = synth.AdversarialSweep(sw.query_ranges, sw.query_poses, sw.cand_ranges, sw.cand_poses, sw.chain_start,
                                 (synth.ANGLE_MIN, synth.ANGLE_INC), (synth.ANGLE_MIN, synth.ANGLE_INC))
    for grid, mapper in ((H.GRID_LOOP, MAPPER), (GRID_DIM44, MAPPER), (GRID_DIM8, SMALL_MAPPER)):
        case = Case(asw, mapper, grid)
        _check(case, _opts(clusters=(1, 2, 8), chunks=(0, 5), dedup=(0, 1)))


@pytest.mark.gpu
def test_edge_beams_reach_the_tail_row():
    case = Case(synth.make_dense_sweep((1281,), edge=True), MAPPER, H.GRID_LOOP)
    gm = _check(case, _opts(clusters=(1, 2), chunks=(0, 21), dedup=(0,)))
    assert gm.batch_info()["edge_beams"] > 0 and gm.batch_tile_info()["tail"]
