"""The tiled sweep kernel's planner in the library (b200sm_tile_plan: no handle, no device) against its plain-Python restatement
tile_plan_rule.plan over a few hundred geometries: search windows of 1 to 12 m at 0.02 to 0.1 m resolution, range thresholds of
4 to 40 m, angle windows up to and past the 4096-angle limit, 181 to 4000 beams per query with the longest candidate scan on
both sides of the 4096 readings the cell-list staging takes, penalised and not, 1 to 1000 pairs on 132 and 114 SMs, forced
cluster sizes and chunk counts, and the tail layout allowed or not."""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from slam_toolbox_b200 import api
import tile_plan_rule as T


def library_plan(g: T.Geometry, n: int, pen: bool, npairs: int, sms: int, cluster: int, chunks: int, max_n: int,
                 tail_layout: bool) -> T.Plan:
    max_n = (max(max_n, 1) + 3) & ~3   # the sweep rounds the longest candidate scan up to 4 readings
    inp = np.array([g.stride, g.height, g.nX, g.nY, g.nA, n, max_n, int(pen), npairs, sms, cluster, chunks, int(tail_layout)],
                   dtype=np.int32)
    out = np.zeros(7, dtype=np.int32)
    api._check(api.lib().b200sm_tile_plan(api._ip(inp), api._ip(out)))
    refused, cluster, chunks, bands, band_rows, smem, tail = (int(v) for v in out)
    if refused:
        return T.Plan(refused)
    return T.Plan(0, chunks, bands, band_rows, cluster, smem, bool(tail))


def cases(count: int, seed: int):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        window, res, rt = rng.uniform(1.0, 12.0), rng.uniform(0.02, 0.1), rng.uniform(4.0, 40.0)
        na = int(rng.choice([int(np.exp(rng.uniform(0.0, math.log(4096)))), 4096, 4097, 4200], p=[0.85, 0.05, 0.05, 0.05]))
        ang_res = math.radians(rng.choice([0.25, 0.5, 1.0]))
        g = T.geometry((window, res, 0.03, rt), (na - 1) / 2 * ang_res, ang_res)
        assert g.nA == na
        n = int(rng.integers(181, 4001))
        max_n = int(rng.choice([n, rng.integers(n, 4097), rng.integers(4097, 8000)]))
        cluster = int(rng.choice([0, 0, 1, 2, 4, 8]))
        chunks = int(rng.choice([0, 0, rng.integers(1, na + 1)]))
        npairs = int(np.exp(rng.uniform(0.0, math.log(1000))))
        yield g, n, bool(rng.integers(2)), npairs, int(rng.choice([132, 114])), cluster, chunks, max_n, bool(rng.integers(2))


def test_library_planner_equals_the_restatement():
    seen = set()
    for c in cases(400, 0):
        want, got = T.plan(*c[:7], max_n=c[7], tail_layout=c[8]), library_plan(*c)
        assert got == want, (c, got, want)
        seen.add(want.refused if want.refused else ("tail" if want.tail else "48-row", want.bands > 1, want.cluster))
    # the draw reaches the angle-limit and no-chunk-fits refusals, banded plans, both y-tile layouts and every cluster size
    assert {2, 4} <= seen, seen
    assert {s[0] for s in seen if isinstance(s, tuple)} == {"tail", "48-row"}, seen
    assert {s[2] for s in seen if isinstance(s, tuple)} == {1, 2, 4, 8}, seen
    assert any(s[1] for s in seen if isinstance(s, tuple)), seen


def test_library_planner_refusals_outside_the_drawn_windows():
    """an odd row stride (2) and more x-tiles than the item record's 6 bits (9)"""
    g = T.geometry((4.0, 0.05, 0.03, 12.0), math.radians(20.0), math.radians(0.5))
    for geom, want in ((dataclasses.replace(g, stride=g.stride + 1), 2), (dataclasses.replace(g, nX=1030), 9)):
        args = (geom, 1081, False, 2, 132, 0, 0, 1081, True)
        assert T.plan(*args[:7]).refused == want and library_plan(*args).refused == want, (geom, want)


def test_library_planner_rejects_out_of_range_input():
    out = np.zeros(7, dtype=np.int32)
    for i, bad in ((0, 0), (2, 4096), (5, -1), (10, -1)):
        inp = np.array([400, 400, 41, 41, 21, 1081, 1084, 0, 2, 132, 0, 0, 1], dtype=np.int32)
        inp[i] = bad
        assert api.lib().b200sm_tile_plan(api._ip(inp), api._ip(out)) == api.ERR_INVALID_ARG, (i, bad)
