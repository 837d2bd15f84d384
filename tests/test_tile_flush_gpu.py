"""The accumulator flush of the tiled sweep kernel (csrc/sm_tile.cu): every lane reduces all of its 16-bit fields unconditionally,
with the fields that are not poses of the item masked to zero -- columns past nX in the last x-tile, columns before 0 at x-tile 0,
rows past the last pose row of the last y-tile, and the tail row outside lane-row 0 -- and the masked fields' addresses kept
inside the accumulator volume or its guard words.  Each case runs on both y-tile layouts (B200_TILE_TAIL) and on one- and
two-CTA clusters, bit-exact against the oracle (responses, means, covariances) on sampled pairs."""
from __future__ import annotations

import numpy as np
import pytest

from slam_toolbox_b200 import synth
import helpers as H

pytestmark = pytest.mark.gpu

MAPPER = dict(H.MAPPER_LOOP, use_response_expansion=0)

# (search dimension, resolution, smear, range threshold) -> poses per side = floor(dim / res + 0.5) // 2 + 1; sweep seed, queries
CASES = {
    "nx41_headline": ((4.0, 0.05, 0.03, 12.0), 41, 900, 1),   # last x-tile: columns 41..47 masked; 48-row tiles: 7 idle rows
    "nx45_idle_rows": ((4.4, 0.05, 0.03, 12.0), 45, 901, 1),  # 48-row y-tile on both settings: rows 45..47 idle
    "nx23_odd": ((2.2, 0.05, 0.03, 12.0), 23, 902, 1),        # odd window, one and a half x-tiles
    "nx4_tiny": ((0.3, 0.05, 0.03, 12.0), 4, 903, 1),         # a single x-tile: 12 of 16 columns and most row tiles masked
    "nx3_tiny": ((0.2, 0.05, 0.03, 12.0), 3, 904, 1),
    "nx41_edge": ((4.0, 0.05, 0.03, 6.0), 41, 35, 2),         # short range threshold: EDGE items flush through the same path
    "nx81_two_ytiles": ((8.0, 0.05, 0.03, 12.0), 81, 906, 1),  # tail layout: items of the first y-tile carry no tail row
}


def _expected(pm, sw, nq, nch):
    pc, pq = H.port_scans(sw.cand_ranges, sw.cand_poses), H.port_scans(sw.query_ranges, sw.query_poses)
    exp = [pm.match(pq[q], pc[sw.chain_start[c]:sw.chain_start[c + 1]], False, False) for q in range(nq) for c in range(nch)]
    return np.array([e[0] for e in exp]), np.array([e[1] for e in exp]), np.array([e[2] for e in exp])


@pytest.mark.parametrize("tail", [0, 1])
@pytest.mark.parametrize("name", sorted(CASES))
def test_flush_masks_vs_oracle(monkeypatch, name, tail):
    grid, side, seed, nq = CASES[name]
    monkeypatch.setenv("B200_TILE_TAIL", str(tail))
    nch = 6
    sw = synth.make_loop_sweep(seed, n_queries=nq, n_chains=nch, chain_len=2, inf_frac=0.02)
    pm, gm = H.port_matcher(MAPPER, grid), H.gpu_matcher(MAPPER, grid)
    gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
    er, em, ec = _expected(pm, sw, nq, nch)
    assert er.max() > 0.0, "the case must produce responses"
    gm.set_option("sweep_kernel", 2)
    for cluster in (1, 2):
        gm.set_option("sweep_cluster", cluster)
        r, m, c = gm.MatchScanBatch(gq, gc, sw.chain_start, None, False, False)
        info, plan = gm.batch_info(), gm.batch_tile_info()
        assert info["kernel"] == "tile" and plan["available"], (info, plan)
        assert plan["xtiles"] == (side + 3 + 15) // 16, (side, plan)
        if not tail:
            assert not plan["tail"] and plan["ytile_rows"] == 48, plan
        if plan["tail"]:
            assert plan["ytile_rows"] == 40, plan
        if name == "nx81_two_ytiles" and tail:
            assert plan["tail"] and plan["ytiles"] == 2, plan
        if name == "nx45_idle_rows":
            assert not plan["tail"], plan
        if name == "nx41_edge":
            assert info["edge_beams"] > 0, info
        assert np.array_equal(r, er), (name, plan, r, er)
        assert np.array_equal(m, em) and np.array_equal(c, ec), (name, plan)
