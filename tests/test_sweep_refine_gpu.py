"""The refine pass of the batched sweep (MatchScanBatch with doRefineMatch = True: LinkNearChains' near-chain matches and the fine
stage of TryCloseLoop) against the oracle, bit for bit: the per-pair fine plans around each coarse mean, the fine kernel's
re-raster after every coarse kernel, the FP64 host epilogue, and the pairs that leave the batch for the single-match path (tie-list
overflow, response expansion, the fine-covariance fallback) mixed with ordinary pairs.  Tolerances: none.  The inputs and the
branch each pair takes are defined and pinned against the oracle in test_sweep_refine_fixtures.py."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from slam_toolbox_b200 import api, synth
from test_sweep_adversarial_gpu import Case
import helpers as H
import test_sweep_highres_fixtures as HF
import test_sweep_highres_gpu as HG
import test_sweep_refine_fixtures as F

pytestmark = pytest.mark.gpu

# every coarse kernel: generic forced, the default choice, the single-CTA kernel, the tiled kernel
KERNELS = [dict(force_generic_sweep=1, sweep_kernel=0), dict(force_generic_sweep=0, sweep_kernel=0),
           dict(force_generic_sweep=0, sweep_kernel=1), dict(force_generic_sweep=0, sweep_kernel=2)]


def check_kernel(options, grid, info):
    """the coarse kernel that ran is the one intended: the sequential matcher's grids (1 m window at 1 cm) only run on the generic
    kernel -- the YAML smear's raster is order dependent, and the tiled kernel's plan refuses the 2,500-row grid -- the loop
    matcher's 4 m / 5 cm grid on the one asked for"""
    if options["force_generic_sweep"]:
        assert info["kernel"] == "generic", (options, info)
    elif grid == H.GRID_SEQ_YAML:
        assert info["kernel"] == "generic" and info["refused_reason"] == 101, (options, info)
    elif grid == H.GRID_SEQ:
        assert info["kernel"] == "generic" and info["refused_reason"] > 101, (options, info)
    else:
        assert info["kernel"] == ("fast" if options["sweep_kernel"] == 1 else "tile"), (options, info)


class GpuScans:
    """Scans of any sizes and lasers as the C ABI's scan array (what MatchScanBatch / MatchScan read from a ScanBlock)"""

    def __init__(self, scans):
        self.scans = list(scans)
        self.c = (api.CScan * max(1, len(self.scans)))()
        for i, s in enumerate(self.scans):
            dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
            self.c[i] = api.CScan(len(s.ranges), dp(s.ranges), dp(s.points), (C.c_double * 3)(*s.pose))

    def __len__(self):
        return len(self.scans)


def expected(b: F.Batch, mapper, grid, pen, refine):
    """the oracle's MatchScan for every pair of the batch (repeated pairs computed once)"""
    pm, memo = H.port_matcher(mapper, grid), {}
    for q, c in b.pairs():
        if (q, c) not in memo:
            memo[(q, c)] = pm.match(b.queries[q], b.chain(c), pen, refine)
    rows = [memo[p] for p in b.pairs()]
    return np.array([r[0] for r in rows]), np.array([r[1] for r in rows]), np.array([r[2] for r in rows])


def run(gm, b: F.Batch, pen, refine, options=None):
    for k, v in (options or {}).items():
        gm.set_option(k, v)
    return gm.MatchScanBatch(GpuScans(b.queries), GpuScans(b.scans), b.chain_start, (b.pair_query, b.pair_chain), pen, refine)


def single(gm, b: F.Batch, q, c, pen, refine):
    base = b.chain(c)
    return gm.MatchScan(GpuScans([b.queries[q]]), GpuScans(base) if base else None, pen, refine)


def assert_rows(out, exp, names, what):
    for k, name in enumerate(names):
        assert out[0][k] == exp[0][k], (what, k, name, out[0][k], exp[0][k])
        assert np.array_equal(out[1][k], exp[1][k]) and np.array_equal(out[2][k], exp[2][k]), (what, k, name)
    assert np.array_equal(out[0], exp[0]) and np.array_equal(out[1], exp[1]) and np.array_equal(out[2], exp[2]), what


def assert_same(a, b, what):
    assert all(np.array_equal(x, y) for x, y in zip(a, b)), what


@pytest.mark.parametrize("grid", [H.GRID_SEQ, H.GRID_SEQ_YAML], ids=["karto_smear", "yaml_smear"])
def test_near_chain_batch_on_every_kernel(grid):
    """LinkNearChains' shape: three queries at distinct poses against chains of 10, 0, 3 and 1 scans, an explicit pair list out of
    order with a repeated pair; every row equals the oracle and the same pair's MatchScan, after every coarse kernel"""
    b = F.near_chain_batch()
    exp = expected(b, H.MAPPER_SEQ, grid, False, True)
    n_empty = sum(len(b.chain(c)) == 0 for _, c in b.pairs())
    gm = H.gpu_matcher(H.MAPPER_SEQ, grid)
    for o in KERNELS:
        out = run(gm, b, False, True, o)
        check_kernel(o, grid, gm.batch_info())
        assert_rows(out, exp, b.names, o)
        st = gm.batch_fetch_stats()
        assert (st["zero_pairs"], st["fallback_pairs"], st["pairs"]) == (n_empty, 0, len(b.pairs())), (o, st)
    for k, (q, c) in enumerate(b.pairs()):
        assert_same(single(gm, b, q, c, False, True), (out[0][k], out[1][k], out[2][k]), (q, c))


@pytest.mark.parametrize("expansion", [1, 0])
def test_fallbacks_mixed_into_one_refined_batch(expansion):
    """ordinary pairs around a fine-covariance-fallback pair, a tie-list overflow, zero responses with an empty and a non-empty
    raster and an empty chain: every row equals the oracle and the pair's MatchScan, and the fetch counts the closed-form and
    single-match pairs the fixtures predict"""
    mapper = F.MAPPER_EXP if expansion else F.MAPPER_NOEXP
    b = F.mixed_batch()
    zero, fallback = F.fetch_stats(F.branches(b, mapper, F.MIXED_GRID))
    assert fallback >= 3
    exp = expected(b, mapper, F.MIXED_GRID, False, True)
    gm = H.gpu_matcher(mapper, F.MIXED_GRID)
    for o in KERNELS[:2]:
        out = run(gm, b, False, True, o)
        check_kernel(o, F.MIXED_GRID, gm.batch_info())
        assert_rows(out, exp, b.names, o)
        st = gm.batch_fetch_stats()
        assert (st["zero_pairs"], st["fallback_pairs"]) == (zero, fallback), (o, st)
    for k, (q, c) in enumerate(b.pairs()):
        assert_same(single(gm, b, q, c, False, True), (out[0][k], out[1][k], out[2][k]), b.names[k])


def test_loop_closure_two_stage():
    """TryCloseLoop: a coarse batch on the loop matcher, then every query moved to its winner's coarse best pose and refined
    against that chain with the sequential matcher (Karto and YAML smear), against the oracle doing both stages; and the loop
    batch refined on every coarse kernel, the single-CTA kernel included"""
    b = F.loop_batch()
    gl = H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    coarse_exp = expected(b, H.MAPPER_LOOP, H.GRID_LOOP, False, False)
    refined_exp = expected(b, H.MAPPER_LOOP, H.GRID_LOOP, False, True)
    for o in KERNELS:
        for refine, exp in ((False, coarse_exp), (True, refined_exp)):
            out = run(gl, b, False, refine, o)
            check_kernel(o, H.GRID_LOOP, gl.batch_info())
            assert_rows(out, exp, b.names, (o, refine))
    fine = F.refine_stage(b, coarse_exp[0], coarse_exp[1])
    for grid in (H.GRID_SEQ, H.GRID_SEQ_YAML):
        exp = expected(fine, H.MAPPER_SEQ, grid, False, True)
        gs = H.gpu_matcher(H.MAPPER_SEQ, grid)
        for o in KERNELS:
            out = run(gs, fine, False, True, o)
            check_kernel(o, grid, gs.batch_info())
            assert_rows(out, exp, fine.names, (grid, o))


def test_handle_reuse_across_refined_batches():
    """one handle: a large refined batch, a small refined one (other candidate laser, a tie-list overflow), a single MatchScan, the
    large batch unrefined and refined again -- every result equals a fresh handle's, the first also the oracle's"""
    big = F.loop_batch()
    sw = synth.make_tie_sweep((25, 2), n_cands=1)
    small = F.batch([F.laser_scan(r, p, sw.query_laser) for r, p in zip(sw.query_ranges, sw.query_poses)],
                    [[F.laser_scan(r, p, sw.cand_laser) for r, p in zip(sw.cand_ranges, sw.cand_poses)]], [(0, 0), (1, 0)])
    mapper, grid = H.MAPPER_LOOP, H.GRID_LOOP
    steps = [("big", lambda g: run(g, big, False, True)), ("small", lambda g: run(g, small, False, True)),
             ("single", lambda g: single(g, big, 1, 2, True, True)), ("big_unrefined", lambda g: run(g, big, False, False)),
             ("big_again", lambda g: run(g, big, False, True))]
    gm = H.gpu_matcher(mapper, grid)
    results = {}
    for name, step in steps:
        results[name] = step(gm)
        if name == "small":
            assert gm.batch_fetch_stats()["fallback_pairs"] >= 1, gm.batch_fetch_stats()
        assert_same(results[name], step(H.gpu_matcher(mapper, grid)), name)
    assert_rows(results["big"], expected(big, mapper, grid, False, True), big.names, "big")
    assert_same(results["big"], results["big_again"], "big_again")


REFINE_CONFIGS = [c for c in HF.CONFIGS if c[0] in (2701, 3600) and c[1] != "yaml"]


@pytest.mark.parametrize("config", REFINE_CONFIGS, ids=HF.config_id)
def test_refined_highres_sweep_on_every_kernel(config):
    """0.1 deg lidars (2,701 and 3,600 readings) on the 4 m / 8 m windows, 12 m / 20 m ranges, 21 and 41 angles: refined, on the
    generic kernel in angle slices, the tiled kernel's plans and the single-CTA kernel where it fits"""
    n, g, na = config
    c = Case(HF.sweep(n), HF.MAPPERS[na], HF.GRIDS[g], pen=False, refine=True, volumes=False)
    gm = c.matcher()
    for o in HG.kernel_options(config):
        info, plan, st, fs, best = c.run(gm, o)
        HG.check_kernel(o, info, plan, na)
