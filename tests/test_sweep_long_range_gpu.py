"""The batched sweep at long laser ranges and wide search windows (synth.make_long_range_sweep): correlation grids of 1,165 to
6,085 cells, tiled plans of 4 to 167 row bands, the planner's refusals and the hand-over to the generic kernel.  Every result is
np.array_equal to the oracle (response, mean, covariance) and batch_best matches the oracle's integer volume; every plan the
device reports equals the restatement of tile_plan_rule.py at the device's SM count.  The configurations are those of
test_sweep_long_range_fixtures.py."""
from __future__ import annotations

import numpy as np
import pytest

from slam_toolbox_b200 import synth
from test_sweep_adversarial_gpu import Case, gpu_block, port_scans
import helpers as H
import test_sweep_long_range_fixtures as F
import tile_plan_rule as T

pytestmark = pytest.mark.gpu

GENERIC = dict(force_generic_sweep=1, sweep_kernel=0, sweep_cluster=0, sweep_chunks=0)
_CASES = {}


def tile(cluster=0, chunks=0):
    return dict(force_generic_sweep=0, sweep_kernel=2, sweep_cluster=cluster, sweep_chunks=chunks)


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def case(name, pen=False, refine=False, mapper=F.MAPPER):
    key = (name, pen, refine, tuple(sorted(mapper.items())))
    if key not in _CASES:
        _CASES[key] = Case(F.sweep(name), mapper, F.CONFIGS[name][0], pen=pen, refine=refine, volumes=not pen)
    return _CASES[key]


def check_plan(o, info, plan, name, pen, npairs):
    """the kernel that ran and its plan are the restatement's"""
    if o["force_generic_sweep"]:
        assert info["kernel"] == "generic" and info["refused_reason"] == 0, (o, info)
        return None
    want = T.plan(F.geometry(name), F.N_BEAMS, pen, npairs, sms(), o["sweep_cluster"], o["sweep_chunks"])
    if want.refused:
        assert info["kernel"] == "generic" and info["refused_reason"] == 100 + want.refused, (o, info, want)
        assert plan["refused_reason"] == want.refused and not plan["available"], (o, plan, want)
        return want
    got = (info["kernel"], plan["chunks"], plan["bands"], plan["band_rows"], plan["cluster"], plan["refused_reason"],
           plan["smem_kb"], plan["tail"])
    assert got == ("tile", want.chunks, want.bands, want.band_rows, want.cluster, 0, want.smem // 1024, want.tail), (o, got, want)
    return want


def options(na):
    """the generic kernel, the automatic plan (a 2-pair batch: 8-CTA clusters), clusters of 1, 2 and 8, one angle per chunk"""
    return [GENERIC, tile(), tile(1), tile(2), tile(8), tile(2, na)]


@pytest.mark.parametrize("pen", [False, True])
@pytest.mark.parametrize("name", F.NAMES)
def test_long_range_sweep_on_every_kernel(name, pen):
    c = case(name, pen)
    gm = c.matcher()
    grid, beyond, regimes = F.CONFIGS[name]
    for o in options(F.geometry(name).nA):
        info, plan, st, fs, best = c.run(gm, o)
        if not pen:
            c.check_best(best, o)
        want = check_plan(o, info, plan, name, pen, c.nq * c.nch)
        if beyond and want is not None and not want.refused:   # readings past the threshold: windows that leave the grid
            assert info["edge_beams"] > 0 and info["far_beams"] > 0, (o, info)
            assert st["wrap2_entries"] > 0, (o, st)
    # the one-CTA plan the device ran (checked above) is the regime the fixtures pin
    one = T.plan(F.geometry(name), F.N_BEAMS, pen, c.nq * c.nch, sms(), cluster=1)
    assert F.expected_regime(one) == regimes[pen], (name, pen, one)


def test_tie_sweep_above_24_ties_at_150m():
    """tie lists of 25 and 100 poses on a 167-band plan: the pairs fall back to the single-match path, exactly"""
    ks = (1, 24, 25, 100)
    grid = F.CONFIGS["4m-150m"][0]
    c = Case(synth.make_tie_sweep(ks, n_cands=1), F.MAPPER, grid)
    assert [b[2] for b in c.best] == list(ks)
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(1)):
        info, plan, st, fs, best = c.run(gm, o)
        c.check_best(best, o)
        assert fs["fallback_pairs"] == 2, (o, fs)
        if o["sweep_kernel"] == 2:
            assert info["kernel"] == "tile" and plan["bands"] > 100, (o, plan)


@pytest.mark.parametrize("name", ["8m-25m", "8m-80m"])
def test_refined_long_range_sweep(name):
    """doRefineMatch after a coarse pass on 5 and 95 bands"""
    c = case(name, pen=True, refine=True)
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(1)):
        info, plan, st, fs, best = c.run(gm, o)
        if name == "8m-80m" and o["sweep_kernel"] == 2:   # the penalised plan refuses: the generic kernel runs
            assert info["kernel"] == "generic" and info["refused_reason"] == 104, (o, info)


def test_penalised_sweep_at_the_code_default_minimum_distance_penalty():
    """minimum_distance_penalty 0.05 (slam_toolbox's code default; the YAML says 0.5) at 8 m / 40 m"""
    mapper = dict(F.MAPPER, minimum_distance_penalty=0.05)
    c = case("8m-40m", pen=True, mapper=mapper)
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(1)):
        info, plan, st, fs, best = c.run(gm, o)
        check_plan(o, info, plan, "8m-40m", True, c.nq * c.nch)


@pytest.mark.parametrize("name", ["8m-25m", "8m-100m"])
def test_response_expansion_on_non_overlapping_candidates(name):
    """use_response_expansion: every other candidate is 2 km away, so its coarse pass responds 0 and the reference widens the
    search three times; the sweep's closed form must equal it on the long-range grids too"""
    sw = F.sweep(name)
    cp = sw.cand_poses.copy()
    cp[::2, :2] += 2000.0
    sw = synth.AdversarialSweep(sw.query_ranges, sw.query_poses, sw.cand_ranges, cp, sw.chain_start, sw.query_laser, sw.cand_laser)
    c = Case(sw, dict(F.MAPPER, use_response_expansion=1), F.CONFIGS[name][0], volumes=False)
    assert c.r[0] == 0.0 and c.r[1] > 0.0, c.r
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(1)):
        info, plan, st, fs, best = c.run(gm, o)
        assert fs["zero_pairs"] == 1 and fs["fallback_pairs"] == 0, (o, fs)


@pytest.mark.parametrize("name", ["8m-25m", "8m-80m", "4m-150m"])
def test_single_match_at_long_range(name):
    """MatchScan (the single-match path) against the oracle with the candidates as its base scans, plain and penalised + refined"""
    grid = F.CONFIGS[name][0]
    sw = F.sweep(name)
    pm, gm = H.port_matcher(F.MAPPER, grid), H.gpu_matcher(F.MAPPER, grid)
    q = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)[0]
    cs = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
    gq, gc = gpu_block(sw.query_ranges, sw.query_poses, sw.query_laser), gpu_block(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
    for pen, ref in ((False, False), (True, True)):
        r, m, cv = gm.MatchScan(gq, gc, pen, ref)
        e = pm.match(q, cs, pen, ref)
        assert r == e[0] and np.array_equal(m, e[1]) and np.array_equal(cv, e[2]), (name, pen, ref, r, e[0])
        assert r > 0


def test_plan_smem_confirms_the_static_shared_memory():
    """the device's dynamic shared memory at the four shipped geometries equals the restatement's, whose budget subtracts
    sizeof(TileShared) = tile_plan_rule.TILE_SHARED_BYTES"""
    sw = synth.make_loop_sweep(5, n_queries=1, n_chains=2, chain_len=1)
    for window, rt in ((4.0, 12.0), (8.0, 12.0), (4.0, 20.0), (8.0, 20.0)):
        grid = (window, 0.05, 0.03, rt)
        gm = H.gpu_matcher(F.MAPPER, grid)
        gm.set_option("sweep_cluster", 1)
        gm.batch_upload(H.gpu_block(sw.query_ranges, sw.query_poses), H.gpu_block(sw.cand_ranges, sw.cand_poses), sw.chain_start)
        g = T.geometry(grid, F.MAPPER["coarse_search_angle_offset"], F.MAPPER["coarse_angle_resolution"])
        want = T.plan(g, F.N_BEAMS, False, 2, sms(), cluster=1)
        plan = gm.batch_tile_info()
        assert (plan["chunks"], plan["bands"], plan["band_rows"], plan["smem_kb"]) == \
            (want.chunks, want.bands, want.band_rows, want.smem // 1024), (grid, plan, want)
