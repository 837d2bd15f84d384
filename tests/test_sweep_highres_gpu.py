"""The batched sweep on high-resolution lidars and wide angle windows (synth.make_highres_sweep): coarse lookup tables larger
than the generic kernel's 200 KB of shared memory, which it reads in angle slices, and tiled-kernel plans at large n and nA.
Every result is np.array_equal to the oracle (response, mean, covariance) and batch_best matches the oracle's integer volume
(first arg-max index, its sum, the number of tied poses).  The configurations are those of test_sweep_highres_fixtures.py."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import api, synth
from test_sweep_adversarial_gpu import Case, gpu_block
import helpers as H
import test_sweep_highres_fixtures as F

pytestmark = pytest.mark.gpu

GENERIC = dict(force_generic_sweep=1, sweep_kernel=0, sweep_cluster=0, sweep_chunks=0)
_CASES = {}


def case(config, pen=False, refine=False, n_chains=2):
    """the oracle's answers for one configuration, computed once per module"""
    key = (config, pen, refine, n_chains)
    if key not in _CASES:
        n, g, na = config
        _CASES[key] = Case(F.sweep(n, n_chains), F.MAPPERS[na], F.GRIDS[g], pen=pen, refine=refine, volumes=not pen)
    return _CASES[key]


def tile(cluster=0, chunks=0):
    return dict(force_generic_sweep=0, sweep_kernel=2, sweep_cluster=cluster, sweep_chunks=chunks)


def kernel_options(config):
    """the generic kernel (angle slices), the tiled kernel with the automatic plan, clusters of 1 / 2 / 8 and forced chunk
    counts (one angle per chunk, and 5), and the single-CTA kernel where its accumulators fit (4 m / 12 m, 21 angles)"""
    na = config[2]
    opts = [GENERIC, tile(), tile(1), tile(2), tile(8), tile(2, na), tile(1, 5)]
    if config[1] == "4m12" and na == 21:
        opts.append(dict(force_generic_sweep=0, sweep_kernel=1, sweep_cluster=0, sweep_chunks=0))
    return opts


def check_kernel(o, info, plan, na):
    if o["force_generic_sweep"]:
        assert info["kernel"] == "generic", (o, info)
    elif o["sweep_kernel"] == 1:
        assert info["kernel"] == "fast", (o, info)
    else:
        assert info["kernel"] == "tile" and plan["available"] and plan["refused_reason"] == 0, (o, info, plan)
        if o["sweep_cluster"]:
            assert plan["cluster"] == o["sweep_cluster"], (o, plan)
        if o["sweep_chunks"]:
            assert plan["chunks"] >= min(o["sweep_chunks"], na), (o, plan)


SWEEPS = [c for c in F.CONFIGS if c[1] != "yaml"]


@pytest.mark.parametrize("config", SWEEPS, ids=F.config_id)
def test_highres_sweep_on_every_kernel(config):
    c = case(config)
    gm = c.matcher()
    for o in kernel_options(config):
        info, plan, st, fs, best = c.run(gm, o)
        check_kernel(o, info, plan, config[2])
        c.check_best(best, o)


PENALISED = [(2701, "4m12", 41), (3600, "8m12", 21), (3600, "4m20", 41), (1081, "4m12", 91)]


@pytest.mark.parametrize("config", PENALISED, ids=F.config_id)
def test_penalised_highres_sweep(config):
    c = case(config, pen=True)
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(8), tile(1, config[2])):
        info, plan, st, fs, best = c.run(gm, o)
        check_kernel(o, info, plan, config[2])


def test_refined_highres_sweep():
    config = (3600, "4m12", 41)
    c = case(config, pen=True, refine=True)
    gm = c.matcher()
    for o in (GENERIC, tile(), tile(2)):
        info, plan, st, fs, best = c.run(gm, o)
        check_kernel(o, info, plan, config[2])


def test_order_dependent_raster_in_angle_slices():
    """the shipped YAML smear makes the raster order dependent: only the generic kernel runs it, here in two slices"""
    c = case((2701, "yaml", 21))
    gm = c.matcher()
    for o in (dict(GENERIC, force_generic_sweep=0), GENERIC):
        info, plan, st, fs, best = c.run(gm, o)
        assert info["kernel"] == "generic" and plan["refused_reason"] == 1, (o, info, plan)
        c.check_best(best, o)


@pytest.mark.parametrize("pen", [False, True])
def test_winner_records_across_shards(pen):
    """6 candidates in 3 shards: every rank selects the same winner as one rank holding them all, and it is the oracle's best"""
    import torch
    from slam_toolbox_b200 import sweep
    config, n_cands, nranks = (3600, "4m20", 41), 6, 3
    c = case(config, pen=pen, n_chains=n_cands)
    sw = c.sw
    nb = api.ScanMatcher.winner_record_bytes()

    def records(lo, hi):
        gm = c.matcher()
        gc = gpu_block(sw.cand_ranges[lo:hi], sw.cand_poses[lo:hi], sw.cand_laser)
        gm.batch_upload(c.gq, gc, np.arange(hi - lo + 1, dtype=np.int32), None, pen)
        gm.batch_run()
        b = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        gm.batch_winner_records(b.data_ptr(), lo)
        torch.cuda.synchronize()
        return gm, gc, b

    whole = records(0, n_cands)
    one = whole[0].batch_winners_select(whole[2].data_ptr(), 1, 1)
    shards = [records(*sweep.shard_range(n_cands, nranks, r)) for r in range(nranks)]
    gathered = torch.cat([s[2] for s in shards])
    j = int(np.argmax(c.r))
    assert one[0][0] == j and one[1][0] == c.r[j] and np.array_equal(one[2][0], c.m[j]) and np.array_equal(one[3][0], c.c[j])
    for gm, _, _ in shards:
        ids, r, m, cv = gm.batch_winners_select(gathered.data_ptr(), nranks, 1)
        assert ids[0] == one[0][0] and r[0] == one[1][0] and np.array_equal(m, one[2]) and np.array_equal(cv, one[3])


def _laser_block(ranges, pose, laser):
    return api.ScanBlock(ranges, pose, api.LaserRangeFinder(minimum_angle=laser[0], angular_resolution=laser[1]))


def _one_pair(n_query, n_cand):
    """a room-scan query of n_query readings and one candidate of n_cand readings (full circle), same world and poses"""
    sw = synth.make_highres_sweep(1081, 270.0, n_chains=1)
    world = synth.make_world(11)   # make_highres_sweep's default world
    out = []
    for n, pose in ((n_query, sw.query_poses), (n_cand, sw.cand_poses)):
        laser = synth.highres_laser(n, 360.0)
        r = synth.raycast(world, pose, n_beams=n, angle_min=laser[0], angle_inc=laser[1])
        out.append((r, pose, laser))
    return out


def test_lookup_row_and_find_valid_bounds():
    """the two refusals left: a query whose single lookup row exceeds the shared memory (more than 51,200 readings, at upload) and a
    candidate scan above the shared-memory staging of FindValidPoints (more than 12,044 readings, at run); both boundaries
    themselves are accepted and exact (on the small 0.5 m search: the generic kernel runs a 51,200-beam pair on one CTA)"""
    mapper, grid = F.MAPPER, H.GRID_SMALL
    for nq, nc, refused in ((51201, 1081, "lookup row"), (1081, 12045, "FindValidPoints"), (51200, 1081, None), (1081, 12044, None)):
        (qr, qp, ql), (cr, cp, cl) = _one_pair(nq, nc)
        gm = H.gpu_matcher(mapper, grid)
        gq, gc = _laser_block(qr, qp, ql), _laser_block(cr, cp, cl)
        cs = np.array([0, 1], dtype=np.int32)
        if refused:
            with pytest.raises(api.B200Error) as e:
                gm.MatchScanBatch(gq, gc, cs, None, False, False)
            assert e.value.code == api.ERR_UNSUPPORTED and refused in str(e.value), (nq, nc, str(e.value))
            continue
        pm = H.port_matcher(mapper, grid)
        er, em, ec = pm.match(P.PortScan(qr[0], qp[0], *ql), [P.PortScan(cr[0], cp[0], *cl)], False, False)
        for o in (GENERIC, dict(GENERIC, force_generic_sweep=0)):
            for k, v in o.items():
                gm.set_option(k, v)
            r, m, c = gm.MatchScanBatch(gq, gc, cs, None, False, False)
            assert r[0] == er and np.array_equal(m[0], em) and np.array_equal(c[0], ec), (nq, nc, o, gm.batch_info())
