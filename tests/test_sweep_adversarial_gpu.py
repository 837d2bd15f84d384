"""The batched sweep kernels on inputs the room-scan fixtures never produce (synth.make_dense_sweep, make_tie_sweep,
make_long_query_sweep): hundreds of beams in one grid cell (descriptor groups longer than one 16-bit flush, large multiplicities,
EDGE groups, sub-blocks), tied best poses around the 24-entry tie list, and queries on both sides of the integer tie rule.
Every result is bit-exact against the oracle, and batch_best against the oracle's integer volume."""
from __future__ import annotations

import math

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import api, synth
import helpers as H

pytestmark = pytest.mark.gpu

MAPPER = dict(H.MAPPER_LOOP, use_response_expansion=0)
MAPPER_NARROW = dict(MAPPER, coarse_search_angle_offset=math.radians(2.0))
GRID_DIM8 = (8.0, 0.05, 0.03, 12.0)
GRID_RT20 = (4.0, 0.05, 0.03, 20.0)
GRID_SMEAR5 = (4.0, 0.05, 0.05, 12.0)
MAX_TIES = 24
TOL = 1e-6


def port_scans(ranges, poses, laser):
    return [P.PortScan(r, p, laser[0], laser[1]) for r, p in zip(np.atleast_2d(ranges), np.atleast_2d(poses))]


def gpu_block(ranges, poses, laser):
    return api.ScanBlock(ranges, poses, api.LaserRangeFinder(minimum_angle=laser[0], angular_resolution=laser[1]))


class Case:
    """one adversarial sweep with the oracle's answers: per pair (query-major) the MatchScan result and, from the coarse
    volume, the first tied pose's flat index (y * nX + x) * nA + a and integer sum, and the number of poses whose response
    DoubleEquals the best (below 9000 beams: the poses with the best sum)"""

    def __init__(self, sw, mapper, grid, pen=False, refine=False, volumes=True):
        self.sw, self.mapper, self.grid = sw, mapper, grid
        self.nq, self.nch = len(sw.query_ranges), len(sw.chain_start) - 1
        pm = H.port_matcher(mapper, grid)
        qs = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)
        cs = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        self.bases = [cs[sw.chain_start[c]:sw.chain_start[c + 1]] for c in range(self.nch)]
        exp = [pm.match(qs[q], self.bases[c], pen, refine) for q in range(self.nq) for c in range(self.nch)]
        self.r = np.array([e[0] for e in exp])
        self.m = np.array([e[1] for e in exp])
        self.c = np.array([e[2] for e in exp])
        self.best = []
        if volumes:
            off, res = H.coarse_search(grid)
            n = sw.query_ranges.shape[1]
            for q in range(self.nq):
                for c in range(self.nch):
                    pm.raster(qs[q], self.bases[c])
                    vol = pm.correlate(qs[q], qs[q].pose, off, res, mapper["coarse_search_angle_offset"],
                                       mapper["coarse_angle_resolution"], False, False)[3].ravel()
                    resp = vol / float(n * 100)
                    d = resp - resp.max()
                    tie = (d >= -TOL) & (d <= TOL)       # DoubleEqual(response, best), M.cpp:807
                    first = int(np.argmax(tie))
                    self.best.append((int(vol[first]), first, int(tie.sum())))
        self.gq = gpu_block(sw.query_ranges, sw.query_poses, sw.query_laser)
        self.gc = gpu_block(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        self.pen, self.refine = pen, refine

    def matcher(self):
        return H.gpu_matcher(self.mapper, self.grid)

    def run(self, gm, options):
        for k, v in options.items():
            gm.set_option(k, v)
        out = gm.MatchScanBatch(self.gq, self.gc, self.sw.chain_start, None, self.pen, self.refine)
        what = (options, gm.batch_info(), gm.batch_tile_info())
        assert np.array_equal(out[0], self.r), what
        assert np.array_equal(out[1], self.m) and np.array_equal(out[2], self.c), what
        return gm.batch_info(), gm.batch_tile_info(), gm.batch_tile_stats(), gm.batch_fetch_stats(), gm.batch_best()

    def check_best(self, best, what, allow_ambiguous=False):
        for p, (s, i, t) in enumerate(zip(*best)):
            es, ei, et = self.best[p]
            if allow_ambiguous and t == -1:   # FP64 path: a chunk best within the tie tolerance -> single-match path
                continue
            assert (s, i, t) == (es, ei, et), (p, what, (s, i, t), self.best[p])


def kernel_options(grid, clusters=(1, 2, 4, 8), chunks=(0, 5, 21), dedup=(0, 1)):
    """generic, single-CTA (4 m / 12 m only) and tiled kernel configurations"""
    opts = [dict(force_generic_sweep=1)]
    if grid == H.GRID_LOOP:
        opts += [dict(force_generic_sweep=0, sweep_kernel=1, no_beam_dedup=d) for d in dedup]
    opts += [dict(force_generic_sweep=0, sweep_kernel=2, sweep_cluster=cl, sweep_chunks=ch, no_beam_dedup=d)
             for cl in clusters for ch in chunks for d in dedup]
    return opts


DENSE = [((639,), False), ((640,), False), ((641,), False), ((1280,), False), ((1281, 639), False), ((1920,), False),
         ((1281,), True)]


@pytest.mark.parametrize("clusters,edge", DENSE)
def test_dense_groups_on_every_kernel(clusters, edge):
    """hundreds of beams in one cell: group splitting, multiplicities up to 640, dedup switched off above 640, EDGE groups
    above 640 (the separate EDGE flush loop), descriptor sub-blocks"""
    sw = synth.make_dense_sweep(clusters, edge=edge)
    big = max(clusters)
    grids = [H.GRID_LOOP, GRID_DIM8] + ([GRID_RT20] if clusters == (1281, 639) else [])
    for grid in grids:
        case = Case(sw, MAPPER, grid)
        gm = case.matcher()
        if grid == GRID_DIM8:   # 8 m: fewer configurations (the oracle's volume is 4x larger)
            opts = kernel_options(grid, clusters=(1, 4), chunks=(0, 21))
        else:
            opts = kernel_options(grid)
        seen = dict(split=0, mult=0, sub=0, edge=0, bands=0, plain=0)
        for o in opts:
            info, plan, st, fs, best = case.run(gm, o)
            case.check_best(best, o)
            if o.get("sweep_kernel") == 2:
                assert info["kernel"] == "tile" and info["refused_reason"] == 0 and plan["available"], (o, info, plan)
                if o["sweep_cluster"]:
                    assert plan["cluster"] == o["sweep_cluster"], plan
                assert st["max_plain_group"] <= big
                if o["no_beam_dedup"] or len(clusters) == 1 and big > 640:
                    assert st["max_multiplicity"] <= 1, (o, st)     # only the odd-length fix-up entries
                seen["split"] = max(seen["split"], st["split_groups"])
                seen["mult"] = max(seen["mult"], st["max_multiplicity"])
                seen["sub"] = max(seen["sub"], st["sub_blocks"])
                seen["edge"] = max(seen["edge"], st["max_edge_group"])
                seen["bands"] = max(seen["bands"], plan["bands"])
                seen["plain"] = max(seen["plain"], st["max_plain_group"])
            elif o.get("sweep_kernel") == 1:
                assert info["kernel"] == "fast", info
        if big > 641 and not edge:
            assert seen["split"] > 0, seen
        if big == 641:   # dedup is off and the odd-length fix moves one beam to the multi list: 640 plain beams, one item
            assert seen["split"] == 0 and seen["plain"] == 640 and seen["mult"] == 1, seen
        if big == 640:
            assert seen["mult"] == 640, seen
        if big >= 1280 and not edge and grid == H.GRID_LOOP:   # 5 angles of 1280 beams do not fit one staging buffer
            assert seen["sub"] > 0, seen
        if edge:
            assert seen["edge"] > 640, seen
        if grid == GRID_RT20:
            assert seen["bands"] > 1, seen
    # single match (k_correlate / k_correlate_few) on the same inputs
    for grid in (H.GRID_LOOP,):
        pm, gm = H.port_matcher(MAPPER, grid), H.gpu_matcher(MAPPER, grid)
        qs = port_scans(sw.query_ranges, sw.query_poses, sw.query_laser)
        cs = port_scans(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        gq, gc = gpu_block(sw.query_ranges, sw.query_poses, sw.query_laser), gpu_block(sw.cand_ranges, sw.cand_poses, sw.cand_laser)
        for pen, ref in ((False, False), (True, True)):
            r, m, c = gm.MatchScan(gq, gc, pen, ref)
            e = pm.match(qs[0], cs, pen, ref)
            assert r == e[0] and np.array_equal(m, e[1]) and np.array_equal(c, e[2]), (pen, ref)


def test_one_angle_stage_fits_a_split_group():
    """8 m window, one angle per chunk, a 1920-beam query whose beams land in one group: the staging buffer must hold the
    group's three pieces of item records on top of its payload, or the planner refuses the tiled kernel"""
    sw = synth.make_dense_sweep((1920,))
    case = Case(sw, MAPPER, GRID_DIM8)
    gm = case.matcher()
    for cluster in (1, 2):
        info, plan, st, fs, best = case.run(gm, dict(sweep_kernel=2, sweep_cluster=cluster, sweep_chunks=21))
        assert info["kernel"] == "tile" and plan["refused_reason"] == 0 and plan["chunks"] == 21, (info, plan)
        assert st["split_groups"] > 0 and st["max_plain_group"] == 1920, st
        case.check_best(best, cluster)


@pytest.mark.parametrize("pen,refine", [(False, False), (True, False), (False, True), (True, True)])
def test_tie_counts_on_every_kernel(pen, refine):
    """1, 2, 23, 24, 25 and 100 tied best poses spread over the angle chunks: tie lists merged across chunks and cluster
    ranks in array order, the fall back above 24 ties"""
    ks = (1, 2, 23, 24, 25, 100)
    sw = synth.make_tie_sweep(ks, n_cands=2)
    case = Case(sw, MAPPER, H.GRID_LOOP, pen=pen, refine=refine, volumes=not pen)
    if not pen:
        assert [b[2] for b in case.best] == [k for k in ks for _ in range(2)]
    gm = case.matcher()
    opts = kernel_options(H.GRID_LOOP, chunks=(0, 21), dedup=(0,)) if not refine else \
        kernel_options(H.GRID_LOOP, clusters=(1, 4), chunks=(0,), dedup=(0,))
    for o in opts:
        info, plan, st, fs, best = case.run(gm, o)
        if not pen:
            case.check_best(best, o)
            if not refine:
                assert fs["fallback_pairs"] == sum(1 for b in case.best if b[2] > MAX_TIES), (o, fs)
    for q, k in enumerate(ks):   # single match
        r, m, c = gm.MatchScan(case.gq, case.gc, pen, refine, scan_index=q)
        e = P.PortScan(sw.query_ranges[q], sw.query_poses[q], *sw.query_laser)
        er, em, ec = H.port_matcher(MAPPER, H.GRID_LOOP).match(e, case.bases[0] + case.bases[1], pen, refine)
        assert r == er and np.array_equal(m, em) and np.array_equal(c, ec), k


@pytest.mark.parametrize("pen", [False, True])
def test_winner_exchange_with_tied_candidates(pen):
    """identical candidates in different shards: every candidate scores the same, the winner is the lowest global id; a
    winner with more than 24 ties cannot be finished from its record (UNSUPPORTED), its owner's fetched row is still exact"""
    import torch
    from slam_toolbox_b200 import sweep
    n_cands, nranks = 6, 3
    nb = api.ScanMatcher.winner_record_bytes()
    for ks, overflow in (((1, 24), False), ((25,), True)):
        if pen and overflow:   # penalties break the ties
            continue
        sw = synth.make_tie_sweep(ks, n_cands=n_cands)
        case = Case(sw, MAPPER, H.GRID_LOOP, pen=pen, volumes=False)
        gq = case.gq
        bufs, handles, rows = [], [], []
        for r in range(nranks):
            lo, hi = sweep.shard_range(n_cands, nranks, r)
            gm = H.gpu_matcher(MAPPER, H.GRID_LOOP)
            gc = gpu_block(sw.cand_ranges[lo:hi], sw.cand_poses[lo:hi], sw.cand_laser)
            cs = np.arange(hi - lo + 1, dtype=np.int32)
            rows.append(gm.MatchScanBatch(gq, gc, cs, None, pen, False))
            gm.batch_upload(gq, gc, cs, None, pen)
            gm.batch_run()
            b = torch.zeros(len(ks) * nb, dtype=torch.uint8, device="cuda")
            gm.batch_winner_records(b.data_ptr(), lo)
            torch.cuda.synchronize()
            bufs.append(b); handles.append((gm, gc))
        gathered = torch.cat(bufs)
        # the owner of candidate 0 (rank 0) fetches its own rows: bit-exact for every query, overflow or not
        r0, m0, c0 = rows[0]
        nloc = sweep.shard_range(n_cands, nranks, 0)[1]
        for q in range(len(ks)):
            j = q * n_cands
            assert r0[q * nloc] == case.r[j] and np.array_equal(m0[q * nloc], case.m[j]) and np.array_equal(c0[q * nloc], case.c[j])
        for gm, _ in handles:
            if overflow:
                with pytest.raises(api.B200Error) as e:
                    gm.batch_winners_select(gathered.data_ptr(), nranks, len(ks))
                assert e.value.code == api.ERR_UNSUPPORTED
            else:
                ids, r, m, c = gm.batch_winners_select(gathered.data_ptr(), nranks, len(ks))
                for q in range(len(ks)):
                    j = q * n_cands
                    assert ids[q] == 0 and r[q] == case.r[j] and np.array_equal(m[q], case.m[j]) and np.array_equal(c[q], case.c[j])


@pytest.mark.parametrize("n", [8990, 10240])
def test_integer_and_fp64_tie_rules_at_the_boundary(n):
    """n = 8990 beams: the integer tie rule (sum equality).  n = 10240: FP64 responses, and the best two sums of chain 1 differ
    by 1, which the reference counts as two ties (DoubleEqual)"""
    sw = synth.make_long_query_sweep(n)
    case = Case(sw, MAPPER_NARROW, GRID_SMEAR5)
    if n == 10240:
        assert case.best[1][2] == 2, case.best
    gm = case.matcher()
    for o in [dict(force_generic_sweep=1)] + [dict(force_generic_sweep=0, sweep_kernel=2, sweep_cluster=cl, sweep_chunks=ch)
                                             for cl in (1, 2) for ch in (0, 3)]:
        info, plan, st, fs, best = case.run(gm, o)
        if o.get("sweep_kernel") == 2:
            assert info["kernel"] == "tile", (o, info)
        case.check_best(best, o, allow_ambiguous=n >= 9000)
