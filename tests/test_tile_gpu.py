"""The tiled cluster sweep kernel (csrc/sm_tile.cu) on the reference's shipped loop-closure geometries:
loop_search_space_dimension 8 m (config/mapper_params_online_sync.yaml:61, Mapper.cpp:2231 -> 81 x 81 x 21 poses),
max_laser_range 20 m (:32 -> 885..965-cell correlation grids), and BASELINE's 4 m / 12 m -- every cluster size and several
chunkings, bit-exact against the oracle (C restatement pinned to the reference) and against the generic kernel."""
from __future__ import annotations

import numpy as np
import pytest

from slam_toolbox_b200 import synth
import helpers as H

pytestmark = pytest.mark.gpu

GRID_DIM8 = (8.0, 0.05, 0.03, 12.0)
GRID_RT20 = (4.0, 0.05, 0.03, 20.0)
GRID_DIM8_RT20 = (8.0, 0.05, 0.03, 20.0)


def _expected(pm, sw, nq, nch, pen=False):
    pc, pq = H.port_scans(sw.cand_ranges, sw.cand_poses), H.port_scans(sw.query_ranges, sw.query_poses)
    exp = [pm.match(pq[q], pc[sw.chain_start[c]:sw.chain_start[c + 1]], pen, False) for q in range(nq) for c in range(nch)]
    return np.array([e[0] for e in exp]), np.array([e[1] for e in exp]), np.array([e[2] for e in exp])


def _run(gm, gq, gc, sw, pen=False):
    r, m, c = gm.MatchScanBatch(gq, gc, sw.chain_start, None, pen, False)
    return r, m, c, gm.batch_best()


@pytest.mark.parametrize("grid,seed", [(H.GRID_LOOP, 31), (GRID_DIM8, 32), (GRID_RT20, 33), (GRID_DIM8_RT20, 34),
                                       ((4.0, 0.05, 0.03, 6.0), 35), ((2.0, 0.05, 0.05, 8.0), 36)])
def test_tile_kernel_every_cluster_size_vs_oracle(grid, seed):
    nq, nch = 2, 6
    sw = synth.make_loop_sweep(seed, n_queries=nq, n_chains=nch, chain_len=2, inf_frac=0.02)
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
    er, em, ec = _expected(pm, sw, nq, nch)
    gm.set_option("force_generic_sweep", 1)
    gen = _run(gm, gq, gc, sw)
    gm.set_option("force_generic_sweep", 0)
    assert np.array_equal(gen[0], er) and np.array_equal(gen[1], em) and np.array_equal(gen[2], ec)
    gm.set_option("sweep_kernel", 2)
    plans = set()
    for cluster, chunks in ((1, 0), (2, 0), (4, 0), (8, 0), (1, 21), (2, 5), (4, 11), (0, 0)):
        gm.set_option("sweep_cluster", cluster)
        gm.set_option("sweep_chunks", chunks)
        out = _run(gm, gq, gc, sw)
        info, plan = gm.batch_info(), gm.batch_tile_info()
        assert info["kernel"] == "tile" and plan["available"], (info, plan)
        if cluster:
            assert plan["cluster"] == cluster, plan
        plans.add((plan["cluster"], plan["chunks"], plan["bands"]))
        assert np.array_equal(out[0], er), (plan, out[0], er)
        assert np.array_equal(out[1], em) and np.array_equal(out[2], ec), plan
        for a, b in zip(out[3], gen[3]):     # best integer sum, arg-max pose index, tie count
            assert np.array_equal(a, b), plan
    assert len(plans) >= 4, plans
    if grid[3] < 12.0:
        assert gm.batch_info()["edge_beams"] > 0


def test_tile_kernel_with_penalties_and_single_scans():
    """FP64 response path (doPenalize) of the distributed reduction: chunk bests within the tie tolerance fall back, everything
    else is reduced on the device; chain length 1."""
    nq, nch = 2, 8
    sw = synth.make_loop_sweep(41, n_queries=nq, n_chains=nch, chain_len=1)
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    pm, gm = H.port_matcher(mapper, GRID_DIM8), H.gpu_matcher(mapper, GRID_DIM8)
    gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
    er, em, ec = _expected(pm, sw, nq, nch, pen=True)
    gm.set_option("sweep_kernel", 2)
    for cluster in (1, 4):
        gm.set_option("sweep_cluster", cluster)
        r, m, c, _ = _run(gm, gq, gc, sw, pen=True)
        assert np.array_equal(r, er) and np.array_equal(m, em) and np.array_equal(c, ec)


@pytest.mark.parametrize("expansion", [0, 1])
@pytest.mark.parametrize("grid", [H.GRID_LOOP, GRID_DIM8])
def test_non_overlapping_candidates_use_the_closed_form(grid, expansion):
    """A candidate that does not overlap the query's search window: every pose ties at response 0 and the reference averages
    ALL poses (Mapper.cpp:802-829).  No per-pair fall back: the closed form is evaluated once per query."""
    nq, nch = 2, 10
    sw = synth.make_loop_sweep(51, n_queries=nq, n_chains=nch, chain_len=1)
    cand_poses = sw.cand_poses.copy()
    cand_poses[::2, :2] += 300.0            # every other candidate is nowhere near the query
    # with use_response_expansion (the toolbox default) the reference runs three more, wider passes on a zero response
    # (Mapper.cpp:594-619); an empty raster makes them zero as well: closed form of the widest pass
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=expansion)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    pc, pq = H.port_scans(sw.cand_ranges, cand_poses), H.port_scans(sw.query_ranges, sw.query_poses)
    gc, gq = H.gpu_block(sw.cand_ranges, cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
    exp = [pm.match(pq[q], pc[c:c + 1], False, False) for q in range(nq) for c in range(nch)]
    for kernel in (0, 2):
        gm.set_option("sweep_kernel", kernel)
        r, m, c = gm.MatchScanBatch(gq, gc, sw.chain_start, None, False, False)
        st = gm.batch_fetch_stats()
        n_zero = sum(1 for e in exp if e[0] == 0.0)
        assert n_zero >= nq * nch // 2 and st["zero_pairs"] == n_zero and st["fallback_pairs"] == 0, (st, n_zero)
        assert np.array_equal(r, np.array([e[0] for e in exp]))
        assert np.array_equal(m, np.array([e[1] for e in exp])) and np.array_equal(c, np.array([e[2] for e in exp]))
    assert (r[::2] == 0).all() and (r[1::2] > 0).any()


@pytest.mark.parametrize("pen", [False, True])
def test_winner_records_one_gather_equals_the_unsharded_sweep(pen):
    """The multi-GPU exchange behind the C ABI (SURVEY.md 8e): per-rank winner records built on the device, ONE all-gather (here:
    torch.cat of three shards' buffers, rank-major like all_gather_into_tensor), local selection.  Every "rank" must end with the
    unsharded sweep's per-query best (highest response, lowest global id) -- also for a penalised sweep, where the integer-sum key of
    b200sm_batch_reduce_keys is not the response order (and is refused)."""
    import torch
    from slam_toolbox_b200 import api, sweep
    Q, Cn = 3, 24
    sw = synth.make_loop_sweep(61, n_queries=Q, n_chains=Cn, chain_len=1)
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    gq = H.gpu_block(sw.query_ranges, sw.query_poses)
    full = H.gpu_matcher(mapper, H.GRID_LOOP)
    resp, mean, cov = full.MatchScanBatch(gq, H.gpu_block(sw.cand_ranges, sw.cand_poses), sw.chain_start, None, pen, False)
    resp, mean, cov = resp.reshape(Q, Cn), mean.reshape(Q, Cn, 3), cov.reshape(Q, Cn, 3, 3)
    nb = api.ScanMatcher.winner_record_bytes()
    bufs, handles = [], []
    for r in range(3):
        lo, hi = sweep.shard_range(Cn, 3, r)
        gm = H.gpu_matcher(mapper, H.GRID_LOOP)
        gm.batch_upload(gq, H.gpu_block(sw.cand_ranges[lo:hi], sw.cand_poses[lo:hi]), np.arange(hi - lo + 1, dtype=np.int32), None, pen)
        gm.batch_run()
        b = torch.zeros(Q * nb, dtype=torch.uint8, device="cuda")
        gm.batch_winner_records(b.data_ptr(), lo)
        torch.cuda.synchronize()
        bufs.append(b); handles.append(gm)
        if pen:
            with pytest.raises(api.B200Error):
                gm.batch_reduce_keys(torch.zeros(Q, dtype=torch.int64, device="cuda").data_ptr(), lo)
    gathered = torch.cat(bufs)
    for gm in handles:
        ids, r, m, c = gm.batch_winners_select(gathered.data_ptr(), 3, Q)
        for q in range(Q):
            j = int(np.argmax(resp[q]))                 # first maximum = lowest id among equal responses
            assert ids[q] == j and r[q] == resp[q, j] and np.array_equal(m[q], mean[q, j]) and np.array_equal(c[q], cov[q, j])


def test_empty_chains_and_ragged_chain_lengths():
    """Ragged input: chains of 0, 1 and 3 scans in one sweep (an empty chain gives the all-poses-tie result: nothing is rasterised),
    on the generic kernel, the tiled kernel with one CTA per pair and with 4-CTA clusters."""
    sw = synth.make_loop_sweep(71, n_queries=2, n_chains=6, chain_len=1)
    chain_start = np.array([0, 0, 1, 4, 4, 5, 6, 6], dtype=np.int32)     # chains: [], [0], [1, 2, 3], [], [4], [5], []
    nch = len(chain_start) - 1
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    for grid in (H.GRID_LOOP, GRID_DIM8):
        pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
        pc, pq = H.port_scans(sw.cand_ranges, sw.cand_poses), H.port_scans(sw.query_ranges, sw.query_poses)
        gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
        exp = [pm.match(pq[q], pc[chain_start[c]:chain_start[c + 1]], False, False) for q in range(2) for c in range(nch)]
        for opts in ({"force_generic_sweep": 1}, {"sweep_kernel": 2, "sweep_cluster": 1}, {"sweep_kernel": 2, "sweep_cluster": 4}):
            gm.set_option("force_generic_sweep", 0)
            for k, v in opts.items():
                gm.set_option(k, v)
            r, m, c = gm.MatchScanBatch(gq, gc, chain_start, None, False, False)
            assert np.array_equal(r, np.array([e[0] for e in exp])), opts
            assert np.array_equal(m, np.array([e[1] for e in exp])) and np.array_equal(c, np.array([e[2] for e in exp])), opts
        assert r[0] == 0.0 and r[3] == 0.0 and r[6] == 0.0 and r[2] > 0


def test_other_search_windows_and_angle_resolutions():
    """Geometries away from the shipped ones: 41 angles (1 degree steps), a 3 m window at a 10 m range threshold (run-time row pitch
    instantiation), a 0.1 m grid, and a 5 x 5 smear kernel with six distinct values (CAS raster) -- auto plan and 2-CTA clusters.
    Wide smear kernels at 0.05 m cells: 15 x 15 taps (sigma 0.18 m, the last kernel held in TileShared::kern), 17 x 17 (0.19 m,
    read from global memory) and 41 x 41 (0.499 m, the widest order-independent kernel); at sigma 0.4995 m the taps next to the
    centre round to 100, the raster is order dependent and the sweep runs on the generic kernel (refusal 100 + 1)."""
    import math
    loop = dict(H.MAPPER_LOOP, use_response_expansion=0)
    cases = [   # (mapper, grid, smear kernel size or None, refusal of the tiled planner)
        (dict(H.MAPPER_LOOP, coarse_angle_resolution=math.radians(1.0), use_response_expansion=0), (3.0, 0.05, 0.03, 10.0), None, 0),
        (dict(H.MAPPER_LOOP, coarse_search_angle_offset=math.radians(10.0), use_response_expansion=0), (6.0, 0.1, 0.1, 15.0), None, 0),
        (loop, (5.0, 0.05, 0.05, 14.0), None, 0),
        (loop, H.GRID_SMALL, None, 0),                      # 6 x 6 poses: tiny accumulators
        (loop, (0.5, 0.05, 0.03, 20.0), None, 0),           # ... behind a wide row pitch
        (loop, (4.0, 0.05, 0.18, 12.0), 15, 0),
        (loop, (4.0, 0.05, 0.19, 12.0), 17, 0),
        (loop, (4.0, 0.05, 0.499, 12.0), 41, 0),
        (loop, (4.0, 0.05, 0.4995, 12.0), 41, 1),
    ]
    sw = synth.make_loop_sweep(81, n_queries=1, n_chains=5, chain_len=2, inf_frac=0.02)
    for mapper, grid, ksize, refusal in cases:
        pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
        if ksize:
            assert pm.grid()["kernel_size"] == ksize, grid
        gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
        er, em, ec = _expected(pm, sw, 1, 5)
        for cluster in (0, 1, 2):
            gm.set_option("sweep_cluster", cluster)
            r, m, c, _ = _run(gm, gq, gc, sw)
            info, plan = gm.batch_info(), gm.batch_tile_info()
            if refusal:
                assert info["kernel"] == "generic" and info["refused_reason"] == 100 + refusal, (grid, info)
                assert plan["refused_reason"] == refusal, (grid, plan)
            else:
                assert info["kernel"] == "tile", (grid, info)
            assert np.array_equal(r, er) and np.array_equal(m, em) and np.array_equal(c, ec), (grid, cluster, plan)


def test_plan_readouts_describe_the_last_upload():
    """One handle, four uploads: tiled kernel, forced generic kernel, single-CTA kernel, tiled kernel again.  The readouts of the
    kernel choice (batch_info, batch_tile_info, batch_tile_stats) describe the last upload only: the forced generic kernel refused
    nothing and classified no beams, the single-CTA upload has no tiled plan, and the second tiled upload reads like the first.
    Every upload runs on its own kernel to the same results.  An order-dependent raster refuses both parity kernels: the generic
    kernel runs with reason 100 + the tiled planner's refusal code 1."""
    nq, nch = 2, 6
    sw = synth.make_loop_sweep(91, n_queries=nq, n_chains=nch, chain_len=2, inf_frac=0.02)
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    gm = H.gpu_matcher(mapper, H.GRID_LOOP)
    gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)

    def upload(**opts):
        for k, v in opts.items():
            gm.set_option(k, v)
        gm.batch_upload(gq, gc, sw.chain_start, None, False)
        gm.batch_run()
        return (gm.batch_info(), gm.batch_tile_info(), gm.batch_tile_stats()), gm.batch_fetch()

    tile, out = upload(force_generic_sweep=0, sweep_kernel=2)
    info, plan, stats = tile
    assert info["kernel"] == "tile" and plan["available"] and stats["blocks"] > 0 and info["fast_descriptors"] > 0, tile
    results = [out]

    (info, plan, stats), out = upload(force_generic_sweep=1)
    assert info["kernel"] == "generic" and info["refused_reason"] == 0, info
    assert info["fast_descriptors"] == info["edge_beams"] == info["far_beams"] == 0, info
    assert not any(plan.values()) and not any(stats.values()), (plan, stats)
    results.append(out)

    (info, plan, stats), out = upload(force_generic_sweep=0, sweep_kernel=1)
    assert info["kernel"] == "fast" and info["refused_reason"] == 0 and info["fast_descriptors"] > 0, info
    assert not any(plan.values()) and not any(stats.values()), (plan, stats)
    results.append(out)

    again, out = upload(sweep_kernel=2)
    assert again == tile, (again, tile)
    results.append(out)
    for r in results[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(r, results[0]))

    seq = synth.make_loop_sweep(92, n_queries=1, n_chains=2, chain_len=1)
    gs = H.gpu_matcher(H.MAPPER_SEQ, H.GRID_SEQ_YAML)
    gs.batch_upload(H.gpu_block(seq.query_ranges, seq.query_poses), H.gpu_block(seq.cand_ranges, seq.cand_poses), seq.chain_start)
    info, plan = gs.batch_info(), gs.batch_tile_info()
    assert info["kernel"] == "generic" and info["refused_reason"] == 101 and plan["refused_reason"] == 1, (info, plan)
