"""Tiny workloads for compute-sanitizer (memcheck / racecheck / initcheck): a sweep of a few pairs through the fast and the
generic kernel (with refine), a single match, a small pose-graph solve on the PCG kernels, and the same solve on the
Cholesky linear solver ("pg_chol": supernodes with several updating descendants, under LM and dogleg)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import helpers as H
from slam_toolbox_b200 import api, synth

which = sys.argv[1] if len(sys.argv) > 1 else "all"
if which in ("all", "sweep"):
    sw = synth.make_loop_sweep(3, n_queries=1, n_chains=3, chain_len=2, inf_frac=0.02)
    gm = H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    gc, gq = H.gpu_block(sw.cand_ranges, sw.cand_poses), H.gpu_block(sw.query_ranges, sw.query_poses)
    r1 = gm.MatchScanBatch(gq, gc, sw.chain_start, None, False, True)
    gm.set_option("force_generic_sweep", 1)
    r2 = gm.MatchScanBatch(gq, gc, sw.chain_start, None, False, True)
    assert all(np.array_equal(a, b) for a, b in zip(r1, r2))
    print("sweep ok", r1[0])
if which in ("all", "single"):
    case = synth.make_sequential_case(1, buffer_len=3)
    gm = H.gpu_matcher(H.MAPPER_SEQ, H.GRID_SMALL)
    print("single ok", gm.MatchScan(H.gpu_block(case["query_ranges"], case["query_pose"]), H.gpu_block(case["base_ranges"], case["base_poses"]), True, True)[0])
if which in ("all", "pg"):
    g = synth.make_pose_graph(1, 200, 450, sigma_xy=0.03, sigma_th=0.01)
    s = api.ScanSolver(max_num_iterations=3)
    for nid, p in zip(g["ids"], g["init"]): s.AddNode(int(nid), p)
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]): s.AddConstraint(int(a), int(b), z, c)
    print("pg ok", s.Compute(), s.summary.pcg_iterations)
if which in ("all", "pg_chol"):
    g = synth.make_pose_graph(1, 200, 450, sigma_xy=0.03, sigma_th=0.01)
    for strategy in (0, 1):
        s = api.ScanSolver(max_num_iterations=3, linear_solver_type=1, trust_region_strategy=strategy)
        for nid, p in zip(g["ids"], g["init"]): s.AddNode(int(nid), p)
        for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]): s.AddConstraint(int(a), int(b), z, c)
        ok = s.Compute()
        info = s.factor_info()
        assert s.summary.linear_solver == 8 and info["supernodes"] > 1 and info["critical_path"] > 2, info
        print("pg_chol ok", strategy, ok, s.summary.linear_solves, info)
