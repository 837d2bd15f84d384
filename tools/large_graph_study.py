"""The two-level PCG with global-memory aggregates (k_pg_pcg_2lvl_g, linear_solver 13 / 16) against block-Jacobi PCG from
global memory (kernel 0, B200PG_FORCE_GLOBAL_PCG=1) on pose graphs past the shared-memory kernels' reach.

Graphs are seeded synth.make_pose_graph graphs: cfg4 density (4 edges per node, sigma 0.05 m / 0.02 rad) at 10,000 nodes
(the control, which plans the shared-memory two-level kernel 6), 15,000, 30,000 and 100,000 nodes, with the lattice side
scaled with sqrt(N); the density of a recorded mapping run (1.22 edges per node, sigma 0.03 / 0.01) at 60,000 and 200,000
nodes; and 1,000,000 nodes / 4,000,000 edges from the vectorised synth.make_pose_graph_large, whose LM solve is capped at
5 iterations (both kernels run the same steps; a full solve of kernel 0 there takes minutes).  On each graph the default
plan and forced kernel 0 run alternately on fresh handles (--reps of each).  Every row records the planned kernel, LM iterations,
accepted steps, linear solves, total CG iterations, device ms and device ms per CG iteration (whole solve / CG
iterations), for the global two-level kernel the aggregate size and coarse size nc (pg_pcg.cu's rule restated in
coarse_plan; tests/test_posegraph_large_gpu.py checks it against the plan the solver prints), and the algorithmic bytes of
one CG iteration (fine level and the dense coarse mat-vec) over the time per iteration, against the data-sheet HBM3
bandwidth (3.35 TB/s).  Working sets of a few tens of MB sit in L2, so that ratio is a bandwidth share only where the
working set does not fit L2 (50 MB).  --parent-lib loads another build of the library (the parent commit's) and records
which kernel its plan picks on each graph.  Where a graph has at most --chol-max-nodes nodes, the exact Cholesky solve (linear_solver_type = 1)
also runs once and its pose gap to the PCG solves is reported.  The card's name, power limit and max SM clock are read in
the same call.

    python tools/large_graph_study.py [--out profiles/h100_large_graph.json] [--reps 3] [--graphs cfg4_15k,...]
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from dogleg_study import card, pose_diff  # noqa: E402
from slam_toolbox_b200 import api, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
CFG4, RECORDED = (0.05, 0.02), (0.03, 0.01)
# name: (generator, seed, nodes, edges, lattice side, (sigma_xy, sigma_th), max LM iterations)
GRAPHS = {
    "cfg4_10k": (synth.make_pose_graph, 0, 10000, 40000, 100, CFG4, 50),
    "cfg4_15k": (synth.make_pose_graph, 7, 15000, 60000, 122, CFG4, 50),
    "cfg4_30k": (synth.make_pose_graph, 7, 30000, 120000, 173, CFG4, 50),
    "cfg4_100k": (synth.make_pose_graph, 7, 100000, 400000, 316, CFG4, 50),
    "recorded_60k": (synth.make_pose_graph, 7, 60000, 73200, 245, RECORDED, 50),
    "recorded_200k": (synth.make_pose_graph, 7, 200000, 244000, 447, RECORDED, 50),
    "cfg4_1m": (synth.make_pose_graph_large, 11, 1000000, 4000000, 1000, CFG4, 5),
}


def coarse_plan(n, e, cm=6):
    """pg_pcg.cu coarse_aggregates_2lvl_global(): nc <= sqrt(fine bytes / 32), at most 4096, aggregates >= 16 nodes."""
    fine = 240.0 * n + 128.0 * 2 * e
    nc = min(4096, int(math.sqrt(fine / 32.0)))
    want = max(1, min((n + 15) // 16, nc // cm))
    per = -(-n // want)
    na = -(-n // per)
    return dict(aggregates=na, nodes_per_aggregate=per, nc=cm * na, fine_bytes_per_iteration=fine,
                coarse_bytes_per_iteration=8.0 * (cm * na) ** 2)


def load(s, g):
    """AddNode / AddConstraint for every node and edge, through the C entry points with pointers into the graph's arrays
    (the per-call numpy conversions of api.ScanSolver would dominate at 4M edges)."""
    raw = C.CDLL(api.library_path())
    raw.b200pg_add_node.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    raw.b200pg_add_edge.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    init = np.ascontiguousarray(g["init"], dtype=np.float64)
    z = np.ascontiguousarray(g["z"], dtype=np.float64)
    cov = np.ascontiguousarray(g["cov"], dtype=np.float64).reshape(-1, 9)
    h, pi, pz, pc = s._h.value, init.ctypes.data, z.ctypes.data, cov.ctypes.data
    for k, nid in enumerate(g["ids"].tolist()):
        raw.b200pg_add_node(h, nid, pi + 24 * k)
    add = raw.b200pg_add_edge
    for k, (a, b) in enumerate(zip(g["edge_a"].tolist(), g["edge_b"].tolist())):
        assert add(h, a, b, pz + 24 * k, pc + 72 * k) == 0
    return init, z, cov   # keep the arrays alive until the solve has read them


def one(g, env=None, **opts):
    for k, v in (env or {}).items():
        os.environ[k] = v
    try:
        s = api.ScanSolver(**opts)   # the environment switches are read when the handle is created
    finally:
        for k in (env or {}):
            del os.environ[k]
    keep = load(s, g)
    t = time.perf_counter()
    ok = s.Compute()
    wall = time.perf_counter() - t
    sm = s.summary
    row = dict(ok=bool(ok), linear_solver=int(sm.linear_solver), iterations=int(sm.iterations), accepted=int(sm.successful_steps),
               linear_solves=int(sm.linear_solves), pcg_iterations=int(sm.pcg_iterations), device_ms=float(sm.solve_ms),
               setup_ms=float(sm.setup_ms), wall_s=wall, final_cost=float(sm.final_cost), termination=int(sm.termination))
    row["ms_per_cg_iteration"] = row["device_ms"] / max(1, row["pcg_iterations"])
    x = s.GetCorrections()[1].copy()
    s.close()
    del keep
    return row, x


def parent_plan(path, g):
    """The kernel the plan of another build of the library (at `path`) picks on g: one LM iteration on a fresh handle."""
    saved_lib, saved_path = api._lib, api._build.LIB
    api._lib, api._build.LIB = None, path
    try:
        return one(g, max_num_iterations=1)[0]["linear_solver"]
    finally:
        api._lib, api._build.LIB = saved_lib, saved_path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_large_graph.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--graphs", default=",".join(GRAPHS))
    ap.add_argument("--chol-max-nodes", type=int, default=60000)
    ap.add_argument("--parent-lib", default=None, help="another build of libb200slam.so whose planned kernel is recorded")
    a = ap.parse_args()
    api._check(api.lib().b200_set_device(0))
    out = dict(card=card(), reps=a.reps, hbm_bytes_per_s=HBM_BYTES_PER_S, graphs={})
    for name in a.graphs.split(","):
        gen, seed, n, e, lat, sig, max_it = GRAPHS[name]
        t = time.perf_counter()
        g = gen(seed, n, e, lattice=lat, sigma_xy=sig[0], sigma_th=sig[1])
        rec = dict(generator=gen.__name__, seed=seed, nodes=n, edges=e, lattice=lat, sigma=list(sig), max_num_iterations=max_it,
                   generate_s=time.perf_counter() - t, runs={"default": [], "kernel0": []})
        if a.parent_lib:
            rec["parent_plan_kernel"] = parent_plan(a.parent_lib, g)
            print(name, "parent plan", rec["parent_plan_kernel"], flush=True)
        xs = {}
        for _ in range(a.reps):
            for label, env in (("default", None), ("kernel0", {"B200PG_FORCE_GLOBAL_PCG": "1"})):
                row, x = one(g, env, max_num_iterations=max_it)
                rec["runs"][label].append(row)
                xs[label] = x
                print(name, label, row, flush=True)
        plan = coarse_plan(n, e)
        if rec["runs"]["default"][-1]["linear_solver"] in (13, 16):
            rec["plan"] = plan
        for label, rows in rec["runs"].items():
            r = rows[-1]
            byts = plan["fine_bytes_per_iteration"] + (plan["coarse_bytes_per_iteration"] if r["linear_solver"] in (13, 16) else 0.0)
            ms = statistics.median(x["ms_per_cg_iteration"] for x in rows)
            rec[label] = dict(linear_solver=r["linear_solver"], iterations=r["iterations"], accepted=r["accepted"],
                              pcg_iterations=r["pcg_iterations"], device_ms_median=statistics.median(x["device_ms"] for x in rows),
                              device_ms_spread=max(x["device_ms"] for x in rows) - min(x["device_ms"] for x in rows),
                              ms_per_cg_iteration=ms, bytes_per_cg_iteration=byts,
                              bytes_rate_over_hbm_bandwidth=byts / (ms * 1e-3) / HBM_BYTES_PER_S if ms > 0 else None,
                              working_set_fits_l2=byts < 50e6,
                              reproducible=len({(x["pcg_iterations"], x["final_cost"]) for x in rows}) == 1)
        rec["pose_gap_default_vs_kernel0"] = pose_diff(xs["default"], xs["kernel0"])
        if n <= a.chol_max_nodes:
            row, x = one(g, linear_solver_type=1, max_num_iterations=max_it)
            rec["cholesky"] = dict(row, pose_gap_to_default=pose_diff(x, xs["default"]))
            print(name, "cholesky", rec["cholesky"], flush=True)
        else:
            rec["cholesky"] = f"not run: more than {a.chol_max_nodes} nodes"
        out["graphs"][name] = rec
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({k: {l: v.get(l) for l in ("default", "kernel0")} for k, v in out["graphs"].items()}, indent=1))


if __name__ == "__main__":
    main()
