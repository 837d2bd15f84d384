"""PCG against the exact block-sparse Cholesky linear solver (linear_solver_type = 1) on cfg4 (10,000 nodes / 40,000
edges) at both noise levels and on a graph of the reference's own shape (4,265 nodes / 5,210 edges), each under
Levenberg-Marquardt, traditional dogleg and subspace dogleg. The two solvers are alternated and repeated on fresh
handles; every row records device and wall time, setup time, iterations, accepted steps, linear solves, PCG iterations,
final cost and the pose gap to the exact-solve oracle, and the Cholesky rows the analysis record (b200pg_factor_info).
Then the one-constraint incremental re-solve, and the split of a Cholesky solve's device time between the factor (with
the forward solve folded in), the backward solve and the residual: the kernel's %globaltimer stamps around its two grid
barriers, which the solver prints per LM step under B200PG_DEBUG=1 (read here from a child process).

    python tools/cholesky_study.py [--out profiles/h100_cholesky.json] [--reps 3]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

import posegraph_dogleg as DL  # noqa: E402
from dogleg_study import ORACLE, STRATEGIES, card, pose_diff  # noqa: E402
from slam_toolbox_b200 import api, synth  # noqa: E402

SOLVERS = {"pcg": 0, "cholesky": 1}
GRAPHS = {"cfg4_s0.03": (0, 10000, 40000, 0.03, 0.01), "cfg4_s0.05": (0, 10000, 40000, 0.05, 0.02),
          "ref_4265_5210": (3, 4265, 5210, 0.03, 0.01)}


def load(s, g, upto=None):
    s.Reset()
    for nid, p in zip(g["ids"], g["init"]):
        s.AddNode(int(nid), p)
    m = len(g["z"]) if upto is None else upto
    for k in range(m):
        s.AddConstraint(int(g["edge_a"][k]), int(g["edge_b"][k]), g["z"][k], g["cov"][k])


def one(g, **opts):
    s = api.ScanSolver(**opts)
    load(s, g)
    assert s.Compute()
    sm = s.summary
    row = dict(device_ms=float(sm.solve_ms), wall_ms=float(sm.wall_ms), setup_ms=float(sm.setup_ms),
               iterations=int(sm.iterations), accepted=int(sm.successful_steps), linear_solves=int(sm.linear_solves),
               pcg_iterations=int(sm.pcg_iterations), final_cost=float(sm.final_cost), linear_solver=int(sm.linear_solver))
    info = s.factor_info() if opts.get("linear_solver_type") == 1 else None
    x = s.GetCorrections()[1]
    s.close()
    return row, info, x


def incremental(g, **opts):
    """All but the last constraint solved, then the last one appended and solved again: the re-solve's numbers."""
    s = api.ScanSolver(**opts)
    load(s, g, len(g["z"]) - 1)
    assert s.Compute()
    k = len(g["z"]) - 1
    s.AddConstraint(int(g["edge_a"][k]), int(g["edge_b"][k]), g["z"][k], g["cov"][k])
    assert s.Compute()
    sm = s.summary
    row = dict(device_ms=float(sm.solve_ms), wall_ms=float(sm.wall_ms), setup_ms=float(sm.setup_ms),
               iterations=int(sm.iterations), linear_solves=int(sm.linear_solves), pcg_iterations=int(sm.pcg_iterations),
               uploaded_edges=int(sm.uploaded_edges))
    if opts.get("linear_solver_type") == 1:
        row["factor_info"] = s.factor_info()
    s.close()
    return row


def split(gname):
    """Per-LM-step factor + forward / backward / residual microseconds of the Cholesky kernel on one graph (medians)."""
    seed, n, e, sxy, sth = GRAPHS[gname]
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from cholesky_study import one\nfrom slam_toolbox_b200 import synth\n"
            "g = synth.make_pose_graph(%d, %d, %d, sigma_xy=%r, sigma_th=%r)\n"
            "one(g, linear_solver_type=1)\none(g, linear_solver_type=1)\n") % (ROOT, os.path.join(ROOT, "tools"), seed, n, e, sxy, sth)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, B200PG_DEBUG="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    pat = re.compile(r"cholesky factor\+forward ([0-9.]+) us, backward ([0-9.]+) us, residual ([0-9.]+) us")
    steps = [tuple(float(v) for v in m.groups()) for m in pat.finditer(r.stderr)]
    steps = steps[len(steps) // 2:]   # the second solve: modules loaded, buffers allocated
    cols = list(zip(*steps))
    return dict(graph=gname, strategy="lm", steps=len(steps), factor_forward_us_median=statistics.median(cols[0]),
                backward_us_median=statistics.median(cols[1]), residual_us_median=statistics.median(cols[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_cholesky.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--split-only", action="store_true", help="only the factor / backward split")
    args = ap.parse_args()
    api._check(api.lib().b200_set_device(0))
    result = dict(card=card(), reps=args.reps, rows=[], incremental=[], split=[])
    for gname, (seed, n, e, sxy, sth) in ([] if args.split_only else GRAPHS.items()):
        g = synth.make_pose_graph(seed, n, e, sigma_xy=sxy, sigma_th=sth)
        for strat, kw in STRATEGIES.items():
            xo, so = DL.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=ORACLE[strat])
            runs = {k: [] for k in SOLVERS}
            last = {}
            for _ in range(args.reps):   # alternated
                for sname, lst in SOLVERS.items():
                    row, info, x = one(g, linear_solver_type=lst, **kw)
                    runs[sname].append(row)
                    last[sname] = (row, info, x)
            for sname in SOLVERS:
                row, info, x = last[sname]
                dxy, dth = pose_diff(x, xo)
                out = dict(graph=gname, nodes=n, edges=e, sigma=[sxy, sth], strategy=strat, solver=sname,
                           device_ms_all=[r["device_ms"] for r in runs[sname]],
                           device_ms_median=statistics.median(r["device_ms"] for r in runs[sname]),
                           wall_ms_median=statistics.median(r["wall_ms"] for r in runs[sname]),
                           setup_ms_median=statistics.median(r["setup_ms"] for r in runs[sname]),
                           **{k: row[k] for k in ("iterations", "accepted", "linear_solves", "pcg_iterations", "final_cost",
                                                  "linear_solver")},
                           device_ms_per_linear_solve=statistics.median(r["device_ms"] for r in runs[sname]) /
                           max(1, row["linear_solves"]),
                           oracle=dict(iterations=so.iterations, accepted=so.successful_steps,
                                       linear_solves=so.linear_solves, final_cost=so.final_cost),
                           same_sequence=(row["iterations"], row["accepted"], row["linear_solves"]) ==
                           (so.iterations, so.successful_steps, so.linear_solves),
                           cost_rel_vs_oracle=abs(row["final_cost"] - so.final_cost) / so.final_cost,
                           dxy_vs_oracle=dxy, dth_vs_oracle=dth, factor_info=info)
                result["rows"].append(out)
                print(json.dumps(out), flush=True)
        if gname != "cfg4_s0.05":
            for sname, lst in SOLVERS.items():
                r = incremental(g, linear_solver_type=lst)
                r.update(graph=gname, solver=sname)
                result["incremental"].append(r)
                print(json.dumps(r), flush=True)
    for gname in GRAPHS:
        r = split(gname)
        result["split"].append(r)
        print(json.dumps(r), flush=True)
    result["card_after"] = card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(args.out)


if __name__ == "__main__":
    main()
