"""cfg4 (10,000 nodes / 40,000 edges) at both noise levels under Levenberg-Marquardt, traditional dogleg and subspace dogleg:
iterations, accepted steps, linear solves, PCG iterations, device time and final cost, next to the exact-solve oracle's counts.
Then the PCG tolerance sweep of the dogleg Gauss-Newton solve (as tools/pcg_tolerance_study.py does for LM): whether the
accept / reject sequence stays the oracle's and how far the poses move from the tightest solve.

    python tools/dogleg_study.py [--out profiles/h100_dogleg_cfg4.json] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import posegraph_dogleg as DL  # noqa: E402
from slam_toolbox_b200 import api, synth  # noqa: E402

STRATEGIES = {"lm": dict(), "traditional": dict(trust_region_strategy=1, dogleg_type=0),
              "subspace": dict(trust_region_strategy=1, dogleg_type=1)}
ORACLE = {"lm": DL.Options(), "traditional": DL.Options(trust_region_strategy="dogleg", dogleg_type="traditional"),
          "subspace": DL.Options(trust_region_strategy="dogleg", dogleg_type="subspace")}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the numbers below are still valid; say why the card is not described
        return dict(error=repr(e))


def solve(g, reps, **opts):
    """Best device time of `reps` solves of a freshly loaded graph on one handle; summary and poses of the last."""
    s = api.ScanSolver(**opts)
    best = None
    for _ in range(reps):
        s.Reset()
        for nid, p in zip(g["ids"], g["init"]):
            s.AddNode(int(nid), p)
        for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
            s.AddConstraint(int(a), int(b), z, c)
        assert s.Compute()
        best = s.summary.solve_ms if best is None else min(best, s.summary.solve_ms)
    sm = s.summary
    row = dict(iterations=int(sm.iterations), accepted=int(sm.successful_steps), linear_solves=int(sm.linear_solves),
               pcg_iterations=int(sm.pcg_iterations), device_ms=round(float(best), 3), final_cost=float(sm.final_cost),
               linear_solver=int(sm.linear_solver))
    x = s.GetCorrections()[1]
    s.close()
    return row, x


def pose_diff(x, y):
    d = x - y
    d[:, 2] = synth.wrap(d[:, 2])
    return float(np.abs(d[:, :2]).max()), float(np.abs(d[:, 2]).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_dogleg_cfg4.json"))
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    # under dogleg the Gauss-Newton solve runs to pcg_tolerance / 10 (pose_graph.cu, kDlPcgTolFactor)
    result = dict(card=card(), graph="synth.make_pose_graph(0, 10000, 40000)", pcg_tolerance_default=1e-9,
                  dogleg_gauss_newton_tolerance="pcg_tolerance / 10", rows=[], sweep=[])
    for sig in ((0.03, 0.01), (0.05, 0.02)):
        g = synth.make_pose_graph(0, 10000, 40000, sigma_xy=sig[0], sigma_th=sig[1])
        for name, kw in STRATEGIES.items():
            xo, so = DL.solve(g["init"], g["edge_a"], g["edge_b"], g["z"], cov=g["cov"], opts=ORACLE[name])
            row, x = solve(g, args.reps, **kw)
            dxy, dth = pose_diff(x, xo)
            row.update(sigma=list(sig), strategy=name, oracle=dict(iterations=so.iterations, accepted=so.successful_steps,
                                                                      linear_solves=so.linear_solves, final_cost=so.final_cost),
                       same_sequence=(row["iterations"], row["accepted"], row["linear_solves"]) ==
                       (so.iterations, so.successful_steps, so.linear_solves),
                       dxy_vs_oracle=dxy, dth_vs_oracle=dth)
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
            if name == "lm":
                continue
            ref = None
            for tol in (1e-12, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6):
                r, x = solve(g, 1, pcg_tolerance=tol, **kw)
                ref = x if ref is None else ref
                dxy_t, dth_t = pose_diff(x, ref)
                dxy_o, dth_o = pose_diff(x, xo)
                r.update(sigma=list(sig), strategy=name, pcg_tolerance=tol, gauss_newton_tolerance=tol / 10,
                         same_sequence=(r["iterations"], r["accepted"], r["linear_solves"]) ==
                         (so.iterations, so.successful_steps, so.linear_solves),
                         dxy_vs_tightest=dxy_t, dth_vs_tightest=dth_t, dxy_vs_oracle=dxy_o, dth_vs_oracle=dth_o)
                result["sweep"].append(r)
                print(json.dumps(r), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(args.out)


if __name__ == "__main__":
    main()
