"""Batched loop-closure sweep on dense lidars: 1 query x 1000 candidate scans of synth.make_highres_sweep at 1081 / 2701 / 3600 /
8192 beams, on the 4 m / 12 m and 8 m / 12 m geometries, at +-20 deg / 2 deg and +-20 deg / 1 deg.  Per case: the correlation
kernel's time (b200sm_batch_kernel_ms), the step time (k_find_valid + correlation, events around batch_run with L2 flushed before
each step, as bench.py times its headline), matches/s, lookups/s (nX * nY * nA * n per match), the kernel and tile plan that ran,
and an exact comparison of sampled pairs with the oracle.  Then the same measurement on bench.py's headline input (a control for
the 1081-beam rows and the measurement method), and the generic kernel (forced, angle slices) on one case.  The GPU's
name, power limit and maximum SM clock are read in the same run.
usage: python tools/highres_sweep.py [--out FILE] [--steps K] [--warmup W] [--candidates N] [--beams 1081,2701,3600,8192]"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import bench
from slam_toolbox_b200 import api, synth

FOV = {1081: 270.0, 2701: 270.0, 3600: 360.0, 8192: 360.0}
GRIDS = {"4 m / 12 m": (4.0, 0.05, 0.03, 12.0), "8 m / 12 m": (8.0, 0.05, 0.03, 12.0)}
WINDOWS = {"+-20 deg / 2 deg": 2.0, "+-20 deg / 1 deg": 1.0}
TABLE_BYTES = 200 * 1024   # lookup rows the generic kernel stages in shared memory at once


def mapper_kw(res_deg):
    return dict(bench.LOOP_MAPPER, coarse_angle_resolution=math.radians(res_deg))


def run_case(sw, grid, res_deg, steps, warmup, stream, flush, options=None, parity_samples=3):
    import torch
    kw = mapper_kw(res_deg)
    mapper = api.MapperParams(**{k: (bool(v) if k == "use_response_expansion" else v) for k, v in kw.items()})
    sm = api.ScanMatcher.Create(mapper, *grid)
    sm.set_stream(stream.cuda_stream)
    for k, v in (options or {}).items():
        sm.set_option(k, v)
    laser = api.LaserRangeFinder(minimum_angle=sw.query_laser[0], angular_resolution=sw.query_laser[1])
    q, c = api.ScanBlock(sw.query_ranges, sw.query_poses, laser), api.ScanBlock(sw.cand_ranges, sw.cand_poses, laser)
    npairs = sm.batch_upload(q, c, sw.chain_start, None, False)
    info, plan = sm.batch_info(), sm.batch_tile_info()
    for _ in range(warmup):
        sm.batch_run()
    torch.cuda.synchronize()
    step_ms, kern_ms = [], []
    for k in range(steps):
        flush.fill_(k & 0xFF)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); sm.batch_run(); b.record(stream)
        kern_ms.append(sm.batch_kernel_ms())   # waits for the step
        step_ms.append(a.elapsed_time(b))
    resp, mean, cov = sm.batch_fetch()
    fs = sm.batch_fetch_stats()
    sm.close()
    n = sw.query_ranges.shape[1]
    side = math.floor(grid[0] / grid[1] + 0.5) + 1
    nxy = side // 2 + 1
    na = int(math.floor(2 * kw["coarse_search_angle_offset"] / kw["coarse_angle_resolution"] + 0.5)) + 1
    lookups = nxy * nxy * na * n
    ok = True
    picks = []
    if parity_samples:
        pm = bench._port_matcher(grid, kw)
        from oracle import karto_port as P
        pq = P.PortScan(sw.query_ranges[0], sw.query_poses[0], *sw.query_laser)
        rng = np.random.default_rng(5)
        picks = sorted({0, npairs - 1, int(np.argmax(resp))} | set(rng.integers(0, npairs, max(0, parity_samples - 3)).tolist()))
        for j in picks:
            base = [P.PortScan(sw.cand_ranges[i], sw.cand_poses[i], *sw.cand_laser) for i in range(sw.chain_start[j], sw.chain_start[j + 1])]
            e = pm.match(pq, base, False, False)
            ok = ok and e[0] == resp[j] and np.array_equal(e[1], mean[j]) and np.array_equal(e[2], cov[j])
    km, sms = float(np.median(kern_ms)), float(np.median(step_ms))
    rows = TABLE_BYTES // (4 * n)
    return {"beams": n, "search": f"{nxy}x{nxy}x{na} poses", "pairs": int(npairs), "lookup_table_kb": round(na * n * 4 / 1024, 1),
            "generic_slices": -(-na // rows), "kernel": info["kernel"],
            "plan": {k: plan[k] for k in ("cluster", "chunks", "bands", "band_rows", "clusters", "smem_kb")} if info["kernel"] == "tile" else None,
            "tile_refused_reason": plan["refused_reason"], "kernel_ms": km, "kernel_ms_min": float(np.min(kern_ms)),
            "kernel_ms_max": float(np.max(kern_ms)), "step_ms": sms, "matches_per_s": npairs / (sms * 1e-3),
            "kernel_matches_per_s": npairs / (km * 1e-3), "lookups_per_match": lookups, "lookups_per_s": npairs * lookups / (km * 1e-3),
            "single_match_fallbacks": fs["fallback_pairs"], "parity_pairs": picks, "parity_exact": bool(ok),
            "best_response": float(resp.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the JSON record here")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--candidates", type=int, default=1000)
    ap.add_argument("--beams", default="1081,2701,3600,8192")
    ap.add_argument("--generic-steps", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("highres_sweep.py: no CUDA device")
    torch.cuda.set_device(0)
    api._check(api.lib().b200_set_device(0))
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > the 50 MB L2 of an H100
    dev = bench.device_info(0)
    print(json.dumps({"device": dev}), flush=True)
    rows = []
    sweeps = {}
    for n in (int(b) for b in args.beams.split(",")):
        sweeps[n] = synth.make_highres_sweep(n, FOV[n], n_chains=args.candidates)
        for gname, grid in GRIDS.items():
            for wname, res in WINDOWS.items():
                r = dict(geometry=gname, window=wname, fov_deg=FOV[n], **run_case(sweeps[n], grid, res, args.steps, args.warmup, stream, flush))
                print(json.dumps(r), flush=True)
                rows.append(r)
    # the same measurement on bench.py's headline input (other scans than make_highres_sweep's 1081-beam row)
    qr, qp, cr, cp, cs = bench.make_inputs(0, args.candidates, 1, 1)
    control = dict(geometry="4 m / 12 m", window="+-20 deg / 2 deg", fov_deg=270.0, input="bench.py headline (bench.make_inputs)",
                   **run_case(synth.AdversarialSweep(qr, qp, cr, cp, cs), GRIDS["4 m / 12 m"], 2.0, args.steps, args.warmup, stream, flush))
    print(json.dumps(control), flush=True)
    n = 2701 if 2701 in sweeps else next(iter(sweeps))
    g = dict(geometry="4 m / 12 m", window="+-20 deg / 2 deg", fov_deg=FOV[n], forced="force_generic_sweep = 1",
             **run_case(sweeps[n], GRIDS["4 m / 12 m"], 2.0, args.generic_steps, 1, stream, flush, {"force_generic_sweep": 1}))
    print(json.dumps(g), flush=True)
    rec = {"what": f"batched sweep, 1 query x {args.candidates} candidate scans of synth.make_highres_sweep (room scans from one dense "
                   "laser), all pairs per step; kernel_ms = b200sm_batch_kernel_ms (correlation kernel), step_ms = events around "
                   "batch_run (k_find_valid + correlation), medians of the timed steps, L2 flushed before each step",
           "device": dev, "steps": args.steps, "warmup": args.warmup, "rows": rows, "headline_input": control, "generic": g}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
