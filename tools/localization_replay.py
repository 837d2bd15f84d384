"""Localization-mode replay: map a trajectory with slam_toolbox's shipped parameters (Mapper::Process), then localize a second
pass with config/mapper_params_localization.yaml (Mapper::ProcessLocalization, rolling buffer of 3 scans), once with the GPU
matcher (libreplay_b200.so) and once with the reference CPU matcher (libreplay_ref.so), both with the GPU solver adapter.
The mapping phase of each arm warms its process up; the localization phase is what is reported.  The reference matcher's loop
searches (8 m window, a chain of 3 is enough for a closure) take it seconds per localization step, so its arm localizes only the
first --ref-loc-scans scans; localization is causal, so those steps must equal the GPU arm's first steps bit for bit.
    python tools/localization_replay.py [--map-scans 2000] [--loc-scans 1000] [--ref-loc-scans 60] [--out profiles/h100_localization.json]
Writes one JSON record (also printed) with the device name, SM count and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import replay  # noqa: E402


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": p.name, "sm_count": p.multi_processor_count, "power_limit_and_max_sm_clock": q.stdout.strip()}


def arm(r, n_loc):
    done = int(r["flags"].sum())
    k = r["map_computes"]
    ms, up = r["compute_ms"][k:], r["compute_uploaded"][k:]
    return {"loc_scans_in": n_loc, "loc_scans_processed": done, "loc_seconds": float(r["loc_seconds"]),
            "loc_scans_per_s": done / float(r["loc_seconds"]),
            "map_scans_kept": int(r["map_counts"][0]), "map_seconds": float(r["map_seconds"]),
            "solver_computes": int(len(ms)), "solver_device_ms_total": float(ms.sum()),
            "solver_device_ms_per_compute": float(ms.mean()) if len(ms) else None,
            "uploaded_edges_per_compute": {"mean": float(up.mean()) if len(up) else None, "min": int(up.min()) if len(up) else None,
                                           "max": int(up.max()) if len(up) else None},
            "mapper_edges_at_end": int(r["step_counts"][-1, 1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--map-scans", type=int, default=2000)
    ap.add_argument("--loc-scans", type=int, default=1000)
    ap.add_argument("--ref-loc-scans", type=int, default=60)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_localization.json"))
    a = ap.parse_args()
    t0 = time.time()

    def heartbeat():   # the replays run in child processes that print nothing until they end
        while True:
            time.sleep(30)
            print(f"... {time.time() - t0:.0f} s", flush=True)
    threading.Thread(target=heartbeat, daemon=True).start()
    if not replay.available():
        sys.exit("oracle/_ref/libreplay_*.so not built (needs the reference sources at build time)")
    mr, mo, _ = replay.make_trajectory(6, a.map_scans)
    lr, lo, lt = replay.make_localization_trajectory(6, a.loc_scans, map_scans=a.map_scans)
    ev = [(0, "process_near", lo[0])]   # the robot starts on the map from a pose estimate
    out = {"workload": f"map {a.map_scans} posed 1081-beam scans (shipped YAML parameters), then localize {a.loc_scans} scans of a "
                       f"second pass (localization YAML: rolling buffer 3, loop chains of 3), first scan near a pose estimate",
           "device": device()}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)

    def save():
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    b = replay.run_localization("b200", mr, mo, lr, lo, replay.YAML_PARAMS, events=ev)
    out["b200"] = arm(b, a.loc_scans)
    out["b200"]["matches_per_loc_step"] = b["loc_match_calls"] / a.loc_scans
    done = b["flags"] == 1
    out["b200"]["max_xy_error_m"] = float(np.abs(b["poses"][done, :2] - lt[done, :2]).max())
    out["b200"]["max_xy_odometry_error_m"] = float(np.abs(lo[done, :2] - lt[done, :2]).max())
    save()
    k = a.ref_loc_scans
    r = replay.run_localization("ref", mr, mo, lr[:k], lo[:k], replay.YAML_PARAMS, events=ev)
    out["ref"] = arm(r, k)
    n_b = int(b["flags"][:k].sum())
    secs_b = float(np.cumsum(b["step_seconds"])[k - 1]) if "step_seconds" in b else None
    out["b200_on_ref_prefix"] = {"loc_scans_in": k, "loc_scans_processed": n_b, "loc_seconds": secs_b,
                                 "loc_scans_per_s": n_b / secs_b if secs_b else None}
    out["identical_localization_on_ref_prefix"] = bool(np.array_equal(b["poses"][:k], r["poses"], equal_nan=True)
                                                       and np.array_equal(b["flags"][:k], r["flags"]))
    if secs_b:
        out["speedup_loc_scans_per_s_on_ref_prefix"] = out["b200_on_ref_prefix"]["loc_scans_per_s"] / out["ref"]["loc_scans_per_s"]
    out["wall_s"] = time.time() - t0
    save()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
