"""Scan removal from the resident map store at the size of a long session: 5,000 synthetic 1081-beam scans (make_mapping_run),
resolution 0.05 m.  For each removal pattern:
  compact : b200og_remove_scans (host wall, its synchronise included) and its compaction kernel's own time (CUDA events),
            then the build of the compacted store
  reload  : the only way without it: clear the store, upload the survivors again from host buffers, build
Patterns: the oldest scan (the localization rolling buffer: every other scan moves), 3 and 50 random scans (interior
scans), the last 3 scans (nothing moves).  Medians (and minima) of reps.
Where oracle/_ref holds the replay libraries, a localization replay also publishes the map after every localization step
through the resident store (karto::b200::ResidentOccupancyMap) and the reference's CreateFromScans, and reports both.
Writes profiles/h100_remove_scans.json (or the path given).  Device name, SM count, power limit and max SM clock are read in
the run.
    python tools/remove_scans_study.py [out.json] [--reps 7]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "integration"))

from slam_toolbox_b200 import api, synth  # noqa: E402

N_SCANS, RES = 5000, 0.05


def card():
    q = "name,power.limit,clocks.max.sm"
    out = dict()
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
        out.update(zip(("name", "power_limit", "max_sm_clock"), [s.strip() for s in line.split(",")]))
    except Exception as e:
        out["error"] = repr(e)
    import torch
    out["sm_count"] = torch.cuda.get_device_properties(0).multi_processor_count
    return out


def stat(v):
    return dict(median=float(np.median(v)), min=float(np.min(v)))


def patterns(rng):
    return {"oldest": np.array([0]),
            "random_3": np.sort(rng.choice(N_SCANS, 3, replace=False)),
            "random_50": np.sort(rng.choice(N_SCANS, 50, replace=False)),
            "last_3": np.arange(N_SCANS - 3, N_SCANS)}


def study(reps):
    laser = api.LaserRangeFinder()
    run = synth.make_mapping_run(300, N_SCANS)
    block = api.ScanBlock(run["ranges"], run["poses"], laser)
    g = api.OccupancyGrid(RES, laser)
    rng = np.random.default_rng(1)
    out = {}
    for name, idx in patterns(rng).items():
        keep = np.setdiff1d(np.arange(N_SCANS), idx)
        survivors = api.ScanBlock(block.ranges[keep], block.poses[keep], laser, points=block.points[keep])
        rec = dict(removed=int(len(idx)), moved_scans=int(N_SCANS - idx[0] - len(idx)))
        comp_wall, comp_kernel, comp_build, reload_wall, build_dev = [], [], [], [], []
        for r in range(reps + 1):   # rep 0 warms up (buffer growth, module load)
            g.ClearScans()
            g.AddScans(block)
            g.Build()
            t0 = time.perf_counter()
            g.RemoveScans(idx)
            t1 = time.perf_counter()
            kms = g.kernel_ms()
            g.Build()
            t2 = time.perf_counter()
            bms = g.kernel_ms()
            compact = g.GetData()
            t3 = time.perf_counter()
            g.ClearScans()
            g.AddScans(survivors)
            g.Build()
            t4 = time.perf_counter()
            assert np.array_equal(compact, g.GetData()), name
            if r:
                comp_wall.append((t1 - t0) * 1e3)
                comp_kernel.append(kms)
                comp_build.append((t2 - t1) * 1e3)
                reload_wall.append((t4 - t3) * 1e3)
                build_dev.append(bms)
        rec.update(remove_scans_host_ms=stat(comp_wall), compaction_kernel_ms=stat(comp_kernel),
                   remove_plus_build_host_ms=stat(np.add(comp_wall, comp_build)), build_device_ms=stat(build_dev),
                   reload_plus_build_host_ms=stat(reload_wall))
        out[name] = rec
    return out


def replay_publishes():
    import replay
    if not replay.available():
        return dict(skipped="oracle/_ref replay libraries not built")
    m_r, m_o, _ = replay.make_trajectory(4, 120)
    l_r, l_o, _ = replay.make_localization_trajectory(4, 80, map_scans=120)
    params = dict(replay.YAML_PARAMS, correlation_search_space_smear_deviation=0.03, loop_search_space_dimension=4.0)
    res = {}
    for which in ("b200",):
        o = replay.run_localization(which, m_r, m_o, l_r, l_o, params, events=[(0, "process_near", l_o[0])], map_resolution=RES,
                                    publish_every=1)
        p = o["publishes"]
        res[which] = dict(publishes=int(len(p)), all_equal=bool(p[:, 1].all()), removed=int(p[:, 2].sum()),
                          appended=int(p[:, 3].sum()), reloads=int(p[:, 4].sum()),
                          resident_publish_ms=stat(p[1:, 5] * 1e3), reference_publish_ms=stat(p[1:, 6] * 1e3),
                          resident_build_device_ms=stat(p[1:, 7]),
                          note="localization replay: 120 mapped scans, 80 localization steps, a publish after every step; "
                               "times exclude the first publish (initial load)")
    return res


def main():
    path = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else os.path.join(ROOT, "profiles", "h100_remove_scans.json")
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 7
    api._check(api.lib().b200_set_device(0))
    res = dict(workload=f"{N_SCANS} synthetic 1081-beam scans (make_mapping_run), resolution {RES} m", device=card(), reps=reps,
               patterns=study(reps), replay=replay_publishes())
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
