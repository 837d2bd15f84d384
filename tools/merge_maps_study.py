"""Map merge at the scale of a multi-session merge: 4 submaps of 5,000 synthetic 1081-beam scans each (make_mapping_run,
the sessions offset and rotated against each other), resident on the device.  One marker move, then a merge:
  device   : transform of every submap's scans (its accumulated correction) + the merged build, CUDA events, median of reps
  host     : the same merge host-to-host, fetch_nav (the nav_msgs payload) included, median of reps
  reupload : the alternative without resident scans: correct the points on the host (numpy, the same formula), clear,
             re-upload, build, fetch_nav
  reference: the reference's transformScan + CreateFromScans on one core (oracle/_ref/libmerge_b200.so), measured on one
             submap of 5,000 scans and scaled by 4 (labelled so); skipped without oracle/_ref
Writes profiles/h100_merge_maps.json (or the path given).  Device name, power limit and max SM clock are read in the run.
    python tools/merge_maps_study.py [out.json] [--reps 5]"""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from slam_toolbox_b200 import api, merge_maps, synth  # noqa: E402

N_SUB, N_SCANS, RES = 4, 5000, 0.05


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:
        return dict(error=repr(e))


def sessions(laser):
    out = []
    for k in range(N_SUB):
        run = synth.make_mapping_run(200 + k, N_SCANS)
        t = math.radians(35.0 * k)
        c, s = math.cos(t), math.sin(t)
        p = run["poses"].copy()
        p[:, 0] = c * run["poses"][:, 0] - s * run["poses"][:, 1] + 30.0 * k
        p[:, 1] = s * run["poses"][:, 0] + c * run["poses"][:, 1] - 12.0 * k
        p[:, 2] = synth.wrap(p[:, 2] + t)
        out.append(api.ScanBlock(run["ranges"], p, laser))
    return out


def host_transform(points, t):
    b, o = t.basis, t.origin
    x, y = points[..., 0], points[..., 1]
    out = np.empty_like(points)
    out[..., 0] = ((b[0, 0] * x + b[0, 1] * y) + b[0, 2] * 0.0) + o[0]
    out[..., 1] = ((b[1, 0] * x + b[1, 1] * y) + b[1, 2] * 0.0) + o[1]
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    path = args[0] if args else os.path.join(ROOT, "profiles", "h100_merge_maps.json")
    laser = api.LaserRangeFinder()
    blocks = sessions(laser)
    mm = merge_maps.MergeMapsKinematic(RES, laser)
    t0 = time.perf_counter()
    for b in blocks:
        mm.AddSubmap(b)
    add_s = time.perf_counter() - t0
    mm.MoveSubmap(2, 5.0, -3.0, 0.3)
    mm.Merge()
    mm.grid.toNavMap()   # warm-up: first transform computes the per-scan boxes
    dev, host = [], []
    for r in range(reps):
        mm.MoveSubmap(3, 1.0 + 0.1 * r, 2.0, 0.05)
        t = time.perf_counter()
        ms = 0.0
        for sid, (first, count) in mm.ranges.items():
            c = mm.corrections[sid]
            mm.grid.TransformScans(first, count, c.basis, c.origin)
            ms += mm.grid.kernel_ms()
        mm.grid.Build()
        ms += mm.grid.kernel_ms()
        nav = mm.grid.toNavMap()
        host.append((time.perf_counter() - t) * 1e3)
        dev.append(ms)
    dims = (mm.grid.GetWidth(), mm.grid.GetHeight())
    # the alternative: host-side correction, clear, re-upload, build
    g = api.OccupancyGrid(RES, laser)
    pts = [b.points.copy() for b in blocks]
    re = []
    for r in range(reps):
        t = time.perf_counter()
        g.ClearScans()
        for k, b in enumerate(blocks):
            pts[k] = host_transform(pts[k], mm.corrections[k + 1])
            poses = b.poses.copy()
            poses[:, :2] = host_transform(b.poses[:, :2], mm.corrections[k + 1])
            g.AddScans(api.ScanBlock(b.ranges, poses, laser, points=pts[k]))
        g.Build()
        g.toNavMap()
        re.append((time.perf_counter() - t) * 1e3)
    out = dict(workload=f"{N_SUB} submaps x {N_SCANS} synthetic 1081-beam scans (make_mapping_run, offset and rotated), "
                        f"resolution {RES} m; one marker move then a merge", device=card(),
               merged_grid=dict(width=dims[0], height=dims[1]), nav_cells=int(nav.size), reps=reps,
               add_submaps_s=add_s,
               resident=dict(device_ms_transform_plus_build=dict(median=float(np.median(dev)), min=float(np.min(dev))),
                             host_ms_incl_fetch_nav=dict(median=float(np.median(host)), min=float(np.min(host)))),
               reupload=dict(host_ms_transform_clear_upload_build_fetch_nav=dict(median=float(np.median(re)), min=float(np.min(re))),
                             note="correction of the points on the host in numpy; the grid differs from the tool's (point boxes)"))
    try:
        import merge_ref as R
        if not R.available():
            raise RuntimeError("oracle/_ref/libmerge_b200.so not built")
        b = blocks[0]
        scans = R.scans(b.ranges, b.poses)
        c = mm.corrections[1]
        t = time.perf_counter()
        for s in scans:
            s.transform(c.basis, c.origin)
        tr = time.perf_counter() - t
        gr = R.occupancy(scans, RES, counters=False)
        out["reference_one_core"] = dict(measured_scans=N_SCANS, transform_s=tr, create_from_scans_s=gr["seconds"],
                                         estimated_merge_s_for_all=N_SUB * (tr + gr["seconds"]),
                                         note="one submap measured, the 4-submap merge estimated as 4 x that (not measured)")
    except Exception as e:
        out["reference_one_core"] = dict(not_measured=repr(e))
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
