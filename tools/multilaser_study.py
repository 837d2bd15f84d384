"""Cost of per-scan laser limits in the occupancy-grid build, 5,000 synthetic 1081-beam scans at 0.05 m (bench.py's
occupancy_grid workload: make_mapping_run(3, 5000) in a 60 m world).
  mixed    : the same scans stored with two alternating lasers (12 m / 0.1 m / 30 m and 8 m / 0.5 m / 20 m) against all on
             one laser (b200og_add_scans_lasers vs b200og_add_scans): build device time (b200og_kernel_ms) and the
             upload's host wall time.  A third store holds every scan through b200og_add_scans_lasers with the first laser's
             limits, so that the cost of per-scan limits is told apart from the cost of the other laser's different work.
  parent   : the existing workload (one laser, b200og_add_scans + b200og_build) on the parent commit's library and on this
             tree's, alternated round by round in one process; both libraries are driven through the same C calls.  The same
             store then takes `--builds` compactions (b200og_remove_scans of its first scan, so every other scan moves) and
             `--builds` transforms of every scan (b200og_transform_scans), each timed by b200og_kernel_ms, and a last build
             of the compacted, transformed store whose output must be identical too.
Medians of `--builds` calls per round, over `--rounds` rounds; the spread is (max - min) / median of the round medians.
Writes the JSON to the path given (default profiles/h100_multilaser.json).  Card name and power limit are read in the run.
    python tools/multilaser_study.py [out.json] [--parent-lib build/parent/libb200slam.so] [--rounds 7] [--builds 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from slam_toolbox_b200 import api, synth  # noqa: E402

N_SCANS, RES = 5000, 0.05
LASER_B = api.LaserRangeFinder(range_threshold=8.0, minimum_range=0.5, maximum_range=20.0)


def card():
    out = dict()
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out.update(zip(("name", "power_limit", "max_sm_clock"), [s.strip() for s in line.split(",")]))
    except Exception as e:
        out["error"] = repr(e)
    return out


def bind(L):
    """the b200og calls both libraries share"""
    L.b200og_create.argtypes = [C.POINTER(api.OgParams), C.POINTER(C.c_void_p)]
    L.b200og_destroy.argtypes = [C.c_void_p]
    L.b200og_add_scans.argtypes = [C.c_void_p, C.POINTER(api.CScan), C.c_int32]
    L.b200og_build.argtypes = [C.c_void_p, C.POINTER(api.OgInfo)]
    L.b200og_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.b200og_fetch.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.b200og_remove_scans.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]
    L.b200og_num_scans.argtypes = [C.c_void_p]
    L.b200og_transform_scans.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                         C.POINTER(C.c_double)]
    return L


def builds(L, h, n):
    info, ms, out = api.OgInfo(), C.c_float(), []
    assert L.b200og_build(h, C.byref(info)) == 0   # warm-up
    for _ in range(n):
        assert L.b200og_build(h, C.byref(info)) == 0
        L.b200og_kernel_ms(h, C.byref(ms))
        out.append(ms.value)
    return out, info


def timed(L, h, n, call):
    """b200og_kernel_ms of n calls of call()"""
    ms, out = C.c_float(), []
    for _ in range(n):
        assert call() == 0
        L.b200og_kernel_ms(h, C.byref(ms))
        out.append(ms.value)
    return out


def compactions(L, h, n):
    first = (C.c_int32 * 1)(0)
    return timed(L, h, n, lambda: L.b200og_remove_scans(h, first, 1))


def transforms(L, h, n):
    t = 0.001   # a small rotation and shift per call, so that the grid keeps its size
    basis = (C.c_double * 9)(np.cos(t), -np.sin(t), 0.0, np.sin(t), np.cos(t), 0.0, 0.0, 0.0, 1.0)
    origin = (C.c_double * 3)(0.01, -0.005, 0.0)
    return timed(L, h, n, lambda: L.b200og_transform_scans(h, 0, L.b200og_num_scans(h), basis, origin, None))


def one_laser_store(L, block):
    laser = api.LaserRangeFinder()
    p = api.OgParams(RES, laser.range_threshold, laser.minimum_range, laser.maximum_range, 2, 0.1)
    h = C.c_void_p()
    assert L.b200og_create(C.byref(p), C.byref(h)) == 0
    assert L.b200og_add_scans(h, block.c, len(block)) == 0
    return h


def digest(L, h, info):
    n = info.stride * info.height
    cells, ps, ht = np.zeros(n, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    assert L.b200og_fetch(h, cells.ctypes.data_as(C.POINTER(C.c_uint8)), ps.ctypes.data_as(C.POINTER(C.c_uint32)),
                          ht.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
    return (info.width, info.height, info.stride, info.offset[0], info.offset[1], cells.tobytes(), ps.tobytes(), ht.tobytes())


def summary(rounds):
    med = [float(np.median(r)) for r in rounds]
    m = float(np.median(med))
    return dict(median_ms=m, round_medians_ms=med, spread=(max(med) - min(med)) / m)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=os.path.join(ROOT, "profiles", "h100_multilaser.json"))
    ap.add_argument("--parent-lib", default=os.path.join(ROOT, "build", "parent", "libb200slam.so"))
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--builds", type=int, default=20)
    a = ap.parse_args()
    api._check(api.lib().b200_set_device(0))
    run = synth.make_mapping_run(3, N_SCANS, world=synth.make_world(3, size=60.0), odd_readings=False)
    laser = api.LaserRangeFinder()
    block = api.ScanBlock(run["ranges"], run["poses"], laser)
    res = dict(card=card(), scans=N_SCANS, beams=int(run["ranges"].size), resolution=RES)

    # mixed lasers against one laser, this tree
    two = [laser if s % 2 == 0 else LASER_B for s in range(N_SCANS)]
    one_r, mix_r, same_r, up1, up2 = [], [], [], [], []
    for _ in range(a.rounds):
        g1 = api.OccupancyGrid(RES, laser)
        t = time.perf_counter(); g1.AddScans(block); up1.append((time.perf_counter() - t) * 1e3)
        g2 = api.OccupancyGrid(RES, laser)
        t = time.perf_counter(); g2.AddScans(block, laser=two); up2.append((time.perf_counter() - t) * 1e3)
        g3 = api.OccupancyGrid(RES, laser)
        g3.AddScans(block, laser=[laser] * N_SCANS)
        ms1, info1 = builds(api.lib(), g1._h, a.builds)
        ms2, info2 = builds(api.lib(), g2._h, a.builds)
        ms3, _ = builds(api.lib(), g3._h, a.builds)
        g3.close()
        one_r.append(ms1)
        mix_r.append(ms2)
        same_r.append(ms3)
        grids = [[info1.width, info1.height], [info2.width, info2.height]]
        # pass-counter sums: the traced cells, which the second laser's shorter threshold changes
        updates = [int(np.frombuffer(digest(api.lib(), h, i)[6], np.uint32).sum()) for h, i in ((g1._h, info1), (g2._h, info2))]
        g1.close(); g2.close()
    res["mixed"] = dict(one_laser=summary(one_r), two_lasers=summary(mix_r), per_scan_same_limits=summary(same_r), laser_b=[LASER_B.range_threshold, LASER_B.minimum_range,
                        LASER_B.maximum_range], grid_one_laser=grids[0], grid_two_lasers=grids[1],
                        cell_updates_one_laser=updates[0], cell_updates_two_lasers=updates[1], upload_ms_one_laser=float(np.median(up1)),
                        upload_ms_two_lasers=float(np.median(up2)))

    # the existing workload: parent library against this tree's, alternated
    if os.path.exists(a.parent_lib):
        libs = {"parent": bind(C.CDLL(a.parent_lib)), "change": bind(C.CDLL(api.library_path()))}
        rounds = {op: {k: [] for k in libs} for op in ("occupancy_grid", "compaction", "transform")}
        digests = {op: {} for op in ("occupancy_grid", "after_compaction_and_transform")}
        for r in range(a.rounds):
            for k in (("parent", "change") if r % 2 == 0 else ("change", "parent")):
                L = libs[k]
                h = one_laser_store(L, block)
                ms, info = builds(L, h, a.builds)
                rounds["occupancy_grid"][k].append(ms)
                if r == 0:
                    digests["occupancy_grid"][k] = digest(L, h, info)
                rounds["compaction"][k].append(compactions(L, h, a.builds))
                rounds["transform"][k].append(transforms(L, h, a.builds))
                if r == 0:
                    info = api.OgInfo()
                    assert L.b200og_build(h, C.byref(info)) == 0
                    digests["after_compaction_and_transform"][k] = digest(L, h, info)
                L.b200og_destroy(h)
        for op, v in rounds.items():
            res[op] = {k: summary(x) for k, x in v.items()}
            res[op]["change_over_parent"] = res[op]["change"]["median_ms"] / res[op]["parent"]["median_ms"]
        res["occupancy_grid"]["identical_output"] = digests["occupancy_grid"]["parent"] == digests["occupancy_grid"]["change"]
        res["compaction"]["identical_output"] = (digests["after_compaction_and_transform"]["parent"] ==
                                                 digests["after_compaction_and_transform"]["change"])
        res["transform"]["identical_output"] = res["compaction"]["identical_output"]
    else:
        res["occupancy_grid"] = dict(error=f"no parent library at {a.parent_lib}")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
