"""Section timers of k_sweep_tile: where the SM cycles of a pair go.

Builds the library with -DB200_TILE_TIMERS into a scratch directory (the shipped library has no timers), runs the
bench's cfg2 loop-closure batch (1 query x N candidates, +-2 m / +-20 deg, 41 x 41 x 21 poses) or another geometry,
and prints every section as a share of the warp cycles of the launch and as SM cycles per pair.

usage: tile_timers.py [--n 1000] [--geom 4:12] [--runs 5] [--build-dir DIR [--reuse]] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from slam_toolbox_b200 import build as _build  # noqa: E402

SECTIONS = ["clear+raster", "descriptor wait", "items: correlation", "items: flush", "stage-end barrier",
            "chunk reduction", "pair epilogue"]


def build_instrumented(out_dir: str) -> str:
    nvcc = os.environ.get("NVCC", "nvcc")

    def one(unit):
        obj = os.path.join(out_dir, unit.replace(".cu", ".o"))
        cmd = [nvcc] + _build.ARCH + _build.COMMON + _build.UNITS[unit] + ["-DB200_TILE_TIMERS", "-c",
                                                                           os.path.join(_build.CSRC, unit), "-o", obj]
        subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(len(_build.UNITS)) as ex:
        objs = list(ex.map(one, _build.UNITS))
    lib = os.path.join(out_dir, "libb200slam_timers.so")
    subprocess.run([nvcc] + _build.ARCH + ["-shared", "--cudart", "shared", "-Xlinker", "-rpath,/usr/local/cuda/lib64",
                                           "-o", lib] + objs + ["-ldl"], check=True)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000, help="candidate scans (pairs)")
    ap.add_argument("--geom", default="4:12", help="search dimension [m]:range threshold [m]")
    ap.add_argument("--runs", type=int, default=5, help="timed launches (after one warm-up)")
    ap.add_argument("--build-dir", default=None, help="where the instrumented library goes (default: a temporary directory)")
    ap.add_argument("--reuse", action="store_true", help="take the instrumented library already in --build-dir")
    ap.add_argument("--json", default=None, help="also write the result here")
    a = ap.parse_args()

    build_dir = a.build_dir or tempfile.mkdtemp(prefix="b200_tile_timers_")
    os.makedirs(build_dir, exist_ok=True)
    prebuilt = os.path.join(build_dir, "libb200slam_timers.so")
    _build.LIB = prebuilt if (a.reuse and os.path.exists(prebuilt)) else build_instrumented(build_dir)
    import bench
    from slam_toolbox_b200 import api
    L = api.lib()
    L.b200_tile_timers.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    L.b200_tile_timers.restype = C.c_int
    nsec = L.b200_tile_timers(None, 1)
    assert nsec == len(SECTIONS) + 1, nsec

    dim, rt = (float(v) for v in a.geom.split(":"))
    qr, qp, cr, cp, cs = bench.make_inputs(0, a.n, 1, 1)
    laser = api.LaserRangeFinder()
    mapper = api.MapperParams(**{k: (bool(v) if k == "use_response_expansion" else v) for k, v in bench.LOOP_MAPPER.items()})
    sm = api.ScanMatcher.Create(mapper, dim, 0.05, 0.03, rt)
    sm.set_option("sweep_kernel", 2)
    sm.batch_upload(api.ScanBlock(qr, qp, laser), api.ScanBlock(cr, cp, laser), cs, None, False)
    info, plan = sm.batch_info(), sm.batch_tile_info()
    assert info["kernel"] == "tile", info
    sm.batch_run()
    L.b200_tile_timers(None, 1)
    ms = []
    for _ in range(a.runs):
        sm.batch_run()
        ms.append(sm.batch_kernel_ms())
    buf = (C.c_ulonglong * nsec)()
    assert L.b200_tile_timers(buf, 1) == nsec
    sm.close()

    total = buf[nsec - 1]
    warps = 1024 // 32
    cyc_pair = total / warps / (a.n * a.runs)   # SM cycles per pair (every CTA runs 32 warps, one CTA per SM)
    split = {name: buf[i] / total for i, name in enumerate(SECTIONS)}
    res = {"geom": a.geom, "pairs": a.n, "runs": a.runs, "plan": plan, "kernel_ms_instrumented": min(ms),
           "sm_cycles_per_pair": round(cyc_pair), "split": {k: round(v, 4) for k, v in split.items()},
           "unaccounted": round(1.0 - sum(split.values()), 4)}
    print(f"k_sweep_tile section split, geometry {a.geom}, {a.n} pairs, plan {plan}")
    print(f"  kernel {min(ms):.3f} ms (instrumented build), {cyc_pair:,.0f} SM cycles per pair")
    for k, v in split.items():
        print(f"  {k:22s} {100 * v:6.2f} %   {v * cyc_pair:10,.0f} cycles/pair")
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
