"""The Cholesky linear solver with its device invariants checked: builds libb200slam.so with -DB200_CHOL_CHECKS into a
temporary directory (device asserts of the schedule's deadlock-freedom conditions -- a CTA waits only on children numbered
below its supernode, or on a parent numbered above it in the reverse phase -- and of the panel layout: every assembled
block, updated element and row mapping inside the supernode's panel), then runs small solves under LM and both dogleg
types on graphs whose supernodes have several updating descendants, and checks them against the unchecked build's
results (bit-identical).

    python tools/chol_checked.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from slam_toolbox_b200 import build as B  # noqa: E402

CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, %(root)r)
from slam_toolbox_b200 import build as B
if %(lib)r:
    B.LIB = %(lib)r
from slam_toolbox_b200 import api, synth
out = []
for seed, n, e in ((1, 200, 450), (2, 1500, 4500)):
    g = synth.make_pose_graph(seed, n, e, sigma_xy=0.05, sigma_th=0.02)
    for strategy, dl in ((0, 0), (1, 0), (1, 1)):
        s = api.ScanSolver(linear_solver_type=1, trust_region_strategy=strategy, dogleg_type=dl)
        for nid, p in zip(g["ids"], g["init"]): s.AddNode(int(nid), p)
        for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]): s.AddConstraint(int(a), int(b), z, c)
        assert s.Compute() and s.summary.linear_solver == 8
        out.append(dict(n=n, strategy=strategy, dogleg_type=dl, info=s.factor_info(), linear_solves=s.summary.linear_solves,
                        poses=s.GetCorrections()[1].tobytes().hex()))
print(json.dumps(out))
"""


def run(lib):
    r = subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, lib=lib)], capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(r.stderr[-3000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    tmp = tempfile.mkdtemp(prefix="b200_chol_checked_")
    objs = []
    for unit, extra in B.UNITS.items():
        obj = os.path.join(tmp, unit.replace(".cu", ".o"))
        flags = extra + (["-DB200_CHOL_CHECKS"] if unit == "pg_cholesky.cu" else [])
        subprocess.run(["nvcc"] + B.ARCH + B.COMMON + flags + ["-c", os.path.join(B.CSRC, unit), "-o", obj], check=True)
        objs.append(obj)
    lib = os.path.join(tmp, "libb200slam.so")
    subprocess.run(["nvcc"] + B.ARCH + ["-shared", "--cudart", "shared", "-o", lib] + objs + ["-ldl"], check=True)
    checked, plain = run(lib), run("")
    for a, b in zip(checked, plain):
        assert a["poses"] == b["poses"] and a["info"] == b["info"], (a["n"], a["strategy"], a["dogleg_type"])
        print(json.dumps({k: a[k] for k in ("n", "strategy", "dogleg_type", "info", "linear_solves")}))
    print(f"chol_checked ok: {len(checked)} solves, every device invariant held, bit-identical to the unchecked build")


if __name__ == "__main__":
    main()
