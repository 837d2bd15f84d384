"""Generates tests/golden/merge_golden.npz from the UNMODIFIED reference (oracle/_ref/libmerge_b200.so, oracle/merge.mk):
slam_toolbox's merge_maps_kinematic data path -- MergeMapsKinematic::transformScan (src/merge_maps_kinematic.cpp:195-248,
restated with Karto's own setters by oracle/merge_ref_driver.cpp's kref_transform_scan) on every scan of every submap, then
karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961) over all of them.  Run where the reference sources are present
(after building the oracle):
    python tests/golden/make_merge_golden.py

A case is a list of submaps and a list of merges; merge m applies corr[m][i] (tf2 basis 3x3 + origin 3) to every scan of
submap i and builds.  The scans are transformed in place, so merge m + 1 transforms merge m's scans again, as the tool does.
  rot30        a mapping run under a 30 degree rotation: the corner box and the point box give other dims and offsets
  fma_point    res 1 m: corrected beam end points at half cells +-1-2 ulps where a fused b0*x + b1*y lands in another cell
  fma_corner   res 1 m: a corrected corner that sets the width, where a fused b0*x + b1*y gives another Round(width)
  round_half   res 1 m: the corrected box is exactly k + 0.5 cells wide (k even): Round gives k + 1, rint and truncation k
  compound     two merges in a row with the same correction (the second one compounds)
  empty        a submap without in-range readings (its boxes are the sensor positions), rotated, next to a mapping run
  three        three submaps with an identity, a pure translation and a rotated correction, merged twice

Each case stores per submap the inputs (ranges, poses), the reference's unfiltered points and sensor poses before any
transform, and per merge the reference's grid (dims, offset, cells, digests + sums of the counters) and stored boxes."""
import hashlib
import math
import os
import sys
from fractions import Fraction

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import helpers as H  # noqa: E402
from slam_toolbox_b200 import synth  # noqa: E402

PATH = os.path.join(HERE, "merge_golden.npz")
N = synth.N_BEAMS
# the correction of the crafted res-1 cases: 33 degrees about the origin, then (0.3, 0.2); anchor (0, 0) lands on the
# origin exactly, so the grid offset is (0.3, 0.2).  (30 degrees would give b1 * y products that are nearly exact, where
# fusing rarely changes a result.)
CRAFT_ORIGIN = (0.3, 0.2, 0.0)
CRAFT_DEG = 33.0


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def rot(deg, origin=(0.0, 0.0, 0.0)):
    """a correction (basis [3, 3], origin [3]) rotating by deg about z"""
    t = math.radians(deg)
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]), np.array(origin, dtype=np.float64)


def ident(origin=(0.0, 0.0, 0.0)):
    return np.eye(3), np.array(origin, dtype=np.float64)


def pack(basis, origin):
    return np.concatenate([np.asarray(basis, dtype=np.float64).ravel(), np.asarray(origin, dtype=np.float64)])


def apply_x(b, o, x, y):
    """x of tf2::Transform(b, o) applied to (x, y, 0), every operation rounded (Python floats never fuse)"""
    return ((b[0][0] * x + b[0][1] * y) + b[0][2] * 0.0) + o[0]


def apply_x_fused(b, o, x, y, which):
    """the same with b0*x + b1*y contracted into one fused multiply-add: which = 0 fma(b0, x, b1*y), 1 fma(b1, y, b0*x)"""
    if which == 0:
        t = float(Fraction(b[0][0]) * Fraction(x) + Fraction(b[0][1] * y))
    else:
        t = float(Fraction(b[0][1]) * Fraction(y) + Fraction(b[0][0] * x))
    return (t + b[0][2] * 0.0) + o[0]


def cell(v, off, scale=1.0):
    return synth.grid_cell(v, off, scale)


def anchor(x, y):
    """an all-inf scan: its box is its sensor position, and it traces nothing"""
    return np.full(N, np.inf), np.array([float(x), float(y), 0.0])


def walk(x0, n):
    """x0 and the n representable values either side of it"""
    out, lo, hi = [x0], x0, x0
    for _ in range(n):
        lo, hi = float(np.nextafter(lo, -np.inf)), float(np.nextafter(hi, np.inf))
        out += [lo, hi]
    return out


def craft_anchors():
    """anchors whose corrected positions bracket every crafted beam: (0, 0) -> (0.3, 0.2), and one beyond (14, 14)"""
    b, o = rot(CRAFT_DEG, CRAFT_ORIGIN)
    t = math.radians(CRAFT_DEG)
    far = (math.cos(t) * 13.7 + math.sin(t) * 13.8, -math.sin(t) * 13.7 + math.cos(t) * 13.8)
    return [anchor(0.0, 0.0), anchor(*far)], (b, o)


def fma_point_case():
    """beams along +x from (8, sy) whose corrected end x' sits at a half cell, unfused and both fused forms on either side"""
    sc, (b, o) = craft_anchors()
    off = o[0]
    found = 0
    for sy in np.random.default_rng(5).uniform(3.0, 5.0, 40):
        sy = float(sy)
        for k in (6, 7, 8, 9):
            target = off + k + 0.5
            px0 = (target - o[0] - b[0][1] * sy) / b[0][0]
            for px in walk(px0, 300):
                u = cell(apply_x(b, o, px, sy), off)
                if all(cell(apply_x_fused(b, o, px, sy, w), off) != u for w in (0, 1)) and px - 8.0 + 8.0 == px:
                    sc.append(synth.axis_scan((8.0, sy), "+x", px - 8.0))
                    found += 1
                    break
    assert found >= 6, found
    return dict(subs=[sc], corr=[[(b, o)]], res=1.0)


def corner_anchor(pred):
    """a pre-image (x, y) of the far anchor whose corrected x is near 0.3 + k + 0.5 (k = 14, 16) and satisfies pred"""
    sc, (b, o) = craft_anchors()
    for by in [sc[1][1][1]] + [float(v) for v in np.random.default_rng(9).uniform(6.0, 8.0, 60)]:
        for k in (14, 16):
            bx0 = (o[0] + k + 0.5 - o[0] - b[0][1] * by) / b[0][0]
            for bx in walk(bx0, 400):
                if pred(b, o, bx, by):
                    return bx, by
    raise RuntimeError("no anchor found")


def width_of(v, off, scale=1.0):
    """ComputeDimensions' math::Round(size * scale) (Math.h:87-90)"""
    return synth.grid_cell(v, off, scale)


def fma_corner_case():
    sc, (b, o) = craft_anchors()
    off = o[0]

    def pred(b, o, x, y):
        w = width_of(apply_x(b, o, x, y), off)
        return all(width_of(apply_x_fused(b, o, x, y, k), off) != w for k in (0, 1))
    bx, by = corner_anchor(pred)
    sc[1] = anchor(bx, by)
    sc.append(synth.axis_scan((6.0, 4.0), "+x", 3.0))
    return dict(subs=[sc], corr=[[(b, o)]], res=1.0)


def round_half_case():
    sc, (b, o) = craft_anchors()
    off = o[0]

    def pred(b, o, x, y):
        v = (apply_x(b, o, x, y) - off) * 1.0
        return v == math.floor(v) + 0.5 and int(math.floor(v)) % 2 == 0
    bx, by = corner_anchor(pred)
    sc[1] = anchor(bx, by)
    sc.append(synth.axis_scan((6.0, 4.0), "+x", 3.0))
    return dict(subs=[sc], corr=[[(b, o)]], res=1.0)


def run_scans(seed, n):
    run = synth.make_mapping_run(seed, n)
    return [(r, p) for r, p in zip(run["ranges"], run["poses"])]


def crafted_cases():
    out = {}
    out["rot30"] = dict(subs=[run_scans(81, 6)], corr=[[rot(30.0, (1.3, -0.7, 0.0))]], res=0.05)
    out["fma_point"] = fma_point_case()
    out["fma_corner"] = fma_corner_case()
    out["round_half"] = round_half_case()
    t = rot(12.0, (0.4, 0.25, 0.0))
    out["compound"] = dict(subs=[run_scans(82, 5)], corr=[[t], [t]], res=0.05)
    empty = [anchor(2.0, 1.0), (np.full(N, 20.0), np.array([3.0, 1.5, 0.4])),
             synth.axis_scan((4.0, 2.0), "+x", 25.0), anchor(5.0, -1.0)]
    out["empty"] = dict(subs=[run_scans(83, 4), empty], corr=[[ident(), rot(45.0, (-1.0, 2.0, 0.0))]], res=0.05)
    three = [ident(), ident((3.1, -1.7, 0.0)), rot(-40.0, (-2.0, 5.5, 0.0))]
    out["three"] = dict(subs=[run_scans(84, 4), run_scans(85, 4), run_scans(86, 4)], corr=[three, three], res=0.05)
    return out


def reference(case):
    """the reference's points / sensor poses before any transform, and per merge its grid and stored boxes"""
    import merge_ref as R
    subs = []
    for i, sub in enumerate(case["subs"]):
        ranges = np.array([s[0] for s in sub])
        poses = np.array([s[1] for s in sub])
        subs.append(dict(ranges=ranges, poses=poses, scans=R.scans(ranges, poses, uid0=1000 * i)))
    for s in subs:
        s["points"] = np.stack([sc.points() for sc in s["scans"]])
        s["sensor"] = np.stack([sc.sensor_pose() for sc in s["scans"]])
    merges = []
    for corr in case["corr"]:
        for s, (b, o) in zip(subs, corr):
            for sc in s["scans"]:
                sc.transform(b, o)
        allscans = [sc for s in subs for sc in s["scans"]]
        g = R.occupancy(allscans, case["res"])
        g["boxes"] = np.stack([sc.box() for sc in allscans])
        merges.append(g)
    return subs, merges


def main():
    out = {}
    cases = crafted_cases()
    for name, c in cases.items():
        subs, merges = reference(c)
        out[f"{name}/nsub"] = np.array([len(subs)])
        out[f"{name}/res"] = np.array([c["res"]])
        out[f"{name}/corr"] = np.array([[pack(b, o) for b, o in corr] for corr in c["corr"]])
        for i, s in enumerate(subs):
            for k in ("ranges", "poses", "points", "sensor"):
                out[f"{name}/sub{i}/{k}"] = s[k]
        for m, g in enumerate(merges):
            p = f"{name}/m{m}"
            out[f"{p}/dims"] = np.array([g["width"], g["height"], g["stride"]])
            out[f"{p}/offset"] = g["offset"]
            out[f"{p}/cells"] = g["cells"]
            out[f"{p}/pass_sha"] = np.array([digest(g["passes"])])
            out[f"{p}/hits_sha"] = np.array([digest(g["hits"])])
            out[f"{p}/sums"] = np.array([int(g["passes"].sum()), int(g["hits"].sum())])
            out[f"{p}/boxes"] = g["boxes"]
            print(name, m, (g["width"], g["height"], g["stride"]), tuple(g["offset"]), "occupied", int((g["cells"] == 100).sum()),
                  "free", int((g["cells"] == 255).sum()), "pass", int(g["passes"].sum()), "hits", int(g["hits"].sum()))
    out["names"] = np.array(list(cases))
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
