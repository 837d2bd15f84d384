"""Generates tests/golden/occupancy_edge_golden.npz from the UNMODIFIED reference (oracle/_ref/libkarto_ref.so):
karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961) on crafted scans that reach the places where a grid build can
be subtly wrong.  Run where the reference sources are present (after building the oracle):
    python tests/golden/make_occupancy_edge_golden.py

Case families (every scan is the standard laser; crafted scans are exact-axis beams, synth.axis_scan, the rest inf):
  half_*      sensor cells, end points and clipped ends at offset + (k + 0.5) * res, each moved by 0..2 ulps; a sensor at
              (w - offset) * scale == 0.49999999999999994; clipped ends of angle-pi beams at negative half cells
  fma_clip_*  over-range beams whose clipped end s + (rt / r) * dx lands in another in-grid cell when the product is fused
  merge_*     resolutions of 1 m and 2 m (whole warps share a cell), alternating inf / valid and 0.15 m / 29 m readings, only
              lane 0 or only lane 31 of each group of 32 beams valid
  dims_*      box sizes of (k + 0.5) * res, widths 8k and 8k + 1, a sensor at the box maximum, 0 x 0 / N x 0 / 0 x N grids,
              all-inf scans, box edges set by readings exactly at the range threshold and at the minimum range
  far_*       make_mapping_run moved rigidly to UTM-like coordinates and to large negative ones (stored as seed + digests)
  update_*    UpdateCell boundaries: hits / pass == threshold, pass == min_pass_through, thresholds 0 and 1

Each crafted case stores the inputs (ranges, poses, parameters), the reference's own unfiltered points and sensor poses,
and the reference's grid: dimensions, offset, the cell bytes and digests + sums of the pass / hit counters."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import helpers as H  # noqa: E402
from slam_toolbox_b200 import synth  # noqa: E402
from oracle import karto_ref as R  # noqa: E402

PATH = os.path.join(HERE, "occupancy_edge_golden.npz")
N = synth.N_BEAMS
RT = H.LASER["range_threshold"]

# far_*: name -> (seed, scans, resolution, translation of the whole run)
FAR_CASES = {
    "far_utm": (71, 8, 0.1, (5e5 + 0.37, 4.4e6 - 0.61)),
    "far_negative": (72, 8, 0.1, (-1e4, -1e4)),
}


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def far_inputs(name):
    """(ranges, poses) of a far_* case: a mapping run translated rigidly"""
    seed, n, _, shift = FAR_CASES[name]
    run = synth.make_mapping_run(seed, n)
    return run["ranges"], run["poses"] + np.array([shift[0], shift[1], 0.0])


def anchor(x, y):
    """an all-inf scan: its sensor position is all it adds to the bounding box, and it traces nothing"""
    return np.full(N, np.inf), np.array([float(x), float(y), 0.0])


def case(scans, res, rt=RT, mp=-1, th=-1.0):
    return dict(ranges=np.array([s[0] for s in scans]), poses=np.array([s[1] for s in scans]), params=np.array([res, rt, mp, th]))


def clip_search(target, rt, direction, seed, tries=400000):
    """(sensor x, range) of an over-range beam along +-x whose clipped end is exactly `target`"""
    rng = np.random.default_rng(seed)
    sign = 1.0 if direction == "+x" else -1.0
    steps = synth._ulp_steps(target - sign * rt, 64)
    for it in range(tries):
        s = steps[it % len(steps)]
        r = float(rng.uniform(rt * 1.0001, synth.RANGE_MAX * 0.999))
        if synth.clipped_end(s, s + sign * r, r, rt) == target:
            return s, r
    raise RuntimeError(f"no clipped end at {target!r}")


def half_cases():
    out = {}
    # res 1: sensors at half cells in x (then y), end points of +y / +x beams at half cells; one sensor at 0.49999999999999994
    sc = [anchor(0, 0), anchor(20, 12)]
    for x in synth.half_cell_centres(0.0, 1.0, (3, 6), 2):
        sc.append(synth.axis_scan((x, 4.0), "+y", 2.5))               # ends at y = 6.5
    for y in synth.half_cell_centres(0.0, 1.0, (8,), 2):
        sc.append(synth.axis_scan((10.0, y), "+x", 3.5))              # ends at x = 13.5
    sc.append(synth.axis_scan((0.49999999999999994, 2.0), "+y", 5.0))
    sc.append(synth.axis_scan((0.49999999999999994, 9.0), "+x", 4.0))
    out["half_sensor_r1"] = case(sc, 1.0)
    # res 0.05: end points of +x beams and sensors in y at half cells
    sc = [anchor(0, 0), anchor(4, 3)]
    for t in synth.half_cell_centres(0.0, 0.05, (25, 30, 34, 41), 2):
        sc.append(synth.axis_scan((1.0, 1.0), "+x", t - 1.0))
    for y in synth.half_cell_centres(0.0, 0.05, (20, 27), 2):
        sc.append(synth.axis_scan((2.5, y), "+x", 0.5))
    out["half_end_r005"] = case(sc, 0.05)
    # clipped ends of over-range +x beams at half cells (res 1 and 0.05)
    for name, res, ks, top in (("half_clip_r1", 1.0, (15, 18), (30, 6)), ("half_clip_r005", 0.05, (300, 361), (25, 2))):
        sc = [anchor(0, 0), anchor(*top)]
        for i, t in enumerate(synth.half_cell_centres(0.0, res, ks, 2)):
            s, r = clip_search(t, RT, "+x", seed=100 + i)
            sc.append(synth.axis_scan((s, 1.0), "+x", r))
        out[name] = case(sc, res)
    # clipped ends of angle-pi beams that leave the box on its low side, at negative half cells (the ceil branch)
    sc = [anchor(0, 0), anchor(20, 6)]
    for i, t in enumerate(synth.half_cell_centres(0.0, 1.0, (-1, -2, -3), 0)):
        s, r = clip_search(t, RT, "-x", seed=200 + i)
        sc.append(synth.axis_scan((s, 3.0), "-x", r))
    out["half_low_r1"] = case(sc, 1.0)
    # ... and one at v = -0.49999999999999994 (range threshold 1 m)
    sc = [anchor(0, 0), anchor(3, 2)]
    s, r = clip_search(-0.49999999999999994, 1.0, "-x", seed=300)
    sc.append(synth.axis_scan((s, 1.0), "-x", r))
    out["half_low_tiny"] = case(sc, 1.0, rt=1.0)
    return out


def fma_cases():
    out = {}
    for name, res, boundary, direction, top in (("fma_clip_r005", 0.05, 20.025, "+x", (25, 2)),
                                                ("fma_clip_r1", 1.0, 19.5, "+x", (30, 4)),
                                                ("fma_clip_low_r005", 0.05, 5.025, "-x", (25, 2))):
        sc = [anchor(0, 0), anchor(*top)]
        for s, r in synth.fma_sensitive_beams(boundary, 0.0, res, RT, 20, seed=17, direction=direction):
            sc.append(synth.axis_scan((s, 1.0), direction, r))
        out[name] = case(sc, res)
    return out


def merge_cases():
    out = {}
    for name, seed, res in (("merge_r1", 61, 1.0), ("merge_r2", 62, 2.0)):
        run = synth.make_mapping_run(seed, 6)
        out[name] = dict(ranges=run["ranges"], poses=run["poses"], params=np.array([res, RT, -1, -1.0]))
    run = synth.make_mapping_run(63, 4)
    r = run["ranges"].copy()
    r[:, 1::2] = np.inf
    out["merge_alt_inf"] = dict(ranges=r, poses=run["poses"], params=np.array([0.05, RT, -1, -1.0]))
    run = synth.make_mapping_run(64, 4)
    r = np.where(np.arange(N) % 2 == 0, 0.15, 29.0)[None, :].repeat(4, axis=0)
    out["merge_near_far"] = dict(ranges=r, poses=run["poses"], params=np.array([0.05, RT, -1, -1.0]))
    for name, seed, lane in (("merge_lane0", 65, 0), ("merge_lane31", 66, 31)):
        run = synth.make_mapping_run(seed, 4)
        r = np.where(np.arange(N) % 32 == lane, run["ranges"], np.inf)
        out[name] = dict(ranges=r, poses=run["poses"], params=np.array([0.1, RT, -1, -1.0]))
    return out


def dims_cases():
    out = {}
    beams = lambda xy: [synth.axis_scan(xy, "+x", 2.0), synth.axis_scan(xy, "+y", 1.5), synth.axis_scan(xy, "-x", 1.0)]   # noqa: E731
    out["dims_half_box"] = case([anchor(0, 0), anchor(10.5, 6.5)] + beams((5.0, 3.0)), 1.0)         # 11 x 7 (rint: 10 x 6)
    out["dims_w16"] = case([anchor(0, 0), anchor(4.0, 2.0)] + beams((1.0, 0.5)), 0.25)              # width 16, stride 16
    out["dims_w17"] = case([anchor(0, 0), anchor(4.25, 2.0)] + beams((1.0, 0.5)), 0.25)             # width 17, stride 24
    # a sensor at the box maximum in x: its traces start at fx == width
    out["dims_sensor_max"] = case([anchor(0, 0), anchor(3, 5), synth.axis_scan((10.0, 2.0), "-x", 4.0),
                                   synth.axis_scan((10.0, 2.0), "-x", 25.0), synth.axis_scan((10.0, 2.0), "+y", 2.0)], 1.0)
    # zero-sized grids: nothing within the range threshold, so the box is made of the sensors; the beams are still traced
    far = lambda xy: [synth.axis_scan(xy, d, 20.0) for d in ("+x", "-x", "+y", "-y")] + [(np.full(N, 20.0), np.array([xy[0], xy[1], 0.3]))]   # noqa: E731
    out["dims_zero"] = case(far((3.0, 4.0)), 1.0)
    out["dims_n_by_0"] = case(far((0.0, 1.0)) + far((7.0, 1.0)), 1.0)
    out["dims_0_by_n"] = case(far((2.0, 0.0)) + far((2.0, 9.0)), 1.0)
    out["dims_all_inf"] = case([anchor(1.0, 1.0), anchor(4.0, 3.0)], 1.0)
    # box edges set by a reading exactly at the range threshold (traced, no hit) and one exactly at the minimum range
    # (in the box, not traced)
    out["dims_range_edges"] = case([anchor(5.0, 3.0), synth.axis_scan((1.0, 1.0), "+x", RT), synth.axis_scan((1.0, 1.0), "-x", 0.1),
                                    synth.axis_scan((1.0, 1.0), "-y", 0.1)], 0.05)
    return out


def update_scans():
    """res 1 m, sensors on rows 0..2 of a 9 x 3 box, +x beams:
    row 0: one beam ends at x = 3, eight end at x = 8 -> cell (3, 0) has pass 10, hits 1 (hits / pass == 0.1)
    row 1: 25 beams end at x = 4 -> cell (4, 1) has pass 50, hits 25
    row 2: one beam ends at x = 5 -> cell (5, 2) has pass 2 == the default min_pass_through"""
    sc = [anchor(9, 3), synth.axis_scan((0.0, 0.0), "+x", 3.0)]
    sc += [synth.axis_scan((0.0, 0.0), "+x", 8.0, which=i) for i in range(8)]
    sc += [synth.axis_scan((0.0, 1.0), "+x", 4.0, which=i) for i in range(25)]
    sc += [synth.axis_scan((0.0, 2.0), "+x", 5.0)]
    return sc


def update_cases():
    sc = update_scans()
    return {"update_default": case(sc, 1.0, mp=-1, th=-1.0), "update_mp0_th0": case(sc, 1.0, mp=0, th=0.0),
            "update_th1": case(sc, 1.0, mp=2, th=1.0), "update_mp50": case(sc, 1.0, mp=50, th=0.1)}


def crafted_cases():
    out = {}
    for f in (half_cases, fma_cases, merge_cases, dims_cases, update_cases):
        out.update(f())
    return out


def reference(ranges, poses, res, rt, mp, th):
    """the reference's grid, points and sensor poses; the range threshold is the laser's, so it is set around the call"""
    R.init_laser(**H.LASER)
    R.lib().kref_laser_set_range_threshold(rt)
    scans = H.ref_scans(ranges, poses)
    g = R.occupancy(scans, res, int(mp), th)
    pts = np.stack([s.points() for s in scans])
    sensor = np.stack([s.sensor_pose() for s in scans])
    R.lib().kref_laser_set_range_threshold(RT)
    return g, pts, sensor


def store(out, name, g):
    out[f"{name}/dims"] = np.array([g["width"], g["height"], g["stride"]])
    out[f"{name}/offset"] = g["offset"]
    out[f"{name}/cells"] = g["cells"]
    out[f"{name}/pass_sha"] = np.array([digest(g["passes"])])
    out[f"{name}/hits_sha"] = np.array([digest(g["hits"])])
    out[f"{name}/sums"] = np.array([int(g["passes"].sum()), int(g["hits"].sum())])
    print(name, (g["width"], g["height"], g["stride"]), "occupied", int((g["cells"] == 100).sum()), "free",
          int((g["cells"] == 255).sum()), "pass", int(g["passes"].sum()), "hits", int(g["hits"].sum()))


def main():
    out = {}
    crafted = crafted_cases()
    for name, c in crafted.items():
        res, rt, mp, th = c["params"]
        g, pts, sensor = reference(c["ranges"], c["poses"], res, rt, mp, th)
        out[f"{name}/ranges"] = c["ranges"]
        out[f"{name}/poses"] = c["poses"]
        out[f"{name}/params"] = c["params"]
        out[f"{name}/points"] = pts
        out[f"{name}/sensor"] = sensor
        store(out, name, g)
    for name, (seed, n, res, shift) in FAR_CASES.items():
        ranges, poses = far_inputs(name)
        g, pts, sensor = reference(ranges, poses, res, RT, -1, -1.0)
        out[f"{name}/params"] = np.array([res, RT, -1, -1.0])
        out[f"{name}/inputs"] = np.array([H.digest(np.concatenate([ranges.ravel(), poses.ravel()]))])
        out[f"{name}/points_digest"] = np.array([H.digest(pts)])
        out[f"{name}/sensor"] = sensor
        store(out, name, g)
    out["names"] = np.array(list(crafted) + list(FAR_CASES))
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
