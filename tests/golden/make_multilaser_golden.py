"""Generates tests/golden/multilaser_golden.npz from the UNMODIFIED reference (oracle/_ref/libmultilaser_ref.so,
oracle/multilaser.mk): karto::OccupancyGrid::CreateFromScans (Karto.h:5946-5961) over scans of several named lasers, each
scan taking its own laser's range threshold, minimum and maximum range.  Run where the reference sources are present
(after building the oracle):
    python tests/golden/make_multilaser_golden.py

The cases are tests/multilaser.py's cases():
  thr_only / minr_only / maxr_only   two lasers that differ in that one limit, scans alternating between them
  tolerance     readings at each laser's threshold - KT_TOLERANCE and one ulp either side (the end cell is hit below only)
  box_long      the longer-threshold laser's far readings set the grid box
  interleaved   A / B / A blocks of scans
  no_inrange    a laser with no in-range reading: its scans add their sensor positions to the box and trace up to 0.5 m
  merge_rot     two submaps on different lasers, the second under a rotated merge correction (the tool's transformScan,
                oracle/merge_ref_driver.cpp), then one grid over both

Each case stores its inputs (ranges, poses, per-scan limits, laser ids, resolution), a digest of the reference's unfiltered
points, and the reference's grid (dims, offset, cells, digests + sums of the counters); merge_rot also its corrections, the
submap of every scan, the stored boxes after the merge and the merged grid."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import multilaser as M  # noqa: E402


def put_grid(out, key, g):
    out[f"{key}/dims"] = np.array([g["width"], g["height"], g["stride"]], dtype=np.int64)
    out[f"{key}/offset"] = np.asarray(g["offset"], dtype=np.float64)
    out[f"{key}/cells"] = g["cells"]
    out[f"{key}/sums"] = np.array([int(g["passes"].sum()), int(g["hits"].sum())], dtype=np.int64)
    out[f"{key}/pass_sha"] = np.array([M.sha(g["passes"])])
    out[f"{key}/hits_sha"] = np.array([M.sha(g["hits"])])


def main():
    assert M.ref_available(), M.REF_PATH
    out = {}
    for name, c in M.cases().items():
        scans = M.ref_scans(c, f"{name}_laser")
        pts = np.stack([s.points() for s in scans])
        for k in ("ranges", "poses", "lasers", "laser_id", "laser_table"):
            out[f"{name}/{k}"] = c[k]
        out[f"{name}/res"] = np.array([c["res"]])
        out[f"{name}/points_sha"] = np.array([M.sha(pts)])
        g = M.ref_occupancy(scans, c["res"])
        put_grid(out, name, g)
        if "corr" in c:
            out[f"{name}/submap"] = c["submap"]
            out[f"{name}/corr"] = c["corr"]
            for s, sc in zip(c["submap"], scans):
                sc.transform(c["corr"][s][:9].reshape(3, 3), c["corr"][s][9:])
            out[f"{name}/boxes"] = np.stack([sc.box() for sc in scans])
            put_grid(out, f"{name}/merged", M.ref_occupancy(scans, c["res"]))
        print(f"{name}: {len(scans)} scans, {g['width']}x{g['height']}, sums {out[f'{name}/sums'].tolist()}")
    np.savez_compressed(M.GOLDEN, **out)
    print("wrote", M.GOLDEN, os.path.getsize(M.GOLDEN), "bytes")


if __name__ == "__main__":
    main()
