"""slam_toolbox's merge_maps_kinematic restated on the host, for the map-merge tests: MergeMapsKinematic::transformScan
(src/merge_maps_kinematic.cpp:195-248) in numpy, and the merged grid through the unchanged C port (oracle/karto_port.c).

The transform is elementwise IEEE FP64 in tf2's order, ((b0*x + b1*y) + b2*0) + o; numpy never fuses a multiply and an
add.  Each stored box becomes the box of its four corrected corners, added in the tool's order with BoundingBox2's strict
comparisons.

kp_occupancy_create sizes its grid from the scans' sensor positions and in-range points (LocalizedRangeScan::Update's rule).
For a transformed store, every scan's stored box goes in first as two zero-beam scans, one at each corner, in the order
ComputeDimensions adds them (Add(min), Add(max), Karto.h:2906-2910).  A zero-beam scan adds its sensor position to the box
and traces nothing.  The real scans add nothing more: the transform is monotone in x and in y, because every IEEE
multiplication by a constant and every addition is.  So each corrected point and sensor position lies inside its corrected
corner box, and the port's box is the union of the stored boxes."""
from __future__ import annotations

import numpy as np

import helpers as H

BIG = 999999999999999999.99999   # BoundingBox2's initial bounds, Karto.h:2845-2849


def apply(basis, origin, x, y):
    """tf2::Transform(basis, origin) applied to (x, y, 0): row dot products, then + origin, every operation rounded"""
    b = np.asarray(basis, dtype=np.float64).reshape(3, 3)
    o = np.asarray(origin, dtype=np.float64).reshape(3)
    with np.errstate(invalid="ignore"):   # points of inf / NaN readings become NaN, as on the device and in the tool
        return ((b[0, 0] * x + b[0, 1] * y) + b[0, 2] * 0.0) + o[0], ((b[1, 0] * x + b[1, 1] * y) + b[1, 2] * 0.0) + o[1]


def corner_boxes(boxes, basis, origin):
    """(S, 4) boxes -> the boxes of their corrected corners, added as min, max, (max x, min y), (min x, max y)"""
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 4)
    out = np.empty_like(boxes)
    mnx = np.full(len(boxes), BIG)
    mny, mxx, mxy = mnx.copy(), -mnx, -mnx
    for cx, cy in ((0, 1), (2, 3), (2, 1), (0, 3)):
        x, y = apply(basis, origin, boxes[:, cx], boxes[:, cy])
        mnx, mny = np.where(x < mnx, x, mnx), np.where(y < mny, y, mny)
        mxx, mxy = np.where(x > mxx, x, mxx), np.where(y > mxy, y, mxy)
    out[:, 0], out[:, 1], out[:, 2], out[:, 3] = mnx, mny, mxx, mxy
    return out


class MergeStore:
    """Flat ranges / points of a set of submaps, their sensor positions and per-scan boxes, corrected in place and built
    with the stored boxes once transformed."""

    def __init__(self, ranges, points, counts, sensor_xy, range_threshold, minimum_range, maximum_range):
        self.ranges = np.ascontiguousarray(ranges, dtype=np.float64).ravel()
        self.points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 2).copy()
        self.counts = np.asarray(counts, dtype=np.int64)
        self.start = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)
        self.sensor = np.ascontiguousarray(sensor_xy, dtype=np.float64).reshape(-1, 2).copy()
        self.rt, self.minr, self.maxr = float(range_threshold), float(minimum_range), float(maximum_range)
        self.boxes = np.zeros((len(self.counts), 4))
        inr = (self.ranges >= self.minr) & (self.ranges <= self.rt)    # math::InRange, Karto.h:5662
        for s in range(len(self.counts)):                               # Update's box, Karto.h:5692-5698
            lo, hi = self.start[s], self.start[s + 1]
            p = self.points[lo:hi][inr[lo:hi]]
            xs = np.concatenate([p[:, 0], self.sensor[s, :1]])
            ys = np.concatenate([p[:, 1], self.sensor[s, 1:]])
            self.boxes[s] = (xs.min(), ys.min(), xs.max(), ys.max())
        self.transformed = False

    def transform(self, first, count, basis, origin):
        lo, hi = self.start[first], self.start[first + count]
        p = self.points[lo:hi]
        p[:, 0], p[:, 1] = apply(basis, origin, p[:, 0].copy(), p[:, 1].copy())
        s = self.sensor[first:first + count]
        s[:, 0], s[:, 1] = apply(basis, origin, s[:, 0].copy(), s[:, 1].copy())
        self.boxes[first:first + count] = corner_boxes(self.boxes[first:first + count], basis, origin)
        self.transformed = True

    def build(self, resolution, first=0, count=None, min_pass_through=2, occupancy_threshold=0.1):
        """kp_occupancy_create over scans [first, first + count): dict(width, height, stride, offset, cells, passes, hits)"""
        count = len(self.counts) - first if count is None else count
        lo = self.start[first]
        rec = H.scan_records(self.ranges[lo:self.start[first + count]], self.points[lo:self.start[first + count]],
                             self.counts[first:first + count],
                             np.column_stack([self.sensor[first:first + count], np.zeros(count)]))
        if self.transformed:
            anchors = np.zeros(2 * count, dtype=H.SCAN_DTYPE)
            anchors["ranges"] = rec["ranges"][0]
            anchors["points_xy"] = rec["points_xy"][0]
            b = self.boxes[first:first + count]
            anchors["sensor_pose"][0::2, :2] = b[:, :2]
            anchors["sensor_pose"][1::2, :2] = b[:, 2:]
            rec = np.concatenate([anchors, rec])
        return H.port_occupancy(rec, resolution, self.rt, min_pass_through, occupancy_threshold)
