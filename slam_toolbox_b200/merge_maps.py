"""slam_toolbox's map-merge tool (MergeMapsKinematic, src/merge_maps_kinematic.cpp) on the GPU occupancy grid.

The submaps' scans stay resident in one device store (api.OccupancyGrid).  Moving a submap's marker composes its correction
on the host; a merge applies every submap's accumulated correction to its scans on the device (in place: each merge
corrects the already corrected scans again, as the tool's transformScan does to the scans it keeps) and builds one grid.

Parity contract: given a correction's tf2 basis and origin, the merged grid (width, height, offset, cells, counters) equals
the reference's transformScan + OccupancyGrid::CreateFromScans bit for bit.  The composition of the corrections in
MoveSubmap restates tf2's quaternion and matrix arithmetic in FP64 on the host; tf2 itself is not available to test that
composition against, so a caller that holds tf2 transforms should pass their basis and origin to TransformScans directly.

    mm = MergeMapsKinematic(resolution=0.05, laser=laser)
    sid, nav, origin = mm.AddSubmap(block)       # addSubmapCallback: the submap's own grid and its re-centred origin
    mm.MoveSubmap(sid, x, y, yaw)                # processInteractiveFeedback, MOUSE_UP
    grid = mm.Merge()                            # mergeMapCallback -> api.OccupancyGrid of all submaps
"""
from __future__ import annotations

import math

import numpy as np

from . import api


class Transform:
    """tf2::Transform restated in FP64: basis (3, 3) and origin (3,), with tf2's operation order."""

    def __init__(self, basis=None, origin=None):
        self.basis = np.eye(3) if basis is None else np.array(basis, dtype=np.float64).reshape(3, 3)
        self.origin = np.zeros(3) if origin is None else np.array(origin, dtype=np.float64).reshape(3)

    @staticmethod
    def from_quaternion(q, origin) -> "Transform":
        """tf2::Matrix3x3::setRotation (x, y, z, w)"""
        x, y, z, w = (float(v) for v in q)
        d = x * x + y * y + z * z + w * w
        s = 2.0 / d
        xs, ys, zs = x * s, y * s, z * s
        wx, wy, wz = w * xs, w * ys, w * zs
        xx, xy, xz = x * xs, x * ys, x * zs
        yy, yz, zz = y * ys, y * zs, z * zs
        b = [[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]]
        return Transform(b, origin)

    @staticmethod
    def _dot(a, b):
        return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]

    def apply(self, v):
        """operator()(Vector3): basis row dot products, then + origin"""
        b = self.basis.tolist()
        return np.array([self._dot(b[r], [float(x) for x in v]) + float(self.origin[r]) for r in range(3)])

    def __mul__(self, t: "Transform") -> "Transform":
        a, c = self.basis.tolist(), t.basis.tolist()
        m = [[self._dot(a[r], [c[0][k], c[1][k], c[2][k]]) for k in range(3)] for r in range(3)]
        return Transform(m, self.apply(t.origin))

    def inverse(self) -> "Transform":
        inv = Transform(self.basis.T.copy())
        neg = [-float(v) for v in self.origin]
        b = inv.basis.tolist()
        inv.origin = np.array([self._dot(b[r], neg) for r in range(3)])
        return inv


def quaternion_yaw(yaw: float):
    """the (x, y, z, w) quaternion of a marker pose turned by yaw about z"""
    return (0.0, 0.0, math.sin(0.5 * yaw), math.cos(0.5 * yaw))


class MergeMapsKinematic:
    """The tool's state: submaps (scan ranges of one resident store), their marker locations and accumulated corrections."""

    def __init__(self, resolution: float = 0.05, laser: api.LaserRangeFinder | None = None):
        self.resolution = float(resolution)
        self.grid = api.OccupancyGrid(resolution, laser)
        self.ranges: dict[int, tuple[int, int]] = {}       # id -> (first scan, count)
        self.locations: dict[int, np.ndarray] = {}         # submap_locations_: x, y, accumulated yaw
        self.corrections: dict[int, Transform] = {}        # submap_marker_transform_

    def AddSubmap(self, block: api.ScanBlock, laser=None):
        """addSubmapCallback (:105-140): stores the scans, builds the submap's own grid from the shared store.  Returns
        (id, nav map [height, width] int8, (x, y) of the submap frame) with the frame at the grid's centre (:115-122).
        laser = the submap's own laser (each pose-graph file brings its own; a per-scan sequence is accepted too), None =
        the tool's default laser given to the constructor."""
        first = self.grid.NumScans()
        self.grid.AddScans(block, laser)
        sid = len(self.ranges) + 1
        self.ranges[sid] = (first, len(block))
        self.grid.Build(first, len(block))
        nav = self.grid.toNavMap()
        w, h, off = self.grid.GetWidth(), self.grid.GetHeight(), self.grid.GetOffset()
        cx = off[0] + w * self.resolution / 2.0
        cy = off[1] + h * self.resolution / 2.0
        self.locations[sid] = np.array([cx, cy, 0.0])
        self.corrections[sid] = Transform()
        return sid, nav, (cx, cy)

    def MoveSubmap(self, sid: int, x: float, y: float, yaw: float):
        """processInteractiveFeedback on MOUSE_UP (:313-352): the marker of submap sid released at (x, y) turned by yaw
        (relative); correction = correction * previous_location^-1 * new_location."""
        q = quaternion_yaw(yaw)
        prev = Transform(origin=[self.locations[sid][0], self.locations[sid][1], 0.0])
        self.locations[sid] = np.array([float(x), float(y), self.locations[sid][2] + math.atan2(
            2.0 * q[3] * q[2], 1.0 - 2.0 * q[2] * q[2])])
        new = Transform.from_quaternion(q, [float(x), float(y), 0.0])
        self.corrections[sid] = self.corrections[sid] * prev.inverse() * new

    def Merge(self) -> api.OccupancyGrid:
        """mergeMapCallback (:251-291): every submap's accumulated correction applied to its resident scans, then one
        grid over all of them"""
        for sid, (first, count) in self.ranges.items():
            t = self.corrections[sid]
            self.grid.TransformScans(first, count, t.basis, t.origin)
        return self.grid.Build()
