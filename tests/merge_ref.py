"""ctypes binding of oracle/_ref/libmerge_b200.so (oracle/merge.mk): the UNMODIFIED reference karto_sdk with
oracle/ref_driver.cpp, the tool's transformScan restated with Karto's setters (oracle/merge_ref_driver.cpp) and the
map-merge binding's driver (integration/merge_maps_driver.cpp), all in one library so that the reference's scans and the
binding share one karto::SensorManager."""
from __future__ import annotations

import ctypes as C
import os
import time

import numpy as np

import helpers as H

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libmerge_b200.so")
_DP = C.POINTER(C.c_double)
_lib = None


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        L.kref_init_laser.restype = C.c_int
        L.kref_init_laser.argtypes = [C.c_double] * 6
        L.kref_scan_create.restype = C.c_void_p
        L.kref_scan_create.argtypes = [_DP, C.c_int, _DP, C.c_int]
        L.kref_scan_destroy.argtypes = [C.c_void_p]
        L.kref_scan_points.restype = C.c_int
        L.kref_scan_points.argtypes = [C.c_void_p, _DP, C.c_int]
        L.kref_scan_sensor_pose.argtypes = [C.c_void_p, _DP]
        L.kref_transform_scan.argtypes = [C.c_void_p, _DP, _DP]
        L.kref_scan_box.argtypes = [C.c_void_p, _DP]
        L.kref_occupancy_create.restype = C.c_void_p
        L.kref_occupancy_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_double, C.c_int, C.c_double]
        L.kref_occupancy_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), _DP]
        L.kref_occupancy_copy.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.kref_occupancy_destroy.argtypes = [C.c_void_p]
        L.kmm_store_create.restype = C.c_void_p
        L.kmm_store_create.argtypes = [C.c_double]
        L.kmm_store_destroy.argtypes = [C.c_void_p]
        L.kmm_add_submap.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
        L.kmm_apply.argtypes = [C.c_void_p, C.c_int, _DP, _DP]
        L.kmm_merge.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_int), _DP, C.POINTER(C.c_uint8), C.c_long]
        L.kref_init_laser(*(H.LASER[k] for k in ("min_angle", "max_angle", "ang_res", "min_range", "max_range", "range_threshold")))
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(_DP)


class Scan:
    """a karto::LocalizedRangeScan of the standard laser"""

    def __init__(self, ranges, pose, uid=0):
        r = np.ascontiguousarray(ranges, dtype=np.float64)
        p = np.ascontiguousarray(pose, dtype=np.float64)
        self.n = len(r)
        self.h = lib().kref_scan_create(_dp(r), len(r), _dp(p), uid)

    def points(self):
        out = np.empty((self.n, 2))
        n = lib().kref_scan_points(self.h, _dp(out), self.n)
        return out[:n]

    def sensor_pose(self):
        out = np.empty(3)
        lib().kref_scan_sensor_pose(self.h, _dp(out))
        return out

    def transform(self, basis, origin):
        """MergeMapsKinematic::transformScan with tf2's basis (3x3) and origin (3)"""
        b = np.ascontiguousarray(basis, dtype=np.float64).reshape(9)
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        lib().kref_transform_scan(self.h, _dp(b), _dp(o))

    def box(self):
        """the stored bounding box {min x, min y, max x, max y}"""
        out = np.empty(4)
        lib().kref_scan_box(self.h, _dp(out))
        return out

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.kref_scan_destroy(self.h)
            self.h = None


def scans(ranges, poses, uid0=0):
    return [Scan(r, p, uid0 + i) for i, (r, p) in enumerate(zip(np.atleast_2d(ranges), np.atleast_2d(poses)))]


def _ptrs(objs):
    return (C.c_void_p * max(1, len(objs)))(*[o.h for o in objs])


def occupancy(scan_list, resolution, counters=True):
    """the reference's OccupancyGrid::CreateFromScans (defaults 2 / 0.1): dict(width, height, stride, offset, cells,
    passes, hits, seconds), None for no scans"""
    t = time.perf_counter()
    h = lib().kref_occupancy_create(_ptrs(scan_list), len(scan_list), float(resolution), -1, -1.0)
    dt = time.perf_counter() - t
    if not h:
        return None
    info = (C.c_int * 3)()
    off = np.zeros(2)
    lib().kref_occupancy_info(h, info, _dp(off))
    w, hh, st = info[0], info[1], info[2]
    cells = np.zeros((hh, st), dtype=np.uint8)
    ps = np.zeros((hh, st), dtype=np.uint32) if counters else None
    ht = np.zeros((hh, st), dtype=np.uint32) if counters else None
    lib().kref_occupancy_copy(h, cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                              ps.ctypes.data_as(C.POINTER(C.c_uint32)) if counters else None,
                              ht.ctypes.data_as(C.POINTER(C.c_uint32)) if counters else None)
    lib().kref_occupancy_destroy(h)
    return dict(width=w, height=hh, stride=st, offset=off, cells=cells, passes=ps, hits=ht, seconds=dt)


class SubmapStore:
    """karto::b200::SubmapStore (integration/merge_maps_b200.hpp) on Scan objects"""

    def __init__(self, resolution):
        self.h = lib().kmm_store_create(float(resolution))

    def add_submap(self, scan_list):
        return lib().kmm_add_submap(self.h, _ptrs(scan_list), len(scan_list), None, None, None, 0)

    def apply(self, sid, basis, origin):
        b = np.ascontiguousarray(basis, dtype=np.float64).reshape(9)
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        return lib().kmm_apply(self.h, int(sid), _dp(b), _dp(o))

    def merge(self, resolution, cap):
        """(info [width, height, stride], offset [2], cells bytes) or None"""
        info, off = (C.c_int * 3)(), np.zeros(2)
        cells = np.zeros(cap, dtype=np.uint8)
        if lib().kmm_merge(self.h, float(resolution), info, _dp(off), cells.ctypes.data_as(C.POINTER(C.c_uint8)), cap) != 0:
            return None
        return list(info), off, cells

    def close(self):
        if self.h:
            lib().kmm_store_destroy(self.h)
            self.h = None
