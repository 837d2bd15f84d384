"""ORACLE (test infrastructure): ctypes binding of oracle/karto_port.c."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import REF_DIR, build

_lib = None


class KpParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "search_size", "resolution", "smear_deviation", "range_threshold",
        "coarse_search_angle_offset", "coarse_angle_resolution", "fine_search_angle_offset",
        "distance_variance_penalty", "angle_variance_penalty", "minimum_distance_penalty",
        "minimum_angle_penalty")] + [("use_response_expansion", C.c_int32)]


class KpScan(C.Structure):
    _fields_ = [("n", C.c_int32), ("ranges", C.POINTER(C.c_double)), ("points_xy", C.POINTER(C.c_double)),
                ("sensor_pose", C.c_double * 3)]


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(REF_DIR, "libkarto_port.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        L.kp_create.restype = C.c_void_p
        L.kp_create.argtypes = [C.POINTER(KpParams)]
        L.kp_destroy.argtypes = [C.c_void_p]
        L.kp_match.restype = C.c_double
        L.kp_match.argtypes = [C.c_void_p, C.POINTER(KpScan), C.POINTER(KpScan), C.c_int32, C.c_int32, C.c_int32,
                               C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.kp_raster.argtypes = [C.c_void_p, C.POINTER(KpScan), C.POINTER(KpScan), C.c_int32]
        L.kp_correlate.restype = C.c_double
        L.kp_correlate.argtypes = [C.c_void_p, C.POINTER(KpScan)] + [C.POINTER(C.c_double)] * 3 + \
            [C.c_double, C.c_double, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double),
             C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32)]
        L.kp_find_valid_points.restype = C.c_int32
        L.kp_find_valid_points.argtypes = [C.POINTER(KpScan), C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.kp_offsets.restype = C.c_int32
        L.kp_offsets.argtypes = [C.c_void_p, C.POINTER(KpScan), C.c_double, C.c_double, C.c_double, C.POINTER(C.c_int32)]
        L.kp_grid.restype = C.POINTER(C.c_uint8)
        L.kp_grid.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_double)]
        L.kp_kernel.restype = C.POINTER(C.c_uint8)
        L.kp_kernel.argtypes = [C.c_void_p]
        L.kp_point_readings.argtypes = [C.POINTER(C.c_double), C.c_int32, C.POINTER(C.c_double), C.c_double, C.c_double,
                                        C.POINTER(C.c_double)]
        L.kp_occupancy_create.restype = C.c_void_p
        L.kp_occupancy_create.argtypes = [C.POINTER(KpScan), C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double,
                                          C.c_uint32, C.c_double]
        L.kp_occupancy_destroy.argtypes = [C.c_void_p]
        L.kp_occupancy_info.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_double)]
        for f, t in (("cells", C.c_uint8), ("pass", C.c_uint32), ("hits", C.c_uint32)):
            getattr(L, "kp_occupancy_" + f).restype = C.POINTER(t)
            getattr(L, "kp_occupancy_" + f).argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def point_readings(ranges, sensor_pose, minimum_angle, angular_resolution):
    r = np.ascontiguousarray(ranges, dtype=np.float64)
    sp = np.ascontiguousarray(sensor_pose, dtype=np.float64)
    out = np.empty((len(r), 2), dtype=np.float64)
    lib().kp_point_readings(_dp(r), len(r), _dp(sp), minimum_angle, angular_resolution, _dp(out))
    return out


class PortScan:
    """Keeps the numpy buffers alive behind a kp_scan."""

    def __init__(self, ranges, sensor_pose, minimum_angle, angular_resolution):
        self.ranges = np.ascontiguousarray(ranges, dtype=np.float64)
        self.pose = np.ascontiguousarray(sensor_pose, dtype=np.float64)
        self.points = point_readings(self.ranges, self.pose, minimum_angle, angular_resolution)
        self.c = KpScan(len(self.ranges), _dp(self.ranges), _dp(self.points), (C.c_double * 3)(*self.pose))


def scan_array(scans):
    arr = (KpScan * max(1, len(scans)))()
    for i, s in enumerate(scans):
        arr[i] = s.c
    return arr


class PortMatcher:
    def __init__(self, **kw):
        self.params = KpParams(**kw)
        self.h = lib().kp_create(C.byref(self.params))
        if not self.h:
            raise ValueError("kp_create returned NULL (invalid parameters)")

    def close(self):
        if self.h:
            lib().kp_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def match(self, query, base, do_penalize=True, do_refine=True):
        mean = np.zeros(3)
        cov = np.zeros(9)
        arr = scan_array(base)
        r = lib().kp_match(self.h, C.byref(query.c), arr, len(base), int(do_penalize), int(do_refine), _dp(mean), _dp(cov))
        return r, mean, cov.reshape(3, 3)

    def raster(self, query, base):
        arr = scan_array(base)
        lib().kp_raster(self.h, C.byref(query.c), arr, len(base))

    def grid(self):
        info = (C.c_int32 * 9)()
        off = (C.c_double * 2)()
        p = lib().kp_grid(self.h, info, off)
        info = list(info)
        data = np.ctypeslib.as_array(p, shape=(info[7],)).copy()
        return dict(width=info[0], height=info[1], stride=info[2], roi=(info[3], info[4], info[5], info[6]),
                    data_size=info[7], kernel_size=info[8], offset=(off[0], off[1]), data=data)

    def kernel(self):
        k = self.grid()["kernel_size"]
        return np.ctypeslib.as_array(lib().kp_kernel(self.h), shape=(k * k,)).copy().reshape(k, k)

    def offsets(self, query, angle_center, angle_offset, angle_res):
        n_angles = int(np.floor(angle_offset * 2.0 / angle_res + 0.5)) + 1
        out = np.empty((n_angles, query.c.n), dtype=np.int32)
        na = lib().kp_offsets(self.h, C.byref(query.c), angle_center, angle_offset, angle_res,
                              out.ctypes.data_as(C.POINTER(C.c_int32)))
        assert na == n_angles
        return out

    def correlate(self, query, center, sp_off, sp_res, ang_off, ang_res, do_penalize, fine, cov=None, want_sums=True):
        mean = np.zeros(3)
        cov = np.zeros(9) if cov is None else np.ascontiguousarray(cov, dtype=np.float64).reshape(9).copy()
        c = np.ascontiguousarray(center, dtype=np.float64)
        o = np.ascontiguousarray(sp_off, dtype=np.float64)
        rs = np.ascontiguousarray(sp_res, dtype=np.float64)
        dims = (C.c_int32 * 3)()
        cap = 1 << 22
        sums = np.zeros(cap, dtype=np.int32) if want_sums else None
        r = lib().kp_correlate(self.h, C.byref(query.c), _dp(c), _dp(o), _dp(rs), ang_off, ang_res, int(do_penalize),
                               int(fine), _dp(mean), _dp(cov),
                               sums.ctypes.data_as(C.POINTER(C.c_int32)) if want_sums else None, cap if want_sums else 0, dims)
        nx, ny, na = dims[0], dims[1], dims[2]
        vol = sums[:nx * ny * na].reshape(ny, nx, na).copy() if want_sums else None
        return r, mean, cov.reshape(3, 3), vol


def find_valid_points(scan, viewpoint):
    vp = np.ascontiguousarray(viewpoint, dtype=np.float64)
    out = np.empty((scan.c.n, 2), dtype=np.float64)
    n = lib().kp_find_valid_points(C.byref(scan.c), _dp(vp), _dp(out))
    return out[:n].copy()


def occupancy(scans, resolution, range_threshold, minimum_range, maximum_range, min_pass_through=2,
              occupancy_threshold=0.1):
    """kp_occupancy_create on PortScan objects; same dict as oracle.karto_ref.occupancy (None when empty)."""
    return occupancy_array(scan_array(scans), len(scans), resolution, range_threshold, minimum_range, maximum_range,
                           min_pass_through, occupancy_threshold)


def occupancy_array(arr, n, resolution, range_threshold, minimum_range, maximum_range, min_pass_through=2,
                    occupancy_threshold=0.1):
    """kp_occupancy_create on n KpScan records at arr (a KpScan array or pointer): dict(width, height, stride, offset,
    cells, passes, hits, seconds), None when n is 0.  seconds is the host time of kp_occupancy_create."""
    import time
    t = time.perf_counter()
    h = lib().kp_occupancy_create(arr, n, resolution, range_threshold, minimum_range, maximum_range, min_pass_through,
                                  occupancy_threshold)
    dt = time.perf_counter() - t
    if not h:
        return None
    info = (C.c_int32 * 3)()
    off = np.zeros(2)
    lib().kp_occupancy_info(h, info, _dp(off))
    w, hh, st = info[0], info[1], info[2]
    n = hh * st
    def grab(fn, dt_):
        p = fn(h)
        return np.ctypeslib.as_array(p, shape=(max(n, 1),))[:n].reshape(hh, st).astype(dt_, copy=True)
    out = dict(width=w, height=hh, stride=st, offset=off, cells=grab(lib().kp_occupancy_cells, np.uint8),
               passes=grab(lib().kp_occupancy_pass, np.uint32), hits=grab(lib().kp_occupancy_hits, np.uint32), seconds=dt)
    lib().kp_occupancy_destroy(h)
    return out
