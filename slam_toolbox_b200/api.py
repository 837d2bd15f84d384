"""Host-side mirror of the reference interface for the hot path, over the C ABI (ctypes).

The names follow karto (lib/karto_sdk/include/karto_sdk/{Karto,Mapper}.h) and
solver_plugins::CeresSolver (solvers/ceres_solver.hpp) so that the parity tests read like
calls into the reference:

    ScanMatcher.Create(mapper_params, searchSize, resolution, smearDeviation, rangeThreshold)
    ScanMatcher.MatchScan(scan, baseScans, doPenalize, doRefineMatch) -> (response, mean, cov)
    ScanSolver.AddNode / AddConstraint / Compute / GetCorrections / ...

Every call goes through include/b200slam.h into libb200slam.so; there is no Python or CPU
implementation of the path here, and importing fails loudly if the library is missing.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np

from . import build as _build

_DP = C.POINTER(C.c_double)
_IP = C.POINTER(C.c_int32)
_lib = None

OK, ERR_INVALID_ARG, ERR_CUDA, ERR_UNSUPPORTED, ERR_NOT_FOUND, ERR_NUMERIC = range(6)


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200slam error {code}: {msg}")
        self.code = code


class SmParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "search_size", "resolution", "smear_deviation", "range_threshold",
        "coarse_search_angle_offset", "coarse_angle_resolution", "fine_search_angle_offset",
        "distance_variance_penalty", "angle_variance_penalty", "minimum_distance_penalty",
        "minimum_angle_penalty")] + [("use_response_expansion", C.c_int32)]


class CScan(C.Structure):
    _fields_ = [("n", C.c_int32), ("ranges", _DP), ("points_xy", _DP), ("sensor_pose", C.c_double * 3)]


class PgOpts(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("parameter_tolerance", C.c_double), ("min_relative_decrease", C.c_double),
                ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double), ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double),
                ("jacobi_scaling", C.c_int32), ("use_nonmonotonic_steps", C.c_int32),
                ("max_consecutive_nonmonotonic_steps", C.c_int32), ("max_num_consecutive_invalid_steps", C.c_int32),
                ("pcg_tolerance", C.c_double), ("pcg_max_iterations", C.c_int32),
                ("loss_function", C.c_int32), ("loss_scale", C.c_double),
                ("trust_region_strategy", C.c_int32), ("dogleg_type", C.c_int32), ("linear_solver_type", C.c_int32)]


class OgParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("range_threshold", C.c_double), ("minimum_range", C.c_double),
                ("maximum_range", C.c_double), ("min_pass_through", C.c_uint32), ("occupancy_threshold", C.c_double)]


class OgInfo(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32), ("offset", C.c_double * 2)]


class PgSummary(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("successful_steps", C.c_int32), ("pcg_iterations", C.c_int32),
                ("termination", C.c_int32), ("usable", C.c_int32), ("initial_cost", C.c_double), ("final_cost", C.c_double),
                ("solve_ms", C.c_float), ("kernel_launches", C.c_int64),
                ("setup_ms", C.c_float), ("wall_ms", C.c_float), ("uploaded_edges", C.c_int32), ("linear_solver", C.c_int32),
                ("linear_solves", C.c_int32)]


def library_path() -> str:
    return _build.LIB


def lib():
    """Loads libb200slam.so (building it in-tree first if the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if not os.path.exists(path) or os.environ.get("B200SLAM_REBUILD"):
        _build.build()
    L = C.CDLL(path)
    L.b200_last_error.restype = C.c_char_p
    L.b200_set_device.argtypes = [C.c_int]
    L.b200_point_readings.argtypes = [_DP, C.c_int32, _DP, C.c_double, C.c_double, _DP]
    L.b200sm_create.argtypes = [C.POINTER(SmParams), C.POINTER(C.c_void_p)]
    L.b200sm_destroy.argtypes = [C.c_void_p]
    L.b200sm_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    L.b200sm_match.argtypes = [C.c_void_p, C.POINTER(CScan), C.POINTER(CScan), C.c_int32, C.c_int32, C.c_int32, _DP, _DP, _DP]
    L.b200sm_raster.argtypes = [C.c_void_p, C.POINTER(CScan), C.POINTER(CScan), C.c_int32]
    L.b200sm_correlate.argtypes = [C.c_void_p, C.POINTER(CScan), _DP, _DP, _DP, C.c_double, C.c_double, C.c_int32, C.c_int32,
                                   _DP, _DP, _DP, _IP, C.c_int32, _IP]
    L.b200sm_grid_info.argtypes = [C.c_void_p, _IP, _DP]
    L.b200sm_grid_copy.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_int32]
    L.b200sm_match_batch.argtypes = [C.c_void_p, C.POINTER(CScan), C.c_int32, C.POINTER(CScan), C.c_int32, _IP, C.c_int32,
                                     _IP, _IP, C.c_int32, C.c_int32, C.c_int32, _DP, _DP, _DP]
    L.b200sm_batch_upload.argtypes = [C.c_void_p, C.POINTER(CScan), C.c_int32, C.POINTER(CScan), C.c_int32, _IP, C.c_int32,
                                      _IP, _IP, C.c_int32, C.c_int32]
    L.b200sm_batch_run.argtypes = [C.c_void_p]
    L.b200sm_batch_fetch.argtypes = [C.c_void_p, _DP, _DP, _DP]
    L.b200sm_batch_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.b200sm_batch_best.argtypes = [C.c_void_p, _IP, _IP, _IP]
    L.b200sm_batch_info.argtypes = [C.c_void_p, _IP]
    L.b200sm_batch_winner_record_bytes.restype = C.c_int32
    L.b200sm_batch_winner_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.b200sm_batch_winners_select.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int64), _DP, _DP, _DP]
    L.b200sm_batch_tile_info.argtypes = [C.c_void_p, _IP]
    L.b200sm_batch_tile_stats.argtypes = [C.c_void_p, _IP]
    L.b200sm_batch_tile_layout.argtypes = [C.c_void_p, _IP]
    L.b200sm_batch_fetch_stats.argtypes = [C.c_void_p, _IP]
    L.b200sm_batch_upload_timing.argtypes = [C.c_void_p, _DP]
    L.b200sm_batch_reduce_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.b200sm_batch_transfer_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int32]
    L.b200sm_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int32]
    L.b200sm_match_timing.argtypes = [C.c_void_p, _DP, C.c_int32]
    L.b200sm_launch_count.restype = C.c_int64
    L.b200sm_launch_count.argtypes = [C.c_void_p]
    if hasattr(L, "b200pg_create"):
        L.b200pg_default_opts.argtypes = [C.POINTER(PgOpts)]
        L.b200pg_create.argtypes = [C.POINTER(PgOpts), C.POINTER(C.c_void_p)]
        L.b200pg_destroy.argtypes = [C.c_void_p]
        L.b200pg_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        L.b200pg_reset.argtypes = [C.c_void_p]
        L.b200pg_clear.argtypes = [C.c_void_p]
        L.b200pg_add_node.argtypes = [C.c_void_p, C.c_int32, _DP]
        L.b200pg_add_edge.argtypes = [C.c_void_p, C.c_int32, C.c_int32, _DP, _DP]
        L.b200pg_remove_node.argtypes = [C.c_void_p, C.c_int32]
        L.b200pg_remove_edge.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.b200pg_modify_node.argtypes = [C.c_void_p, C.c_int32, _DP]
        L.b200pg_get_node.argtypes = [C.c_void_p, C.c_int32, _DP]
        L.b200pg_num_nodes.argtypes = [C.c_void_p]
        L.b200pg_num_edges.argtypes = [C.c_void_p]
        L.b200pg_solve.argtypes = [C.c_void_p, C.POINTER(PgSummary)]
        L.b200pg_get_corrections.argtypes = [C.c_void_p, _IP, _DP, C.c_int32]
        L.b200pg_cholesky_analyze.argtypes = [C.c_int32, C.c_int32, _IP, C.c_int32, C.POINTER(C.c_int64), _IP, C.c_int32]
        L.b200pg_factor_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.b200og_default_params.argtypes = [C.POINTER(OgParams)]
    L.b200og_create.argtypes = [C.POINTER(OgParams), C.POINTER(C.c_void_p)]
    L.b200og_destroy.argtypes = [C.c_void_p]
    L.b200og_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    L.b200og_add_scans.argtypes = [C.c_void_p, C.POINTER(CScan), C.c_int32]
    L.b200og_clear_scans.argtypes = [C.c_void_p]
    L.b200og_num_scans.argtypes = [C.c_void_p]
    L.b200og_build.argtypes = [C.c_void_p, C.POINTER(OgInfo)]
    L.b200og_fetch.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.b200og_fetch_nav.argtypes = [C.c_void_p, C.POINTER(C.c_int8)]
    L.b200og_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.b200og_launch_count.restype = C.c_int64
    L.b200og_launch_count.argtypes = [C.c_void_p]
    L.b200og_create_from_scans.argtypes = [C.POINTER(OgParams), C.POINTER(CScan), C.c_int32, C.POINTER(OgInfo),
                                           C.POINTER(C.c_void_p)]
    _lib = L
    return L


def _check(rc: int):
    if rc != OK:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))


def _dp(a):
    return a.ctypes.data_as(_DP)


def _ip(a):
    return a.ctypes.data_as(_IP) if a is not None else None


@dataclass
class LaserRangeFinder:
    """The fields of karto::LaserRangeFinder (Karto.h:3874-4368) the path reads."""
    minimum_angle: float = math.radians(-135.0)
    maximum_angle: float = math.radians(135.0)
    angular_resolution: float = math.radians(0.25)
    minimum_range: float = 0.1
    maximum_range: float = 30.0
    range_threshold: float = 12.0


def point_readings(ranges: np.ndarray, sensor_poses: np.ndarray, laser: LaserRangeFinder) -> np.ndarray:
    """LocalizedRangeScan::Update for a (S, n) block of scans -> (S, n, 2) unfiltered points."""
    r = np.ascontiguousarray(np.atleast_2d(ranges), dtype=np.float64)
    p = np.ascontiguousarray(np.atleast_2d(sensor_poses), dtype=np.float64)
    out = np.empty(r.shape + (2,), dtype=np.float64)
    for s in range(r.shape[0]):
        _check(lib().b200_point_readings(_dp(r[s]), r.shape[1], _dp(p[s]), laser.minimum_angle, laser.angular_resolution,
                                         _dp(out[s])))
    return out


class ScanBlock:
    """A contiguous block of scans (ranges, unfiltered points, sensor poses) plus the b200_scan
    array pointing into it -- the flattened form of a LocalizedRangeScanVector."""

    def __init__(self, ranges, sensor_poses, laser: LaserRangeFinder, points=None):
        self.ranges = np.ascontiguousarray(np.atleast_2d(ranges), dtype=np.float64)
        self.poses = np.ascontiguousarray(np.atleast_2d(sensor_poses), dtype=np.float64)
        self.points = point_readings(self.ranges, self.poses, laser) if points is None else \
            np.ascontiguousarray(points, dtype=np.float64).reshape(self.ranges.shape + (2,))
        self.laser = laser
        S, n = self.ranges.shape
        self.c = (CScan * max(S, 1))()
        rb, pb = self.ranges.ctypes.data, self.points.ctypes.data
        for s in range(S):
            self.c[s].n = n
            self.c[s].ranges = C.cast(rb + s * n * 8, _DP)
            self.c[s].points_xy = C.cast(pb + s * n * 16, _DP)
            self.c[s].sensor_pose = (C.c_double * 3)(*self.poses[s])

    def __len__(self):
        return self.ranges.shape[0]


@dataclass
class MapperParams:
    """The karto::Mapper parameters ScanMatcher reads at match time (Mapper.cpp:590-594, 626-627,
    675-682), with the toolbox/YAML names; the two variance penalties are squared on the way in
    exactly like Mapper::setParamDistanceVariancePenalty / AngleVariancePenalty (Mapper.cpp:2562-2570)."""
    coarse_search_angle_offset: float = math.radians(20.0)
    coarse_angle_resolution: float = math.radians(2.0)
    fine_search_angle_offset: float = math.radians(0.2)
    distance_variance_penalty: float = 0.5
    angle_variance_penalty: float = 1.0
    minimum_distance_penalty: float = 0.5
    minimum_angle_penalty: float = 0.9
    use_response_expansion: bool = False


class ScanMatcher:
    """karto::ScanMatcher (Mapper.h:1322-1544) on the GPU."""

    def __init__(self, handle, params):
        self._h = handle
        self.params = params

    @staticmethod
    def Create(mapper: MapperParams, searchSize: float, resolution: float, smearDeviation: float,
               rangeThreshold: float) -> "ScanMatcher":
        p = SmParams(searchSize, resolution, smearDeviation, rangeThreshold, mapper.coarse_search_angle_offset,
                     mapper.coarse_angle_resolution, mapper.fine_search_angle_offset,
                     mapper.distance_variance_penalty * mapper.distance_variance_penalty,
                     mapper.angle_variance_penalty * mapper.angle_variance_penalty,
                     mapper.minimum_distance_penalty, mapper.minimum_angle_penalty, int(mapper.use_response_expansion))
        h = C.c_void_p()
        _check(lib().b200sm_create(C.byref(p), C.byref(h)))
        return ScanMatcher(h, p)

    def close(self):
        if self._h:
            lib().b200sm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int):
        _check(lib().b200sm_set_stream(self._h, C.c_void_p(cuda_stream)))

    # --- single match -------------------------------------------------------------------------
    def MatchScan(self, scan: ScanBlock, baseScans: ScanBlock | None, doPenalize: bool = True, doRefineMatch: bool = True,
                  scan_index: int = 0):
        mean, cov, resp = np.zeros(3), np.zeros(9), C.c_double()
        nb = len(baseScans) if baseScans is not None else 0
        _check(lib().b200sm_match(self._h, C.byref(scan.c[scan_index]), baseScans.c if nb else None, nb, int(doPenalize),
                                  int(doRefineMatch), _dp(mean), _dp(cov), C.byref(resp)))
        return resp.value, mean, cov.reshape(3, 3)

    def raster(self, scan: ScanBlock, baseScans: ScanBlock, scan_index: int = 0):
        _check(lib().b200sm_raster(self._h, C.byref(scan.c[scan_index]), baseScans.c, len(baseScans)))

    def CorrelateScan(self, scan: ScanBlock, searchCenter, searchSpaceOffset, searchSpaceResolution, searchAngleOffset,
                      searchAngleResolution, doPenalize, doingFineMatch, cov=None, scan_index: int = 0):
        """Returns (response, mean, cov, integer volume [nY, nX, nAngles])."""
        mean = np.zeros(3)
        cov = np.zeros(9) if cov is None else np.ascontiguousarray(cov, dtype=np.float64).reshape(9).copy()
        c = np.ascontiguousarray(searchCenter, dtype=np.float64)
        o = np.ascontiguousarray(searchSpaceOffset, dtype=np.float64)
        r = np.ascontiguousarray(searchSpaceResolution, dtype=np.float64)
        cap = 1 << 22
        sums = np.zeros(cap, dtype=np.int32)
        dims = (C.c_int32 * 3)()
        resp = C.c_double()
        _check(lib().b200sm_correlate(self._h, C.byref(scan.c[scan_index]), _dp(c), _dp(o), _dp(r), searchAngleOffset,
                                      searchAngleResolution, int(doPenalize), int(doingFineMatch), _dp(mean), _dp(cov),
                                      C.byref(resp), _ip(sums), cap, dims))
        nx, ny, na = dims[0], dims[1], dims[2]
        return resp.value, mean, cov.reshape(3, 3), sums[:nx * ny * na].reshape(ny, nx, na).copy()

    def GetCorrelationGrid(self):
        info = (C.c_int32 * 9)()
        off = np.zeros(2)
        _check(lib().b200sm_grid_info(self._h, info, _dp(off)))
        info = list(info)
        data = np.empty(info[7], dtype=np.uint8)
        _check(lib().b200sm_grid_copy(self._h, data.ctypes.data_as(C.POINTER(C.c_uint8)), info[7]))
        return dict(width=info[0], height=info[1], stride=info[2], roi=(info[3], info[4], info[5], info[6]),
                    data_size=info[7], kernel_size=info[8], offset=(off[0], off[1]), data=data)

    # --- batched sweep ------------------------------------------------------------------------
    def _pairs(self, pairs):
        if pairs is None:
            return None, None, 0
        pq = np.ascontiguousarray(pairs[0], dtype=np.int32)
        pc = np.ascontiguousarray(pairs[1], dtype=np.int32)
        return pq, pc, len(pq)

    def MatchScanBatch(self, queries: ScanBlock, candidates: ScanBlock, chain_start, pairs=None, doPenalize=False,
                       doRefineMatch=False):
        """MatchScan for every (query, candidate chain) pair. Returns (response[np], mean[np,3], cov[np,3,3])."""
        cs = np.ascontiguousarray(chain_start, dtype=np.int32)
        nch = len(cs) - 1
        pq, pc, npairs = self._pairs(pairs)
        if pq is None:
            npairs = len(queries) * nch
        self._npairs = npairs
        resp, mean, cov = np.zeros(npairs), np.zeros((npairs, 3)), np.zeros((npairs, 9))
        _check(lib().b200sm_match_batch(self._h, queries.c, len(queries), candidates.c, len(candidates), _ip(cs), nch,
                                        _ip(pq), _ip(pc), npairs, int(doPenalize), int(doRefineMatch), _dp(resp), _dp(mean),
                                        _dp(cov)))
        return resp, mean, cov.reshape(npairs, 3, 3)

    def batch_upload(self, queries: ScanBlock, candidates: ScanBlock, chain_start, pairs=None, doPenalize=False):
        cs = np.ascontiguousarray(chain_start, dtype=np.int32)
        nch = len(cs) - 1
        pq, pc, npairs = self._pairs(pairs)
        if pq is None:
            npairs = len(queries) * nch
        self._keep = (queries, candidates, cs, pq, pc)
        self._npairs = npairs
        _check(lib().b200sm_batch_upload(self._h, queries.c, len(queries), candidates.c, len(candidates), _ip(cs), nch,
                                         _ip(pq), _ip(pc), npairs, int(doPenalize)))
        return npairs

    def batch_run(self):
        _check(lib().b200sm_batch_run(self._h))

    def batch_fetch(self):
        n = self._npairs
        resp, mean, cov = np.zeros(n), np.zeros((n, 3)), np.zeros((n, 9))
        _check(lib().b200sm_batch_fetch(self._h, _dp(resp), _dp(mean), _dp(cov)))
        return resp, mean, cov.reshape(n, 3, 3)

    def batch_kernel_ms(self) -> float:
        ms = C.c_float()
        _check(lib().b200sm_batch_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def batch_best(self):
        n = self._npairs
        s, i, t = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        _check(lib().b200sm_batch_best(self._h, _ip(s), _ip(i), _ip(t)))
        return s, i, t

    def batch_reduce_keys(self, device_ptr: int, id_offset: int = 0):
        """Per-query packed best-response keys into a device buffer (see b200sm_batch_reduce_keys)."""
        _check(lib().b200sm_batch_reduce_keys(self._h, C.c_void_p(device_ptr), int(id_offset)))

    @staticmethod
    def winner_record_bytes() -> int:
        return int(lib().b200sm_batch_winner_record_bytes())

    def batch_winner_records(self, device_ptr: int, id_offset: int = 0):
        """This rank's best candidate per query (+ its raw device reduction) into a device buffer of
        n_queries * winner_record_bytes() bytes -- the send buffer of the one all-gather of the multi-GPU sweep."""
        _check(lib().b200sm_batch_winner_records(self._h, C.c_void_p(device_ptr), int(id_offset)))

    def batch_winners_select(self, gathered_device_ptr: int, nranks: int, n_queries: int):
        """Per-query winner over the gathered records of all ranks: (global ids, response, mean[Q,3], cov[Q,3,3])."""
        ids = np.zeros(n_queries, dtype=np.int64)
        resp, mean, cov = np.zeros(n_queries), np.zeros((n_queries, 3)), np.zeros((n_queries, 9))
        _check(lib().b200sm_batch_winners_select(self._h, C.c_void_p(gathered_device_ptr), int(nranks),
                                                 ids.ctypes.data_as(C.POINTER(C.c_int64)), _dp(resp), _dp(mean), _dp(cov)))
        return ids, resp, mean, cov.reshape(n_queries, 3, 3)

    def batch_info(self):
        info = np.zeros(8, dtype=np.int32)
        _check(lib().b200sm_batch_info(self._h, _ip(info)))
        return dict(fast=bool(info[0]), kernel=("generic", "fast", "tile")[int(info[0])], fast_descriptors=int(info[1]), edge_beams=int(info[2]), far_beams=int(info[3]),
                    refused_reason=int(info[4]), ctas=int(info[5]), pairs=int(info[6]), items=int(info[7]))

    def batch_tile_info(self):
        """Plan of the tiled cluster kernel for the uploaded sweep (b200sm_batch_tile_info)."""
        info = np.zeros(8, dtype=np.int32)
        _check(lib().b200sm_batch_tile_info(self._h, _ip(info)))
        lay = np.zeros(4, dtype=np.int32)
        _check(lib().b200sm_batch_tile_layout(self._h, _ip(lay)))
        return dict(available=bool(info[0]), cluster=int(info[1]), chunks=int(info[2]), bands=int(info[3]), band_rows=int(info[4]),
                    refused_reason=int(info[5]), clusters=int(info[6]), smem_kb=int(info[7]), ytile_rows=int(lay[0]),
                    ytiles=int(lay[1]), xtiles=int(lay[2]), tail=bool(lay[3]))

    def batch_tile_stats(self):
        """What the tiled kernel's descriptor blocks hold for the uploaded sweep (b200sm_batch_tile_stats)."""
        st = np.zeros(8, dtype=np.int32)
        _check(lib().b200sm_batch_tile_stats(self._h, _ip(st)))
        return dict(blocks=int(st[0]), sub_blocks=int(st[1]), max_edge_group=int(st[2]), split_groups=int(st[3]),
                    multi_entries=int(st[4]), max_multiplicity=int(st[5]), max_plain_group=int(st[6]), wrap2_entries=int(st[7]))

    def batch_upload_timing(self):
        t = np.zeros(3)
        _check(lib().b200sm_batch_upload_timing(self._h, _dp(t)))
        return dict(lookup_tables_ms=float(t[0]), kernel_tables_ms=float(t[1]), total_ms=float(t[2]))

    def batch_fetch_stats(self):
        st = np.zeros(4, dtype=np.int32)
        _check(lib().b200sm_batch_fetch_stats(self._h, _ip(st)))
        return dict(zero_pairs=int(st[0]), fallback_pairs=int(st[1]), pairs=int(st[2]))

    def transfer_bytes(self, reset: bool = False):
        a, b = C.c_int64(), C.c_int64()
        _check(lib().b200sm_batch_transfer_bytes(self._h, C.byref(a), C.byref(b), int(reset)))
        return a.value, b.value

    def set_option(self, name: str, value: int):
        _check(lib().b200sm_set_option(self._h, name.encode(), int(value)))

    def launch_count(self) -> int:
        return int(lib().b200sm_launch_count(self._h))

    def match_timing(self, reset: bool = False):
        """Per-phase host wall time of the single-match path, averaged per match (ms)."""
        t = np.zeros(6)
        _check(lib().b200sm_match_timing(self._h, _dp(t), int(reset)))
        n = max(t[5], 1.0)
        return dict(valid_points=t[0] / n, raster=t[1] / n, lookup_tables=t[2] / n, volume=t[3] / n, epilogue=t[4] / n, matches=int(t[5]))


FACTOR_INFO = ("columns", "nnz_blocks", "supernodes", "critical_path", "max_width", "max_rows", "flops", "analyses")


def cholesky_analyze(n: int, edge_nodes, fixed: int = 0):
    """b200pg_cholesky_analyze: the host analysis of the Cholesky linear solver for nodes 0..n-1 and edges [e, 2] of node
    indices, `fixed` the constant node (-1 for none). Returns (info dict keyed by FACTOR_INFO, free nodes in elimination
    order)."""
    ed = np.ascontiguousarray(np.asarray(edge_nodes, dtype=np.int32).reshape(-1, 2))
    info = np.zeros(8, dtype=np.int64)
    order = np.zeros(max(n, 1), dtype=np.int32)
    _check(lib().b200pg_cholesky_analyze(int(n), len(ed), _ip(ed), int(fixed), info.ctypes.data_as(C.POINTER(C.c_int64)),
                                         _ip(order), max(n, 1)))
    return dict(zip(FACTOR_INFO, (int(v) for v in info))), order[:int(info[0])].copy()


class ScanSolver:
    """karto::ScanSolver (Mapper.h:954-1065) as implemented by solver_plugins::CeresSolver
    (solvers/ceres_solver.cpp), on the GPU."""

    def __init__(self, **opts):
        o = PgOpts()
        lib().b200pg_default_opts(C.byref(o))
        for k, v in opts.items():
            if not hasattr(o, k):
                raise KeyError(k)
            setattr(o, k, v)
        self.opts = o
        self._h = C.c_void_p()
        _check(lib().b200pg_create(C.byref(o), C.byref(self._h)))
        self.summary = None

    def close(self):
        if self._h:
            lib().b200pg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int):
        _check(lib().b200pg_set_stream(self._h, C.c_void_p(cuda_stream)))

    def Reset(self):
        _check(lib().b200pg_reset(self._h))

    def Clear(self):
        _check(lib().b200pg_clear(self._h))

    def AddNode(self, unique_id: int, corrected_pose):
        p = np.ascontiguousarray(corrected_pose, dtype=np.float64)
        _check(lib().b200pg_add_node(self._h, int(unique_id), _dp(p)))

    def AddConstraint(self, source_id: int, target_id: int, pose_difference, covariance) -> bool:
        """LinkInfo::GetPoseDifference() / GetCovariance(). Returns False where the reference warns and ignores."""
        z = np.ascontiguousarray(pose_difference, dtype=np.float64)
        c = np.ascontiguousarray(covariance, dtype=np.float64).reshape(9)
        rc = lib().b200pg_add_edge(self._h, int(source_id), int(target_id), _dp(z), _dp(c))
        if rc == ERR_NOT_FOUND:
            return False
        _check(rc)
        return True

    def RemoveNode(self, unique_id: int) -> bool:
        rc = lib().b200pg_remove_node(self._h, int(unique_id))
        if rc == ERR_NOT_FOUND:
            return False
        _check(rc)
        return True

    def RemoveConstraint(self, source_id: int, target_id: int) -> bool:
        rc = lib().b200pg_remove_edge(self._h, int(source_id), int(target_id))
        if rc == ERR_NOT_FOUND:
            return False
        _check(rc)
        return True

    def ModifyNode(self, unique_id: int, pose):
        p = np.ascontiguousarray(pose, dtype=np.float64)
        rc = lib().b200pg_modify_node(self._h, int(unique_id), _dp(p))
        if rc != ERR_NOT_FOUND:
            _check(rc)

    def GetNodeOrientation(self, unique_id: int):
        p = np.zeros(3)
        rc = lib().b200pg_get_node(self._h, int(unique_id), _dp(p))
        return None if rc == ERR_NOT_FOUND else p[2]

    def getGraph(self):
        n = lib().b200pg_num_nodes(self._h)
        return {i: self.get_node(i) for i in self._ids()} if n else {}

    def get_node(self, unique_id: int):
        p = np.zeros(3)
        _check(lib().b200pg_get_node(self._h, int(unique_id), _dp(p)))
        return p

    def Compute(self) -> bool:
        """ScanSolver::Compute: returns False (and leaves corrections untouched) when no usable solution was found."""
        s = PgSummary()
        rc = lib().b200pg_solve(self._h, C.byref(s))
        self.summary = s
        if rc == ERR_NUMERIC:
            return False
        _check(rc)
        return True

    def GetCorrections(self):
        n = lib().b200pg_num_nodes(self._h)
        ids = np.zeros(max(n, 1), np.int32)
        poses = np.zeros((max(n, 1), 3))
        m = lib().b200pg_get_corrections(self._h, _ip(ids), _dp(poses), n)
        return ids[:m], poses[:m]

    def factor_info(self):
        """b200pg_factor_info: the analysis the last Cholesky solve used (dict keyed by FACTOR_INFO; zeros before one),
        with 'analyses' = the analyses this solver has run."""
        info = np.zeros(8, dtype=np.int64)
        _check(lib().b200pg_factor_info(self._h, info.ctypes.data_as(C.POINTER(C.c_int64))))
        return dict(zip(FACTOR_INFO, (int(v) for v in info)))

    def num_nodes(self):
        return lib().b200pg_num_nodes(self._h)

    def num_edges(self):
        return lib().b200pg_num_edges(self._h)


GridStates_Unknown, GridStates_Occupied, GridStates_Free = 0, 100, 255   # Karto.h:4379-4381


class OccupancyGrid:
    """karto::OccupancyGrid (Karto.h:5883-6330) on the GPU: the map slam_toolbox publishes
    (SMapper::getOccupancyGrid, src/slam_mapper.cpp:63-69).

        grid = OccupancyGrid.CreateFromScans(scans, resolution)       # None for no scans, like the reference's NULL
        grid.GetWidth(), grid.GetHeight(), grid.GetOffset(), grid.GetData() ...

    or, keeping the scans resident in HBM between map updates:

        grid = OccupancyGrid(resolution, laser); grid.AddScans(block); grid.Build(); grid.AddScans(more); grid.Build()
    """

    def __init__(self, resolution: float, laser: LaserRangeFinder | None = None, min_pass_through: int = 2,
                 occupancy_threshold: float = 0.1):
        laser = laser or LaserRangeFinder()
        self.params = OgParams(resolution, laser.range_threshold, laser.minimum_range, laser.maximum_range,
                               min_pass_through, occupancy_threshold)
        self._h = C.c_void_p()
        self.info = OgInfo()
        _check(lib().b200og_create(C.byref(self.params), C.byref(self._h)))

    @staticmethod
    def CreateFromScans(rScans: ScanBlock | None, resolution: float, min_pass_through: int = 2,
                        occupancy_threshold: float = 0.1) -> "OccupancyGrid | None":
        if rScans is None or len(rScans) == 0:
            return None
        g = OccupancyGrid(resolution, rScans.laser, min_pass_through, occupancy_threshold)
        g.AddScans(rScans)
        g.Build()
        return g

    def close(self):
        if self._h:
            lib().b200og_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int):
        _check(lib().b200og_set_stream(self._h, C.c_void_p(cuda_stream)))

    def AddScans(self, scans: ScanBlock):
        _check(lib().b200og_add_scans(self._h, scans.c, len(scans)))

    def ClearScans(self):
        _check(lib().b200og_clear_scans(self._h))

    def NumScans(self) -> int:
        return lib().b200og_num_scans(self._h)

    def Build(self):
        _check(lib().b200og_build(self._h, C.byref(self.info)))
        return self

    def GetWidth(self) -> int:
        return self.info.width

    def GetHeight(self) -> int:
        return self.info.height

    def GetWidthStep(self) -> int:
        return self.info.stride

    def GetOffset(self) -> np.ndarray:
        return np.array([self.info.offset[0], self.info.offset[1]])

    def GetResolution(self) -> float:
        return self.params.resolution

    def GetData(self, counters: bool = False):
        """cells [height, width step] uint8 (GridStates_*); with counters=True also (pass, hits) uint32."""
        h, st = self.info.height, self.info.stride
        cells = np.zeros((h, st), dtype=np.uint8)
        ps = np.zeros((h, st), dtype=np.uint32) if counters else None
        ht = np.zeros((h, st), dtype=np.uint32) if counters else None
        _check(lib().b200og_fetch(self._h, cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                  ps.ctypes.data_as(C.POINTER(C.c_uint32)) if counters else None,
                                  ht.ctypes.data_as(C.POINTER(C.c_uint32)) if counters else None))
        return (cells, ps, ht) if counters else cells

    def toNavMap(self) -> np.ndarray:
        """vis_utils::toNavMap: [height, width] int8 with -1 unknown / 100 occupied / 0 free."""
        out = np.zeros((self.info.height, self.info.width), dtype=np.int8)
        _check(lib().b200og_fetch_nav(self._h, out.ctypes.data_as(C.POINTER(C.c_int8))))
        return out

    def kernel_ms(self) -> float:
        ms = C.c_float()
        _check(lib().b200og_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def launch_count(self) -> int:
        return lib().b200og_launch_count(self._h)
