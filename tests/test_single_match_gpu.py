"""The single-match path (b200sm_match / b200sm_raster / b200sm_correlate: k_stamp, k_correlate, k_correlate_few and the FP64 host
epilogue) against the oracle, bit for bit, where the sequential cases of test_matcher_gpu.py never go: the shipped 20 m geometries
with the YAML's radian angles, smear kernels at both accepted bounds, queries at the origin / across the heading wrap / beyond 2 pi /
far from the origin, queries of 10,240 to 51,200 readings, windows either side of the two correlation kernels' boundary, more angles
than a CUDA grid holds in y, the fine-covariance fallback, dense / ROI-edge / ragged base lists, and one handle serving all of these
in turn and on a caller's stream.  Tolerances: none.  The cases are defined and pinned against the oracle in
test_single_match_fixtures.py."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
import test_single_match_fixtures as F
from oracle import karto_port as P
from slam_toolbox_b200 import api, synth

pytestmark = pytest.mark.gpu
FLAGS = ((True, True), (False, False), (True, False), (False, True))


def laser(geometry):
    return api.LaserRangeFinder(minimum_angle=geometry[0], angular_resolution=geometry[1])


def gpu_case(case: synth.SingleMatchCase):
    return (api.ScanBlock(case.query_ranges[None, :], case.query_pose[None, :], laser(case.query_laser)),
            api.ScanBlock(case.base_ranges, case.base_poses, laser(case.base_laser)))


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def same_grid(pm, gm):
    return np.array_equal(pm.grid()["data"], gm.GetCorrelationGrid()["data"])


class BaseList:
    """A base list of scans of any sizes, (ranges, points, pose) each, as the scan arrays of both implementations"""

    def __init__(self, scans):
        self.keep, self.n = [], len(scans)
        self.g, self.p = (api.CScan * max(1, self.n))(), (P.KpScan * max(1, self.n))()
        for s, (r, pts, pose) in enumerate(scans):
            r = np.ascontiguousarray(r, dtype=np.float64)
            pts = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 2)
            self.keep += [r, pts]
            dp = r.ctypes.data_as(C.POINTER(C.c_double)), pts.ctypes.data_as(C.POINTER(C.c_double))
            self.g[s] = api.CScan(len(r), dp[0], dp[1], (C.c_double * 3)(*pose))
            self.p[s] = P.KpScan(len(r), dp[0], dp[1], (C.c_double * 3)(*pose))

    def raster(self, pm, pq, gm, gq):
        P.lib().kp_raster(pm.h, C.byref(pq.c), self.p, self.n)
        api._check(api.lib().b200sm_raster(gm._h, C.byref(gq.c[0]), self.g, self.n))

    def match(self, pm, pq, gm, gq, pen, refine):
        pmean, pcov, gmean, gcov, resp = np.zeros(3), np.zeros(9), np.zeros(3), np.zeros(9), C.c_double()
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
        r = P.lib().kp_match(pm.h, C.byref(pq.c), self.p, self.n, int(pen), int(refine), dp(pmean), dp(pcov))
        api._check(api.lib().b200sm_match(gm._h, C.byref(gq.c[0]), self.g, self.n, int(pen), int(refine), dp(gmean), dp(gcov),
                                          C.byref(resp)))
        return (r, pmean, pcov), (resp.value, gmean, gcov)


def room_scans(case: synth.SingleMatchCase):
    pts = api.point_readings(case.base_ranges, case.base_poses, laser(case.base_laser))
    return [(r, p, pose) for r, p, pose in zip(case.base_ranges, pts, case.base_poses)]


# --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("expansion", [1, 0])
@pytest.mark.parametrize("name", list(F.GEOMETRIES))
def test_geometry_flags_and_query_kinds(name, expansion):
    """Every (penalise, refine) pair on a matching, a partly overlapping and an out-of-window query (zero best response on a
    non-empty raster: with expansion on, three more coarse passes run), then the grid bytes and the coarse volume"""
    mapper, grid, _ = F.GEOMETRIES[name]
    mapper = dict(mapper, use_response_expansion=expansion)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    so, sr = H.coarse_search(grid)
    for kind in F.QUERIES:
        case = F.geometry_case(name, kind)
        pq, pb = F.port_case(case)
        gq, gb = gpu_case(case)
        for pen, refine in FLAGS:
            assert same(pm.match(pq, pb, pen, refine), gm.MatchScan(gq, gb, pen, refine)), (kind, pen, refine)
        assert same_grid(pm, gm), kind
        for pen in (False, True):
            a = pm.correlate(pq, case.query_pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], pen,
                             False)
            b = gm.CorrelateScan(gq, case.query_pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"],
                                 pen, False)
            assert same(a, b) and np.array_equal(a[3], b[3]), (kind, pen)


@pytest.mark.parametrize("name", list(F.POSES))
def test_query_poses(name):
    case = F.pose_case(name)
    pq, pb = F.port_case(case)
    gq, gb = gpu_case(case)
    for mapper, grid in ((H.MAPPER_SEQ, H.GRID_SEQ), (F.MAPPER_YAML, F.GEOMETRIES["seq_shipped"][1]), (H.MAPPER_LOOP, H.GRID_LOOP)):
        pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
        for pen, refine in ((True, True), (True, False), (False, True)):
            assert same(pm.match(pq, pb, pen, refine), gm.MatchScan(gq, gb, pen, refine)), (grid, pen, refine)
        assert same_grid(pm, gm), grid


@pytest.mark.parametrize("n", F.LONG_BEAMS)
def test_long_query(n):
    """lookup rows of 40 KB, just above, 48 KB, just above, 117 KB and 200 KB of dynamic shared memory (coarse pass) and the
    warp-per-(pose, angle) fine pass over the same rows"""
    case = F.long_case(n)
    pq, pb = F.port_case(case)
    gq, gb = gpu_case(case)
    pm, gm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP), H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    for pen, refine in ((False, False), (True, True)):
        assert same(pm.match(pq, pb, pen, refine), gm.MatchScan(gq, gb, pen, refine)), (pen, refine)


def test_query_above_the_row_limit_is_refused_before_any_correlation():
    case = synth.make_single_match_case(7, n_beams=F.REFUSED_BEAMS, fov_deg=360.0)
    gq, gb = gpu_case(case)
    gm = H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    l0 = gm.launch_count()
    with pytest.raises(api.B200Error) as e:
        gm.MatchScan(gq, gb, True, True)
    assert e.value.code == api.ERR_UNSUPPORTED
    assert gm.launch_count() - l0 == 1   # the raster's k_stamp, nothing else
    ok = F.window_case()                 # the handle still serves a normal query
    pm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    assert same(pm.match(*F.port_case(ok), True, True), gm.MatchScan(*gpu_case(ok), True, True))


@pytest.mark.parametrize("name", list(F.WINDOWS))
def test_explicit_windows(name):
    so, sr, ao, ar, (nx, ny, na) = F.WINDOWS[name]
    case = F.window_case()
    pq, pb = F.port_case(case)
    gq, gb = gpu_case(case)
    pm, gm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP), H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    pm.raster(pq, pb)
    gm.raster(gq, gb)
    for pen in (False, True):
        a = pm.correlate(pq, case.query_pose, so, sr, ao, ar, pen, False)
        l0 = gm.launch_count()
        b = gm.CorrelateScan(gq, case.query_pose, so, sr, ao, ar, pen, False)
        assert gm.launch_count() - l0 == 1
        assert b[3].shape == (ny, nx, na)
        assert same(a, b) and np.array_equal(a[3], b[3]), pen


def test_wide_angle_window_then_a_narrow_one():
    """+-180 deg at 0.005 deg: 72,001 angles, more than gridDim.y can hold, through CorrelateScan and MatchScan; then a narrow
    window and a coarse pass of the default size on the same handle"""
    mapper, grid = F.WIDE["mapper"], F.WIDE["grid"]
    case = F.wide_case()
    pq, pb = F.port_case(case)
    gq, gb = gpu_case(case)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    so, sr = H.coarse_search(grid)
    pm.raster(pq, pb)
    gm.raster(gq, gb)
    nx, ny, na = F.WIDE["dims"]
    for pen in (False, True):
        a = pm.correlate(pq, case.query_pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], pen, False)
        b = gm.CorrelateScan(gq, case.query_pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], pen,
                             False)
        assert b[3].shape == (ny, nx, na)
        assert same(a, b) and np.array_equal(a[3], b[3]), pen
    assert same(pm.match(pq, pb, True, True), gm.MatchScan(gq, gb, True, True))
    so2, sr2, ao2, ar2, _ = F.WINDOWS["block_2112"]
    a = pm.correlate(pq, case.query_pose, so2, sr2, ao2, ar2, True, False)
    b = gm.CorrelateScan(gq, case.query_pose, so2, sr2, ao2, ar2, True, False)
    assert same(a, b) and np.array_equal(a[3], b[3])
    pm2, gm2 = H.port_matcher(H.MAPPER_LOOP, grid), H.gpu_matcher(H.MAPPER_LOOP, grid)
    assert same(pm2.match(pq, pb, True, True), gm2.MatchScan(gq, gb, True, True))


@pytest.mark.parametrize("n", F.FALLBACK_READINGS)
def test_fine_covariance_fallback(n):
    """fine passes centred on half-cell boundaries: where the averaged best pose rounds to a cell the 3 x 3 search did not visit,
    the angular covariance needs that cell's column, computed by one more launch"""
    mapper, grid = H.MAPPER_SEQ, H.GRID_SEQ_YAML
    case = F.fallback_case(n)
    gq, gb = gpu_case(case)
    gm = H.gpu_matcher(mapper, grid)
    gm.raster(gq, gb)
    so, sr, ao, ar = F.fine_window(mapper, grid)
    flagged = 0
    for pen in (False, True):
        for c, extra, exp in F.fallback_centres(n, pen):
            l0 = gm.launch_count()
            r, mean, cov, _ = gm.CorrelateScan(gq, c, so, sr, ao, ar, pen, True)
            assert same(exp, (r, mean, cov)), (c, pen)
            assert gm.launch_count() - l0 == (2 if extra else 1), (c, pen, extra)
            flagged += extra
    assert flagged > 0


def test_one_handle_many_sizes_and_streams():
    """long, short, long queries, then a dense and a sparse raster, on one handle (grow-only buffers, the kernel's shared-memory
    attribute left raised), then the same calls on a caller's torch stream and back on the handle's own"""
    import torch
    pm, gm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP), H.gpu_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    cases = [F.long_case(30000), F.window_case(), F.long_case(12289), F.long_case(10240)]
    ports = [F.port_case(c) for c in cases]
    gpus = [gpu_case(c) for c in cases]
    exp = [pm.match(pq, pb, True, True) for pq, pb in ports]
    dense = BaseList(synth.make_dense_base(cases[1].query_pose, H.GRID_LOOP[1]))
    sparse = BaseList(room_scans(cases[1])[:1])
    rasters = []
    for bl in (dense, sparse):
        bl.raster(pm, ports[1][0], gm, gpus[1][0])
        rasters.append(pm.grid()["data"])
        assert np.array_equal(rasters[-1], gm.GetCorrelationGrid()["data"])

    def run_all():
        for (gq, gb), e in zip(gpus, exp):
            assert same(e, gm.MatchScan(gq, gb, True, True))
        for bl, g in zip((dense, sparse), rasters):
            bl.raster(pm, ports[1][0], gm, gpus[1][0])
            assert np.array_equal(g, gm.GetCorrelationGrid()["data"])

    run_all()
    s = torch.cuda.Stream()
    gm.set_stream(s.cuda_stream)
    run_all()
    gm.set_stream(0)
    run_all()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", ["smear_half", "smear_10x", "seq_shipped"])
def test_dense_edge_and_ragged_rasters(name):
    """hundreds of points per cell (contended byte-max updates), points on the first / last ROI rows and columns (kernel rows reach
    the border and the stride padding) and just outside them, and a base list with a zero-reading scan and scans of different beam
    counts: grid bytes after raster() and a match against each list"""
    mapper, grid, _ = F.GEOMETRIES[name]
    case = F.window_case()
    pq, pb = F.port_case(case)
    gq, gb = gpu_case(case)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    pm.raster(pq, pb)
    roi_x, roi_y, roi_w, roi_h = pm.grid()["roi"]
    rooms = room_scans(case)
    short = (rooms[1][0][:400], rooms[1][1][:400], rooms[1][2])
    empty = (np.zeros(0), np.zeros((0, 2)), rooms[2][2])
    lists = {"dense": synth.make_dense_base(case.query_pose, grid[1]),
             "edge": synth.make_roi_edge_base(case.query_pose, grid[1], roi_w),
             "ragged": [rooms[0], empty, short] + synth.make_dense_base(case.query_pose, grid[1], n_clusters=5) + [rooms[3]]}
    for key, scans in lists.items():
        bl = BaseList(scans)
        bl.raster(pm, pq, gm, gq)
        g = pm.grid()
        assert np.array_equal(g["data"], gm.GetCorrelationGrid()["data"]), key
        img = g["data"].reshape(g["data_size"] // g["stride"], g["stride"])
        if key == "edge":   # every ROI corner cell is stamped
            for y in (roi_y, roi_y + roi_h - 1):
                for x in (roi_x, roi_x + roi_w - 1):
                    assert img[y, x] == 100, (y, x)
        else:
            assert img.max() == 100
        a, b = bl.match(pm, pq, gm, gq, True, True)
        assert same(a, b), key
