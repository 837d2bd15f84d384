"""cfg3 replay: the reference's own karto::Mapper::Process over a sequence of posed scans, through one of
the two integration libraries oracle/Makefile builds into oracle/_ref/ (where the reference sources are present):

  libreplay_ref.so   reference CPU ScanMatcher            + GPU ScanSolver adapter (B200Solver)
  libreplay_b200.so  GPU ScanMatcher (link-time seam)     + GPU ScanSolver adapter

Each run happens in its own process (both libraries define the same karto symbols):
    python integration/replay.py <ref|b200> <in.npz> <out.npz>
    python integration/replay.py localize-<ref|b200> <in.npz> <out.npz>     (run_localization)
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_DP = C.POINTER(C.c_double)

# slam_toolbox's shipped parameter set (config/mapper_params_online_sync.yaml:39-74), with Karto's default
# smear so that the sequential raster is order independent; BASELINE cfg3
YAML_PARAMS = dict(
    use_scan_matching=1, use_scan_barycenter=1, minimum_travel_distance=0.5, minimum_travel_heading=0.5, scan_buffer_size=10,
    scan_buffer_maximum_scan_distance=10.0, link_match_minimum_response_fine=0.1, link_scan_maximum_distance=1.5,
    loop_search_maximum_distance=3.0, do_loop_closing=1, loop_match_minimum_chain_size=10, loop_match_maximum_variance_coarse=3.0,
    loop_match_minimum_response_coarse=0.35, loop_match_minimum_response_fine=0.45,
    correlation_search_space_dimension=0.5, correlation_search_space_resolution=0.01, correlation_search_space_smear_deviation=0.1,
    loop_search_space_dimension=8.0, loop_search_space_resolution=0.05, loop_search_space_smear_deviation=0.03,
    distance_variance_penalty=0.5, angle_variance_penalty=1.0, fine_search_angle_offset=0.00349, coarse_search_angle_offset=0.349,
    coarse_angle_resolution=0.0349, minimum_angle_penalty=0.9, minimum_distance_penalty=0.5, use_response_expansion=1)
# config/mapper_params_localization.yaml where it differs from the mapping set above: a rolling buffer of 3 scans, and
# loop closures against the map from chains of 3
LOCALIZATION_PARAMS = dict(scan_buffer_size=3, loop_match_minimum_chain_size=3)
DEFAULT_LASER = dict(min_angle=math.radians(-135), max_angle=math.radians(135), ang_res=math.radians(0.25), min_range=0.1,
                     max_range=30.0, range_threshold=12.0)


def library(which: str) -> str:
    return os.path.join(ROOT, "oracle", "_ref", f"libreplay_{which}.so")


def available() -> bool:
    return os.path.exists(library("ref")) and os.path.exists(library("b200"))


def _bind(which: str):
    L = C.CDLL(library(which))
    L.krep_create.restype = C.c_void_p
    L.krep_create.argtypes = [C.c_int]
    L.krep_set.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
    L.krep_process.argtypes = [C.c_void_p, _DP, C.c_int, _DP, C.c_int]
    L.krep_process_localization.argtypes = [C.c_void_p, _DP, C.c_int, _DP, C.c_int, _DP, _DP]
    L.krep_process_near.argtypes = [C.c_void_p, _DP, C.c_int, _DP, C.c_int, _DP, _DP, _DP]
    L.krep_clear_localization_buffer.argtypes = [C.c_void_p]
    L.krep_num_scans.argtypes = [C.c_void_p]
    L.krep_poses.argtypes = [C.c_void_p, _DP, C.POINTER(C.c_int)]
    L.krep_stats.argtypes = [C.c_void_p, _DP]
    L.krep_counts.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.krep_edges.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), _DP, _DP, C.c_int]
    L.krep_solver_graph.argtypes = [C.c_void_p, C.POINTER(C.c_int), _DP, C.c_int]
    L.krep_solver_computes.argtypes = [C.c_void_p, _DP, C.POINTER(C.c_int), C.c_int]
    L.krep_occupancy.restype = C.c_double
    L.krep_occupancy.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(C.c_int), _DP, C.POINTER(C.c_uint8), C.c_long]
    L.krep_init_laser.argtypes = [C.c_double] * 6
    return L


def _create(L, laser: dict, params: dict, use_solver: bool):
    L.krep_init_laser(laser["min_angle"], laser["max_angle"], laser["ang_res"], laser["min_range"], laser["max_range"],
                      laser["range_threshold"])
    h = L.krep_create(int(use_solver))
    _set_params(L, h, params)
    return h


def _set_params(L, h, params: dict):
    for k, v in params.items():
        if L.krep_set(h, k.encode(), float(v)) != 0:
            raise KeyError(k)


def _scans(L, h):
    """The scans the mapper holds now: unique ids and corrected poses, in processing order."""
    n = L.krep_num_scans(h)
    ids = np.zeros(max(n, 1), dtype=np.int32)
    poses = np.zeros((max(n, 1), 3))
    L.krep_poses(h, poses.ctypes.data_as(_DP), ids.ctypes.data_as(C.POINTER(C.c_int)))
    return ids[:n], poses[:n]


def _solver_graph(L, h, cap: int):
    """ScanSolver::getGraph() of the adapter, sorted by id: (node count, ids, poses)."""
    gids = np.zeros(max(cap, 1), dtype=np.int32)
    gposes = np.zeros((max(cap, 1), 3))
    gn = L.krep_solver_graph(h, gids.ctypes.data_as(C.POINTER(C.c_int)), gposes.ctypes.data_as(_DP), cap)
    order = np.argsort(gids[:min(gn, cap)])
    return gn, gids[:min(gn, cap)][order], gposes[:min(gn, cap)][order]


def _occupancy(L, h, map_resolution: float, out: dict):
    """The map-publish step over the mapper's scans: reference CPU build and the b200og binding, same process."""
    for tag, gpu in (("cpu", 0), ("gpu", 1)):
        info = (C.c_int * 3)()
        off = np.zeros(2)
        sec = L.krep_occupancy(h, map_resolution, gpu, info, off.ctypes.data_as(_DP), None, 0)   # sizes (and warm-up)
        cells = np.zeros((max(info[1], 0), max(info[2], 0)), dtype=np.uint8)
        if sec >= 0:
            sec = L.krep_occupancy(h, map_resolution, gpu, info, off.ctypes.data_as(_DP), cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                   cells.size)
        out[f"map_{tag}_seconds"] = sec
        out[f"map_{tag}_dims"] = np.array([info[0], info[1], info[2]])
        out[f"map_{tag}_offset"] = off
        out[f"map_{tag}_cells"] = cells


def run_inprocess(which: str, ranges: np.ndarray, odom: np.ndarray, params: dict, laser: dict, use_solver: bool = True,
                  map_resolution: float = 0.0):
    L = _bind(which)
    h = _create(L, laser, params, use_solver)
    ranges = np.ascontiguousarray(ranges, dtype=np.float64)
    odom = np.ascontiguousarray(odom, dtype=np.float64)
    kept = []
    for i in range(len(ranges)):
        if L.krep_process(h, ranges[i].ctypes.data_as(_DP), ranges.shape[1], odom[i].ctypes.data_as(_DP), i):
            kept.append(i)
    _, poses = _scans(L, h)
    n = len(poses)
    st = np.zeros(5)
    L.krep_stats(h, st.ctypes.data_as(_DP))
    matches = 0
    if which == "b200":
        L.b200_shim_match_calls.restype = C.c_long
        matches = int(L.b200_shim_match_calls())
    gn, gids, gposes = _solver_graph(L, h, n) if use_solver else (0, np.zeros(0, dtype=np.int32), np.zeros((0, 3)))
    out = dict(graph_nodes=gn, graph_ids=gids, graph_poses=gposes, poses=poses, kept=np.array(kept),
               process_seconds=st[0], solver_computes=int(st[1]), solver_ms=st[2], edges=int(st[3]), scans=int(st[4]), match_calls=matches)
    if map_resolution:
        _occupancy(L, h, map_resolution, out)
    return out


def run(which: str, ranges, odom, params=None, laser=None, use_solver=True, tmpdir=None, map_resolution=0.0):
    """Runs the replay in a fresh process and returns its result dict."""
    import tempfile
    params = params or YAML_PARAMS
    laser = laser or DEFAULT_LASER
    d = tmpdir or tempfile.mkdtemp(prefix="replay_")
    fin, fout = os.path.join(d, f"in_{which}.npz"), os.path.join(d, f"out_{which}.npz")
    np.savez(fin, ranges=ranges, odom=odom, pkeys=np.array(list(params.keys())), pvals=np.array(list(params.values()), dtype=np.float64),
             lkeys=np.array(list(laser.keys())), lvals=np.array(list(laser.values()), dtype=np.float64), use_solver=int(use_solver),
             map_resolution=float(map_resolution))
    env = dict(os.environ)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), which, fin, fout], capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise RuntimeError(f"replay {which} failed:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    z = np.load(fout)
    return {k: (z[k] if z[k].shape else z[k].item()) for k in z.files}


def make_trajectory(seed: int, n_scans: int, step: float = 0.5):
    """A wandering path with revisits through the synthetic world: posed scans + drifting odometry."""
    sys.path.insert(0, ROOT)
    from slam_toolbox_b200 import synth
    rng = np.random.default_rng(seed)
    world = synth.make_world(seed)
    # a loop through a few room centres, repeated, so that later passes revisit earlier ones
    start = synth.free_pose(world, rng)
    half = synth.chain_poses(world, start, max(8, n_scans // 2), rng, step=step)
    back = half[::-1].copy()
    back[:, 2] = synth.wrap(back[:, 2] + math.pi)
    traj = np.concatenate([half, back])[:n_scans]
    ranges = synth.noisy(synth.raycast(world, traj), rng)
    # odometry = truth + slowly accumulating drift
    drift = np.cumsum(np.column_stack([rng.normal(0, 0.004, (len(traj), 2)), rng.normal(0, 0.0015, len(traj))]), axis=0)
    odom = traj + drift
    return ranges, odom, traj


def localization_inprocess(which: str, map_ranges, map_odom, loc_ranges, loc_odom, params: dict, loc_params: dict, laser: dict,
                           events, map_resolution: float = 0.0):
    """Maps with Mapper::Process, then applies loc_params and localizes scan by scan as the localization node does.
    events: (step, kind, pose) with kind "process_near" (that step's scan goes through ProcessAgainstNodesNearBy at pose) or
    "clear_localization_buffer" (Mapper::ClearLocalizationBuffer before that step's scan)."""
    L = _bind(which)
    if which == "b200":
        L.b200_shim_match_calls.restype = C.c_long
    h = _create(L, laser, params, True)
    map_ranges = np.ascontiguousarray(map_ranges, dtype=np.float64)
    map_odom = np.ascontiguousarray(map_odom, dtype=np.float64)
    for i in range(len(map_ranges)):
        L.krep_process(h, map_ranges[i].ctypes.data_as(_DP), map_ranges.shape[1], map_odom[i].ctypes.data_as(_DP), i)
    counts = (C.c_int * 4)()
    L.krep_counts(h, counts)
    map_counts = np.array(counts[:])
    st = np.zeros(5)
    L.krep_stats(h, st.ctypes.data_as(_DP))
    map_seconds, map_computes = st[0], int(st[1])
    map_matches = int(L.b200_shim_match_calls()) if which == "b200" else 0
    _set_params(L, h, loc_params)

    near = {int(s): np.asarray(p, dtype=np.float64) for s, k, p in events if k == "process_near"}
    clear = {int(s) for s, k, _ in events if k == "clear_localization_buffer"}
    loc_ranges = np.ascontiguousarray(loc_ranges, dtype=np.float64)
    loc_odom = np.ascontiguousarray(loc_odom, dtype=np.float64)
    n = len(loc_ranges)
    flags = np.zeros(n, dtype=np.int32)
    poses = np.full((n, 3), np.nan)
    covs = np.full((n, 3, 3), np.nan)
    step_counts = np.zeros((n, 4), dtype=np.int32)
    step_seconds = np.zeros(n)
    clear_counts = []
    for i in range(n):
        if i in clear:
            if L.krep_clear_localization_buffer(h) != 0:
                raise RuntimeError("krep_clear_localization_buffer refused")
            L.krep_counts(h, counts)
            clear_counts.append([i] + counts[:])
        rp, op = loc_ranges[i].ctypes.data_as(_DP), loc_odom[i].ctypes.data_as(_DP)
        pose, cov = np.zeros(3), np.zeros(9)
        sid = len(map_ranges) + i
        if i in near:
            rc = L.krep_process_near(h, rp, loc_ranges.shape[1], op, sid, near[i].ctypes.data_as(_DP), pose.ctypes.data_as(_DP),
                                     cov.ctypes.data_as(_DP))
        else:
            rc = L.krep_process_localization(h, rp, loc_ranges.shape[1], op, sid, pose.ctypes.data_as(_DP), cov.ctypes.data_as(_DP))
        if rc < 0:
            raise RuntimeError("the driver refused to localize")
        flags[i] = rc
        if rc:
            poses[i], covs[i] = pose, cov.reshape(3, 3)
        L.krep_counts(h, counts)
        step_counts[i] = counts[:]
        before = st[0]
        L.krep_stats(h, st.ctypes.data_as(_DP))
        step_seconds[i] = st[0] - before
    L.krep_stats(h, st.ctypes.data_as(_DP))
    ids, scan_poses = _scans(L, h)
    ne = L.krep_edges(h, None, None, None, None, 0)
    src, dst = np.zeros(max(ne, 1), dtype=np.int32), np.zeros(max(ne, 1), dtype=np.int32)
    diff, ecov = np.zeros((max(ne, 1), 3)), np.zeros((max(ne, 1), 3, 3))
    L.krep_edges(h, src.ctypes.data_as(C.POINTER(C.c_int)), dst.ctypes.data_as(C.POINTER(C.c_int)), diff.ctypes.data_as(_DP),
                 ecov.ctypes.data_as(_DP), ne)
    gn, gids, gposes = _solver_graph(L, h, len(ids) + 16)
    nc = L.krep_solver_computes(h, None, None, 0)
    cms, cup = np.zeros(max(nc, 1)), np.zeros(max(nc, 1), dtype=np.int32)
    L.krep_solver_computes(h, cms.ctypes.data_as(_DP), cup.ctypes.data_as(C.POINTER(C.c_int)), nc)
    out = dict(flags=flags, poses=poses, covs=covs, step_counts=step_counts, step_seconds=step_seconds, map_counts=map_counts,
               clear_counts=np.array(clear_counts, dtype=np.int32).reshape(-1, 5), scan_ids=ids, scan_poses=scan_poses,
               edge_src=src[:ne], edge_dst=dst[:ne], edge_diff=diff[:ne], edge_cov=ecov[:ne], graph_nodes=gn, graph_ids=gids,
               graph_poses=gposes, map_computes=map_computes, map_seconds=map_seconds, loc_seconds=st[0] - map_seconds,
               compute_ms=cms[:nc], compute_uploaded=cup[:nc], map_match_calls=map_matches,
               loc_match_calls=(int(L.b200_shim_match_calls()) - map_matches) if which == "b200" else 0)
    if map_resolution:
        _occupancy(L, h, map_resolution, out)
    return out


def run_localization(which: str, map_ranges, map_odom, loc_ranges, loc_odom, params=None, events=(), loc_params=None, laser=None,
                     map_resolution=0.0, tmpdir=None):
    """Maps map_* with Mapper::Process, then localizes loc_* with Mapper::ProcessLocalization (params updated by loc_params,
    LOCALIZATION_PARAMS by default), in a fresh process; events as localization_inprocess.  Returns per-step processed flags,
    published poses and covariances, graph sizes (mapper vertices, mapper edges, solver nodes, solver edges) and mapper seconds
    of every step,
    the final processed scans, the mapper's edges, the solver graph, every solver compute and (map_resolution > 0) both map
    publishes over the final scans."""
    import tempfile
    params = params or YAML_PARAMS
    loc_params = LOCALIZATION_PARAMS if loc_params is None else loc_params
    laser = laser or DEFAULT_LASER
    d = tmpdir or tempfile.mkdtemp(prefix="localize_")
    fin, fout = os.path.join(d, f"loc_in_{which}.npz"), os.path.join(d, f"loc_out_{which}.npz")
    kinds = {"process_near": 0, "clear_localization_buffer": 1}
    ev = np.array([[s, kinds[k]] + list(np.zeros(3) if p is None else p) for s, k, p in events], dtype=np.float64).reshape(-1, 5)
    np.savez(fin, map_ranges=map_ranges, map_odom=map_odom, loc_ranges=loc_ranges, loc_odom=loc_odom,
             pkeys=np.array(list(params.keys())), pvals=np.array(list(params.values()), dtype=np.float64),
             qkeys=np.array(list(loc_params.keys())), qvals=np.array(list(loc_params.values()), dtype=np.float64),
             lkeys=np.array(list(laser.keys())), lvals=np.array(list(laser.values()), dtype=np.float64), events=ev,
             map_resolution=float(map_resolution))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), f"localize-{which}", fin, fout], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"localization replay {which} failed:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    z = np.load(fout)
    return {k: (z[k] if z[k].shape else z[k].item()) for k in z.files}


def make_localization_trajectory(seed: int, n_scans: int, map_scans: int = 120, step: float = 0.5, offset=(0.15, -0.12, 0.04)):
    """A second pass through the world of make_trajectory(seed, map_scans): it starts beside a pose of the mapped path (a
    different free pose, its own heading), wanders out and comes back the same way, so that it crosses the mapped area.
    Odometry = truth seen from a frame `offset` (x, y, heading) off the map frame about the start, plus its own drift.
    Returns ranges, odometry, truth."""
    sys.path.insert(0, ROOT)
    from slam_toolbox_b200 import synth
    _, _, mapped = make_trajectory(seed, map_scans, step)
    rng = np.random.default_rng(seed + 7919)
    world = synth.make_world(seed)
    centre = mapped[int(rng.integers(len(mapped) // 4, max(len(mapped) // 2, len(mapped) // 4 + 1)))]
    start = synth.poses_near(world, centre[:2], 1.0, 1, rng)[0]
    half = synth.chain_poses(world, start, max(8, (n_scans + 1) // 2), rng, step=step)
    back = half[::-1].copy()
    back[:, 2] = synth.wrap(back[:, 2] + math.pi)
    traj = np.concatenate([half, back])[:n_scans]
    ranges = synth.noisy(synth.raycast(world, traj), rng)
    dx, dy, dth = offset
    c, s = math.cos(dth), math.sin(dth)
    rel = traj[:, :2] - start[:2]
    odom = np.column_stack([start[0] + dx + c * rel[:, 0] - s * rel[:, 1], start[1] + dy + s * rel[:, 0] + c * rel[:, 1],
                            synth.wrap(traj[:, 2] + dth)])
    odom += np.cumsum(np.column_stack([rng.normal(0, 0.004, (len(traj), 2)), rng.normal(0, 0.0015, len(traj))]), axis=0)
    return ranges, odom, traj


def lifecycle_inprocess():
    """Adapter hardening checks that need the integration library in this process: option mapping of B200Solver (the ceres_* keys
    CeresSolver::Configure reads) and release of the matchers' device state on Mapper::Reset / destruction."""
    L = C.CDLL(library("b200"))
    L.krep_create.restype = C.c_void_p
    L.krep_create.argtypes = [C.c_int]
    L.krep_process.argtypes = [C.c_void_p, _DP, C.c_int, _DP, C.c_int]
    L.krep_set.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
    L.krep_solver_configure.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.krep_reset_mapper.argtypes = [C.c_void_p]
    L.krep_destroy.argtypes = [C.c_void_p]
    L.b200_shim_live_handles.restype = C.c_long
    L.krep_init_laser.argtypes = [C.c_double] * 6
    L.krep_init_laser(math.radians(-135), math.radians(135), math.radians(0.25), 0.1, 30.0, 12.0)
    ranges, odom, _ = make_trajectory(3, 24)
    h = L.krep_create(1)
    for k, v in YAML_PARAMS.items():
        L.krep_set(h, k.encode(), float(v))
    out = {"configure": {}}
    for key, val in (("ceres_loss_function", "HuberLoss"), ("ceres_loss_function", "CauchyLoss"), ("ceres_loss_function", "None"),
                     ("ceres_loss_function", "Bogus"), ("ceres_trust_strategy", "LEVENBERG_MARQUARDT"), ("ceres_trust_strategy", "DOGLEG"),
                     ("ceres_linear_solver", "SPARSE_NORMAL_CHOLESKY"), ("ceres_preconditioner", "SCHUR_JACOBI"), ("no_such_key", "1")):
        out["configure"][f"{key}={val}"] = int(L.krep_solver_configure(h, key.encode(), val.encode()))
    live = [int(L.b200_shim_live_handles())]

    def feed(lo, hi):
        for i in range(lo, hi):
            L.krep_process(h, np.ascontiguousarray(ranges[i]).ctypes.data_as(_DP), ranges.shape[1], np.ascontiguousarray(odom[i]).ctypes.data_as(_DP), i)
    feed(0, 12)
    live.append(int(L.b200_shim_live_handles()))     # sequential + loop matcher
    L.krep_reset_mapper(h)
    live.append(int(L.b200_shim_live_handles()))     # Mapper::Reset deleted both
    feed(12, 24)
    live.append(int(L.b200_shim_live_handles()))
    L.krep_destroy(h)
    live.append(int(L.b200_shim_live_handles()))
    out["live_handles"] = live
    return out


if __name__ == "__main__":
    if sys.argv[1] == "lifecycle":
        import json
        devnull = os.open(os.devnull, os.O_WRONLY)
        saved = os.dup(1)
        os.dup2(devnull, 1)
        try:
            res = lifecycle_inprocess()
        finally:
            os.dup2(saved, 1)
        print(json.dumps(res))
        sys.exit(0)
    which, fin, fout = sys.argv[1], sys.argv[2], sys.argv[3]
    z = np.load(fin)
    params = {str(k): float(v) for k, v in zip(z["pkeys"], z["pvals"])}
    laser = {str(k): float(v) for k, v in zip(z["lkeys"], z["lvals"])}
    devnull = os.open(os.devnull, os.O_WRONLY)
    saved = os.dup(1)
    os.dup2(devnull, 1)   # the reference prints progress to stdout
    try:
        if which.startswith("localize-"):
            loc_params = {str(k): float(v) for k, v in zip(z["qkeys"], z["qvals"])}
            events = [(int(e[0]), ("process_near", "clear_localization_buffer")[int(e[1])], e[2:]) for e in z["events"]]
            out = localization_inprocess(which[len("localize-"):], z["map_ranges"], z["map_odom"], z["loc_ranges"], z["loc_odom"],
                                         params, loc_params, laser, events, float(z["map_resolution"]))
        else:
            out = run_inprocess(which, z["ranges"], z["odom"], params, laser, bool(int(z["use_solver"])), float(z["map_resolution"]))
    finally:
        os.dup2(saved, 1)
    np.savez(fout, **out)
