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
import json
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
    L.krep_remove_node.argtypes = [C.c_void_p, C.c_int]
    L.krep_num_scans.argtypes = [C.c_void_p]
    L.krep_poses.argtypes = [C.c_void_p, _DP, C.POINTER(C.c_int)]
    L.krep_stats.argtypes = [C.c_void_p, _DP]
    L.krep_counts.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.krep_edges.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), _DP, _DP, C.c_int]
    L.krep_solver_graph.argtypes = [C.c_void_p, C.POINTER(C.c_int), _DP, C.c_int]
    L.krep_solver_computes.argtypes = [C.c_void_p, _DP, C.POINTER(C.c_int), C.c_int]
    L.krep_occupancy.restype = C.c_double
    L.krep_occupancy.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(C.c_int), _DP, C.POINTER(C.c_uint8), C.c_long]
    L.krep_occupancy_resident.restype = C.c_double
    L.krep_occupancy_resident.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_int), _DP, C.POINTER(C.c_uint8), C.c_long,
                                          C.POINTER(C.c_int), C.POINTER(C.c_float)]
    L.krep_init_laser.argtypes = [C.c_double] * 6
    L.krep_laser.argtypes = [C.c_char_p] + [C.c_double] * 6
    L.krep_process_on.argtypes = [C.c_void_p, C.c_char_p, _DP, C.c_int, _DP, C.c_int]
    return L


SECOND_LASER = "laser1"


def _second_laser(L, laser: dict):
    """registers (or sets the limits of) the second laser, SECOND_LASER"""
    n = L.krep_laser(SECOND_LASER.encode(), laser["min_angle"], laser["max_angle"], laser["ang_res"], laser["min_range"],
                     laser["max_range"], laser["range_threshold"])
    if n <= 0:
        raise RuntimeError("krep_laser refused the second laser")


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


def _edges(L, h):
    """The mapper's graph edges (krep_edges, insertion order): source ids, target ids, pose differences, covariances."""
    ne = L.krep_edges(h, None, None, None, None, 0)
    src, dst = np.zeros(max(ne, 1), dtype=np.int32), np.zeros(max(ne, 1), dtype=np.int32)
    diff, cov = np.zeros((max(ne, 1), 3)), np.zeros((max(ne, 1), 3, 3))
    L.krep_edges(h, src.ctypes.data_as(C.POINTER(C.c_int)), dst.ctypes.data_as(C.POINTER(C.c_int)), diff.ctypes.data_as(_DP),
                 cov.ctypes.data_as(_DP), ne)
    return src[:ne], dst[:ne], diff[:ne], cov[:ne]


def lifelong_candidates(ids, src, dst, buffer: int):
    """The scans lifelong mode may remove (src/experimental/slam_toolbox_lifelong.cpp:271-278, 313), sorted: not ids 0 and 1,
    at least `buffer` (scan_buffer_size) ids older than the newest scan, and with two or more graph edges."""
    ids = np.asarray(ids)
    if len(ids) == 0:
        return ids
    deg = {int(i): 0 for i in ids}
    for a, b in zip(np.asarray(src).tolist(), np.asarray(dst).tolist()):
        deg[a] += 1
        deg[b] += 1
    newest = int(ids.max())
    return np.array(sorted(i for i, d in deg.items() if i > 1 and newest - i >= buffer and d >= 2), dtype=np.int64)


def _remove_node(L, h, step: int, nid: int, buffer: int, log: list):
    """krep_remove_node on nid, or (nid < 0) on a lifelong candidate picked from the mapper's edges by a generator seeded with
    the step.  Appends [step, id, its edges, its index among the stored scans, scans, return code, mapper vertices, mapper
    edges, solver nodes, solver edges, solver node set == mapper scan set]."""
    ids, _ = _scans(L, h)
    src, dst, _, _ = _edges(L, h)
    if nid < 0:
        cand = lifelong_candidates(ids, src, dst, buffer)
        nid = int(cand[np.random.default_rng(step).integers(len(cand))]) if len(cand) else 0
    deg = int(np.sum(src == nid) + np.sum(dst == nid))
    pos = int(np.searchsorted(ids, nid)) if nid in ids else -1
    rc = L.krep_remove_node(h, nid)
    counts = (C.c_int * 4)()
    L.krep_counts(h, counts)
    after, _ = _scans(L, h)
    _, gids, _ = _solver_graph(L, h, len(after) + 16)
    log.append([step, nid, deg, pos, len(ids), rc] + counts[:] + [int(np.array_equal(gids, np.sort(after)))])


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


def _publish_pair(L, h, map_resolution: float, step: int, log: list):
    """One map publish through the resident store (krep_occupancy_resident) and through the reference's CreateFromScans over
    the same scans.  Appends [step, equal, removed, appended, reloaded, resident seconds, reference seconds, resident device ms]."""
    info, off, stats, dms = (C.c_int * 3)(), np.zeros(2), (C.c_int * 3)(), C.c_float()
    cells = np.zeros(1, dtype=np.uint8)
    sec = L.krep_occupancy_resident(h, map_resolution, info, off.ctypes.data_as(_DP), None, 0, stats, C.byref(dms))
    if sec >= 0:   # the store is current after the first call: the second one only rebuilds and fetches
        cells = np.zeros(max(info[1], 0) * max(info[2], 0), dtype=np.uint8)
        L.krep_occupancy_resident(h, map_resolution, info, off.ctypes.data_as(_DP), cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                  cells.size, None, None)
    rinfo, roff = (C.c_int * 3)(), np.zeros(2)
    rsec = L.krep_occupancy(h, map_resolution, 0, rinfo, roff.ctypes.data_as(_DP), None, 0)
    rcells = np.zeros(max(rinfo[1], 0) * max(rinfo[2], 0), dtype=np.uint8)
    if rsec >= 0:
        rsec = L.krep_occupancy(h, map_resolution, 0, rinfo, roff.ctypes.data_as(_DP), rcells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                rcells.size)
    equal = sec >= 0 and rsec >= 0 and rinfo[:] == info[:] and roff.tobytes() == off.tobytes() and np.array_equal(cells, rcells)
    log.append([step, int(equal), stats[0], stats[1], stats[2], sec, rsec, dms.value])


def run_inprocess(which: str, ranges: np.ndarray, odom: np.ndarray, params: dict, laser: dict, use_solver: bool = True,
                  map_resolution: float = 0.0, publish_every: int = 0, events=(), sensors=None, laser2=None, laser2_changes=()):
    L = _bind(which)
    h = _create(L, laser, params, use_solver)
    if laser2 is not None:
        _second_laser(L, laser2)
    ranges = np.ascontiguousarray(ranges, dtype=np.float64)
    odom = np.ascontiguousarray(odom, dtype=np.float64)
    kept, publishes, removals = [], [], []
    buffer = int(params.get("scan_buffer_size", YAML_PARAMS["scan_buffer_size"]))
    for i in range(len(ranges)):
        if sensors is not None and sensors[i]:
            done = L.krep_process_on(h, SECOND_LASER.encode(), ranges[i].ctypes.data_as(_DP), ranges.shape[1],
                                     odom[i].ctypes.data_as(_DP), i)
        else:
            done = L.krep_process(h, ranges[i].ctypes.data_as(_DP), ranges.shape[1], odom[i].ctypes.data_as(_DP), i)
        if done:
            kept.append(i)
        for step, lim in laser2_changes:
            if step == i:   # a publish with the store current, the change, then two publishes with no scan in between
                _publish_pair(L, h, map_resolution, i, publishes)
                _second_laser(L, dict(laser2, **lim))
                _publish_pair(L, h, map_resolution, i, publishes)
                _publish_pair(L, h, map_resolution, i, publishes)
        if publish_every and (i + 1) % publish_every == 0:
            _publish_pair(L, h, map_resolution, i, publishes)
        for ev in events:
            if ev[0] != i:
                continue
            if ev[1] == "remove_node":
                _remove_node(L, h, i, int(ev[2]), buffer, removals)
            else:
                _publish_pair(L, h, map_resolution, i, publishes)
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
    if publish_every or events or laser2_changes:
        out["publishes"] = np.array(publishes, dtype=np.float64).reshape(-1, 8)
    if events:
        out["removals"] = np.array(removals, dtype=np.int64).reshape(-1, 11)
        out["edge_src"], out["edge_dst"], out["edge_diff"], out["edge_cov"] = _edges(L, h)
        out["scan_ids"] = _scans(L, h)[0]
    return out


def run(which: str, ranges, odom, params=None, laser=None, use_solver=True, tmpdir=None, map_resolution=0.0, publish_every=0,
        events=(), sensors=None, laser2=None, laser2_changes=()):
    """Runs the replay in a fresh process and returns its result dict.  publish_every = k > 0 (with map_resolution) also
    publishes the map after every k-th scan through the resident store and the reference, 'publishes' rows as _publish_pair.
    events: after step i's scan, in list order, (i, "remove_node", id) removes a scan as lifelong mode does (krep_remove_node;
    id < 0 picks one of lifelong_candidates, see _remove_node; 'removals' rows) and (i, "publish") publishes as
    publish_every does.  With events the result also holds the mapper's final edges and scan ids.
    Two lasers: laser2 (a dict like laser, same angles) is registered as SECOND_LASER, and scan i is processed on it where
    sensors[i] is nonzero (krep_process_on), on the first laser elsewhere.  laser2_changes = [(i, {key: value})] sets those
    limits of the second laser after step i's scan: one publish before the change, then two after it with no scan in between
    ('publishes' rows with step i)."""
    import tempfile
    params = params or YAML_PARAMS
    laser = laser or DEFAULT_LASER
    d = tmpdir or tempfile.mkdtemp(prefix="replay_")
    fin, fout = os.path.join(d, f"in_{which}.npz"), os.path.join(d, f"out_{which}.npz")
    np.savez(fin, ranges=ranges, odom=odom, pkeys=np.array(list(params.keys())), pvals=np.array(list(params.values()), dtype=np.float64),
             lkeys=np.array(list(laser.keys())), lvals=np.array(list(laser.values()), dtype=np.float64), use_solver=int(use_solver),
             map_resolution=float(map_resolution), publish_every=int(publish_every),
             events=np.array([[e[0], e[1] == "remove_node", e[2] if len(e) > 2 else -1] for e in events], dtype=np.int64).reshape(-1, 3),
             sensors=np.zeros(0, dtype=np.int64) if sensors is None else np.asarray(sensors, dtype=np.int64),
             l2keys=np.array(list((laser2 or {}).keys())), l2vals=np.array(list((laser2 or {}).values()), dtype=np.float64),
             l2steps=np.array([c[0] for c in laser2_changes], dtype=np.int64),
             l2changes=np.array([json.dumps(c[1]) for c in laser2_changes]))
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


def make_two_laser_trajectory(seed: int, n_scans: int, block: int = 6, step: float = 0.5):
    """make_trajectory with a second laser: scans alternate between the two lasers in blocks of `block` (A / B / A ...), so that
    the mapper meets a new sensor's first scan, and the second laser (TWO_LASER) has a shorter threshold, a larger minimum
    range and a shorter maximum range.  Returns ranges, odom, truth, sensors (0 / 1 per scan)."""
    ranges, odom, traj = make_trajectory(seed, n_scans, step)
    sensors = (np.arange(len(ranges)) // block) % 2
    return ranges, odom, traj, sensors


TWO_LASER = dict(DEFAULT_LASER, min_range=0.3, max_range=20.0, range_threshold=8.0)


def localization_inprocess(which: str, map_ranges, map_odom, loc_ranges, loc_odom, params: dict, loc_params: dict, laser: dict,
                           events, map_resolution: float = 0.0, publish_every: int = 0):
    """Maps with Mapper::Process, then applies loc_params and localizes scan by scan as the localization node does.
    events: (step, kind, pose) with kind "process_near" (that step's scan goes through ProcessAgainstNodesNearBy at pose) or
    "clear_localization_buffer" (Mapper::ClearLocalizationBuffer before that step's scan).  publish_every as run_inprocess, over
    the localization steps (the resident store holds the map's scans from the first publish on)."""
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
    clear_counts, publishes = [], []
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
        if publish_every and (i + 1) % publish_every == 0:
            _publish_pair(L, h, map_resolution, i, publishes)
    L.krep_stats(h, st.ctypes.data_as(_DP))
    ids, scan_poses = _scans(L, h)
    src, dst, diff, ecov = _edges(L, h)
    gn, gids, gposes = _solver_graph(L, h, len(ids) + 16)
    nc = L.krep_solver_computes(h, None, None, 0)
    cms, cup = np.zeros(max(nc, 1)), np.zeros(max(nc, 1), dtype=np.int32)
    L.krep_solver_computes(h, cms.ctypes.data_as(_DP), cup.ctypes.data_as(C.POINTER(C.c_int)), nc)
    out = dict(flags=flags, poses=poses, covs=covs, step_counts=step_counts, step_seconds=step_seconds, map_counts=map_counts,
               clear_counts=np.array(clear_counts, dtype=np.int32).reshape(-1, 5), scan_ids=ids, scan_poses=scan_poses,
               edge_src=src, edge_dst=dst, edge_diff=diff, edge_cov=ecov, graph_nodes=gn, graph_ids=gids,
               graph_poses=gposes, map_computes=map_computes, map_seconds=map_seconds, loc_seconds=st[0] - map_seconds,
               compute_ms=cms[:nc], compute_uploaded=cup[:nc], map_match_calls=map_matches,
               loc_match_calls=(int(L.b200_shim_match_calls()) - map_matches) if which == "b200" else 0)
    if map_resolution:
        _occupancy(L, h, map_resolution, out)
    if publish_every:
        out["publishes"] = np.array(publishes, dtype=np.float64).reshape(-1, 8)
    return out


def run_localization(which: str, map_ranges, map_odom, loc_ranges, loc_odom, params=None, events=(), loc_params=None, laser=None,
                     map_resolution=0.0, tmpdir=None, publish_every=0):
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
             map_resolution=float(map_resolution), publish_every=int(publish_every))
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
                                         params, loc_params, laser, events, float(z["map_resolution"]),
                                         int(z["publish_every"]) if "publish_every" in z.files else 0)
        else:
            events = [(int(e[0]), "remove_node", int(e[2])) if e[1] else (int(e[0]), "publish") for e in z["events"]]
            two = "sensors" in z.files and len(z["l2keys"]) > 0
            out = run_inprocess(which, z["ranges"], z["odom"], params, laser, bool(int(z["use_solver"])), float(z["map_resolution"]),
                                int(z["publish_every"]), events, sensors=z["sensors"] if two else None,
                                laser2={str(k): float(v) for k, v in zip(z["l2keys"], z["l2vals"])} if two else None,
                                laser2_changes=[(int(i), json.loads(str(c))) for i, c in zip(z["l2steps"], z["l2changes"])] if two else ())
    finally:
        os.dup2(saved, 1)
    np.savez(fout, **out)
