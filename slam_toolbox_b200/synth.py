"""Synthetic inputs for the scan-matching / pose-graph hot path (SURVEY.md section 8d).

Everything here is *workload generation* for tests and bench.py: a Manhattan world of
axis-aligned wall segments on a 0.5 m lattice, exact ray casting for a 1081-beam laser
(-135 deg .. +135 deg @ 0.25 deg, like the reference survey's LaserRangeFinder_Custom set-up),
posed scans, loop-closure candidate sets and a Manhattan-world SE(2) pose graph.  Nothing in
this file is on the product path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

N_BEAMS = 1081
ANGLE_MIN = math.radians(-135.0)
ANGLE_MAX = math.radians(135.0)
ANGLE_INC = math.radians(0.25)
RANGE_MIN = 0.1
RANGE_MAX = 30.0


@dataclass
class World:
    vert: np.ndarray   # (V,3) x, y0, y1   wall segments x = const
    horz: np.ndarray   # (H,3) y, x0, x1   wall segments y = const
    rooms: np.ndarray  # (R,4) x0, y0, x1, y1
    size: float

    @property
    def n_segments(self) -> int:
        return len(self.vert) + len(self.horz)


def make_world(seed: int, size: float = 36.0, min_room: float = 4.0, max_room: float = 12.0) -> World:
    """BSP split of [0,size]^2 into rooms with sides in [min_room, max_room] on a 0.5 m lattice;
    each interior wall gets one 1 m door."""
    rng = np.random.default_rng(seed)
    vert, horz, rooms = [], [], []

    def lattice(a: float, b: float) -> float:
        k0, k1 = int(math.ceil(a * 2 - 1e-9)), int(math.floor(b * 2 + 1e-9))
        return 0.5 * int(rng.integers(k0, k1 + 1))

    def split(x0, y0, x1, y1):
        w, h = x1 - x0, y1 - y0
        can_x, can_y = w >= 2 * min_room, h >= 2 * min_room
        must = w > max_room or h > max_room
        if not (can_x or can_y) or (not must and rng.random() < 0.5):
            rooms.append((x0, y0, x1, y1))
            return
        if can_x and (not can_y or w >= h):
            c = lattice(x0 + min_room, x1 - min_room)
            d = lattice(y0 + 0.5, y1 - 1.5)
            if d - y0 > 1e-9:
                vert.append((c, y0, d))
            if y1 - (d + 1.0) > 1e-9:
                vert.append((c, d + 1.0, y1))
            split(x0, y0, c, y1)
            split(c, y0, x1, y1)
        else:
            c = lattice(y0 + min_room, y1 - min_room)
            d = lattice(x0 + 0.5, x1 - 1.5)
            if d - x0 > 1e-9:
                horz.append((c, x0, d))
            if x1 - (d + 1.0) > 1e-9:
                horz.append((c, d + 1.0, x1))
            split(x0, y0, x1, c)
            split(x0, c, x1, y1)

    split(0.0, 0.0, size, size)
    vert += [(0.0, 0.0, size), (size, 0.0, size)]
    horz += [(0.0, 0.0, size), (size, 0.0, size)]
    return World(np.array(vert, dtype=np.float64), np.array(horz, dtype=np.float64),
                 np.array(rooms, dtype=np.float64), size)


def raycast(world: World, poses: np.ndarray, n_beams: int = N_BEAMS, angle_min: float = ANGLE_MIN,
            angle_inc: float = ANGLE_INC, range_max: float = RANGE_MAX, chunk: int = 16) -> np.ndarray:
    """Exact ranges (P, n_beams) for sensor poses (P,3) against the axis-aligned segments."""
    poses = np.atleast_2d(np.asarray(poses, dtype=np.float64))
    out = np.empty((len(poses), n_beams), dtype=np.float64)
    beam = angle_min + np.arange(n_beams) * angle_inc
    vx, vy0, vy1 = world.vert[:, 0], world.vert[:, 1], world.vert[:, 2]
    hy, hx0, hx1 = world.horz[:, 0], world.horz[:, 1], world.horz[:, 2]
    for s in range(0, len(poses), chunk):
        p = poses[s:s + chunk]
        ang = p[:, 2:3] + beam[None, :]
        dx, dy = np.cos(ang)[..., None], np.sin(ang)[..., None]       # (c,n,1)
        ox, oy = p[:, 0][:, None, None], p[:, 1][:, None, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            tv = (vx[None, None, :] - ox) / dx
            yv = oy + tv * dy
            okv = (tv > 1e-9) & (yv >= vy0 - 1e-12) & (yv <= vy1 + 1e-12)
            tv = np.where(okv, tv, np.inf)
            th = (hy[None, None, :] - oy) / dy
            xh = ox + th * dx
            okh = (th > 1e-9) & (xh >= hx0 - 1e-12) & (xh <= hx1 + 1e-12)
            th = np.where(okh, th, np.inf)
        r = np.minimum(tv.min(axis=2), th.min(axis=2))
        out[s:s + chunk] = np.minimum(r, range_max)
    return out


def free_pose(world: World, rng: np.random.Generator, margin: float = 0.6) -> np.ndarray:
    r = world.rooms[int(rng.integers(len(world.rooms)))]
    return np.array([rng.uniform(r[0] + margin, r[2] - margin), rng.uniform(r[1] + margin, r[3] - margin),
                     rng.uniform(-math.pi, math.pi)])


def wall_clearance(world: World, xy: np.ndarray) -> np.ndarray:
    """Distance from points (N,2) to the closest wall segment."""
    x, y = xy[:, 0:1], xy[:, 1:2]
    dv = np.hypot(x - world.vert[None, :, 0], np.clip(y, world.vert[None, :, 1], world.vert[None, :, 2]) - y)
    dh = np.hypot(np.clip(x, world.horz[None, :, 1], world.horz[None, :, 2]) - x, y - world.horz[None, :, 0])
    return np.minimum(dv.min(axis=1), dh.min(axis=1))


def poses_near(world: World, center_xy, radius: float, n: int, rng: np.random.Generator,
               margin: float = 0.4) -> np.ndarray:
    """n sensor poses uniformly within `radius` of center_xy, at least `margin` from any wall."""
    out = np.empty((0, 3))
    c = np.asarray(center_xy, dtype=np.float64)
    while len(out) < n:
        m = 2 * (n - len(out)) + 16
        rr = radius * np.sqrt(rng.random(m))
        aa = rng.uniform(-math.pi, math.pi, m)
        xy = c[None, :] + np.stack([rr * np.cos(aa), rr * np.sin(aa)], axis=1)
        ok = (xy[:, 0] > margin) & (xy[:, 0] < world.size - margin) & (xy[:, 1] > margin) & (xy[:, 1] < world.size - margin)
        ok &= wall_clearance(world, xy) >= margin
        th = rng.uniform(-math.pi, math.pi, m)
        out = np.concatenate([out, np.column_stack([xy, th])[ok]])
    return out[:n]


def noisy(ranges: np.ndarray, rng: np.random.Generator, sigma: float = 0.01, inf_frac: float = 0.0,
          nan_frac: float = 0.0) -> np.ndarray:
    r = ranges + rng.normal(0.0, sigma, ranges.shape)
    r = np.clip(r, 0.0, RANGE_MAX)
    if inf_frac > 0:
        r = np.where(rng.random(r.shape) < inf_frac, np.inf, r)
    if nan_frac > 0:
        r = np.where(rng.random(r.shape) < nan_frac, np.nan, r)
    return r


def chain_poses(world: World, start: np.ndarray, n: int, rng: np.random.Generator, step: float = 0.5) -> np.ndarray:
    """A short trajectory of n poses, `step` apart, staying clear of walls (running-scan chain)."""
    poses = [np.array(start, dtype=np.float64)]
    heading = start[2]
    tries = 0
    while len(poses) < n:
        h = heading + rng.normal(0, 0.15)
        nxt = poses[-1][:2] + step * np.array([math.cos(h), math.sin(h)])
        ok = 0.4 < nxt[0] < world.size - 0.4 and 0.4 < nxt[1] < world.size - 0.4 and \
            wall_clearance(world, nxt[None, :])[0] > 0.4
        if ok:
            poses.append(np.array([nxt[0], nxt[1], h]))
            heading = h
            tries = 0
        else:
            heading = rng.uniform(-math.pi, math.pi)
            tries += 1
            if tries > 200:
                poses.append(poses[-1].copy())
    return np.array(poses)


@dataclass
class LoopSweep:
    """cfg2 / cfg5 shaped input: query scans and candidate chains (SURVEY.md 8d)."""
    query_ranges: np.ndarray          # (Q, n)
    query_poses: np.ndarray           # (Q, 3)  believed (drifted) sensor poses
    query_true: np.ndarray            # (Q, 3)
    cand_ranges: np.ndarray           # (S, n)  all candidate scans
    cand_poses: np.ndarray            # (S, 3)  corrected sensor poses
    chain_start: np.ndarray           # (C+1,)  chain j = scans [chain_start[j], chain_start[j+1])
    world: World = field(repr=False, default=None)


def make_loop_sweep(seed: int, n_queries: int = 1, n_chains: int = 1000, chain_len: int = 1,
                    drift_xy: float = 0.5, drift_th: float = 0.08, radius: float = 3.0,
                    inf_frac: float = 0.0, world: World | None = None) -> LoopSweep:
    rng = np.random.default_rng(seed)
    world = world or make_world(seed)
    qtrue = np.array([free_pose(world, rng) for _ in range(n_queries)])
    qr = noisy(raycast(world, qtrue), rng, inf_frac=inf_frac)
    qpose = qtrue + np.column_stack([rng.normal(0, drift_xy, (n_queries, 2)), rng.normal(0, drift_th, n_queries)])
    # candidates live around the first query's true position (one revisit area per sweep)
    starts = poses_near(world, qtrue[0, :2], radius, n_chains, rng)
    if chain_len == 1:
        cposes = starts
    else:
        cposes = np.concatenate([chain_poses(world, s, chain_len, rng) for s in starts])
    cr = noisy(raycast(world, cposes), rng, inf_frac=inf_frac)
    chain_start = np.arange(0, n_chains * chain_len + 1, chain_len, dtype=np.int32)
    return LoopSweep(qr, qpose, qtrue, cr, cposes, chain_start, world)


def make_sequential_case(seed: int, buffer_len: int = 10, odo_xy: float = 0.03, odo_th: float = 0.01,
                         inf_frac: float = 0.0, nan_frac: float = 0.0):
    """cfg1: one query against a running buffer of `buffer_len` scans spaced 0.5 m."""
    rng = np.random.default_rng(seed)
    world = make_world(seed)
    traj = chain_poses(world, free_pose(world, rng), buffer_len + 1, rng)
    ranges = noisy(raycast(world, traj), rng, inf_frac=inf_frac, nan_frac=nan_frac)
    qtrue = traj[-1]
    qpose = qtrue + np.array([rng.normal(0, odo_xy), rng.normal(0, odo_xy), rng.normal(0, odo_th)])
    return dict(world=world, base_ranges=ranges[:-1], base_poses=traj[:-1], query_ranges=ranges[-1],
                query_pose=qpose, query_true=qtrue)


def make_mapping_run(seed: int, n_scans: int = 24, step: float = 0.5, inf_frac: float = 0.02, nan_frac: float = 0.005,
                     odd_readings: bool = True, world: World | None = None):
    """Input of the map-publish step (OccupancyGrid::CreateFromScans over all processed scans): a trajectory of
    n_scans sensor poses `step` apart with their scans.  odd_readings sprinkles the values AddScan treats specially
    (Karto.h:6158-6171): below the minimum range, at / beyond the maximum range, exactly at the range threshold."""
    rng = np.random.default_rng(seed)
    world = world or make_world(seed)
    poses = chain_poses(world, free_pose(world, rng), n_scans, rng, step=step)
    ranges = noisy(raycast(world, poses), rng, inf_frac=inf_frac, nan_frac=nan_frac)
    if odd_readings and ranges.size:
        m = ranges.shape[1]
        for s in range(len(ranges)):
            k = rng.integers(0, m, 6)
            ranges[s, k[0]] = 0.05
            ranges[s, k[1]] = 0.1          # == minimum range: ignored (<=)
            ranges[s, k[2]] = 30.0         # == maximum range: ignored (>=)
            ranges[s, k[3]] = 12.0         # == range threshold: traced, no hit
            ranges[s, k[4]] = 12.0 - 5e-7  # inside the KT_TOLERANCE band: traced to the end point, no hit
            ranges[s, k[5]] = 25.0         # beyond the threshold: traced up to it
    return dict(world=world, ranges=ranges, poses=poses)


def wrap(a):
    """[-pi, pi) like solvers/ceres_utils.h:27-32 NormalizeAngle."""
    a = np.asarray(a, dtype=np.float64)
    return a - 2.0 * math.pi * np.floor((a + math.pi) / (2.0 * math.pi))


def make_pose_graph(seed: int, n_nodes: int = 10000, n_edges: int = 40000, lattice: int = 100,
                    sigma_xy: float = 0.05, sigma_th: float = 0.02, min_gap: int = 50):
    """cfg4: Manhattan-world SE(2) graph (SURVEY.md 8d): random walk on a lattice (1 m steps, 90 deg
    turns), n_nodes-1 odometry edges + loop edges between nodes on the same/adjacent lattice site
    with index gap > min_gap.  Edge = (a, b, z = pose_b in frame a + noise, cov = diag(sigma^2) rotated
    like LinkInfo::Update, Mapper.h:174-188).  Initial guess = dead-reckoned odometry."""
    rng = np.random.default_rng(seed)
    dirs = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]])
    cell = np.zeros((n_nodes, 2), dtype=np.int64)
    head = np.zeros(n_nodes, dtype=np.int64)
    cell[0] = lattice // 2
    for i in range(1, n_nodes):
        h = head[i - 1]
        r = rng.random()
        if r < 0.25:
            h = (h + 1) % 4
        elif r < 0.5:
            h = (h + 3) % 4
        nxt = cell[i - 1] + dirs[h]
        k = 0
        while not (0 <= nxt[0] < lattice and 0 <= nxt[1] < lattice):
            h = (h + 1) % 4
            nxt = cell[i - 1] + dirs[h]
            k += 1
        head[i] = h
        cell[i] = nxt
    truth = np.column_stack([cell[:, 0].astype(float), cell[:, 1].astype(float), wrap(head * (math.pi / 2))])

    def rel(pa, pb):
        c, s = np.cos(pa[:, 2]), np.sin(pa[:, 2])
        dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
        return np.column_stack([c * dx + s * dy, -s * dx + c * dy, wrap(pb[:, 2] - pa[:, 2])])

    ea = list(range(n_nodes - 1))
    eb = list(range(1, n_nodes))
    # loop edges: bucket nodes by lattice site
    site = {}
    for i in range(n_nodes):
        site.setdefault((int(cell[i, 0]), int(cell[i, 1])), []).append(i)
    pairs = set()
    want = n_edges - (n_nodes - 1)
    order = rng.permutation(n_nodes)
    nb = [(0, 0), (1, 0), (0, 1), (-1, 0), (0, -1)]
    rounds = 0
    while len(pairs) < want and rounds < 64:
        for i in order:
            if len(pairs) >= want:
                break
            dxy = nb[int(rng.integers(len(nb)))]
            lst = site.get((int(cell[i, 0]) + dxy[0], int(cell[i, 1]) + dxy[1]))
            if not lst:
                continue
            j = lst[int(rng.integers(len(lst)))]
            a, b = (int(i), int(j)) if i < j else (int(j), int(i))
            if b - a > min_gap:
                pairs.add((a, b))
        rounds += 1
    pairs = sorted(pairs)
    ea += [p[0] for p in pairs]
    eb += [p[1] for p in pairs]
    ea, eb = np.array(ea, dtype=np.int32), np.array(eb, dtype=np.int32)
    z = rel(truth[ea], truth[eb])
    z += np.column_stack([rng.normal(0, sigma_xy, (len(ea), 2)), rng.normal(0, sigma_th, len(ea))])
    z[:, 2] = wrap(z[:, 2])
    # covariance in the frame of pose a: R(-th_a) diag R(-th_a)^T  (Mapper.h:183-186)
    base = np.diag([sigma_xy ** 2, sigma_xy ** 2, sigma_th ** 2])
    cov = np.empty((len(ea), 3, 3))
    for k in range(len(ea)):
        t = -truth[ea[k], 2]
        R = np.array([[math.cos(t), -math.sin(t), 0], [math.sin(t), math.cos(t), 0], [0, 0, 1]])
        cov[k] = R @ base @ R.T
    # dead-reckoned initial guess from the odometry edges
    init = np.zeros_like(truth)
    init[0] = truth[0]
    for i in range(1, n_nodes):
        c, s = math.cos(init[i - 1, 2]), math.sin(init[i - 1, 2])
        init[i, 0] = init[i - 1, 0] + c * z[i - 1, 0] - s * z[i - 1, 1]
        init[i, 1] = init[i - 1, 1] + s * z[i - 1, 0] + c * z[i - 1, 1]
        init[i, 2] = wrap(init[i - 1, 2] + z[i - 1, 2])
    ids = np.arange(n_nodes, dtype=np.int32)
    return dict(ids=ids, init=init, truth=truth, edge_a=ea, edge_b=eb, z=z, cov=cov)


def make_pose_graph_large(seed: int, n_nodes: int, n_edges: int, lattice: int, sigma_xy: float = 0.05,
                          sigma_th: float = 0.02, min_gap: int = 50) -> dict:
    """make_pose_graph's kind of graph at sizes its per-edge loops make slow (10^6 nodes): vectorised, with its own random
    stream, so it does not reproduce make_pose_graph's graphs.  The lattice walk (1 m steps, 90 deg turns with probability
    1/4 each way) is folded back into [0, lattice)^2 (a step across a border stays on its site) instead of turning; loop edges join nodes on the same or an
    adjacent site with index gap > min_gap, drawn in rounds of one candidate per node until n_edges - (n_nodes - 1) distinct
    pairs are found.  Measurements, covariances and the dead-reckoned initial guess as in make_pose_graph."""
    rng = np.random.default_rng(seed)
    r = rng.random(n_nodes - 1)
    turn = np.where(r < 0.25, 1, np.where(r < 0.5, 3, 0))
    head = np.concatenate([[0], np.cumsum(turn) % 4])
    dirs = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]])
    raw = lattice // 2 + np.concatenate([np.zeros((1, 2), dtype=np.int64), np.cumsum(dirs[head[1:]], axis=0)])
    period = 2 * lattice   # fold the unbounded walk into [0, lattice): a reflection at each border
    m = np.mod(raw, period)
    cell = np.where(m < lattice, m, period - 1 - m)
    truth = np.column_stack([cell[:, 0].astype(float), cell[:, 1].astype(float), wrap(head * (math.pi / 2))])
    key = cell[:, 0] * lattice + cell[:, 1]
    order = np.argsort(key, kind="stable")
    skey = key[order]
    want = n_edges - (n_nodes - 1)
    nb = np.array([(0, 0), (1, 0), (0, 1), (-1, 0), (0, -1)])
    found = np.zeros(0, dtype=np.int64)
    for _ in range(64):
        if len(found) >= want:
            break
        i = rng.permutation(n_nodes)
        c = cell[i] + nb[rng.integers(len(nb), size=n_nodes)]
        ok = (c[:, 0] >= 0) & (c[:, 0] < lattice) & (c[:, 1] >= 0) & (c[:, 1] < lattice)
        k = c[:, 0] * lattice + c[:, 1]
        lo, hi = np.searchsorted(skey, k, "left"), np.searchsorted(skey, k, "right")
        ok &= hi > lo
        pick = lo + np.floor(rng.random(n_nodes) * np.maximum(hi - lo, 1)).astype(np.int64)
        j = order[np.minimum(pick, n_nodes - 1)]
        a, b = np.minimum(i, j), np.maximum(i, j)
        ok &= (b - a) > min_gap
        cand = np.concatenate([found, (a * n_nodes + b)[ok]])
        _, first = np.unique(cand, return_index=True)
        found = cand[np.sort(first)]
    pairs = np.sort(found[:want])
    ea = np.concatenate([np.arange(n_nodes - 1), pairs // n_nodes]).astype(np.int32)
    eb = np.concatenate([np.arange(1, n_nodes), pairs % n_nodes]).astype(np.int32)
    z = _pose_rel(truth[ea], truth[eb])
    z += np.column_stack([rng.normal(0, sigma_xy, (len(ea), 2)), rng.normal(0, sigma_th, len(ea))])
    z[:, 2] = wrap(z[:, 2])
    t = -truth[ea, 2]
    R = np.zeros((len(ea), 3, 3))
    R[:, 0, 0] = np.cos(t); R[:, 0, 1] = -np.sin(t); R[:, 1, 0] = np.sin(t); R[:, 1, 1] = np.cos(t); R[:, 2, 2] = 1.0
    cov = R @ np.diag([sigma_xy ** 2, sigma_xy ** 2, sigma_th ** 2]) @ R.transpose(0, 2, 1)
    odo = z[: n_nodes - 1]
    th = np.concatenate([[truth[0, 2]], truth[0, 2] + np.cumsum(odo[:, 2])])
    c, s = np.cos(th[:-1]), np.sin(th[:-1])
    init = np.zeros_like(truth)
    init[0] = truth[0]
    init[1:, 0] = truth[0, 0] + np.cumsum(c * odo[:, 0] - s * odo[:, 1])
    init[1:, 1] = truth[0, 1] + np.cumsum(s * odo[:, 0] + c * odo[:, 1])
    init[:, 2] = wrap(th)
    return dict(ids=np.arange(n_nodes, dtype=np.int32), init=init, truth=truth, edge_a=ea, edge_b=eb, z=z, cov=cov)


def _pose_rel(pa, pb):
    """pb in the frame of pa, rows (x, y, theta) -> (dx, dy, wrap(dtheta))."""
    c, s = np.cos(pa[:, 2]), np.sin(pa[:, 2])
    dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
    return np.column_stack([c * dx + s * dy, -s * dx + c * dy, wrap(pb[:, 2] - pa[:, 2])])


def _lattice_walk(rng: np.random.Generator, n: int, lattice: int, start) -> np.ndarray:
    """Random walk of n lattice sites (1 m steps, 90 deg turns) inside [0, lattice)^2; returns (n, 3) cells + heading index."""
    dirs = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]])
    out = np.zeros((n, 3), dtype=np.int64)
    out[0, :2] = start
    for i in range(1, n):
        h = out[i - 1, 2]
        r = rng.random()
        h = (h + 1) % 4 if r < 0.25 else (h + 3) % 4 if r < 0.5 else h
        nxt = out[i - 1, :2] + dirs[h]
        while not (0 <= nxt[0] < lattice and 0 <= nxt[1] < lattice):
            h = (h + 1) % 4
            nxt = out[i - 1, :2] + dirs[h]
        out[i, :2], out[i, 2] = nxt, h
    return out


def _base_covariance(rng: np.random.Generator, model: str, sigma_xy: float, sigma_th: float) -> np.ndarray:
    """Edge covariance before the LinkInfo rotation.  iso: diag(sxy^2, sxy^2, sth^2).  karto: an anisotropic xy block
    R(phi) diag(s1^2, s2^2) R(phi)^T with s1 / s2 in [1, 10] (a corridor) and a separate theta variance.  full: the karto
    xy block with x-theta and y-theta correlations, a general SPD 3x3."""
    if model == "iso":
        return np.diag([sigma_xy ** 2, sigma_xy ** 2, sigma_th ** 2])
    ratio = rng.uniform(1.0, 10.0)
    s1, s2 = sigma_xy * math.sqrt(ratio), sigma_xy / math.sqrt(ratio)
    phi = rng.uniform(-math.pi, math.pi)
    c, s = math.cos(phi), math.sin(phi)
    R = np.array([[c, -s], [s, c]])
    cov = np.zeros((3, 3))
    cov[:2, :2] = R @ np.diag([s1 * s1, s2 * s2]) @ R.T
    cov[2, 2] = (sigma_th * rng.uniform(0.5, 2.0)) ** 2
    if model == "full":
        # correlation of theta with a random xy direction, |rho| <= 0.7: the Schur complement stays positive definite
        rho = rng.uniform(-0.7, 0.7)
        u = rng.normal(size=2)
        u /= np.linalg.norm(u)
        sd = np.sqrt(np.diag(cov[:2, :2]))
        w = rho * math.sqrt(cov[2, 2]) * (cov[:2, :2] @ u) / math.sqrt(u @ cov[:2, :2] @ u)
        cov[:2, 2] = cov[2, :2] = w
        assert np.all(np.abs(w) < sd * math.sqrt(cov[2, 2]))
    elif model != "karto":
        raise ValueError(f"unknown covariance model {model!r}")
    return cov


def _rot_z(t: float) -> np.ndarray:
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def make_pose_graph_family(seed: int, n_nodes: int = 2000, n_loops: int = 4000, *, cov_model: str = "iso",
                           sigma_xy: float = 0.03, sigma_th: float = 0.01, reversed_frac: float = 0.0,
                           duplicate_frac: float = 0.0, order: str = "chain", ids: str = "dense",
                           world_rotation: float = 0.0, world_translation=(0.0, 0.0), isolated_runs=(),
                           detached_nodes: int = 0, hub_degree: int = 0, lattice: int = 60, min_gap: int = 20,
                           heading_jitter: float = 0.05) -> dict:
    """SE(2) pose graphs of the shapes a mapper produces and make_pose_graph does not (it stays as it is: bench.py's cfg4).

    A lattice random walk of n_nodes poses (headings jittered off the lattice directions) with odometry and up to
    n_loops loop edges between poses on the same / adjacent site, plus:
      cov_model        'iso' | 'karto' | 'full' (see _base_covariance), then rotated into the source frame like
                       LinkInfo::Update (Mapper.h:174-188); measurement noise is drawn from that covariance
      reversed_frac    fraction of edges stored target -> source, with z and cov of the reversed direction
      duplicate_frac   fraction of edges repeated as parallel edges with independent noise
      order            insertion order of the connected nodes: 'chain', 'reversed' or 'shuffled'; the first inserted
                       node is the solver's anchor, which may then sit anywhere along the chain
      ids              'dense' (0..N-1) or 'sparse' (unique int32 ids including negative ones and both extremes)
      world_rotation / world_translation   rigid transform of the whole world (truth and initial guess)
      isolated_runs    ((fraction, length), ...): runs of consecutive nodes without edges, inserted at that fraction of
                       the insertion order (never first)
      detached_nodes   a second walk of that many nodes with its own odometry / loop edges, not connected to the first
      hub_degree       extra loop edges from the walk's middle node to nodes at least 64 steps away along the walk
    Returns ids, init, truth (insertion order), edge_a / edge_b (ids), ia / ib (insertion positions), z, cov,
    component (0 main walk, 1 detached walk, -1 isolated) and anchor (insertion position of the anchor, 0)."""
    rng = np.random.default_rng(seed)
    comps = [(0, n_nodes)] + ([(1, detached_nodes)] if detached_nodes else [])
    truth_l, comp_l, src, dst, kinds = [], [], [], [], []
    base = 0
    for cid, n in comps:
        walk = _lattice_walk(rng, n, lattice, (lattice // 2, lattice // 2) if cid == 0 else (lattice // 4, lattice // 4))
        th = wrap(walk[:, 2] * (math.pi / 2) + rng.normal(0.0, heading_jitter, n))
        truth_l.append(np.column_stack([walk[:, 0].astype(float), walk[:, 1].astype(float), th]))
        comp_l.append(np.full(n, cid))
        src += list(range(base, base + n - 1)); dst += list(range(base + 1, base + n)); kinds += [0] * (n - 1)
        site = {}
        for i in range(n):
            site.setdefault((int(walk[i, 0]), int(walk[i, 1])), []).append(i)
        want = n_loops if cid == 0 else max(1, (n_loops * n) // max(n_nodes, 1))
        pairs, tries = set(), 0
        while len(pairs) < want and tries < 64 * max(want, 1):
            tries += 1
            i = int(rng.integers(n))
            dx, dy = [(0, 0), (1, 0), (0, 1), (-1, 0), (0, -1)][int(rng.integers(5))]
            lst = site.get((int(walk[i, 0]) + dx, int(walk[i, 1]) + dy))
            if lst:
                j = lst[int(rng.integers(len(lst)))]
                if abs(j - i) > min_gap:
                    pairs.add((min(i, j), max(i, j)))
        for a, b in sorted(pairs):
            src.append(base + a); dst.append(base + b); kinds.append(1)
        if cid == 0 and hub_degree:
            h = n // 2
            far = np.nonzero(np.abs(np.arange(n) - h) > 64)[0]
            far = far if len(far) else np.setdiff1d(np.arange(n), [h])
            for j in rng.choice(far, size=hub_degree, replace=True):
                src.append(base + h); dst.append(base + int(j)); kinds.append(2)
        base += n
    truth = np.concatenate(truth_l)
    comp = np.concatenate(comp_l)
    src, dst = np.array(src, dtype=np.int64), np.array(dst, dtype=np.int64)
    E0 = len(src)
    dup = np.nonzero(rng.random(E0) < duplicate_frac)[0]
    src, dst = np.concatenate([src, src[dup]]), np.concatenate([dst, dst[dup]])
    kinds = np.concatenate([np.array(kinds), np.full(len(dup), 3)])
    E = len(src)
    # measurement and covariance of every edge in its forward (walk) direction
    cov_f = np.empty((E, 3, 3))
    z_f = _pose_rel(truth[src], truth[dst])
    for k in range(E):
        cb = _base_covariance(rng, cov_model, sigma_xy, sigma_th)
        R = _rot_z(-truth[src[k], 2])
        cov_f[k] = R @ cb @ R.T
        z_f[k] += np.linalg.cholesky(cov_f[k]) @ rng.normal(size=3)
    z_f[:, 2] = wrap(z_f[:, 2])
    # dead-reckoned initial guess of every walk from its odometry edges (forward direction)
    init = truth.copy()
    for k in np.nonzero(kinds == 0)[0]:
        a, b = src[k], dst[k]
        c, s = math.cos(init[a, 2]), math.sin(init[a, 2])
        init[b, 0] = init[a, 0] + c * z_f[k, 0] - s * z_f[k, 1]
        init[b, 1] = init[a, 1] + s * z_f[k, 0] + c * z_f[k, 1]
        init[b, 2] = wrap(init[a, 2] + z_f[k, 2])
    # reversed edges: z^-1 and the covariance pushed through the Jacobian of the inverse
    z, cov = z_f.copy(), cov_f.copy()
    rev = np.nonzero(rng.random(E) < reversed_frac)[0]
    for k in rev:
        tx, ty, ph = z_f[k]
        c, s = math.cos(ph), math.sin(ph)
        z[k] = [-(c * tx + s * ty), -(-s * tx + c * ty), wrap(-ph)]
        Jinv = np.array([[-c, -s, s * tx - c * ty], [s, -c, c * tx + s * ty], [0.0, 0.0, -1.0]])
        cov[k] = Jinv @ cov_f[k] @ Jinv.T
        src[k], dst[k] = dst[k], src[k]
    cov = 0.5 * (cov + np.transpose(cov, (0, 2, 1)))
    # world transform
    if world_rotation or np.any(world_translation):
        Rw = _rot_z(world_rotation)[:2, :2]
        t = np.asarray(world_translation, dtype=np.float64)
        for P in (truth, init):
            P[:, :2] = P[:, :2] @ Rw.T + t
            P[:, 2] = wrap(P[:, 2] + world_rotation)
    # insertion order of the connected nodes, then the isolated runs spliced in
    nc = len(truth)
    perm = {"chain": np.arange(nc), "reversed": np.arange(nc)[::-1], "shuffled": rng.permutation(nc)}[order]
    seq = [("c", int(i)) for i in perm]
    iso_poses = []
    for frac, length in sorted(isolated_runs, reverse=True):
        pos = max(1, min(len(seq), int(round(frac * len(seq)))))
        run = [("i", len(iso_poses) + k) for k in range(length)]
        iso_poses += [[rng.uniform(-50, 50), rng.uniform(-50, 50), rng.uniform(-math.pi, math.pi)] for _ in range(length)]
        seq[pos:pos] = run
    iso_poses = np.array(iso_poses, dtype=np.float64).reshape(-1, 3)
    N = len(seq)
    pos_of = np.empty(nc, dtype=np.int64)
    out_truth, out_init, out_comp = np.empty((N, 3)), np.empty((N, 3)), np.empty(N, dtype=np.int64)
    for p, (kind, i) in enumerate(seq):
        if kind == "c":
            pos_of[i] = p
            out_truth[p], out_init[p], out_comp[p] = truth[i], init[i], comp[i]
        else:
            out_truth[p] = out_init[p] = iso_poses[i]
            out_comp[p] = -1
    if ids == "dense":
        id_arr = np.arange(N, dtype=np.int32)
    elif ids == "sparse":
        lo, hi = np.iinfo(np.int32).min, np.iinfo(np.int32).max
        pool = np.setdiff1d(np.unique(np.concatenate([[-1, 0], rng.integers(lo + 1, hi, 4 * N + 8)])), [lo, hi])
        id_arr = rng.permutation(np.concatenate([[lo, hi], rng.permutation(pool)])[:N]).astype(np.int32)
    else:
        raise ValueError(f"unknown id scheme {ids!r}")
    ia, ib = pos_of[src], pos_of[dst]
    return dict(ids=id_arr, init=out_init, truth=out_truth, edge_a=id_arr[ia], edge_b=id_arr[ib], ia=ia, ib=ib,
                z=z, cov=cov, component=out_comp, anchor=0)


# ---------------------------------------------------------------------------------------------------------------------------
# Adversarial inputs for the batched sweep kernels: beams piled into one grid cell, tied best poses, very long queries.
# Each query and candidate block carries its own laser geometry (angle_min, angle_increment).
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class AdversarialSweep:
    query_ranges: np.ndarray          # (Q, n)
    query_poses: np.ndarray           # (Q, 3)
    cand_ranges: np.ndarray           # (S, m)
    cand_poses: np.ndarray            # (S, 3)
    chain_start: np.ndarray           # (C+1,)
    query_laser: tuple = (ANGLE_MIN, ANGLE_INC)
    cand_laser: tuple = (ANGLE_MIN, ANGLE_INC)


DENSE_INC = 1e-9   # rad: a cluster of 2000 beams at 13 m spans 26 um, so it sits in one 5 cm cell at every search angle


def make_dense_sweep(clusters=(640,), *, edge: bool = False, n_chains: int = 2, seed: int = 101) -> AdversarialSweep:
    """One query whose beams pile up in a few grid cells: cluster i is clusters[i] beams at one range, fanned over a few
    nano-radians, so every search angle puts the whole cluster in one cell (one descriptor group of that many beams).
    Candidates are room scans of make_loop_sweep around the query plus, per cluster, a scan from the query's pose that draws a
    ring at the cluster's range (so that the cluster's cell is occupied near the zero-offset pose).

    edge=True puts the clusters 12.3 m (and further) behind the query along -x: their pose window leaves the correlation grid
    (range threshold 12 m) through its left side, so they are EDGE beams with row-wrapped (wrap2) entries."""
    ls = make_loop_sweep(seed, n_queries=1, n_chains=n_chains, chain_len=1)
    q = ls.query_poses[0].copy()
    if edge:
        q[2] = math.pi
        radii = [12.3 + 0.35 * i for i in range(len(clusters))]
    else:
        radii = [0.55 + 0.35 * i for i in range(len(clusters))]
    qr = np.concatenate([np.full(k, r) for k, r in zip(clusters, radii)])
    rings = np.array([np.full(N_BEAMS, r) for r in radii])
    cr = np.concatenate([ls.cand_ranges, rings])
    cp = np.concatenate([ls.cand_poses, np.repeat(q[None, :], len(radii), axis=0)])
    chain_start = np.append(np.arange(n_chains + 1), len(cr)).astype(np.int32)   # one room scan per chain, then the rings
    return AdversarialSweep(qr[None, :], q[None, :], cr, cp, chain_start, (0.0, DENSE_INC), (ANGLE_MIN, ANGLE_INC))


# Query beams (index into the 1081-beam laser, range in m) whose coarse volume against make_tie_sweep's one-point candidate has
# exactly k maximal poses (response 1/1081), on the 4 m / 0.05 m grid with +-20 deg at 2 deg.  Found once with the oracle; pinned
# by tests/test_sweep_fixtures.py.
TIE_BEAMS = {
    1: ((770, 0.15),),
    2: ((536, 0.15),),
    23: ((16, 0.3), (224, 1.9), (640, 1.9), (1069, 0.3)),
    24: ((107, 0.5), (172, 1.9), (237, 1.6), (744, 0.5)),
    25: ((367, 1.9), (601, 0.5), (770, 0.15), (848, 1.6), (939, 1.6), (1056, 1.6)),
    100: ((55, 0.15), (68, 1.6), (81, 1.9), (120, 1.6), (198, 1.6), (302, 0.3), (432, 1.9), (536, 0.5), (705, 0.3), (757, 1.9),
          (809, 0.5), (848, 1.9), (887, 1.6), (913, 0.3), (965, 1.9), (1043, 0.5)),
}
TIE_POSE = (10.0, 12.0, 0.3)
TIE_CAND_LASER = (0.0, 0.5 * math.pi)
TIE_CAND_RANGES = (0.3, 5.0)   # FindValidPoints keeps the first reading only: one occupied cell, 0.3 m ahead of the query


def make_tie_sweep(ks=(1, 2, 23, 24, 25, 100), n_cands: int = 1) -> AdversarialSweep:
    """Queries with a few finite readings (the rest inf) against a candidate that rasterises to a single occupied cell: every
    pose that puts one reading on that cell scores 100, nothing scores more, and the readings are far enough apart that no pose
    puts two of them near it.  Query i has exactly ks[i] tied best poses, spread over the angles.  n_cands identical candidates,
    one per chain."""
    qr = np.full((len(ks), N_BEAMS), np.inf)
    for row, k in enumerate(ks):
        for i, d in TIE_BEAMS[k]:
            qr[row, i] = d
    qp = np.repeat(np.array([TIE_POSE]), len(ks), axis=0)
    cr = np.repeat(np.array([TIE_CAND_RANGES]), n_cands, axis=0)
    cp = np.repeat(np.array([TIE_POSE]), n_cands, axis=0)
    return AdversarialSweep(qr, qp, cr, cp, np.arange(n_cands + 1, dtype=np.int32), (ANGLE_MIN, ANGLE_INC), TIE_CAND_LASER)


def highres_laser(n_beams: int, fov_deg: float) -> tuple:
    """(angle_min, angle_increment) of a laser with n_beams readings centred on the sensor's x axis: fov_deg from the first
    to the last reading, or, for a full circle (fov_deg >= 360), n_beams readings spaced 360 / n_beams degrees."""
    fov = math.radians(fov_deg)
    inc = fov / n_beams if fov_deg >= 360.0 else fov / (n_beams - 1)
    return -0.5 * fov, inc


def make_highres_sweep(n_beams: int, fov_deg: float, *, seed: int = 11, n_queries: int = 1, n_chains: int = 2,
                       chain_len: int = 1, radius: float = 3.0, inf_frac: float = 0.0) -> AdversarialSweep:
    """Room scans from one dense laser (highres_laser(n_beams, fov_deg)) for the queries and the candidates: the shape of a
    0.1 deg lidar (2701 beams over 270 deg, 3600 over 360 deg) or of a 3-D lidar flattened to a scan.  Queries sit in a
    room of make_world(seed) with make_loop_sweep's drift; candidate chains start within `radius` of the first query."""
    rng = np.random.default_rng(seed)
    world = make_world(seed)
    amin, inc = highres_laser(n_beams, fov_deg)
    qtrue = np.array([free_pose(world, rng) for _ in range(n_queries)])
    qr = noisy(raycast(world, qtrue, n_beams=n_beams, angle_min=amin, angle_inc=inc), rng, inf_frac=inf_frac)
    qpose = qtrue + np.column_stack([rng.normal(0, 0.5, (n_queries, 2)), rng.normal(0, 0.08, n_queries)])
    starts = poses_near(world, qtrue[0, :2], radius, n_chains, rng)
    cposes = starts if chain_len == 1 else np.concatenate([chain_poses(world, s, chain_len, rng) for s in starts])
    cr = noisy(raycast(world, cposes, n_beams=n_beams, angle_min=amin, angle_inc=inc), rng, inf_frac=inf_frac)
    chain_start = np.arange(0, n_chains * chain_len + 1, chain_len, dtype=np.int32)
    return AdversarialSweep(qr, qpose, cr, cposes, chain_start, (amin, inc), (amin, inc))


WEIGHTED_BEAMS = 8192   # laser of make_weighted_sweep: 360 deg at 0.044 deg


def make_weighted_sweep(weights, *, resolution: float = 0.05, r_min: float = 1.5, r_max: float = 4.0,
                        seed: int = 111) -> AdversarialSweep:
    """One query whose beams land in chosen cells: cell i is hit by weights[i] neighbouring beams of a 8192-beam, 360 deg laser.
    At the query's own heading (the central search angle) every cell is 8 columns x 2 rows apart on the query-centred cell
    lattice, so they all fall in ONE (parity phase, alignment) descriptor group, whose weight is sum(weights); the other angles
    shuffle them over the groups.  The cells lie r_min..r_max from the query (at most 12 mm off a cell centre at 4 m for a
    weight of 10), the other readings are inf.  Candidates: chain 0 a room scan, chain 1 the query's own scan, chain 2 both."""
    ls = make_loop_sweep(seed, n_queries=1, n_chains=2, chain_len=1)
    q = ls.query_poses[0].copy()
    q[2] = 0.0
    amin, inc = highres_laser(WEIGHTED_BEAMS, 360.0)
    lim = int(r_max / resolution) + 8
    u = np.arange(-lim, lim + 1, 8)
    v = np.arange(-lim, lim + 1, 2)
    gx, gy = np.meshgrid(u, v)
    pts = np.column_stack([gx.ravel(), gy.ravel()]) * resolution
    rad = np.hypot(pts[:, 0], pts[:, 1])
    pts, rad = pts[(rad >= r_min) & (rad <= r_max)], rad[(rad >= r_min) & (rad <= r_max)]
    beam = np.rint((np.arctan2(pts[:, 1], pts[:, 0]) - amin) / inc).astype(int) % WEIGHTED_BEAMS
    order = np.argsort(beam, kind="stable")
    qr = np.full(WEIGHTED_BEAMS, np.inf)
    nxt, k = 0, 0
    for i in order:   # cells in bearing order, each on its own run of beams with one beam between runs
        if k == len(weights):
            break
        w = int(weights[k])
        b0 = beam[i] - w // 2
        if b0 < nxt or b0 + w > WEIGHTED_BEAMS:
            continue
        qr[b0:b0 + w] = rad[i]
        nxt, k = b0 + w + 1, k + 1
    if k < len(weights):
        raise ValueError(f"only {k} of {len(weights)} cells fit r_min..r_max")
    room = raycast(ls.world, ls.cand_poses, n_beams=WEIGHTED_BEAMS, angle_min=amin, angle_inc=inc)
    cr = np.concatenate([room[:1], qr[None, :], room[1:2], qr[None, :]])
    cp = np.concatenate([ls.cand_poses[:1], q[None, :], ls.cand_poses[1:2], q[None, :]])
    return AdversarialSweep(qr[None, :], q[None, :], cr, cp, np.array([0, 1, 2, 4], dtype=np.int32), (amin, inc), (amin, inc))


def make_long_query_sweep(n: int, seed: int = 7, n_chains: int = 3, inf_frac: float = 0.97) -> AdversarialSweep:
    """One query of n beams over the usual 270 deg field of view (a room scan at n / 1081 times the angular density, a fraction
    inf_frac of the readings replaced by inf) and n_chains room-scan candidates.  With the defaults, n = 10240 and the 4 m /
    0.05 m grid with a 0.05 m smear (5 x 5 kernel) at +-2 deg / 2 deg, chain 1's best two integer sums are s and s - 1: their
    responses differ by 1 / (100 n) < 1e-6, so both count as ties of the best."""
    ls = make_loop_sweep(seed, n_queries=1, n_chains=n_chains, chain_len=1)
    inc = (ANGLE_MAX - ANGLE_MIN) / (n - 1)
    rng = np.random.default_rng(seed)
    qr = noisy(raycast(ls.world, ls.query_true, n_beams=n, angle_inc=inc), rng)
    qr[:, rng.random(n) < inf_frac] = np.inf
    return AdversarialSweep(qr, ls.query_poses, ls.cand_ranges, ls.cand_poses, ls.chain_start, (ANGLE_MIN, inc), (ANGLE_MIN, ANGLE_INC))


# ---------------------------------------------------------------------------------------------------------------------------
# Single-match inputs (one query against a running buffer of base scans) at the poses, beam counts and rasters the sequential
# cases never produce.  A base scan given as points carries them directly (ranges = distances from its pose), so a test can build
# rasters no laser draws.
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class SingleMatchCase:
    query_ranges: np.ndarray          # (n,)
    query_pose: np.ndarray            # (3,)  reported sensor pose
    base_ranges: np.ndarray           # (B, m)
    base_poses: np.ndarray            # (B, 3)
    query_laser: tuple = (ANGLE_MIN, ANGLE_INC)
    base_laser: tuple = (ANGLE_MIN, ANGLE_INC)


def _move_scene(poses: np.ndarray, src: np.ndarray, dst: np.ndarray) -> np.ndarray:
    """poses (N,3) under the rigid motion that takes pose src to pose dst (headings are not wrapped)"""
    c, s = math.cos(dst[2] - src[2]), math.sin(dst[2] - src[2])
    dx, dy = poses[:, 0] - src[0], poses[:, 1] - src[1]
    return np.column_stack([dst[0] + c * dx - s * dy, dst[1] + s * dx + c * dy, poses[:, 2] + (dst[2] - src[2])])


def make_single_match_case(seed: int, *, query: str = "match", search_size: float = 1.0, buffer_len: int = 6,
                           n_beams: int = N_BEAMS, fov_deg: float = 270.0, pose=None, inf_frac: float = 0.02) -> SingleMatchCase:
    """One query against a chain of buffer_len room scans (the standard laser) spaced 0.5 m, ending at the query's true pose.

    query      'match'    reported pose = true pose + odometry noise
               'partial'  reported 0.75 * search_size off in x (beyond the search window's half width) and 0.05 rad off: only
                          part of the scan lines up anywhere in the window
               'far'      all but the shortest tenth of the readings dropped (inf), reported left of every base point by more
                          than those readings, the search window and the smear can bridge: the best response is zero, but the correlation grid (centred on the
                          reported pose, range threshold >= 6 m) still holds base points
    n_beams, fov_deg   the query's laser (highres_laser); the base scans keep the standard laser
    pose       if given, the whole scene is moved rigidly so that the reported query pose is exactly `pose` (the origin, a
               heading near +-pi or beyond 2 pi, large world coordinates)"""
    rng = np.random.default_rng(seed)
    world = make_world(seed)
    traj = chain_poses(world, free_pose(world, rng), buffer_len + 1, rng)
    qtrue = traj[-1]
    base_ranges = noisy(raycast(world, traj[:-1]), rng, inf_frac=inf_frac)
    amin, inc = highres_laser(n_beams, fov_deg) if n_beams != N_BEAMS else (ANGLE_MIN, ANGLE_INC)
    qr = noisy(raycast(world, qtrue, n_beams=n_beams, angle_min=amin, angle_inc=inc), rng, inf_frac=inf_frac)[0]
    reported = qtrue + np.array([rng.normal(0, 0.03), rng.normal(0, 0.03), rng.normal(0, 0.01)])
    if query == "partial":
        reported = qtrue + np.array([0.75 * search_size, 0.0, 0.05])
    elif query == "far":
        short_range = np.sort(qr[np.isfinite(qr)])[np.isfinite(qr).sum() // 10]
        qr = np.where(qr > short_range, np.inf, qr)
        ang = traj[:-1, 2:3] + ANGLE_MIN + np.arange(N_BEAMS) * ANGLE_INC
        px = np.where(np.isfinite(base_ranges), traj[:-1, 0:1] + base_ranges * np.cos(ang), np.inf)
        reported = np.array([px.min() - (short_range + 0.75 * search_size + 1.5), qtrue[1], qtrue[2]])
    elif query != "match":
        raise ValueError(f"unknown query kind {query!r}")
    base_poses = traj[:-1]
    if pose is not None:
        pose = np.asarray(pose, dtype=np.float64)
        base_poses = _move_scene(base_poses, reported, pose)
        reported = pose.copy()
    return SingleMatchCase(qr, reported, base_ranges, base_poses, (amin, inc), (ANGLE_MIN, ANGLE_INC))


def make_few_beam_query(case: SingleMatchCase, n_readings: int) -> SingleMatchCase:
    """The case's query with all but n_readings evenly spread readings replaced by inf"""
    keep = np.linspace(0, len(case.query_ranges) - 1, n_readings).astype(int)
    qr = np.full_like(case.query_ranges, np.inf)
    qr[keep] = case.query_ranges[keep]
    return SingleMatchCase(qr, case.query_pose, case.base_ranges, case.base_poses, case.query_laser, case.base_laser)


def half_cell_centres(offset: float, resolution: float, cells, ulps: int = 2) -> np.ndarray:
    """Coordinates offset + (k + 0.5) * resolution for every k in cells, each also moved by 1..ulps units in the last place either
    way: the centres where a fine search's cell map rounds in both directions"""
    scale = 1.0 / resolution
    out = []
    for k in cells:
        c = offset + (k + 0.5) / scale
        for d in range(-ulps, ulps + 1):
            x = c
            for _ in range(abs(d)):
                x = float(np.nextafter(x, np.inf if d > 0 else -np.inf))
            out.append(x)
    return np.array(out)


def points_scan(points: np.ndarray, pose) -> tuple:
    """(ranges, points, pose) of a base scan given by its points"""
    pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 2)
    pose = np.asarray(pose, dtype=np.float64)
    return np.hypot(pts[:, 0] - pose[0], pts[:, 1] - pose[1]), pts, pose


def make_dense_base(center, resolution: float, n_clusters: int = 12, per_cluster: int = 300, radius: float = 1.2,
                    seed: int = 5) -> list:
    """One base scan whose points pile up in few cells: n_clusters clusters of per_cluster points, each within a tenth of a cell,
    on a circle of `radius` around `center` (a sensor there), visited counter-clockwise so that FindValidPoints keeps every
    cluster but the last"""
    rng = np.random.default_rng(seed)
    c = np.asarray(center, dtype=np.float64)
    pts = []
    for k in range(n_clusters):
        a = 2 * math.pi * k / n_clusters
        p = c[:2] + radius * np.array([math.cos(a), math.sin(a)])
        pts.append(p + rng.uniform(-0.05 * resolution, 0.05 * resolution, (per_cluster, 2)))
    return [points_scan(np.concatenate(pts), c)]


def make_roi_edge_base(query_pose, resolution: float, roi_w: int) -> list:
    """Base scans on the border of the correlation grid's region of interest around query_pose (roi_w cells wide, the grid
    offset of ScanMatcher::MatchScan, Mapper.cpp:560-569): one scan along the first and last ROI rows and columns, one along
    the cells just outside them, both counter-clockwise around the query"""
    q = np.asarray(query_pose, dtype=np.float64)
    res = 1.0 / (1.0 / resolution)
    off = q[:2] - 0.5 * (roi_w - 1) * res
    out = []
    for lo, hi in ((0, roi_w - 1), (-1, roi_w)):
        k = np.arange(lo, hi)
        ring = np.concatenate([np.column_stack([k, np.full_like(k, lo)]), np.column_stack([np.full_like(k, hi), k]),
                               np.column_stack([hi - (k - lo), np.full_like(k, hi)]),
                               np.column_stack([np.full_like(k, lo), hi - (k - lo)])])
        out.append(points_scan(off[None, :] + ring * res, q))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# Crafted occupancy-grid inputs: readings along exact axes, at half cells and where a fused multiply-add would round the
# clipped end of an over-range beam into another cell.  LocalizedRangeScan::Update computes a beam's angle as
# (heading + angle_min) + k * angle_increment; a heading can make that exactly 0, +-pi/2 (as doubles) or pi for many beams k.
# cos(0) = 1, sin(0) = 0 and cos(pi) = -1 in double, so such a beam's point is (x + r, y), (x - r, ~y); at +-pi/2 the y
# coordinate is y +- r.  Scans are the standard laser with every other reading inf.
# ---------------------------------------------------------------------------------------------------------------------------
AXIS_ANGLES = {"+x": 0.0, "+y": math.pi / 2, "-y": -math.pi / 2, "-x": math.pi}


def _ulp_steps(x: float, n: int):
    """x moved by -n..n units in the last place"""
    out = [x]
    lo = hi = x
    for _ in range(n):
        lo, hi = float(np.nextafter(lo, -np.inf)), float(np.nextafter(hi, np.inf))
        out += [lo, hi]
    return out


def exact_axis_heading(k: int, direction: str, angle_min: float = ANGLE_MIN, angle_inc: float = ANGLE_INC):
    """A heading h in [-pi, pi] with (h + angle_min) + k * angle_inc == AXIS_ANGLES[direction] in double, or None"""
    target = AXIS_ANGLES[direction]
    a = k * angle_inc
    for b in _ulp_steps(target - a, 2):
        if b + a != target:
            continue
        for h in _ulp_steps(b - angle_min, 3):
            if h + angle_min == b and -math.pi <= h <= math.pi:
                return h
    return None


def exact_axis_beams(direction: str, n_beams: int = N_BEAMS) -> list:
    """[(beam index, heading)] of every beam that a heading puts exactly on the axis direction"""
    out = []
    for k in range(n_beams):
        h = exact_axis_heading(k, direction)
        if h is not None:
            out.append((k, h))
    return out


def axis_scan(sensor_xy, direction: str, readings, n_beams: int = N_BEAMS, which: int = 0) -> tuple:
    """(ranges, pose) of one scan whose exact-axis beams point along `direction` from sensor_xy.  readings = the ranges of
    the beams: only one beam of a scan can lie exactly on an axis, so readings[0] goes there and any further readings go to
    the beams right after it (a few hundredths of a degree off the axis).  `which` picks one of the exact beams."""
    k, h = exact_axis_beams(direction, n_beams)[which]
    r = np.full(n_beams, np.inf)
    readings = np.atleast_1d(np.asarray(readings, dtype=np.float64))
    assert k + len(readings) <= n_beams
    r[k:k + len(readings)] = readings
    return r, np.array([float(sensor_xy[0]), float(sensor_xy[1]), h])


def clipped_end(s: float, p: float, r: float, rt: float) -> float:
    """AddScan's end of an over-range beam along one axis, rounded like the reference (no fused multiply-add):
    s + (rt / r) * (p - s)"""
    return s + (rt / r) * (p - s)


def clipped_end_fused(s: float, p: float, r: float, rt: float) -> float:
    """the same end with s + ratio * dx fused into one rounding (exact rational arithmetic, rounded once)"""
    from fractions import Fraction
    ratio, dx = rt / r, p - s
    return float(Fraction(s) + Fraction(ratio) * Fraction(dx))


def grid_cell(w: float, offset: float, scale: float) -> int:
    """CoordinateConverter::WorldToGrid on one axis: round half away from zero of (w - offset) * scale"""
    v = (w - offset) * scale
    return int(math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5))


def fma_sensitive_beams(boundary: float, offset: float, resolution: float, rt: float, n: int, seed: int, direction: str = "+x",
                        max_r: float = RANGE_MAX) -> list:
    """n (sensor coordinate, range) pairs of over-range axis beams (rt < r < max_r) whose clipped end lands in a different
    grid cell when s + ratio * dx is fused: sensor coordinates step by units in the last place around boundary -+ rt."""
    rng = np.random.default_rng(seed)
    scale = 1.0 / resolution
    sign = 1.0 if direction in ("+x", "+y") else -1.0
    s0 = boundary - sign * rt
    out, seen = [], set()
    steps = _ulp_steps(s0, 64)
    while len(out) < n:
        s = steps[int(rng.integers(len(steps)))]
        r = float(rng.uniform(rt * 1.0001, max_r * 0.999))
        p = s + sign * r
        e, f = clipped_end(s, p, r, rt), clipped_end_fused(s, p, r, rt)
        if grid_cell(e, offset, scale) != grid_cell(f, offset, scale) and (s, r) not in seen:
            seen.add((s, r))
            out.append((s, r))
    return out
