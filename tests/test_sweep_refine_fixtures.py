"""The inputs of tests/test_sweep_refine_gpu.py checked against the oracle alone: every pair of the refined batches reaches the
branch of the batch's fetch it was built for, so that a generator that drifts off its branch fails on any machine.

A refined batch (MatchScanBatch with doRefineMatch) finishes each pair in one of these ways:
  plain     the coarse reduction is finished on the host, then the fine pass (3 x 3 x nA around the coarse mean) runs on the
            device and its FP64 epilogue on the host;
  zero      every coarse pose ties at response 0: the closed form of the all-poses average (counted in zero_pairs), then the
            fine pass;
  fallback  more than 24 tied coarse poses, or a zero response under use_response_expansion while the raster holds cells: the
            pair is re-run whole through the single-match path during the coarse fetch (counted in fallback_pairs) and the fine
            pass must leave its row alone.
A plain or zero pair whose averaged fine pose rounds to a cell outside the 3 x 3 searched ones is re-run through the single-match
path after the fine pass (the fine-covariance fallback, also counted in fallback_pairs).

The cases are defined here and imported by the GPU test."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import pytest

from oracle import karto_port as P
from slam_toolbox_b200 import synth
import helpers as H
import test_single_match_fixtures as SM

MAX_TIES = 24   # tie indices a pair returns from the device; more -> the single-match path

# the near-chain and loop-closure fine stages: the sequential matcher's parameters, doPenalize = false
MAPPER_EXP = H.MAPPER_SEQ                                     # use_response_expansion = 1, the toolbox default
MAPPER_NOEXP = dict(H.MAPPER_SEQ, use_response_expansion=0)
MIXED_GRID = H.GRID_SEQ_YAML                                  # the shipped smear: order-dependent raster, generic kernel only

# Shifts of fallback_case(n)'s reported pose whose coarse pass ties at four poses that average onto a half-cell boundary of the
# query's grid, so that the fine pass centred there averages its best poses onto a cell between the searched ones.  A batch
# only reaches the fine-covariance fallback through such a coarse mean (the grid is centred on the query, so a single coarse
# winner always sits on a whole cell).  Found once with the oracle; pinned by test_fallback_shifts_reach_the_fine_fallback.
# The 7- and 9-reading queries of SM.FALLBACK_READINGS seldom tie at four coarse poses: none of 6,000 random shifts of either
# reached the fallback, so only the 3-reading query is used here.
FALLBACK_SHIFTS = {3: ((-0.3198, -0.3406, -0.0593), (0.2607, 0.2804, -0.0912))}

TIE_BEAM, TIE_RANGE = 540, 1.0   # the one finite reading of the tie query: straight ahead, 1 m
WALL_HALF, WALL_STEP = 0.8, 0.004
FAR_SHIFT = 300.0                # a chain this far away puts no point in the query's grid
BEHIND_RANGE, BEHIND_HALF = 8.3, 0.3   # a short wall this far behind the query: inside its grid, where no reading looks


class Scan:
    """one scan as both implementations take it (ranges, points, sensor pose), the buffers kept alive here; .c is the oracle's
    record, the GPU test builds its own from the same buffers"""

    def __init__(self, ranges, points, pose):
        self.ranges = np.ascontiguousarray(ranges, dtype=np.float64).reshape(-1)
        self.points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 2)
        self.pose = np.ascontiguousarray(pose, dtype=np.float64).reshape(3)
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
        self.c = P.KpScan(len(self.ranges), dp(self.ranges), dp(self.points), (C.c_double * 3)(*self.pose))


def laser_scan(ranges, pose, laser=(synth.ANGLE_MIN, synth.ANGLE_INC)) -> Scan:
    return Scan(ranges, P.point_readings(ranges, pose, *laser), pose)


def points_scan(points, pose) -> Scan:
    return Scan(*synth.points_scan(points, pose))


def wall_scan(pose, bearing, distance, half) -> Scan:
    """a straight wall of points WALL_STEP apart, `distance` from the pose along `bearing` and perpendicular to it, 2 * half long,
    in counter-clockwise order around the pose like a laser's readings (FindValidPoints' side test keeps them)"""
    u, v = np.array([math.cos(bearing), math.sin(bearing)]), np.array([-math.sin(bearing), math.cos(bearing)])
    s = np.arange(-half, half + WALL_STEP / 2, WALL_STEP)
    return points_scan(pose[:2] + distance * u + s[:, None] * v[None, :], pose)


@dataclass
class Batch:
    """queries, candidate scans, chain_start and an explicit pair list (pair_query, pair_chain), with a name per pair"""
    queries: list
    scans: list
    chain_start: np.ndarray
    pair_query: np.ndarray
    pair_chain: np.ndarray
    names: list

    def chain(self, c):
        return self.scans[self.chain_start[c]:self.chain_start[c + 1]]

    def pairs(self):
        return [(int(q), int(c)) for q, c in zip(self.pair_query, self.pair_chain)]


def batch(queries, chains, pairs, names=None) -> Batch:
    scans = [s for ch in chains for s in ch]
    chain_start = np.concatenate([[0], np.cumsum([len(ch) for ch in chains])]).astype(np.int32)
    pq = np.array([p[0] for p in pairs], dtype=np.int32)
    pc = np.array([p[1] for p in pairs], dtype=np.int32)
    return Batch(queries, scans, chain_start, pq, pc, names or [f"q{q}c{c}" for q, c in pairs])


# ---- the mixed batch -------------------------------------------------------------------------------------------------------------
def mixed_batch() -> Batch:
    """One refined batch on MIXED_GRID whose pairs take every branch of the fetch, fallbacks between ordinary pairs:
    the queries are the few-reading queries of fallback_case (all 1081 readings long, the rest inf) and one single-reading query;
    the chains are fallback_case's room scans, an empty chain, the room scans 300 m away, a short wall behind the query, and a
    long wall across the single reading."""
    plain = SM.fallback_case(9)
    true = plain.query_pose
    base = [laser_scan(r, p) for r, p in zip(plain.base_ranges, plain.base_poses)]
    queries = [laser_scan(plain.query_ranges, true)]
    for n, shifts in FALLBACK_SHIFTS.items():
        c = SM.fallback_case(n)
        queries += [laser_scan(c.query_ranges, c.query_pose + np.array(s)) for s in shifts]
    tie = np.full(synth.N_BEAMS, np.inf)
    tie[TIE_BEAM] = TIE_RANGE
    queries.append(laser_scan(tie, true))
    q_tie = len(queries) - 1
    # the wall: through the reading's end point, perpendicular to the beam, points in counter-clockwise order around the query
    # (FindValidPoints keeps them all); at every search angle a band of poses along the wall puts the reading on it
    wall = wall_scan(true, true[2] + synth.ANGLE_MIN + TIE_BEAM * synth.ANGLE_INC, TIE_RANGE, WALL_HALF)
    far = [Scan(b.ranges, b.points + FAR_SHIFT, b.pose + np.array([FAR_SHIFT, FAR_SHIFT, 0.0])) for b in base]
    behind = wall_scan(true, true[2] + math.pi, BEHIND_RANGE, BEHIND_HALF)
    chains = [base, [], far, [behind], [wall]]
    pairs = [(0, 0, "plain")]
    pairs += [(1 + k, 0, f"fine_fallback_{k}") for k in range(len(queries) - 2)]
    pairs += [(q_tie, 4, "tie_overflow"), (0, 0, "plain_repeat"), (0, 2, "zero_far"), (q_tie, 0, "plain_tie_query"),
              (0, 3, "zero_behind"), (0, 1, "empty_chain"), (0, 0, "plain_after_empty")]
    return batch(queries, chains, [p[:2] for p in pairs], [p[2] for p in pairs])


# ---- branch of a pair, from the oracle ---------------------------------------------------------------------------------------------
@dataclass
class Branch:
    coarse: str          # plain / zero / fallback
    fine_outside: bool   # the fine pass's averaged pose rounds outside its 3 x 3 cells (plain / zero only)
    ties: int            # poses with the best coarse integer sum
    best_sum: int
    empty_raster: bool


def fine_rounds_outside(pm, mapper, grid, q, centre) -> bool:
    """the fine pass of MatchScan centred on `centre` (the raster of the pair must be the oracle's current one): does its
    averaged best pose round to a cell outside the 3 x 3 cells it searched?"""
    offx, offy = pm.grid()["offset"]
    so, sr, ao, ar = SM.fine_window(mapper, grid)
    _, mean, _, _ = pm.correlate(q, centre, so, sr, ao, ar, False, True)
    xs = {SM.world_to_grid(centre[0] + (-so[0] + k * sr[0]), offx, grid[1]) for k in range(3)}
    ys = {SM.world_to_grid(centre[1] + (-so[1] + k * sr[1]), offy, grid[1]) for k in range(3)}
    return SM.world_to_grid(mean[0], offx, grid[1]) not in xs or SM.world_to_grid(mean[1], offy, grid[1]) not in ys


def branch(pm, mapper, grid, q, base) -> Branch:
    """which branch of the refined batch's fetch the pair (q, base) takes, doPenalize = false"""
    pm.raster(q, base)
    empty = int(pm.grid()["data"].max()) == 0
    so, sr = H.coarse_search(grid)
    vol = pm.correlate(q, q.pose, so, sr, mapper["coarse_search_angle_offset"], mapper["coarse_angle_resolution"], False, False)[3]
    best = int(vol.max())
    ties = int((vol == best).sum())   # below 9000 readings DoubleEqual of the responses is equality of the integer sums
    if best == 0 and mapper["use_response_expansion"]:
        coarse = "zero" if empty else "fallback"
    elif best == 0 and ties == vol.size and ties > MAX_TIES:
        coarse = "zero"
    elif ties > MAX_TIES:
        coarse = "fallback"
    else:
        coarse = "plain"
    outside = False
    if coarse != "fallback":
        mean = pm.match(q, base, False, False)[1]   # the coarse result, after the response-expansion passes
        outside = fine_rounds_outside(pm, mapper, grid, q, mean)
    return Branch(coarse, outside, ties, best, empty)


def branches(b: Batch, mapper, grid):
    pm = H.port_matcher(mapper, grid)
    return [branch(pm, mapper, grid, b.queries[q], b.chain(c)) for q, c in b.pairs()]


def fetch_stats(brs):
    """(zero_pairs, fallback_pairs) that batch_fetch_stats reports after a refined batch with these branches"""
    zero = sum(br.coarse == "zero" for br in brs)
    fallback = sum(br.coarse == "fallback" for br in brs) + sum(br.fine_outside for br in brs)
    return zero, fallback


# ---- the near-chain batch (LinkNearChains: one query against each near chain) ------------------------------------------------------
NEAR_CHAIN_LENGTHS = (10, 0, 3, 1)


def near_chain_batch() -> Batch:
    """Three queries at distinct poses (the case's query as reported and moved, and a scan of the running buffer moved off its
    pose) against chains of 10, 0, 3 and 1 scans of the buffer; every (query, chain) pair, out of order, one of them twice"""
    c = synth.make_sequential_case(5, buffer_len=sum(NEAR_CHAIN_LENGTHS))
    scans = [laser_scan(r, p) for r, p in zip(c["base_ranges"], c["base_poses"])]
    queries = [laser_scan(c["query_ranges"], c["query_pose"]),
               laser_scan(c["query_ranges"], c["query_true"] + np.array([0.04, -0.03, 0.02])),
               laser_scan(c["base_ranges"][-2], c["base_poses"][-2] + np.array([-0.05, 0.02, -0.015]))]
    starts = np.concatenate([[0], np.cumsum(NEAR_CHAIN_LENGTHS)])
    chains = [scans[starts[k]:starts[k + 1]] for k in range(len(NEAR_CHAIN_LENGTHS))]
    pairs = [(2, 3), (0, 3), (1, 0), (0, 2), (2, 2), (1, 1), (0, 0), (2, 0), (1, 3), (0, 3), (2, 1), (1, 2), (0, 1)]
    return batch(queries, chains, pairs)


# ---- the loop-closure two-stage batch ----------------------------------------------------------------------------------------------
LOOP_DRIFTS = ((0.3, -0.2, 0.05), (-0.25, 0.35, -0.04), (0.1, 0.15, 0.07))


def loop_batch() -> Batch:
    """TryCloseLoop's coarse stage: one room scan reported at three drifted poses against six chains of three scans around it"""
    sw = synth.make_loop_sweep(17, n_queries=1, n_chains=6, chain_len=3, radius=2.0, inf_frac=0.02)
    queries = [laser_scan(sw.query_ranges[0], sw.query_true[0] + np.array(d)) for d in LOOP_DRIFTS]
    scans = [laser_scan(r, p) for r, p in zip(sw.cand_ranges, sw.cand_poses)]
    chains = [scans[sw.chain_start[k]:sw.chain_start[k + 1]] for k in range(len(sw.chain_start) - 1)]
    return batch(queries, chains, [(q, c) for q in range(len(queries)) for c in range(len(chains))])


def refine_stage(b: Batch, response, mean) -> Batch:
    """TryCloseLoop's fine stage: each query moved to the coarse best pose of its best chain (the first of equal responses; its
    points recomputed at that pose, as SetSensorPose makes the scan do), against that chain"""
    nq = len(b.queries)
    r = np.asarray(response).reshape(nq, -1)
    win = [int(np.argmax(r[q])) for q in range(nq)]
    queries = [laser_scan(b.queries[q].ranges, np.asarray(mean).reshape(nq, -1, 3)[q, win[q]]) for q in range(nq)]
    chains = [b.chain(c) for c in range(len(b.chain_start) - 1)]
    return batch(queries, chains, [(q, win[q]) for q in range(nq)])


# --------------------------------------------------------------------------------------------------------------------------------
def test_generators_are_deterministic():
    for make in (mixed_batch, near_chain_batch, loop_batch):
        a, b = make(), make()
        assert a.names == b.names and np.array_equal(a.chain_start, b.chain_start)
        assert np.array_equal(a.pair_query, b.pair_query) and np.array_equal(a.pair_chain, b.pair_chain)
        for x, y in zip(a.queries + a.scans, b.queries + b.scans):
            assert np.array_equal(x.ranges, y.ranges) and np.array_equal(x.points, y.points) and np.array_equal(x.pose, y.pose)


@pytest.mark.parametrize("n", sorted(FALLBACK_SHIFTS))
def test_fallback_shifts_reach_the_fine_fallback(n):
    """the coarse pass is finished on the host (at most 24 ties, a positive best) and its mean centres a fine pass whose
    averaged best pose rounds outside the 3 x 3 searched cells"""
    mapper, grid = MAPPER_EXP, MIXED_GRID
    case = SM.fallback_case(n)
    assert np.isfinite(case.query_ranges).sum() == n
    pm = H.port_matcher(mapper, grid)
    base = [laser_scan(r, p) for r, p in zip(case.base_ranges, case.base_poses)]
    for s in FALLBACK_SHIFTS[n]:
        q = laser_scan(case.query_ranges, case.query_pose + np.array(s))
        br = branch(pm, mapper, grid, q, base)
        assert br.coarse == "plain" and br.best_sum > 0 and br.fine_outside, (s, br)
        assert br.ties % 4 == 0, (s, br)   # a half-cell mean needs a multiple of four tied poses


def test_mixed_batch_reaches_every_branch():
    b = mixed_batch()
    assert len({len(q.ranges) for q in b.queries}) == 1                # one reading count for every query of a batch
    assert [len(b.chain(c)) for c in range(len(b.chain_start) - 1)] == [4, 0, 4, 1, 1]
    wall = b.chain(4)[0]
    assert len(P.find_valid_points(wall, b.queries[-1].pose)) >= 0.9 * len(wall.ranges)   # the side test keeps the wall
    for mapper in (MAPPER_EXP, MAPPER_NOEXP):
        brs = dict(zip(b.names, branches(b, mapper, MIXED_GRID)))
        exp = bool(mapper["use_response_expansion"])
        for name, br in brs.items():
            if name.startswith("plain"):
                assert br.coarse == "plain" and br.best_sum > 0 and not br.fine_outside, (name, br)
            elif name.startswith("fine_fallback"):
                assert br.coarse == "plain" and br.fine_outside, (name, br)
        assert brs["tie_overflow"].coarse == "fallback" and brs["tie_overflow"].ties > MAX_TIES and brs["tie_overflow"].best_sum == 100
        for name in ("zero_far", "empty_chain"):
            assert brs[name].empty_raster and brs[name].best_sum == 0 and brs[name].coarse == "zero", (name, brs[name])
        # the wall behind the query is in its grid but under no reading: zero response with a raster -> the expansion passes
        # could see it, so the pair goes through the single-match path; without expansion it is the closed form
        zb = brs["zero_behind"]
        assert not zb.empty_raster and zb.best_sum == 0 and zb.coarse == ("fallback" if exp else "zero"), zb
        n_fine = sum(len(v) for v in FALLBACK_SHIFTS.values())
        assert fetch_stats(brs.values()) == ((2, 2 + n_fine) if exp else (3, 1 + n_fine))


@pytest.mark.parametrize("grid", [H.GRID_SEQ, H.GRID_SEQ_YAML], ids=["karto_smear", "yaml_smear"])
def test_near_chain_pairs_have_real_answers(grid):
    b = near_chain_batch()
    assert sorted({len(b.chain(c)) for c in range(len(b.chain_start) - 1)}) == [0, 1, 3, 10]
    assert len(set(b.pairs())) == len(b.pairs()) - 1 and b.pairs() != sorted(b.pairs())   # one repeat, out of order
    assert len({tuple(q.pose) for q in b.queries}) == len(b.queries)
    brs = branches(b, H.MAPPER_SEQ, grid)
    for (q, c), br in zip(b.pairs(), brs):
        if len(b.chain(c)) == 0:
            assert br.coarse == "zero" and br.empty_raster
        else:
            assert br.coarse == "plain" and br.best_sum > 0 and not br.fine_outside, ((q, c), br)


def test_yaml_smear_drops_cells_of_the_near_chains():
    """the shipped smear has 100s off the kernel's centre, so AddScan skips points that land on an occupied cell and the raster
    depends on the scan order: the fine pass must re-rasterise with the coarse pass's dropped cells left out"""
    b = near_chain_batch()
    pm = H.port_matcher(H.MAPPER_SEQ, H.GRID_SEQ_YAML)
    assert int((pm.kernel() == 100).sum()) > 1
    q, long_chain = b.queries[0], b.chain(0)
    rasters = []
    for order in (long_chain, long_chain[::-1]):
        pm.raster(q, order)
        rasters.append(pm.grid()["data"])
    assert not np.array_equal(rasters[0], rasters[1])


def test_loop_two_stage_winners():
    """every query's coarse winner has a positive response, and the fine stage centred on it is finished on the host"""
    b = loop_batch()
    pm = H.port_matcher(H.MAPPER_LOOP, H.GRID_LOOP)
    coarse = [pm.match(b.queries[q], b.chain(c), False, False) for q, c in b.pairs()]
    fine = refine_stage(b, [r for r, _, _ in coarse], [m for _, m, _ in coarse])
    assert all(coarse[q * 6 + c][0] > 0 for q, c in fine.pairs())
    for grid in (H.GRID_SEQ, H.GRID_SEQ_YAML):
        for br in branches(fine, H.MAPPER_SEQ, grid):
            assert br.coarse == "plain" and br.best_sum > 0, br
