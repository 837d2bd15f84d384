"""Plain-Python restatement of the tiled sweep kernel's planner (plan_tile in csrc/sm_tile.cu), written from the code, for tests
that check which plan the device reports at geometries the shipped parameters never reach.

The planner takes the correlation grid (stride, height), the coarse pose window (nX x nY poses, nA angles), the query's beam
count n, whether the sweep is penalised (the per-cell image is then FP64 instead of int32 sums), the batch size and the device's
SM count, and returns the plan (chunks V, bands, band rows, cluster size C) or a refusal code:
  2  odd grid stride or more than 4096 angles;
  9  more x-tiles (16 columns of poses) than the item record's 6 bits, or more y-tiles than its 8 bits;
  4  no chunk count V leaves room for 8 band rows next to the accumulators, the image and the two staging buffers;
  5  the chosen plan's shared memory (with the idle lanes' over-read of the last y-tile) exceeds 227 KB.
The refusals that depend on the encoded descriptor blocks (8, 10 to 13) and the parity preconditions (1, 6, 7) are not restated.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

SMEM_LIMIT = 227 * 1024
TILE_SHARED_BYTES = 1936       # sizeof(TileShared): the kernel's static shared memory
TILE_THREADS = 1024
TILE_MAX_CLUSTER = 8
CHUNK_BEAMS = 640
A_GUARD_LO, A_GUARD_HI = 4, 20
ITEM_MAX_XTILES, ITEM_MAX_YTILES = 64, 256
OCCUPIED = 100


@dataclass(frozen=True)
class Geometry:
    """what ScanMatcher::Create and the coarse pass make of (search size, resolution, smear, range threshold) and the angle
    window: the correlation grid (width x height, row stride) and the coarse pose window"""
    width: int
    height: int
    stride: int
    nX: int
    nY: int
    nA: int
    ksize: int


def round_half_away(v: float) -> int:
    return int(math.floor(v + 0.5)) if v >= 0 else int(math.ceil(v - 0.5))


def geometry(grid, angle_offset: float, angle_res: float) -> Geometry:
    """grid = (search size, resolution, smear deviation, range threshold) as ScanMatcher::Create takes them"""
    search, res, smear, rt = grid
    side = round_half_away(search / res) + 1
    margin = math.ceil(rt / res)
    grid_size = side + 2 * margin
    half = round_half_away(2.0 * smear / res)
    width = grid_size + 2 * (half + 1)
    stride = (width + 7) & ~7
    n_xy = (side - 1) // 2 + 1                     # coarse pass: 2-cell steps over the side
    na = round_half_away(2 * angle_offset / angle_res) + 1
    return Geometry(width, width, stride, n_xy, n_xy, na, 2 * half + 1)


@dataclass(frozen=True)
class Plan:
    refused: int                 # 0 = the tiled kernel runs with the plan below
    chunks: int = 0
    bands: int = 0
    band_rows: int = 0
    cluster: int = 0
    smem: int = 0                # dynamic shared memory, bytes
    tail: bool = False


def plan(g: Geometry, n: int, pen: bool, npairs: int, sms: int, cluster: int = 0, chunks: int = 0, max_n: int | None = None,
         tail_layout: bool = True) -> Plan:
    """the plan of build_tile_tables.  cluster / chunks are the sweep_cluster / sweep_chunks options (0 = automatic); max_n is
    the longest candidate scan's reading count (it only decides whether the first scan's cells are staged in shared memory)"""
    nX, nY, nA = g.nX, g.nY, g.nA
    P = nX * nY
    if g.stride & 1 or nA < 1 or nA > 4096:
        return Plan(2)
    pitch_w = (g.stride // 2 + 16 + 3) // 4
    while pitch_w & 7 != 4:
        pitch_w += 1
    yt48, yt40 = (nY + 47) // 48, max(1, (nY - 1 + 39) // 40)
    tail = tail_layout and 8 * 5 * yt40 + 2 < 8 * 6 * yt48
    ytile_rows = 40 if tail else 48
    xtiles, ytiles = (nX + 3 + 15) // 16, (yt40 if tail else yt48)
    if xtiles > ITEM_MAX_XTILES or ytiles > ITEM_MAX_YTILES:
        return Plan(9)
    rows_valid = (g.height + 1) // 2
    halo = nY + 2
    base_rows = max(1, rows_valid - nY + 1)
    want_c = cluster
    if want_c <= 0:
        want_c = 1
        while want_c < TILE_MAX_CLUSTER and npairs * want_c * 2 <= sms:
            want_c *= 2
    cc = 1
    while cc * 2 <= min(want_c, TILE_MAX_CLUSTER):
        cc *= 2
    cc = min(cc, nA)
    while cc & (cc - 1):
        cc -= 1
    budget = SMEM_LIMIT - TILE_SHARED_BYTES - 256
    int_ties = not pen and n * OCCUPIED < 0.9e6
    probs_bytes = (P * (4 if int_ties else 8) + 15) & ~15
    best = None
    for V in range(cc, nA + 1):
        if chunks > 0 and V < min(chunks, nA):
            continue
        nAc = -(-nA // V)
        if -(-nA // nAc) != V or nAc > 63:
            continue
        a_bytes = (4 * (A_GUARD_LO + nAc * P + A_GUARD_HI) + 15) & ~15
        one_angle = 8 * xtiles * ytiles * (4 + max(n - 1, 0) // CHUNK_BEAMS) + 2 * n + 4 * 12 + 6 + 10
        stage = 16 + nAc * 52 + (nAc * n * 2 * 3) // 8 + 64 * nAc
        stage = max(stage, one_angle + 64)
        stage = (stage + 127) & ~127
        s_avail = budget - a_bytes - probs_bytes - 2 * stage
        if s_avail <= 0:
            continue
        rows_avail = s_avail // (pitch_w * 4)
        if rows_avail * pitch_w > 65535:
            rows_avail = 65535 // pitch_w
        B = rows_avail - halo
        if B < 8:
            continue
        B = min(B, base_rows)
        nbv = -(-base_rows // B)
        B = -(-base_rows // nbv)
        loads = 5.0 * ytiles + 0.25 if tail else 6.0 * ytiles
        flush_wi = 124 if tail else 112
        # C's integer arithmetic: (long)(double) truncates toward zero, / on non-negative ints floors
        w_angle = int(n * xtiles * loads * 32 * 2.3 / TILE_THREADS) + 4 * nbv * ((4 * xtiles * ytiles * flush_wi) // 32)
        w_raster = 4 * (700 + (3 * min(B + halo, rows_valid + halo - nY) * pitch_w) // TILE_THREADS)
        cost = ((V + cc - 1) // cc) * (nbv * w_raster + nAc * w_angle)
        if best is None or cost < best[0]:
            best = (cost, V, nbv, B, stage)
    if best is None:
        return Plan(4)
    _, V, nbands, B, stage = best
    nAc = -(-nA // V)
    C = min(cc, V)
    alloc_rows = max(min(B + halo, rows_valid + halo - nY), 1)
    s_bytes = (alloc_rows * pitch_w * 4 + 15) & ~15
    a_bytes = (4 * (A_GUARD_LO + nAc * P + A_GUARD_HI) + 15) & ~15
    off_probs = s_bytes + a_bytes
    off_stage = (off_probs + probs_bytes + 127) & ~127
    off_cells = off_stage + 2 * stage
    max_n = (max(n if max_n is None else max_n, 1) + 3) & ~3
    cell_cap = max_n if max_n <= 4096 else 0
    if off_cells + 2 * cell_cap * 4 + TILE_SHARED_BYTES + 64 > SMEM_LIMIT:
        cell_cap = 0
    smem = off_cells + 2 * cell_cap * 4
    overrun = max(ytile_rows * ytiles - nY + 1, 1) * pitch_w * 4
    if smem - s_bytes < overrun:
        smem = s_bytes + overrun
    if smem + TILE_SHARED_BYTES + 64 > SMEM_LIMIT:
        return Plan(5)
    return Plan(0, V, nbands, B, C, smem, tail)


def stages_per_pair(p: Plan) -> int:
    """(chunk, phase, band) stages one pair runs through, over all CTAs of its cluster"""
    return p.chunks * 4 * p.bands
