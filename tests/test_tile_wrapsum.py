"""Wrapped-word accumulation of the tiled sweep kernel (csrc/sm_tile.cu).

The item loops add every loaded word whole into Tw (wrapping mod 2^32) and only its odd bytes into To; the flush recovers the
even-byte fields as E = Tw - (To << 8) mod 2^32.  This holds exactly while every 16-bit field of an item stays below 2^16, which
the host guarantees by capping an item at kChunkBeams = 640 beams of cell values <= 100 (64,000).

The CPU tests restate the kernel's loops in numpy (uint32 arithmetic, as on the device) and compare E and To with the direct even /
odd byte sums.  The GPU test runs saturated sweeps -- candidates that are the query itself, so the best poses score (nearly) 1 and
every beam of an item adds 100 -- on both y-tile layouts and one- and two-CTA clusters, bit-exact against the oracle."""
from __future__ import annotations

import numpy as np
import pytest

K_CHUNK_BEAMS = 640
MAX_CELL = 100
U32 = np.uint32


def odd_bytes(w):
    return (w >> U32(8)) & U32(0x00FF00FF)


def even_bytes(w):
    return w & U32(0x00FF00FF)


def derive_even(tw, to):
    with np.errstate(over="ignore"):
        return (tw - (to << U32(8))).astype(U32)


def cells(rng, shape, lo=0, hi=MAX_CELL):
    """Words of four cell bytes in [lo, hi] (the sub-grid holds smear values 0..100)."""
    b = rng.integers(lo, hi + 1, size=shape + (4,), dtype=np.uint64)
    return (b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16) | (b[..., 3] << 24)).astype(U32)


def accumulate(plain, singles=(), pairs=()):
    """The kernel's loops for one lane and row tile: plain words in 4-beam steps (two byte-wise pair sums, then one add of each
    into Tw and one add of their odd bytes into To), then 2- and 1-beam steps, weighted singles (word, k) and weighted pairs
    (word, word, k).  Returns (Tw, To) and the direct sums (E, O) the reference loops would have formed."""
    tw, to = U32(0), U32(0)
    e, o = 0, 0
    with np.errstate(over="ignore"):
        b = 0
        n = len(plain)
        while b + 3 < n:
            wa, wb = plain[b] + plain[b + 1], plain[b + 2] + plain[b + 3]   # bytes <= 200: no carry between bytes
            tw = tw + wa + wb
            to = to + odd_bytes(wa) + odd_bytes(wb)
            b += 4
        while b < n:
            tw = tw + plain[b]
            to = to + odd_bytes(plain[b])
            b += 1
        for w, k in singles:
            tw = tw + w * U32(k)
            to = to + odd_bytes(w) * U32(k)
        for w0, w1, k in pairs:
            w = w0 + w1
            tw = tw + w * U32(k)
            to = to + odd_bytes(w) * U32(k)
    for w in plain:
        e += int(even_bytes(w)); o += int(odd_bytes(w))
    for w, k in singles:
        e += k * int(even_bytes(w)); o += k * int(odd_bytes(w))
    for w0, w1, k in pairs:
        e += k * (int(even_bytes(w0)) + int(even_bytes(w1))); o += k * (int(odd_bytes(w0)) + int(odd_bytes(w1)))
    return tw, to, e, o


def fields(v):
    return v & 0xFFFF, v >> 16


def check(tw, to, e, o):
    assert max(fields(e)) < 1 << 16 and max(fields(o)) < 1 << 16, "an item's fields must stay below 2^16"
    assert int(to) == o
    assert int(derive_even(tw, to)) == e
    if int(tw) == 0 and int(to) == 0:   # the flush skips an item whose Tw and To are zero: then E is zero too
        assert e == 0


@pytest.mark.parametrize("seed", range(8))
def test_random_items(seed):
    rng = np.random.default_rng(seed)
    for _ in range(50):
        n = int(rng.integers(0, K_CHUNK_BEAMS + 1))
        check(*accumulate(list(cells(rng, (n,)))))


def test_every_cell_100_at_full_weight():
    w = cells(np.random.default_rng(0), (K_CHUNK_BEAMS,), MAX_CELL, MAX_CELL)
    tw, to, e, o = accumulate(list(w))
    assert fields(e) == (64000, 64000) and fields(o) == (64000, 64000)
    check(tw, to, e, o)
    for n4 in range(0, K_CHUNK_BEAMS + 1, 37):   # the 4-, 2- and 1-beam steps at every remainder
        check(*accumulate(list(w[:n4])))


def test_weighted_pairs_and_singles_at_full_weight():
    rng = np.random.default_rng(1)
    full = lambda n: list(cells(rng, (n,), MAX_CELL, MAX_CELL))
    # pairs of weight 36 (the largest weight of one group's pairs: 2 + 3 + ... + 36 > 640), singles of the next weights, plain rest
    pairs = [(a, b, 36) for a, b in zip(full(8), full(8))]                      # 576 beams
    singles = [(full(1)[0], k) for k in (30, 20)]                                # 50 beams
    plain = full(K_CHUNK_BEAMS - 576 - 50)
    tw, to, e, o = accumulate(plain, singles, pairs)
    assert fields(e) == (64000, 64000)
    check(tw, to, e, o)
    for k in range(2, 37):   # every pair weight with random cells, the rest of the item plain
        npair = K_CHUNK_BEAMS // (2 * k)
        pr = [(a, b, k) for a, b in zip(cells(rng, (npair,)), cells(rng, (npair,)))]
        check(*accumulate(list(cells(rng, (K_CHUNK_BEAMS - 2 * k * npair,))), (), pr))


def test_single_of_full_weight():
    w = cells(np.random.default_rng(2), (1,), MAX_CELL, MAX_CELL)[0]
    tw, to, e, o = accumulate([], [(w, K_CHUNK_BEAMS)])
    assert fields(e) == (64000, 64000)
    check(tw, to, e, o)


def test_tail_row_butterfly():
    """The tail row: 8 lane-rows each sum every 8th entry, the flush adds Tw and To over the lane-rows with three butterfly
    steps (wrapping), then derives E once."""
    rng = np.random.default_rng(3)
    for hi in (MAX_CELL, None):
        w = cells(rng, (K_CHUNK_BEAMS,), MAX_CELL if hi else 0, MAX_CELL)
        tws, tos = np.zeros(8, U32), np.zeros(8, U32)
        with np.errstate(over="ignore"):
            for y in range(8):
                for k in range(y, K_CHUNK_BEAMS, 8):
                    tws[y] = tws[y] + w[k]
                    tos[y] = tos[y] + odd_bytes(w[k])
            for step in (4, 2, 1):   # lanes 4 and 8 apart in the kernel: lane-rows 1, 2, 4 apart
                tws = (tws + tws[np.arange(8) ^ step]).astype(U32)
                tos = (tos + tos[np.arange(8) ^ step]).astype(U32)
        e = sum(int(even_bytes(x)) for x in w)
        o = sum(int(odd_bytes(x)) for x in w)
        for y in range(8):
            check(tws[y], tos[y], e, o)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: saturated sweeps against the oracle
# ---------------------------------------------------------------------------------------------------------------------------
# both cases run the cfg2 geometry (4 m search, 0.05 m cells); they differ in the scan every candidate copies
SCANS = {
    # the query's own ranges: at the centre pose every beam reads 100
    "world_self": "world",
    # every range just above the minimum: the 1081 beams pile into a few cells, so weighted singles and pairs of large weight carry
    # whole items at the centre pose
    "short_ring": "ring",
}


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [0, 1])
@pytest.mark.parametrize("name", sorted(SCANS))
def test_saturated_sweep_vs_oracle(monkeypatch, name, tail):
    from slam_toolbox_b200 import synth
    import helpers as H

    grid = H.GRID_LOOP
    monkeypatch.setenv("B200_TILE_TAIL", str(tail))
    mapper = dict(H.MAPPER_LOOP, use_response_expansion=0)
    sw = synth.make_loop_sweep(970 + tail, n_queries=1, n_chains=1, chain_len=1)
    rng = np.random.default_rng(971)
    qr = np.array(sw.query_ranges, dtype=np.float64, copy=True)
    if SCANS[name] == "ring":
        qr[:] = rng.uniform(0.105, 0.125, size=qr.shape)
    qp = np.array(sw.query_poses, dtype=np.float64).reshape(1, 3)
    # six candidates: the query itself, and the query shifted by whole cells / rotated by one angle step
    shifts = np.array([[0, 0, 0], [0.05, 0, 0], [0, -0.1, 0], [0.15, 0.05, 0], [0, 0, np.radians(2.0)], [-0.05, 0.1, 0]])
    cp = qp + shifts
    cr = np.repeat(qr.reshape(1, -1), len(cp), axis=0)
    chain_start = np.arange(len(cp) + 1, dtype=np.int32)
    pm, gm = H.port_matcher(mapper, grid), H.gpu_matcher(mapper, grid)
    pc, pq = H.port_scans(cr, cp), H.port_scans(qr, qp)
    exp = [pm.match(pq[0], pc[c:c + 1], False, False) for c in range(len(cp))]
    er = np.array([x[0] for x in exp])
    em, ec = np.array([x[1] for x in exp]), np.array([x[2] for x in exp])
    assert er.max() > 0.99, er   # saturated: the best poses read 100 at (nearly) every beam
    gc, gq = H.gpu_block(cr, cp), H.gpu_block(qr, qp)
    gm.set_option("sweep_kernel", 2)
    for cluster in (1, 2):
        gm.set_option("sweep_cluster", cluster)
        r, m, c = gm.MatchScanBatch(gq, gc, chain_start, None, False, False)
        info, plan = gm.batch_info(), gm.batch_tile_info()
        assert info["kernel"] == "tile" and plan["available"], (info, plan)
        assert bool(plan["tail"]) == bool(tail), plan
        if SCANS[name] == "ring":
            assert gm.batch_tile_stats()["max_multiplicity"] >= 16, gm.batch_tile_stats()
        assert np.array_equal(r, er), (name, plan, r, er)
        assert np.array_equal(m, em) and np.array_equal(c, ec), (name, plan)
