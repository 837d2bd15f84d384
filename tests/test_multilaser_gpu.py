"""Occupancy grids over scans of several lasers on the device (b200og_add_scans_lasers, OccupancyGrid.AddScans(laser=...)):
each scan keeps its own range threshold, minimum and maximum range, as the reference reads each scan's own laser.  Every
result must equal, bit for bit (dimensions, stride, offset, cells, both counters), the reference's fixtures
(tests/golden/multilaser_golden.npz) or the host oracle of tests/multilaser.py."""
import numpy as np
import pytest

import multilaser as M
from slam_toolbox_b200 import api, merge_maps

pytestmark = pytest.mark.gpu
Z = np.load(M.GOLDEN)
NAMES = ["thr_only", "minr_only", "maxr_only", "tolerance", "box_long", "interleaved", "no_inrange", "merge_rot"]


def laser(lim):
    return api.LaserRangeFinder(range_threshold=float(lim[0]), minimum_range=float(lim[1]), maximum_range=float(lim[2]))


def case(name):
    return {k: Z[f"{name}/{k}"] for k in ("ranges", "poses", "lasers", "laser_id", "laser_table")} | {"res": float(Z[f"{name}/res"][0])}


def grid_of(g):
    cells, ps, ht = g.GetData(counters=True)
    return dict(width=g.GetWidth(), height=g.GetHeight(), stride=g.GetWidthStep(), offset=g.GetOffset(), cells=cells, passes=ps, hits=ht)


def runs(ids):
    """[first, end) of every run of equal laser ids"""
    out, a = [], 0
    for k in range(1, len(ids) + 1):
        if k == len(ids) or ids[k] != ids[a]:
            out.append((a, k))
            a = k
    return out


@pytest.mark.parametrize("name", NAMES)
def test_per_scan_lasers_equal_reference(name):
    c = case(name)
    block = api.ScanBlock(c["ranges"], c["poses"], laser(c["laser_table"][0]))
    g = api.OccupancyGrid(c["res"], laser(c["laser_table"][0]))
    g.AddScans(block, laser=[laser(v) for v in c["lasers"]])
    M.assert_equals_golden(grid_of(g.Build()), Z, name)


@pytest.mark.parametrize("name", NAMES)
def test_create_from_blocks_equals_reference(name):
    """CreateFromScans over one ScanBlock per run of scans of one laser, each block built with its own laser"""
    c = case(name)
    blocks = [api.ScanBlock(c["ranges"][a:b], c["poses"][a:b], laser(c["lasers"][a])) for a, b in runs(c["laser_id"].tolist())]
    M.assert_equals_golden(grid_of(api.OccupancyGrid.CreateFromScans(blocks, c["res"])), Z, name)


def test_merge_with_per_submap_lasers_equals_reference():
    name = "merge_rot"
    c = case(name)
    corr, sub = Z[f"{name}/corr"], Z[f"{name}/submap"]
    mm = merge_maps.MergeMapsKinematic(c["res"], laser(c["laser_table"][0]))
    for k in range(len(corr)):
        m = sub == k
        sid, _, _ = mm.AddSubmap(api.ScanBlock(c["ranges"][m], c["poses"][m], laser(c["lasers"][m][0])), laser(c["lasers"][m][0]))
        mm.corrections[sid] = merge_maps.Transform(corr[k][:9].reshape(3, 3), corr[k][9:])
    M.assert_equals_golden(grid_of(mm.Merge()), Z, f"{name}/merged")
    assert np.array_equal(mm.grid.ScanBoxes(), Z[f"{name}/boxes"])


def test_submap_grid_uses_its_own_laser():
    """a submap built from the shared store (a range build) equals the reference's grid of its scans on its laser"""
    c = case("interleaved")
    g = api.OccupancyGrid(c["res"])
    g.AddScans(api.ScanBlock(c["ranges"], c["poses"], laser(c["laser_table"][0])), laser=[laser(v) for v in c["lasers"]])
    block = api.ScanBlock(c["ranges"], c["poses"], laser(c["laser_table"][0]))
    for a, b in ((0, 6), (6, 6), (3, 9), (12, 6)):
        e = M.host_occupancy(c["ranges"][a:a + b], block.points[a:a + b], c["poses"][a:a + b], c["lasers"][a:a + b], c["res"])
        M.assert_grid_equal(grid_of(g.Build(a, b)), e)


@pytest.mark.parametrize("seed,n_scans,n_lasers", [(301, 40, 2), (302, 150, 3), (303, 400, 5)])
def test_random_mixed_store_equals_host_oracle(seed, n_scans, n_lasers):
    s = M.random_store(seed, n_scans, n_lasers)
    block = api.ScanBlock(s["ranges"], s["poses"], api.LaserRangeFinder())
    g = api.OccupancyGrid(s["res"])
    # in three appends, so that the limits of later appends land after earlier ones
    cut = [0, n_scans // 3, (2 * n_scans) // 3, n_scans]
    for a, b in zip(cut[:-1], cut[1:]):
        g.AddScans(api.ScanBlock(s["ranges"][a:b], s["poses"][a:b], api.LaserRangeFinder(), points=block.points[a:b]),
                   laser=[laser(v) for v in s["lasers"][a:b]])
    e = M.host_occupancy(s["ranges"], block.points, s["poses"], s["lasers"], s["res"])
    M.assert_grid_equal(grid_of(g.Build()), e)
    boxes = np.array([M.scan_box(s["ranges"][k], block.points[k], s["poses"][k], s["lasers"][k]) for k in range(n_scans)])
    assert np.array_equal(g.ScanBoxes(), boxes)


def test_one_laser_calls_are_unchanged():
    """AddScans without a laser, with the handle's own laser and with the same laser per scan store the same limits"""
    s = M.random_store(311, 60, 1)
    lz = api.LaserRangeFinder()
    block = api.ScanBlock(s["ranges"], s["poses"], lz)
    out = []
    for how in (None, lz, [lz] * 60):
        g = api.OccupancyGrid(s["res"], lz)
        g.AddScans(block, laser=how)
        out.append(grid_of(g.Build()))
    for o in out[1:]:
        M.assert_grid_equal(o, out[0])
    M.assert_grid_equal(grid_of(api.OccupancyGrid.CreateFromScans([block], s["res"])), out[0])


def test_remove_scans_of_a_mixed_store():
    s = M.random_store(321, 120, 3)
    block = api.ScanBlock(s["ranges"], s["poses"], api.LaserRangeFinder())
    lasers = [laser(v) for v in s["lasers"]]
    g = api.OccupancyGrid(s["res"])
    g.AddScans(block, laser=lasers)
    alive = np.arange(120)
    rng = np.random.default_rng(5)
    plans = [np.flatnonzero(s["laser_id"] == 1),                           # every scan of one laser
             np.sort(rng.choice(120 - int((s["laser_id"] == 1).sum()), 17, replace=False)),
             np.array([0]), np.array([], dtype=np.int64)]
    for idx in plans:
        g.RemoveScans(idx)
        alive = np.delete(alive, idx)
        fresh = api.OccupancyGrid(s["res"])
        fresh.AddScans(api.ScanBlock(s["ranges"][alive], s["poses"][alive], api.LaserRangeFinder(), points=block.points[alive]),
                       laser=[lasers[k] for k in alive])
        got, exp = grid_of(g.Build()), grid_of(fresh.Build())
        M.assert_grid_equal(got, exp)
        M.assert_grid_equal(got, M.host_occupancy(s["ranges"][alive], block.points[alive], s["poses"][alive], s["lasers"][alive], s["res"]))
        assert np.array_equal(g.ScanBoxes(), fresh.ScanBoxes())
    assert not np.any(s["laser_id"][alive] == 1)


@pytest.mark.parametrize("bad", [dict(range_threshold=np.nan), dict(minimum_range=np.inf), dict(maximum_range=-np.inf)])
def test_non_finite_limits_are_refused(bad):
    s = M.random_store(331, 10, 2)
    block = api.ScanBlock(s["ranges"], s["poses"], api.LaserRangeFinder())
    g = api.OccupancyGrid(s["res"])
    g.AddScans(block, laser=[laser(v) for v in s["lasers"]])
    before = grid_of(g.Build())
    lasers = [laser(v) for v in s["lasers"]]
    lasers[7] = api.LaserRangeFinder(**bad)
    with pytest.raises(api.B200Error) as e:
        g.AddScans(block, laser=lasers)
    assert e.value.code == api.ERR_INVALID_ARG
    assert g.NumScans() == 10
    M.assert_grid_equal(grid_of(g.Build()), before)
    with pytest.raises(ValueError):
        g.AddScans(block, laser=lasers[:3])
