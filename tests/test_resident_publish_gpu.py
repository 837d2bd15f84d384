"""The resident map publish (karto::b200::ResidentOccupancyMap, integration/occupancy_b200.hpp) inside the reference's own
Mapper: after every publish step its grid equals the reference's OccupancyGrid::CreateFromScans over the scans the mapper holds
then (dimensions, offset, cell bytes).  A localization run exercises the in-place removals of the rolling buffer's oldest
scans; a mapping run exercises the reloads after MapperGraph::CorrectPoses, which move stored scans."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import replay  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not replay.available(), reason="oracle/_ref/libreplay_*.so not built")]

SEED = 4
PARAMS = dict(replay.YAML_PARAMS, correlation_search_space_smear_deviation=0.03, loop_search_space_dimension=4.0)
# publishes rows: step, equal, removed, appended, reloaded, resident s, reference s, resident device ms


def test_localization_publishes_equal_the_reference():
    mr, mo, _ = replay.make_trajectory(SEED, 120)
    lr, lo, _ = replay.make_localization_trajectory(SEED, 60, map_scans=120)
    out = replay.run_localization("b200", mr, mo, lr, lo, PARAMS, events=[(0, "process_near", lo[0])], map_resolution=0.05,
                                  publish_every=1)
    p = out["publishes"]
    assert len(p) == 60
    assert p[:, 1].all(), p[p[:, 1] == 0, 0]
    assert p[0, 4] == 1                            # the first publish loads the map
    removal_steps = p[(p[:, 2] > 0) & (p[:, 4] == 0)]
    assert len(removal_steps) >= 10                # the rolling buffer's oldest scans leave in place
    assert p[:, 3].sum() > 0


def test_mapping_publishes_equal_the_reference_across_loop_closures():
    ranges, odom, _ = replay.make_trajectory(SEED, 160)
    out = replay.run("b200", ranges, odom, PARAMS, map_resolution=0.05, publish_every=5)
    p = out["publishes"]
    assert p[:, 1].all(), p[p[:, 1] == 0, 0]
    assert out["solver_computes"] > 0
    later = p[1:]
    assert (later[:, 4] == 1).sum() >= 1           # a publish after CorrectPoses reloads
    assert ((later[:, 4] == 0) & (later[:, 3] > 0)).sum() >= 1   # and the others only append
