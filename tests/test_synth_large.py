"""synth.make_pose_graph_large, the vectorised generator of the million-node study graph, on small sizes (no GPU): the edge
count, odometry chain, loop edges between the same or adjacent lattice sites past the index gap, no repeated pair, and the
dead-reckoned start."""
import numpy as np

from slam_toolbox_b200 import synth


def test_large_generator_shape():
    n, e, lat = 20000, 80000, 141
    g = synth.make_pose_graph_large(3, n, e, lat, sigma_xy=0.05, sigma_th=0.02)
    ea, eb = g["edge_a"], g["edge_b"]
    assert len(ea) == e and g["z"].shape == (e, 3) and g["cov"].shape == (e, 3, 3)
    assert np.array_equal(ea[: n - 1], np.arange(n - 1)) and np.array_equal(eb[: n - 1], np.arange(1, n))
    la, lb = ea[n - 1:], eb[n - 1:]
    assert np.all(lb - la > 50)
    assert len(np.unique(la.astype(np.int64) * n + lb)) == len(la)
    t = g["truth"]
    assert np.all((t[:, :2] >= 0) & (t[:, :2] < lat))
    step = np.abs(t[1:, :2] - t[:-1, :2]).sum(axis=1)
    assert np.all(step <= 1) and np.mean(step == 1) > 0.99     # 1 m lattice steps; a step across a border stays on its site
    assert np.all(np.abs(t[la, :2] - t[lb, :2]).sum(axis=1) <= 1)      # same or adjacent site
    # the initial guess integrates the odometry measurements
    c, s = np.cos(g["init"][:-1, 2]), np.sin(g["init"][:-1, 2])
    d = g["init"][1:, :2] - g["init"][:-1, :2]
    assert np.allclose(np.column_stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1]]), g["z"][: n - 1, :2])
    assert np.array_equal(synth.make_pose_graph_large(3, n, e, lat)["edge_b"], eb)
