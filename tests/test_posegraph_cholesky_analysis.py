"""The host analysis of the Cholesky linear solver (b200pg_cholesky_analyze), without a device: the elimination order is a
permutation of exactly the free nodes and a function of the adjacency pattern alone, the fill of L in that order equals
an independent symbolic factorisation (SciPy's SuperLU), the ordering's fill is close to SciPy's minimum-degree ordering,
and linear_solver_type is validated through the ABI."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from slam_toolbox_b200 import api, synth
from test_posegraph_shapes_gpu import FAMILIES, family


def free_nodes(n, ia, ib, fixed):
    f = np.zeros(n, dtype=bool)
    f[ia] = True
    f[ib] = True
    if fixed >= 0:
        f[fixed] = False
    return np.flatnonzero(f)


def node_matrix(n, ia, ib, nodes, seed=0):
    """The free nodes' block pattern as a scalar matrix (one entry per node), diagonally dominant with random weights, so
    that no numerical cancellation can hide a structural nonzero."""
    pos = np.full(n, -1)
    pos[nodes] = np.arange(len(nodes))
    keep = (pos[ia] >= 0) & (pos[ib] >= 0)
    a, b = pos[ia[keep]], pos[ib[keep]]
    w = np.random.default_rng(seed).uniform(0.1, 1.0, len(a))
    m = len(nodes)
    A = sp.coo_matrix((np.concatenate([w, w]), (np.concatenate([a, b]), np.concatenate([b, a]))), shape=(m, m)).tocsr()
    A.sum_duplicates()
    d = np.asarray(abs(A).sum(axis=1)).reshape(-1) + 1.0
    return (A + sp.diags(d)).tocsc(), pos


def superlu_fill(A, perm=None):
    """nnz of L (unit diagonal included) and its column counts, from SuperLU without pivoting."""
    if perm is not None:
        A = A[perm][:, perm].tocsc()
    lu = spla.splu(A, permc_spec="NATURAL", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True))
    L = lu.L.tocsc()
    assert np.array_equal(lu.perm_r, np.arange(A.shape[0])) and np.array_equal(lu.perm_c, np.arange(A.shape[0]))
    return L.nnz, np.diff(L.indptr)


GRAPHS = [("synth", 0, 60, 120), ("synth", 1, 500, 1400), ("synth", 2, 3000, 9000), ("synth", 7, 1500, 4500)] + \
    [("family", name, 0, 0) for name in sorted(FAMILIES)]


def graph(kind, a, n, e):
    if kind == "synth":
        g = synth.make_pose_graph(a, n, e, sigma_xy=0.03, sigma_th=0.01)
        return len(g["ids"]), g["edge_a"].astype(np.int64), g["edge_b"].astype(np.int64), 0
    g = family(a)
    return len(g["ids"]), np.asarray(g["ia"], dtype=np.int64), np.asarray(g["ib"], dtype=np.int64), int(g["anchor"])


@pytest.mark.parametrize("kind,a,n,e", GRAPHS)
def test_order_and_fill_against_superlu(kind, a, n, e):
    n, ia, ib, fixed = graph(kind, a, n, e)
    info, order = api.cholesky_analyze(n, np.column_stack([ia, ib]), fixed)
    nodes = free_nodes(n, ia, ib, fixed)
    # a permutation of exactly the free nodes: not the constant node, not a node outside every edge
    assert info["columns"] == len(nodes) == len(order)
    assert np.array_equal(np.sort(order), nodes)
    assert fixed not in set(order.tolist())
    # deterministic
    info2, order2 = api.cholesky_analyze(n, np.column_stack([ia, ib]), fixed)
    assert info2 == info and np.array_equal(order2, order)
    # the fill in that order equals an independent symbolic factorisation
    A, pos = node_matrix(n, ia, ib, nodes)
    nnz, counts = superlu_fill(A, pos[order])
    assert info["nnz_blocks"] == nnz, (info, nnz)
    assert info["flops"] == sum((3 * c - k) ** 2 for c in counts.tolist() for k in range(3))
    # shapes of the supernodal structure
    assert 1 <= info["max_width"] <= 16 and info["max_rows"] >= counts.max()
    assert 1 <= info["critical_path"] <= info["supernodes"] <= info["columns"]
    assert info["analyses"] == 0


def test_order_ignores_edge_multiplicity_and_order():
    g = synth.make_pose_graph(4, 800, 2400, sigma_xy=0.03, sigma_th=0.01)
    ed = np.column_stack([g["edge_a"], g["edge_b"]])
    info, order = api.cholesky_analyze(800, ed, 0)
    rng = np.random.default_rng(1)
    shuffled = ed[rng.permutation(len(ed))]
    flipped = shuffled.copy()
    flip = rng.random(len(ed)) < 0.5
    flipped[flip] = flipped[flip][:, ::-1]
    doubled = np.concatenate([flipped, flipped[rng.choice(len(ed), 300)]])
    for variant in (shuffled, flipped, doubled):
        i2, o2 = api.cholesky_analyze(800, variant, 0)
        assert i2 == info and np.array_equal(o2, order)


def test_isolated_nodes_and_no_fixed_node():
    # nodes 5..9 are outside every edge; without a fixed node every node in an edge is a column
    ed = np.array([[0, 1], [1, 2], [2, 3], [3, 4], [4, 0], [1, 3]])
    info, order = api.cholesky_analyze(10, ed, -1)
    assert info["columns"] == 5 and np.array_equal(np.sort(order), np.arange(5))
    info, order = api.cholesky_analyze(10, ed, 2)
    assert info["columns"] == 4 and 2 not in order.tolist()
    # no free node at all
    info, order = api.cholesky_analyze(2, np.array([[0, 1]]), 0)
    assert info["columns"] == 1 and order.tolist() == [1]
    info, order = api.cholesky_analyze(3, np.zeros((0, 2), dtype=np.int32), 0)
    assert info["columns"] == 0 and info["nnz_blocks"] == 0 and info["supernodes"] == 0
    info, order = api.cholesky_analyze(0, np.zeros((0, 2), dtype=np.int32), -1)
    assert info["columns"] == 0 and len(order) == 0


def test_invalid_arguments():
    L = api.lib()
    info = np.zeros(8, dtype=np.int64)
    ip = info.ctypes.data_as(C.POINTER(C.c_int64))
    bad = np.array([[0, 5]], dtype=np.int32)
    assert L.b200pg_cholesky_analyze(3, 1, bad.ctypes.data_as(C.POINTER(C.c_int32)), 0, ip, None, 0) == api.ERR_INVALID_ARG
    loop = np.array([[1, 1]], dtype=np.int32)
    assert L.b200pg_cholesky_analyze(3, 1, loop.ctypes.data_as(C.POINTER(C.c_int32)), 0, ip, None, 0) == api.ERR_INVALID_ARG
    ok = np.array([[0, 1], [1, 2]], dtype=np.int32)
    order = np.zeros(1, dtype=np.int32)
    assert L.b200pg_cholesky_analyze(3, 2, ok.ctypes.data_as(C.POINTER(C.c_int32)), -1, ip,
                                     order.ctypes.data_as(C.POINTER(C.c_int32)), 1) == api.ERR_INVALID_ARG
    assert L.b200pg_cholesky_analyze(3, 2, ok.ctypes.data_as(C.POINTER(C.c_int32)), 3, ip, None, 0) == api.ERR_INVALID_ARG
    # no nodes: only fixed = -1 names no node
    assert L.b200pg_cholesky_analyze(0, 0, None, 0, ip, None, 0) == api.ERR_INVALID_ARG
    with pytest.raises(api.B200Error) as e:
        api.cholesky_analyze(0, np.zeros((0, 2), dtype=np.int32))
    assert e.value.code == api.ERR_INVALID_ARG
    assert L.b200pg_cholesky_analyze(0, 0, None, -1, ip, None, 0) == api.OK and info[0] == 0 and info[1] == 0
    assert L.b200pg_cholesky_analyze(3, 2, ok.ctypes.data_as(C.POINTER(C.c_int32)), -1, ip, None, 0) == api.OK
    assert info[0] == 3
    assert L.b200pg_factor_info(None, ip) == api.ERR_INVALID_ARG


def test_fill_quality_on_cfg4():
    """cfg4 (10k nodes / 40k edges): the ordering's fill stays within 2x of SciPy's multiple-minimum-degree ordering on
    the same node graph (177,967 blocks)."""
    g = synth.make_pose_graph(0, 10000, 40000, sigma_xy=0.03, sigma_th=0.01)
    ia, ib = g["edge_a"].astype(np.int64), g["edge_b"].astype(np.int64)
    info, order = api.cholesky_analyze(10000, np.column_stack([ia, ib]), 0)
    nodes = free_nodes(10000, ia, ib, 0)
    A, pos = node_matrix(10000, ia, ib, nodes)
    mmd = spla.splu(A, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True)).L.nnz
    assert info["nnz_blocks"] <= 2 * mmd, (info, mmd)
    nnz, _ = superlu_fill(A, pos[order])
    assert info["nnz_blocks"] == nnz


def test_linear_solver_type_through_the_abi():
    L = api.lib()
    o = api.PgOpts()
    L.b200pg_default_opts(C.byref(o))
    assert o.linear_solver_type == 0
    assert (o.trust_region_strategy, o.dogleg_type) == (0, 0)   # the fields before it are in place
    assert [f for f, _ in api.PgOpts._fields_][-1] == "linear_solver_type"
    h = C.c_void_p()
    for value in (2, -1):
        bad = api.PgOpts()
        L.b200pg_default_opts(C.byref(bad))
        bad.linear_solver_type = value
        assert L.b200pg_create(C.byref(bad), C.byref(h)) == api.ERR_INVALID_ARG
