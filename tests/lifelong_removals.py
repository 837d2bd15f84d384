"""Removal traffic of slam_toolbox's lifelong mode on a pose graph, planned on the host for the solver tests
(test_lifelong_removals_gpu.py) and their fixture checks (test_lifelong_removals_fixtures.py).

LifelongSlamToolbox::removeFromSlamGraph (src/experimental/slam_toolbox_lifelong.cpp:332-344) removes interior nodes through
Mapper::RemoveNodeFromGraph (lib/karto_sdk/src/Mapper.cpp:2964-3003): RemoveConstraint(source, target) for each edge of each
neighbour that touches the node, neighbours in the node's edge order, then RemoveNode.  It never removes ids 0 and 1, nodes
within scan_buffer_size of the newest id, or nodes with fewer than two edges (:271-278, :313).  The solver keeps its nodes
in slots in insertion order and RemoveNode moves the last slot's node into the freed one (b200pg_remove_node); Book mirrors
both, so that a test can rebuild the solver's problem in its slot order."""
import numpy as np

from slam_toolbox_b200 import synth

BUFFER = 10          # scan_buffer_size of the shipped mapping parameters (config/mapper_params_online_sync.yaml)
SIGMA = (0.03, 0.03, 0.01)
COV = np.diag(np.square(SIGMA))


class Book:
    """The solver's graph as the removals leave it: node ids in slot order, edges in insertion order (None once removed) and
    every node's edge list (Vertex::GetEdges: indices into edges)."""

    def __init__(self):
        self.order, self.edges, self.vedges, self.anchor = [], [], {}, None

    def add_node(self, nid):
        if self.anchor is None:
            self.anchor = nid          # the first node ever added: the one CeresSolver holds constant
        self.order.append(nid)
        self.vedges[nid] = []

    def add_edge(self, a, b, z, c):
        self.edges.append((a, b, np.asarray(z, dtype=np.float64), np.asarray(c, dtype=np.float64)))
        self.vedges[a].append(len(self.edges) - 1)
        self.vedges[b].append(len(self.edges) - 1)

    def degree(self, nid):
        return len(self.vedges[nid])

    def remove(self, nid):
        """Mapper::RemoveNodeFromGraph's solver calls for nid: returns ([(source, target) of each RemoveConstraint], whether
        RemoveNode moves another node into nid's slot)."""
        calls = []
        for v in [self.edges[j][0] if self.edges[j][1] == nid else self.edges[j][1] for j in self.vedges[nid]]:
            for j in list(self.vedges[v]):
                if nid in self.edges[j][:2]:
                    self.vedges[v].remove(j)
                    calls.append(self.edges[j][:2])
                    self.edges[j] = None
        del self.vedges[nid]
        slot = self.order.index(nid)
        swapped = slot != len(self.order) - 1
        self.order[slot] = self.order[-1]
        self.order.pop()
        return calls, swapped

    def live(self):
        return [e for e in self.edges if e is not None]

    def removable(self, nid, buffer=BUFFER):
        """Lifelong's guards: not ids 0 and 1, at least `buffer` ids older than the newest node, two or more edges."""
        return nid > 1 and max(self.order) - nid >= buffer and self.degree(nid) >= 2

    def components(self):
        """(components with an edge that do not hold the anchor, ids of nodes without an edge)."""
        parent = {n: n for n in self.order}

        def find(n):
            while parent[n] != n:
                parent[n] = parent[parent[n]]
                n = parent[n]
            return n
        for e in self.live():
            parent[find(e[0])] = find(e[1])
        isolated = sorted(n for n in self.order if self.degree(n) == 0)
        roots = {find(n) for n in self.order if self.degree(n) > 0}
        if self.anchor in parent:
            roots.discard(find(self.anchor))
        return len(roots), isolated

    def problem(self, poses):
        """The oracle's problem in slot order from {id: pose}: (init, ea, eb, z, cov, fixed), fixed = the anchor's slot, None
        once the anchor is gone (CeresSolver never fixes another node: was_constant_set_ stays true,
        solvers/ceres_solver.cpp:228-240)."""
        pos = {n: i for i, n in enumerate(self.order)}
        live = self.live()
        init = np.array([poses[n] for n in self.order], dtype=np.float64)
        ea = np.array([pos[e[0]] for e in live], dtype=np.int64)
        eb = np.array([pos[e[1]] for e in live], dtype=np.int64)
        z = np.array([e[2] for e in live]).reshape(-1, 3)
        cov = np.array([e[3] for e in live]).reshape(-1, 3, 3)
        return init, ea, eb, z, cov, pos.get(self.anchor)


def _rel(pa, pb):
    return synth._pose_rel(pa[None], pb[None])[0]


def _graph(seed, n, m, lattice):
    return synth.make_pose_graph(seed, n, m, lattice=lattice, sigma_xy=SIGMA[0], sigma_th=SIGMA[2])


def _base(g):
    book = Book()
    for nid in g["ids"]:
        book.add_node(int(nid))
    for a, b, z, c in zip(g["edge_a"], g["edge_b"], g["z"], g["cov"]):
        book.add_edge(int(a), int(b), z, c)
    return book


def _measured(g, a, b, rng):
    return ("edge", a, b, _rel(g["truth"][a], g["truth"][b]) + rng.normal(0, SIGMA), COV)


def scenario(name):
    """The graph and the plan of case `name`: dict(graph, steps, shapes).  steps: the operations before each Compute, each
    ("remove", id) | ("edge", a, b, z, cov) | ("yaw", id, yaw) (ModifyNode with that yaw added); the first step is empty
    (the first Compute of the full graph).  shapes: per step, after its operations, dict(fragments, isolated, swaps,
    guarded), what the case claims and the fixture tests pin."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "batches":
        # (a) a 600-node mapping graph with revisits; four batches of 12 interior removals
        g = _graph(71, 600, 900, 30)
        book, steps = _base(g), [[]]
        for _ in range(4):
            ops = []
            for _ in range(12):
                cand = [n for n in book.order if book.removable(n)]
                nid = int(rng.choice(cand))
                book.remove(nid)
                ops.append(("remove", nid))
            steps.append(ops)
    elif name.startswith("fragments"):
        # (b) removals that each cut the chain, until `target` components are without the anchor: few loop closures
        target = int(name.split("_")[1])
        g = _graph(72, 400, 440, 60)
        book, steps = _base(g), [[]]
        frags = 0
        for nid in rng.permutation(np.array(book.order)):
            nid = int(nid)
            if frags == target:
                break
            if nid not in book.vedges or not book.removable(nid):
                continue
            trial = Book()
            trial.order, trial.edges, trial.vedges, trial.anchor = list(book.order), list(book.edges), \
                {k: list(v) for k, v in book.vedges.items()}, book.anchor
            trial.remove(nid)
            f, iso = trial.components()
            if f == frags + 1 and not iso:
                book.remove(nid)
                frags = f
                steps.append([("remove", nid)])
    elif name == "isolated":
        # (c) all neighbours of a node go; it stays with no edge, its yaw pushed outside [-pi, pi) (AngleLocalParameterization
        # would wrap it if the solve took the node as a parameter block)
        g = _graph(73, 300, 330, 60)
        book, steps = _base(g), [[]]
        v = next(n for n in book.order[40:] if book.degree(n) == 2 and book.degree(n - 1) == 2 and book.degree(n + 1) == 2)
        ops = [("remove", v - 1), ("remove", v + 1)]
        for _, nid in ops:
            book.remove(nid)
        ops.append(("yaw", v, 7.0))
        steps.append(ops)
        steps.append([("remove", int(next(n for n in book.order[150:] if book.removable(n))))])
        book.remove(steps[-1][0][1])
    elif name == "slots":
        # (d) the node in the last slot leaves (the newest: no swap; outside lifelong's guards, which keep it), then an
        # interior node whose slot receives the last slot's node
        g = _graph(74, 300, 360, 40)
        book, steps = _base(g), [[]]
        newest = book.order[-1]
        book.remove(newest)
        mid = int(next(n for n in book.order[100:] if book.removable(n)))
        book.remove(mid)
        steps += [[("remove", newest)], [("remove", mid)]]
    elif name == "anchor":
        # (e) the anchor (id 0) leaves after the first Compute: no node is held constant from then on.  Lifelong mode keeps
        # ids 0 and 1; localization's rolling buffer and ClearLocalizationBuffer reach the solver the same way.  Removing the
        # anchor before the first Compute makes the reference dereference a stale iterator (first_node_,
        # ceres_solver.cpp:228-240, 333-335): not exercised.
        g = _graph(75, 300, 360, 40)
        book, steps = _base(g), [[]]
        book.remove(0)
        mid = int(next(n for n in book.order[120:] if book.removable(n)))
        book.remove(mid)
        steps += [[("remove", 0)], [("remove", mid)]]
    elif name == "append":
        # (f) a Compute after a removal uploads every edge; k constraints appended afterwards travel alone, and a parallel
        # edge after those (the same node pair, so the same Cholesky pattern) too
        g = _graph(76, 300, 360, 40)
        book, steps = _base(g), [[]]
        mid = int(next(n for n in book.order[100:] if book.removable(n)))
        book.remove(mid)
        steps.append([("remove", mid)])
        ops = []
        for _ in range(5):
            a, b = sorted(int(x) for x in rng.choice(book.order[:-BUFFER], 2, replace=False))
            ops.append(_measured(g, a, b, rng))
        steps.append(ops)
        e = book.live()[7]
        steps.append([_measured(g, e[0], e[1], rng)])
    else:
        raise KeyError(name)
    return dict(graph=g, steps=steps, shapes=replay_shapes(g, steps))


def replay_shapes(g, steps):
    """Runs the plan on a fresh Book: per step, the anchorless components and isolated nodes after it, how many removals
    swapped and did not, and whether every removal of a node other than the newest or the anchor met lifelong's guards."""
    book = _base(g)
    out = []
    for ops in steps:
        swaps, plain, guarded = 0, 0, True
        for op in ops:
            if op[0] == "remove":
                nid = op[1]
                if nid != max(book.order) and nid != book.anchor:
                    guarded &= book.removable(nid)
                _, sw = book.remove(nid)
                swaps += sw
                plain += not sw
            elif op[0] == "edge":
                book.add_edge(*op[1:])
        f, iso = book.components()
        out.append(dict(fragments=f, isolated=iso, swaps=swaps, plain=plain, guarded=guarded))
    return out


CASES = ("batches", "fragments_1", "fragments_2", "fragments_8", "isolated", "slots", "anchor", "append")
