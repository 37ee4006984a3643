"""Plain-Python restatement of the APLS metric of the reference (cityscale_metrics/apls/convert.py + main.go), for
tests only.  It is written line by line from main.go, with dicts where Go has maps, and shares no code with
sam_road_b200/apls_metric.py: it is the check on that module's host stages and on csrc/apls_metric.cu.

Go iterates its maps in a random order.  `order_seed=None` walks every map in ascending key order (the order the
product defines); an integer seeds a shuffle of every map iteration, which emulates one run of the Go program.
rtreego's NearestNeighbors(10, q) is the exact 10 nearest by squared distance to each node's +-1e-6 box in degree
space, ties by ascending node id.  Shortest paths are Dijkstra with heapq on the densified graph, and the pair sum
is math.fsum: the exactly rounded sum, independent of the order.
"""
from __future__ import annotations

import heapq
import math
import random

TOL = 0.000001


class GoParams:
    """main.go's globals; `spacenet=True` is the small-tile branch that a fourth argument switches on."""

    def __init__(self, spacenet=False):
        self.interval_1, self.interval_2 = 37, 25.0
        self.min_distance_filter, self.prop_step = 100.0, 4
        self.region_size, self.margin_size = 2048.0, 100.0
        if spacenet:
            self.interval_2 = 10.0
            self.interval_1 = int(self.interval_2 * 1.5)
            self.min_distance_filter = 30.0
            self.prop_step = 3
            self.margin_size = 30.0
            self.region_size = 352.0


class GoOrder:
    def __init__(self, seed=None):
        self.rng = None if seed is None else random.Random(seed)

    def keys(self, m):
        ks = sorted(m)
        if self.rng is not None:
            self.rng.shuffle(ks)
        return ks


def convert_pickle(neighbors):
    """convert.py: the [nodes, edges] it dumps to JSON (Python repr floats; Go reads them back exactly)."""
    nodes, edges, nodemap, edge_map = [], [], {}, {}
    for k, v in neighbors.items():
        nodemap[k] = len(nodes)
        lat1 = 41.0 - k[0] * 1.0 / 111111.0
        lon1 = -71.0 + (k[1] * 1.0 / 111111.0) / math.cos(math.radians(41.0))
        nodes.append([float(lat1), float(lon1)])
    for k, v in neighbors.items():
        n1 = k
        for n2 in v:
            if (n1, n2) in edge_map or (n2, n1) in edge_map:
                continue
            else:
                edge_map[(n1, n2)] = True
            edges.append([nodemap[n1], nodemap[n2]])
    return [nodes, edges]


class Graph:
    def __init__(self):
        self.Nodes = []
        self.Edges = []
        self.loc2index = {}
        self.neighbors = {}

    def propagate(self, nid, step, action, order):
        visited = {nid: 0}
        queue = [nid]
        while len(queue) > 0:
            current_nid = queue[0]
            queue = queue[1:]
            if visited[current_nid] > step:
                continue
            action(current_nid)
            for k in order.keys(self.neighbors.get(current_nid, {})):
                if k in visited:
                    pass
                else:
                    queue.append(k)
                    visited[k] = visited[current_nid] + 1

    def addEdge(self, loc1, loc2):
        sk1, sk2 = loc2key(loc1), loc2key(loc2)
        if sk1 in self.loc2index:
            nid1 = self.loc2index[sk1]
        else:
            nid1 = len(self.Nodes)
            self.Nodes.append(loc1)
            self.loc2index[sk1] = nid1
        if sk2 in self.loc2index:
            nid2 = self.loc2index[sk2]
        else:
            nid2 = len(self.Nodes)
            self.Nodes.append(loc2)
            self.loc2index[sk2] = nid2
        self.Edges.append([nid1, nid2])
        self.neighbors.setdefault(nid1, {})[nid2] = True
        self.neighbors.setdefault(nid2, {})[nid1] = True

    def arc(self, u, v):
        return int(GPSDistance(self.Nodes[u], self.Nodes[v]) * 100.0)

    def ShortestPaths(self, nid1, targets, order):
        """Dijkstra on integer centimetres; result[v] = cm / 100.0, -1.0 when v is unreachable."""
        result = {v: -1.0 for v in targets}
        mindistance = {nid: 100000000000 for nid in range(len(self.Nodes))}
        mindistance[nid1] = 0
        pq = [(0, nid1)]
        done = set()
        while pq:
            d, cur = heapq.heappop(pq)
            if cur in done or d != mindistance[cur]:
                continue
            done.add(cur)
            if cur in result:
                result[cur] = float(d) / 100.0
            for nxt in order.keys(self.neighbors.get(cur, {})):
                w = self.arc(cur, nxt)
                if w + mindistance[cur] < mindistance[nxt]:
                    mindistance[nxt] = w + mindistance[cur]
                    heapq.heappush(pq, (mindistance[nxt], nxt))
        return result


def GPSDistance(p1, p2):
    a = (p1[0] - p2[0]) * 111111.0
    b = (p1[1] - p2[1]) * 111111.0 * math.cos(p1[0] / 360.0 * 2.0 * math.pi)
    return math.sqrt(a * a + b * b)


def GPSInBound(p1, P):
    lat_top_left = 41.0
    lon_top_left = -71.0
    lat2 = lat_top_left - P.region_size / 111111.0
    lon2 = lon_top_left + P.region_size / 111111.0 / math.cos(lat_top_left / 180.0 * 3.1415926)
    if p1[0] > lat2 + P.margin_size / 111111.0 and p1[0] < lat_top_left - P.margin_size / 111111.0 and \
            p1[1] > lon_top_left + P.margin_size / 111111.0 / math.cos(lat_top_left / 180.0 * 3.1415926) and \
            p1[1] < lon2 - P.margin_size / 111111.0 / math.cos(lat_top_left / 180.0 * 3.1415926):
        return True
    return False


def loc2key(loc):
    return "%.7f_%.7f" % (loc[0], loc[1])


def lockey(loc, dist):
    return "%d_%d" % (int(loc[0] * 111111.0 / dist), int(loc[1] * 111111.0 / dist))


def LoadGraph(raw):
    g = Graph()
    nodes, edges = raw
    for ind, node in enumerate(nodes):
        loc = [float(node[0]), float(node[1])]
        g.Nodes.append(loc)
        sk = loc2key(loc)
        if sk not in g.loc2index:
            g.loc2index[sk] = ind
    for edge in edges:
        g.Edges.append([int(edge[0]), int(edge[1])])
    return g


def GraphDensify(g):
    ng = Graph()
    for n1, n2 in g.Edges:
        d = GPSDistance(g.Nodes[n1], g.Nodes[n2])
        if d > 3.0:
            n = int(d / 2.0) + 1
            for i in range(n):
                alpha1 = float(i) / float(n)
                alpha2 = float(i + 1) / float(n)
                A, B = g.Nodes[n1], g.Nodes[n2]
                if i == 0:
                    loc1 = A
                    loc2 = [A[0] * (1 - alpha2) + B[0] * alpha2, A[1] * (1 - alpha2) + B[1] * alpha2]
                elif i == n - 1:
                    loc1 = [A[0] * (1 - alpha1) + B[0] * alpha1, A[1] * (1 - alpha1) + B[1] * alpha1]
                    loc2 = B
                else:
                    loc1 = [A[0] * (1 - alpha1) + B[0] * alpha1, A[1] * (1 - alpha1) + B[1] * alpha1]
                    loc2 = [A[0] * (1 - alpha2) + B[0] * alpha2, A[1] * (1 - alpha2) + B[1] * alpha2]
                ng.addEdge(loc1, loc2)
        else:
            ng.addEdge(g.Nodes[n1], g.Nodes[n2])
    return ng


def box_d2(node, q):
    s = 0.0
    for i in range(2):
        lo, hi = node[i] - TOL, node[i] + TOL
        if q[i] < lo:
            d = lo - q[i]
        elif q[i] > hi:
            d = q[i] - hi
        else:
            d = 0.0
        s = s + d * d
    return s


def nearest_numpy(nodes, k, queries):
    """NearestNeighbors for many queries at once: the same float64 expressions, vectorised (large tiles)."""
    import numpy as np
    ll = np.asarray(nodes, dtype=np.float64).reshape(-1, 2)
    ids = np.arange(ll.shape[0])
    out = []
    for q in queries:
        s = 0.0
        for i in range(2):
            lo, hi = ll[:, i] - TOL, ll[:, i] + TOL
            d = np.where(q[i] < lo, lo - q[i], np.where(q[i] > hi, q[i] - hi, 0.0))
            s = s + d * d
        order = np.lexsort((ids, s))[:k]
        out.append([int(x) for x in order] + [-1] * (k - len(order)))
    return out


def NearestNeighbors(nodes, k, q):
    keyed = sorted((box_d2(loc, q), nid) for nid, loc in enumerate(nodes))
    return [nid for _, nid in keyed[:k]]


def select_control_points(graph_gt, graph_prop, P, order):
    """The first loop of apls_one_way: control_point_gt with every value -1."""
    visited, lockeys, control_point_gt = {}, {}, {}
    node_cover_map_gt = {nid: False for nid in range(len(graph_gt.Nodes))}

    def cover(nid):
        node_cover_map_gt[nid] = True

    for nid in range(len(graph_gt.Nodes)):
        nb = graph_gt.neighbors.get(nid, {})
        if len(nb) != 2:
            for next_nid in order.keys(nb):
                if next_nid in visited:
                    continue
                chain = [nid, next_nid]
                last_nid, current_nid = nid, next_nid
                while len(graph_gt.neighbors.get(current_nid, {})) == 2:
                    s = 0
                    for k in order.keys(graph_gt.neighbors[current_nid]):
                        s = s + k
                    current_nid, last_nid = s - last_nid, current_nid
                    chain.append(current_nid)
                if len(chain) > P.interval_1:
                    n = int(float(len(chain)) / P.interval_2) + 1
                    for i in range(1, n):
                        idx = int(float(len(chain)) * float(i) / float(n))
                        if GPSInBound(graph_gt.Nodes[chain[idx]], P) and not node_cover_map_gt[chain[idx]]:
                            lk = lockey(graph_gt.Nodes[chain[idx]], 2.0)
                            if lk not in lockeys:
                                lockeys[lk] = True
                                control_point_gt[chain[idx]] = -1
                                graph_prop.propagate(chain[idx], 4, cover, order)
                for cnid in chain:
                    visited[cnid] = True
            if GPSInBound(graph_gt.Nodes[nid], P) and (not node_cover_map_gt[nid] or len(nb) == 1):
                lk = lockey(graph_gt.Nodes[nid], 2.0)
                if lk not in lockeys:
                    lockeys[lk] = True
                    control_point_gt[nid] = -1
                    graph_prop.propagate(nid, 4, cover, order)
    return control_point_gt


def snap(graph_gt, graph_prop, control_point_gt, P, order, nearest=None):
    """The second loop: one-to-one snapping in (shuffled) map order.  Returns the candidate lists by control point."""
    node_cover_map = {nid: False for nid in range(len(graph_prop.Nodes))}
    cands = {}

    def cover(nid):
        node_cover_map[nid] = True

    for nid1 in order.keys(control_point_gt):
        q = graph_gt.Nodes[nid1]
        results = nearest(nid1) if nearest else NearestNeighbors(graph_prop.Nodes, 10, q)
        cands[nid1] = results
        for r in results:
            if node_cover_map.get(r, False):
                continue
            if GPSDistance(graph_prop.Nodes[r], q) < 10.0:
                control_point_gt[nid1] = r
                graph_prop.propagate(r, P.prop_step, cover, order)
                break
    return cands


def distances(g, sources, order, solver=None):
    """{source: {target: cm}} between `sources` (cm = -1 when unreachable), by Dijkstra or by `solver`."""
    if solver is not None:
        return solver(g, sources)
    out = {}
    for s in sources:
        r = g.ShortestPaths(s, sources, order)
        out[s] = {t: (-1 if v < 0 else int(round(v * 100.0))) for t, v in r.items()}
    return out


def score_pairs(control_point_gt, sp_gt, sp_prop, min_distance_filter, order):
    """The pair loop: counts per rule and math.fsum of the terms (penalties included)."""
    terms, penalty, skipped, scored = [], 0, 0, 0
    for cp1_gt in order.keys(control_point_gt):
        cp1_prop = control_point_gt[cp1_gt]
        for cp2_gt in order.keys(control_point_gt):
            cp2_prop = control_point_gt[cp2_gt]
            if cp2_gt <= cp1_gt:
                continue
            if cp1_prop == -1 or cp2_prop == -1:
                terms.append(1.0)
                penalty += 1
                continue
            d1 = float(sp_gt[cp1_gt][cp2_gt]) / 100.0
            if d1 > min_distance_filter:
                d2 = float(sp_prop[cp1_prop][cp2_prop]) / 100.0
                if d2 < 0:
                    d2 = 0
                s = abs(d1 - d2) / d1
                if s > 1.0:
                    s = 1.0
                terms.append(s)
                scored += 1
            else:
                skipped += 1
    cc = penalty + scored
    total = math.fsum(terms)
    return dict(cc=cc, penalty=penalty, skipped=skipped, scored=scored, sum=total,
                apls=float("nan") if cc == 0 else 1.0 - total / float(cc))


def apls_one_way(graph_gt, graph_prop, P, order, solver=None):
    control_point_gt = select_control_points(graph_gt, graph_prop, P, order)
    cps = sorted(control_point_gt)
    cands = snap(graph_gt, graph_prop, control_point_gt, P, order)
    gt_list = [c for c in cps if control_point_gt[c] >= 0]
    prop_list = list(dict.fromkeys(control_point_gt[c] for c in gt_list))
    sp_gt = distances(graph_gt, gt_list, order, solver)
    sp_prop = distances(graph_prop, prop_list, order, solver)
    r = score_pairs(control_point_gt, sp_gt, sp_prop, P.min_distance_filter, order)
    r.update(control_points=cps, matches=[control_point_gt[c] for c in cps], candidates=[cands[c] for c in cps],
             dist_gt=[[sp_gt[a][b] for b in gt_list] for a in gt_list],
             dist_prop=[[sp_prop[a][b] for b in prop_list] for a in prop_list])
    return r


def go_f(x):
    return "NaN" if math.isnan(x) else "%f" % x


def apls(gt_raw, prop_raw, spacenet=False, order_seed=None, solver=None):
    """main.go on [nodes, edges] of both graphs: (apls_gt, apls_prop, the line, the dense graphs, both directions)."""
    P = GoParams(spacenet)
    order = GoOrder(order_seed)
    g = GraphDensify(LoadGraph(gt_raw))
    p = GraphDensify(LoadGraph(prop_raw))
    a = apls_one_way(g, p, P, order, solver)
    b = apls_one_way(p, g, P, order, solver)
    line = "%s %s %s\n" % (go_f(a["apls"]), go_f(b["apls"]), go_f((a["apls"] + b["apls"]) / 2.0))
    return a["apls"], b["apls"], line, (g, p), (a, b)


def scipy_solver(g, sources):
    """Integer Dijkstra by scipy.sparse.csgraph on the same arcs: a second, independent solver for large graphs."""
    import numpy as np
    import scipy.sparse as sp
    from scipy.sparse.csgraph import dijkstra
    if not sources:
        return {}
    rows, cols, ws = [], [], []
    for u, nb in g.neighbors.items():
        for v in nb:
            if u != v:
                rows.append(u)
                cols.append(v)
                ws.append(g.arc(u, v))
    n = len(g.Nodes)
    # explicitly stored zeros are arcs for csgraph; integer sums stay exact in float64
    m = sp.csr_matrix((np.asarray(ws, dtype=np.float64), (rows, cols)), shape=(n, n))
    d = dijkstra(m, directed=True, indices=list(sources))
    out = {}
    for i, s in enumerate(sources):
        out[s] = {t: (int(d[i, t]) if np.isfinite(d[i, t]) else -1) for t in sources}
    return out


class _Scorer:
    """The device's three stages for sam_road_b200.apls_metric (scorer=apls_oracle.scorer), from this module's
    Dijkstra (or `solver`) and math.fsum, on the product's densified graphs."""

    def __init__(self, gt, prop, solver=None, vectorised=False):
        self.graphs = [self._graph(gt), self._graph(prop)]
        self.solver = solver
        self.vectorised = vectorised
        self.order = GoOrder(None)

    @staticmethod
    def _graph(dg):
        g = Graph()
        g.Nodes = [list(x) for x in dg.nodes]
        g.neighbors = {u: {v: True for v in nb} for u, nb in enumerate(dg.nbrs)}
        return g

    def candidates(self, which, queries):
        if self.vectorised:
            return nearest_numpy(self.graphs[which].Nodes, 10, queries)
        return [NearestNeighbors(self.graphs[which].Nodes, 10, q) + [-1] * max(0, 10 - len(self.graphs[which].Nodes))
                for q in queries]

    def one_way(self, gt_role, cps, matches, min_distance_filter):
        cpg = dict(zip([int(c) for c in cps], [int(m) for m in matches]))
        gt_list = [c for c in cpg if cpg[c] >= 0]
        prop_list = list(dict.fromkeys(cpg[c] for c in gt_list))
        sp_gt = distances(self.graphs[gt_role], gt_list, self.order, self.solver)
        sp_prop = distances(self.graphs[1 - gt_role], prop_list, self.order, self.solver)
        r = score_pairs(cpg, sp_gt, sp_prop, min_distance_filter, self.order)
        n = len(cpg)
        r.update(pairs=n * (n - 1) // 2, dist_gt=[[sp_gt[a][b] for b in gt_list] for a in gt_list],
                 dist_prop=[[sp_prop[a][b] for b in prop_list] for a in prop_list])
        return r


def scorer(gt, prop):
    return _Scorer(gt, prop)


def scipy_scorer(gt, prop):
    """For tiles too large for the heapq Dijkstra: scipy's solver and the vectorised nearest-node search."""
    return _Scorer(gt, prop, scipy_solver, vectorised=True)
