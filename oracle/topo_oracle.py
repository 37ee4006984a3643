"""NumPy / Python restatement of the per-pair work of the TOPO metric (tests only): the three TOPOWalks of
graph.py (newstyle, direction=False, metaData=None), the candidate test of topo.py TOPOWithPairs and the size of a
maximum matching (augmenting paths), written independently of csrc/topo_metric.cu.  `scorer(gt, prop)` plugs into
sam_road_b200.topo_metric.topo_tile(scorer=...) in place of the device, with the same [pairs, 6] counts.
"""
from __future__ import annotations

import math

import numpy as np

COS40 = math.cos(math.radians(40))


def _dist(p1, p2):
    a = p1[0] - p2[0]
    b = (p1[1] - p2[1]) * math.cos(math.radians(p1[0]))
    return math.sqrt(a * a + b * b)


def topo_walk(g, nid1, nid2, dist1, dist2, r, step, bidirection=False):
    """RoadGraph.TOPOWalk(1, step, r, direction=False, newstyle=True, nid1, nid2, dist1, dist2, bidirection)."""
    mables, seen = [], set()

    def add(t, twin):
        if t in seen:
            return
        seen.add(t)
        mables.append(t)
        if twin:
            tw = (t[0] + 0.00001, t[1] + 0.00001, t[2], t[3])
            seen.add(tw)
            mables.append(tw)

    lat1, lon1 = g.nodes[nid1]
    lat2, lon2 = g.nodes[nid2]
    l = _dist((lat2, lon2), (lat1, lon1))
    twin = bidirection and nid1 in g.link[nid2] and nid2 in g.link[nid1]
    alpha = 0
    while True:
        latI = lat1 * alpha + lat2 * (1 - alpha)
        lonI = lon1 * alpha + lon2 * (1 - alpha)
        d1 = _dist((latI, lonI), (lat1, lon1))
        d2 = _dist((latI, lonI), (lat2, lon2))
        if dist1 - d1 < r or dist2 - d2 < r:
            add((latI, lonI, lat2 - lat1, lon2 - lon1), twin)
        alpha += step / l
        if alpha > 1.0:
            break

    dmap, covered = {}, {}
    queue = [(nid1, -1, dist1), (nid2, -1, dist2)]
    head = 0
    while head < len(queue):
        cur, prev, dist = queue[head]
        head += 1
        old = 1
        if cur in dmap:
            old = dmap[cur]
            if old <= dist:
                continue
        if dist > r:
            continue
        dmap[cur] = dist
        done = []
        lat1, lon1 = g.nodes[cur]
        for nx in g.link[cur] + g.rlink[cur]:
            if nx == prev or nx == cur or nx == nid1 or nx == nid2 or nx in done:
                continue
            done.append(nx)
            lat2, lon2 = g.nodes[nx]
            l = _dist((lat2, lon2), (lat1, lon1))
            c = step * math.ceil(dist / step) - dist
            if old + l < r:
                queue.append((nx, cur, dist + l))
                continue
            start_lim = covered.get((cur, nx), 0)
            end_lim = l - covered[(nx, cur)] if (nx, cur) in covered else l
            twin = bidirection and nx in g.link[cur] and cur in g.link[nx]
            while c < l:
                alpha = c / l
                if dist + l * alpha > r:
                    break
                if l * alpha < start_lim:
                    c += step
                    continue
                if l * alpha > end_lim:
                    break
                add((lat2 * alpha + lat1 * (1 - alpha), lon2 * alpha + lon1 * (1 - alpha), lat2 - lat1, lon2 - lon1),
                    twin)
                c += step
            covered[(cur, nx)] = c - step
            queue.append((nx, cur, dist + l))
    return mables


def _norm(p0, p1):
    p11 = p1 * COS40
    l = math.sqrt(p11 * p11 + p0 * p0)
    return p0 / l, p11 / l


def is_candidate(marble, hole, query_is_marble, threshold):
    """The rtree box test (query +-1.8 threshold, indexed point +-0.00001, inclusive), distance < threshold and the
    angle test of TOPOWithPairs."""
    rr = threshold * 1.8
    q, x = (marble, hole) if query_is_marble else (hole, marble)
    if not (x[0] - 0.00001 <= q[0] + rr and x[0] + 0.00001 >= q[0] - rr and
            x[1] - 0.00001 <= q[1] + rr and x[1] + 0.00001 >= q[1] - rr):
        return False
    ddd = _dist(marble, hole)
    angle_d = 0.0
    if marble[2] != marble[3] and hole[2] != hole[3]:
        n1, n2 = _norm(marble[2], marble[3]), _norm(hole[2], hole[3])
        angle_d = 1.0 - abs(n1[0] * n2[0] + n1[1] * n2[1])
    return ddd < threshold and angle_d < 0.29


def candidate_graph(left, right, left_is_marble, threshold):
    """{left key (tuple): set of right indices}, keyed as TOPOWithPairs' bigraph (equal tuples merge)."""
    out = {}
    for a in left:
        for j, b in enumerate(right):
            ok = is_candidate(a, b, True, threshold) if left_is_marble else is_candidate(b, a, False, threshold)
            if ok:
                out.setdefault(a, set()).add(j)
    return out


def matching_size(adj: dict) -> int:
    """Size of a maximum matching of a bipartite graph {left: iterable of right} (Kuhn's augmenting paths)."""
    match_r = {}
    keys = list(adj)

    def augment(u, seen):
        for v in sorted(adj[u]):
            if v in seen:
                continue
            seen.add(v)
            if v not in match_r or augment(match_r[v], seen):
                match_r[v] = u
                return True
        return False

    return sum(1 for u in keys if augment(u, set()))


def pair_counts(gt, prop, n, d, r, step, threshold):
    """[6] counts of one pair: marbles, holes, bidirectional holes, matched (precision), matched (recall), 0."""
    marbles = topo_walk(prop, n[0], n[1], d[0], d[1], r, step)
    holes = topo_walk(gt, n[2], n[3], d[2], d[3], r, step)
    holes_b = topo_walk(gt, n[2], n[3], d[2], d[3], r, step, bidirection=True)
    mp = matching_size(candidate_graph(marbles, holes_b, True, threshold))
    mr = matching_size(candidate_graph(holes, marbles, False, threshold))
    return [len(marbles), len(holes), len(holes_b), mp, mr, 0]


def scorer(gt, prop):
    def score(pn, pd, r, step, threshold):
        return np.array([pair_counts(gt, prop, [int(v) for v in n], [float(v) for v in d], r, step, threshold)
                         for n, d in zip(pn, pd)], dtype=np.int32).reshape(-1, 6)
    return score
