"""The APLS graph metric of the reference (cityscale_metrics/apls/convert.py + main.go + apls.py, spacenet_metrics/
likewise), scored on the device.  DESIGN.md §15.

    python -m sam_road_b200.apls_metric --savedir save/<run> --dataset cityscale|spacenet [--gt-root DIR]

reads `<savedir>/graph/<tile>.p` (what `inferencer.main` writes) and the ground-truth pickles, and writes
`<savedir>/results/apls/<tile>.txt` and the dataset's `apls.json`, as `apls.bash` + `apls.py` do.  No Go toolchain
and no rtree library are needed.

The host part is main.go's, restated in Python in its operation order: convert.py's node and edge lists,
GraphDensify (the `%.7f` key merge, the `d > 3.0` split), the directed integer arc weights
int(GPSDistance(u, v) * 100.0), the control points of apls_one_way (chains, lockeys, the cover through the *other*
graph's 4-hop BFS) and the greedy one-to-one snapping, the text lines and both aggregators.  Go leaves two orders
to its randomised map iteration; here both are ascending node id: a junction's neighbours during the control-point
walk, and the control points during the snapping.  rtreego's 10-nearest query is the exact 10 nearest by squared
distance to each node's +-1e-6 degree box, ties by ascending node id.  The snapping candidates, the shortest paths
and the pair score run in csrc/apls_metric.cu; the sum over pairs is exact there, rounded once.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import pickle
from dataclasses import dataclass, field

import numpy as np

from . import _lib, ranks
from .topo_metric import gt_path, tile_list, xy2latlon

COVER_STEP = 4          # apls_one_way's graph_prop.propagate(nid, 4, ...): prop_step is not used there
SNAP_RADIUS = 10.0      # GPSDistance(candidate, control point) < 10.0
DEFAULT_CAPS = dict(max_nodes=1 << 17, max_arcs=1 << 19, max_control_points=8192)


@dataclass(frozen=True)
class AplsParams:
    interval_1: int
    interval_2: float
    min_distance_filter: float
    prop_step: int
    region_size: float
    margin_size: float


# cityscale's apls.bash runs main.go with three arguments; spacenet's passes a fourth, which switches to the
# small-tile branch (spacenet_metrics/apls/main.go: interval_2 = 10.0, interval_1 = int(interval_2 * 1.5))
PARAMS = {"cityscale": AplsParams(37, 25.0, 100.0, 4, 2048.0, 100.0),
          "spacenet": AplsParams(int(10.0 * 1.5), 10.0, 30.0, 3, 352.0, 30.0)}


def params_of(dataset: str) -> AplsParams:
    if dataset not in PARAMS:
        raise ValueError(f"dataset must be 'cityscale' or 'spacenet' (got {dataset!r})")
    return PARAMS[dataset]


def convert(adj: dict):
    """convert.py: ([lat, lon] per key in dict order, [i, j] per unordered neighbour pair in dict / list order)."""
    nodes, edges, nodemap, seen = [], [], {}, set()
    for k in adj:
        nodemap[k] = len(nodes)
        lat, lon = xy2latlon(k[0], k[1])
        nodes.append([float(lat), float(lon)])
    for n1, v in adj.items():
        for n2 in v:
            if (n1, n2) in seen or (n2, n1) in seen:
                continue
            seen.add((n1, n2))
            if n2 not in nodemap:
                raise ValueError(f"node {n1!r} lists the neighbour {n2!r}, which is not a key of the graph; "
                                 f"convert.py raises KeyError there")
            edges.append([nodemap[n1], nodemap[n2]])
    return nodes, edges


def gps_distance(p1, p2):
    """main.go GPSDistance: the cosine of p1's latitude, written p1[0] / 360.0 * 2.0 * pi."""
    a = (p1[0] - p2[0]) * 111111.0
    b = (p1[1] - p2[1]) * 111111.0 * math.cos(p1[0] / 360.0 * 2.0 * math.pi)
    return math.sqrt(a * a + b * b)


def gps_in_bound(p, params: AplsParams):
    """main.go GPSInBound: strict inequalities, with the literal 3.1415926."""
    lat_top_left, lon_top_left = 41.0, -71.0
    c = math.cos(lat_top_left / 180.0 * 3.1415926)
    lat2 = lat_top_left - params.region_size / 111111.0
    lon2 = lon_top_left + params.region_size / 111111.0 / c
    return (p[0] > lat2 + params.margin_size / 111111.0 and p[0] < lat_top_left - params.margin_size / 111111.0 and
            p[1] > lon_top_left + params.margin_size / 111111.0 / c and p[1] < lon2 - params.margin_size / 111111.0 / c)


def loc2key(loc):
    return "%.7f_%.7f" % (loc[0], loc[1])


def lockey(loc, dist=2.0):
    return int(loc[0] * 111111.0 / dist), int(loc[1] * 111111.0 / dist)


@dataclass
class DenseGraph:
    """GraphDensify's result: nodes by id, the edge list, and each node's neighbour set in ascending id."""
    nodes: list = field(default_factory=list)
    edges: list = field(default_factory=list)
    nbrs: list = field(default_factory=list)


def densify(nodes, edges) -> DenseGraph:
    """main.go GraphDensify + addEdge: ids in order of first appearance, endpoints merged by loc2key."""
    index, out, nb = {}, DenseGraph(), []

    def node(loc):
        k = loc2key(loc)
        i = index.get(k)
        if i is None:
            i = index[k] = len(out.nodes)
            out.nodes.append(loc)
            nb.append(set())
        return i

    def add(l1, l2):
        a, b = node(l1), node(l2)
        out.edges.append((a, b))
        nb[a].add(b)
        nb[b].add(a)

    for n1, n2 in edges:
        p, q = nodes[n1], nodes[n2]
        d = gps_distance(p, q)
        if d > 3.0:
            n = int(d / 2.0) + 1
            for i in range(n):
                a1 = float(i) / float(n)
                a2 = float(i + 1) / float(n)
                l1 = p if i == 0 else [p[0] * (1 - a1) + q[0] * a1, p[1] * (1 - a1) + q[1] * a1]
                l2 = q if i == n - 1 else [p[0] * (1 - a2) + q[0] * a2, p[1] * (1 - a2) + q[1] * a2]
                add(l1, l2)
        else:
            add(p, q)
    out.nbrs = [sorted(s) for s in nb]
    return out


def propagate(g: DenseGraph, nid: int, step: int) -> set:
    """graph.propagate: the nodes within `step` hops of nid (nid alone when it is not a node of g)."""
    depth = {nid: 0}
    queue, head, acted = [nid], 0, set()
    while head < len(queue):
        cur = queue[head]
        head += 1
        if depth[cur] > step:
            continue
        acted.add(cur)
        for k in (g.nbrs[cur] if 0 <= cur < len(g.nbrs) else ()):
            if k not in depth:
                depth[k] = depth[cur] + 1
                queue.append(k)
    return acted


def control_points(gt: DenseGraph, prop: DenseGraph, params: AplsParams) -> list:
    """The control points of apls_one_way on gt, ascending id; a junction's neighbours are walked in ascending id."""
    visited, lockeys, cps, covered = set(), set(), set(), set()

    def take(c):
        lk = lockey(gt.nodes[c])
        if lk in lockeys:
            return
        lockeys.add(lk)
        cps.add(c)
        covered.update(propagate(prop, c, COVER_STEP))

    for nid in range(len(gt.nodes)):
        nb = gt.nbrs[nid]
        if len(nb) == 2:
            continue
        for nx in nb:
            if nx in visited:
                continue
            chain = [nid, nx]
            last, cur = nid, nx
            while len(gt.nbrs[cur]) == 2:
                s = gt.nbrs[cur][0] + gt.nbrs[cur][1]
                cur, last = s - last, cur
                chain.append(cur)
                if len(chain) > 2 * len(gt.nodes) + 2:
                    raise RuntimeError(f"the chain from node {nid} does not end")
            if len(chain) > params.interval_1:
                n = int(float(len(chain)) / params.interval_2) + 1
                for i in range(1, n):
                    c = chain[int(float(len(chain)) * float(i) / float(n))]
                    if gps_in_bound(gt.nodes[c], params) and c not in covered:
                        take(c)
            visited.update(chain)
        if gps_in_bound(gt.nodes[nid], params) and (nid not in covered or len(nb) == 1):
            take(nid)
    return sorted(cps)


def snap(gt: DenseGraph, prop: DenseGraph, cps, candidates, params: AplsParams) -> list:
    """The greedy one-to-one snapping, control points in ascending id: the first candidate that is not covered and
    lies within 10 m; its prop_step-hop neighbourhood on the proposal graph is then covered.  -1: unmatched."""
    covered, match = set(), []
    for i, c in enumerate(cps):
        m = -1
        for k in candidates[i]:
            k = int(k)
            if k < 0:
                break
            if k in covered:
                continue
            if gps_distance(prop.nodes[k], gt.nodes[c]) < SNAP_RADIUS:
                m = k
                covered.update(propagate(prop, k, params.prop_step))
                break
        match.append(m)
    return match


def arc_csr(g: DenseGraph):
    """Directed arcs in ascending (u, v) with weights int(GPSDistance(u, v) * 100.0): u's cosine, so the two
    directions of an edge can differ by 1 cm."""
    start = np.zeros(len(g.nodes) + 1, dtype=np.int32)
    start[1:] = np.cumsum([len(x) for x in g.nbrs])
    col = np.array([v for x in g.nbrs for v in x], dtype=np.int32)
    w = np.array([int(gps_distance(g.nodes[u], g.nodes[v]) * 100.0) for u, x in enumerate(g.nbrs) for v in x],
                 dtype=np.int64)
    if w.size and int(w.sum()) >= 2 ** 31 - 1:
        raise ValueError(f"the arc weights of a graph sum to {int(w.sum())} cm, so a distance could exceed int32")
    return start, col, w.astype(np.int32)


def fmt_f(x: float) -> str:
    """Go's %f: six decimals, NaN as `NaN`."""
    return "NaN" if math.isnan(x) else "%f" % x


def apls_line(apls_gt: float, apls_prop: float) -> str:
    return "%s %s %s\n" % (fmt_f(apls_gt), fmt_f(apls_prop), fmt_f((apls_gt + apls_prop) / 2.0))


class AplsDevice:
    """One samroad_apls object: both densified graphs of a tile on the device, candidates, shortest paths, pairs."""

    def __init__(self, device: int = 0, **caps):
        self._lib = _lib.load()
        self.caps = _lib.SamRoadAplsCaps(**dict(DEFAULT_CAPS, **caps))
        self._h = _lib.Handle("samroad_apls_create", "samroad_apls_destroy", device, C.byref(self.caps))

    __getstate__ = _lib.refuse_copy

    def close(self):
        self._h.close()

    def upload_csr(self, which: int, latlon, start, col, w):
        ll = np.ascontiguousarray(np.asarray(latlon, dtype=np.float64).reshape(-1, 2))
        st = np.ascontiguousarray(start, dtype=np.int32)
        co = np.ascontiguousarray(col, dtype=np.int32)
        wt = np.ascontiguousarray(w, dtype=np.int32)
        p = lambda a: a.ctypes.data if a.size else None  # noqa: E731
        _lib.check(self._lib.samroad_apls_upload_graph(self._h, which, ll.shape[0], p(ll), p(st), p(co), p(wt)),
                   "samroad_apls_upload_graph")

    def upload(self, which: int, g: DenseGraph):
        self.upload_csr(which, g.nodes, *arc_csr(g))

    def candidates(self, which: int, queries) -> np.ndarray:
        q = np.ascontiguousarray(np.asarray(queries, dtype=np.float64).reshape(-1, 2))
        out = np.full((q.shape[0], _lib.APLS_CANDIDATES), -1, dtype=np.int32)
        if q.shape[0]:
            _lib.check(self._lib.samroad_apls_candidates(self._h, which, q.shape[0], q.ctypes.data, out.ctypes.data),
                       "samroad_apls_candidates")
        return out

    def one_way(self, gt_role: int, cps, matches, min_distance_filter: float, export: bool = False) -> dict:
        cp = np.ascontiguousarray(cps, dtype=np.int32)
        mt = np.ascontiguousarray(matches, dtype=np.int32)
        ng = int((mt >= 0).sum())
        npr = len({int(m) for m in mt if m >= 0})
        dg = np.zeros((ng, ng), dtype=np.int32) if export else None
        dp = np.zeros((npr, npr), dtype=np.int32) if export else None
        r = _lib.SamRoadAplsResult()
        p = lambda a: a.ctypes.data if a is not None and a.size else None  # noqa: E731
        _lib.check(self._lib.samroad_apls_one_way(self._h, gt_role, cp.size, p(cp), p(mt), min_distance_filter,
                                                  C.byref(r), p(dg), p(dp)), "samroad_apls_one_way")
        out = dict(pairs=r.pairs, cc=r.cc, penalty=r.penalty, skipped=r.skipped, scored=r.scored, sum=r.sum,
                   sum_fixed=[int(x) for x in r.sum_fixed], terminals=(r.terminals_gt, r.terminals_prop))
        if export:
            out["dist_gt"], out["dist_prop"] = dg, dp
        return out


class _DeviceScorer:
    def __init__(self, dev: AplsDevice, gt: DenseGraph, prop: DenseGraph, export: bool):
        self.dev, self.export = dev, export
        dev.upload(0, gt)
        dev.upload(1, prop)

    def candidates(self, which, queries):
        return self.dev.candidates(which, queries)

    def one_way(self, gt_role, cps, matches, min_distance_filter):
        return self.dev.one_way(gt_role, cps, matches, min_distance_filter, export=self.export)


@dataclass
class OneWay:
    control_points: list     # ascending node ids of the GT-role graph
    candidates: np.ndarray   # [control points, 10] node ids of the other graph, nearest first, -1 padded
    matches: list            # per control point: its node of the other graph, or -1
    result: dict             # cc, penalty, skipped, scored, sum (and the distance matrices when exported)
    apls: float


@dataclass
class AplsDetails:
    gt: DenseGraph
    prop: DenseGraph
    gt_way: OneWay           # apls_one_way(gt, prop)
    prop_way: OneWay         # apls_one_way(prop, gt)
    line: str


def one_way(graphs, gt_role: int, params: AplsParams, score) -> OneWay:
    gt, prop = graphs[gt_role], graphs[1 - gt_role]
    cps = control_points(gt, prop, params)
    cand = score.candidates(1 - gt_role, [gt.nodes[c] for c in cps])
    matches = snap(gt, prop, cps, cand, params)
    r = score.one_way(gt_role, cps, matches, params.min_distance_filter)
    apls = float("nan") if r["cc"] == 0 else 1.0 - r["sum"] / float(r["cc"])
    return OneWay(cps, np.asarray(cand), matches, r, apls)


def apls_graphs(gt_nodes, gt_edges, prop_nodes, prop_edges, dataset: str = "cityscale",
                device: int | AplsDevice = 0, scorer=None, export: bool = False):
    """main.go on two converted graphs (its gt.json / prop.json: [lat, lon] nodes, [i, j] edges)."""
    params = params_of(dataset)
    graphs = (densify(gt_nodes, gt_edges), densify(prop_nodes, prop_edges))
    own = None
    if scorer is None:
        dev = device if isinstance(device, AplsDevice) else None
        if dev is None:
            dev = own = AplsDevice(device)
        score = _DeviceScorer(dev, graphs[0], graphs[1], export)
    else:
        score = scorer(graphs[0], graphs[1])
    try:
        a = one_way(graphs, 0, params, score)
        b = one_way(graphs, 1, params, score)
    finally:
        if own is not None:
            own.close()
    return a.apls, b.apls, (a.apls + b.apls) / 2.0, AplsDetails(graphs[0], graphs[1], a, b, apls_line(a.apls, b.apls))


def apls_tile(gt_adj: dict, prop_adj: dict, dataset: str = "cityscale", device: int | AplsDevice = 0,
              scorer=None, export: bool = False):
    """One tile as apls.bash scores it: returns (apls_gt, apls_prop, apls, AplsDetails).

    gt_adj / prop_adj: adjacency dicts in the pickle format ({(x, y): [(x, y), ...]}).  A direction without a
    scored pair is NaN, and so is then the mean.  `scorer(gt, prop)`, when given, returns an object with
    `candidates(which, queries)` and `one_way(gt_role, cps, matches, min_distance_filter)` used instead of the
    device (the test oracle plugs in here).  `export` adds the two distance matrices to each direction's result."""
    params_of(dataset)
    return apls_graphs(*convert(gt_adj), *convert(prop_adj), dataset=dataset, device=device, scorer=scorer,
                       export=export)


def run_tiles(savedir: str, dataset: str, gt_root: str, tiles=None, device: int = 0, scorer=None, rank: int = 0,
              world: int = 1):
    """apls.bash's loop: every tile of the dataset's list that has a proposal graph; each file is overwritten.  With
    world > 1 only the tiles rank::world of the list."""
    tiles = tile_list(dataset, gt_root) if tiles is None else tiles
    tiles = [tiles[i] for i in ranks.shard(len(tiles), rank, world)]
    os.makedirs(os.path.join(savedir, "results", "apls"), exist_ok=True)
    dev = AplsDevice(device) if scorer is None and tiles else None
    try:
        for tile in tiles:
            prop_path = os.path.join(savedir, "graph", "%s.p" % tile)
            if not os.path.isfile(prop_path):
                continue
            with open(gt_path(dataset, gt_root, tile), "rb") as f:
                gt_adj = pickle.load(f)
            with open(prop_path, "rb") as f:
                prop_adj = pickle.load(f)
            d = apls_tile(gt_adj, prop_adj, dataset, device=dev, scorer=scorer)[3]
            with open(os.path.join(savedir, "results", "apls", "%s.txt" % tile), "w") as f:
                f.write(d.line)
    finally:
        if dev is not None:
            dev.close()


def aggregate(savedir: str, dataset: str, verbose: bool = False):
    """The dataset's apls.py.  cityscale: files in sorted order, the value `split(' ')[-1][:-2]` (the sixth decimal
    dropped), reading stops at the first file that does not parse (a NaN line); score/apls.json.  spacenet: files
    whose line holds `NaN` are skipped, the full last token is kept; results/apls.json.  Returns the JSON object."""
    rdir = os.path.join(savedir, "results", "apls")
    names = sorted(os.listdir(rdir))
    apls, listed = [], []
    with np.errstate(all="ignore"):
        for name in names:
            with open(os.path.join(rdir, name)) as f:
                lines = f.readlines()
            if dataset == "cityscale":
                try:
                    v = float(lines[0].split(' ')[-1][:-2])
                except (ValueError, IndexError):
                    break
                if verbose:
                    print(name, lines[0].split(' ')[-1][:-2])
                apls.append(v)
            elif 'NaN' not in lines[0]:
                v = float(lines[0].split(' ')[-1])
                apls.append(v)
                listed.append([name, v])
        if dataset == "cityscale":
            out = {'apls': apls, 'final_APLS': np.mean(apls)}
            path = os.path.join(savedir, "score", "apls.json")
            os.makedirs(os.path.dirname(path), exist_ok=True)
        else:
            out = {'apls': listed, 'final_APLS': np.mean(apls)}
            path = os.path.join(savedir, "results", "apls.json")
    with open(path, 'w') as jf:
        json.dump(out, jf)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description="APLS metric of a run's graph/*.p, on the device (replaces apls.bash)")
    ap.add_argument("--savedir", required=True, help="the run directory holding graph/<tile>.p")
    ap.add_argument("--dataset", required=True, choices=["cityscale", "spacenet"])
    ap.add_argument("--gt-root", default=None,
                    help="the dataset directory: cityscale/ (with 20cities/) or spacenet/ (with RGB_1.0_meter/ and "
                         "data_split.json); default ./<dataset>")
    ap.add_argument("--device", type=int, default=0, help="GPU index (GPU LOCAL_RANK under torchrun with several ranks)")
    a = ap.parse_args(argv)
    gt_root = a.gt_root or a.dataset
    with ranks.process_group() as (rank, world):    # rank r of W scores the tiles r::W, rank 0 then aggregates
        device = ranks.local_gpu() if world > 1 else a.device
        ranks.run_checked(run_tiles, a.savedir, a.dataset, gt_root, device=device, rank=rank, world=world)
        if rank == 0:
            out = aggregate(a.savedir, a.dataset, verbose=True)
            print('APLS', out['final_APLS'])


if __name__ == "__main__":
    main()
