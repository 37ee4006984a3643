"""The TOPO graph metric of the reference (cityscale_metrics/topo/main.py + topo.py, spacenet_metrics/ likewise),
scored on the device.  DESIGN.md §14.

    python -m sam_road_b200.topo_metric --savedir save/<run> --dataset cityscale|spacenet [--gt-root DIR]

reads `<savedir>/graph/<tile>.p` (what `inferencer.main` writes) and the ground-truth pickles, and writes
`<savedir>/results/topo/<tile>.txt`, `<tile>.topo.p` and the dataset's `topo.json`, as `topo.bash` does.

The host part is the reference's, restated: graph construction (node ids in dict order, float64 lat/lon, the
`min_lat` / `max_lon` that carry over from tile to tile), the starting points, the pair search (rtree box queries
become an inclusive bounding-box test in ascending edge id, what the rtree shim returns), TOPO121's competitor
sets (distanceBetweenTwoLocation) and its stable-sorted greedy keep, and the text lines.  Per pair, the three
walks, the candidate marble-hole edges and the two maximum matchings run in csrc/topo_metric.cu.
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

from . import _lib

LAT_TOP_LEFT = 41.0
LON_TOP_LEFT = -71.0
DENSITY = 0.00050
MARGIN = 0.07
PAIR_THRESHOLD = 0.00010
MATCHING_THRESHOLD = 0.00010
INTERVAL = 0.00005
COS40 = math.cos(math.radians(40))
CITYSCALE_TILES = [8, 9, 19, 28, 29, 39, 48, 49, 59, 68, 69, 79, 88, 89, 99, 108, 109, 119, 128, 129, 139, 148, 149,
                   159, 168, 169, 179]
# about 3 MB of device workspace per slot (0.8 GB at 264 slots, allocated only for the pairs a tile has); the
# synthetic 2048² city tile of tools/topo_bench.py needs at most 1244 marbles per walk
DEFAULT_CAPS = dict(max_marbles=8192, max_queue=8192, max_covered=4096, max_candidates=1 << 17, slots=264)


@dataclass
class TopoState:
    """main.py's globals: min_lat / max_lon start at the top-left corner and carry over from tile to tile."""
    min_lat: float = LAT_TOP_LEFT
    max_lon: float = LON_TOP_LEFT


@dataclass
class RoadGraph:
    """graph.RoadGraph as create_graph leaves it: nodes by id, edges by id, nodeLink / nodeLinkReverse lists."""
    nodes: list = field(default_factory=list)       # [lat, lon] by node id
    edges: list = field(default_factory=list)       # (n1, n2) by edge id
    link: list = field(default_factory=list)
    rlink: list = field(default_factory=list)


def xy2latlon(x, y):
    lat = LAT_TOP_LEFT - x * 1.0 / 111111.0
    lon = LON_TOP_LEFT + (y * 1.0 / 111111.0) / math.cos(math.radians(LAT_TOP_LEFT))
    return lat, lon


def distance(p1, p2):
    a = p1[0] - p2[0]
    b = (p1[1] - p2[1]) * math.cos(math.radians(p1[0]))
    return math.sqrt(a * a + b * b)


def create_graph(m: dict, state: TopoState) -> RoadGraph:
    """main.py create_graph + RoadGraph.addEdge + ReverseDirectionLink; updates state.min_lat / max_lon."""
    g = RoadGraph()
    idmap = {}
    edge_set = set()

    def node(k, lat, lon):
        if k not in idmap:
            idmap[k] = len(g.nodes)
            g.nodes.append([lat, lon])
            g.link.append([])
        return idmap[k]

    for n1, v in m.items():
        lat1, lon1 = xy2latlon(n1[0], n1[1])
        if lat1 < state.min_lat:
            state.min_lat = lat1
        if lon1 > state.max_lon:
            state.max_lon = lon1
        for n2 in v:
            lat2, lon2 = xy2latlon(n2[0], n2[1])
            id1 = node(n1, lat1, lon1)
            id2 = node(n2, lat2, lon2)
            if (id1, id2) in edge_set:          # addEdge: "Duplicated Edge !!!"
                continue
            edge_set.add((id1, id2))
            g.edges.append((id1, id2))
            if id2 not in g.link[id1]:
                g.link[id1].append(id2)
    g.rlink = [[] for _ in g.nodes]
    for a, b in g.edges:
        if a not in g.rlink[b]:
            g.rlink[b].append(a)
    for a, b in g.edges:
        if g.nodes[a] == g.nodes[b]:
            keys = {v: k for k, v in idmap.items()}
            raise ValueError(f"edge {keys[a]} -> {keys[b]} has length zero; the reference divides by the length of "
                             f"an edge and gets inf / NaN for it")
    return g


def region_of(state: TopoState):
    return [state.min_lat - 300 * 1.0 / 111111.0, LON_TOP_LEFT - 500 * 1.0 / 111111.0,
            LAT_TOP_LEFT + 300 * 1.0 / 111111.0, state.max_lon + 500 * 1.0 / 111111.0]


def starting_points(g: RoadGraph, region, density=DENSITY, mergin=MARGIN):
    """topo.py TOPOGenerateStartingPoints(check=False, image='NULL', metaData=None)."""
    result = []
    visited = set()
    for nodeid in range(len(g.nodes)):
        if nodeid in visited:
            continue
        next_nodes = dict.fromkeys(g.link[nodeid] + g.rlink[nodeid])
        if len(next_nodes) == 2:
            continue
        for nextnode in next_nodes:
            if nextnode in visited:
                continue
            node_list = [nodeid]
            cur = nextnode
            while True:
                node_list.append(cur)
                nb = list(dict.fromkeys(g.link[cur] + g.rlink[cur]))
                if len(nb) != 2:
                    break
                cur = nb[1] if node_list[-2] == nb[0] else nb[0]
            visited.update(node_list[1:-1])
            dists = []
            dist = 0
            for i in range(len(node_list) - 1):
                dists.append(dist)
                dist += distance(g.nodes[node_list[i]], g.nodes[node_list[i + 1]])
            dists.append(dist)
            if dist < density / 2:
                continue
            n = max(int(dist / density), 1)
            alphas = [float(x + 1) / float(n + 1) for x in range(n)]
            for alpha in alphas:
                for j in range(len(node_list) - 1):
                    if alpha * dist >= dists[j] and alpha * dist <= dists[j + 1]:
                        a = (alpha * dist - dists[j]) / (dists[j + 1] - dists[j])
                        lat = (1 - a) * g.nodes[node_list[j]][0] + a * g.nodes[node_list[j + 1]][0]
                        lon = (1 - a) * g.nodes[node_list[j]][1] + a * g.nodes[node_list[j + 1]][1]
                        lat_m = mergin * (region[2] - region[0])
                        lon_m = mergin * (region[3] - region[1])
                        if lat - region[0] > lat_m and region[2] - lat > lat_m and lon - region[1] > lon_m and \
                                region[3] - lon > lon_m:
                            result.append((lat, lon, node_list[j], node_list[j + 1], alpha * dist - dists[j],
                                           dists[j + 1] - alpha * dist))
    return result


def latlon_norm(p1, lat=40):
    p11 = p1[1] * math.cos(math.radians(lat))
    l = math.sqrt(p11 * p11 + p1[0] * p1[0])
    return p1[0] / l, p11 / l


def _point_to_line(p2, p3):
    dist = math.sqrt(p2[0] * p2[0] + p2[1] * p2[1])
    proj = (p2[0] * p3[0] + p2[1] * p3[1]) / dist
    if proj > dist:
        a, b = p3[0] - p2[0], p3[1] - p2[1]
        return math.sqrt(a * a + b * b)
    if proj < 0:
        a, b = p3[0] - 0, p3[1] - 0
        return math.sqrt(a * a + b * b)
    alpha = proj / dist
    a, b = p3[0] - alpha * p2[0], p3[1] - alpha * p2[1]
    return math.sqrt(a * a + b * b)


def _point_to_line_latlon(p1, p2, p3):
    c = math.cos(math.radians(p1[0]))
    return _point_to_line((p2[0] - p1[0], (p2[1] - p1[1]) * c), (p3[0] - p1[0], (p3[1] - p1[1]) * c))


def generate_pairs(gps: RoadGraph, osm: RoadGraph, osm_list, threshold=PAIR_THRESHOLD):
    """topo.py TOPOGeneratePairs(edgeids=None): {start index: [edge, n1, n2, d1, d2, lat, lon]}, ascending index."""
    result = {}
    if not gps.edges:
        return result
    e = np.asarray(gps.edges, dtype=np.int64)
    ll = np.asarray(gps.nodes, dtype=np.float64)
    b0 = np.minimum(ll[e[:, 0], 0], ll[e[:, 1], 0])
    b1 = np.minimum(ll[e[:, 0], 1], ll[e[:, 1], 1])
    b2 = np.maximum(ll[e[:, 0], 0], ll[e[:, 1], 0])
    b3 = np.maximum(ll[e[:, 0], 1], ll[e[:, 1], 1])
    for i, item in enumerate(osm_list):
        lat, lon = item[0], item[1]
        q0, q1, q2, q3 = lat - threshold * 2, lon - threshold * 2, lat + threshold * 2, lon + threshold * 2
        cand = np.nonzero((b0 <= q2) & (b2 >= q0) & (b1 <= q3) & (b3 >= q1))[0]
        min_dist, min_edge = 10000, -1
        lat3, lon3 = osm.nodes[item[2]]
        lat4, lon4 = osm.nodes[item[3]]
        nlat2, nlon2 = latlon_norm((lat4 - lat3, lon4 - lon3))
        for edgeid in cand.tolist():
            n1, n2 = gps.edges[edgeid]
            lat1, lon1 = gps.nodes[n1]
            lat2, lon2 = gps.nodes[n2]
            nlat1, nlon1 = latlon_norm((lat2 - lat1, lon2 - lon1))
            dist = _point_to_line_latlon((lat1, lon1), (lat2, lon2), (lat, lon))
            if dist < threshold and dist < min_dist:
                if 1.0 - abs(nlat1 * nlat2 + nlon1 * nlon2) < 0.04:
                    min_edge, min_dist = edgeid, dist
        if min_edge != -1:
            n1, n2 = gps.edges[min_edge]
            lat1, lon1 = gps.nodes[n1]
            lat2, lon2 = gps.nodes[n2]
            result[i] = [min_edge, n1, n2, distance((lat1, lon1), (lat, lon)), distance((lat2, lon2), (lat, lon)),
                         lat, lon]
    return result


def distance_between_locations(g: RoadGraph, loc1, loc2, max_distance):
    """graph.py RoadGraph.distanceBetweenTwoLocation."""
    if loc1[0] == loc2[0] and loc1[1] == loc2[1]:
        return abs(loc1[2] - loc2[2])
    elif loc1[0] == loc2[1] and loc1[1] == loc2[0]:
        return abs(loc1[2] - loc2[3])
    ans = 100000
    dmap = {}
    queue = [(loc1[0], -1, loc1[2]), (loc1[1], -1, loc1[2])]
    head = 0
    while head < len(queue):
        cur, prev, dist = queue[head]
        head += 1
        if cur in dmap and dmap[cur] <= dist:
            continue
        if dist > max_distance:
            continue
        dmap[cur] = dist
        seen = []
        lat1, lon1 = g.nodes[cur]
        for nx in g.link[cur] + g.rlink[cur]:
            if nx == prev or nx == cur or nx == loc1[0] or nx == loc1[1] or nx in seen:
                continue
            seen.append(nx)
            if cur == loc2[0] and nx == loc2[1]:
                if dist + loc2[2] < ans:
                    ans = dist + loc2[2]
            elif cur == loc2[1] and nx == loc2[0]:
                if dist + loc2[3] < ans:
                    ans = dist + loc2[3]
            queue.append((nx, cur, dist + distance(g.nodes[nx], (lat1, lon1))))
    return ans


def topo121(results, gps: RoadGraph):
    """topo.py TOPO121: competitor sets, stable sort by precision, greedy keep from the end."""
    n = len(results)
    lat = np.array([t[0] for t in results], dtype=np.float64)
    lon = np.array([t[1] for t in results], dtype=np.float64)
    new_list = []
    for ind in range(n):
        la, lo = results[ind][0], results[ind][1]
        r_lat = 0.00030
        r_lon = 0.00030 / math.cos(math.radians(la))
        # rtree boxes [lat - 1e-6, lon - 1e-6, lat + 1e-6, lon + 1e-6] against the query box, bounds inclusive
        hit = (lat - 0.000001 <= la + r_lat) & (lat + 0.000001 >= la - r_lat) & \
              (lon - 0.000001 <= lo + r_lon) & (lon + 0.000001 >= lo - r_lon)
        loc1 = tuple(results[ind][4:8])
        comp = [c for c in np.nonzero(hit)[0].tolist()
                if distance_between_locations(gps, loc1, tuple(results[c][4:8]), 0.00030) < 0.00020]
        new_list.append((results[ind], ind, comp))
    new_list = sorted(new_list, key=lambda item: item[0][2])
    kept, mark = [], set()
    for ind in range(len(new_list) - 1, -1, -1):
        if new_list[ind][1] in mark and new_list[ind][0][2] < 0.9:
            continue
        kept.append(new_list[ind][0])
        mark.update(new_list[ind][2])
    return kept


def topo_avg(kept):
    p = 0
    r = 0
    for item in kept:
        p = p + item[2]
        r = r + item[3]
    if len(kept) == 0:
        return 0, 0
    return p / len(kept), r / len(kept)


def _csr(lists):
    start = np.zeros(len(lists) + 1, dtype=np.int32)
    start[1:] = np.cumsum([len(x) for x in lists])
    flat = np.array([v for x in lists for v in x], dtype=np.int32)
    return start, flat if flat.size else np.zeros(1, dtype=np.int32)


class TopoDevice:
    """One samroad_topo object: both graphs of a tile on the device, and the per-pair scoring."""

    def __init__(self, device: int = 0, **caps):
        c = dict(DEFAULT_CAPS, **caps)
        self._lib = _lib.load()
        self.caps = _lib.SamRoadTopoCaps(**c)
        self._h = _lib.Handle("samroad_topo_create", "samroad_topo_destroy", device, C.byref(self.caps))

    __getstate__ = _lib.refuse_copy

    def close(self):
        self._h.close()

    def upload(self, which: int, g: RoadGraph):
        ll = np.ascontiguousarray(np.asarray(g.nodes, dtype=np.float64).reshape(-1, 2))
        cl = np.array([math.cos(math.radians(p[0])) for p in g.nodes], dtype=np.float64)
        ls, li = _csr(g.link)
        rs, ri = _csr(g.rlink)
        p = lambda a: a.ctypes.data  # noqa: E731
        _lib.check(self._lib.samroad_topo_upload_graph(self._h, which, len(g.nodes), p(ll), p(cl) if cl.size else None,
                                                       p(ls), p(li), p(rs), p(ri)), "samroad_topo_upload_graph")

    def run(self, pair_nodes: np.ndarray, pair_dists: np.ndarray, r: float, step: float, threshold: float):
        n = int(pair_nodes.shape[0])
        counts = np.zeros((n, 6), dtype=np.int32)
        if n == 0:
            return counts
        pn = np.ascontiguousarray(pair_nodes, dtype=np.int32)
        pd = np.ascontiguousarray(pair_dists, dtype=np.float64)
        _lib.check(self._lib.samroad_topo_run(self._h, n, pn.ctypes.data, pd.ctypes.data, r, step, threshold, COS40,
                                              counts.ctypes.data), "samroad_topo_run")
        return counts


@dataclass
class TileDetails:
    results: list            # per starting point that found a pair and scored: (lat, lon, p, r, n1, n2, d1, d2)
    kept: list               # TOPO121's kept results
    lines: list              # the .txt lines, as written
    starts: list             # TOPOGenerateStartingPoints
    pairs: dict              # TOPOGeneratePairs
    region: list
    r: float
    counts: np.ndarray       # [pairs, 6] per pair in pair order: marbles, holes, holes_bidirection, mp, mr, status


def pair_counts(gt: RoadGraph, prop: RoadGraph, starts, pairs, r, step, threshold, scorer):
    """The per-pair work of TOPOWithPairs, by `scorer(pair_nodes, pair_dists, r, step, threshold)`."""
    keys = list(pairs.keys())
    pn = np.array([[pairs[k][1], pairs[k][2], starts[k][2], starts[k][3]] for k in keys],
                  dtype=np.int32).reshape(-1, 4)
    pd = np.array([[pairs[k][3], pairs[k][4], starts[k][4], starts[k][5]] for k in keys],
                  dtype=np.float64).reshape(-1, 4)
    return keys, scorer(pn, pd, r, step, threshold)


def score_pairs(gt: RoadGraph, prop: RoadGraph, starts, pairs, r, step, threshold, scorer, cityscale=True):
    """TOPOWithPairs(one2oneMatching=True, metaData=None) with the per-pair counts from `scorer`."""
    if cityscale:
        float(len(pairs)) / float(len(starts))   # `rrr`: cityscale's topo.py divides by the start count here
    keys, counts = pair_counts(gt, prop, starts, pairs, r, step, threshold, scorer)
    lines, results = [], []
    i = 0
    psum = rsum = 0
    for k, c in zip(keys, counts.tolist()):
        nm, nh, _, mp, mr, _ = c
        if nm == 0 or nh == 0:
            continue
        gps = pairs[k]
        lat, lon = starts[k][0], starts[k][1]
        prec = float(mp) / nm
        rec = float(mr) / nh
        psum += prec
        rsum += rec
        lines.append(str(i) + " " + str(lat) + " " + str(lon) + " " + str(gps[1]) + " " + str(gps[2]) + " Precesion " +
                     str(prec) + " Recall " + str(rec) + " Avg Precesion " + str(psum / (i + 1)) + " Avg Recall " +
                     str(rsum / (i + 1)) + " \n")
        results.append((lat, lon, prec, rec, gps[1], gps[2], gps[3], gps[4]))
        i += 1
    kept = topo121(results, prop)
    p, rr = topo_avg(kept)
    try:
        tail = [str(p) + " " + str(rr) + " " + str(len(kept) / float(len(starts))) + " " +
                str(rr * len(kept) / float(len(starts))) + "\n",
                "precision=" + str(p) + " overall-recall=" + str(rr * len(kept) / float(len(starts)))]
    except ZeroDivisionError:
        tail = [str(0) + " " + str(0) + " " + str(0) + " " + str(0) + "\n"]
    return results, kept, lines + tail, counts


def device_scorer(dev: TopoDevice, gt: RoadGraph, prop: RoadGraph):
    def score(pn, pd, r, step, threshold):
        if pn.shape[0] == 0:
            return np.zeros((0, 6), dtype=np.int32)
        dev.upload(0, gt)
        dev.upload(1, prop)
        return dev.run(pn, pd, r, step, threshold)
    return score


def topo_tile(gt_adj: dict, prop_adj: dict, state: TopoState | None = None, dataset: str = "cityscale",
              device: int | TopoDevice = 0, scorer=None):
    """One tile, as main.py's loop body does it: returns (precision, overall recall, TileDetails).

    gt_adj / prop_adj: adjacency dicts in the pickle format ({(x, y): [(x, y), ...]}).  `state` carries
    min_lat / max_lon from the previous tiles (a fresh TopoState when None).  The precision and recall are those of
    the file's last line (0 and 0 when the file's except branch writes zeros).  `scorer(gt, prop)`, when given,
    returns the per-pair scoring function used instead of the device (the test oracle plugs in here)."""
    if dataset not in ("cityscale", "spacenet"):
        raise ValueError(f"dataset must be 'cityscale' or 'spacenet' (got {dataset!r})")
    state = TopoState() if state is None else state
    gt = create_graph(gt_adj, state)
    prop = create_graph(prop_adj, state)
    region = region_of(state)
    starts = starting_points(gt, region)
    pairs = generate_pairs(prop, gt, starts) if starts else {}
    r = 0.00300
    if dataset == "spacenet" or LAT_TOP_LEFT - state.min_lat < 0.01000:
        r = 0.00150
    own = None
    if scorer is None:
        dev = device if isinstance(device, TopoDevice) else None
        if dev is None:
            dev = own = TopoDevice(device)
        score = device_scorer(dev, gt, prop)
    else:
        score = scorer(gt, prop)
    try:
        results, kept, lines, counts = score_pairs(gt, prop, starts, pairs, r, INTERVAL, MATCHING_THRESHOLD, score,
                                                   cityscale=dataset == "cityscale")
    finally:
        if own is not None:
            own.close()
    p, rec = parse_last_line(lines[-1])
    return p, rec, TileDetails(results, kept, lines, starts, pairs, region, r, counts)


def parse_last_line(line: str):
    """topo.py: p and r from the last line of a tile's file."""
    p = float(line.split(' ')[0].split('=')[-1])
    r = float(line.split(' ')[-1].split('=')[-1])
    return p, r


def tile_list(dataset: str, gt_root: str):
    if dataset == "cityscale":
        return list(CITYSCALE_TILES)
    with open(os.path.join(gt_root, "data_split.json")) as jf:
        return json.load(jf)["test"]


def gt_path(dataset: str, gt_root: str, tile):
    if dataset == "cityscale":
        return os.path.join(gt_root, "20cities", "region_%s_graph_gt.pickle" % tile)
    return os.path.join(gt_root, "RGB_1.0_meter", "%s__gt_graph.p" % tile)


def run_tiles(savedir: str, dataset: str, gt_root: str, tiles=None, device: int = 0, scorer=None):
    """main.py: every tile of the dataset's list, in order, with min_lat / max_lon carried over."""
    tiles = tile_list(dataset, gt_root) if tiles is None else tiles
    state = TopoState()
    dev = TopoDevice(device) if scorer is None else None
    try:
        for tile in tiles:
            output = os.path.join(savedir, "results", "topo", "%s.txt" % tile)
            os.makedirs(os.path.dirname(output), exist_ok=True)
            with open(gt_path(dataset, gt_root, tile), "rb") as f:
                gt_adj = pickle.load(f)
            with open(os.path.join(savedir, "graph", "%s.p" % tile), "rb") as f:
                prop_adj = pickle.load(f)
            _, _, d = topo_tile(gt_adj, prop_adj, state, dataset, device=dev, scorer=scorer)
            with open(output, "a") as fout:    # the reference appends
                fout.write("".join(d.lines))
            with open(output.replace('txt', 'topo.p'), 'wb') as f:
                pickle.dump([d.starts, d.kept, d.region], f)
    finally:
        if dev is not None:
            dev.close()


def aggregate(savedir: str, dataset: str):
    """topo.py of the dataset: per-tile F1 from each file's last line, the means, and topo.json."""
    topo, precision, recall = [], [], []
    rdir = os.path.join(savedir, "results", "topo")
    for file_name in os.listdir(rdir):
        if '.txt' not in file_name:
            continue
        with open(os.path.join(rdir, file_name)) as f:
            lines = f.readlines()
        p, r = parse_last_line(lines[-1])
        if dataset == "cityscale":
            topo.append(2 * p * r / (p + r))
            precision.append(p)
            recall.append(r)
        elif p + r:
            precision.append(p)
            recall.append(r)
    if dataset == "cityscale":
        out = {'mean topo': [np.mean(topo), np.mean(precision), np.mean(recall)], 'prec': precision,
               'recall': recall, 'f1': topo}
        save_path = os.path.join(savedir, "score", "topo.json")
        os.makedirs(os.path.dirname(save_path), exist_ok=True)
    else:
        t = 2 * np.mean(precision) * np.mean(recall) / (np.mean(precision) + np.mean(recall))
        out = {'mean topo': [t, np.mean(precision), np.mean(recall)], 'prec': precision, 'recall': recall, 'f1': t}
        save_path = os.path.join(savedir, "topo.json")
    with open(save_path, 'w') as jf:
        json.dump(out, jf)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description="TOPO metric of a run's graph/*.p, on the device (replaces topo.bash)")
    ap.add_argument("--savedir", required=True, help="the run directory holding graph/<tile>.p")
    ap.add_argument("--dataset", required=True, choices=["cityscale", "spacenet"])
    ap.add_argument("--gt-root", default=None,
                    help="the dataset directory: cityscale/ (with 20cities/) or spacenet/ (with RGB_1.0_meter/ and "
                         "data_split.json); default ./<dataset>")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    gt_root = a.gt_root or a.dataset
    run_tiles(a.savedir, a.dataset, gt_root, device=a.device)
    out = aggregate(a.savedir, a.dataset)
    print('TOPO', out['mean topo'][0], 'Precision', out['mean topo'][1], 'Recall', out['mean topo'][2])


if __name__ == "__main__":
    main()
