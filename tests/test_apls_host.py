"""APLS metric, host side (sam_road_b200/apls_metric.py) and its oracle (oracle/apls_oracle.py), without a GPU.

Each rule of main.go has a hand-derived case on which its plausible misreading gives a different answer, derived
with the reference's float64 expressions.  The product's host stages (densified graphs, control points, matches)
equal the oracle's on the reference's spacenet sample and synthetic tiles; the oracle's Dijkstra equals scipy's;
the aggregators and the file text follow apls.py and Go's %f."""
import json
import math
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import dijkstra

from oracle import apls_oracle as O
from sam_road_b200 import apls_metric as AM
from sam_road_b200 import synth

SAMPLE = os.path.join(os.path.dirname(__file__), "golden", "apls_spacenet_sample")
SN, CS = AM.PARAMS["spacenet"], AM.PARAMS["cityscale"]


def sample():
    with open(os.path.join(SAMPLE, "gt.json")) as f:
        gt = json.load(f)
    with open(os.path.join(SAMPLE, "prop.json")) as f:
        prop = json.load(f)
    return gt, prop


def ll(x, y):
    lat, lon = AM.xy2latlon(x, y)
    return [float(lat), float(lon)]


def dense(nodes, nbrs):
    return AM.DenseGraph(nodes=nodes, edges=[], nbrs=[sorted(n) for n in nbrs])


def star_pair():
    """Junction 0 (leaves 1, 2, 3) and junction 4 (leaves 5, 6, 7), joined by the chain 8..13: 7 hops apart."""
    pos = {0: (100, 100), 1: (80, 100), 2: (100, 80), 3: (80, 80), 4: (100, 240), 5: (120, 240), 6: (100, 260),
           7: (120, 260)}
    for k in range(8, 14):
        pos[k] = (100, 100 + 20 * (k - 7))
    nb = {0: {1, 2, 3, 8}, 1: {0}, 2: {0}, 3: {0}, 4: {5, 6, 7, 13}, 5: {4}, 6: {4}, 7: {4}}
    chain = [0] + list(range(8, 14)) + [4]
    for a, b in zip(chain[1:-1], chain[2:]):
        nb.setdefault(a, set()).add(b)
        nb.setdefault(b, set()).add(a)
    nb[8].add(0)
    return dense([ll(*pos[k]) for k in range(14)], [nb[k] for k in range(14)])


def to_oracle(g):
    return O._Scorer._graph(g)


def test_cover_through_the_other_graph_and_the_degree_one_exception():
    gt = star_pair()
    # the proposal graph joins ids 0 - 4 - 5: covering from GT node 0 there covers GT nodes 4 and 5
    prop = dense([ll(300, 300 + k) for k in range(6)], [{4}, set(), set(), set(), {0, 5}, {4}])
    cps = AM.control_points(gt, prop, SN)
    assert cps == [0, 1, 2, 3, 5, 6, 7]            # 4 covered (not a cp); 5 covered too but has degree 1
    assert 4 in AM.propagate(prop, 0, 4) and 4 not in AM.propagate(gt, 0, 4)   # the misreading would keep 4
    o = O.select_control_points(to_oracle(gt), to_oracle(prop), O.GoParams(True), O.GoOrder())
    assert sorted(o) == cps
    # an id past the other graph's node count covers only itself
    assert AM.propagate(prop, 11, 4) == {11}


def test_lockey_deduplicates():
    a, b = ll(100, 100), ll(100.5, 100.2)
    assert AM.lockey(a) == AM.lockey(b)
    nodes = [a, ll(80, 100), ll(100, 80), ll(80, 80), b, ll(130, 150), ll(150, 130), ll(150, 150)]
    gt = dense(nodes, [{1, 2, 3}, {0}, {0}, {0}, {5, 6, 7}, {4}, {4}, {4}])
    cps = AM.control_points(gt, dense([], []), SN)
    assert 0 in cps and 4 not in cps and cps == [0, 1, 2, 3, 5, 6, 7]
    assert sorted(O.select_control_points(to_oracle(gt), to_oracle(dense([], [])), O.GoParams(True),
                                          O.GoOrder())) == cps


def test_loc2key_half_even_tie_merges():
    # 40.98828125 = 40 + 253/256 is exact and sits on a tie at the 8th decimal: half-even gives ...812
    assert AM.loc2key([40.98828125, -70.9921875]) == "40.9882812_-70.9921875"
    assert "%.7f" % 40.99609375 == "40.9960938"
    lon = -70.9921875
    nodes = [[40.98828125, lon], [40.98828125 - 2e-5, lon], [40.9882812, lon], [40.9882812 + 2e-5, lon]]
    g = AM.densify(nodes, [[0, 1], [2, 3]])
    assert len(g.nodes) == 3 and g.nbrs[0] == [1, 2]       # half-up would give 40.9882813: four nodes
    og = O.GraphDensify(O.LoadGraph([nodes, [[0, 1], [2, 3]]]))
    assert og.Nodes == g.nodes and og.Edges == [list(e) for e in g.edges]


def test_self_loop_from_a_key_merge():
    p = ll(100, 100)
    nodes = [p, [p[0] + 1e-9, p[1]], ll(102, 100)]     # 0 and 1 share the key
    g = AM.densify(nodes, [[0, 1]])
    assert g.edges == [(0, 0)] and g.nbrs == [[0]]                      # degree 1
    g = AM.densify(nodes, [[0, 1], [0, 2]])
    assert g.nbrs == [[0, 1], [0]]                                       # degree 2 with one other neighbour
    # node 1 is the only junction; its chain walks 1 -> 0 -> 0 (the loop) -> 1
    cps = AM.control_points(g, dense([], []), SN)
    assert cps == [1]
    assert sorted(O.select_control_points(to_oracle(g), to_oracle(dense([], [])), O.GoParams(True),
                                          O.GoOrder())) == cps


@pytest.mark.parametrize("extra", [0, 1])
def test_chain_indices_at_interval_1(extra):
    n = SN.interval_1 + extra                      # a path of 15 or 16 nodes 2.5 m apart, no split
    nodes = [[41.0 - (100 + 2.5 * k) / 111111.0, ll(0, 150)[1]] for k in range(n)]
    g = AM.densify(nodes, [[k, k + 1] for k in range(n - 1)])
    assert len(g.nodes) == n
    cps = AM.control_points(g, dense([], []), SN)
    if extra == 0:
        assert cps == [0, n - 1]                   # len(chain) == interval_1: no interior point
    else:
        assert cps == [0, int(float(16) * 1.0 / 2.0), n - 1]     # n = int(16 / 10.0) + 1 = 2: index 8
    o = O.select_control_points(to_oracle(g), to_oracle(dense([], [])), O.GoParams(True), O.GoOrder())
    assert sorted(o) == cps


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_in_bound_exactly_at_the_margins(dataset):
    P = AM.PARAMS[dataset]
    c = math.cos(41.0 / 180.0 * 3.1415926)
    lat_lo = 41.0 - P.region_size / 111111.0 + P.margin_size / 111111.0
    lat_hi = 41.0 - P.margin_size / 111111.0
    lon_lo = -71.0 + P.margin_size / 111111.0 / c
    lon_hi = (-71.0 + P.region_size / 111111.0 / c) - P.margin_size / 111111.0 / c
    mid = [(lat_lo + lat_hi) / 2, (lon_lo + lon_hi) / 2]
    op = O.GoParams(dataset == "spacenet")
    for i, v, inward in ((0, lat_lo, math.inf), (0, lat_hi, -math.inf), (1, lon_lo, math.inf), (1, lon_hi, -math.inf)):
        p = list(mid)
        p[i] = v
        assert not AM.gps_in_bound(p, P) and not O.GPSInBound(p, op)
        p[i] = math.nextafter(v, inward)
        assert AM.gps_in_bound(p, P) and O.GPSInBound(p, op)


def test_gps_distance_uses_p1_cosine():
    a, b = [40.99, -70.99], [40.90, -70.80]
    assert AM.gps_distance(a, b) != AM.gps_distance(b, a)
    assert AM.gps_distance(a, b) == O.GPSDistance(a, b)
    # an edge under 3 m (kept whole by densify) whose two directed weights differ by a centimetre: 2.98999996 m
    # with u's cosine, 2.99000030 m with v's
    u, v = [40.99864999865, -70.99821123067021], [40.99862819434305, -70.99823212690804]
    g = AM.densify([u, v], [[0, 1]])
    assert g.nodes == [u, v]
    start, col, w = AM.arc_csr(g)
    assert start.tolist() == [0, 1, 2] and col.tolist() == [1, 0] and w.tolist() == [298, 299]
    assert w.tolist() == [int(O.GPSDistance(u, v) * 100.0), int(O.GPSDistance(v, u) * 100.0)]


def test_degree_space_nearest_is_not_the_metre_nearest():
    q = [40.99, -70.99]
    nodes = [[q[0], q[1] + 1e-4], [q[0] + 0.9e-4, q[1]]]
    assert AM.gps_distance(nodes[0], q) < AM.gps_distance(nodes[1], q)
    assert O.NearestNeighbors(nodes, 10, q) == [1, 0]
    gt = dense([q], [set()])
    prop = dense(nodes, [set(), set()])
    assert AM.snap(gt, prop, [0], [[1, 0] + [-1] * 8], SN) == [1]


def test_covered_nearest_falls_through_and_prop_step():
    # proposal path P0 - P1 - P2 - P3 - P4 (2 m hops); GT control points g0 at P0 and g1 with candidates [P0, P4]
    prop = dense([[40.99 - 2 * k / 111111.0, -70.99] for k in range(5)], [{1}, {0, 2}, {1, 3}, {2, 4}, {3}])
    gt = dense([prop.nodes[0], [prop.nodes[4][0], -70.99 + 1e-6]], [set(), set()])
    cand = [[0, 1, 2, 3, 4] + [-1] * 5, [0, 4] + [-1] * 8]
    assert AM.snap(gt, prop, [0, 1], cand, SN) == [0, 4]       # prop_step 3: P4 is not covered, the second candidate
    assert AM.snap(gt, prop, [0, 1], cand, CS) == [0, -1]      # prop_step 4 covers P4 as well: unmatched
    assert AM.snap(gt, prop, [0, 1], [cand[0], [0, 2, 4] + [-1] * 7], SN) == [0, 4]   # P2 covered too


def test_snap_radius_is_strict():
    # GPSDistance(p, q) is exactly 10.0 here; one ulp of p's latitude northwards brings it to 9.9999999995
    q, p = [40.99864999865, -70.99821123067021], [40.99859600337601, -70.99811582692163]
    assert AM.gps_distance(p, q) == 10.0 == O.GPSDistance(p, q)
    near = [math.nextafter(p[0], math.inf), p[1]]
    assert AM.gps_distance(near, q) < 10.0
    gt, cand = dense([q], [set()]), [[0] + [-1] * 9]
    assert AM.snap(gt, dense([p], [set()]), [0], cand, SN) == [-1]        # `<= 10.0` would match it
    assert AM.snap(gt, dense([near], [set()]), [0], cand, SN) == [0]


def test_pair_score_rules():
    """Penalties, d1 == filter, d1 unreachable, d2 unreachable, the clamp and the asymmetric pair, by hand."""
    order = O.GoOrder()
    cpg = {0: 0, 1: 1, 2: 2, 3: -1}
    sp_gt = {0: {0: 0, 1: 15000, 2: 10000}, 1: {0: 10000, 1: 0, 2: 20000}, 2: {0: 30000, 1: 20000, 2: 0}}
    sp_prop = {0: {0: 0, 1: 40000, 2: -1}, 1: {0: -1, 1: 0, 2: -1}, 2: {0: -1, 1: 90000, 2: 0}}
    r = O.score_pairs(cpg, sp_gt, sp_prop, 100.0, order)
    assert (r["penalty"], r["skipped"], r["scored"], r["cc"], r["sum"]) == (3, 1, 2, 5, 5.0) and r["apls"] == 0.0
    sp_gt[1][0] = 20000                        # read from the larger id, (0, 1) would still score; it reads 0 -> 1
    sp_gt[0][1] = 10000                        # now d1 == the filter: skipped
    r = O.score_pairs(cpg, sp_gt, sp_prop, 100.0, order)
    assert (r["skipped"], r["scored"]) == (2, 1)
    r = O.score_pairs({0: 0, 1: 1}, {0: {0: 0, 1: 15000}, 1: {0: 0, 1: 0}}, {0: {0: 0, 1: 12000}, 1: {0: 0, 1: 0}},
                      100.0, order)
    assert r["sum"] == abs(150.0 - 120.0) / 150.0 and r["apls"] == 1.0 - r["sum"] / 1.0
    r = O.score_pairs({0: -1}, {}, {}, 100.0, order)
    assert r["cc"] == 0 and math.isnan(r["apls"])


def test_lines_and_nan():
    assert AM.apls_line(float("nan"), float("nan")) == "NaN NaN NaN\n"
    assert AM.apls_line(1.0, float("nan")) == "1.000000 NaN NaN\n"
    assert AM.apls_line(0.1234565, 0.5) == "%f %f %f\n" % (0.1234565, 0.5, (0.1234565 + 0.5) / 2.0)
    assert AM.fmt_f(0.0000005) == "0.000000" and AM.fmt_f(0.0000015) == "0.000002"   # the binary value rounds


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_straight_road_against_itself_is_one(dataset):
    x = 1000.0 if dataset == "cityscale" else 150.0
    road = {(x, 60.0 if dataset == "spacenet" else 150.0): [(x, 300.0)]}
    road[(x, 300.0)] = [next(iter(road))]
    a = AM.apls_tile(road, road, dataset, scorer=O.scorer)
    assert a[:3] == (1.0, 1.0, 1.0) and a[3].gt_way.result["cc"] > 0 and a[3].line == "1.000000 1.000000 1.000000\n"


def test_convert_dict_order_and_missing_key():
    adj = {(5, 5): [(1, 1), (5, 5)], (1, 1): [(5, 5), (9, 9)], (9, 9): [(1, 1)]}
    nodes, edges = AM.convert(adj)
    assert nodes == [ll(5, 5), ll(1, 1), ll(9, 9)] and edges == [[0, 1], [0, 0], [1, 2]]
    assert [nodes, edges] == O.convert_pickle(adj)
    with pytest.raises(ValueError, match=r"\(7, 7\)"):
        AM.convert({(1, 1): [(7, 7)]})


def equal_host_stages(gt_raw, prop_raw, dataset):
    a = AM.apls_graphs(*gt_raw, *prop_raw, dataset=dataset, scorer=O.scorer)
    o = O.apls(gt_raw, prop_raw, spacenet=dataset == "spacenet")
    d = a[3]
    for mine, theirs in ((d.gt, o[3][0]), (d.prop, o[3][1])):
        assert mine.nodes == theirs.Nodes and [list(e) for e in mine.edges] == theirs.Edges
        assert mine.nbrs == [sorted(theirs.neighbors.get(i, {})) for i in range(len(theirs.Nodes))]
    for w, ow in ((d.gt_way, o[4][0]), (d.prop_way, o[4][1])):
        assert w.control_points == ow["control_points"] and w.matches == ow["matches"]
        assert [list(c) for c in w.candidates] == [c + [-1] * (10 - len(c)) for c in ow["candidates"]]
    assert d.line == o[2]
    return a


@pytest.mark.parametrize("dataset", ["spacenet", "cityscale"])
def test_host_stages_equal_oracle_on_the_sample(dataset):
    equal_host_stages(*sample(), dataset)


@pytest.mark.parametrize("dataset,seed", [("spacenet", 0), ("spacenet", 1), ("cityscale", 2)])
def test_host_stages_equal_oracle_on_synthetic_tiles(dataset, seed):
    extent = 400 if dataset == "spacenet" else 700
    gt = AM.convert(synth.make_road_graph(extent, seed=seed))
    prop = AM.convert(synth.make_road_graph(extent, seed=seed + 7, spacing=40))
    a = equal_host_stages(gt, prop, dataset)
    assert a[3].gt_way.result["scored"] > 0


class IntGraph(O.Graph):
    def __init__(self, n, arcs):
        super().__init__()
        self.Nodes = [[0.0, 0.0]] * n
        self.w = {}
        for u, v, w in arcs:
            self.neighbors.setdefault(u, {})[v] = True
            self.w[(u, v)] = w

    def arc(self, u, v):
        return self.w[(u, v)]


def check_dijkstra(n, arcs, sources):
    g = IntGraph(n, arcs)
    a = np.array(arcs, dtype=np.int64).reshape(-1, 3)
    m = sp.csr_matrix((a[:, 2].astype(np.float64), (a[:, 0], a[:, 1])), shape=(n, n))
    ref = dijkstra(m, directed=True, indices=sources)
    for i, s in enumerate(sources):
        r = g.ShortestPaths(s, list(range(n)), O.GoOrder())
        got = np.array([r[t] for t in range(n)])
        exp = np.where(np.isfinite(ref[i]), ref[i] / 100.0, -1.0)
        assert np.array_equal(got, exp)


@pytest.mark.parametrize("seed", range(3))
def test_oracle_dijkstra_equals_scipy_on_random_digraphs(seed):
    rng = np.random.default_rng(seed)
    n = 300
    pairs = {(int(u), int(v)) for u, v in rng.integers(0, n, size=(900, 2)) if u != v}
    arcs = [(u, v, int(rng.integers(0, 50))) for u, v in sorted(pairs)]
    check_dijkstra(n, arcs, [0, 5, 77])


def test_oracle_dijkstra_long_path_and_zero_cycles():
    n = 20000
    arcs = [(k, k + 1, 3) for k in range(n - 1)] + [(k + 1, k, 2) for k in range(n - 1)]
    check_dijkstra(n, arcs, [0, n - 1])
    arcs = [(k, (k + 1) % 50, 0) for k in range(50)] + [(k, 50 + k, k) for k in range(50)] + [(60, 3, 1)]
    check_dijkstra(100, arcs, [0, 60])


def write_results(tmp_path, lines):
    d = tmp_path / "results" / "apls"
    d.mkdir(parents=True)
    for name, text in lines.items():
        (d / name).write_text(text)


def test_cityscale_aggregator(tmp_path):
    write_results(tmp_path, {"9.txt": "0.5 0.5 0.512345\n", "19.txt": "0.1 0.2 0.150000\n", "8.txt": "NaN NaN NaN\n",
                             "28.txt": "0.9 0.9 0.987654\n"})
    out = AM.aggregate(str(tmp_path), "cityscale")
    # sorted: 19, 28, 8 (NaN: reading stops), 9 never read; the sixth decimal is dropped
    assert out["apls"] == [0.15, 0.98765] and out["final_APLS"] == np.mean([0.15, 0.98765])
    assert json.loads((tmp_path / "score" / "apls.json").read_text()) == {"apls": [0.15, 0.98765],
                                                                          "final_APLS": np.mean([0.15, 0.98765])}


def test_spacenet_aggregator(tmp_path):
    write_results(tmp_path, {"b.txt": "0.5 0.5 0.512345\n", "a.txt": "NaN 0.2 NaN\n", "c.txt": "0.1 0.2 0.150000\n"})
    out = AM.aggregate(str(tmp_path), "spacenet")
    assert out["apls"] == [["b.txt", 0.512345], ["c.txt", 0.15]]
    assert json.loads((tmp_path / "results" / "apls.json").read_text()) == {
        "apls": [["b.txt", 0.512345], ["c.txt", 0.15]], "final_APLS": np.mean([0.512345, 0.15])}


def test_go_order_spread(report_dir):
    """Go randomises its map iteration; the oracle emulates 32 runs per tile.  Information for DESIGN.md §15."""
    tiles = {"spacenet_sample/spacenet": (sample(), True), "spacenet_sample/cityscale": (sample(), False),
             "make_road_graph_300/spacenet": ((O.convert_pickle(synth.make_road_graph(300, seed=4)),
                                               O.convert_pickle(synth.make_road_graph(300, seed=9, spacing=40))),
                                              True)}
    report = {}
    for name, ((gt, prop), spacenet) in tiles.items():
        base = O.apls(gt, prop, spacenet=spacenet)
        mine = AM.apls_graphs(*gt, *prop, dataset="spacenet" if spacenet else "cityscale", scorer=O.scorer)
        assert mine[3].line == base[2]
        vals = []
        for seed in range(32):
            a, b, _, _, _ = O.apls(gt, prop, spacenet=spacenet, order_seed=seed)
            vals.append((a + b) / 2.0)
        report[name] = dict(ascending_ids=(base[0] + base[1]) / 2.0, min=min(vals), max=max(vals),
                            median=float(np.median(vals)))
    with open(os.path.join(report_dir, "apls_go_order_spread.json"), "w") as f:
        json.dump(report, f, indent=1)
