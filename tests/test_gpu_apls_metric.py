"""APLS metric on the device (csrc/apls_metric.cu): the snapping candidates, both distance matrices, the counts, the
bits of the exact pair sum, the scores and the file line equal the oracle (oracle/apls_oracle.py) on the reference's
spacenet sample, synthetic tiles and edge cases; shortest paths equal scipy on random digraphs; capacities are
refused exactly past the need without spoiling the handle; a handle is reusable and two runs are bitwise equal."""
import json
import math
import os
import pickle

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import dijkstra

from oracle import apls_oracle as O
from sam_road_b200 import apls_metric as AM
from sam_road_b200 import synth

pytestmark = pytest.mark.gpu

SAMPLE = os.path.join(os.path.dirname(__file__), "golden", "apls_spacenet_sample")
# a straight two-way road of 200 px (200 m) along one row, well inside both datasets' bounds
ROAD = {(1000.0, 100.0): [(1000.0, 300.0)], (1000.0, 300.0): [(1000.0, 100.0)]}
SMALL_ROAD = {(150.0, 60.0): [(150.0, 260.0)], (150.0, 260.0): [(150.0, 60.0)]}


def sample():
    with open(os.path.join(SAMPLE, "gt.json")) as f:
        gt = json.load(f)
    with open(os.path.join(SAMPLE, "prop.json")) as f:
        prop = json.load(f)
    return gt, prop


@pytest.fixture(scope="module")
def dev():
    d = AM.AplsDevice(0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def city():
    return synth.city_tile()


def same_float(a, b):
    return (math.isnan(a) and math.isnan(b)) or np.float64(a).tobytes() == np.float64(b).tobytes()


def check_equal(a, b):
    """Device run `a` against oracle-scored run `b` (both apls_graphs / apls_tile results with export=True)."""
    da, db = a[3], b[3]
    assert da.line == db.line
    for x, y in zip(a[:3], b[:3]):
        assert same_float(x, y)
    for wa, wb in ((da.gt_way, db.gt_way), (da.prop_way, db.prop_way)):
        assert wa.control_points == wb.control_points
        assert np.array_equal(np.asarray(wa.candidates).reshape(-1, 10), np.asarray(wb.candidates).reshape(-1, 10))
        assert wa.matches == wb.matches
        ra, rb = wa.result, wb.result
        for k in ("cc", "penalty", "skipped", "scored", "pairs"):
            assert ra[k] == rb[k], k
        assert np.float64(ra["sum"]).tobytes() == np.float64(rb["sum"]).tobytes()
        assert np.array_equal(ra["dist_gt"], np.asarray(rb["dist_gt"], dtype=np.int32).reshape(ra["dist_gt"].shape))
        assert np.array_equal(ra["dist_prop"],
                              np.asarray(rb["dist_prop"], dtype=np.int32).reshape(ra["dist_prop"].shape))
        assert same_float(wa.apls, wb.apls)


def both_raw(dev, gt_raw, prop_raw, dataset, scorer=O.scorer):
    a = AM.apls_graphs(*gt_raw, *prop_raw, dataset=dataset, device=dev, export=True)
    b = AM.apls_graphs(*gt_raw, *prop_raw, dataset=dataset, scorer=scorer, export=True)
    check_equal(a, b)
    return a


def both(dev, gt, prop, dataset, scorer=O.scorer):
    return both_raw(dev, AM.convert(gt), AM.convert(prop), dataset, scorer)


@pytest.mark.parametrize("dataset", ["spacenet", "cityscale"])
def test_spacenet_sample_equals_oracle(dev, dataset):
    gt, prop = sample()
    a = both_raw(dev, gt, prop, dataset)
    o = O.apls(gt, prop, spacenet=dataset == "spacenet")    # the oracle end to end, its own host stages
    assert a[3].line == o[2]
    assert a[3].gt_way.result["cc"] > 0 and a[3].prop_way.result["cc"] > 0


@pytest.mark.parametrize("dataset,seed", [("spacenet", 0), ("spacenet", 3), ("cityscale", 0)])
def test_road_graph_tiles(dev, dataset, seed):
    extent = 400 if dataset == "spacenet" else 600
    gt = synth.make_road_graph(extent, seed=seed)
    prop = synth.make_road_graph(extent, seed=seed + 1, spacing=40)
    a = both(dev, gt, prop, dataset)
    assert a[3].gt_way.result["scored"] > 0


def test_city_tile(dev, city):
    gt, prop = city
    a = both(dev, gt, prop, "cityscale", scorer=O.scipy_scorer)
    assert len(a[3].gt_way.control_points) > 900 and a[3].gt_way.result["scored"] > 100000
    # the chains collapse: far fewer terminals than nodes
    assert a[3].gt_way.result["terminals"][0] < len(a[3].gt.nodes) // 10


def test_empty_proposal(dev):
    gt = synth.make_road_graph(400, seed=0)
    a = both(dev, gt, {}, "spacenet")
    assert math.isnan(a[1]) and a[3].prop_way.result["cc"] == 0
    assert a[3].gt_way.result["penalty"] == a[3].gt_way.result["pairs"] > 0     # nothing matched: all penalties
    assert a[3].line.endswith(" NaN NaN\n")


def test_proposal_equals_gt(dev):
    gt = synth.make_road_graph(400, seed=2)
    a = both(dev, gt, gt, "spacenet")
    assert a[3].gt_way.result["penalty"] == 0 and a[0] == 1.0 and a[1] == 1.0


@pytest.mark.parametrize("dataset", ["spacenet", "cityscale"])
def test_single_edge(dev, dataset):
    road = SMALL_ROAD if dataset == "spacenet" else ROAD
    a = both(dev, road, road, dataset)
    assert a[:3] == (1.0, 1.0, 1.0) and a[3].gt_way.result["scored"] > 0


def test_disconnected_components(dev):
    # two roads far apart on both sides: pairs across the components are unreachable (skipped); a third GT road
    # that the proposal lacks gives penalties
    gt = dict(ROAD)
    gt.update({(1400.0, 500.0): [(1400.0, 900.0)], (1400.0, 900.0): [(1400.0, 500.0)]})
    prop = {(x + 1.0, y): [(u + 1.0, v) for u, v in nb] for (x, y), nb in gt.items()}
    gt.update({(600.0, 1200.0): [(600.0, 1500.0)], (600.0, 1500.0): [(600.0, 1200.0)]})
    a = both(dev, gt, prop, "cityscale")
    d = a[3].gt_way.result["dist_gt"]
    assert (d == -1).any() and a[3].gt_way.result["skipped"] > 0 and a[3].gt_way.result["penalty"] > 0


def test_zero_weight_arcs(dev):
    # a longitude step of 1e-7 degree is 0.84 cm here: distinct %.7f keys, arc weight int(0.84) = 0
    lat0, lon0 = 40.999, -70.997
    lat1, e = lat0 - 150 / 111111.0, 1e-7
    nodes = [[lat0, lon0], [lat1, lon0], [lat1, lon0 + e], [lat0 - 300 / 111111.0, lon0 + e], [lat1, lon0 + 0.001]]
    edges = [[0, 1], [1, 2], [2, 3], [1, 4], [2, 4]]
    a = both_raw(dev, [nodes, edges], [nodes, edges], "cityscale")
    w = AM.arc_csr(a[3].gt)[2]
    assert (w == 0).any()


def test_component_without_junction(dev):
    # a closed ring: every node has degree 2, so it has no control point; the open road beside it has
    ring = {}
    pts = [(1000.0 + 150 * math.cos(k * math.pi / 8), 1000.0 + 150 * math.sin(k * math.pi / 8)) for k in range(16)]
    for k, p in enumerate(pts):
        ring.setdefault(p, []).append(pts[(k + 1) % 16])
        ring.setdefault(pts[(k + 1) % 16], []).append(p)
    gt = dict(ROAD)
    gt.update(ring)
    a = both(dev, gt, gt, "cityscale")
    ring_ids = {i for i, nb in enumerate(a[3].gt.nbrs) if len(nb) == 2}
    assert a[3].gt_way.control_points and a[3].gt_way.result["scored"] > 0
    assert len(ring_ids) > len(a[3].gt.nodes) // 2


def test_pair_rules_on_hand_distances(dev):
    # GT role: 0 -> 1 150 m but 1 -> 0 100 m (the smaller id's row is read), 0 -> 2 exactly the 100 m filter, node 3
    # unreachable; proposal: 0 -> 1 400 m (the term clamps to 1), nothing from 1 to 2 (d2 = 0, the term is 1)
    ll = [[40.99, -70.99], [40.98, -70.99], [40.97, -70.99], [40.96, -70.99]]
    dev.upload_csr(0, ll, [0, 2, 3, 4, 4], [1, 2, 0, 1], [15000, 10000, 10000, 20000])
    dev.upload_csr(1, ll, [0, 1, 1, 2, 2], [1, 1], [40000, 90000])
    r = dev.one_way(0, [0, 1, 2, 3], [0, 1, 2, -1], 100.0, export=True)
    assert r["dist_gt"].tolist() == [[0, 15000, 10000], [10000, 0, 20000], [30000, 20000, 0]]
    assert r["dist_prop"].tolist() == [[0, 40000, -1], [-1, 0, -1], [-1, 90000, 0]]
    assert (r["penalty"], r["skipped"], r["scored"], r["cc"], r["sum"]) == (3, 1, 2, 5, 5.0)
    r = dev.one_way(0, [0, 1, 2, 3], [0, 1, 2, 3], 100.0)       # d1 unreachable: the pairs with 3 are skipped
    assert (r["penalty"], r["skipped"], r["scored"], r["cc"], r["sum"]) == (0, 4, 2, 2, 2.0)
    r = dev.one_way(1, [0, 1, 2], [0, 1, 2], 100.0)             # the proposal as GT: only (0, 1) is reachable
    assert (r["penalty"], r["skipped"], r["scored"], r["sum"]) == (0, 2, 1, abs(400.0 - 150.0) / 400.0)


def test_candidates_in_degree_space(dev):
    # B is nearer in degrees (0.9 * 1e-4 of latitude) than A (1e-4 of longitude) but farther in metres
    q = [40.99, -70.99]
    ll = [[q[0], q[1] + 1e-4], [q[0] + 0.9e-4, q[1]]] + [[q[0] + 0.01 * k, q[1]] for k in range(1, 12)]
    dev.upload_csr(1, ll, np.zeros(len(ll) + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32))
    c = dev.candidates(1, [q])[0].tolist()
    assert c[:2] == [1, 0] and c == O.NearestNeighbors(ll, 10, q)
    assert AM.gps_distance(ll[0], q) < AM.gps_distance(ll[1], q)
    # ties: four nodes at the same box distance come out in ascending id
    ll = [[q[0] + 1e-4, q[1]], [q[0] - 1e-4, q[1]], [q[0], q[1] + 1e-4], [q[0], q[1] - 1e-4]]
    dev.upload_csr(1, ll, np.zeros(5, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32))
    assert dev.candidates(1, [q])[0].tolist() == O.NearestNeighbors(ll, 10, q) + [-1] * 6


def test_shortest_paths_enter_a_chain_from_a_one_way_arc(dev):
    # c has out-neighbours {a, b}, both with arcs back, and an extra in-arc from x: c is a terminal, not a chain node,
    # or the path x -> c -> b (17) would be lost
    x, c, a, b = 0, 1, 2, 3
    rows = np.array([x, c, a, c, b], dtype=np.int32)
    cols = np.array([c, a, c, b, c], dtype=np.int32)
    w = np.array([10, 5, 5, 7, 7], dtype=np.int32)
    r = sssp_check(dev, 4, rows, cols, w, [x, a, b])
    assert r["dist_gt"][0].tolist() == [0, 15, 17]


def test_shortest_paths_one_way_arcs_into_chains(dev):
    # a two-way path with random weights, plus one-way arcs from random nodes into (and out of) random path nodes
    rng = np.random.default_rng(11)
    n = 4000
    k = np.arange(n - 1, dtype=np.int32)
    extra = rng.integers(0, n, size=(400, 2)).astype(np.int32)
    extra = extra[extra[:, 0] != extra[:, 1]]
    pairs = np.unique(np.concatenate([np.stack([k, k + 1], 1), np.stack([k + 1, k], 1), extra]), axis=0)
    rows, cols = pairs[:, 0].astype(np.int32), pairs[:, 1].astype(np.int32)
    w = rng.integers(0, 500, size=rows.size).astype(np.int32)
    sssp_check(dev, n, rows, cols, w, rng.choice(n, 40, replace=False))


def upload_digraph(dev, n, rows, cols, w):
    order = np.lexsort((cols, rows))
    rows, cols, w = rows[order], cols[order], w[order]
    start = np.zeros(n + 1, dtype=np.int32)
    np.add.at(start, rows + 1, 1)
    start = np.cumsum(start).astype(np.int32)
    ll = np.stack([41.0 - np.arange(n) * 1e-5, np.full(n, -70.99)], 1)
    for which in (0, 1):
        dev.upload_csr(which, ll, start, cols, w)


def sssp_check(dev, n, rows, cols, w, sources):
    upload_digraph(dev, n, rows, cols, w)
    sources = np.sort(np.asarray(sources))
    r = dev.one_way(0, sources, sources, 0.0, export=True)
    m = sp.csr_matrix((w.astype(np.float64), (rows, cols)), shape=(n, n))
    d = dijkstra(m, directed=True, indices=sources)[:, sources]
    ref = np.where(np.isfinite(d), d, -1).astype(np.int64)
    assert np.array_equal(r["dist_gt"], ref) and np.array_equal(r["dist_prop"], ref)
    return r


@pytest.mark.parametrize("n,seed", [(2000, 0), (30000, 1), (AM.DEFAULT_CAPS["max_nodes"], 2)])
def test_shortest_paths_random_digraphs(dev, n, seed):
    rng = np.random.default_rng(seed)
    m = min(3 * n, AM.DEFAULT_CAPS["max_arcs"])
    pairs = np.unique(rng.integers(0, n, size=(m, 2)), axis=0)
    rows, cols = pairs[:, 0].astype(np.int32), pairs[:, 1].astype(np.int32)
    w = rng.integers(0, 2000, size=rows.size).astype(np.int32)
    w[rng.random(rows.size) < 0.05] = 0
    sssp_check(dev, n, rows, cols, w, rng.choice(n, 48, replace=False))


def test_shortest_paths_on_a_pure_cycle(dev):
    n = 5000
    a = np.arange(n, dtype=np.int32)
    rows = np.concatenate([a, (a + 1) % n]).astype(np.int32)
    cols = np.concatenate([(a + 1) % n, a]).astype(np.int32)
    rng = np.random.default_rng(7)
    w = rng.integers(0, 300, size=rows.size).astype(np.int32)
    r = sssp_check(dev, n, rows, cols, w, [17, 1200, 2500, 4999])
    assert r["terminals"][0] == 4          # every node is a chain node: only the sources remain


def test_shortest_paths_thousands_of_hops(dev):
    n = 20000
    a = np.arange(n - 1, dtype=np.int32)
    rows = np.concatenate([a, a + 1]).astype(np.int32)
    cols = np.concatenate([a + 1, a]).astype(np.int32)
    w = np.concatenate([np.full(n - 1, 200), np.full(n - 1, 201)]).astype(np.int32)
    r = sssp_check(dev, n, rows, cols, w, np.arange(0, n, 7))      # 2858 sources, routes up to 2857 arcs
    assert r["terminals"][0] >= 2858


def test_weight_sum_beyond_int32_refused(dev):
    w = np.array([2 ** 30, 2 ** 30], dtype=np.int32)
    with pytest.raises(RuntimeError, match="exceed int32"):
        dev.upload_csr(0, [[41.0, -71.0], [40.9, -71.0]], np.array([0, 1, 2], np.int32), np.array([1, 0], np.int32), w)
    both(dev, ROAD, ROAD, "cityscale")


def needs(gt_raw, prop_raw, dataset):
    r = AM.apls_graphs(*gt_raw, *prop_raw, dataset=dataset, scorer=O.scorer)
    d = r[3]
    return dict(max_nodes=max(len(d.gt.nodes), len(d.prop.nodes)),
                max_arcs=max(sum(map(len, d.gt.nbrs)), sum(map(len, d.prop.nbrs))),
                max_control_points=max(len(d.gt_way.control_points), len(d.prop_way.control_points)))


@pytest.mark.parametrize("cap", ["max_nodes", "max_arcs", "max_control_points"])
def test_capacity_exact_and_one_below(cap):
    gt, prop = sample()
    need = needs(gt, prop, "spacenet")[cap]
    d = AM.AplsDevice(0, **{cap: need})
    try:
        both_raw(d, gt, prop, "spacenet")
    finally:
        d.close()
    d = AM.AplsDevice(0, **{cap: need - 1})
    try:
        with pytest.raises(RuntimeError, match=cap):
            AM.apls_graphs(*gt, *prop, dataset="spacenet", device=d)
        both(d, SMALL_ROAD, SMALL_ROAD, "spacenet")
    finally:
        d.close()


def test_handle_reuse_small_city_small(city):
    gt, prop = sample()
    d = AM.AplsDevice(0)
    try:
        runs = [("raw", gt, prop, "spacenet"), ("adj", city[0], city[1], "cityscale"), ("raw", prop, gt, "spacenet")]
        for kind, g, p, ds in runs:
            f = AM.apls_graphs if kind == "raw" else AM.apls_tile
            args = (*g, *p) if kind == "raw" else (g, p)
            a = f(*args, dataset=ds, device=d, export=True)
            fresh = AM.AplsDevice(0)
            try:
                b = f(*args, dataset=ds, device=fresh, export=True)
            finally:
                fresh.close()
            check_equal(a, b)
    finally:
        d.close()


def test_two_runs_bitwise_equal(dev, city):
    a = AM.apls_tile(*city, "cityscale", device=dev, export=True)
    b = AM.apls_tile(*city, "cityscale", device=dev, export=True)
    check_equal(a, b)
    assert a[3].gt_way.result["sum_fixed"] == b[3].gt_way.result["sum_fixed"]


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_cli_end_to_end(tmp_path, dataset):
    root = tmp_path / dataset
    tiles = [8, 9, 19] if dataset == "cityscale" else ["AOI_2_t0", "AOI_2_t1", "AOI_2_t2"]
    extent = 500 if dataset == "cityscale" else 400
    for out in ("dev", "ora"):
        (tmp_path / out / "graph").mkdir(parents=True)
    if dataset == "cityscale":
        (root / "20cities").mkdir(parents=True)
    else:
        (root / "RGB_1.0_meter").mkdir(parents=True)
        (root / "data_split.json").write_text(json.dumps({"test": tiles + ["AOI_2_missing"]}))
    for k, t in enumerate(tiles):
        g = synth.make_road_graph(extent, seed=k)
        p = {} if k == 1 else synth.make_road_graph(extent, seed=k + 5, spacing=40)
        with open(AM.gt_path(dataset, str(root), t), "wb") as f:
            pickle.dump(g, f)
        for out in ("dev", "ora"):
            with open(tmp_path / out / "graph" / f"{t}.p", "wb") as f:
                pickle.dump(p, f)
    AM.main(["--savedir", str(tmp_path / "dev"), "--dataset", dataset, "--gt-root", str(root)])
    AM.run_tiles(str(tmp_path / "ora"), dataset, str(root), scorer=O.scorer)
    AM.aggregate(str(tmp_path / "ora"), dataset)
    files = sorted(os.listdir(tmp_path / "dev" / "results" / "apls"))
    assert files == sorted(f"{t}.txt" for t in tiles)
    for name in files:
        assert (tmp_path / "dev" / "results" / "apls" / name).read_bytes() == \
            (tmp_path / "ora" / "results" / "apls" / name).read_bytes()
    js = "score/apls.json" if dataset == "cityscale" else "results/apls.json"
    assert (tmp_path / "dev" / js).read_bytes() == (tmp_path / "ora" / js).read_bytes()
