"""TOPO metric at the limits of csrc/topo_metric.cu, against oracle/topo_oracle.py with exact equality: several
chunks of pair slots, one handle across graphs of changing size, capacities exactly at and one below the need,
matchings that need long augmenting paths, the candidate test on its boundaries, walks on awkward graphs and a
city-sized tile, and the argument refusals of samroad_topo_upload_graph / samroad_topo_run."""
import math

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import maximum_bipartite_matching

from oracle import topo_oracle
from sam_road_b200 import _lib
from sam_road_b200 import topo_metric as TM
from sam_road_b200.synth import city_tile
from test_gpu_topo_metric import TINY_GT, TINY_PROP, both, lat_path
from test_topo_host import GOLDEN, check_tile, load_tiles

pytestmark = pytest.mark.gpu

D = 1 / 1024.0          # node spacing of the exact-geometry graphs, in degrees
KINDS = {"max_marbles": "marbles", "max_queue": "queued", "max_covered": "covered", "max_candidates": "candidate"}


@pytest.fixture(scope="module")
def dev():
    d = TM.TopoDevice(0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def tiles():
    return load_tiles(np.load(GOLDEN))


def make_graph(nodes, edges):
    """A RoadGraph with the link lists exactly as given: directed edges in order, repeats kept."""
    g = TM.RoadGraph()
    g.nodes = [list(p) for p in nodes]
    g.edges = list(edges)
    g.link = [[] for _ in nodes]
    g.rlink = [[] for _ in nodes]
    for a, b in edges:
        g.link[a].append(b)
        g.rlink[b].append(a)
    return g


def meridian(n, lat0=40.0, lon=-70.0, two_way=True):
    """n nodes D apart along a meridian: every length, distance sum and sample position is exact in float64."""
    edges = [(k, k + 1) for k in range(n - 1)]
    if two_way:
        edges = [e for a, b in edges for e in ((a, b), (b, a))]
    return make_graph([(lat0 + k * D, lon) for k in range(n)], edges)


def oracle_rows(gt, prop, pn, pd, r, step, threshold):
    stats = [{} for _ in pn]
    ref = np.array([topo_oracle.pair_counts(gt, prop, [int(v) for v in n], [float(v) for v in d], r, step,
                                            threshold, stats=s) for n, d, s in zip(pn, pd, stats)],
                   dtype=np.int32).reshape(-1, 6)
    return ref, stats


def score(dev, gt, prop, pn, pd, r, step, threshold):
    """Device counts of hand-made pairs, asserted equal to the oracle's; returns (counts, oracle statistics)."""
    dev.upload(0, gt)
    dev.upload(1, prop)
    got = dev.run(np.array(pn, dtype=np.int32), np.array(pd, dtype=np.float64), r, step, threshold)
    ref, stats = oracle_rows(gt, prop, pn, pd, r, step, threshold)
    assert np.array_equal(got, ref), (got, ref)
    return got, stats


def tile_pairs(gt_adj, prop_adj):
    """Graphs, pair arrays and r of a tile scored alone, as topo_tile hands them to the device."""
    state = TM.TopoState()
    gt, prop = TM.create_graph(gt_adj, state), TM.create_graph(prop_adj, state)
    starts = TM.starting_points(gt, TM.region_of(state))
    pairs = TM.generate_pairs(prop, gt, starts)
    got = {}
    TM.pair_counts(gt, prop, starts, pairs, 0, 0, 0, lambda pn, pd, *a: got.update(pn=pn, pd=pd))
    r = 0.0015 if TM.LAT_TOP_LEFT - state.min_lat < 0.01 else 0.003
    return gt, prop, got["pn"], got["pd"], r


# ---------------------------------------------------------------------------------------------- 1. chunked slots

@pytest.fixture(scope="module")
def default_counts(dev, tiles):
    state, out = TM.TopoState(), []
    for t in (0, 1):
        out.append(TM.topo_tile(*tiles[t], state, "cityscale", device=dev)[2].counts)
    return out


@pytest.mark.parametrize("slots", [1, 3, 7, 35, 36, 37, 38, 39])
def test_golden_tiles_in_chunks(tiles, default_counts, slots):
    z = np.load(GOLDEN)
    d = TM.TopoDevice(0, slots=slots)
    try:
        state = TM.TopoState()
        for t in (0, 1):
            p, rr, det = TM.topo_tile(*tiles[t], state, "cityscale", device=d)
            check_tile(z, "cityscale", t, p, rr, det)
            assert np.array_equal(det.counts, default_counts[t])
            assert (det.counts.shape[0] > slots) == (slots < (38, 36)[t])   # 38 and 36 pairs: chunked below that
    finally:
        d.close()


@pytest.mark.parametrize("slots", [1, 2])
def test_slot_reuse_after_a_large_pair(slots):
    # A: a long walk from the middle (many marbles and covered edges); Z: start distances beyond r, so nothing is
    # placed and no node is expanded; B: a short walk at the far end; every ordered succession of two of them
    # happens in one slot, for one slot and for two
    g = meridian(40)
    h = D / 2
    A, Z, B = ([19, 20, 19, 20], [h, h, h, h]), ([19, 20, 5, 6], [1.0] * 4), ([38, 39, 37, 38], [h, h, h, h])
    order = [A, Z, B, A, A, B, Z, A] if slots == 1 else [A, A, Z, Z, B, B, A, A, A, B, B, Z, Z, A, A, A]
    d = TM.TopoDevice(0, slots=slots)
    try:
        got, stats = score(d, g, g, [p[0] for p in order], [p[1] for p in order], 12 * D, D / 4, D / 4)
    finally:
        d.close()
    assert len(order) > slots
    ia, iz, ib = order.index(A), order.index(Z), order.index(B)
    assert (got[iz] == 0).all() and got[ia, 0] > got[ib, 0] > 0 and min(stats[ia]["covered"]) >= 20


# ---------------------------------------------------------------------------------------------- 2. handle reuse

@pytest.fixture(scope="module")
def city(dev):
    gt, prop = city_tile()
    return gt, prop, TM.topo_tile(gt, prop, TM.TopoState(), "cityscale", device=dev)[2]


def test_one_handle_across_graph_sizes(tiles, city):
    # small -> large -> small, the GT larger than the proposal and then the reverse, the first tile again at the end
    seq = [(TINY_GT, TINY_PROP), tiles[0], (city[0], city[1]), (tiles[1][1], tiles[1][0]), (city[1], city[0]),
           tiles[3], (TINY_GT, TINY_PROP)]
    sizes = [(len(a), len(b)) for a, b in seq]
    assert sizes[1][0] < sizes[2][0] > sizes[3][0] and sizes[2][0] < sizes[2][1] and sizes[4][0] > sizes[4][1]
    one = TM.TopoDevice(0)
    try:
        for i, (gt, prop) in enumerate(seq):
            a = TM.topo_tile(gt, prop, TM.TopoState(), "cityscale", device=one)[2]
            if (gt, prop) == (city[0], city[1]):
                b = city[2]
            else:
                fresh = TM.TopoDevice(0)
                try:
                    b = TM.topo_tile(gt, prop, TM.TopoState(), "cityscale", device=fresh)[2]
                finally:
                    fresh.close()
            assert np.array_equal(a.counts, b.counts) and a.lines == b.lines, i
    finally:
        one.close()


def test_node_count_changes_without_a_new_layout():
    # 10 and then 13 nodes: the dense distance maps round to the same 256 bytes and both runs use two slots, so the
    # workspace is neither laid out again nor cleared; only the serial separates the second tile's stamps
    small, large = lat_path(9), lat_path(12)
    for width in (8, 4):
        assert (width * len(small.nodes) + 255) // 256 == (width * len(large.nodes) + 255) // 256
    h = D / 2
    pn, pd = [[3, 4, 3, 4], [4, 3, 3, 4], [2, 3, 3, 4]], [[h, h, h, h], [h, h, h, h], [h, 3 * h, h, h]]
    d = TM.TopoDevice(0, slots=2)
    try:
        a, _ = score(d, small, small, pn, pd, 12 * h, D / 4, D / 4)
        b, _ = score(d, large, large, pn, pd, 12 * h, D / 4, D / 4)
        c, _ = score(d, small, large, pn, pd, 12 * h, D / 4, D / 4)
        assert not np.array_equal(a, b)      # the longer path is walked further north
        assert np.array_equal(c[:, 0], b[:, 0]) and np.array_equal(c[:, 1:3], a[:, 1:3])
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------- 3. exact capacities

@pytest.fixture(scope="module")
def cap_scene(tiles):
    gt, prop, pn, pd, r = tile_pairs(*tiles[0])
    ref, stats = oracle_rows(gt, prop, pn, pd, r, TM.INTERVAL, TM.MATCHING_THRESHOLD)
    need = {"max_marbles": [max(s["marbles"]) for s in stats], "max_queue": [max(s["queue"]) for s in stats],
            "max_covered": [max(s["covered"]) for s in stats], "max_candidates": [max(s["candidates"]) for s in stats]}
    return gt, prop, pn, pd, r, ref, stats, need


@pytest.mark.parametrize("later_chunk", [False, True])
@pytest.mark.parametrize("kind", list(KINDS))
def test_capacity_exactly_at_the_need(cap_scene, kind, later_chunk):
    gt, prop, pn, pd, r, ref, stats, need = cap_scene
    need = np.array(need[kind])
    caps = {}
    order = np.arange(len(need))
    if later_chunk:                      # the pairs that need the most go last, beyond the first chunks of 7 slots
        order = np.argsort(need, kind="stable")
        caps["slots"] = 7
    pn, pd, ref, need = pn[order], pd[order], ref[order], need[order]
    top = int(need.max())
    first = int(np.argmax(need == top))
    assert top >= 4 and first >= 7 * later_chunk
    if kind == "max_queue":              # the ring wraps: more entries pass through it than it holds
        assert max(max(s["pushes"]) for s in stats) > top
    d = TM.TopoDevice(0, **caps, **{kind: top})
    try:
        for g, p in ((gt, 0), (prop, 1)):
            d.upload(p, g)
        assert np.array_equal(d.run(pn, pd, r, TM.INTERVAL, TM.MATCHING_THRESHOLD), ref)
    finally:
        d.close()
    d = TM.TopoDevice(0, **caps, **{kind: top - 1})
    try:
        for g, p in ((gt, 0), (prop, 1)):
            d.upload(p, g)
        with pytest.raises(RuntimeError, match=rf"pair {first}: .*{KINDS[kind]}"):
            d.run(pn, pd, r, TM.INTERVAL, TM.MATCHING_THRESHOLD)
        both(d, TINY_GT, TINY_PROP)
    finally:
        d.close()


def test_twin_needs_two_free_marble_slots():
    # a two-way path: every bidirectional hole is placed with its twin, so the walk ends on a twin pair
    g = meridian(12)
    h = D / 2
    pn, pd, args = [[5, 6, 5, 6]], [[h, h, h, h]], (4 * D, D / 4, D / 4)
    ref, stats = oracle_rows(g, g, pn, pd, *args)
    nm, nh, nhb = ref[0, :3]
    assert nhb == 2 * nh == 2 * nm and stats[0]["marbles"] == [nm, nh, nhb]
    for cap, ok in ((nhb, True), (nhb - 1, False)):      # two free slots before the last twin pair, then one
        d = TM.TopoDevice(0, max_marbles=int(cap))
        try:
            if ok:
                score(d, g, g, pn, pd, *args)
            else:
                with pytest.raises(RuntimeError, match="pair 0: .*marbles"):
                    score(d, g, g, pn, pd, *args)
                score(d, g, g, pn, pd, 2 * D, D / 4, D / 4)
        finally:
            d.close()


def test_covered_table_half_full():
    # the densest covered-edge table the layout allows: twice the need is a power of two, so the table is half full
    g = meridian(80)
    h = D / 2
    pn, pd = [[39, 40, 39, 40]], [[h, h, h, h]]
    for k in range(8, 70):
        ref, stats = oracle_rows(g, g, pn, pd, k * h, D / 2, D / 2)
        need = max(stats[0]["covered"])
        if need >= 32 and need & (need - 1) == 0:
            break
    else:
        pytest.fail("no r gives a power-of-two number of covered edges")
    d = TM.TopoDevice(0, max_covered=need)
    try:
        score(d, g, g, pn, pd, k * h, D / 2, D / 2)
    finally:
        d.close()
    d = TM.TopoDevice(0, max_covered=need - 1)
    try:
        with pytest.raises(RuntimeError, match="pair 0: .*covered"):
            score(d, g, g, pn, pd, k * h, D / 2, D / 2)
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------- 4. matchings

def scipy_matching(adj, left, n_right):
    rows = [(i, j) for i, a in enumerate(left) for j in adj.get(a, ())]
    if not rows:
        return 0
    m = csr_matrix((np.ones(len(rows), dtype=np.int8), tuple(zip(*rows))), shape=(len(left), n_right))
    return int((maximum_bipartite_matching(m, perm_type="column") >= 0).sum())


def greedy(adj, left):
    """The device's start: every left vertex in order takes its lowest free right vertex."""
    taken, free = set(), []
    for a in left:
        v = next((j for j in sorted(adj.get(a, ())) if j not in taken), None)
        if v is None:
            free.append(a)
        else:
            taken.add(v)
    return len(taken), free


def chain_scene(n_nodes=100):
    """A one-way proposal street walked from its south end and the same street one and a half samples further south
    as GT, walked from its north end, with a threshold of one sample spacing.  A walk samples every node but the far
    end, so marble i (i samples north of the proposal's first node) sees the holes half a spacing below and above
    it, and the top marble only the one below."""
    prop = meridian(n_nodes, two_way=False)
    gt = meridian(n_nodes, lat0=40.0 - 3 * D / 8, two_way=False)
    h, t = D / 2, n_nodes - 1
    return gt, prop, [[0, 1, t, t - 1]], [[h, h, h, h]], (n_nodes * D, D / 4, D / 4)


def test_chain_needs_one_augmenting_path_through_every_vertex(dev):
    gt, prop, pn, pd, args = chain_scene()
    got, _ = score(dev, gt, prop, pn, pd, *args)
    marbles = topo_oracle.topo_walk(prop, 0, 1, pd[0][0], pd[0][1], *args[:2])
    holes = topo_oracle.topo_walk(gt, pn[0][2], pn[0][3], pd[0][2], pd[0][3], *args[:2], bidirection=True)
    adj = topo_oracle.candidate_graph(marbles, holes, True, args[2])
    n = len(marbles)
    assert n == len(holes) == 4 * 99 and got[0, 0] == n
    # a chain, in half samples north of the proposal's first node: marbles at 0, 2, ..., holes at -1, 1, ...
    mpos = {m: round((m[0] - 40.0) / (D / 8)) for m in marbles}
    hpos = [round((x[0] - 40.0) / (D / 8)) for x in holes]
    assert sorted(mpos.values()) == list(range(0, 2 * n, 2)) and sorted(hpos) == list(range(-1, 2 * n - 1, 2))
    for m, i in mpos.items():
        assert {hpos[j] for j in adj[m]} == {i - 1, i + 1} & set(hpos)
    # the greedy start takes the upper hole for every marble and strands the top one; the only free hole is the
    # bottom one, so the one augmenting path alternates through every marble and every hole
    size, free = greedy(adj, marbles)
    assert size == n - 1 and [mpos[m] for m in free] == [2 * n - 2]
    assert scipy_matching(adj, marbles, n) == n == got[0, 3]
    assert got[0, 4] == scipy_matching(topo_oracle.candidate_graph(
        topo_oracle.topo_walk(gt, pn[0][2], pn[0][3], pd[0][2], pd[0][3], *args[:2]), marbles, False, args[2]),
        topo_oracle.topo_walk(gt, pn[0][2], pn[0][3], pd[0][2], pd[0][3], *args[:2]), n)


def test_chain_with_the_match_workspace_exactly_full():
    gt, prop, pn, pd, args = chain_scene(60)
    ref, stats = oracle_rows(gt, prop, pn, pd, *args)
    n = int(ref[0, 0])
    assert stats[0]["marbles"] == [n, n, n]
    d = TM.TopoDevice(0, max_marbles=n)
    try:
        got, _ = score(d, gt, prop, pn, pd, *args)
    finally:
        d.close()
    assert got[0, 3] == n


def comb_scene(n_nodes=40, extra=12):
    """Two one-way proposal streets 2^-20 degree apart, joined at the south end, against one GT street that runs
    `extra` nodes further north: south of the proposal's end two marbles compete for every hole, north of it the
    holes have no marble."""
    e = 2.0 ** -20
    nodes = [(40.0 + k * D, -70.0) for k in range(n_nodes)] + [(40.0 + k * D, -70.0 + e) for k in range(n_nodes)]
    edges = [(k, k + 1) for k in range(n_nodes - 1)] + [(n_nodes + k, n_nodes + k + 1) for k in range(n_nodes - 1)]
    prop = make_graph(nodes, edges + [(0, n_nodes)])
    gt = meridian(n_nodes + extra, lat0=40.0 - D / 8, two_way=False)
    h, t = D / 2, n_nodes + extra - 1
    return gt, prop, [[0, 1, t, t - 1]], [[h, h, h, h]], ((n_nodes + extra) * D, D / 4, D / 4)


def test_comb_matching_smaller_than_both_sides(dev):
    gt, prop, pn, pd, args = comb_scene()
    got, _ = score(dev, gt, prop, pn, pd, *args)
    nm, nh, nhb, mp, mr = got[0, :5]
    marbles = topo_oracle.topo_walk(prop, 0, 1, pd[0][0], pd[0][1], *args[:2])
    holes = topo_oracle.topo_walk(gt, pn[0][2], pn[0][3], pd[0][2], pd[0][3], *args[:2])
    adj = topo_oracle.candidate_graph(marbles, holes, True, args[2])
    assert mp == scipy_matching(adj, marbles, len(holes)) and 0 < mp < min(nm, nhb)
    # many marbles that do see holes stay unmatched: their searches walk the alternating tree and fail
    assert sum(1 for m in greedy(adj, marbles)[1] if adj.get(m)) >= 100
    rec = topo_oracle.candidate_graph(holes, marbles, False, args[2])
    assert mr == scipy_matching(rec, holes, len(marbles)) and 0 < mr < min(nm, nh)


# ---------------------------------------------------------------------------------------------- 5. candidate test

def edge_graph(a, b):
    return make_graph([a, b], [(0, 1)])


def crossing(dev, gt_dir, prop_dir):
    """One GT edge and one proposal edge crossing at their midpoints, each walked over its whole length; returns
    the candidate edges of the precision graph."""
    c = (40.0, -70.0)
    gt = edge_graph((c[0] - gt_dir[0] / 2, c[1] - gt_dir[1] / 2), (c[0] + gt_dir[0] / 2, c[1] + gt_dir[1] / 2))
    prop = edge_graph((c[0] - prop_dir[0] / 2, c[1] - prop_dir[1] / 2),
                      (c[0] + prop_dir[0] / 2, c[1] + prop_dir[1] / 2))
    got, stats = score(dev, gt, prop, [[0, 1, 0, 1]], [[D, D, D, D]], 4 * D, D / 16, D / 8)
    assert got[0, 0] >= 16 and got[0, 1] >= 16
    return stats[0]["candidates"][0]


def test_equal_dlat_and_dlon_switch_the_angle_test_off(dev):
    # a GT segment with dlat == dlon is never tested for its angle: the crossing proposal segment matches it near
    # the crossing; one unit in dlon's 11th bit switches the test back on, and nothing matches
    assert crossing(dev, (D, D), (D, -D)) > 0
    assert crossing(dev, (D, D + D / 1024), (D, -D)) == 0
    assert crossing(dev, (D, D + D / 1024), (D, D + D / 512)) > 0     # nearly parallel: the angle test passes


def test_angle_boundary(dev):
    # the proposal street turns away from the GT meridian in steps of atan(1/64 / cos 40): the candidate edges stop
    # between the two slopes whose angle_d lie either side of 0.29
    def angle_d(k):
        n = topo_oracle._norm(D, k * D / 64)
        return 1.0 - abs(n[0])
    k = next(k for k in range(1, 200) if angle_d(k + 1) >= 0.29)
    assert angle_d(k) < 0.29 <= angle_d(k + 1)
    assert crossing(dev, (D, 0.0), (D, k * D / 64)) > 0
    assert crossing(dev, (D, 0.0), (D, (k + 1) * D / 64)) == 0


@pytest.mark.parametrize("shift,near_only", [(-1, True), (0, False), (1, True)])
def test_distance_boundary(dev, shift, near_only):
    # holes half a sample spacing from the marbles, moved by 2^-30 degree either way; the threshold is exactly half
    # a spacing and the test is a strict `<`: on the boundary nothing matches, off it each marble has the nearer hole
    prop = meridian(6, two_way=False)
    gt = meridian(6, lat0=40.0 + D / 8 + shift * 2.0 ** -30, two_way=False)
    h = D / 2
    got, stats = score(dev, gt, prop, [[2, 3, 2, 3]], [[h, h, h, h]], 2 * D, D / 4, D / 8)
    marbles = topo_oracle.topo_walk(prop, 2, 3, h, h, 2 * D, D / 4)
    holes = topo_oracle.topo_walk(gt, 2, 3, h, h, 2 * D, D / 4)
    near = sorted(min(abs(m[0] - x[0]) for x in holes) for m in marbles)
    assert (near[0] < D / 8) == (shift != 0) and (near[0] == D / 8) == (shift == 0)
    cand = stats[0]["candidates"][0]
    assert got[0, 0] == got[0, 1] >= 12 and (cand >= got[0, 0] if near_only else cand == 0)


def test_box_boundary(dev):
    # at 64 degrees north a degree of longitude is short enough for the box (1.8 threshold + 0.00001) to decide
    # before the distance does.  The marble at the proposal's node and the hole at the GT's node are the only close
    # pair; the hole's box touches the marble's query box exactly, then misses it by one ulp
    thr, lat, lon = 1e-4, 64.0, -70.0
    edge = lon + thr * 1.8                                  # the query box's east side, as the kernel rounds it
    x = edge + 0.00001
    while x - 0.00001 > edge:
        x = math.nextafter(x, -math.inf)
    while math.nextafter(x, math.inf) - 0.00001 <= edge:
        x = math.nextafter(x, math.inf)
    prop = edge_graph((lat, lon - D), (lat, lon))           # nid2 = node 1 is the marble at `lon`
    counts = []
    for hole_lon in (x, math.nextafter(x, math.inf)):
        gt = edge_graph((lat, hole_lon + D), (lat, hole_lon))
        got, stats = score(dev, gt, prop, [[0, 1, 0, 1]], [[D, 0.0, D, 0.0]], 3e-4, 1e-4, thr)
        assert topo_oracle._dist((lat, lon), (lat, hole_lon)) < thr
        counts.append(stats[0]["candidates"][0])
    assert counts == [1, 0]


# ---------------------------------------------------------------------------------------------- 6. walks

def awkward_graphs():
    base = (40.0, -70.0)

    def at(i, j):
        return (base[0] + i * D, base[1] + j * D)

    def two_way(pairs):
        return [e for a, b in pairs for e in ((a, b), (b, a))]

    out = {}
    # a triangle on the pair's edge 0-1 with a tail: with node 0 far from the start and node 1 at it, node 2 is
    # reached from node 0 first and again, nearer, from node 1
    out["triangle"] = make_graph([at(0, 0), at(1, 0), at(1, 1), at(2, 1), at(3, 1)],
                                 two_way([(0, 1), (0, 2), (1, 2), (2, 3), (3, 4)]))
    # node 2 is listed twice in node 1's link list and once more in its reverse list
    out["repeated"] = make_graph([at(0, 0), at(1, 0), at(2, 0), at(3, 0)],
                                 [(0, 1), (1, 0), (1, 2), (1, 2), (2, 1), (2, 3), (3, 2)])
    star = [at(1, 0)] + [at(1 + i, j) for i, j in ((1, 0), (1, 1), (0, 1), (-1, 1), (-1, 0), (-1, -1), (0, -1),
                                                    (1, -1))]
    out["star"] = make_graph(star + [at(-2, 0)], two_way([(0, k) for k in range(1, 9)] + [(5, 9)]))
    # a ring: the two fronts leave the pair's edge 0-1 in opposite directions and meet on the far side
    ring = [at(0, 0), at(1, 0), at(2, 1), at(2, 2), at(1, 3), at(0, 3), at(-1, 2), at(-1, 1)]
    out["ring"] = make_graph(ring, two_way([(k, (k + 1) % 8) for k in range(8)]))
    out["one_way_dead_end"] = make_graph([at(k, 0) for k in range(5)], [(0, 1), (1, 0), (1, 2), (2, 3), (3, 4)])
    # a short cycle 1-2-3-0 that leads back to the pair's own edge 0-1
    out["short_cycle"] = make_graph([at(0, 0), at(1, 0), at(1, 1), at(0, 1), at(2, 0)],
                                    two_way([(0, 1), (1, 2), (2, 3), (3, 0), (1, 4)]))
    return out


@pytest.mark.parametrize("name", list(awkward_graphs()))
def test_walks_on_awkward_graphs(dev, name):
    g = awkward_graphs()[name]
    h = D / 2
    pn = [[0, 1, 0, 1], [1, 0, 0, 1], [0, 1, 1, 0], [0, 1, 0, 1]]
    pd = [[h, h, h, h], [h / 2, 3 * h / 2, h, h], [h, h, 0.0, D], [3 * D, 0.0, 2 * D, h]]
    seen = set()
    for k in range(1, 15):
        got, stats = score(dev, g, g, pn, pd, k / 2048.0, D / 4, D / 4)
        seen.add(tuple(got[:, :3].ravel()))
    assert len(seen) >= 4                       # the walks do grow with r
    # a neighbour expanded twice would change no count here, only queue an entry too many: the queue holds the
    # oracle's high-water mark exactly
    d = TM.TopoDevice(0, max_queue=max(max(s["queue"]) for s in stats))
    try:
        score(d, g, g, pn, pd, 14 / 2048.0, D / 4, D / 4)
    finally:
        d.close()


def test_triangle_relaxes_a_node_twice():
    # what the triangle is for, on the oracle's own walk: node 2 is expanded at two distances within the sweep
    g = awkward_graphs()["triangle"]
    stats = {}
    topo_oracle.topo_walk(g, 0, 1, 3 * D, 0.0, 14 / 2048.0, D / 4, stats=stats)
    assert stats["lowered"] >= 1


def test_city_tile(dev, city):
    gt_adj, prop_adj, det = city
    gt, prop, pn, pd, r = tile_pairs(gt_adj, prop_adj)
    counts = np.asarray(det.counts)
    slots = TM.DEFAULT_CAPS["slots"]
    n = counts.shape[0]
    assert n == pn.shape[0] > 3 * slots and r == det.r and (counts[:, 5] == 0).all()
    again = TM.topo_tile(gt_adj, prop_adj, TM.TopoState(), "cityscale", device=dev)[2]
    assert np.array_equal(again.counts, counts) and again.lines == det.lines
    d = TM.TopoDevice(0, slots=97)
    try:
        assert np.array_equal(TM.topo_tile(gt_adj, prop_adj, TM.TopoState(), "cityscale", device=d)[2].counts, counts)
    finally:
        d.close()
    # the oracle on a fixed sample: the largest walks, pairs whose matching leaves marbles or holes over, and the
    # first, a middle and the last pair of every chunk
    short = np.nonzero((counts[:, 3] < counts[:, 0]) | (counts[:, 4] < counts[:, 1]))[0]
    sample = set(np.argsort(-counts[:, 0], kind="stable")[:4].tolist()) | set(short[:: max(1, len(short) // 6)][:6].tolist())
    for ch in range((n + slots - 1) // slots):
        lo, hi = ch * slots, min(n, (ch + 1) * slots) - 1
        sample |= {lo, (lo + hi) // 2, hi}
    sample = sorted(sample)
    assert len(short) > 0 and 16 <= len(sample) <= 26
    ref, _ = oracle_rows(gt, prop, pn[sample], pd[sample], r, TM.INTERVAL, TM.MATCHING_THRESHOLD)
    assert np.array_equal(counts[sample], ref)


# ---------------------------------------------------------------------------------------------- 7. refusals

def upload_raw(dev, which, ll, ls, li, rs, ri):
    ll = np.array(ll, dtype=np.float64)
    cl = np.cos(np.radians(ll[:, 0]))
    a = [np.array(v, dtype=np.int32) for v in (ls, li, rs, ri)]
    rc = _lib.load().samroad_topo_upload_graph(dev._h, which, len(ll), ll.ctypes.data, cl.ctypes.data,
                                               *[v.ctypes.data for v in a])
    return rc, _lib.last_error()


def test_run_refuses_bad_arguments_and_recovers():
    g = lat_path()
    h = D / 2
    good = ([[3, 4, 3, 4]], [[h, h, h, h]], 3 * h, D / 4, D / 4)
    d = TM.TopoDevice(0)
    try:
        with pytest.raises(RuntimeError, match="both graphs must be uploaded"):
            d.run(np.array(good[0], dtype=np.int32), np.array(good[1]), *good[2:])
        d.upload(0, g)
        with pytest.raises(RuntimeError, match="both graphs must be uploaded"):
            d.run(np.array(good[0], dtype=np.int32), np.array(good[1]), *good[2:])
        score(d, g, g, *good)
        n = len(g.nodes)
        for pn, pd, step, msg in (
                ([[3, 4, 3, 4], [3, n, 3, 4]], [[h] * 4] * 2, D / 4, f"pair 1 names node {n}, outside its graph"),
                ([[3, 4, -1, 4]], [[h] * 4], D / 4, "pair 0 names node -1, outside its graph"),
                ([[3, 4, 3, 4], [3, 4, 3, 4], [5, 5, 3, 4]], [[h] * 4] * 3, D / 4, "pair 2 names an edge from a node"),
                ([[3, 4, 4, 4]], [[h] * 4], D / 4, "pair 0 names an edge from a node"),
                ([[3, 4, 3, 4]], [[h, h, math.inf, h]], D / 4, "pair 0 has a distance that is not finite"),
                ([[3, 4, 3, 4]], [[math.nan, h, h, h]], D / 4, "pair 0 has a distance that is not finite"),
                ([[3, 4, 3, 4]], [[h] * 4], 0.0, "step positive"),
                ([[3, 4, 3, 4]], [[h] * 4], -D, "step positive"),
                ([[3, 4, 3, 4]], [[h] * 4], math.nan, "step positive")):
            with pytest.raises(RuntimeError, match=msg):
                d.run(np.array(pn, dtype=np.int32), np.array(pd, dtype=np.float64), 3 * h, step, D / 4)
            score(d, g, g, *good)
        # no pair: success, and neither the arguments nor the handle are touched
        lib = _lib.load()
        assert lib.samroad_topo_run(d._h, 0, None, None, 3 * h, D / 4, D / 4, TM.COS40, None) == 0
        assert d.run(np.zeros((0, 4), dtype=np.int32), np.zeros((0, 4)), 3 * h, D / 4, D / 4).shape == (0, 6)
        score(d, g, g, *good)
    finally:
        d.close()


def test_upload_refuses_bad_adjacency_and_recovers():
    g = lat_path()
    h = D / 2
    good = ([[3, 4, 3, 4]], [[h, h, h, h]], 3 * h, D / 4, D / 4)
    ll = [[40.0, -70.0], [40.0 + D, -70.0], [40.0 + 2 * D, -70.0]]
    d = TM.TopoDevice(0)
    try:
        score(d, g, g, *good)
        for ls, li, rs, ri, msg in (
                ([0, 2, 1, 2], [1, 2], [0, 0, 1, 2], [0, 0], "adjacency offsets decrease at 1"),
                ([0, 1, 2, 2], [1, 2], [0, 0, 2, 1], [0, 1], "adjacency offsets decrease at 2"),
                ([1, 1, 2, 2], [1, 2], [0, 0, 1, 2], [0, 1], "adjacency offsets must start at 0"),
                ([0, 1, 2, 2], [1, 3], [0, 0, 1, 2], [0, 1], "neighbour 3 out of range"),
                ([0, 1, 2, 2], [1, 2], [0, 0, 1, 2], [0, -1], "neighbour -1 out of range")):
            rc, err = upload_raw(d, 1, ll, ls, li, rs, ri)
            assert rc != 0 and msg in err
            # the refused upload left the proposal that was there in place
            got = d.run(np.array(good[0], dtype=np.int32), np.array(good[1]), *good[2:])
            assert np.array_equal(got, oracle_rows(g, g, *good)[0])
        rc, err = upload_raw(d, 2, ll, [0, 1, 2, 2], [1, 2], [0, 0, 1, 2], [0, 1])
        assert rc != 0 and "which must be 0" in err
        score(d, g, g, *good)
    finally:
        d.close()
