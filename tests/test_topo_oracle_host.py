"""The TOPO oracle itself (oracle/topo_oracle.py): its matching size against scipy's on graphs far larger than a
tile's, on paths thousands of vertices long and on the chain and comb scenes of the GPU tests; its walk and
candidate statistics against its own counts on the golden tiles; the boxed candidate search against the scalar
one.  No GPU needed."""
import random

import numpy as np
import pytest

from oracle import topo_oracle
from test_gpu_topo_limits import chain_scene, comb_scene, oracle_rows, scipy_matching, tile_pairs
from test_topo_host import GOLDEN, load_tiles
from sam_road_b200 import topo_metric as TM


@pytest.mark.parametrize("density", [0.002, 0.01, 0.05, 0.5])
def test_matching_size_equals_scipy(density):
    rng = random.Random(int(density * 1000))
    for nl, nr in ((600, 600), (600, 150), (97, 411), (1, 1), (0, 5)):
        left = [("m", i) for i in range(nl)]
        adj = {a: {j for j in range(nr) if rng.random() < density} for a in left}
        adj = {a: v for a, v in adj.items() if v}
        assert topo_oracle.matching_size(adj) == scipy_matching(adj, left, nr), (nl, nr)


def test_matching_size_on_a_path_of_ten_thousand_vertices():
    # left i sees right n - 2 - i, which it prefers, and right n - 1 - i, which the vertex before it took; the last
    # left vertex sees only a taken one, so its augmenting path runs back through all 5000 left vertices
    n = 5000
    left = list(range(n))
    adj = {i: {n - 1 - i, n - 2 - i} & set(range(n)) for i in left}
    assert topo_oracle.matching_size(adj) == n == scipy_matching(adj, left, n)
    adj[0] = {n - 2}                      # now the path's far end is gone: one vertex stays unmatched
    assert topo_oracle.matching_size(adj) == n - 1 == scipy_matching(adj, left, n)


@pytest.mark.parametrize("scene", [chain_scene, comb_scene])
def test_matching_size_on_the_chain_and_comb_scenes(scene):
    gt, prop, pn, pd, (r, step, thr) = scene()
    marbles = topo_oracle.topo_walk(prop, pn[0][0], pn[0][1], pd[0][0], pd[0][1], r, step)
    for bidirection in (True, False):
        holes = topo_oracle.topo_walk(gt, pn[0][2], pn[0][3], pd[0][2], pd[0][3], r, step, bidirection=bidirection)
        prec = topo_oracle.candidate_graph(marbles, holes, True, thr)
        rec = topo_oracle.candidate_graph(holes, marbles, False, thr)
        assert topo_oracle.matching_size(prec) == scipy_matching(prec, marbles, len(holes)) > 100
        assert topo_oracle.matching_size(rec) == scipy_matching(rec, holes, len(marbles)) > 100


@pytest.fixture(scope="module")
def golden_pairs():
    out = []
    for gt_adj, prop_adj in load_tiles(np.load(GOLDEN))[:4]:
        gt, prop, pn, pd, r = tile_pairs(gt_adj, prop_adj)
        out.append((gt, prop, pn, pd, r) + oracle_rows(gt, prop, pn, pd, r, TM.INTERVAL, TM.MATCHING_THRESHOLD))
    return out


def test_statistics_agree_with_the_counts(golden_pairs):
    total = 0
    for gt, prop, pn, pd, r, ref, stats in golden_pairs:
        for row, s in zip(ref.tolist(), stats):
            assert s["marbles"] == row[:3]
            for w, g in enumerate((prop, gt, gt)):
                assert 2 <= s["queue"][w] <= s["pushes"][w]
                assert s["covered"][w] <= len(g.edges) + sum(len(x) for x in g.rlink)
                assert s["lowered"][w] <= s["pushes"][w]
            assert s["covered"][1] == s["covered"][2] and s["queue"][1] == s["queue"][2]   # twins change no walk
            assert row[3] <= min(row[0], row[2], s["candidates"][0])
            assert row[4] <= min(row[1], row[0], s["candidates"][1])
            assert (row[3] == 0) == (s["candidates"][0] == 0) and (row[4] == 0) == (s["candidates"][1] == 0)
            total += 1
    assert total >= 90


def test_boxed_candidates_equal_the_scalar_search(golden_pairs):
    for gt, prop, pn, pd, r, ref, stats in golden_pairs:
        for n, d in zip(pn.tolist(), pd.tolist()):
            marbles = topo_oracle.topo_walk(prop, n[0], n[1], d[0], d[1], r, TM.INTERVAL)
            holes = topo_oracle.topo_walk(gt, n[2], n[3], d[2], d[3], r, TM.INTERVAL)
            holes_b = topo_oracle.topo_walk(gt, n[2], n[3], d[2], d[3], r, TM.INTERVAL, bidirection=True)
            for left, right, lm in ((marbles, holes_b, True), (holes, marbles, False)):
                assert topo_oracle.candidate_graph_boxed(left, right, lm, TM.MATCHING_THRESHOLD) == \
                    topo_oracle.candidate_graph(left, right, lm, TM.MATCHING_THRESHOLD)
