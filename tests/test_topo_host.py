"""TOPO metric on the host: the restated graph construction, starting points, pairs, TOPO121 and lines, with the
oracle's per-pair counts, reproduce the unmodified reference (tests/golden/topo_synth.npz, tools/make_golden.py
--topo) bit for bit; the oracle's matching size equals networkx's.  No GPU needed."""
import json
import os
import random

import numpy as np
import pytest

from oracle import topo_oracle
from sam_road_b200 import topo_metric as TM

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "topo_synth.npz")


def load_tiles(z):
    tiles = []
    t = 0
    while f"tile{t}/gt_keys" in z:
        pair = []
        for name in ("gt", "prop"):
            keys, cnt, nb = z[f"tile{t}/{name}_keys"], z[f"tile{t}/{name}_cnt"], z[f"tile{t}/{name}_nbrs"]
            adj, o = {}, 0
            for k, c in zip(keys.tolist(), cnt.tolist()):
                adj[tuple(k)] = [tuple(v) for v in nb[o:o + c].tolist()]
                o += c
            pair.append(adj)
        tiles.append(tuple(pair))
        t += 1
    return tiles


def check_tile(z, dataset, t, p, rr, d):
    pre = f"{dataset}/tile{t}/"
    assert d.r == float(z[pre + "r"])
    assert np.array_equal(np.array(d.region), z[pre + "region"])
    assert np.array_equal(np.array(d.starts, dtype=np.float64).reshape(-1, 6), z[pre + "starts"])
    assert list(d.pairs) == z[pre + "pair_keys"].tolist()
    assert np.array_equal(np.array(list(d.pairs.values()), dtype=np.float64).reshape(-1, 7), z[pre + "pairs"])
    ref = z[pre + "counts"]
    mine = np.asarray(d.counts)[:, :5]
    defined = ref[:, 4] >= 0
    assert np.array_equal(mine[:, :4], ref[:, :4])
    assert np.array_equal(mine[defined, 4], ref[defined, 4])
    res = np.array(d.results, dtype=np.float64).reshape(-1, 8)
    assert res.tobytes() == z[pre + "results"].tobytes()
    assert np.array(d.kept, dtype=np.float64).reshape(-1, 8).tobytes() == z[pre + "kept"].tobytes()
    assert "".join(d.lines) == str(z[pre + "text"])
    assert (p, rr) == TM.parse_last_line(str(z[pre + "text"]).splitlines()[-1])


def dataset_tiles(z, dataset):
    """The tiles the dataset's driver ran, in order (spacenet's list adds one with no starting point)."""
    tiles = load_tiles(z)
    return [tiles[t] for t in range(len(tiles)) if f"{dataset}/tile{t}/r" in z]


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_oracle_reproduces_reference(dataset):
    z = np.load(GOLDEN)
    state = TM.TopoState()
    for t, (gt, prop) in enumerate(dataset_tiles(z, dataset)):
        p, rr, d = TM.topo_tile(gt, prop, state, dataset, scorer=topo_oracle.scorer)
        check_tile(z, dataset, t, p, rr, d)


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_fixture_exercises_topo121_and_the_zeros_line(dataset):
    z = np.load(GOLDEN)
    # tile 3: the reference's TOPO121 drops scored starting points (competitors below precision 0.9)
    kept, results = z[f"{dataset}/tile3/kept"], z[f"{dataset}/tile3/results"]
    assert 0 < len(kept) < len(results)
    assert (results[:, 2] < 0.9).any()
    if dataset == "spacenet":
        # tile 4: no starting point; spacenet's topo.py takes its except branch
        assert str(z["spacenet/tile4/text"]) == "0 0 0 0\n"
    else:
        assert "cityscale/tile4/r" not in z


def test_tile_order_carries_min_lat():
    z = np.load(GOLDEN)
    tiles = load_tiles(z)
    # tile 2 alone is scored at r = 0.0015; after tile 1 (x up to 1250 px) the cityscale driver uses 0.003
    assert TM.topo_tile(*tiles[2], TM.TopoState(), "cityscale", scorer=topo_oracle.scorer)[2].r == 0.0015
    assert float(z["cityscale/tile2/r"]) == 0.003 and float(z["spacenet/tile2/r"]) == 0.0015


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_aggregate_matches_reference_json(tmp_path, dataset, monkeypatch):
    z = np.load(GOLDEN)
    rdir = tmp_path / "results" / "topo"
    rdir.mkdir(parents=True)
    names = []
    for t in range(len(dataset_tiles(z, dataset))):
        (rdir / f"{t}.txt").write_text(str(z[f"{dataset}/tile{t}/text"]))
        names.append(f"{t}.txt")
    monkeypatch.setattr(TM.os, "listdir", lambda p: list(names))
    TM.aggregate(str(tmp_path), dataset)
    path = tmp_path / ("score/topo.json" if dataset == "cityscale" else "topo.json")
    assert path.read_text() == str(z[f"{dataset}/topo_json"])
    json.loads(path.read_text())


def test_cityscale_without_starting_points_raises():
    gt, prop = load_tiles(np.load(GOLDEN))[4]
    with pytest.raises(ZeroDivisionError):       # cityscale's topo.py divides by the start count (`rrr`)
        TM.topo_tile(gt, prop, TM.TopoState(), "cityscale", scorer=topo_oracle.scorer)
    p, rr, d = TM.topo_tile(gt, prop, TM.TopoState(), "spacenet", scorer=topo_oracle.scorer)
    assert (p, rr) == (0.0, 0.0) and d.lines == ["0 0 0 0\n"]


def test_zero_length_edge_is_refused():
    adj = {(10.0, 10.0): [(10.0, 10.0)]}
    with pytest.raises(ValueError, match=r"\(10.0, 10.0\) -> \(10.0, 10.0\) has length zero"):
        TM.create_graph(adj, TM.TopoState())


def test_matching_size_equals_networkx():
    nx = pytest.importorskip("networkx")
    rng = random.Random(3)
    for trial in range(200):
        nl, nr = rng.randint(0, 12), rng.randint(0, 12)
        p = rng.random()
        adj = {("m", i): {j for j in range(nr) if rng.random() < p} for i in range(nl)}
        adj = {k: v for k, v in adj.items() if v}
        g = nx.Graph()
        g.add_nodes_from([("L", k) for k in adj])
        for k, vs in adj.items():
            for v in vs:
                g.add_edge(("L", k), ("R", v))
        ref = len(nx.bipartite.hopcroft_karp_matching(g, top_nodes=[("L", k) for k in adj])) // 2
        assert topo_oracle.matching_size(adj) == ref, trial
