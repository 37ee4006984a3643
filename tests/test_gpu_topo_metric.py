"""TOPO metric on the device (csrc/topo_metric.cu): the per-pair walks, candidate edges and maximum matchings equal
the unmodified reference (tests/golden/topo_synth.npz) bit for bit, and the oracle on edge cases; capacity limits
and zero-length edges are refused without spoiling the handle; two runs are bitwise equal."""
import json
import pickle

import numpy as np
import pytest

from oracle import topo_oracle
from sam_road_b200 import topo_metric as TM
from test_topo_host import GOLDEN, check_tile, dataset_tiles, load_tiles

pytestmark = pytest.mark.gpu

TINY_GT = {(100.0, 100.0): [(100.0, 160.0)], (100.0, 160.0): [(100.0, 100.0)]}
TINY_PROP = {(102.0, 100.0): [(102.0, 160.0)], (102.0, 160.0): [(102.0, 100.0)]}


@pytest.fixture(scope="module")
def dev():
    d = TM.TopoDevice(0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return z, load_tiles(z)


def both(dev, gt, prop, dataset="cityscale", state=None, state2=None):
    a = TM.topo_tile(gt, prop, state, dataset, device=dev)
    b = TM.topo_tile(gt, prop, state2, dataset, scorer=topo_oracle.scorer)
    assert np.array_equal(a[2].counts, b[2].counts)
    assert a[2].lines == b[2].lines
    assert a[2].kept == b[2].kept
    assert a[:2] == b[:2]
    return a


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_device_equals_reference(dev, golden, dataset):
    z, tiles = golden
    state = TM.TopoState()
    for t, (gt, prop) in enumerate(dataset_tiles(z, dataset)):
        p, rr, d = TM.topo_tile(gt, prop, state, dataset, device=dev)
        check_tile(z, dataset, t, p, rr, d)
        assert (np.asarray(d.counts)[:, 5] == 0).all()


def test_cli_writes_reference_files(golden, tmp_path):
    z, tiles = golden
    save, root = tmp_path / "save", tmp_path / "spacenet"
    (save / "graph").mkdir(parents=True)
    (root / "RGB_1.0_meter").mkdir(parents=True)
    tiles = dataset_tiles(z, "spacenet")
    names = [f"t{t}" for t in range(len(tiles))]
    (root / "data_split.json").write_text(json.dumps({"test": names}))
    for n, (gt, prop) in zip(names, tiles):
        pickle.dump(gt, open(root / "RGB_1.0_meter" / f"{n}__gt_graph.p", "wb"))
        pickle.dump(prop, open(save / "graph" / f"{n}.p", "wb"))
    TM.main(["--savedir", str(save), "--dataset", "spacenet", "--gt-root", str(root)])
    for t, n in enumerate(names):
        assert (save / "results" / "topo" / f"{n}.txt").read_text() == str(z[f"spacenet/tile{t}/text"])
        starts, kept, region = pickle.load(open(save / "results" / "topo" / f"{n}.topo.p", "rb"))
        assert np.array(kept, dtype=np.float64).reshape(-1, 8).tobytes() == z[f"spacenet/tile{t}/kept"].tobytes()
    got = json.loads((save / "topo.json").read_text())
    ref = json.loads(str(z["spacenet/topo_json"]))
    # the means follow the directory's listing order (byte-identical output under a pinned order: test_topo_host)
    assert sorted(got["prec"]) == sorted(ref["prec"]) and sorted(got["recall"]) == sorted(ref["recall"])
    assert np.allclose(got["mean topo"], ref["mean topo"], rtol=1e-15, atol=0)


def test_empty_proposal(dev, golden):
    _, tiles = golden
    p, rr, d = both(dev, tiles[0][0], {})
    assert (p, rr) == (0.0, 0.0) and d.lines[-1] == "precision=0 overall-recall=0.0"


def test_proposal_equals_gt_and_equal_precisions(dev, golden):
    _, tiles = golden
    p, rr, d = both(dev, tiles[0][0], tiles[0][0])
    precs = [x[2] for x in d.results]
    assert len(set(precs)) < len(precs)       # TOPO121 sorts equal precisions: the stable order decides the keep


def test_single_edge(dev):
    p, rr, d = both(dev, TINY_GT, TINY_PROP)
    # both dead ends start a chain over the one edge: two starting points at the same place, as in the reference
    assert len(d.results) == 2 and p > 0


def test_spacenet_fixed_r_and_carry_over(dev, golden):
    _, tiles = golden
    s1, s2 = TM.TopoState(), TM.TopoState()
    for t in (1, 2):
        d = both(dev, *tiles[t], dataset="spacenet", state=s1, state2=s2)[2]
        assert d.r == 0.0015
    s1, s2 = TM.TopoState(), TM.TopoState()
    rs = [both(dev, *tiles[t], state=s1, state2=s2)[2].r for t in (2, 1, 2)]
    assert rs == [0.0015, 0.003, 0.003]


@pytest.mark.parametrize("cap", [dict(max_marbles=40), dict(max_queue=2), dict(max_covered=1),
                                 dict(max_candidates=200)])
def test_capacity_refused_then_handle_works(golden, cap):
    _, tiles = golden
    what = {"max_marbles": "marbles", "max_queue": "queued", "max_covered": "covered",
            "max_candidates": "candidate"}[next(iter(cap))]
    d = TM.TopoDevice(0, **cap)
    try:
        with pytest.raises(RuntimeError, match=what):
            TM.topo_tile(*tiles[0], device=d)
        both(d, TINY_GT, TINY_PROP)
    finally:
        d.close()


def test_zero_length_edge_refused_by_device(dev):
    from sam_road_b200 import _lib
    lib = _lib.load()
    ll = np.array([[41.0, -71.0], [41.0, -71.0]], dtype=np.float64)
    cl = np.cos(np.radians(ll[:, 0]))
    ls, li = np.array([0, 1, 1], dtype=np.int32), np.array([1], dtype=np.int32)
    rs, ri = np.array([0, 0, 1], dtype=np.int32), np.array([0], dtype=np.int32)
    rc = lib.samroad_topo_upload_graph(dev._h, 0, 2, ll.ctypes.data, cl.ctypes.data, ls.ctypes.data,
                                       li.ctypes.data, rs.ctypes.data, ri.ctypes.data)
    assert rc != 0 and "edge 0 -> 1 has length zero" in _lib.last_error()
    both(dev, TINY_GT, TINY_PROP)


def test_two_runs_bitwise_equal(dev, golden):
    _, tiles = golden
    a = TM.topo_tile(*tiles[1], device=dev)[2]
    b = TM.topo_tile(*tiles[1], device=dev)[2]
    assert np.array_equal(a.counts, b.counts) and a.lines == b.lines


def lat_path(n=9):
    """A two-way path along a meridian with nodes 1/1024 degree apart, and a side street at node 4: every length on
    the path, every distance sum and every sample position is exact in float64."""
    g = TM.RoadGraph()
    g.nodes = [[40.0 + k / 1024.0, -70.0] for k in range(n)] + [[40.0 + 4 / 1024.0, -70.0 + 1 / 1024.0]]
    pairs = [(k, k + 1) for k in range(n - 1)] + [(4, n)]
    g.edges = [e for a, b in pairs for e in ((a, b), (b, a))]
    g.link = [[] for _ in g.nodes]
    g.rlink = [[] for _ in g.nodes]
    for a, b in g.edges:
        g.link[a].append(b)
        g.rlink[b].append(a)
    return g


def run_pairs(dev, g, pn, pd, r, step, threshold):
    dev.upload(0, g)
    dev.upload(1, g)
    got = dev.run(np.array(pn, dtype=np.int32), np.array(pd, dtype=np.float64), r, step, threshold)
    ref = np.array([topo_oracle.pair_counts(g, g, n, d, r, step, threshold) for n, d in zip(pn, pd)],
                   dtype=np.int32)
    assert np.array_equal(got, ref), (got, ref)
    return got


@pytest.mark.parametrize("k", range(2, 10))
def test_walk_exhausts_r_exactly_at_a_node(dev, k):
    # the walks start mid-edge 3-4 at 1/2048 from both ends; r = k/2048 reaches a node exactly for odd k (the
    # `dist > r` and `old + l < r` boundaries) and a sample exactly for every k (step 1/4096); the threshold equals
    # the sample spacing, so neighbouring samples sit exactly on `ddd < threshold`
    g = lat_path()
    h = 1 / 2048.0
    got = run_pairs(dev, g, [[3, 4, 3, 4], [4, 3, 3, 4], [2, 3, 3, 4]], [[h, h, h, h], [h, h, h, h], [h, 3 * h, h, h]],
                    k / 2048.0, 1 / 4096.0, 1 / 4096.0)
    assert (got[:, :3] > 0).all()


def test_pair_with_zero_holes(dev):
    # start distances beyond r place nothing on the first segment and expand no node: zero holes (and, in the
    # second pair, zero marbles as well)
    g = lat_path()
    h = 1 / 2048.0
    got = run_pairs(dev, g, [[3, 4, 3, 4], [3, 4, 5, 6]], [[h, h, 1.0, 1.0], [1.0, 1.0, 1.0, 1.0]],
                    0.0015, 0.00005, 0.0001)
    assert got[0, 0] > 0 and (got[0, 1:] == 0).all() and (got[1] == 0).all()
