"""CPU: the OpenCV restatement of oracle/label_mask_oracle.py against live cv2 (exhaustive small sweeps, long
segments far outside the tile) and against tests/golden/label_masks.npz, which the reference scripts' own drawing
functions wrote (tools/make_golden.py --label-masks); sam_road_b200.label_masks.tile_arrays against networkx; the
argument refusals of samroad_label_masks, which come before any CUDA call."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import label_mask_oracle as LM
from sam_road_b200 import _lib, synth
from sam_road_b200 import label_masks as L

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "label_masks.npz")
GRID = [int(v) for v in np.linspace(-3, 26, 9).astype(int)]   # 9 positions across and around a 24-pixel image


def golden_tiles():
    """{name: (dataset, adjacency dict, keypoint mask, road mask)} of the golden file."""
    fx = np.load(GOLDEN)
    out = {}
    for name in sorted({k.split("/")[0] for k in fx.files if "/" in k}):
        dataset = str(fx[f"{name}/dataset"])
        size = L.IMAGE_SIZE[dataset]
        adj = {tuple(n): [] for n in fx[f"{name}/lonely"].tolist()}
        for r0, c0, r1, c1 in fx[f"{name}/pairs"].tolist():
            adj.setdefault((r0, c0), []).append((r1, c1))
        unpack = lambda k: np.unpackbits(fx[k])[:size * size].reshape(size, size) * np.uint8(255)  # noqa: E731
        out[name] = (dataset, adj, unpack(f"{name}/keypoint"), unpack(f"{name}/road"))
    return out


@pytest.mark.parametrize("width", range(2, 9))
def test_thick_lines_match_cv2_on_every_grid_segment(width):
    cv2 = pytest.importorskip("cv2")
    pts = [(x, y) for x in GRID for y in GRID]
    bad = []
    for p in pts:
        for q in pts:
            want = np.zeros((24, 24), np.uint8)
            cv2.line(want, p, q, 255, width)
            got = np.zeros((24, 24), np.uint8)
            LM.thick_line(got, p, q, width)
            if not np.array_equal(got, want):
                bad.append((p, q))
    assert not bad, f"{len(bad)} of {len(pts) ** 2} segments differ, e.g. {bad[:3]}"


def test_filled_discs_match_cv2_near_the_border():
    cv2 = pytest.importorskip("cv2")
    bad = []
    for r in range(11):
        for cx in range(-12, 36):
            for cy in (-12, -4, -1, 0, 1, 3, 11, 20, 22, 23, 24, 27, 35):
                for c in ((cx, cy), (cy, cx)):
                    want = np.zeros((24, 24), np.uint8)
                    cv2.circle(want, c, r, 255, -1)
                    got = np.zeros((24, 24), np.uint8)
                    LM.circle_fill(got, c[0], c[1], r)
                    if not np.array_equal(got, want):
                        bad.append((c, r))
    assert not bad, bad[:5]


def test_long_segments_far_outside_match_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    for k in range(40):
        p = tuple(int(v) for v in rng.integers(-100000, 100001, 2))
        q = tuple(int(v) for v in rng.integers(-300, 2400, 2))
        if k % 2:
            p, q = q, p
        width = int(rng.integers(2, 6))
        want = np.zeros((2048, 2048), np.uint8)
        cv2.line(want, p, q, 255, width)
        got = np.zeros((2048, 2048), np.uint8)
        LM.thick_line(got, p, q, width)
        assert np.array_equal(got, want), (p, q, width)


def test_oracle_matches_golden():
    fx = np.load(GOLDEN)
    assert str(fx["cv2_version"]) and str(fx["networkx_version"])
    tiles = golden_tiles()
    assert {"city_empty", "city_special", "space_special"} <= set(tiles)
    for name, (dataset, adj, kp, road) in tiles.items():
        okp, oroad = LM.tile_masks(adj, dataset, L.IMAGE_SIZE[dataset])
        assert np.array_equal(okp, kp) and np.array_equal(oroad, road), name


def test_tile_arrays_follow_networkx():
    nx = pytest.importorskip("networkx")
    tiles = golden_tiles()
    cases = [(dataset, adj) for dataset, adj, _, _ in tiles.values()]
    cases += [("cityscale", synth.city_tile(2048, seed=3)[1]), ("spacenet", synth.make_road_graph(400, seed=4))]
    for dataset, adj in cases:
        kp, edges = L.tile_arrays(adj, dataset)
        assert kp.dtype == np.int32 and edges.dtype == np.int32
        g = nx.Graph()
        for n, neis in adj.items():
            for nei in neis:
                g.add_edge(LM.node_key(n, dataset), LM.node_key(nei, dataset))
        assert sorted(tuple(p) for p in kp.tolist()) == sorted(n for n, d in g.degree() if d != 2)
        assert sorted((tuple(e[:2]), tuple(e[2:])) for e in edges.tolist()) == \
            sorted((min(u, v), max(u, v)) for u, v in g.edges())


def test_tile_arrays_graph_rules():
    adj = {(5.0, 5.0): [(5.0, 5.0), (9.0, 7.0)],       # self-loop + one edge: degree 3
           (20.0, 20.0): [(20.0, 20.0)],               # lone self-loop: degree 2, no keypoint
           (30.7, 1.2): [(40.0, 1.0)], (30.2, 1.9): [(35.0, 9.0)],   # merge into (1, 30): degree 2
           (50.0, 50.0): []}                            # no neighbours: no node
    kp, edges = L.tile_arrays(adj, "cityscale")
    assert kp.tolist() == [[1, 40], [5, 5], [7, 9], [9, 35]]
    assert [5, 5, 5, 5] in edges.tolist() and [20, 20, 20, 20] in edges.tolist() and len(edges) == 5
    kp, edges = L.tile_arrays({(0.5, 3.0): [(-2.0, 3.0)]}, "spacenet")
    assert edges.tolist() == [[3, 400, 3, 402]]
    assert L.tile_arrays({(1.0, 1.0): []}, "cityscale")[1].shape == (0, 4)
    with pytest.raises(ValueError, match="dataset"):
        L.tile_arrays({}, "deepglobe")


def test_missing_pickle_is_named(tmp_path):
    with pytest.raises(FileNotFoundError, match="region_0_refine_gt_graph.p"):
        L.write_dataset_masks("cityscale", str(tmp_path))
    assert not (tmp_path / "processed").exists()


@pytest.mark.parametrize("args,msg", [
    (dict(T=-1), "tile count"), (dict(size=0), "size"), (dict(road_width=1), "road_width"),
    (dict(road_width=32768), "road_width"), (dict(keypoint_radius=-1), "keypoint_radius"),
    (dict(keypoint_radius=40000), "keypoint_radius"), (dict(null=True), "null pointer")])
def test_argument_refusals(args, msg):
    lib = _lib.load()
    a = dict(T=2, size=16, keypoint_radius=3, road_width=3, null=False)
    a.update(args)
    buf = (C.c_int64 * 64)()
    p = None if a["null"] else C.addressof(buf)
    rc = lib.samroad_label_masks(a["T"], a["size"], C.addressof(buf), C.addressof(buf), C.addressof(buf),
                                 C.addressof(buf), a["keypoint_radius"], a["road_width"], C.addressof(buf), p, None)
    assert rc != 0 and msg in _lib.last_error() and "samroad_label_masks" in _lib.last_error()
