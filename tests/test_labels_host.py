"""CPU: the per-scene precompute of sam_road_b200.dataset and the numpy sample_patch oracle
(oracle/label_oracle.py) against tests/golden/labels_synth.npz, which the unmodified reference's
GraphLabelGenerator made (tools/make_golden.py --labels; its contents are described in DESIGN.md §13 and in
labels_fixture's docstring); BFS against networkx; refusals without a GPU."""
import ctypes as C
import os

import networkx as nx
import numpy as np
import pytest

from oracle import label_oracle as LO
from sam_road_b200 import dataset as D
from sam_road_b200 import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "labels_synth.npz")
GOLDEN_EDGES = os.path.join(os.path.dirname(__file__), "golden", "labels_edges.npz")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def scene(fx):
    return D.precompute_scene(synth.make_road_graph(int(fx["extent"]), seed=0), D.cityscale_transform)


def _lc(fx):
    c = dict(zip([str(k) for k in fx["cfg_keys"]], fx["cfg"].tolist()))
    return dict(P=c["PATCH_SIZE"], S=c["TOPO_SAMPLE_NUM"], Np=c["MAX_NEIGHBOR_QUERIES"], r_nms=c["ROAD_NMS_RADIUS"],
                r_nbr=c["NEIGHBOR_RADIUS"])


def _patches(fx):
    for k, (x0, y0, rot) in enumerate(fx["patches"].tolist()):
        yield k, x0, y0, rot, {key.split("/", 1)[1]: v for key, v in fx.items() if key.startswith(f"p{k}/")}


def test_precompute_matches_reference(fx, scene):
    assert np.array_equal(scene.points, fx["subdivide_points"])          # ids and coordinates
    assert np.array_equal(np.unique(scene.crossovers, axis=0), np.unique(fx["crossovers"], axis=0))
    assert scene.crossovers.shape[0] == fx["crossovers"].shape[0] > 0
    assert np.array_equal(np.nonzero(scene.excluded)[0], fx["excluded"])
    assert np.array_equal(scene.nms_override, fx["nms_override"])
    assert np.array_equal(scene.weights, fx["sample_weights"])
    deg = np.diff(scene.adj_start)
    assert np.array_equal(deg != 2, scene.nms_override > 1) and (scene.flags[scene.excluded] & D.EXCLUDED).all()


def test_oracle_reproduces_reference_samples(fx, scene):
    lc = _lc(fx)
    seen_rot, seen_empty = set(), False
    for k, x0, y0, rot, rec in _patches(fx):
        draws = {} if "score" not in rec else dict(score=rec["score"], source_index=rec["source_index"],
                                                    noise=rec["noise"])
        o = LO.sample_patch(scene, x0, y0, rot, lc, draws, ties="scipy")
        if "candidates" in rec:
            assert np.array_equal(o["candidates"], rec["candidates"])
            assert np.array_equal(o["survivors"], rec["survivors"])
            assert np.array_equal(o["points"], rec["points"].astype(np.float32))
            seen_rot.add(rot)
        else:
            seen_empty = True
            assert np.array_equal(o["points"], np.zeros((1, 2), np.float32))
        for key in ("pairs", "connected", "valid"):
            assert np.array_equal(o[key], rec[key]), (k, key)
    assert seen_rot == {0, 1, 2, 3} and seen_empty


def test_index_ties_differ_only_among_equidistant_neighbours(fx, scene):
    lc = _lc(fx)
    for k, x0, y0, rot, rec in _patches(fx):
        if "candidates" not in rec:
            continue
        score_by_id = dict(zip(rec["candidates"].tolist(), rec["score"].tolist()))
        cand = LO.candidates(scene.points, scene.excluded, x0, y0, lc["P"], "index")
        assert sorted(cand.tolist()) == sorted(rec["candidates"].tolist())
        surv_ref = rec["survivors"]
        src_ids = surv_ref[rec["source_index"]]
        # the index-mode survivor order, then the same sources and per-survivor noise
        keep = LO.nms(scene.points[cand], np.maximum([score_by_id[c] for c in cand.tolist()],
                                                     scene.nms_override[cand]), lc["r_nms"], "index")
        surv = cand[keep]
        assert set(surv.tolist()) == set(surv_ref.tolist())
        at = {s: i for i, s in enumerate(surv.tolist())}
        noise_by_id = dict(zip(surv_ref.tolist(), rec["noise"]))
        draws = dict(score=np.array([score_by_id[c] for c in cand.tolist()]),
                     source_index=np.array([at[s] for s in src_ids.tolist()]),
                     noise=np.array([noise_by_id[s] for s in surv.tolist()]))
        o = LO.sample_patch(scene, x0, y0, rot, lc, draws, ties="index")
        assert np.array_equal(o["survivors"], surv)
        pts_ref = dict(zip(surv_ref.tolist(), rec["points"].astype(np.float32)))
        assert all(np.array_equal(p, pts_ref[s]) for s, p in zip(surv.tolist(), o["points"]))
        P = scene.points
        for s in range(lc["S"]):
            def targets(pairs, valid, conn, ids):
                t = ids[pairs[s, valid[s], 1]]
                return t, dict(zip(t.tolist(), conn[s, valid[s]].tolist()))
            t_ref, c_ref = targets(rec["pairs"], rec["valid"], rec["connected"], surv_ref)
            t_new, c_new = targets(o["pairs"], o["valid"], o["connected"], surv)
            assert len(t_ref) == len(t_new)
            src = P[src_ids[s]]
            d_ref = ((P[t_ref] - src) ** 2).sum(1)
            d_new = ((P[t_new] - src) ** 2).sum(1)
            assert np.array_equal(d_ref, d_new)      # same distances in the same order: only ties may swap
            last = d_ref.max() if len(d_ref) else 0.0
            inner_ref = set(t_ref[d_ref < last].tolist())
            assert inner_ref == set(t_new[d_new < last].tolist())
            for t in set(t_ref.tolist()) & set(t_new.tolist()):
                assert c_ref[t] == c_new[t]


def test_bfs_matches_networkx(fx, scene):
    g = nx.DiGraph()
    g.add_nodes_from(range(scene.points.shape[0]))
    lc = _lc(fx)
    depth = lc["r_nbr"] // 4
    rng = np.random.RandomState(0)
    for _ in range(60):
        src = int(rng.randint(scene.points.shape[0]))
        near = np.nonzero(((scene.points - scene.points[src]) ** 2).sum(1) < 64.0 ** 2)[0]
        stops = set(rng.choice(near, size=min(len(near), int(rng.randint(0, 8))), replace=False).tolist()) - {src}
        # a stop node is entered but never left: drop its outgoing arcs
        dg = nx.DiGraph()
        dg.add_nodes_from(range(scene.points.shape[0]))
        dg.add_edges_from((int(a), int(b)) for a, b in scene.edges if a not in stops)
        dg.add_edges_from((int(b), int(a)) for a, b in scene.edges if b not in stops)
        want = set(nx.single_source_shortest_path_length(dg, src, cutoff=depth))
        assert LO.bfs_reached(scene.adj_start, scene.adj, src, stops, depth) == want


def test_segment_crossings_rules():
    p = lambda *v: np.array([v], dtype=np.float64)  # noqa: E731
    hit, pt = D.segment_crossings(p(0, 0), p(4, 4), p(0, 4), p(4, 0))
    assert hit[0] and np.array_equal(pt[0], [2, 2])
    for seg in ((p(2, 2), p(6, 2)), (p(0, 4), p(2, 2)), (p(1, 1), p(3, 3)), (p(0, 1), p(4, 5))):
        assert not D.segment_crossings(p(0, 0), p(4, 4), *seg)[0][0]    # touching, endpoint, collinear, parallel


def test_max_window_points_is_exact():
    rng = np.random.RandomState(1)
    pts = rng.randint(0, 60, (200, 2)).astype(np.float64) + rng.rand(200, 2) * (rng.rand(200, 1) < 0.5)
    keep = rng.rand(200) < 0.8
    got = D.max_window_points(pts, keep, 3, 40, 16)
    want = max(int((keep & (pts[:, 0] >= x) & (pts[:, 0] <= x + 16) & (pts[:, 1] >= y) & (pts[:, 1] <= y + 16)).sum())
               for x in range(3, 41) for y in range(3, 41))
    assert got == want


@pytest.mark.parametrize("key,value", [("MAX_NEIGHBOR_QUERIES", 0), ("MAX_NEIGHBOR_QUERIES", 33),
                                       ("TOPO_SAMPLE_NUM", 0), ("ROAD_NMS_RADIUS", -1.0),
                                       ("NEIGHBOR_RADIUS", float("nan")), ("NEIGHBOR_RADIUS", 2.0 ** 33),
                                       ("PATCH_SIZE", 4096),
                                       ("PATCH_SIZE", 2.5)])
def test_bad_config_is_refused(key, value):
    cfg = dict(PATCH_SIZE=512, TOPO_SAMPLE_NUM=512, MAX_NEIGHBOR_QUERIES=16, ROAD_NMS_RADIUS=16, NEIGHBOR_RADIUS=64)
    cfg[key] = value
    with pytest.raises(ValueError, match=key):
        D.label_config(cfg, 2048, 64)


def test_bad_dataset_and_loader_arguments_are_refused():
    with pytest.raises(ValueError, match="DATASET"):
        D.SatMapDataset(dict(DATASET="mapillary", PATCH_SIZE=256), is_train=True)
    with pytest.raises(ValueError, match="batch_size"):
        D.BatchLoader(None, 0)
    ds = D.SatMapDataset.__new__(D.SatMapDataset)
    with pytest.raises(RuntimeError, match="loader"):
        ds[0]
    with pytest.raises(TypeError, match="pickle"):
        ds.__getstate__()


def test_c_abi_refuses_bad_label_config_before_any_device_call():
    from sam_road_b200 import _lib
    lib = _lib.load()
    good = dict(patch_size=512, image_size=2048, sample_margin=64, topo_sample_num=512, max_neighbor_queries=16,
                max_patch_points=100, road_nms_radius=16.0, neighbor_radius=64.0)
    for key, value, msg in (("max_neighbor_queries", 33, "MAX_NEIGHBOR_QUERIES"),
                            ("patch_size", 2000, "does not fit"), ("road_nms_radius", 0.0, "ROAD_NMS_RADIUS"),
                            ("max_patch_points", 0, "max_patch_points"), ("topo_sample_num", 0, "TOPO_SAMPLE_NUM"),
                            ("neighbor_radius", 2.0 ** 33, "BFS depth")):
        cfg = _lib.SamRoadLabelCfg(**dict(good, **{key: value}))
        h = C.c_void_p()
        assert lib.samroad_labels_create(0, C.byref(cfg), C.byref(h)) == 2
        assert msg in _lib.last_error() and not h.value
    assert lib.samroad_labels_batch(None, 1, 0, None, *([None] * 7), None, None) != 0
    assert "null labels object" in _lib.last_error()


def test_oracle_reproduces_reference_at_edge_settings(scene):
    """labels_edges.npz (tools/make_golden.py --labels-edges): the unmodified reference at NMS / neighbour radii
    10 / 30 (depth 7) with Np 4 and S 5, at NEIGHBOR_RADIUS 3 (depth 3 // 4 = 0) with S 3, and one PATCH_SIZE 1024
    window.  The oracle's depth rule (r // 4 on a float) and its inclusive NMS / exclusive kNN radius tests must
    reproduce scipy's samples there, not only at 16 / 64."""
    fx = dict(np.load(GOLDEN_EDGES))
    assert int(fx["extent"]) == 360
    seen = set()
    for g in (str(v) for v in fx["groups"]):
        c = dict(zip([str(k) for k in fx[f"{g}/cfg_keys"]], fx[f"{g}/cfg"].tolist()))
        lc = dict(P=int(c["PATCH_SIZE"]), S=int(c["TOPO_SAMPLE_NUM"]), Np=int(c["MAX_NEIGHBOR_QUERIES"]),
                  r_nms=c["ROAD_NMS_RADIUS"], r_nbr=c["NEIGHBOR_RADIUS"])
        for k, (x0, y0, rot) in enumerate(fx[f"{g}/patches"].tolist()):
            rec = {key.split("/", 2)[2]: v for key, v in fx.items() if key.startswith(f"{g}/p{k}/")}
            o = LO.sample_patch(scene, x0, y0, rot, lc, dict(score=rec["score"], source_index=rec["source_index"],
                                                             noise=rec["noise"]), ties="scipy")
            assert np.array_equal(o["candidates"], rec["candidates"]), (g, k)
            assert np.array_equal(o["survivors"], rec["survivors"]), (g, k)
            assert np.array_equal(o["points"], rec["points"].astype(np.float32)), (g, k)
            for key in ("pairs", "connected", "valid"):
                assert o[key].shape == (lc["S"], lc["Np"]) + (() if key != "pairs" else (2,))
                assert np.array_equal(o[key], rec[key]), (g, k, key)
            seen.add((g, int(rec["valid"].sum()) > 0, int(rec["connected"].sum()) > 0))
    # radii 10 / 30 and P 1024 have connected and unconnected targets; radius 3 has none in range
    assert {("r10_30", True, True), ("p1024", True, True), ("r3", False, False)} <= seen
    r = dict(zip([str(k) for k in fx["r10_30/cfg_keys"]], fx["r10_30/cfg"].tolist()))
    assert r["NEIGHBOR_RADIUS"] // 4 == 7 and r["ROAD_NMS_RADIUS"] == 10


# P with an inexact float32 np.linalg.inv of the reference's centring matrix (DESIGN.md §13): there the reference's
# point transform may differ from the device's float64 one by one float64 ulp before the float32 rounding
INEXACT_TRANSFORM_P = (1488, 1584, 1680, 1872)


def _transform_like_device(pts, x0, y0, P, rot, noise):
    c = 0.5 * P
    x, y = (pts[:, 0] - x0) - c, (pts[:, 1] - y0) - c
    for _ in range(rot):
        x, y = y, -x
    return np.stack([(x + c) + noise[:, 0], (y + c) + noise[:, 1]], 1)


def test_point_transform_is_exact_except_listed_patch_sizes():
    """The float64 transform of labels.cu (subtract, rotate, add) equals the reference's matrix product with the
    float32 inverse of the centring matrix for every multiple of 16 up to 1920 except INEXACT_TRANSFORM_P."""
    inexact = []
    rng = np.random.RandomState(3)
    for P in range(16, 1921, 16):
        t = np.array([[1, 0, -0.5 * P], [0, 1, -0.5 * P], [0, 0, 1]], dtype=np.float32)
        exact_inv = np.array([[1, 0, 0], [0, 1, 0], [0.5 * P, 0.5 * P, 1]], dtype=np.float32)
        if not np.array_equal(np.linalg.inv(t.T), exact_inv):
            inexact.append(P)
            continue
        x0, y0 = 64, 37
        pts = np.concatenate([rng.rand(64, 2) * P, rng.randint(0, P + 1, (16, 2))]) + [x0, y0]
        noise = rng.randn(pts.shape[0], 2)
        for rot in range(4):
            want = LO.transform_points(pts, x0, y0, P, rot, noise)
            assert np.array_equal(_transform_like_device(pts, x0, y0, P, rot, noise), want), (P, rot)
    assert tuple(inexact) == INEXACT_TRANSFORM_P
    assert not {256, 512, 1024} & set(inexact)
    P = INEXACT_TRANSFORM_P[0]   # the documented bound where the inverse is inexact: one float32 ulp
    pts = rng.rand(4096, 2) * P
    noise = rng.randn(4096, 2)
    for rot in range(4):
        a = _transform_like_device(pts, 0, 0, P, rot, noise).astype(np.float32)
        b = LO.transform_points(pts, 0, 0, P, rot, noise).astype(np.float32)
        assert (np.abs(a - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all(), rot
