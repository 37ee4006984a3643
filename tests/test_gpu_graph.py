"""Bit-exact parity of the device-side graph stage (csrc/graph.cu behind sam_road_b200.graph.SceneGraph)
against the oracle's restatement of the reference host code:
    graph_extraction.extract_graph_points / graph_utils.nms_points   graph_extraction.py:130-139, graph_utils.py:572-591
    pair-query construction                                          inferencer.py:126-197
    edge aggregation                                                 inferencer.py:206-230
Integer / index work: the bar is identical arrays (same points in the same order, same pairs, same
valid mask, same edges in the same order), not a tolerance."""
import os
from collections import defaultdict

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200.graph import SceneGraph  # noqa: E402
from sam_road_b200.inferencer import batch_plan, get_patch_info_one_img  # noqa: E402

DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def gx():
    return SceneGraph(DEV)


def _extract(gx, kp, road, thr0, thr1, r0, r1, tie):
    out = gx.extract_graph_points(torch.as_tensor(kp).to(DEV), torch.as_tensor(road).to(DEV), thr0, thr1, r0, r1,
                                  tie_order=tie)
    return out.cpu().numpy()


@pytest.mark.parametrize("tie", ["numpy", "stable"])
def test_keypoints_golden_masks(gx, tie):
    """The mask pair of tests/golden/tileloop.npz (blobs and bars: thousands of equal scores)."""
    g = np.load(os.path.join(GOLD, "tileloop.npz"))
    mine = _extract(gx, g["kp_mask"], g["road_mask"], 0.3, 0.4, 8, 16, tie)
    ref = O.extract_graph_points(g["kp_mask"], g["road_mask"], 0.3, 0.4, 8, 16, tie)
    assert mine.dtype == np.int64 and np.array_equal(mine, ref)
    assert gx.stats["n_points"] == ref.shape[0] and gx.stats["nms_rounds"][2] >= 1


@pytest.mark.parametrize("tie", ["numpy", "stable"])
@pytest.mark.parametrize("shape,thr,radii", [
    ((400, 400), (0.97, 0.93), (8, 16)),        # spacenet-sized scene, noise masks
    ((300, 517), (0.95, 0.90), (3, 7)),         # non-square, odd width, small radii
    ((257, 129), (0.90, 0.80), (16, 40)),       # radius 40 > shared-memory halo: generic kernel
    ((128, 128), (0.5, 0.5), (8, 32)),          # dense candidates, halo 32 (largest tiled radius)
    ((256, 256), (0.7, 0.6), (8, 16)),          # > 16 384 candidates: the stable order's histogram spans scan tiles
    ((2048, 2052), (0.996, 0.99), (8, 16)),     # > 4096 x 1024 pixels: the compaction's chunk counts span scan tiles
])
def test_keypoints_noise_masks(gx, tie, shape, thr, radii):
    rng = np.random.RandomState(shape[0] + shape[1])
    kp = rng.randint(0, 256, size=shape).astype(np.uint8)
    road = rng.randint(0, 256, size=shape).astype(np.uint8)
    mine = _extract(gx, kp, road, thr[0], thr[1], radii[0], radii[1], tie)
    ref = O.extract_graph_points(kp, road, thr[0], thr[1], radii[0], radii[1], tie)
    assert ref.shape[0] > 5
    assert np.array_equal(mine, ref), (mine.shape, ref.shape)
    cand = gx.stats["candidates"]
    assert cand[0] == int((kp > thr[0] * 255).sum()) and cand[1] == int((road > thr[1] * 255).sum())


@pytest.mark.parametrize("tie", ["numpy", "stable"])
def test_keypoints_mortal_scores_and_edge_cases(gx, tie):
    """Thresholds below 1/255 admit score 1, which is not immune (graph_utils.py:573): passes 1 and 2
    then really suppress.  Also: empty masks, thresholds nothing passes (ITSC_THRESHOLD: 128 exists in
    the reference configs), one mask empty, fractional radius."""
    rng = np.random.RandomState(7)
    kp = rng.randint(0, 4, size=(90, 110)).astype(np.uint8)
    road = rng.randint(0, 3, size=(90, 110)).astype(np.uint8)
    t = 0.5 / 255
    assert np.array_equal(_extract(gx, kp, road, t, t, 2, 3, tie), O.extract_graph_points(kp, road, t, t, 2, 3, tie))
    assert gx.stats["nms_rounds"][0] >= 1 and gx.stats["nms_rounds"][1] >= 1
    assert np.array_equal(_extract(gx, kp, road, t, t, 2.5, 4.3, tie),
                          O.extract_graph_points(kp, road, t, t, 2.5, 4.3, tie))
    z = np.zeros((64, 80), np.uint8)
    assert _extract(gx, z, z, 0.3, 0.4, 8, 16, tie).shape == (0, 2)
    assert _extract(gx, kp, road, 128, 128, 8, 16, tie).shape == (0, 2)
    big = rng.randint(0, 256, size=(120, 120)).astype(np.uint8)
    assert np.array_equal(_extract(gx, z[:64, :64], big[:64, :64], 0.3, 0.9, 8, 16, tie),
                          O.extract_graph_points(z[:64, :64], big[:64, :64], 0.3, 0.9, 8, 16, tie))
    assert np.array_equal(_extract(gx, big[:64, :64], z[:64, :64], 0.9, 0.3, 8, 16, tie),
                          O.extract_graph_points(big[:64, :64], z[:64, :64], 0.9, 0.3, 8, 16, tie))
    # radius 0: only exact duplicates (a pixel above both thresholds) are merged
    assert np.array_equal(_extract(gx, big, big, 0.9, 0.8, 0, 0, tie), O.extract_graph_points(big, big, 0.9, 0.8, 0, 0, tie))


def test_keypoints_full_scene_2048(gx):
    """City-scale scene size (2048^2) with ~5 % road and ~0.4 % intersection candidates: 2e5 candidates
    through the three passes, both tie orders."""
    rng = np.random.RandomState(11)
    # low-frequency field + noise so that candidates form blobs like a road mask does
    base = rng.rand(64, 64).astype(np.float32)
    up = torch.nn.functional.interpolate(torch.tensor(base)[None, None], size=(2048, 2048), mode="bicubic",
                                         align_corners=False)[0, 0].numpy()
    kp = np.clip((up + 0.15 * rng.rand(2048, 2048)) * 210, 0, 255).astype(np.uint8)
    road = np.clip((up[::-1] + 0.15 * rng.rand(2048, 2048)) * 210, 0, 255).astype(np.uint8)
    t0 = float(np.quantile(kp, 0.996)) / 255
    t1 = float(np.quantile(road, 0.95)) / 255
    for tie in ("numpy", "stable"):
        mine = _extract(gx, kp, road, t0, t1, 8, 16, tie)
        ref = O.extract_graph_points(kp, road, t0, t1, 8, 16, tie)
        assert ref.shape[0] > 200 and np.array_equal(mine, ref), (tie, mine.shape, ref.shape)
        assert gx.stats["candidates"][1] > 150000


def _nms_like_points(rng, size, n_try, min_dist):
    pts = rng.randint(0, size + 1, size=(n_try, 2)).astype(np.int64)
    keep = []
    import scipy.spatial
    for p in pts:
        if all((p[0] - q[0]) ** 2 + (p[1] - q[1]) ** 2 > min_dist ** 2 for q in keep[-400:]):
            keep.append(p)
    pts = np.array(keep, dtype=np.int64)
    tree = scipy.spatial.KDTree(pts)
    bad = {j for _, j in tree.query_pairs(r=min_dist)}
    return pts[[i for i in range(len(pts)) if i not in bad]]


@pytest.mark.parametrize("grid", [(400, 0, 256, 4), (400, 0, 256, 16), (2048, 64, 512, 8), (2048, 64, 512, 16)])
def test_pair_queries_match_oracle(gx, grid):
    """Box query + kNN of every tile of the BASELINE grids vs the oracle (ties by index), including
    tiles with no point, points on the inclusive tile border and more than 16 neighbours in range."""
    size, margin, P, per_edge = grid
    rng = np.random.RandomState(size + per_edge)
    tiles = get_patch_info_one_img(0, size, margin, P, per_edge)
    pts = _nms_like_points(rng, size, 900 if size == 400 else 5000, 9 if size == 400 else 17)
    # force border cases: points exactly on tile corners / edges, and an empty region
    x0, y0 = tiles[len(tiles) // 2][1]
    pts = pts[~((pts[:, 0] < size * 0.4) & (pts[:, 1] < size * 0.4))]
    pts = np.unique(np.concatenate([pts, np.array([[x0, y0], [x0 + P, y0 + P], [x0 + P, y0 + 7]])]), axis=0)
    rng.shuffle(pts)
    K, R = 16, 64.0
    txy = np.array([t[1] for t in tiles], dtype=np.int32)
    counts = gx.plan_pair_queries(torch.as_tensor(pts).to(DEV), txy, P, R)
    ref = [O.build_pair_queries(pts, t, K, R, "index") for t in tiles]
    assert list(counts) == [r[1].shape[0] for r in ref]
    assert (counts == 0).any() or size == 400
    bs = 64
    for b0 in range(0, len(tiles), bs):
        nb = min(bs, len(tiles) - b0)
        nmax = int(counts[b0:b0 + nb].max())
        if nmax == 0:
            continue
        p_d, q_d, v_d = gx.fill_batch(b0, nb, nmax, K)
        p_h, q_h, v_h = p_d.cpu().numpy(), q_d.cpu().numpy(), v_d.cpu().numpy()
        assert v_d.dtype == torch.bool
        for i in range(nb):
            idx, rp, rq, rv = ref[b0 + i]
            n = rp.shape[0]
            assert np.array_equal(p_h[i, :n], rp) and np.array_equal(q_h[i, :n], rq) and np.array_equal(v_h[i, :n], rv)
            assert not p_h[i, n:].any() and not q_h[i, n:].any() and not v_h[i, n:].any()   # np.pad zeros
    assert max(int(r[3].sum(1).max()) for r in ref if r[3].size) == K        # some query is truncated at 16


def _reference_edge_loop(ref, batches, scores_by_tile, K):
    """inferencer.py:206-222 verbatim on float32 scores; returns the two dicts."""
    es, ec = defaultdict(float), defaultdict(float)
    for (b0, nb) in batches:
        for ti in range(b0, b0 + nb):
            idx, pts, pairs, valid = ref[ti]
            sc = scores_by_tile[ti]
            if sc is None:
                continue
            for si in range(pts.shape[0]):
                for pi in range(K):
                    if not valid[si, pi]:
                        continue
                    s, t = pairs[si, pi]
                    score = sc[si, pi]
                    assert 0.0 <= score <= 1.0
                    es[(int(idx[s]), int(idx[t]))] += score
                    ec[(int(idx[s]), int(idx[t]))] += 1.0
    return es, ec


@pytest.mark.parametrize("grid,world,min_dist", [((400, 0, 256, 4), 1, 10), ((400, 0, 256, 16), 2, 10),
                                                 ((2048, 64, 512, 16), 1, 17), ((2048, 64, 512, 8), 4, 17),
                                                 ((400, 0, 256, 4), 1, 6),      # 64 < neighbours in range <= 128
                                                 ((400, 0, 256, 4), 2, 3)])     # > 128: one-thread-per-source fallback
def test_edge_aggregation_bit_exact(gx, grid, world, min_dist):
    """Random float32 scores through the device aggregation vs the reference triple loop: identical
    edges in identical (dict insertion) order for several thresholds; the score-buffer layout is the
    one infer_one_img uses (per batch [n, nmax_of_batch, K], batch plan of `world` ranks)."""
    size, margin, P, per_edge = grid
    rng = np.random.RandomState(3 * size + per_edge)
    tiles = get_patch_info_one_img(0, size, margin, P, per_edge)
    pts = _nms_like_points(rng, size, (700 if min_dist >= 10 else 6000) if size == 400 else 4000, min_dist)
    pts = pts[~((pts[:, 0] > size * 0.7) & (pts[:, 1] > size * 0.6))]       # an empty corner: empty tiles
    K, R, bs = 16, 64.0, 64 if size > 400 else 6
    txy = np.array([t[1] for t in tiles], dtype=np.int32)
    counts = gx.plan_pair_queries(torch.as_tensor(pts).to(DEV), txy, P, R)
    ref = [O.build_pair_queries(pts, t, K, R, "index") for t in tiles]
    plan = batch_plan(len(tiles), bs, world)
    tile_off = np.full(len(tiles), -1, dtype=np.int64)
    cursor, scores_by_tile, chunks = 0, [None] * len(tiles), []
    for (_, b0, nb) in plan:
        nmax = int(counts[b0:b0 + nb].max())
        if nmax == 0:
            continue
        block = rng.rand(nb, nmax, K).astype(np.float32)
        block[rng.rand(nb, nmax, K) < 0.02] = 1.0
        block[rng.rand(nb, nmax, K) < 0.02] = 0.0
        for i in range(nb):
            tile_off[b0 + i] = cursor + i * nmax * K
            scores_by_tile[b0 + i] = block[i]
        chunks.append(block.reshape(-1))
        cursor += nb * nmax * K
    flat = torch.as_tensor(np.concatenate(chunks)).to(DEV)
    batches = [(b0, nb) for (_, b0, nb) in plan]
    es, ec = _reference_edge_loop(ref, batches, scores_by_tile, K)
    for thr in (0.3, 0.5, 0.705):
        mine = gx.aggregate_edges(flat, tile_off, K, thr).cpu().numpy()
        want = np.array([e for e, v in es.items() if v / ec[e] > thr]).reshape(-1, 2)   # inferencer.py:223-229
        assert mine.dtype == np.int64 and np.array_equal(mine, want), (thr, mine.shape, want.shape)
        assert want.shape[0] > 10
    # NaN scores become -100 and trip the reference's assert (inferencer.py:206,219)
    bad = flat.clone()
    first_valid_tile = next(t for t in range(len(tiles)) if ref[t][3].any())
    si, pi = np.argwhere(ref[first_valid_tile][3])[0]
    bad[int(tile_off[first_valid_tile]) + int(si) * K + int(pi)] = float("nan")
    with pytest.raises(AssertionError):
        gx.aggregate_edges(bad, tile_off, K, 0.5)


def test_graph_stage_requires_cuda():
    with pytest.raises(RuntimeError):
        SceneGraph("cpu")
