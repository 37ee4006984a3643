"""MAX_NEIGHBOR_QUERIES / n_pairs from 17 to 32: TopoNet on the layered path (17..31) and on the
32-pair fused kernel against the fp32 oracle, pair queries and edge aggregation at K = 24 and 32 against
the oracle's restatement of inferencer.py:126-230, one scene end to end, and the errors above 32."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200.graph import SceneGraph  # noqa: E402
from sam_road_b200.inferencer import batch_plan, get_patch_info_one_img, infer_one_img  # noqa: E402
from sam_road_b200 import synth  # noqa: E402
from test_gpu_graph import _nms_like_points, _reference_edge_loop  # noqa: E402
from test_gpu_scene import _check_scene, _scene_cfg  # noqa: E402
from test_gpu_shapes import TOL_LOGIT, _build, _config, _topo_check  # noqa: E402

DEV = "cuda:0"
C2, C3, C4 = (2048, 64, 512, 16), (400, 0, 256, 16), (2048, 64, 512, 8)


@pytest.fixture(scope="module", autouse=True)
def _fp32_oracle_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def gx():
    return SceneGraph(DEV)


# --------------------------------------------------------------------------------------------------
# TopoNet
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_pairs", [17, 24, 31, 32])
def test_toponet_wide_npairs(n_pairs):
    """17..31: layered path (topo_attention over up to 32 keys); 32: the fused kernel, 4 samples x 32
    pairs per tile.  int64 / int32 / float inputs, an all-invalid row, a masked key in front of valid
    ones, logit_gain 12.  The neighbour radius covers the whole tile, so slots up to 32 are valid."""
    spec, sd, net = _build(_config(256), seed=2, gain=12.0)
    g = torch.Generator().manual_seed(60 + n_pairs)
    feat = torch.randn(2, 256, 16, 16, generator=g).to(DEV)
    pts, prs, val = synth.make_topo_inputs(2, 256, 40, seed=61 + n_pairs, max_nbr=n_pairs, radius=400.0)
    assert prs.shape[2] == n_pairs and val[0].all(dim=1).any()
    val[1, 2] = False                                    # all-invalid row: flipped to all-valid
    val[0, 5, 0] = False                                 # a masked key in front of valid ones
    pts, prs, val = pts.to(DEV), prs.to(DEV), val.to(DEV)
    _topo_check(net, sd, spec, feat, pts, prs, val, "int64")
    _topo_check(net, sd, spec, feat, pts.int(), prs.int(), val, "int32")
    _topo_check(net, sd, spec, feat, pts.float() + 0.25, prs, val, "float")


def test_toponet_32_pairs_tiles_straddle_images():
    """Ns = 21 samples of N = 30 points at B = 3: 21 * 32 tokens per image, so 128-token tiles of the
    fused kernel straddle images."""
    spec, sd, net = _build(_config(256), seed=3, gain=12.0)
    g = torch.Generator().manual_seed(70)
    feat = torch.randn(3, 256, 16, 16, generator=g).to(DEV)
    pts, prs, val = synth.make_topo_inputs(3, 256, 30, seed=71, max_nbr=32, ragged=False, radius=400.0)
    prs, val = prs[:, :21].contiguous(), val[:, :21].contiguous()
    val[2, 4] = False
    val[1, 7, :3] = False
    _topo_check(net, sd, spec, feat, pts.to(DEV), prs.to(DEV), val.to(DEV), "Ns=21 np=32")


def test_toponet_padding_to_32_pairs_keeps_valid_logits():
    """A 16-pair input extended to 32 slots with invalid ones: masked keys are left out of the softmax,
    so every valid slot's logit agrees with the 16-pair call (fused 16 vs fused 32 kernel).  Every row
    has a valid slot: an all-invalid row is flipped over 32 slots instead of 16."""
    _, _, net = _build(_config(256), seed=4, gain=12.0)
    g = torch.Generator().manual_seed(80)
    feat = torch.randn(2, 256, 16, 16, generator=g).to(DEV)
    pts, prs, val = synth.make_topo_inputs(2, 256, 36, seed=81, max_nbr=16, ragged=False)
    val[:, :, 0] = True                                  # slot 0 valid everywhere (a self pair if isolated)
    val[0, 3, 0] = False
    val[0, 3, 5] = True
    assert val.any(dim=2).all()
    src = prs[..., :1, 0:1].expand(-1, -1, 16, 2)        # padding slots point back at the source
    prs32 = torch.cat([prs, src], dim=2).contiguous()
    val32 = torch.cat([val, torch.zeros_like(val)], dim=2).contiguous()
    pts, prs, val, prs32, val32 = (t.to(DEV) for t in (pts, prs, val, prs32, val32))
    l16, _ = net._topo(feat, pts, prs, val, True)
    l32, _ = net._topo(feat, pts, prs32, val32, True)
    torch.cuda.synchronize()
    span = (l16.max() - l16.min()).item()
    v = val.unsqueeze(-1)
    err = ((l32[:, :, :16] - l16).abs() * v).max().item()
    assert err <= max(TOL_LOGIT, 2e-3 * span), (err, span)
    bias = l32[:, :, 16:]                                # masked slots report output_proj.bias
    assert torch.equal(bias, bias.flatten()[0].expand_as(bias))


def test_toponet_rejects_33_pairs():
    _, _, net = _build(_config(256), seed=2)
    feat = torch.zeros(1, 256, 16, 16, device=DEV)
    pts, prs, val = synth.make_topo_inputs(1, 256, 40, seed=1, max_nbr=33, radius=400.0)
    with pytest.raises(RuntimeError, match="n_pairs=33"):
        net._topo(feat, pts.to(DEV), prs.to(DEV), val.to(DEV), True)


# --------------------------------------------------------------------------------------------------
# graph stage
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [24, 32])
@pytest.mark.parametrize("grid", [C2, C3, C4])
def test_wide_pair_queries_match_oracle(gx, grid, K):
    """Box query + kNN with K slots per query vs the oracle (ties by index): identical points, pairs
    and valid mask per tile, some query truncated at K.  A K = 32 plan also serves K = 16 fills."""
    size, margin, P, per_edge = grid
    rng = np.random.RandomState(size + per_edge + K)
    tiles = get_patch_info_one_img(0, size, margin, P, per_edge)
    pts = _nms_like_points(rng, size, 900 if size == 400 else 5000, 9 if size == 400 else 17)
    x0, y0 = tiles[len(tiles) // 2][1]
    pts = np.unique(np.concatenate([pts, np.array([[x0, y0], [x0 + P, y0 + P], [x0 + P, y0 + 7]])]), axis=0)
    rng.shuffle(pts)
    R = 64.0 if size == 400 else 128.0                 # the 2048 scenes are sparser: > 32 neighbours in range
    txy = np.array([t[1] for t in tiles], dtype=np.int32)
    counts = gx.plan_pair_queries(torch.as_tensor(pts).to(DEV), txy, P, R, max_nbr=K)
    ref = [O.build_pair_queries(pts, t, K, R, "index") for t in tiles]
    assert list(counts) == [r[1].shape[0] for r in ref]
    bs = 64
    for b0 in range(0, len(tiles), bs):
        nb = min(bs, len(tiles) - b0)
        nmax = int(counts[b0:b0 + nb].max())
        if nmax == 0:
            continue
        for k in ((K, 16) if K == 32 else (K,)):
            p_d, q_d, v_d = gx.fill_batch(b0, nb, nmax, k)
            p_h, q_h, v_h = p_d.cpu().numpy(), q_d.cpu().numpy(), v_d.cpu().numpy()
            for i in range(nb):
                idx, rp, rq, rv = ref[b0 + i]
                n = rp.shape[0]
                assert np.array_equal(p_h[i, :n], rp) and np.array_equal(q_h[i, :n], rq[:, :k])
                assert np.array_equal(v_h[i, :n], rv[:, :k])
                assert not p_h[i, n:].any() and not q_h[i, n:].any() and not v_h[i, n:].any()
    assert max(int(r[3].sum(1).max()) for r in ref if r[3].size) == K        # some query is truncated at K


@pytest.mark.parametrize("grid,world,min_dist", [((400, 0, 256, 4), 1, 10), ((2048, 64, 512, 16), 2, 17),
                                                 ((400, 0, 256, 4), 1, 6),      # 64 < neighbours in range <= 128
                                                 ((400, 0, 256, 4), 2, 3)])     # > 128: one-thread-per-source fallback
def test_edge_aggregation_32_bit_exact(gx, grid, world, min_dist):
    """K = 32: every lane of the warp kernel loads one pair slot.  Random float32 scores vs the
    reference triple loop: identical edges in identical order at several thresholds; NaN trips the
    assert."""
    size, margin, P, per_edge = grid
    rng = np.random.RandomState(5 * size + per_edge + min_dist)
    tiles = get_patch_info_one_img(0, size, margin, P, per_edge)
    pts = _nms_like_points(rng, size, (700 if min_dist >= 10 else 6000) if size == 400 else 4000, min_dist)
    pts = pts[~((pts[:, 0] > size * 0.7) & (pts[:, 1] > size * 0.6))]       # an empty corner: empty tiles
    K, R, bs = 32, 64.0 if size == 400 else 128.0, 64 if size > 400 else 6
    txy = np.array([t[1] for t in tiles], dtype=np.int32)
    counts = gx.plan_pair_queries(torch.as_tensor(pts).to(DEV), txy, P, R, max_nbr=K)
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
    es, ec = _reference_edge_loop(ref, [(b0, nb) for (_, b0, nb) in plan], scores_by_tile, K)
    assert max(int(r[3].sum(1).max()) for r in ref if r[3].size) > 16     # slots above 16 are in play
    for thr in (0.3, 0.5, 0.705):
        mine = gx.aggregate_edges(flat, tile_off, K, thr).cpu().numpy()
        want = np.array([e for e, v in es.items() if v / ec[e] > thr]).reshape(-1, 2)
        assert mine.dtype == np.int64 and np.array_equal(mine, want), (thr, mine.shape, want.shape)
        assert want.shape[0] > 10
    bad = flat.clone()
    t = next(t for t in range(len(tiles)) if ref[t][3].any())
    si, pi = np.argwhere(ref[t][3])[0]
    bad[int(tile_off[t]) + int(si) * K + int(pi)] = float("nan")
    with pytest.raises(AssertionError):
        gx.aggregate_edges(bad, tile_off, K, 0.5)


def test_wide_pair_queries_errors(gx):
    """MAX_NEIGHBOR_QUERIES 33 is refused by the plan; fill and aggregate refuse a K above the
    planned one."""
    tiles = get_patch_info_one_img(0, 400, 0, 256, 4)
    txy = np.array([t[1] for t in tiles], dtype=np.int32)
    pts = torch.as_tensor(_nms_like_points(np.random.RandomState(1), 400, 300, 10)).to(DEV)
    with pytest.raises(RuntimeError, match="MAX_NEIGHBOR_QUERIES=33"):
        gx.plan_pair_queries(pts, txy, 256, 64.0, max_nbr=33)
    counts = gx.plan_pair_queries(pts, txy, 256, 64.0, max_nbr=16)
    nmax = int(counts[:4].max())
    with pytest.raises(RuntimeError, match="MAX_NEIGHBOR_QUERIES=24"):
        gx.fill_batch(0, 4, nmax, 24)
    scores = torch.full((len(tiles) * nmax * 24,), 0.5, device=DEV)
    offs = np.arange(len(tiles), dtype=np.int64) * nmax * 24
    with pytest.raises(RuntimeError, match="MAX_NEIGHBOR_QUERIES=24"):
        gx.aggregate_edges(scores, offs, 24, 0.5)
    with pytest.raises(RuntimeError, match="MAX_NEIGHBOR_QUERIES=33"):
        gx.aggregate_edges(scores, offs, 33, 0.5)


# --------------------------------------------------------------------------------------------------
# scene
# --------------------------------------------------------------------------------------------------
def test_scene_with_32_neighbour_queries():
    """infer_one_img on the C3 grid with MAX_NEIGHBOR_QUERIES = 32 (fused 32-pair TopoNet, 32-slot
    pair queries and aggregation), checked like test_gpu_scene: masks within 1 LSB, identical nodes,
    identical edges from our topology scores, edges within 2e-3 of the threshold otherwise."""
    size, patch, per_edge, margin = 400, 256, 16, 0
    img = np.random.RandomState(size + per_edge).randint(0, 256, size=(size, size, 3)).astype(np.uint8)
    cfg = dict(_scene_cfg(patch, per_edge, margin), INFER_BATCH_SIZE=64, MAX_NEIGHBOR_QUERIES=32)
    timings, _ = _check_scene(cfg, img, seed=11, gain=6.0, cand_frac=(0.004, 0.05), tie="numpy", min_points=50)
    assert timings["n_points"] >= 50


def test_scene_rejects_33_neighbour_queries():
    _, _, net = _build(_config(256), seed=2)
    img = np.random.RandomState(0).randint(0, 256, size=(256, 256, 3)).astype(np.uint8)
    cfg = dict(_scene_cfg(256, 1, 0), MAX_NEIGHBOR_QUERIES=33, ITSC_THRESHOLD=0.0, ROAD_THRESHOLD=0.0)
    with pytest.raises(RuntimeError, match="MAX_NEIGHBOR_QUERIES=33"):
        infer_one_img(net, img, cfg, device=torch.device(DEV))
