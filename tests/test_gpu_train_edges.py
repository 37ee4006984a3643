"""GPU: the training step (train.cu) where its kernels change path, against the float64 oracle
(oracle/train_oracle.py in float64) on the engine's own image embeddings, slice by slice.

Cases: decoder rows that are not a multiple of the 64-row GEMM tile and a 25 x 25 token grid (@400); the benched
shape with dropout (B*N = 8192 points in the CSR scan, 128-chunk weight gradients over 131 072 pair tokens);
B*N = 4098 points, one more tile of the CSR scan holding two;
pair batches drawn the way the reference's dataset draws them (sources with replacement, (src, src) padding, so
CSR segments that are long, empty or hold a point both as src and as tgt); the other input dtypes; one point, one
sample, one pair; ViT-L; a batch without a valid slot; and decoder GEMMs of more than 65 535 row tiles.

Every gradient slice that one kernel call writes is compared on its own (`_slices`), so an error confined to a
few columns cannot hide behind a large neighbour.  The fp32 oracle's own error against float64 is printed beside
the engine's, for scale.
"""
import numpy as np
import pytest
import scipy.spatial
import torch

from oracle import train_oracle as TO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200 import train as T

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# Per slice, engine against float64.  Measured on an H100 (DESIGN.md §12): worst 1.6e-4 (inf) and 1.4e-4 (2-norm),
# both at B=16 @1024 where the weight-gradient chunks sum 32 768 rows each in fp32; every other case stays below
# 5e-5.  The fp32 oracle itself is off by up to 2.6e-3 (cuDNN runs its convolutions in TF32).
TAU_INF = 5e-4     # ||g - g64||_inf <= TAU_INF * ||g64||_inf
TAU_2 = 5e-4       # ||g - g64||_2   <= TAU_2   * ||g64||_2
KEY_BIAS = 1e-6    # |d in_proj_bias[128:256]| (exactly 0) <= KEY_BIAS * max |d in_proj_bias| of q and v (seen: 1.3e-7)
LOSS_RTOL = 1e-5


def _cfg(P=256, version="normal", focal=False, sam="vit_b"):
    return {"SAM_VERSION": sam, "PATCH_SIZE": P, "FREEZE_ENCODER": True, "BASE_LR": 1e-3,
            "TOPONET_VERSION": version, "FOCAL_LOSS": focal}


def _net(cfg, seed=0):
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=seed, logit_gain=4.0))
    return net.to(DEV)


def _masks(B, P, g):
    return {"keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
            "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}


def _knn_batch(B, P, N, Ns, Np, seed):
    """kNN pair queries, one source point per sample row (synth.make_topo_inputs), with one all-invalid row."""
    g = torch.Generator().manual_seed(seed)
    pts, pairs, valid = synth.make_topo_inputs(B, P, N, seed=seed, max_nbr=Np)
    pairs, valid = pairs[:, :Ns], valid[:, :Ns].clone()
    valid[0, 0] = False
    return {"rgb": synth.make_tiles(B, P, seed=seed), "graph_points": pts, "pairs": pairs, "valid": valid,
            "connected": torch.rand(valid.shape, generator=g) < 0.4, **_masks(B, P, g)}


def _reference_style_batch(P, Ns, Np, seed, radius=48.0):
    """Three tiles whose pairs are drawn like the reference's SatMapDataset draws them: Ns sources with
    replacement, weighted; each source's neighbours within `radius` (nearest first, the source itself dropped);
    the missing ones padded with (src, src), valid and connected False.
      tile 0: 5 close points, point 0 weighted 50:1, so it is the src of ~470 samples (> 1000 tokens for Np >= 3)
              and a tgt of the others and of every padding slot;
      tile 1: 34 points in the middle with heavy-tailed weights, and 6 isolated points on the border that are
              never sampled and lie outside everyone's radius: unreferenced, empty CSR segments;
      tile 2: a single point: every pair is (0, 0) and invalid.
    The tiles are padded to 40 points with (0, 0) points nothing refers to."""
    rng = np.random.RandomState(seed)
    N = 40
    iso = np.array([[0, 0], [P, 0], [0, P], [P, P], [P // 2, 0], [0, P // 2]], dtype=np.float64)
    tiles = [
        (P / 2 + rng.uniform(-12, 12, (5, 2)), np.array([50.0, 1, 1, 1, 1])),
        (np.concatenate([rng.uniform(P / 4, 3 * P / 4, (34, 2)), iso]),
         np.concatenate([rng.exponential(size=34) ** 3, np.zeros(6)])),
        (rng.uniform(0, P, (1, 2)), np.ones(1)),
    ]
    pts = np.zeros((3, N, 2), np.int64)
    pairs = np.zeros((3, Ns, Np, 2), np.int64)
    valid = np.zeros((3, Ns, Np), bool)
    conn = np.zeros((3, Ns, Np), bool)
    for b, (xy, w) in enumerate(tiles):
        xy = np.clip(np.round(xy), 0, P).astype(np.int64)
        n = xy.shape[0]
        pts[b, :n] = xy
        src = rng.choice(n, size=Ns, replace=True, p=w / w.sum())
        _, knn = scipy.spatial.KDTree(xy).query(xy[src], k=Np + 1, distance_upper_bound=radius)
        for i in range(Ns):
            nb = knn[i][knn[i] < n][1:]
            pairs[b, i, :, 0] = src[i]
            pairs[b, i, :, 1] = src[i]
            pairs[b, i, :len(nb), 1] = nb
            valid[b, i, :len(nb)] = True
            conn[b, i, :len(nb)] = rng.rand(len(nb)) < 0.4
    g = torch.Generator().manual_seed(seed)
    return {"rgb": synth.make_tiles(3, P, seed=seed), "graph_points": torch.from_numpy(pts),
            "pairs": torch.from_numpy(pairs), "valid": torch.from_numpy(valid), "connected": torch.from_numpy(conn),
            **_masks(3, P, g)}


def _dev(b):
    return {k: v.to(DEV) for k, v in b.items()}


def _engine_step(net, b, dropout_p=0.0, seed=0, topo=True):
    """(losses, grads by key, image embeddings) of one device step; the incoming gradient of the topology loss
    is 1, or absent (a mask-only backward) when not `topo`."""
    net._enable_training()
    heads = net._head_params()
    bb = T.validate_batch(b, net.image_size, DEV)
    args = T.make_args(bb, net.focal_loss, dropout_p, seed)
    s = net.image_size // 16
    emb = torch.empty((bb["B"], 256, s, s), device=DEV)
    ml, tl = T.head_losses(net._handle(DEV), bb, args, [k for k, _ in heads], [p for _, p in heads], emb)
    grads = torch.autograd.grad(ml + tl if topo else ml, [p for _, p in heads])
    return (ml.detach(), tl.detach()), dict(zip([k for k, _ in heads], grads)), emb


def _oracle(net, emb, b, version, dtype, keep=None, dropout_p=0.0):
    params = {k: p.detach().to(dtype).requires_grad_(True) for k, p in net._head_params()}
    ml, tl = TO.heads_losses(params, emb.to(dtype), b, net.image_size, net.focal_loss, version, keep, dropout_p)
    (ml + tl).backward()
    return (ml.detach(), tl.detach()), {k: p.grad for k, p in params.items()}


def _keep_masks(b, seed, p=0.1):
    B, Ns, Np = b["valid"].shape
    rows, tok = B * Ns, B * Ns * Np
    keep = {}
    for l in range(3):
        keep[(l, 0)] = T.dropout_keep(p, seed, l, 0, rows * 4 * Np * Np, DEV).view(rows, 4, Np, Np)
        for site in (1, 2, 3):
            keep[(l, site)] = T.dropout_keep(p, seed, l, site, tok * 128, DEV).view(rows, Np, 128)
    return keep


def _slices(k, shape):
    """(name, index) of the parts of gradient `k` that separate kernel calls or separate GEMM columns write."""
    if k.endswith("in_proj_weight"):
        return [("q", slice(0, 128)), ("k", slice(128, 256)), ("v", slice(256, 384))]
    if k.endswith("in_proj_bias"):      # the key block is exactly 0: checked on its own
        return [("q", slice(0, 128)), ("v", slice(256, 384))]
    if k == "topo_net.pair_proj.weight":
        return [("src", (slice(None), slice(0, 128))), ("tgt", (slice(None), slice(128, 256))),
                ("offset", (slice(None), slice(256, 258)))]
    if k.startswith("map_decoder.") and len(shape) == 4:     # ConvTranspose [Cin, Cout, 2, 2]: per output channel
        return [(f"co{c}", (slice(None), c)) for c in range(shape[1])]
    return [("", slice(None))]


def _errors(g, r):
    """{(key, slice): (inf-norm error, 2-norm error) relative to r}; slices where r is exactly 0 give None."""
    out = {}
    for k, rk in r.items():
        gk = g[k].to(torch.float64)
        for name, ix in _slices(k, rk.shape):
            a, w = gk[ix], rk[ix]
            ri, r2 = w.abs().max().item(), w.norm().item()
            if ri == 0:
                out[(k, name)] = None if (a == 0).all() else (float("inf"), float("inf"))
                continue
            d = a - w
            out[(k, name)] = (d.abs().max().item() / ri, d.norm().item() / r2)
    return out


def _key_bias_ratio(g):
    """Largest |d in_proj_bias[128:256]| over the q / v blocks' largest, over the layers (None without them)."""
    worst = None
    for k, v in g.items():
        if k.endswith("in_proj_bias"):
            scale = max(v[:128].abs().max().item(), v[256:].abs().max().item())
            r = v[128:256].abs().max().item() / scale
            worst = r if worst is None else max(worst, r)
    return worst


def _worst(err):
    ok = {s: e for s, e in err.items() if e is not None}
    wi = max(ok, key=lambda s: ok[s][0])
    w2 = max(ok, key=lambda s: ok[s][1])
    return ok[wi][0], wi, ok[w2][1], w2


def _check(tag, net, got, b, version, keep=None, dropout_p=0.0, fp32=True):
    """Engine against the float64 oracle: losses within LOSS_RTOL, every slice within TAU_INF / TAU_2, exactly-zero
    slices exactly zero, the key bias below KEY_BIAS.  Prints the engine's and the fp32 oracle's worst errors."""
    (gl, gg, emb) = got
    wl, wg = _oracle(net, emb, b, version, torch.float64, keep, dropout_p)
    err = _errors(gg, wg)
    ei, si, e2, s2 = _worst(err)
    line = f"[{tag}] engine vs float64: inf {ei:.2e} ({si[0]} {si[1]}), l2 {e2:.2e} ({s2[0]} {s2[1]})"
    if fp32:
        _, og = _oracle(net, emb, b, version, torch.float32, keep, dropout_p)
        fi, fsi, f2, fs2 = _worst(_errors(og, wg))
        line += f" | fp32 oracle vs float64: inf {fi:.2e} ({fsi[0]} {fsi[1]}), l2 {f2:.2e} ({fs2[0]} {fs2[1]})"
    kb = _key_bias_ratio(gg)
    if kb is not None:
        line += f" | key bias / q,v bias {kb:.2e}"
    print(line)
    bad = {s: e for s, e in err.items() if e is not None and (e[0] > TAU_INF or e[1] > TAU_2)}
    bad.update({("loss", i): (a.item(), w.item()) for i, (a, w) in enumerate(zip(gl, wl))
                if not abs(a.item() - w.item()) <= LOSS_RTOL * abs(w.item())})
    if kb is not None and not kb <= KEY_BIAS:
        bad["key bias"] = kb
    assert not bad, (tag, sorted(bad.items(), key=str))
    return err


# ---- cases -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,version,focal", [(2, "normal", False), (1, "no_transformer", True)])
def test_partial_row_tiles_at_400(B, version, focal):
    """@400 the token grid is 25 x 25: every decoder stage has B*625*4^i rows, never a multiple of 64, and the
    mask loss decodes pixels with s = 25; the last weight-gradient chunk holds a few rows."""
    net = _net(_cfg(400, version, focal))
    b = _dev(_knn_batch(B, 400, 40, 12, 7, seed=400 + B))
    _check(f"@400 B={B} {version}", net, _engine_step(net, b), b, version)


def test_benched_shape_with_dropout():
    """B=16 @512, N = Ns = 512, Np = 16 with dropout, the shape tools/train_bench.py times: 8192 points (two
    4096-point tiles of the CSR scan), 131 072 pair tokens (weight gradients in 128 chunks of 1024 rows)."""
    net = _net(_cfg(512))
    b = _dev(_knn_batch(16, 512, 512, 512, 16, seed=16))
    keep = _keep_masks(b, seed=77)
    got = _engine_step(net, b, dropout_p=0.1, seed=77)
    _check("bench B=16 @512 dropout", net, got, b, "normal", keep=keep, dropout_p=0.1)


def test_csr_scan_with_a_partial_tile():
    """B*N = 3 * 1366 = 4098 points: the CSR offsets are scanned in two 4096-point tiles, the second holding two."""
    net = _net(_cfg(256))
    b = _dev(_knn_batch(3, 256, 1366, 24, 8, seed=3))
    _check("B*N = 4098", net, _engine_step(net, b), b, "normal")


@pytest.mark.parametrize("Np,version", [(1, "normal"), (2, "no_offset"), (16, "normal"), (31, "normal")])
def test_reference_style_pair_batch(Np, version):
    b = _reference_style_batch(256, 512, Np, seed=Np)
    src = b["pairs"][0, :, :, 0].reshape(-1)
    assert (src == 0).sum() > 256 * min(Np, 4)      # one long src segment (> 1000 tokens from Np = 3 on)
    net = _net(_cfg(256, version, Np == 31))
    b = _dev(b)
    err = _check(f"reference-style Np={Np} {version}", net, _engine_step(net, b), b, version)
    if version == "no_offset":
        assert err[("topo_net.pair_proj.weight", "offset")] is None


@pytest.mark.parametrize("kind", ["f32_points_u8_masks_f32_rgb", "i32_points_and_pairs"])
def test_input_dtypes(kind):
    b = _knn_batch(2, 256, 40, 20, 16, seed=5)
    if kind == "f32_points_u8_masks_f32_rgb":
        g = torch.Generator().manual_seed(9)
        pts = b["graph_points"].float() + torch.rand(b["graph_points"].shape, generator=g) - 0.5
        b["graph_points"] = pts.clamp(0, 256)
        assert (b["graph_points"] != b["graph_points"].round()).float().mean() > 0.9
        b["valid"], b["connected"] = b["valid"].to(torch.uint8), b["connected"].to(torch.uint8)
        b["rgb"] = b["rgb"].float()
    else:
        b["graph_points"], b["pairs"] = b["graph_points"].int(), b["pairs"].int()
    net = _net(_cfg(256))
    b = _dev(b)
    _check(kind, net, _engine_step(net, b), b, "normal")


def test_one_point_one_sample_one_pair():
    """B = N = Ns = Np = 1: the only pair is (0, 0) (zero offset: the offset columns' gradient is exactly 0), the
    attention has one key (softmax 1: the q and k blocks' gradients are exactly 0), every matrix has one row."""
    g = torch.Generator().manual_seed(1)
    b = {"rgb": synth.make_tiles(1, 256, seed=1), "graph_points": torch.tensor([[[100, 60]]]),
         "pairs": torch.zeros((1, 1, 1, 2), dtype=torch.int64), "valid": torch.ones((1, 1, 1), dtype=torch.bool),
         "connected": torch.ones((1, 1, 1), dtype=torch.bool), **_masks(1, 256, g)}
    net = _net(_cfg(256))
    b = _dev(b)
    err = _check("B=N=Ns=Np=1", net, _engine_step(net, b), b, "normal")
    assert err[("topo_net.pair_proj.weight", "offset")] is None
    for l in range(3):
        k = f"topo_net.transformer_encoder.layers.{l}.self_attn.in_proj_weight"
        assert err[(k, "q")] is None and err[(k, "k")] is None


def test_vit_l_encoder():
    cfg = _cfg(256, "normal", False, sam="vit_l")
    net = _net(cfg)
    b = _dev(_knn_batch(2, 256, 40, 20, 16, seed=12))
    _check("ViT-L @256", net, _engine_step(net, b), b, "normal")


def test_batch_without_a_valid_slot():
    """The topology loss is 0/0 = NaN as in the reference; the decoder's gradients are those of the mask loss alone,
    bit for bit, and each TopoNet gradient is NaN wherever the float64 oracle's is."""
    b = _knn_batch(2, 256, 40, 20, 16, seed=8)
    b["valid"] = torch.zeros_like(b["valid"])
    net = _net(_cfg(256))
    b = _dev(b)
    (ml, tl), g, emb = _engine_step(net, b)
    _, gm, _ = _engine_step(net, b, topo=False)
    (wml, wtl), wg = _oracle(net, emb, b, "normal", torch.float64)
    assert torch.isnan(tl) and torch.isnan(wtl)
    assert abs(ml.item() - wml.item()) <= LOSS_RTOL * abs(wml.item())
    nan = 0
    for k, w in wg.items():
        if k.startswith("map_decoder."):
            assert torch.equal(g[k], gm[k]), k
        else:
            assert g[k][w.isnan()].isnan().all(), k
            nan += int(w.isnan().sum())
    assert nan > 0
    dec = {k: v for k, v in wg.items() if k.startswith("map_decoder.")}
    bad = {s: e for s, e in _errors(gm, dec).items() if e is not None and (e[0] > TAU_INF or e[1] > TAU_2)}
    assert not bad, bad


def test_decoder_rows_beyond_65535_tiles():
    """B=16 @1024: the decoder's stage-3 GEMM and its input-gradient GEMM have 64 * 16 * 64^2 = 4 194 304 rows,
    65 536 row tiles, one more than a grid.y dimension holds."""
    net = _net(_cfg(1024))
    b = _dev(_knn_batch(16, 1024, 64, 64, 16, seed=1024))
    _check("B=16 @1024", net, _engine_step(net, b), b, "normal", fp32=False)
