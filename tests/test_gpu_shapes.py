"""Parity at the shapes the library accepts beyond the benched configurations: tile sizes whose token
grid is odd (the mask epilogue pairs tokens across row and image ends), smaller than one 14x14 window
(P < 224: the window blocks become one padded window) or not a divisor of 128 (the neck's 3x3 conv
runs through im2col); TopoNet with n_pairs != 16 (the layered path: pair features, per-layer GEMMs
and topo_attention instead of the fused kernel) and with fewer samples than points; the GEMM
epilogues at partial column tiles with padded output rows.

Model parity uses the fp32 oracle and the 1e-3 logit tolerance of test_gpu_model.py and adds its
numbers to parity_report.json in the test report directory.  Every output buffer is filled with NaN before the call, so
an element the kernels never write fails as NaN instead of passing on stale memory."""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402

DEV = "cuda:0"
TOL_LOGIT = 1e-3
# image embeddings against the fp32 oracle, max-abs relative to their max-abs: measured at most 8.4e-4 over
# test_encode_and_topo_parity and test_tile_size_parity on an H100 80GB HBM3 at 700 W
TOL_FEAT_REL = 3.5e-3
_REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _fp32_oracle_math(report_dir):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    path = os.path.join(report_dir, "parity_report.json")
    old = {}
    if os.path.exists(path):
        try:
            old = json.load(open(path))
        except Exception:
            old = {}
    old.update(_REPORT)
    json.dump(old, open(path, "w"), indent=1, sort_keys=True)


def _config(patch, version="vit_b", topo="normal", samdec=False):
    return dict(SAM_VERSION=version, PATCH_SIZE=patch, USE_SAM_DECODER=samdec,
                ENCODER_LORA=False, LORA_RANK=0, TOPONET_VERSION=topo, NO_SAM=False)


def _build(cfg, seed=0, gain=1.0):
    spec = O.ModelSpec.from_config(cfg)
    sd = synth.make_state_dict(cfg, seed=seed, logit_gain=gain)
    net = SAMRoad(cfg)
    net.load_state_dict(sd, strict=True)
    net.eval().to(DEV)
    return spec, {k: v.to(DEV) for k, v in sd.items()}, net


def _st():
    return torch.cuda.current_stream().cuda_stream


def _maxabs(a, b):
    return (a.float() - b.float()).abs().max().item()


def _nan_blocks(x, limit=8):
    """(image, row // 16, col // 16) of the first 16x16 mask blocks holding a NaN ([B, P, P, C] input)."""
    bad = torch.isnan(x).any(dim=-1)
    B, P, _ = bad.shape
    blk = bad.view(B, P // 16, 16, P // 16, 16).any(dim=4).any(dim=2)
    return [tuple(i) for i in blk.nonzero().tolist()[:limit]], int(blk.sum().item())


# --------------------------------------------------------------------------------------------------
# whole model at other tile sizes
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,patch,version,samdec", [
    ("vitb_192", 192, "vit_b", False),          # s = 12 < 14: one padded window
    ("vitb_192_samdec", 192, "vit_b", True),
    ("vitb_208", 208, "vit_b", False),          # s = 13: odd grid, smaller than the window
    ("vitb_384", 384, "vit_b", False),          # s = 24: padded windows, im2col neck
    ("vitb_400", 400, "vit_b", False),          # s = 25: odd grid and s*s odd (pairs cross images)
    ("vitb_400_samdec", 400, "vit_b", True),
    ("vitb_448", 448, "vit_b", False),          # s = 28: windows tile the grid exactly
    ("vith_400", 400, "vit_h", False),          # head_dim 80 (ViT-H: 1280 / 16)
])
def test_tile_size_parity(name, patch, version, samdec):
    B = 2
    cfg = _config(patch, version, samdec=samdec)
    spec, sd, net = _build(cfg, seed=1)
    rgb = synth.make_tiles(B, patch, seed=7).to(DEV).float()
    with torch.no_grad():
        o_scores, o_feat, o_logits = O.infer_masks_and_img_features(sd, spec, rgb, return_logits=True)
    pts, prs, val = [t.to(DEV) for t in synth.make_topo_inputs(B, patch, 40, seed=8)]
    with torch.no_grad():
        o_ts, o_tl = O.infer_toponet(sd, spec, o_feat, pts, prs, val, return_logits=True)

    # the C ABI straight, into NaN-filled outputs
    lib = _lib.load()
    s = patch // 16
    scores = torch.full((B, patch, patch, 2), float("nan"), device=DEV)
    logits = torch.full((B, patch, patch, 2), float("nan"), device=DEV)
    feat = torch.full((B, 256, s, s), float("nan"), device=DEV)
    _lib.check(lib.samroad_encode_masks(net._handle(rgb.device), rgb.data_ptr(), _lib.F32, B,
                                        scores.data_ptr(), logits.data_ptr(), feat.data_ptr(), _st()),
               "samroad_encode_masks")
    torch.cuda.synchronize()
    nan_blocks, n_nan_blocks = _nan_blocks(logits)
    _, scores_module, t_logits, _ = net(rgb, pts, prs, val)
    rep = {
        "B": B, "grid": s,
        "feat_maxabs": _maxabs(feat, o_feat), "feat_absmax": o_feat.abs().max().item(),
        "mask_logit_maxabs": _maxabs(logits, o_logits),
        "mask_logit_range": [o_logits.min().item(), o_logits.max().item()],
        "mask_score_maxabs": _maxabs(scores, o_scores),
        "mask_nan_blocks_16x16": n_nan_blocks,
        "topo_logit_maxabs_valid": ((t_logits - o_tl).abs() * val.unsqueeze(-1)).max().item(),
        "topo_logit_maxabs_all": _maxabs(t_logits, o_tl),
        "tolerance_logit": TOL_LOGIT,
    }
    _REPORT[f"shapes_{name}"] = rep
    print(name, json.dumps(rep))
    assert n_nan_blocks == 0, f"16x16 mask blocks never written (image, row/16, col/16): {nan_blocks}"
    assert not torch.isnan(scores).any() and not torch.isnan(feat).any()
    assert torch.equal(scores_module, scores)            # the module path computes the same masks
    assert rep["mask_logit_maxabs"] <= TOL_LOGIT and rep["mask_score_maxabs"] <= TOL_LOGIT, rep
    assert rep["feat_maxabs"] <= TOL_FEAT_REL * rep["feat_absmax"], rep
    assert rep["topo_logit_maxabs_valid"] <= TOL_LOGIT and rep["topo_logit_maxabs_all"] <= 3 * TOL_LOGIT, rep


# --------------------------------------------------------------------------------------------------
# TopoNet: the layered path (n_pairs != 16) and Ns != N on both paths
# --------------------------------------------------------------------------------------------------
def _topo_check(net, sd, spec, feat, pts, prs, val, tag):
    with torch.no_grad():
        o_ts, o_tl = O.infer_toponet(sd, spec, feat, pts, prs, val, return_logits=True)
    t_logits, t_scores = net._topo(feat, pts, prs, val, True)
    torch.cuda.synchronize()
    span = (o_tl.max() - o_tl.min()).item()
    v = val.unsqueeze(-1)
    err_valid = ((t_logits - o_tl).abs() * v).max().item()
    err_all = _maxabs(t_logits, o_tl)
    assert torch.isfinite(t_logits).all() and torch.isfinite(t_scores).all(), tag
    # logit_gain 12 spreads the logits over several units: tolerance relative to their span, as in
    # test_gpu_model.test_parity_with_wide_logits
    tol = max(TOL_LOGIT, 2e-3 * span)
    assert err_valid <= tol and err_all <= 3 * tol, (tag, err_valid, err_all, span)
    assert _maxabs(t_scores, o_ts) <= tol, tag
    return err_valid, span


@pytest.mark.parametrize("topo,n_pairs", [("normal", 1), ("normal", 2), ("normal", 5), ("normal", 8),
                                          ("normal", 15), ("normal", 7), ("no_offset", 7),
                                          ("no_transformer", 7)])
def test_toponet_layered_path(topo, n_pairs):
    """n_pairs != 16 runs topo_pair_features, per-layer wgmma GEMMs with LayerNorm epilogues and
    topo_attention over sequences of n_pairs; int64 / int32 / float inputs, an all-invalid row."""
    cfg = _config(256, topo=topo)
    spec, sd, net = _build(cfg, seed=2, gain=12.0)
    g = torch.Generator().manual_seed(30 + n_pairs)
    feat = torch.randn(2, 256, 16, 16, generator=g).to(DEV)
    pts, prs, val = synth.make_topo_inputs(2, 256, 30, seed=31 + n_pairs, max_nbr=n_pairs)
    assert prs.shape[2] == n_pairs
    val[1, 2] = False                                    # all-invalid row: flipped to all-valid
    val[0, 5, 0] = False                                 # a masked key in front of valid ones
    pts, prs, val = pts.to(DEV), prs.to(DEV), val.to(DEV)
    err, span = _topo_check(net, sd, spec, feat, pts, prs, val, "int64")
    _topo_check(net, sd, spec, feat, pts.int(), prs.int(), val, "int32")
    _topo_check(net, sd, spec, feat, pts.float() + 0.25, prs, val, "float")
    _REPORT[f"shapes_toponet_{topo}_np{n_pairs}"] = {"topo_logit_maxabs_valid": err, "topo_logit_span": span}


@pytest.mark.parametrize("n_pairs", [16, 7])
def test_toponet_fewer_samples_than_points(n_pairs):
    """pairs / valid cover Ns = 21 samples of N = 30 points (B = 3: 21 * n_pairs tokens per image, so
    128-token tiles of the fused kernel straddle images); n_pairs 16 = fused kernel, 7 = layered path."""
    cfg = _config(256)
    spec, sd, net = _build(cfg, seed=3, gain=12.0)
    g = torch.Generator().manual_seed(40 + n_pairs)
    feat = torch.randn(3, 256, 16, 16, generator=g).to(DEV)
    pts, prs, val = synth.make_topo_inputs(3, 256, 30, seed=41 + n_pairs, max_nbr=n_pairs, ragged=False)
    Ns = 21
    prs, val = prs[:, :Ns].contiguous(), val[:, :Ns].contiguous()
    val[2, 4] = False
    pts, prs, val = pts.to(DEV), prs.to(DEV), val.to(DEV)
    err, span = _topo_check(net, sd, spec, feat, pts, prs, val, f"Ns={Ns}")
    _REPORT[f"shapes_toponet_ns{Ns}_np{n_pairs}"] = {"topo_logit_maxabs_valid": err, "topo_logit_span": span}


# --------------------------------------------------------------------------------------------------
# op level
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,hd", [(12, 64), (13, 64), (25, 64), (28, 64), (40, 64), (13, 80), (25, 80)])
def test_window_attention_grid_sizes(s, hd):
    """14x14 window attention on grids smaller than one window (s = 12, 13), with padded edge windows
    (25, 40) and exact tiling (28): the fp32 reference with the pad semantics of
    test_gpu_ops.test_encoder_attention, and the tensor-core kernel against the SIMT kernel."""
    lib = _lib.load()
    B, win = 2, 14
    heads = 12 if hd == 64 else 16
    D = heads * hd
    g = torch.Generator().manual_seed(100 + s)
    x = torch.randn(B, s, s, D, generator=g).to(DEV)
    w = (torch.randn(3 * D, D, generator=g) / math.sqrt(D)).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(DEV)
    rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    qkv16 = F.linear(x, w, bias).to(torch.float16).contiguous()
    bias16 = bias.to(torch.float16).float()
    xw, padded = O.window_split(qkv16.float(), win)
    mask, _ = O.window_split(torch.ones(B, s, s, 1, device=DEV), win)
    xw = torch.where(mask.bool(), xw, bias16.view(1, 1, 1, -1).expand_as(xw))
    ref = O.window_merge(O.attention_core(xw, rel_h, rel_w, heads), win, padded, (s, s))
    outs = []
    try:
        for simt in (0, 1):
            lib.samroad_debug_force_simt_attention(simt)
            out = torch.full((B * s * s, D), float("nan"), dtype=torch.float16, device=DEV)
            _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias16.data_ptr(), rel_h.data_ptr(),
                                                rel_w.data_ptr(), B, s, win, heads, hd, out.data_ptr(),
                                                _st()), "attention")
            torch.cuda.synchronize()
            outs.append(out.float().view(B, s, s, D))
    finally:
        lib.samroad_debug_force_simt_attention(0)
    mag = ref.abs().max().item()
    errs = [(o - ref).abs().max().item() for o in outs]
    print(f"s={s} hd={hd}: tc {errs[0]:.3e} simt {errs[1]:.3e} |ref|max {mag:.3f}")
    assert all(torch.isfinite(o).all() for o in outs)
    assert errs[0] < 1.5e-3 * max(1.0, mag) and errs[1] < 1.5e-3 * max(1.0, mag), errs
    assert (outs[0] - outs[1]).abs().max().item() <= 2.5e-3 * outs[1].abs().max().item()


def _ln_ref(x, group, gamma, beta, eps, act):
    M, N = x.shape
    y = F.layer_norm(x.view(M, N // group, group), (group,), gamma, beta, eps).view(M, N)
    return F.gelu(y) if act == 1 else y


@pytest.mark.parametrize("M,N,K,group,act,tokens", [
    (2 * 144, 256, 256, 64, 1, 144),        # SAM upscaler at P = 192 (128-column tiles)
    (128 * 144, 256, 256, 64, 1, 144),      # enough rows for 256-column tiles: two groups per half
    (2 * 625, 256, 2304, 256, 0, 625),      # neck 3x3 conv at P = 400 (im2col operand)
    (3 * 784, 512, 256, 128, 1, 784),       # decoder stage 1 at P = 448
])
def test_gemm_ln_groups_and_nchw(M, N, K, group, act, tokens):
    lib = _lib.load()
    A = (torch.randn(M, K, generator=torch.Generator().manual_seed(M + group)) * 1.0).half().to(DEV)
    W = (torch.randn(N, K, generator=torch.Generator().manual_seed(N + K)) / math.sqrt(K)).half().to(DEV)
    bias = 0.3 * torch.randn(N, device=DEV)
    resid = torch.randn(M, N, device=DEV)
    gamma = 1 + 0.1 * torch.randn(group, device=DEV)
    beta = 0.1 * torch.randn(group, device=DEV)
    y = _ln_ref(A.float() @ W.float().t() + bias + resid, group, gamma, beta, 1e-6, act)
    o16 = torch.full((M, N), float("nan"), dtype=torch.float16, device=DEV)
    o32 = torch.full((M, N), float("nan"), device=DEV)
    onchw = torch.full((M // tokens, N, tokens), float("nan"), device=DEV)
    _lib.check(lib.samroad_op_gemm_ln(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                      resid.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-6, group, act,
                                      o16.data_ptr(), o32.data_ptr(), onchw.data_ptr(), tokens, N, _st()),
               "gemm_ln")
    torch.cuda.synchronize()
    assert (o32 - y).abs().max().item() < 2e-3
    assert (o16.float() - y).abs().max().item() < 6e-3
    assert torch.equal(onchw.permute(0, 2, 1).reshape(M, N), o32)


@pytest.mark.parametrize("epi,N", [("f16", 96), ("f16", 160), ("f16", 288), ("f32", 96), ("f32", 160),
                                   ("f32", 288), ("ln", 192), ("ln", 320)])
def test_gemm_partial_column_tiles_padded_rows(epi, N):
    """N not a multiple of the 128-column tile (last tile partial, or one column half empty), output
    row pitch ldo > N: every column < N correct, the padding columns untouched (still NaN).  The
    LayerNorm epilogue needs whole 64-column groups, hence N = 192 / 320 there."""
    lib = _lib.load()
    M, K = 300, 256
    ldo = N + 32
    A = torch.randn(M, K, generator=torch.Generator().manual_seed(N)).half().to(DEV)
    W = (torch.randn(N, K, generator=torch.Generator().manual_seed(N + 1)) / math.sqrt(K)).half().to(DEV)
    bias = torch.randn(N, device=DEV)
    acc = A.float() @ W.float().t() + bias
    if epi == "f16":
        out = torch.full((M, ldo), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(lib.samroad_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), 1,
                                           out.data_ptr(), ldo, _st()), "gemm_f16")
        ref, tol, outs = F.gelu(acc), 2e-3 * max(1.0, acc.abs().max().item()), [out]
    elif epi == "f32":
        T = 7
        pos = torch.randn(T, N, device=DEV)
        out = torch.full((M, ldo), float("nan"), device=DEV)
        out[:, :N] = torch.randn(M, N, device=DEV)           # in-place residual with the same pitch
        ref = acc + out[:, :N] + pos[torch.arange(M, device=DEV) % T]
        _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                           out.data_ptr(), pos.data_ptr(), T, out.data_ptr(), ldo, _st()),
                   "gemm_f32")
        tol, outs = 2e-4 * max(1.0, ref.abs().max().item()), [out]
    else:
        group = 64
        resid = torch.full((M, ldo), float("nan"), device=DEV)
        resid[:, :N] = torch.randn(M, N, device=DEV)
        gamma = 1 + 0.1 * torch.randn(group, device=DEV)
        beta = 0.1 * torch.randn(group, device=DEV)
        ref = _ln_ref(acc + resid[:, :N], group, gamma, beta, 1e-6, 0)
        o16 = torch.full((M, ldo), float("nan"), dtype=torch.float16, device=DEV)
        o32 = torch.full((M, ldo), float("nan"), device=DEV)
        _lib.check(lib.samroad_op_gemm_ln(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                          resid.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-6, group, 0,
                                          o16.data_ptr(), o32.data_ptr(), None, 1, ldo, _st()), "gemm_ln")
        tol, outs = 6e-3, [o16, o32]
    torch.cuda.synchronize()
    for o in outs:
        assert not torch.isnan(o[:, :N]).any(), "columns below N left unwritten"
        assert torch.isnan(o[:, N:]).all(), "padding columns beyond N overwritten"
        err = (o[:, :N].float() - ref).abs().max().item()
        assert err <= tol, (o.dtype, err, tol)
