"""The image encoder and the naive map decoder (samroad_encode_masks) stage by stage, against a float64
reference of the same operation.

`samroad_op_encoder_taps` runs samroad_encode_masks and copies chosen intermediates out of the workspace.
Each is compared with oracle/encoder_oracle.py evaluated in float64 on the GPU, with the fp16 rounding of
the CUDA path emulated, and fed from the device's own previous intermediate, so that one stage (one or two
launches) is judged at a time:

    tokens0            im2col + patch-embed GEMM (+ pos_embed)     from the pixels
    ln1                layernorm_f16                               from the block's input X
    qkv                qkv GEMM (fp16 out)                         from the device's ln1
    att                encoder attention                           from the device's qkv
    x_attn             proj GEMM + residual (fp32 out)             from the device's att and X
    ln2                layernorm_f16                               from the device's x_attn
    h                  lin1 GEMM + GELU                            from the device's ln2
    x_lin2, block      lin2 GEMM + residual / the whole block      from the device's h / the previous block
    n1                 fp16(X), neck conv1 + LN2d (gemm_ln)        from the device's last block
    emb, feat16        neck conv3 + LN2d (implicit or im2col)      from the device's n1
    d1                 dec1 + LN2d + GELU (gemm_ln, group 128)     from the device's feat16
    d2                 dec2 + GELU                                 from the device's d1
    logits             dec3 + GELU + dec4 (gemm_dec_final)         from the device's d2
    scores             sigmoid                                     from the device's logits

fp32 stages are judged by max |err| over the reference's RMS per token row (logits: over their span, scores:
absolute).  fp16 stages are judged in units of the fp16 ulp of the reference value (the ulp at RMS / 256 for
smaller values, whose error is set by the row's scale, not their own): the max, and the fraction of elements
more than 1 ulp off.  Stages with the GELU fit (h, d1, d2) get its 6.1e-6 absolute error as an allowance.
The bounds are about 4x the worst error measured on an H100 (DESIGN.md, image encoder stage by stage); the
measured errors go to encoder_stages_report.json in the test report directory.

The shapes are where the kernels branch: s = 12 (one padded window, im2col neck), 13 (odd grid, per-token
dec_final layout), 16 (implicit-conv neck), 25 (odd s * s, partial windows), 32 (the benched shape), 64
(64-slot key rows, one Q stage in the global attention kernel); B = 1, 3 (row tails) and 64.  Models ViT-B, ViT-L, ViT-H (head
dim 80, D = 1280) and LoRA rank 4.  Weight regimes, each aimed at one path (see REGIMES)."""
import ctypes
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import attention_oracle as A  # noqa: E402
from oracle import encoder_oracle as E  # noqa: E402
from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402

DEV = "cuda:0"
GELU_FIT = 6.1e-6          # max abs error of gelu_erf_fast2 (csrc/common.cuh)
# fp32 stages: max |err| / RMS of the reference row (logits: / span; scores: absolute).  fp16 stages:
# (max error in ulp, fraction of elements more than 1 ulp off).  About 4x the worst value measured on an
# H100 80GB HBM3 at 700 W over the cases below (DESIGN.md, "Image encoder, stage by stage").
BOUNDS = {
    "tokens0": 3e-5, "x_attn": 2e-5, "x_lin2": 8e-5, "block": 8e-3, "emb": 4e-5, "logits": 2.5e-4, "scores": 4e-7,
    "ln1": (9, 8e-3), "ln2": (8, 5e-3), "qkv": (8, 1e-4), "att": (1000, 2.6e-3), "h": (4, 1e-5), "n1": (4, 1e-5),
    "feat16": (8, 8e-4), "d1": (4, 1e-5), "d2": (4, 1e-5),
}
# rows at +300 with a variance near 1: the float32 row mean carries an absolute error of ~4e-5, which shifts
# the whole normalised row by that much, i.e. several ulps of its smallest elements (measured 15.5 ulp and
# 1.1 % of the elements; a single-pass variance gives 853 ulp and 89 %)
BOUNDS_BY_REGIME = {"offset_even": {"ln1": (62, 0.045), "ln2": (62, 0.045)}}
# the whole encoder chained in float64 with the fp16 emulation, from the pixels, against the device:
# embeddings over their RMS, logits over their span (test_whole_encoder_against_float64_chain)
BOUNDS_CHAIN = {"emb": 0.075, "logits": 5e-3}

MODELS = {"vit_b": ("vit_b", 0), "vit_l": ("vit_l", 0), "vit_h": ("vit_h", 0), "lora4": ("vit_b", 4)}
# weight regime -> what it changes in synth.make_state_dict's weights; the path it exercises
REGIMES = {
    "default": "none; baseline",
    "peaked": "q and k rows of every qkv.weight x4: softmax across K/V chunks, exp underflow, P rounding",
    "relpos": "rel_pos_h / rel_pos_w ~ N(0, 1): the hi/lo rel-pos split, masked slots of every window",
    "offset": "patch-embed bias +300 on every channel, +500 on one, +100 on another: the fp32 residual at a "
              "large offset, fp16 range of the neck input, LayerNorm rows whose variance two channels set",
    "offset_even": "patch-embed bias +300 on every channel: rows at +300 with a variance near 1, where a "
                   "single-pass E[x^2] - E[x]^2 in float32 loses the variance (two-pass variance of every LayerNorm)",
    "flat": "patch-embed weight, bias and pos_embed x1e-3: block 0's row variances near the 1e-6 eps",
    "widegelu": "lin1 weights x4: GELU arguments past the fit's 5.6 clamp",
    "gain12": "logit_gain = 12: wide decoder logits",
}
CASES = [   # model, P, B, regime, detail blocks (window and global ones of each model)
    ("vit_b", 192, 1, "default", (0, 2)),      # s = 12: one padded window, im2col neck
    ("vit_b", 208, 3, "default", (0,)),        # s = 13: odd grid, per-token dec_final layout, row tails
    ("vit_b", 256, 3, "default", (2,)),        # s = 16: implicit-conv neck
    ("vit_b", 400, 1, "default", (1, 5)),      # s = 25: partial windows, odd s * s
    ("vit_b", 512, 3, "default", (0, 11)),     # the benched shape
    ("vit_b", 1024, 1, "default", (2,)),       # s = 64: 64-slot key rows, 1 Q / 2 K/V stages
    ("vit_b", 400, 3, "peaked", (0, 2)),
    ("vit_b", 1024, 1, "peaked", (8,)),
    ("vit_b", 208, 3, "relpos", (0, 2)),
    ("vit_b", 512, 1, "relpos", (3, 5)),
    ("vit_b", 256, 3, "offset", (0, 2)),
    ("vit_b", 400, 1, "offset", (11,)),
    ("vit_b", 256, 3, "offset_even", (0, 2)),
    ("vit_b", 256, 3, "flat", (0,)),
    ("vit_b", 192, 1, "flat", (0,)),
    ("vit_b", 400, 3, "widegelu", (0, 2)),
    ("vit_b", 208, 3, "gain12", (0,)),
    ("vit_l", 256, 3, "default", (0, 5)),
    ("vit_l", 256, 1, "peaked", (5,)),
    ("vit_h", 256, 1, "default", (0, 7)),
    ("vit_h", 400, 1, "peaked", (7, 8)),
    ("vit_h", 400, 1, "offset", (0,)),
    ("lora4", 256, 3, "default", (0, 2)),
]
_REPORT = {}
_NET = {}


@pytest.fixture(scope="module", autouse=True)
def _report(report_dir):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    with open(os.path.join(report_dir, "encoder_stages_report.json"), "w") as f:
        json.dump(_REPORT, f, indent=1, sort_keys=True)
    _NET.clear()


def _config(model, patch):
    version, lora = MODELS[model]
    return dict(SAM_VERSION=version, PATCH_SIZE=patch, USE_SAM_DECODER=False, ENCODER_LORA=lora > 0,
                LORA_RANK=lora, TOPONET_VERSION="normal", NO_SAM=False)


def _state_dict(cfg, regime):
    sd = synth.make_state_dict(cfg, seed=1, logit_gain=12.0 if regime == "gain12" else 1.0)
    D = O.ModelSpec.from_config(cfg).embed_dim
    if regime == "peaked":
        for k in [k for k in sd if k.endswith("attn.qkv.weight")]:
            sd[k] = torch.cat([sd[k][:2 * D] * 4, sd[k][2 * D:]])
    elif regime == "relpos":
        g = torch.Generator().manual_seed(7)
        for k in [k for k in sd if "rel_pos" in k]:
            sd[k] = torch.randn(sd[k].shape, generator=g)
    elif regime in ("offset", "offset_even"):
        b = sd["image_encoder.patch_embed.proj.bias"] + 300
        if regime == "offset":
            b[5] += 200
            b[9] -= 200
        sd["image_encoder.patch_embed.proj.bias"] = b
    elif regime == "flat":
        for k in ("image_encoder.patch_embed.proj.weight", "image_encoder.patch_embed.proj.bias",
                  "image_encoder.pos_embed"):
            sd[k] = sd[k] * 1e-3
    elif regime == "widegelu":
        for k in [k for k in sd if k.endswith("mlp.lin1.weight")]:
            sd[k] = sd[k] * 4
    return sd


def _net(model, patch, regime="default"):
    """(net, float64 staged reference) on the device; one configuration is kept at a time (ViT-H is large)"""
    key = (model, patch, regime)
    if key not in _NET:
        _NET.clear()
        torch.cuda.empty_cache()
        cfg = _config(model, patch)
        sd = _state_dict(cfg, regime)
        net = SAMRoad(cfg)
        net.load_state_dict(sd, strict=True)
        net.eval()
        net._handle(torch.device(DEV))
        ref = E.EncoderRef({k: v.to(DEV) for k, v in sd.items() if k.startswith(("image_encoder.", "map_decoder."))},
                           O.ModelSpec.from_config(cfg), fp16=True, p_block=_p_block)
        _NET[key] = (net, ref)
    return _NET[key]


def _p_block(s, win, hd):
    """key slots per running-maximum block of the attention kernel that runs (s, win, hd): P rounding as the
    device does it (oracle/attention_oracle.py)"""
    path = _lib.load().samroad_debug_attention_path(s, win, hd, None, None)
    assert path >= 0, _lib.last_error()
    return A.PATH_BLOCK[path]


def _h(net):
    return net._handle(torch.device(DEV))


def _rgb_code(rgb):
    return _lib.U8 if rgb.dtype == torch.uint8 else _lib.F32


def _taps(net, rgb, mask, detail, decoder=True):
    """samroad_op_encoder_taps into NaN-filled buffers; checks that every requested element was written.
    Returns NHWC grids [B, s, s, C] (blocks: {i: grid}), the NCHW embeddings, the decoder rows and the masks."""
    lib = _lib.load()
    B, P = rgb.shape[0], rgb.shape[1]
    s = P // 16
    M, D = B * s * s, net._vit[0]
    nan = float("nan")
    f32 = lambda *shape: torch.full(shape, nan, device=DEV)                          # noqa: E731
    f16 = lambda *shape: torch.full(shape, nan, device=DEV, dtype=torch.float16)     # noqa: E731
    sel = [i for i in range(64) if mask >> i & 1]
    bufs = {"tokens0": f32(M, D), "n1": f16(M, 256), "feat16": f16(M, 256)}
    if sel:
        bufs["blocks"] = f32(len(sel), M, D)
    if detail >= 0:
        bufs.update(ln1=f16(M, D), qkv=f16(M, 3 * D), att=f16(M, D), x_attn=f32(M, D), ln2=f16(M, D),
                    h=f16(M, 4 * D))
    if decoder:
        bufs.update(d1=f16(4 * M, 128), d2=f16(16 * M, 64))
    t = _lib.SamroadEncoderTaps(block_mask=mask, detail_block=detail)
    for k, v in bufs.items():
        setattr(t, k, v.data_ptr())
    emb = f32(B, 256, s, s)
    scores, logits = (f32(B, P, P, 2), f32(B, P, P, 2)) if decoder else (None, None)
    _lib.check(lib.samroad_op_encoder_taps(_h(net), rgb.data_ptr(), _rgb_code(rgb), B, ctypes.byref(t),
                                           _lib.ptr(scores), _lib.ptr(logits), emb.data_ptr(),
                                           _lib.current_stream_ptr()), "samroad_op_encoder_taps")
    torch.cuda.synchronize()
    out = {"emb": emb}
    if decoder:
        out.update(scores=scores, logits=logits)
    for k, v in list(bufs.items()) + list(out.items()):
        assert not torch.isnan(v).any(), f"{k}: {int(torch.isnan(v).sum())} elements never written (or NaN)"
    grid = lambda v: v.view(B, s, s, -1)                                               # noqa: E731
    for k in ("tokens0", "n1", "feat16", "ln1", "qkv", "att", "x_attn", "ln2", "h"):
        if k in bufs:
            out[k] = grid(bufs[k])
    out["blocks"] = {i: grid(bufs["blocks"][j]) for j, i in enumerate(sel)} if sel else {}
    for k in ("d1", "d2"):
        if k in bufs:
            out[k] = bufs[k]
    return out


# ---- metrics -------------------------------------------------------------------------------------------
def _rms(t):
    return t.double().pow(2).mean().sqrt().item()


def _row_err(dev, ref):
    """max over token rows of max |err| / RMS of the reference row"""
    d, r = dev.double().flatten(0, -2), ref.double().flatten(0, -2)
    return ((d - r).abs().amax(-1) / r.pow(2).mean(-1).sqrt()).max().item()


def _ulp_err(dev, ref, gelu=False):
    """(max error in fp16 ulp of the reference, fraction of elements more than 1 ulp off)"""
    d, r = dev.double(), ref.double()
    mag = r.abs().clamp(min=max(_rms(r) / 256, 2.0 ** -14))
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 10)
    err = (d - r).abs()
    if gelu:
        err = (err - GELU_FIT).clamp(min=0)
    e = err / ulp
    return [e.max().item(), (e > 1).double().mean().item()]


def _span(t):
    return (t.max() - t.min()).double().item()


def _judge(tag, errs, regime="default"):
    _REPORT.setdefault("stages", {})[tag] = errs
    print(tag, json.dumps(errs))
    bounds = {**BOUNDS, **BOUNDS_BY_REGIME.get(regime, {})}
    bad = {}
    for k, v in errs.items():
        name = k.split("@")[0]
        if name not in bounds:
            continue
        b = bounds[name]
        ok = (v[0] <= b[0] and v[1] <= b[1]) if isinstance(b, tuple) else v <= b
        if not ok:
            bad[k] = (v, b)
    assert not bad, f"{tag}: stage error over its bound (measured, bound): {bad}"


def _stage_errors(ref, rgb, out, details, sel=None):
    """errors of every tap in `out` against the reference stage fed from the device's previous tap"""
    B = rgb.shape[0]
    s = rgb.shape[1] // 16
    dt = torch.float64
    g = lambda k: out[k].to(dt)                                                # noqa: E731
    errs = {}
    with torch.no_grad():
        errs["tokens0"] = _row_err(out["tokens0"], ref.patch_embed(rgb))
        blocks = out["blocks"]
        for i, x in sorted(blocks.items()):
            x_in = out["tokens0"] if i == 0 else blocks.get(i - 1)
            if x_in is not None:
                errs[f"block@{i}"] = _row_err(x, ref.block(x_in.to(dt), i))
        for i in details:
            x_in = (out["tokens0"] if i == 0 else blocks[i - 1]).to(dt)
            d = out["detail"][i]
            gd = lambda k: d[k].to(dt)                                        # noqa: E731
            errs[f"ln1@{i}"] = _ulp_err(d["ln1"], ref.ln(x_in, i, 1))
            errs[f"qkv@{i}"] = _ulp_err(d["qkv"], ref.qkv(gd("ln1"), i))
            errs[f"att@{i}"] = _ulp_err(d["att"], ref.attention(gd("qkv"), i))
            errs[f"x_attn@{i}"] = _row_err(d["x_attn"], ref.proj(gd("att"), x_in, i))
            errs[f"ln2@{i}"] = _ulp_err(d["ln2"], ref.ln(gd("x_attn"), i, 2))
            errs[f"h@{i}"] = _ulp_err(d["h"], ref.lin1(gd("ln2"), i), gelu=True)
            if i in blocks:
                errs[f"x_lin2@{i}"] = _row_err(blocks[i], ref.lin2(gd("h"), gd("x_attn"), i))
        last = ref.spec.depth - 1
        if last in blocks:
            errs["n1"] = _ulp_err(out["n1"], ref.neck1(blocks[last].to(dt)))
        emb, feat16 = ref.neck2(g("n1"))
        errs["emb"] = _row_err(out["emb"].permute(0, 2, 3, 1), emb.permute(0, 2, 3, 1))
        errs["feat16"] = _ulp_err(out["feat16"], feat16)
        if "d1" in out:
            d1 = ref.dec1(g("feat16").permute(0, 3, 1, 2))
            errs["d1"] = _ulp_err(out["d1"], E.quad_rows(d1, 1), gelu=True)
            d2 = ref.dec2(E.from_quad_rows(g("d1"), B, s, 1))
            errs["d2"] = _ulp_err(out["d2"], E.quad_rows(d2, 2), gelu=True)
            logits = ref.dec3(E.from_quad_rows(g("d2"), B, s, 2)).permute(0, 2, 3, 1)
            errs["logits"] = (out["logits"].double() - logits).abs().max().item() / _span(logits)
            errs["scores"] = (out["scores"].double() - torch.sigmoid(g("logits"))).abs().max().item()
    return errs


def _select(out, sel, B, s):
    """the tiles `sel` of every tap (decoder rows: the tiles' row ranges)"""
    r = {}
    for k, v in out.items():
        if k == "blocks":
            r[k] = {i: x[sel] for i, x in v.items()}
        elif k in ("d1", "d2"):
            n = (4 if k == "d1" else 16) * s * s
            r[k] = v.view(B, n, -1)[sel].reshape(-1, v.shape[-1])
        elif k == "detail":
            r[k] = {i: {kk: x[sel] for kk, x in d.items()} for i, d in v.items()}
        else:
            r[k] = v[sel]
    return r


def _score_std(qkv, heads):
    """std of (q * scale) k^T over the first 1024 tokens of image 0, all heads: how peaked the softmax is"""
    D = qkv.shape[-1] // 3
    hd = D // heads
    t = qkv[0].reshape(-1, 3, heads, hd)[:1024].double()
    q, k = t[:, 0].transpose(0, 1), t[:, 1].transpose(0, 1)
    return ((q @ k.transpose(-2, -1)) * hd ** -0.5).std().item()


def _run_case(net, rgb, details, mask=None, decoder=True):
    depth = net._vit[1]
    mask = (1 << depth) - 1 if mask is None else mask
    out = None
    detail = {}
    for i in details or (-1,):
        o = _taps(net, rgb, mask if out is None else 0, i, decoder)
        if out is None:
            out = o
        elif i >= 0:
            for k in ("emb", "scores", "logits", "tokens0"):
                if k in o:
                    assert torch.equal(o[k], out[k]), f"{k}: not repeatable across calls"
        if i >= 0:
            detail[i] = {k: o[k] for k in ("ln1", "qkv", "att", "x_attn", "ln2", "h")}
    out["detail"] = detail
    return out


# --------------------------------------------------------------------------------------------------
# every stage against float64
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,P,B,regime,details", CASES,
                         ids=[f"{m}-P{p}-B{b}-{r}" for m, p, b, r, _ in CASES])
def test_stages_against_float64(model, P, B, regime, details):
    net, ref = _net(model, P, regime)
    rgb = synth.make_tiles(B, P, seed=P + B).to(DEV)
    out = _run_case(net, rgb, details)
    errs = _stage_errors(ref, rgb, out, details)
    if regime in ("peaked", "default"):
        i = details[0]
        errs["score_std"] = _score_std(out["detail"][i]["qkv"], ref.spec.num_heads)
    _judge(f"{model}_P{P}_B{B}_{regime}", errs, regime)


def test_b64_sparse_block_mask():
    """B = 64 at the benched P = 512 with taps on blocks {0, 2, 11} only: four tiles against the reference
    (tokens0, block 0 and its operands, the neck from block 11, the decoder).  A second call tapping every
    block gives the same bits in the three selected slots."""
    P, B, sel = 512, 64, [0, 21, 42, 63]
    net, ref = _net("vit_b", P)
    rgb = synth.make_tiles(B, P, seed=61).to(DEV)
    mask = 1 | 1 << 2 | 1 << 11
    out = _run_case(net, rgb, (0,), mask=mask)
    assert sorted(out["blocks"]) == [0, 2, 11]
    full = _taps(net, rgb, (1 << 12) - 1, -1, decoder=False)
    for i in (0, 2, 11):
        assert torch.equal(full["blocks"][i], out["blocks"][i]), i
    assert torch.equal(full["emb"], out["emb"])
    del full
    s = P // 16
    out = _select(out, sel, B, s)
    _judge("vit_b_P512_B64_default", _stage_errors(ref, rgb[sel], out, (0,)))


def test_inputs_against_float64():
    """Pixels the normalisation and the patch im2col must take as they come: uint8 tiles all 0 and all 255,
    float32 non-integer pixels including values outside 0..255; and the same tile as uint8 and as float32
    gives bit-identical taps."""
    P = 208
    net, ref = _net("vit_b", P)
    u8 = synth.make_tiles(3, P, seed=71)
    u8[0] = 0
    u8[1] = 255
    g = torch.Generator().manual_seed(72)
    f32 = torch.rand(2, P, P, 3, generator=g) * 340 - 40          # -40 .. 300, not integers
    for tag, rgb in (("u8_const", u8), ("f32_wide", f32)):
        rgb = rgb.to(DEV)
        out = _run_case(net, rgb, (0,))
        _judge(f"vit_b_P{P}_inputs_{tag}", _stage_errors(ref, rgb, out, (0,)))
    a = _run_case(net, u8.to(DEV), (2,))
    b = _run_case(net, u8.float().to(DEV), (2,))
    for k in ("tokens0", "n1", "feat16", "d1", "d2", "emb", "scores", "logits"):
        assert torch.equal(a[k], b[k]), k
    for i in a["blocks"]:
        assert torch.equal(a["blocks"][i], b["blocks"][i]), i
    for k in a["detail"][2]:
        assert torch.equal(a["detail"][2][k], b["detail"][2][k]), k


# --------------------------------------------------------------------------------------------------
# composition
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["default", "peaked"])
def test_whole_encoder_against_float64_chain(regime):
    """the float64 reference chained from the pixels (not fed from the device) against the device's
    embeddings and logits: how far the stage errors carry through 12 blocks, the neck and the decoder"""
    P, B = 512, 3
    net, ref = _net("vit_b", P, regime)
    rgb = synth.make_tiles(B, P, seed=81).to(DEV)
    scores, logits, emb = net._encode(rgb, True)
    torch.cuda.synchronize()
    with torch.no_grad():
        r_emb, r_feat16 = ref.encoder(rgb)
        r_logits = ref.map_decoder(r_feat16).permute(0, 2, 3, 1)
    errs = {"emb": (emb.double() - r_emb).abs().max().item() / _rms(r_emb),
            "logits": (logits.double() - r_logits).abs().max().item() / _span(r_logits)}
    _REPORT.setdefault("chain", {})[f"vit_b_P{P}_B{B}_{regime}"] = errs
    print(regime, json.dumps(errs))
    for k, v in errs.items():
        assert v <= BOUNDS_CHAIN[k], (k, v, BOUNDS_CHAIN[k])


@pytest.mark.parametrize("P,B", [(208, 3), (256, 2)])
def test_taps_do_not_change_the_forward(P, B):
    """With taps set the outputs are those of samroad_encode_masks bit for bit, and both calls (and the hook
    with taps NULL) issue the same number of launches: the copies are no kernels."""
    lib = _lib.load()
    net, _ = _net("vit_b", P)
    rgb = synth.make_tiles(B, P, seed=91).to(DEV)

    def counted(fn):
        lib.samroad_launch_count(1)
        r = fn()
        torch.cuda.synchronize()
        return r, lib.samroad_launch_count(0)

    (sc, lg, em), n_plain = counted(lambda: net._encode(rgb, True))
    out, n_taps = counted(lambda: _taps(net, rgb, (1 << 12) - 1, 2))
    s = P // 16
    em2, sc2, lg2 = (torch.full((B, 256, s, s), float("nan"), device=DEV),
                     torch.full((B, P, P, 2), float("nan"), device=DEV),
                     torch.full((B, P, P, 2), float("nan"), device=DEV))

    def null_taps():
        _lib.check(lib.samroad_op_encoder_taps(_h(net), rgb.data_ptr(), _lib.U8, B, None, sc2.data_ptr(),
                                               lg2.data_ptr(), em2.data_ptr(), _lib.current_stream_ptr()),
                   "samroad_op_encoder_taps")
    _, n_null = counted(null_taps)
    assert n_plain == n_taps == n_null and n_plain > 0, (n_plain, n_taps, n_null)
    for a, b in ((out["emb"], em), (out["scores"], sc), (out["logits"], lg), (em2, em), (sc2, sc), (lg2, lg)):
        assert torch.equal(a, b)


def test_block_index_refusals_then_a_good_call():
    lib = _lib.load()
    P, B = 192, 1
    net, _ = _net("vit_b", P)
    rgb = synth.make_tiles(B, P, seed=95).to(DEV)
    good = _taps(net, rgb, 1, 0)
    emb = torch.full((B, 256, P // 16, P // 16), float("nan"), device=DEV)
    for mask, detail, msg in ((1 << 12, -1, "block_mask"), (1 << 63, -1, "block_mask"), (0, 12, "detail_block=12"),
                              (0, -2, "detail_block=-2")):
        t = _lib.SamroadEncoderTaps(block_mask=mask, detail_block=detail)
        n0 = lib.samroad_launch_count(0)
        rc = lib.samroad_op_encoder_taps(_h(net), rgb.data_ptr(), _lib.U8, B, ctypes.byref(t), None, None,
                                         emb.data_ptr(), _lib.current_stream_ptr())
        assert rc != 0 and msg in _lib.last_error(), (rc, _lib.last_error())
        assert lib.samroad_launch_count(0) == n0          # refused before any launch
    assert torch.isnan(emb).all()
    again = _taps(net, rgb, 1, 0)
    for k in ("tokens0", "ln1", "h", "emb", "logits"):
        assert torch.equal(again[k], good[k]), k
