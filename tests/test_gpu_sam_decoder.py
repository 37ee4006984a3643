"""The SAM mask decoder (USE_SAM_DECODER: True, csrc/sam_decoder.cu) stage by stage, against a float64
reference of the same operation.

`samroad_op_sam_decoder` runs the decoder alone on given embeddings and returns four of its intermediates
next to the masks.  Each is compared with oracle/sam_decoder_oracle.py evaluated in float64 on the GPU,
with the fp16 rounding of the CUDA path emulated, and fed from the device's previous checkpoint so that one
stage is judged at a time:

    queries, keys   two-way transformer        from the input embeddings
    hyper           hypernetworks              from the device's queries
    lowres          upscaler . hyper           from the device's keys and hyper
    logits          x4 bilinear                from the device's lowres
    scores          sigmoid                    from the device's logits

Errors are relative to the reference's RMS (queries, keys, hyper) or span (lowres, logits); scores are
absolute.  The bounds are about 4x the worst error measured on an H100 (DESIGN.md, SAM decoder); the
measured errors go to sam_decoder_report.json in the test report directory.

The shapes are those the kernels treat specially: T = 1, fewer keys than the 64 softmax partitions of the
token->image attention (T = 9, 49), one key per partition (T = 64), odd grids, T = 4096 (P = 1024), token
batches 4B that leave a partial 32-row tile of the token GEMMs (B = 5, 9) and the benched B = 64.  Inputs
stress the softmax: embeddings x8, one token far larger than the rest (one partition carries the softmax,
the others underflow) and embeddings constant over the tokens (equal V rows).  Weights are the default
synthetic ones, logit_gain = 12 (wide logits) and token LayerNorms scaled to small outputs (their eps matters).

The last tests run the decoder inside the model: the hook composes with samroad_encode_masks bit for bit,
the archived decoder configurations agree with the fp32 model oracle, and the scene path equals the tile
path."""
import copy
import ctypes
import json
import os
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import samroad_oracle as O  # noqa: E402
from oracle import sam_decoder_oracle as SD  # noqa: E402
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402

DEV = "cuda:0"
# max error of each checkpoint over the reference's RMS (queries, keys, hyper), over its span (lowres,
# logits), and absolute (scores).  About 4x the worst error measured on an H100 80GB HBM3 at 700 W over the
# 20 stage cases below: queries 1.1e-4 (P = 16), keys 1.7e-4, hyper 1.8e-6, lowres 3.8e-4, logits 6.8e-8,
# scores 8.5e-8.
BOUNDS = {"queries": 4e-4, "keys": 7e-4, "hyper": 7e-6, "lowres": 1.5e-3, "logits": 2.5e-7, "scores": 3.5e-7}
# model logits against the fp32 oracle, relative to their span under logit_gain = 12 (as
# test_gpu_model.py::test_parity_with_wide_logits); measured at most 5.3e-4 on the same card
TOL_MODEL = 2e-3
# weight variants: logit_gain = 12 widens the logits; "small_ln" scales the token-side LayerNorm weights and
# biases (norm1-3 of both layers, norm_final_attn) by 0.03, so that those LayerNorms see variances of ~1e-3
# and their eps matters
WEIGHTS = {"default": (1.0, 1.0), "gain12": (12.0, 1.0), "small_ln": (1.0, 0.03)}
_TOKEN_LN = re.compile(r"mask_decoder\.transformer\.(layers\.\d\.norm[123]|norm_final_attn)\.")
CHECKPOINTS = ("queries", "keys", "hyper", "lowres", "scores", "logits")
_REPORT = {}
_NETS = {}


@pytest.fixture(scope="module", autouse=True)
def _report(report_dir):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    with open(os.path.join(report_dir, "sam_decoder_report.json"), "w") as f:
        json.dump(_REPORT, f, indent=1, sort_keys=True)
    _NETS.clear()


def _config(patch, lora=0):
    return dict(SAM_VERSION="vit_b", PATCH_SIZE=patch, USE_SAM_DECODER=True, ENCODER_LORA=lora > 0,
                LORA_RANK=lora, TOPONET_VERSION="normal", NO_SAM=False)


def _net(patch, weights="default", lora=0):
    """(net, float32 state_dict, float64 decoder state_dict) on the device; one handle per configuration."""
    key = (patch, weights, lora)
    if key not in _NETS:
        cfg = _config(patch, lora)
        gain, ln = WEIGHTS[weights]
        sd = synth.make_state_dict(cfg, seed=1, logit_gain=gain)
        sd = {k: v * ln if _TOKEN_LN.match(k) else v for k, v in sd.items()}
        net = SAMRoad(cfg)
        net.load_state_dict(sd, strict=True)
        net.eval()
        net._handle(torch.device(DEV))
        sd64 = {k: v.to(DEV, torch.float64) for k, v in sd.items()
                if k.startswith(("mask_decoder.", "prompt_encoder."))}
        _NETS[key] = (net, sd, sd64)
    return _NETS[key]


def _h(net):
    return net._handle(torch.device(DEV))


def _shapes(B, P):
    s = P // 16
    return {"queries": (B, 4, 256), "keys": (B, s * s, 256), "hyper": (B, 2, 32), "lowres": (B, 4 * s, 4 * s, 2),
            "scores": (B, P, P, 2), "logits": (B, P, P, 2)}


_GUARD = 256     # NaN elements after every output: nothing may be written past its end


def _decode(net, emb, want=CHECKPOINTS):
    """samroad_op_sam_decoder into NaN-filled outputs (NULL for those not in `want`); checks that every
    element of every requested output was written and that nothing was written past its end."""
    lib = _lib.load()
    B, P = emb.shape[0], emb.shape[2] * 16
    bufs, out = {}, {}
    for name, shape in _shapes(B, P).items():
        if name in want:
            n = 1
            for d in shape:
                n *= d
            bufs[name] = torch.full((n + _GUARD,), float("nan"), device=DEV)
            out[name] = bufs[name][:n].view(shape)
    p = lambda n: bufs[n].data_ptr() if n in bufs else None    # noqa: E731
    _lib.check(lib.samroad_op_sam_decoder(_h(net), emb.data_ptr(), B, p("queries"), p("keys"), p("hyper"),
                                          p("lowres"), p("scores"), p("logits"), _lib.current_stream_ptr()),
               "samroad_op_sam_decoder")
    torch.cuda.synchronize()
    for name, t in out.items():
        assert not torch.isnan(t).any(), f"{name}: {int(torch.isnan(t).sum())} elements never written"
        assert torch.isnan(bufs[name][t.numel():]).all(), f"{name}: written past its end"
    return out


def _embeddings(B, P, kind, seed):
    s = P // 16
    g = torch.Generator().manual_seed(seed)
    if kind == "const":        # the same vector at every token: the V rows of token->image are equal
        e = torch.randn(B, 256, 1, 1, generator=g).expand(B, 256, s, s)
    else:
        e = torch.randn(B, 256, s, s, generator=g)
    if kind == "x8":
        e = 8 * e
    if kind == "spike":        # one token 200x the rest: its score dominates its partition by far more
        t = (s * s) // 3       # than exp can resolve in fp32, in every head where it is positive
        e[:, :, t // s, t % s] *= 200
    return e.contiguous().to(DEV)


def _rms(t):
    return t.double().pow(2).mean().sqrt().item()


def _span(t):
    return (t.max() - t.min()).double().item()


def _stage_errors(sd64, emb, out, P):
    """error of each device checkpoint against the float64 reference fed from the previous checkpoint"""
    s = P // 16
    with torch.no_grad():
        q_ref, k_ref, _, _ = SD.sam_low_res_masks(emb.double(), sd64, fp16=True, checkpoints=True)
        hyper_ref = SD.hypernetworks(sd64, out["queries"].double())[:, 1:]
        low_ref = SD.low_res_masks(sd64, out["keys"].double(), out["hyper"].double(), s, s, fp16=True)
        low_ref = low_ref.permute(0, 2, 3, 1)
        logit_ref = SD.upsample_masks(out["lowres"].double().permute(0, 3, 1, 2), P).permute(0, 2, 3, 1)
        score_ref = torch.sigmoid(out["logits"].double())
    err = lambda a, r: (a.double() - r).abs().max().item()    # noqa: E731
    return {"queries": err(out["queries"], q_ref) / _rms(q_ref),
            "keys": err(out["keys"], k_ref) / _rms(k_ref),
            "hyper": err(out["hyper"], hyper_ref) / _rms(hyper_ref),
            "lowres": err(out["lowres"], low_ref) / _span(low_ref),
            "logits": err(out["logits"], logit_ref) / _span(logit_ref),
            "scores": err(out["scores"], score_ref)}


def _check_stages(tag, errs):
    _REPORT.setdefault("stages", {})[tag] = errs
    print(tag, json.dumps(errs))
    bad = {k: (v, BOUNDS[k]) for k, v in errs.items() if not v <= BOUNDS[k]}
    assert not bad, f"{tag}: stage error over its bound (measured, bound): {bad}"


# --------------------------------------------------------------------------------------------------
# the decoder alone, stage by stage
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,B,weights,kind", [
    (16, 3, "default", "randn"),      # T = 1: 63 of 64 partitions empty
    (48, 3, "default", "randn"),      # T = 9
    (112, 1, "default", "randn"),     # T = 49 < 64 partitions, one image
    (112, 5, "default", "randn"),     # 4B = 20: one partial token-GEMM row tile
    (128, 3, "default", "randn"),     # T = 64: one key per partition
    (144, 9, "default", "randn"),     # 4B = 36: a full and a partial row tile
    (256, 3, "default", "randn"),
    (400, 2, "default", "randn"),     # s = 25: odd grid
    (400, 3, "gain12", "randn"),      # wide logits
    (1024, 1, "gain12", "randn"),     # T = 4096 (finetune_enc_dec_1024)
    (256, 64, "default", "randn"),    # the benched batch: Bt = 256 token rows, dim3(64, 8) attention CTAs
    (512, 64, "gain12", "randn"),     # B = 64 at P = 512: four images against the reference, all finite
    (112, 3, "default", "x8"),
    (256, 3, "default", "x8"),
    (128, 3, "default", "spike"),
    (1024, 1, "gain12", "spike"),
    (112, 3, "default", "const"),
    (256, 3, "default", "const"),
    (112, 3, "small_ln", "randn"),
    (256, 3, "small_ln", "spike"),
])
def test_stages_against_float64(P, B, weights, kind):
    net, _, sd64 = _net(P, weights)
    emb = _embeddings(B, P, kind, seed=P + B)
    out = _decode(net, emb)
    for name in CHECKPOINTS:
        assert torch.isfinite(out[name]).all(), name
    if B > 8 and P >= 512:
        sel = [0, 21, 42, 63]
        out = {k: v[sel] for k, v in out.items()}
        emb = emb[sel]
    _check_stages(f"P{P}_B{B}_{weights}_{kind}", _stage_errors(sd64, emb, out, P))


def test_partial_outputs_and_batch_permutation():
    """scores-only, logits-only and checkpoint-free calls give the bits of the full call; permuting the
    batch permutes every checkpoint bit for bit."""
    P, B = 144, 9
    net, _, _ = _net(P)
    emb = _embeddings(B, P, "randn", seed=3)
    full = _decode(net, emb)
    assert torch.equal(_decode(net, emb, ("scores",))["scores"], full["scores"])
    assert torch.equal(_decode(net, emb, ("logits",))["logits"], full["logits"])
    part = _decode(net, emb, ("keys", "scores", "logits"))
    assert torch.equal(part["keys"], full["keys"]) and torch.equal(part["logits"], full["logits"])
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(0)).to(DEV)
    permuted = _decode(net, emb[perm].contiguous())
    for name in CHECKPOINTS:
        assert torch.equal(permuted[name], full[name][perm]), name


def test_b64_against_b4_calls_and_handle_reuse():
    """A B = 64 call against 16 calls of B = 4 (within the stage bounds; whether they are bit-equal is
    reported); two identical calls are bit-equal; a handle going B = 64 -> 1 -> 64 gives the results of
    fresh handles."""
    P = 256
    net, _, _ = _net(P)
    emb = _embeddings(64, P, "randn", seed=11)
    r64 = _decode(net, emb)
    r4 = [_decode(net, emb[i:i + 4].contiguous()) for i in range(0, 64, 4)]
    cat = {k: torch.cat([r[k] for r in r4]) for k in CHECKPOINTS}
    scale = {"queries": _rms, "keys": _rms, "hyper": _rms, "lowres": _span, "logits": _span,
             "scores": lambda t: 1.0}
    diff = {k: (r64[k] - cat[k]).abs().max().item() / scale[k](r64[k]) for k in CHECKPOINTS}
    rep = {"b64_vs_16xb4": diff, "bit_equal": {k: torch.equal(r64[k], cat[k]) for k in CHECKPOINTS}}
    _REPORT["b64_vs_b4"] = rep
    print(json.dumps(rep))
    for k in CHECKPOINTS:
        assert diff[k] <= BOUNDS[k], (k, diff[k])

    r64b = _decode(net, emb)                       # same handle, same call
    r1 = _decode(net, emb[5:6].contiguous())       # the workspace is grown for 64 and reused for 1
    r64c = _decode(net, emb)
    fresh1 = copy.deepcopy(net)                    # a copy owns a handle of its own, created on first use
    f1 = _decode(fresh1, emb[5:6].contiguous())
    fresh64 = copy.deepcopy(net)
    f64 = _decode(fresh64, emb)
    for k in CHECKPOINTS:
        assert torch.equal(r64b[k], r64[k]) and torch.equal(r64c[k], r64[k]), k
        assert torch.equal(f64[k], r64[k]) and torch.equal(r1[k], f1[k]), k


def test_refusals_then_a_good_call():
    lib = _lib.load()
    P = 128
    net, _, _ = _net(P)
    emb = _embeddings(2, P, "randn", seed=5)
    good = _decode(net, emb)

    def expect_refusal(h, e, B, scores, logits, msg):
        n0 = lib.samroad_launch_count(0)
        rc = lib.samroad_op_sam_decoder(h, e, B, None, None, None, None, scores, logits,
                                        _lib.current_stream_ptr())
        assert rc != 0 and msg in _lib.last_error(), (rc, _lib.last_error())
        assert lib.samroad_launch_count(0) == n0          # refused before any launch
        again = _decode(net, emb)
        for k in CHECKPOINTS:
            assert torch.equal(again[k], good[k]), k

    out = torch.full((2, P, P, 2), float("nan"), device=DEV)
    for use_dec, msg in ((0, "no SAM mask decoder"), (1, "not finalized")):
        cfg = _lib.SamRoadCfg()
        cfg.patch_size, cfg.embed_dim, cfg.depth, cfg.num_heads, cfg.window_size = P, 768, 12, 12, 14
        for i, g in enumerate((2, 5, 8, 11)):
            cfg.global_attn_indexes[i] = g
        cfg.use_sam_decoder = use_dec
        other = _lib.Handle("samroad_create", "samroad_destroy", ctypes.byref(cfg), 0)
        expect_refusal(other, emb.data_ptr(), 2, out.data_ptr(), None, msg)
        other.close()
    h = _h(net)
    expect_refusal(h, None, 2, out.data_ptr(), None, "null emb_nchw")
    expect_refusal(h, emb.data_ptr(), 0, out.data_ptr(), None, "B=0")
    expect_refusal(h, emb.data_ptr(), -1, out.data_ptr(), None, "B=-1")
    expect_refusal(h, emb.data_ptr(), 2, None, None, "both null")
    assert torch.isnan(out).all()


# --------------------------------------------------------------------------------------------------
# the decoder inside the model
# --------------------------------------------------------------------------------------------------
def test_composition_with_encode_masks():
    """samroad_encode_masks = encoder, then exactly the decoder the hook runs on the embeddings it returned"""
    P, B = 400, 3
    net, _, _ = _net(P, "gain12")
    rgb = synth.make_tiles(B, P, seed=31).to(DEV)
    scores, logits, emb = net._encode(rgb, True)
    torch.cuda.synchronize()
    out = _decode(net, emb, ("scores", "logits"))
    assert torch.equal(out["logits"], logits) and torch.equal(out["scores"], scores)


def _model_parity(tag, net, sd, rgb, sel=None):
    cfg = net.config
    spec = O.ModelSpec.from_config(cfg)
    full = net._encode(rgb, True)[1]
    logits = full
    if sel is not None:
        logits, rgb = full[sel], rgb[sel]
    with torch.no_grad():
        o_logits = O.infer_masks_and_img_features({k: v.to(DEV) for k, v in sd.items()}, spec, rgb.float(),
                                                  return_logits=True)[2]
    span = _span(o_logits)
    em = (logits - o_logits).abs().max().item()
    _REPORT.setdefault("model", {})[tag] = {"mask_logit_maxabs": em, "mask_logit_span": span}
    print(tag, em, span)
    assert torch.isfinite(logits).all()
    assert em <= TOL_MODEL * span, (em, span)
    return full


def test_archived_vitb_512_b64_with_permutation():
    net, sd, _ = _net(512, "gain12")
    B, sel = 64, [0, 21, 42, 63]
    rgb = synth.make_tiles(B, 512, seed=41).to(DEV)
    logits = _model_parity("vitb_512_samdec_b64", net, sd, rgb, sel)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1)).to(DEV)
    assert torch.equal(net._encode(rgb[perm].contiguous(), True)[1], logits[perm])


@pytest.mark.parametrize("patch,lora", [(1024, 0), (512, 8), (512, 16)])
def test_archived_configs_against_fp32_oracle(patch, lora):
    net, sd, _ = _net(patch, "gain12", lora)
    rgb = synth.make_tiles(1 if patch == 1024 else 2, patch, seed=43).to(DEV)
    _model_parity(f"vitb_{patch}_samdec_lora{lora}", net, sd, rgb)


def test_scene_path_with_decoder():
    P = 256
    net, _, _ = _net(P)
    scene = synth.make_tiles(1, 640, seed=45)[0].to(DEV).contiguous()
    xy = torch.tensor([[0, 0], [384, 0], [100, 384], [384, 384], [17, 211]], dtype=torch.int32)
    scores, emb = net.infer_masks_and_img_features_scene(scene, xy)
    tiles = torch.stack([scene[y:y + P, x:x + P] for x, y in xy.tolist()]).contiguous()
    t_scores, t_emb = net.infer_masks_and_img_features(tiles)
    assert torch.equal(scores, t_scores) and torch.equal(emb, t_emb)
