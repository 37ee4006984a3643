"""CPU: the float64 SAM-decoder reference that tests/test_gpu_sam_decoder.py judges the device against.

* With the fp16 rounding emulation off it is the plain oracle, bit for bit, and its stage functions
  (hypernetworks, low_res_masks, upsample_masks) compose to exactly the whole forward.
* In float64 it agrees with the float32 model oracle, and with the goldens of the unmodified reference
  (vitb_256_samdec, vitb_192_samdec), to float32 rounding.
* The emulation changes the result at fp16 level, not more."""
import os

import numpy as np
import pytest
import torch

from oracle import samroad_oracle as O
from oracle import sam_decoder_oracle as SD
from sam_road_b200 import synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5      # tests/test_oracle_golden.py


def _cfg(patch):
    return dict(SAM_VERSION="vit_b", PATCH_SIZE=patch, USE_SAM_DECODER=True, ENCODER_LORA=False, LORA_RANK=0,
                TOPONET_VERSION="normal", NO_SAM=False)


def _span(t):
    return (t.max() - t.min()).item()


@pytest.mark.parametrize("name,patch", [("vitb_256_samdec", 256), ("vitb_192_samdec", 192)])
def test_float64_decoder_against_float32_oracle_and_golden(name, patch):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    seed = int(g["seed"])
    cfg = _cfg(patch)
    sd = synth.make_state_dict(cfg, seed=seed)
    spec = O.ModelSpec.from_config(cfg)
    rgb = synth.make_tiles(1, patch, seed=seed + 21, dtype=torch.float32)
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    with torch.no_grad():
        _, feat, logits32 = O.infer_masks_and_img_features(sd, spec, rgb, return_logits=True)
        sd64 = {k: v.double() for k, v in sd.items()}
        logits64 = SD.sam_mask_logits(feat.double(), sd64, spec).permute(0, 2, 3, 1)
    assert logits64.dtype == torch.float64
    # float32 rounding of ~0.5-valued logits after two transformer layers: a few hundred fp32 ulps at most
    err32 = (logits64 - logits32.double()).abs().max().item()
    assert err32 <= 2e-6, err32
    assert np.abs(logits64[0, ::8, ::8, :].numpy() - g["mask_logits_sub"]).max() < TOL
    # the float64 forward is not the float32 one evaluated again
    assert err32 > 0


def test_emulation_off_is_the_plain_oracle_and_stages_compose():
    cfg = _cfg(192)
    sd = {k: v.double() for k, v in synth.make_state_dict(cfg, seed=4).items()}
    spec = O.ModelSpec.from_config(cfg)
    gen = torch.Generator().manual_seed(5)
    feat = torch.randn(2, 256, 12, 12, generator=gen, dtype=torch.float64)
    with torch.no_grad():
        plain = SD.sam_mask_logits(feat, sd, spec)
        off = SD.sam_mask_logits(feat, sd, spec, fp16=False)
        q, k, hyper, low = SD.sam_low_res_masks(feat, sd, fp16=False, checkpoints=True)
        assert torch.equal(off, plain)
        assert torch.equal(SD.upsample_masks(low, 192), plain)
        assert q.shape == (2, 4, 256) and k.shape == (2, 144, 256) and hyper.shape == (2, 2, 32)
        # the stages the GPU test feeds from device checkpoints reproduce the whole forward bit for bit
        assert torch.equal(SD.hypernetworks(sd, q)[:, 1:], hyper)
        assert torch.equal(SD.low_res_masks(sd, k, hyper, 12, 12), low)

        q16, k16, hyper16, low16 = SD.sam_low_res_masks(feat, sd, fp16=True, checkpoints=True)
    # fp16 operands move every stage, by about fp16 resolution relative to its scale
    for a, b in ((q16, q), (k16, k), (hyper16, hyper), (low16, low)):
        rel = ((a - b).abs().max() / b.pow(2).mean().sqrt()).item()
        assert 1e-5 < rel < 2e-2, rel
    # the token side stays in full precision: with fp16 keys fed in, the hypernetworks are exact
    assert torch.equal(SD.hypernetworks(sd, q16)[:, 1:], hyper16)


def test_dense_pe_dtype():
    cfg = _cfg(256)
    sd = synth.make_state_dict(cfg, seed=0)
    pe32 = SD.dense_pe(sd, 16, 16)
    pe64 = SD.dense_pe({k: v.double() for k, v in sd.items()}, 16, 16, torch.float64)
    assert pe32.dtype == torch.float32 and pe64.dtype == torch.float64 and pe64.shape == (1, 256, 16, 16)
    assert (pe64 - pe32.double()).abs().max().item() < 1e-5
    # channel k < 128 is sin(2 pi (x G[0,k] + y G[1,k])) at the pixel centre (x, y) in [-1, 1]
    G = sd["prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"].double()
    yy, xx = 3, 11
    cx, cy = 2 * (xx + 0.5) / 16 - 1, 2 * (yy + 0.5) / 16 - 1
    want = torch.sin(2 * np.pi * (cx * G[0] + cy * G[1]))
    assert torch.allclose(pe64[0, :128, yy, xx], want, rtol=0, atol=1e-12)
