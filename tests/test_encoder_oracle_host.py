"""CPU: the staged encoder reference (oracle/encoder_oracle.py) is the algorithm of the model oracle.

With fp16=False its stages chained end to end reproduce samroad_oracle.image_encoder (every block's output
and the embeddings) and map_decoder, both in float64, on ViT-B at P = 256 (s = 16: a full window and
partial ones), P = 400 (odd grid) and with LoRA rank 4.  The
model oracle itself is pinned to the unmodified reference by tests/test_oracle_golden.py, so this closes
the chain reference -> fp32 oracle -> staged float64 reference the GPU stage tests compare against.  The
fp16 emulation is checked to move results by fp16 resolution only, and the decoder row order helpers to be
inverse permutations."""
import pytest
import torch

from oracle import encoder_oracle as E
from oracle import samroad_oracle as O
from sam_road_b200 import synth


def _cfg(patch, lora=0):
    return dict(SAM_VERSION="vit_b", PATCH_SIZE=patch, USE_SAM_DECODER=False, ENCODER_LORA=lora > 0,
                LORA_RANK=lora, TOPONET_VERSION="normal", NO_SAM=False)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("patch,lora", [(256, 0), (400, 0), (256, 4)])
def test_stages_chain_to_the_model_oracle(patch, lora):
    cfg = _cfg(patch, lora)
    spec = O.ModelSpec.from_config(cfg)
    sd = {k: v.double() for k, v in synth.make_state_dict(cfg, seed=3).items()}
    rgb = synth.make_tiles(1, patch, seed=5).double()
    with torch.no_grad():
        taps = {}
        feat = O.image_encoder(O.normalize_rgb(rgb), sd, spec, taps)
        logits = O.map_decoder(feat, sd)
        ref = E.EncoderRef(sd, spec)
        mine = {}
        emb, feat16 = ref.encoder(rgb, mine)
        dec = ref.map_decoder(feat16)
    assert _rel(mine["tokens0"], taps["tokens0"]) <= 1e-6
    for i in range(spec.depth):
        assert _rel(mine[f"block{i}"], taps[f"block{i}"]) <= 1e-6, i
    assert _rel(emb, feat) <= 1e-6
    assert torch.equal(feat16.permute(0, 3, 1, 2), emb)        # no rounding with fp16=False
    assert _rel(dec, logits) <= 1e-6


def test_fp16_emulation_moves_results_by_fp16_resolution():
    cfg = _cfg(208)
    spec = O.ModelSpec.from_config(cfg)
    sd = synth.make_state_dict(cfg, seed=4)
    rgb = synth.make_tiles(1, 208, seed=6)
    with torch.no_grad():
        full, half = E.EncoderRef(sd, spec), E.EncoderRef(sd, spec, fp16=True)
        x = full.patch_embed(rgb)
        assert 0 < _rel(half.patch_embed(rgb), x) <= 2e-3
        t_full, t_half = {}, {}
        full.block(x, 0, t_full)
        half.block(x, 0, t_half)
        for k in ("ln1", "qkv", "att", "ln2", "h"):
            v = t_half[k]
            assert torch.equal(v, v.half().double()), k          # stored in fp16
            assert 0 < _rel(v, t_full[k]) <= 2e-2, k
        assert 0 < _rel(t_half["x"], t_full["x"]) <= 2e-3
        emb, f16 = half.neck2(half.neck1(t_half["x"]))
        assert torch.equal(f16, emb.half().double().permute(0, 2, 3, 1))
        d1 = half.dec1(emb)
        assert torch.equal(d1, d1.half().double())
        assert _rel(half.dec3(half.dec2(d1)), full.map_decoder(emb.permute(0, 2, 3, 1))) <= 2e-2


@pytest.mark.parametrize("levels", [1, 2])
def test_quad_rows_round_trip(levels):
    B, s, C = 2, 3, 5
    x = torch.arange(B * C * (s << levels) ** 2, dtype=torch.float64).view(B, C, s << levels, s << levels)
    rows = E.quad_rows(x, levels)
    assert rows.shape == (B * s * s * 4 ** levels, C)
    assert torch.equal(E.from_quad_rows(rows, B, s, levels), x)
    # row ((m * 4 + d1) * 4 + d2) holds pixel (2^L i + sum di_l 2^(L-l), ...) of token m = (b, i, j)
    b, i, j, d = 1, 2, 0, [(1, 0), (0, 1)][:levels]
    m = (b * s + i) * s + j
    r, y, xx = m, i, j
    for di, dj in d:
        r, y, xx = r * 4 + di * 2 + dj, 2 * y + di, 2 * xx + dj
    assert torch.equal(rows[r], x[b, :, y, xx])
