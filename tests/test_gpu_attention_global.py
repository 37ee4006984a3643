"""Global attention blocks (window = grid) on the persistent wgmma kernel at batch sizes where every CTA walks
several work items (image, head, 128 query rows): item to item hand-over of the Q and K/V rings, and item tails
that meet partial 128-slot key blocks, each against the fp32 SIMT kernel; and bitwise repeatability."""
import pytest
import torch

from sam_road_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, s, heads, hd, seed):
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
    rel_h = (0.3 * torch.randn(2 * s - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * s - 1, hd, generator=g)).to(DEV)
    return qkv16, bias, rel_h, rel_w


def _run(lib, simt, B, s, heads, hd, qkv16, bias, rel_h, rel_w):
    lib.samroad_debug_force_simt_attention(simt)
    try:
        out = torch.full((B * s * s, heads * hd), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                            B, s, s, heads, hd, out.data_ptr(), _st()), "attention")
        torch.cuda.synchronize()
    finally:
        lib.samroad_debug_force_simt_attention(0)
    return out


@pytest.mark.parametrize("B,s,heads,hd", [
    (64, 32, 12, 64),    # ViT-B @512: 8 items per unit, 8 whole key blocks
    (64, 16, 16, 80),    # ViT-H @256: 2 items per unit, 16-column tail boxes
    (64, 23, 12, 64),    # 529 queries: a last item of 17 rows; 736 key slots: a last key block of 96
])
def test_attention_global_many_items_tc_vs_simt(B, s, heads, hd):
    lib = _lib.load()
    x = _inputs(B, s, heads, hd, seed=31)
    ref = _run(lib, 1, B, s, heads, hd, *x).float()
    out = _run(lib, 0, B, s, heads, hd, *x).float()
    err = (out - ref).abs().max().item()
    mean_err = (out - ref).abs().mean().item()
    mag = ref.abs().max().item()
    print(f"tc vs simt: max err {err:.3e} mean err {mean_err:.3e} |out|max {mag:.3f}")
    assert torch.isfinite(out).all()
    assert err <= 2.5e-3 * mag and mean_err <= 2e-4 * mag, (err, mean_err, mag)


def test_attention_global_many_items_bitwise_repeatable():
    B, s, heads, hd = 64, 32, 12, 64
    lib = _lib.load()
    x = _inputs(B, s, heads, hd, seed=7)
    a = _run(lib, 0, B, s, heads, hd, *x)
    b = _run(lib, 0, B, s, heads, hd, *x)
    assert torch.equal(a, b)
