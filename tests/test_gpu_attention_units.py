"""Tensor-core encoder attention at the seams of its kernels: window blocks whose whole window is resident in one
CTA (warps walking the window's 16-row tiles), global blocks on the persistent wgmma kernel (128-row work items,
128-slot key blocks), and the streamed one-tile kernel for windows too large to be resident, each against the
fp32 SIMT kernel."""
import pytest
import torch

from sam_road_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _inputs(B, s, win, heads, hd, seed):
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
    rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    return qkv16, bias, rel_h, rel_w


def _run(lib, simt, B, s, win, heads, hd, qkv16, bias, rel_h, rel_w):
    lib.samroad_debug_force_simt_attention(simt)
    try:
        out = torch.full((B * s * s, heads * hd), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                            B, s, win, heads, hd, out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream), "attention")
        torch.cuda.synchronize()
    finally:
        lib.samroad_debug_force_simt_attention(0)
    return out.float()


@pytest.mark.parametrize("B,s,win,heads,hd", [
    (2, 32, 14, 12, 64),    # full windows of 13 tiles over 5 warps, 14x4 edges (4 tiles), a 4x4 corner (1 tile)
    (2, 25, 14, 12, 64),    # 14x11 edges (10 tiles, the last with 10 rows) and an 11x11 corner; s no multiple of 8
    (2, 28, 14, 16, 80),    # head dim 80: 13 tiles over 4 warps, no edge window
    (1, 64, 14, 12, 64),    # 25 windows per image, 14x8 edges
    (1, 64, 64, 12, 64),    # global with 64-slot key rows: 32 items per head, 32 key blocks, 1 Q / 2 K/V stages
    (2, 9, 9, 12, 64),      # global, 81 queries: one item of 128 rows, 47 never stored; one key block of 144 slots
    (1, 23, 23, 16, 80),    # global at head dim 80: a last item of 17 rows, a last key block of 96 slots
    (1, 17, 14, 1, 64),     # one image, one head: 14x3 and 3x3 windows
    (1, 40, 20, 12, 64),    # a window too large to be resident: streamed, with CTAs past a unit's last tile
    (2, 30, 16, 16, 80),    # resident at head dim 64 only: head dim 80 streams 16x16 windows
    (3, 20, 7, 12, 64),     # 8-slot key rows, 4 tiles per window: one warp of five has no tile
])
def test_attention_units_tc_vs_simt(B, s, win, heads, hd):
    lib = _lib.load()
    x = _inputs(B, s, win, heads, hd, seed=31)
    ref = _run(lib, 1, B, s, win, heads, hd, *x)
    out = _run(lib, 0, B, s, win, heads, hd, *x)
    err = (out - ref).abs().max().item()
    mean_err = (out - ref).abs().mean().item()
    mag = ref.abs().max().item()
    print(f"tc vs simt: max err {err:.3e} mean err {mean_err:.3e} |out|max {mag:.3f}")
    assert torch.isfinite(out).all()
    assert err <= 2.5e-3 * mag and mean_err <= 2e-4 * mag, (err, mean_err, mag)


@pytest.mark.parametrize("B,s,win,heads,hd", [(8, 25, 14, 12, 64), (4, 28, 14, 16, 80)])
def test_attention_units_bitwise_repeatable(B, s, win, heads, hd):
    lib = _lib.load()
    x = _inputs(B, s, win, heads, hd, seed=7)
    first = _run(lib, 0, B, s, win, heads, hd, *x)
    for _ in range(4):
        assert torch.equal(first, _run(lib, 0, B, s, win, heads, hd, *x))
