"""Tensor-core encoder attention at tile boundaries of its layout (key rows padded to a power of two,
64-slot chunks whose upper half may hold no key, 16-row tiles of a window's real queries), and the
accuracy of its tensor-core rel-pos terms, each against the fp32 SIMT kernel."""
import pytest
import torch

from sam_road_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, s, win, heads, hd, seed, rel_sigma=0.3):
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
    rel_h = (rel_sigma * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (rel_sigma * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    return qkv16, bias, rel_h, rel_w


def _run(lib, simt, B, s, win, heads, hd, qkv16, bias, rel_h, rel_w):
    lib.samroad_debug_force_simt_attention(simt)
    try:
        out = torch.full((B * s * s, heads * hd), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                            B, s, win, heads, hd, out.data_ptr(), _st()), "attention")
        torch.cuda.synchronize()
    finally:
        lib.samroad_debug_force_simt_attention(0)
    return out.float()


@pytest.mark.parametrize("B,s,win,heads,hd", [
    (2, 25, 25, 12, 64),    # global, key rows padded 25 -> 32, last chunk half empty
    (2, 20, 20, 16, 80),    # global, padded key rows, whole chunks
    (3, 12, 14, 12, 64),    # one window larger than the grid: 144 real queries = 9 row tiles
    (4, 3, 3, 12, 64),      # 8-slot key rows, one half chunk
    (2, 5, 5, 16, 80),      # 8-slot key rows, one full chunk
    (1, 40, 40, 12, 64),    # global, 64-slot key rows
    (2, 48, 14, 16, 80),    # windows with 6-token edges
])
def test_attention_tile_boundaries_tc_vs_simt(B, s, win, heads, hd):
    lib = _lib.load()
    x = _inputs(B, s, win, heads, hd, seed=21)
    ref = _run(lib, 1, B, s, win, heads, hd, *x)
    out = _run(lib, 0, B, s, win, heads, hd, *x)
    err = (out - ref).abs().max().item()
    mean_err = (out - ref).abs().mean().item()
    mag = ref.abs().max().item()
    print(f"tc vs simt: max err {err:.3e} mean err {mean_err:.3e} |out|max {mag:.3f}")
    assert torch.isfinite(out).all()
    assert err <= 2.5e-3 * mag and mean_err <= 2e-4 * mag, (err, mean_err, mag)


@pytest.mark.parametrize("B,s,win,heads,hd", [(2, 16, 16, 12, 64), (2, 16, 16, 16, 80), (2, 32, 14, 12, 64)])
def test_attention_relpos_accuracy(B, s, win, heads, hd):
    """Rel-pos tables 10x the usual scale: rounding them to a single fp16 table moves the output by
    about 7e-3 of its magnitude (float64 evaluation of the reference math); the hi + lo split keeps
    the tensor-core kernel within 1.5e-3 of the fp32 SIMT kernel."""
    lib = _lib.load()
    x = _inputs(B, s, win, heads, hd, seed=3, rel_sigma=3.0)
    ref = _run(lib, 1, B, s, win, heads, hd, *x)
    out = _run(lib, 0, B, s, win, heads, hd, *x)
    err = (out - ref).abs().max().item()
    mag = ref.abs().max().item()
    print(f"rel-pos x10: max err {err:.3e} |out|max {mag:.3f}")
    assert torch.isfinite(out).all()
    assert err <= 1.5e-3 * mag, (err, mag)


def test_attention_determinism_padded_key_rows():
    B, s, win, heads, hd = 16, 25, 25, 12, 64
    lib = _lib.load()
    x = _inputs(B, s, win, heads, hd, seed=5)
    first = _run(lib, 0, B, s, win, heads, hd, *x)
    for _ in range(8):
        assert torch.equal(first, _run(lib, 0, B, s, win, heads, hd, *x))
