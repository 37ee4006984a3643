"""CPU: the float64 attention reference (oracle/attention_oracle.py) is the attention of the model oracle, its
block-wise P rounding reduces to the "P against the row maximum" rule when one block holds every key, and the
analytic inputs of tests/test_gpu_attention_float64.py give the outputs they are built to give."""
import pytest
import torch

from oracle import attention_oracle as A
from oracle import samroad_oracle as O


def _inputs(B, s, win, heads, hd, seed):
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float()
    rel_h = 0.3 * torch.randn(2 * win - 1, hd, generator=g)
    rel_w = 0.3 * torch.randn(2 * win - 1, hd, generator=g)
    return qkv16, bias, rel_h, rel_w


def _model_oracle(qkv16, bias, rel_h, rel_w, B, s, win, heads):
    """samroad_oracle.attention_core in float32 on the windows of a grid padded with fp16(bias) tokens"""
    nwin = -(-s // win)
    x = bias.to(torch.float16).float().expand(B, nwin * win, nwin * win, bias.numel()).clone()
    x[:, :s, :s] = qkv16.float().view(B, s, s, -1)
    wins, padded = O.window_split(x, win)
    out = O.attention_core(wins, rel_h, rel_w, heads)
    return O.window_merge(out, win, padded, (s, s)).reshape(B * s * s, -1)


@pytest.mark.parametrize("B,s,win,heads,hd", [
    (2, 9, 9, 2, 64),       # global
    (1, 12, 12, 1, 80),     # global, head dim 80
    (2, 16, 8, 2, 64),      # whole windows
    (1, 13, 5, 2, 64),      # partial windows at the right and bottom edges
    (2, 12, 14, 2, 80),     # one window larger than the grid
])
def test_exact_is_the_model_attention(B, s, win, heads, hd):
    x = _inputs(B, s, win, heads, hd, seed=s + win)
    ref = A.attention(*x, B, s, win, heads, hd)
    model = _model_oracle(*x, B, s, win, heads)
    err = ((ref["exact"] - model.double()).abs().max() / model.abs().max()).item()
    assert err <= 1e-6, err
    assert torch.equal(ref["exact"], ref["emulated"])          # block=None: the SIMT kernel, P unrounded


def _global_max_rule(scores, v):
    """EncoderRef's former rule: P = fp16(exp(S - max_row S)), l sums the rounded P"""
    pr = torch.exp(scores - scores.amax(-1, keepdim=True)).to(torch.float16).double()
    return (pr @ v) / pr.sum(-1, keepdim=True)


def test_one_block_is_the_global_max_rule():
    g = torch.Generator().manual_seed(1)
    scores = torch.randn(3, 40, 70, generator=g, dtype=torch.float64) * 6
    scores[:, :, 60:] = float("-inf")
    v = torch.randn(3, 70, 16, generator=g, dtype=torch.float64)
    one = torch.zeros(70, dtype=torch.long)
    assert torch.equal(A.softmax_pv(scores, v, one), _global_max_rule(scores, v))
    # through the whole reference: a block of at least win * winP slots
    B, s, heads, hd = 1, 11, 2, 64
    x = _inputs(B, s, s, heads, hd, seed=2)
    big = A.attention(*x, B, s, s, heads, hd, block=s * A.win_pitch(s))
    per_key = A.attention(*x, B, s, s, heads, hd, block=1 << 20)
    assert torch.equal(big["emulated"], per_key["emulated"])
    assert not torch.equal(big["emulated"], big["exact"])
    # and the rule itself: restated from the scores of `exact`
    qkv16, bias, rel_h, rel_w = x
    q, k, v = qkv16.double().view(s * s, 3, heads, hd).permute(1, 2, 0, 3)   # each [heads, L, hd]
    Rh, Rw = A._gather(rel_h.double(), s), A._gather(rel_w.double(), s)
    qg = q.reshape(heads, s, s, hd)
    sc = (hd ** -0.5 * q @ k.transpose(-2, -1)).view(heads, s, s, s, s)
    sc = sc + torch.einsum("ahwc,hkc->ahwk", qg, Rh)[..., :, None] + torch.einsum("ahwc,wkc->ahwk", qg, Rw)[..., None, :]
    want = _global_max_rule(sc.view(heads, s * s, s * s), v).transpose(0, 1).reshape(s * s, -1)
    assert (big["emulated"] - want).abs().max().item() <= 1e-12


def test_running_max_blocks():
    """Two keys in two blocks, the larger second: the first P is taken against its own block's maximum and
    rounded there, then rescaled -- unlike the global-max rule, which rounds exp(-d) itself."""
    d = 3.3
    scores = torch.tensor([[0.0, d]], dtype=torch.float64)
    v = torch.tensor([[1.0], [0.0]], dtype=torch.float64)
    two = A.softmax_pv(scores, v, torch.tensor([0, 1]))
    p0 = 1.0 * torch.exp(torch.tensor(-d, dtype=torch.float64))         # fp16(exp(0 - 0)) = 1, rescaled
    assert torch.allclose(two, (p0 / (p0 + 1)).view(1, 1), rtol=0, atol=1e-15)
    one = A.softmax_pv(scores, v, torch.tensor([0, 0]))
    p0 = torch.exp(torch.tensor(-d, dtype=torch.float64)).half().double()
    assert torch.allclose(one, (p0 / (p0 + 1)).view(1, 1), rtol=0, atol=1e-15)
    assert not torch.equal(one, two)


def test_key_blocks_follow_the_slot_order():
    # win 9 -> winP 16: key (kh, kw) in slot kh * 16 + kw; 64-slot blocks hold four key rows
    b = A.key_blocks(9, 64).view(9, 9)
    assert b[:, 0].tolist() == [0, 0, 0, 0, 1, 1, 1, 1, 2]
    assert (b == b[:, :1]).all()
    # win 40 -> winP 64: 128-slot blocks hold two key rows
    assert A.key_blocks(40, 128).view(40, 40)[:, 0].tolist() == [r // 2 for r in range(40)]
    assert A.win_pitch(1) == 8 and A.win_pitch(8) == 8 and A.win_pitch(9) == 16 and A.win_pitch(64) == 64


# ---- the analytic inputs of the GPU tests ----------------------------------------------------------------
@pytest.mark.parametrize("s,win,hd", [(9, 9, 64), (12, 14, 80), (13, 5, 64)])
@pytest.mark.parametrize("zero", ["q", "k"])
def test_uniform_inputs_give_the_window_mean(s, win, hd, zero):
    B, heads = 2, 3
    x = A.uniform_inputs(B, s, win, heads, hd, zero, seed=4, device="cpu")
    ref = A.attention(*x, B, s, win, heads, hd, block=64)
    want = A.window_mean(x[0], x[1], B, s, win, heads, hd)
    assert torch.allclose(ref["exact"], want, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["emulated"], want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("s,win,hd,dh,dw", [
    (9, 9, 64, 2, -3), (9, 9, 80, -20, 20), (13, 5, 64, 1, 1), (12, 14, 80, -3, 0), (10, 10, 64, 0.5, 0),
])
def test_shifted_peak_inputs_pick_one_key(s, win, hd, dh, dw):
    B, heads = 2, 3
    x = A.peak_inputs(B, s, win, heads, hd, dh, dw, device="cpu")
    ref = A.attention(*x, B, s, win, heads, hd, block=128)
    want = A.peak_target(x[0], x[1], B, s, win, heads, hd, dh, dw)
    # the target's neighbours have P = fp16(e^-40) = 0; keys of earlier blocks may still reach l and O
    # rescaled by e^-40 or less, which fp16 rounding of the output removes
    assert torch.equal(ref["emulated"].half().double(), want)
    assert (ref["exact"] - want).abs().max().item() <= 1e-12
    assert (want == want.half().double()).all()
