"""Float64 reference of one encoder attention call (samroad_op_attention) -- TEST INFRASTRUCTURE ONLY (see
samroad_oracle.py).

The operands are those of the op: fp16 qkv [B * s * s, 3 D] (columns (q | k | v) x head x hd), the fp32 qkv
bias [3 D] and the rel-pos tables [2 win - 1, hd].  Windows of `win` tokens cut the s x s grid from the top
left; a window that runs past the grid is padded with tokens whose q = k = v = fp16(bias), which are real
softmax keys (image_encoder.py:168-172 on a zero LayerNorm output) whose query rows are never written.
win == s is a global block.  For every real query row, in float64:

  exact     softmax(scale q k^T + q Rh + q Rw) v, scale = hd^-1/2, the rel-pos terms from the unscaled q
            (image_encoder.py:224-240, 325-361);
  emulated  the same with P rounded as the tensor-core kernels round it: key slots k = kh * winP + kw
            (winP = the next power of two >= max(win, 8)) are cut into blocks of `block` slots; P =
            fp16(exp(S - m_run)) with m_run the row's running maximum through the key's block; the earlier
            blocks are rescaled by exp(m_old - m_new), and the denominator sums the rounded P.  block=None
            leaves P unrounded (the fp32 SIMT kernel), and a block of at least win * winP slots is the
            "P against the row's global maximum" rule.

and, for the error bound of tests/test_gpu_attention_float64.py, per row r with w the exact softmax weights:

  wv        sum_i w_ri |v_ic|                                                    [rows, hd]
  tail      (sum_{i: w_ri / max w_r < 2^-14} |v_ic|  +  n_small |o_rc|) / sum_i w_ri / max w_r    [rows, hd]
  qk        max_i sum_j |q_j k_ij|  over the row's keys                          [rows]
  rel       sum_j |q_j| (max_t |Rh_tj| + max_t |Rw_tj|)                          [rows]
  qabs      sum_j |q_j|                                                          [rows]

Work is done one (image, heads) chunk at a time on the operands' device: a global block at s = 64 holds
4096 x 4096 float64 scores (134 MB) per head.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

Tensor = torch.Tensor

# score elements of one chunk
_CHUNK = 1 << 24
# key slots per running-maximum block of each kernel, by the number samroad_debug_attention_path returns: the
# one-CTA-per-window and streamed kernels (64-slot chunks), the global wgmma kernel (128-slot blocks), the SIMT
# kernel (P unrounded)
PATH_BLOCK = {0: 64, 1: 64, 2: 128, 3: None}


def win_pitch(win: int) -> int:
    """winP: the key-row pitch of the tensor-core kernels' slot order"""
    p = 8
    while p < win:
        p <<= 1
    return p


def key_blocks(win: int, block: Optional[int], device=None) -> Optional[Tensor]:
    """block index of every key (kh, kw) of a window, in the order kh * win + kw; None for block=None"""
    if block is None:
        return None
    kh, kw = torch.meshgrid(torch.arange(win), torch.arange(win), indexing="ij")
    return ((kh * win_pitch(win) + kw) // block).reshape(-1).to(device)


def softmax_pv(scores: Tensor, v: Tensor, blocks: Optional[Tensor]) -> Tensor:
    """softmax(scores) v over the last axis of scores [..., Lq, Lk] (-inf: no key) and v [..., Lk, hd].
    With blocks [Lk] (the block of every key), P is rounded to fp16 against the running maximum through the
    key's block, as the device does; the blocks' partial sums meet at the final maximum."""
    if blocks is None:
        return scores.softmax(-1) @ v
    nb = int(blocks.max()) + 1
    idx = blocks.expand_as(scores)
    bmax = torch.full((*scores.shape[:-1], nb), float("-inf"), dtype=scores.dtype, device=scores.device)
    bmax = bmax.scatter_reduce(-1, idx, scores, "amax")
    run = torch.cummax(bmax, -1).values                       # m_run after each block
    fin = run[..., -1:]
    m = run.gather(-1, idx)                                   # m_run of every key's block
    p = torch.exp(scores - m).to(torch.float16).to(scores.dtype)
    p = p * torch.exp(m - fin)                                # the later rescales, exact in float64
    return (p @ v) / p.sum(-1, keepdim=True)


def _unit_tokens(qkv: Tensor, bias16: Tensor, b: int, s: int, win: int) -> Tensor:
    """tokens of image b cut into windows: [nwin^2, win * win, 3 D] float64, padding tokens = fp16(bias)"""
    nwin = -(-s // win)
    sp = nwin * win
    x = bias16.expand(sp, sp, bias16.shape[-1]).clone()
    x[:s, :s] = qkv[b * s * s:(b + 1) * s * s].view(s, s, -1).double()
    return x.view(nwin, win, nwin, win, -1).permute(0, 2, 1, 3, 4).reshape(nwin * nwin, win * win, -1)


def _gather(table: Tensor, win: int) -> Tensor:
    """R[q, k] = table[q - k + win - 1]  [win, win, hd]"""
    i = torch.arange(win, device=table.device)
    return table[(i.view(-1, 1) - i.view(1, -1) + win - 1)]


def attention(qkv16: Tensor, qkv_bias: Tensor, rel_h: Tensor, rel_w: Tensor, B: int, s: int, win: int,
              heads: int, hd: int, block: Optional[int] = None, bound_terms: bool = False) -> Dict[str, Tensor]:
    """{'exact', 'emulated'} (and with bound_terms the bound's ingredients, see the module docstring) for the
    real query rows, as [B * s * s, D] (per-row terms [B * s * s, heads])."""
    dev = qkv16.device
    D = heads * hd
    L = win * win
    nwin = -(-s // win)
    nw = nwin * nwin
    scale = hd ** -0.5
    bias16 = qkv_bias.to(dev).to(torch.float16).double()
    Rh, Rw = _gather(rel_h.to(dev).double(), win), _gather(rel_w.to(dev).double(), win)
    rmax = rel_h.to(dev).double().abs().amax(0) + rel_w.to(dev).double().abs().amax(0)     # [hd]
    blocks = key_blocks(win, block, dev)
    names = ["exact", "emulated"] + (["wv", "tail"] if bound_terms else [])
    rows = ["qk", "rel", "qabs"] if bound_terms else []
    out = {k: torch.empty(B, nw, L, heads, hd, dtype=torch.float64, device=dev) for k in names}
    out.update({k: torch.empty(B, nw, L, heads, dtype=torch.float64, device=dev) for k in rows})
    hc = max(1, min(heads, _CHUNK // (nw * L * L)))
    for b in range(B):
        t = _unit_tokens(qkv16, bias16, b, s, win).view(nw, L, 3, heads, hd)
        for h0 in range(0, heads, hc):
            hs = slice(h0, min(heads, h0 + hc))
            q, k, v = (t[:, :, i, hs].transpose(1, 2) for i in range(3))         # [nw, h, L, hd]
            qg = q.reshape(*q.shape[:2], win, win, hd)
            rh = torch.einsum("nahwc,hkc->nahwk", qg, Rh)
            rw = torch.einsum("nahwc,wkc->nahwk", qg, Rw)
            sc = (scale * q @ k.transpose(-2, -1)).view(*q.shape[:2], win, win, win, win)
            sc = (sc + rh[..., :, None] + rw[..., None, :]).view(*q.shape[:2], L, L)
            w = sc.softmax(-1)
            o = w @ v
            res = {"exact": o, "emulated": o if blocks is None else softmax_pv(sc, v, blocks)}
            if bound_terms:
                res["wv"] = w @ v.abs()
                wr = w / w.amax(-1, keepdim=True)
                small = (wr < 2.0 ** -14).double()
                res["tail"] = (small @ v.abs() + small.sum(-1, keepdim=True) * o.abs()) / wr.sum(-1, keepdim=True)
                qa = q.abs()
                res["qk"] = (qa @ k.abs().transpose(-2, -1)).amax(-1)
                res["rel"] = qa @ rmax
                res["qabs"] = qa.sum(-1)
            for key, val in res.items():
                out[key][b, :, :, hs] = val.transpose(1, 2)
    merged = {}
    for key, val in out.items():
        tail = val.shape[3:]
        g = val.view(B, nwin, nwin, win, win, *tail).transpose(2, 3).reshape(B, nwin * win, nwin * win, *tail)
        g = g[:, :s, :s].reshape(B * s * s, -1)
        merged[key] = g
    return merged


# ---- inputs whose correct output is known exactly ------------------------------------------------------------
# V holds small multiples of 1/8, so that every sum of up to 4096 of them, and the mean of two or four, is
# exact in fp32 and in fp16.
def _v_values(shape, g) -> Tensor:
    return torch.randint(-64, 65, shape, generator=g).float() / 8


def uniform_inputs(B: int, s: int, win: int, heads: int, hd: int, zero: str, seed: int, device="cuda:0"):
    """(qkv16, bias, rel_h, rel_w) whose scores are all exactly 0: zero="q" sets q = 0 (every score term has
    q in it), zero="k" sets k = 0, the K third of the bias (padding keys) and both rel-pos tables to 0.  Every
    P is then 1 and the output is the mean of V over the window's keys (window_mean)."""
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * s * s, 3 * D, generator=g) * 1.5
    qkv[:, 2 * D:] = _v_values((B * s * s, D), g)
    bias = 0.5 * torch.randn(3 * D, generator=g)
    bias[2 * D:] = _v_values((D,), g)
    rel_h = 0.3 * torch.randn(2 * win - 1, hd, generator=g)
    rel_w = 0.3 * torch.randn(2 * win - 1, hd, generator=g)
    if zero == "q":
        qkv[:, :D] = 0
    else:
        qkv[:, D:2 * D] = 0
        bias[D:2 * D] = 0
        rel_h.zero_()
        rel_w.zero_()
    return (qkv.to(torch.float16).to(device), bias.to(torch.float16).float().to(device), rel_h.to(device),
            rel_w.to(device))


def window_mean(qkv16: Tensor, bias: Tensor, B: int, s: int, win: int, heads: int, hd: int) -> Tensor:
    """every query row's mean of V over the keys of its window, padding keys included  [B * s * s, D]"""
    D = heads * hd
    nwin = -(-s // win)
    sp = nwin * win
    v = bias[2 * D:].double().expand(B, sp, sp, D).clone()
    v[:, :s, :s] = qkv16[:, 2 * D:].double().view(B, s, s, D)
    m = v.view(B, nwin, win, nwin, win, D).mean(dim=(2, 4), keepdim=True).expand(B, nwin, win, nwin, win, D)
    return m.reshape(B, sp, sp, D)[:, :s, :s].reshape(B * s * s, D)


PEAK_BETA = 40.0


def peak_inputs(B: int, s: int, win: int, heads: int, hd: int, dh: float, dw: float, device="cuda:0"):
    """(qkv16, bias, rel_h, rel_w) that make query (qh, qw) of a window attend to its key (qh - dh, qw - dw),
    clamped into the window: k = 0 (and the K third of the bias, so padding keys score like real ones), q = u
    = (1, .., 1), rel_h[j] = -beta (j - (win - 1) - dh)^2 u / |u|^2 and rel_w alike, so the score of key
    (kh, kw) is -beta ((qh - kh - dh)^2 + (qw - kw - dw)^2).  With beta = 40 every other key's weight is at
    most e^-40 of the target's: its P rounds to 0 against the target, and a key of an earlier block that
    reached O against a lower running maximum is rescaled to below half the smallest fp16 subnormal of the
    output even times |v| = 64.  A half-integer offset makes two keys tie exactly.
    V's columns 0..3 are (y, x, image, head) of a real token and -1 for a padding token."""
    D = heads * hd
    g = torch.Generator().manual_seed(int(1000 + 10 * dh + dw))
    qkv = torch.zeros(B * s * s, 3 * D)
    qkv[:, :D] = 1.0
    v = _v_values((B, s, s, heads, hd), g)
    y, x = torch.meshgrid(torch.arange(s), torch.arange(s), indexing="ij")
    v[..., 0] = y.view(1, s, s, 1).float()
    v[..., 1] = x.view(1, s, s, 1).float()
    v[..., 2] = torch.arange(B).view(B, 1, 1, 1).float()
    v[..., 3] = torch.arange(heads).view(1, 1, 1, heads).float()
    qkv[:, 2 * D:] = v.view(B * s * s, D)
    bias = torch.zeros(3 * D)
    bias[:D] = torch.randn(D, generator=g)                    # q of padding tokens: never a query row
    bv = _v_values((heads, hd), g)
    bv[:, :4] = -1
    bias[2 * D:] = bv.view(-1)
    j = torch.arange(2 * win - 1, dtype=torch.float64) - (win - 1)
    rel_h = (-PEAK_BETA * (j - dh) ** 2 / hd).float().view(-1, 1).expand(-1, hd).contiguous()
    rel_w = (-PEAK_BETA * (j - dw) ** 2 / hd).float().view(-1, 1).expand(-1, hd).contiguous()
    return qkv.to(torch.float16).to(device), bias.to(device), rel_h.to(device), rel_w.to(device)


def _nearest(n: int, d: float) -> Tensor:
    """[n, n] weights: row qh spreads 1 evenly over the keys kh in [0, n) nearest to qh - d"""
    qh = torch.arange(n, dtype=torch.float64).view(-1, 1)
    dist = (qh - torch.arange(n, dtype=torch.float64).view(1, -1) - d).abs()
    near = (dist == dist.amin(-1, keepdim=True)).double()
    return near / near.sum(-1, keepdim=True)


def peak_target(qkv16: Tensor, bias: Tensor, B: int, s: int, win: int, heads: int, hd: int, dh: float,
                dw: float) -> Tensor:
    """what peak_inputs must give: every query row's V at its target key (the mean over tied keys), found by
    index arithmetic alone  [B * s * s, D]"""
    D = heads * hd
    nwin = -(-s // win)
    sp = nwin * win
    v = bias[2 * D:].double().expand(B, sp, sp, D).clone()
    v[:, :s, :s] = qkv16[:, 2 * D:].double().view(B, s, s, D)
    v = v.view(B, nwin, win, nwin, win, D)
    Wh, Ww = _nearest(win, dh).to(v.device), _nearest(win, dw).to(v.device)
    o = torch.einsum("qk,bykxwc->byqxwc", Wh, v)
    o = torch.einsum("qk,byhxkc->byhxqc", Ww, o)
    return o.reshape(B, sp, sp, D)[:, :s, :s].reshape(B * s * s, D)


# P of every key outside the query's own key row: just below the midpoint of 0.5 and the next fp16 value, so
# that fp16 rounds each such P down by nearly 2^-12, all in the same direction
SUM1_P = 0.5 + 2.0 ** -12 - 2.0 ** -15


def sum1_inputs(B: int, s: int, win: int, heads: int, hd: int, device="cuda:0"):
    """(qkv16, bias, rel_h, rel_w) with V = 1 for every token, padding tokens included, so that every output
    is exactly 1 whatever the weights -- when the softmax denominator sums the same P as P V.  k = 0, q = 1,
    rel_w = 0, rel_h = 0 on the query's own key row and ln(SUM1_P) / hd elsewhere: keys of the query's row
    have P = 1, all others P = fp16(SUM1_P) = 0.5.  A denominator of unrounded P is larger by up to 2^-11
    of itself, which moves the output to 1 - 2^-11."""
    D = heads * hd
    g = torch.Generator().manual_seed(s)
    qkv = torch.zeros(B * s * s, 3 * D)
    qkv[:, :D] = 1.0
    qkv[:, 2 * D:] = 1.0
    bias = torch.zeros(3 * D)
    bias[:D] = torch.randn(D, generator=g)
    bias[2 * D:] = 1.0
    rel_h = torch.full((2 * win - 1, hd), float(torch.log(torch.tensor(SUM1_P, dtype=torch.float64))) / hd)
    rel_h[win - 1] = 0.0
    rel_w = torch.zeros(2 * win - 1, hd)
    return qkv.to(torch.float16).to(device), bias.to(device), rel_h.to(device), rel_w.to(device)
