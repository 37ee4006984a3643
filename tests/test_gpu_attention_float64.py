"""Encoder attention (samroad_op_attention) on every kernel and ring depth, against a float64 reference.

samroad_debug_attention_path says which kernel runs a shape: the one-CTA-per-window kernel and the streamed
kernel round P against a running maximum over 64-slot key chunks, the global wgmma kernel over 128-slot
blocks, the SIMT kernel not at all.  oracle/attention_oracle.py computes the exact float64 output and the
output with that rounding emulated (`emulated`).  Four families of inputs:

uniform   every score exactly 0 (q = 0; or k = 0 with zero rel-pos tables), so every P is 1 and the output
          is the mean of V over the window's keys.  V holds multiples of 1/8, so the device's sums are exact
          and the only errors are 1 / l and the product in fp32 (2^-23 of the output) and the fp16 store (half
          an ulp).  A key dropped, counted twice or left unmasked moves the mean by |v - mean| / n, many ulps.
peak      every query attends to one key at a fixed offset (oracle peak_inputs), clamped into the window:
          the output must be that key's V bit for bit, and V's first columns say which key a query got.
          Offsets put the target in the last, partial key block, past the bottom and right grid edges
          (where an unmasked zero-filled slot would win), and half-integer offsets make two keys tie across
          block boundaries, whose exact mean the output must be.
sum1      V = 1 and weights whose fp16 rounding is all one way (oracle sum1_inputs): the output must be 1
          exactly, which holds only when the softmax denominator sums the same rounded P as P V.
random    fp16 qkv of unit scale (diffuse), q and k x4 (peaked), rel-pos tables x10 (relpos), against the
          bound below, and against `emulated` in fp16 ulps (max, and the fraction of elements > 1 ulp off,
          ulps of the value or of RMS / 256 for small values).

The bound.  For element (r, c), with w the float64 softmax weights, o the exact output and u = 2^-24:

    |out - o| <= E + ulp16(|o| + E) / 2,
    E = (2^-11 + eta_r + gamma) (sum_i w_ri |v_ic| + |o_rc|) + 2^-25 tail_rc

The first factor bounds the relative error of every weight as the device forms it, and a relative error
e_i of weight i moves o by sum_i w_i e_i (v_i - o), at most max e times sum w |v - o| <= sum w |v| + |o|
(the form used here; the exact sum w |v - o| is a [rows, keys, hd] reduction).
  2^-11   fp16 rounding of a normal P.  The denominator l sums the same rounded P, so the rounding moves o
          by at most 2^-11 sum w |v - o| whatever running maximum P was taken against.
  tail    P below 2^-14 is subnormal: absolute error <= 2^-25 against a running maximum m_run <= the final
          one, so <= 2^-25 in units of the row's largest weight after the rescale.  tail_rc = (sum over keys
          with w / max w < 2^-14 of |v_ic| + their count |o_rc|) / sum_i w_i / max w.
  eta_r   the score error, in natural-log units (a score error d is a relative weight error of about d):
            q k^T: hd products of fp16 values are exact in fp32; their sum on the tensor cores, which may
              truncate, is off by <= (hd + 4) 2u sum_j |q_j k_j|; times the scale: (hd + 4) 2u scale qk_r,
              qk_r = max over the row's keys of sum_j |q_j k_ij|;
            rel-pos: each table entry R is split into fp16 hi + lo, off by <= 2^-22 |R| + 2^-25 (lo
              subnormal); the 2 hd products summed on the tensor cores: (2 hd + 4) 2u; times log2e: u.  With
              rel_r = sum_j |q_j| (max |Rh_j| + max |Rw_j|) and qabs_r = sum_j |q_j|:
              (4u + (2 hd + 4) 2u + u) rel_r + u qabs_r;
            the fp32 scale, the fma and the bias add, and the subtraction of the maximum before exp2:
              7u T_r, T_r = scale qk_r + rel_r bounding |S| (and |S - m| <= 2 T_r);
            ex2.approx: 4u; each of the nb rescales by ex2.approx(m_old - m_new), applied to O and l: 8u nb.
  gamma   fp32 accumulation: l sums nslots / 4 values per thread (u each) and O adds one k16 product per
          16 slots on the tensor cores (2u each): (nslots / 4 + 32) u + (nslots / 16 + 16) 2u, nslots = win
          winP; then 1 / l and O / l.  The SIMT kernel sums every key in one thread: 2 (keys + 32) u.
  ulp16   the final fp16 store, at most half an ulp of the stored value, |o| + E at most.
No constant here is fitted to a measurement.  The ulp bounds against `emulated` are (ULP_BOUNDS) about 4x
the worst measured on an H100; the measured values and the worst error / bound ratio per case go to
attention_float64_report.json in the test report directory.

Outputs go into a NaN-filled allocation with guard rows on both sides, which must stay NaN, and qkv is
followed by NaN rows, so a tensor map that overshoots the batch reaches a stored output as NaN."""
import ctypes
import json
import math
import os

import pytest
import torch

from oracle import attention_oracle as A
from sam_road_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UNIT, STREAMED, GLOBAL, SIMT = 0, 1, 2, 3
PATH_NAMES = {UNIT: "unit", STREAMED: "streamed", GLOBAL: "global", SIMT: "simt"}
BLOCK = A.PATH_BLOCK
GUARD = 7                     # guard rows around out, NaN rows after qkv
# (max error in fp16 ulps of `emulated`, fraction of elements more than 1 ulp off), about 4x the worst
# measured on an H100 80GB HBM3 at 700 W (DESIGN.md, "Encoder attention against float64")
ULP_BOUNDS = {"diffuse": (1600.0, 0.009), "peaked": (970.0, 0.0034), "relpos": (1400.0, 0.0058)}
# offsets (dh, dw) of the peak family: centre, a small shift, past the bottom-right and top-left corners,
# ties across key rows (and so across blocks) on the right edge, and ties in both directions
PEAK_OFFSETS = [(0, 0), (2, -3), (-64, -64), (64, 64), (0.5, -64), (-1.5, 0.5)]
_REPORT = {}
_HITS = set()


@pytest.fixture(scope="module", autouse=True)
def _report(report_dir):
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    with open(os.path.join(report_dir, "attention_float64_report.json"), "w") as f:
        json.dump(_REPORT, f, indent=1, sort_keys=True)


def _path(s, win, hd, simt=False):
    lib = _lib.load()
    q, kv = ctypes.c_int(-1), ctypes.c_int(-1)
    lib.samroad_debug_force_simt_attention(1 if simt else 0)
    try:
        p = lib.samroad_debug_attention_path(s, win, hd, ctypes.byref(q), ctypes.byref(kv))
    finally:
        lib.samroad_debug_force_simt_attention(0)
    assert p >= 0, _lib.last_error()
    _HITS.add((hd, win == s, p, q.value, kv.value))
    return p


def _run(x, B, s, win, heads, hd, simt=False):
    """the op on guarded buffers; returns out [B * s * s, D] fp16"""
    qkv16, bias, rel_h, rel_w = x
    D = heads * hd
    n = B * s * s
    lib = _lib.load()
    src = torch.full((n + GUARD, 3 * D), float("nan"), dtype=torch.float16, device=DEV)
    src[:n] = qkv16
    buf = torch.full((n + 2 * GUARD, D), float("nan"), dtype=torch.float16, device=DEV)
    lib.samroad_debug_force_simt_attention(1 if simt else 0)
    try:
        _lib.check(lib.samroad_op_attention(src.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                            B, s, win, heads, hd, buf[GUARD].data_ptr(),
                                            torch.cuda.current_stream().cuda_stream), "attention")
        torch.cuda.synchronize()
    finally:
        lib.samroad_debug_force_simt_attention(0)
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), "write outside out"
    out = buf[GUARD:GUARD + n]
    assert torch.isfinite(out).all(), f"{int((~torch.isfinite(out)).sum())} outputs not finite (or never written)"
    return out


def _where(bad, B, s, heads, hd):
    """(image, y, x, head) of the first few True elements of bad [B * s * s, D], and counts per head / y / x"""
    g = bad.view(B, s, s, heads, hd).any(-1)
    idx = g.nonzero().tolist()
    per = lambda d: {int(i): int(c) for i, c in zip(*torch.unique(g.nonzero()[:, d], return_counts=True))}  # noqa
    return f"{len(idx)} rows; first {idx[:6]}; per_head {per(3)} per_y {per(1)} per_x {per(2)}"


# ---- families ------------------------------------------------------------------------------------------------
def _uniform(B, s, win, heads, hd, simt=False):
    for zero in ("q", "k"):
        x = A.uniform_inputs(B, s, win, heads, hd, zero, seed=s * 7 + hd)
        out = _run(x, B, s, win, heads, hd, simt).double()
        m = A.window_mean(x[0], x[1], B, s, win, heads, hd)
        tol = 0.5 * _ulp16(m.abs() * (1 + 2.0 ** -22)) + 2.0 ** -22 * m.abs()
        bad = (out - m).abs() > tol
        assert not bad.any(), f"uniform ({zero} = 0): mean of V missed at " + _where(bad, B, s, heads, hd)


def _peak(B, s, win, heads, hd, simt=False, offsets=PEAK_OFFSETS):
    for dh, dw in offsets:
        x = A.peak_inputs(B, s, win, heads, hd, dh, dw)
        out = _run(x, B, s, win, heads, hd, simt).double()
        want = A.peak_target(x[0], x[1], B, s, win, heads, hd, dh, dw)
        bad = out != want
        if bad.any():
            o, w = out.view(B, s, s, heads, hd), want.view(B, s, s, heads, hd)
            rows = bad.view(B, s, s, heads, hd).any(-1).nonzero().tolist()[:6]
            got = [(r, o[tuple(r)][:4].tolist(), w[tuple(r)][:4].tolist()) for r in rows]
            raise AssertionError(f"peak ({dh}, {dw}): query (image, y, x, head) -> got (y, x, image, head) of key, "
                                 f"wanted: {got}; " + _where(bad, B, s, heads, hd))


def _sum1(B, s, win, heads, hd, simt=False):
    x = A.sum1_inputs(B, s, win, heads, hd)
    out = _run(x, B, s, win, heads, hd, simt)
    bad = out != 1
    assert not bad.any(), f"sum1: outputs {out[bad][:4].tolist()} != 1 at " + _where(bad, B, s, heads, hd)


def _random_inputs(B, s, win, heads, hd, regime, seed):
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * s * s, 3 * D, generator=g) * 1.5
    bias = 0.5 * torch.randn(3 * D, generator=g)
    rs = 3.0 if regime == "relpos" else 0.3
    rel_h = rs * torch.randn(2 * win - 1, hd, generator=g)
    rel_w = rs * torch.randn(2 * win - 1, hd, generator=g)
    if regime == "peaked":
        qkv[:, :2 * D] *= 4
        bias[:2 * D] *= 4
    return (qkv.to(torch.float16).to(DEV), bias.to(torch.float16).float().to(DEV), rel_h.to(DEV), rel_w.to(DEV))


def _ulp16(mag):
    return torch.exp2(torch.floor(torch.log2(mag.clamp(min=2.0 ** -14))) - 10)


def _ulp_err(dev, ref):
    """(max error in fp16 ulp of the reference, fraction of elements more than 1 ulp off); the ulp of RMS /
    256 for smaller values (as tests/test_gpu_encoder_stages.py)"""
    rms = ref.pow(2).mean().sqrt().item()
    e = (dev - ref).abs() / _ulp16(ref.abs().clamp(min=rms / 256))
    return e.max().item(), (e > 1).double().mean().item()


def _bound(ref, s, win, heads, hd, path):
    u = 2.0 ** -24
    scale = hd ** -0.5
    rows = lambda t: t.repeat_interleave(hd, dim=1)            # noqa: E731  [rows, heads] -> [rows, D]
    qk, rel, qabs = rows(ref["qk"]), rows(ref["rel"]), rows(ref["qabs"])
    T = scale * qk + rel
    nslots = win * A.win_pitch(win)
    if path == SIMT:
        nb = math.ceil(win * win / 32)
        gamma = 2 * (win * win + 32) * u
    else:
        nb = math.ceil(nslots / BLOCK[path])
        gamma = (nslots / 4 + 32) * u + (nslots / 16 + 16) * 2 * u
    eta = ((hd + 4) * 2 * u * scale * qk + (4 * u + (2 * hd + 4) * 2 * u + u) * rel + u * qabs + 7 * u * T
           + 4 * u + 8 * u * nb)
    o = ref["exact"]
    E = (2.0 ** -11 + eta + gamma) * (ref["wv"] + o.abs()) + 2.0 ** -25 * ref["tail"]
    return E + 0.5 * _ulp16(o.abs() + E)


def _random(tag, B, s, win, heads, hd, path, regimes=("diffuse",), images=None, simt=False):
    images = list(range(B)) if images is None else images
    D = heads * hd
    for regime in regimes:
        x = _random_inputs(B, s, win, heads, hd, regime, seed=1000 * s + hd + B)
        out = _run(x, B, s, win, heads, hd, simt).view(B, -1, D)[images].reshape(-1, D).double()
        sel = (x[0].view(B, -1, 3 * D)[images].reshape(-1, 3 * D),) + x[1:]
        ref = A.attention(*sel, len(images), s, win, heads, hd, block=BLOCK[path], bound_terms=True)
        err = (out - ref["exact"]).abs()
        ratio = err / _bound(ref, s, win, heads, hd, path)
        ulp_max, frac = _ulp_err(out, ref["emulated"])
        _REPORT[f"{tag}/{regime}"] = {"path": PATH_NAMES[path], "bound_ratio": ratio.max().item(),
                                      "ulp_max": ulp_max, "ulp_frac": frac}
        print(tag, regime, json.dumps(_REPORT[f"{tag}/{regime}"]))
        bad = ratio > 1
        assert not bad.any(), (f"{regime}: error over the float64 bound (worst ratio {ratio.max().item():.3f}) at "
                               + _where(bad, len(images), s, heads, hd))
        lim = ULP_BOUNDS[regime]
        assert ulp_max <= lim[0] and frac <= lim[1], (regime, ulp_max, frac, lim)


# ---- shapes ----------------------------------------------------------------------------------------------------
SWEEP = [(s, hd) for hd in (64, 80) for s in range(1, 65)]


@pytest.mark.parametrize("s,hd", SWEEP, ids=[f"s{s}-hd{hd}" for s, hd in SWEEP])
def test_global_sweep(s, hd):
    """win = s for every s at B = 2 and 3 heads: every winP, partial last query item and key block, and
    every ring depth (and, at head dim 80 and s = 41..64, the streamed kernel)"""
    B, heads = 2, 3
    path = _path(s, s, hd)
    _uniform(B, s, s, heads, hd)
    _peak(B, s, s, heads, hd)
    _sum1(B, s, s, heads, hd)
    _random(f"sweep_s{s}_hd{hd}", B, s, s, heads, hd, path)


MANY = [(64, s, 3, 64) for s in (32, 41, 53, 64)] + [(64, s, 3, 80) for s in (16, 23, 32, 37, 40, 41, 64)] + [
    (1, 23, 1, 64), (1, 32, 1, 80), (1, 64, 1, 80)]     # grids smaller than the SM count: one image, one head
SAMPLE = [0, 5, 6, 17, 30, 47, 62, 63]   # images checked against float64 at B = 64 (batch invariance: all)


@pytest.mark.parametrize("B,s,heads,hd", MANY, ids=[f"B{b}-s{s}-h{h}-hd{hd}" for b, s, h, hd in MANY])
def test_global_many_items(B, s, heads, hd):
    """B = 64: a CTA walks several work items (3 heads x 64 images x ceil(s^2 / 128) items, a count that is
    no multiple of the SM count), so the rings and barrier phases are handed on from item to item"""
    path = _path(s, s, hd)
    images = SAMPLE if B == 64 else None
    _uniform(B, s, s, heads, hd)
    _peak(B, s, s, heads, hd, offsets=[(0, 0), (-64, -64), (0.5, -64)])
    _sum1(B, s, s, heads, hd)
    _random(f"many_B{B}_s{s}_h{heads}_hd{hd}", B, s, s, heads, hd, path, ("diffuse", "peaked", "relpos"), images)


@pytest.mark.parametrize("s,hd", [(32, 64), (41, 64), (37, 80), (64, 80), (25, 64)])
def test_batch_invariance(s, hd):
    """image b alone at B = 1 gives the same bits as inside a batch of 64 (no state leaks from item to item)"""
    B, heads = 64, 3
    win = s if s != 25 else 14
    D = heads * hd
    x = _random_inputs(B, s, win, heads, hd, "diffuse", seed=5)
    full = _run(x, B, s, win, heads, hd).view(B, -1, D)
    for b in (0, 31, 63):
        one = (x[0].view(B, -1, 3 * D)[b].contiguous(),) + x[1:]
        assert torch.equal(_run(one, 1, s, win, heads, hd).view(-1, D), full[b]), b


WINDOWS = [   # (s, win, hd): the path each takes is asserted in test_dispatch_coverage
    (25, 14, 64), (32, 14, 64), (25, 14, 80), (32, 14, 80),      # one CTA per window
    (40, 20, 80), (30, 16, 80),                                  # windows streamed
    (12, 14, 64), (13, 14, 64), (12, 14, 80), (13, 14, 80),      # one window padded past the grid
]


@pytest.mark.parametrize("s,win,hd", WINDOWS, ids=[f"s{s}-w{w}-hd{hd}" for s, w, hd in WINDOWS])
def test_window_paths(s, win, hd):
    B, heads = 3, 3
    path = _path(s, win, hd)
    _uniform(B, s, win, heads, hd)
    _peak(B, s, win, heads, hd)
    _sum1(B, s, win, heads, hd)
    _random(f"window_s{s}_w{win}_hd{hd}", B, s, win, heads, hd, path, ("diffuse", "peaked", "relpos"))


SIMT_CASES = [(16, 16, 64), (25, 14, 64), (12, 14, 80), (23, 23, 80), (64, 64, 64)]


@pytest.mark.parametrize("s,win,hd", SIMT_CASES, ids=[f"s{s}-w{w}-hd{hd}" for s, w, hd in SIMT_CASES])
def test_simt_kernel(s, win, hd):
    """the fp32 SIMT kernel, every other kernel's on-device checker, pinned to float64 itself"""
    B, heads = 2, 3
    path = _path(s, win, hd, simt=True)
    assert path == SIMT
    _uniform(B, s, win, heads, hd, simt=True)
    _peak(B, s, win, heads, hd, simt=True, offsets=[(0, 0), (-64, -64), (0.5, -64)])
    _sum1(B, s, win, heads, hd, simt=True)
    _random(f"simt_s{s}_w{win}_hd{hd}", B, s, win, heads, hd, path, ("diffuse", "peaked", "relpos"), simt=True)


def test_dispatch_coverage():
    """the shapes above reach every (kernel, ring depth) samroad_op_attention can choose at both head dims"""
    for s, hd in SWEEP:
        _path(s, s, hd)
    for s, win, hd in WINDOWS:
        _path(s, win, hd)
    for s, win, hd in SIMT_CASES:
        _path(s, win, hd, simt=True)
    for hd in (64, 80):
        want = {(hd, True, GLOBAL, 2, 3), (hd, True, GLOBAL, 2, 2), (hd, True, GLOBAL, 1, 2),
                (hd, False, UNIT, 0, 0), (hd, False, STREAMED, 0, 0)}
        if hd == 80:
            want.add((hd, True, STREAMED, 0, 0))          # s = 41..64: no ring fits
        assert want <= _HITS, want - _HITS
        assert any(h[0] == hd and h[2] == SIMT for h in _HITS)
    # every s of the sweep at head dim 80 from 41 on takes the streamed kernel, below it the global one
    lib = _lib.load()
    for s in range(1, 65):
        assert lib.samroad_debug_attention_path(s, s, 80, None, None) == (STREAMED if s > 40 else GLOBAL), s
