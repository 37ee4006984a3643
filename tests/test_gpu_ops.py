"""Op-level parity on the GPU, through the C ABI: every kernel against plain fp32 torch math on the
same (fp16-rounded) operands, and the wgmma GEMM additionally against the SIMT checker GEMM."""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from sam_road_b200 import _lib  # noqa: E402
from oracle import samroad_oracle as O  # noqa: E402

DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _fp32_oracle_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rand16(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.float16).to(DEV)


GEMM_SHAPES = [
    (256, 768, 768), (1000, 2304, 768), (20000, 3072, 768), (512, 768, 3072), (300, 128, 128),
    (4099, 384, 128), (640, 256, 64), (130, 512, 256), (19000, 768, 768), (77, 256, 2304),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_f16(M, N, K, act):
    lib = _lib.load()
    A = _rand16((M, K), 1.0, 1)
    W = _rand16((N, K), 1.0 / math.sqrt(K), 2)
    bias = torch.randn(N, device=DEV)
    out = torch.full((M, N), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(lib.samroad_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                       act, out.data_ptr(), N, _st()), "gemm_f16")
    ref = A.float() @ W.float().t() + bias
    ref = [lambda x: x, F.gelu, F.relu][act](ref)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out.float()).all()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), f"max abs err {err}"
    if act == 0:   # independent on-device checker
        chk = torch.empty((M, N), dtype=torch.float32, device=DEV)
        _lib.check(lib.samroad_op_gemm_ref(A.data_ptr(), K, W.data_ptr(), K, M, N, K,
                                           chk.data_ptr(), N, _st()), "gemm_ref")
        torch.cuda.synchronize()
        assert (chk + bias - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("M,N,K", [(256, 768, 768), (3000, 768, 3072), (20000, 768, 768), (500, 256, 128)])
def test_gemm_f32_resid_pos(M, N, K):
    lib = _lib.load()
    A = _rand16((M, K), 1.0, 3)
    W = _rand16((N, K), 1.0 / math.sqrt(K), 4)
    bias = torch.randn(N, device=DEV)
    resid = torch.randn(M, N, device=DEV)
    T = 64
    pos = torch.randn(T, N, device=DEV)
    ref = A.float() @ W.float().t() + bias + resid + pos[torch.arange(M, device=DEV) % T]
    out = resid.clone()   # in-place residual, as the encoder uses it
    _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                       out.data_ptr(), pos.data_ptr(), T, out.data_ptr(), N, _st()),
               "gemm_f32")
    torch.cuda.synchronize()
    err = (out - ref).abs().max().item()
    assert err < 2e-4 * max(1.0, ref.abs().max().item()), err
    out2 = torch.empty_like(out)
    _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, None, None, None,
                                       0, out2.data_ptr(), N, _st()), "gemm_f32 plain")
    torch.cuda.synchronize()
    assert (out2 - A.float() @ W.float().t()).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,N,K", [(65536, 768, 768), (20001, 768, 3072), (9999, 1024, 512)])
def test_gemm_f32_inplace_shortcut_tma(M, N, K):
    """x += A.W^T + b in place (attention proj / MLP lin2 shortcut) at encoder sizes against fp32 torch
    math; a repeated call gives the same bits."""
    lib = _lib.load()
    A = _rand16((M, K), 1.0, 31)
    W = _rand16((N, K), 1.0 / math.sqrt(K), 32)
    bias = torch.randn(N, device=DEV)
    resid = torch.randn(M, N, device=DEV) * 3
    ref = resid + bias
    for m0 in range(0, M, 16384):     # chunked: keeps the fp32 reference product small
        ref[m0:m0 + 16384] += A[m0:m0 + 16384].float() @ W.float().t()
    outs = []
    for _ in range(2):
        out = resid.clone()
        _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                           out.data_ptr(), None, 0, out.data_ptr(), N, _st()),
                   "gemm_f32 in place")
        torch.cuda.synchronize()
        outs.append(out)
    tol = 2e-4 * max(1.0, ref.abs().max().item())
    assert (outs[0] - ref).abs().max().item() < tol
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,T", [(65536, 1024), (20480, 256), (30000, 1024)])
def test_gemm_f32_pos_embed_tma(M, T):
    """out = A.W^T + b + pos[m % T] (patch embedding + pos_embed, image_encoder.py:107-109) at encoder
    sizes against fp32 torch math; a repeated call gives the same bits."""
    lib = _lib.load()
    N = K = 768
    A = _rand16((M, K), 1.0, 41)
    W = _rand16((N, K), 1.0 / math.sqrt(K), 42)
    bias = torch.randn(N, device=DEV)
    pos = torch.randn(T, N, device=DEV)
    ref = bias + pos[torch.arange(M, device=DEV) % T]
    for m0 in range(0, M, 16384):
        ref[m0:m0 + 16384] += A[m0:m0 + 16384].float() @ W.float().t()
    outs = []
    for _ in range(2):
        out = torch.full((M, N), float("nan"), device=DEV)
        _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                           None, pos.data_ptr(), T, out.data_ptr(), N, _st()), "gemm_f32 pos")
        torch.cuda.synchronize()
        outs.append(out)
    tol = 2e-4 * max(1.0, ref.abs().max().item())
    assert (outs[0] - ref).abs().max().item() < tol
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,N,K,group,act", [(1024, 256, 768, 256, 0), (1024, 512, 256, 128, 1),
                                             (333, 128, 128, 128, 0), (20000, 512, 256, 128, 1),
                                             (2048, 256, 2304, 256, 0)])
def test_gemm_ln(M, N, K, group, act):
    lib = _lib.load()
    A = _rand16((M, K), 1.0, 5)
    W = _rand16((N, K), 1.0 / math.sqrt(K), 6)
    bias = torch.randn(N, device=DEV) * 0.3
    resid = torch.randn(M, N, device=DEV)
    gamma = 1 + 0.1 * torch.randn(group, device=DEV)
    beta = 0.1 * torch.randn(group, device=DEV)
    tokens = 64 if M % 64 == 0 else 1
    x = A.float() @ W.float().t() + bias + resid
    y = F.layer_norm(x.view(M, N // group, group), (group,), gamma, beta, 1e-6).view(M, N)
    if act == 1:
        y = F.gelu(y)
    o16 = torch.empty((M, N), dtype=torch.float16, device=DEV)
    o32 = torch.empty((M, N), dtype=torch.float32, device=DEV)
    onchw = torch.empty((M // tokens, N, tokens), dtype=torch.float32, device=DEV)
    _lib.check(lib.samroad_op_gemm_ln(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                      resid.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-6,
                                      group, act, o16.data_ptr(), o32.data_ptr(), onchw.data_ptr(),
                                      tokens, N, _st()), "gemm_ln")
    torch.cuda.synchronize()
    assert (o32 - y).abs().max().item() < 2e-3
    assert (o16.float() - y).abs().max().item() < 6e-3
    assert (onchw.permute(0, 2, 1).reshape(M, N) - o32).abs().max().item() == 0.0


@pytest.mark.parametrize("M,D", [(1000, 768), (64, 1280), (4097, 128), (300, 1024)])
def test_layernorm(M, D):
    lib = _lib.load()
    x = torch.randn(M, D, device=DEV) * 3 + 0.5
    g = 1 + 0.1 * torch.randn(D, device=DEV)
    b = 0.1 * torch.randn(D, device=DEV)
    out = torch.empty((M, D), dtype=torch.float16, device=DEV)
    _lib.check(lib.samroad_op_layernorm(x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-6, M, D,
                                        out.data_ptr(), _st()), "layernorm")
    ref = F.layer_norm(x, (D,), g, b, 1e-6)
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max().item() < 4e-3


@pytest.mark.parametrize("B,s,win,heads,hd", [(2, 16, 14, 12, 64), (2, 16, 16, 12, 64),
                                              (1, 32, 14, 12, 64), (1, 32, 32, 12, 64),
                                              (1, 16, 14, 16, 80), (1, 16, 16, 16, 80),
                                              (2, 32, 14, 16, 80), (1, 32, 32, 16, 80)])
def test_encoder_attention(B, s, win, heads, hd):
    """Window (pad-after-LN semantics) and global attention with decomposed rel-pos."""
    lib = _lib.load()
    D = heads * hd
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, s, s, D, generator=g).to(DEV)
    w = (torch.randn(3 * D, D, generator=g) / math.sqrt(D)).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(DEV)
    rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    qkv16 = F.linear(x, w, bias).to(torch.float16).contiguous()          # real tokens only
    bias16 = bias.to(torch.float16).float()   # pad tokens see the bias rounded like everything else
    # oracle: pad after "LN", qkv of pad tokens = bias, attention per window, merge + crop
    if win < s:
        xw, padded = O.window_split(qkv16.float(), win)
        mask, _ = O.window_split(torch.ones(B, s, s, 1, device=DEV), win)
        xw = torch.where(mask.bool(), xw, bias16.view(1, 1, 1, -1).expand_as(xw))
        ref = O.window_merge(O.attention_core(xw, rel_h, rel_w, heads), win, padded, (s, s))
    else:
        ref = O.attention_core(qkv16.float(), rel_h, rel_w, heads)
    out = torch.full((B * s * s, D), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias16.data_ptr(), rel_h.data_ptr(),
                                        rel_w.data_ptr(), B, s, win, heads, hd, out.data_ptr(),
                                        _st()), "attention")
    torch.cuda.synchronize()
    diff = (out.float().view(B, s, s, D) - ref).abs()
    err = diff.max().item()
    tol = 1.5e-3 * max(1.0, ref.abs().max().item())   # fp16 P / output rounding: a few output ulps
    if not err < tol:   # diagnostics: where is it wrong?
        per_head = diff.view(B, s, s, heads, hd).amax(dim=(0, 1, 2, 4)).tolist()
        per_y = diff.amax(dim=(0, 2, 3)).tolist()
        per_x = diff.amax(dim=(0, 1, 3)).tolist()
        nan = int(torch.isnan(out.float()).sum().item())
        print(f"attention mismatch: max {err} nan {nan}\n per_head {per_head}\n per_y {per_y}\n per_x {per_x}")
    assert err < tol, (err, tol)


@pytest.mark.parametrize("B,s,win,heads,hd", [(3, 32, 14, 12, 64), (3, 32, 32, 12, 64), (5, 16, 14, 12, 64),
                                              (5, 16, 16, 12, 64), (12, 16, 14, 16, 80), (12, 16, 16, 16, 80),
                                              (3, 32, 14, 16, 80), (2, 32, 32, 16, 80),
                                              (2, 64, 64, 12, 64), (1, 64, 14, 12, 64)])   # PATCH_SIZE 1024: 64x64 grid
def test_attention_tc_vs_simt(B, s, win, heads, hd):
    """Tensor-core kernel (head_dim 64 and 80) against the fp32 SIMT kernel on identical inputs
    (independent checker); batches of many windows and heads."""
    lib = _lib.load()
    D = heads * hd
    g = torch.Generator().manual_seed(11)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
    rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    outs = []
    for simt in (1, 0):
        lib.samroad_debug_force_simt_attention(simt)
        out = torch.full((B * s * s, D), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(),
                                            rel_w.data_ptr(), B, s, win, heads, hd, out.data_ptr(),
                                            _st()), "attention")
        torch.cuda.synchronize()
        outs.append(out.float())
    lib.samroad_debug_force_simt_attention(0)
    err = (outs[0] - outs[1]).abs().max().item()
    mean_err = (outs[0] - outs[1]).abs().mean().item()
    mag = outs[0].abs().max().item()
    print(f"tc vs simt: max err {err:.3e} mean err {mean_err:.3e} |out|max {mag:.3f}")
    assert torch.isfinite(outs[1]).all()
    # P is rounded to fp16 (rel 2^-11) before the PV MMA and the output to fp16: a few output ulps
    assert err <= 2.5e-3 * mag and mean_err <= 2e-4 * mag, (err, mean_err, mag)


@pytest.mark.parametrize("B,s,win,heads,hd", [(64, 16, 14, 12, 64), (48, 32, 14, 12, 64), (64, 16, 16, 12, 64),
                                              (64, 16, 14, 16, 80), (3, 64, 64, 12, 64)])
def test_attention_run_to_run_determinism(B, s, win, heads, hd):
    """The same QKV through the tensor-core attention 24 times must give identical bits, on inputs that
    were just rewritten (L2-resident), with thousands of CTAs of window or global units in flight."""
    lib = _lib.load()
    D = heads * hd
    g = torch.Generator().manual_seed(5)
    qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
    bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
    rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
    first = None
    for it in range(24):
        out = torch.full((B * s * s, D), float("nan"), dtype=torch.float16, device=DEV)
        qkv16.copy_(qkv16.clone())
        _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(),
                                            rel_w.data_ptr(), B, s, win, heads, hd, out.data_ptr(),
                                            _st()), "attention")
        if first is None:
            first = out
        else:
            assert torch.equal(first, out), (it, int((first != out).sum()))
    assert torch.isfinite(first.float()).all()
