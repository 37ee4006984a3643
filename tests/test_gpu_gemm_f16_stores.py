"""The fp16 epilogue of the ping-pong GEMM (samroad_op_gemm_f16) stores each row's 32-column chunk after a 4x4
transpose across the lanes of a quad.  Without activation its output must be the fp32 epilogue's acc + bias
(samroad_op_gemm_f32 without residual, the same fp32 sums) rounded to fp16, bit for bit, so any column or lane
mix-up shows.  Covered: K = 768 (12 k-blocks) and K = 3072, N a multiple of 128 and not (a last tile of one to
three 32-column chunks), an M tail, an output wider than N whose other columns must stay untouched, and the
refusal of an output that is not 16-byte aligned."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from sam_road_b200 import _lib

DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _operands(M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(torch.float16).to(DEV)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.float16).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    return A, W, bias


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("N,K", [(768, 768), (800, 768), (96, 768), (768, 3072), (800, 3072)])
def test_f16_epilogue_matches_f32_epilogue(N, K, act):
    lib = _lib.load()
    M = 128 * 3 + 37
    A, W, bias = _operands(M, N, K, seed=N + K + act)
    ldo = N + 64
    out16 = torch.full((M, ldo), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(lib.samroad_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), act,
                                       out16.data_ptr(), ldo, _st()), "gemm_f16")
    out32 = torch.full((M, N), float("nan"), device=DEV)
    _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), None, None, 0,
                                       out32.data_ptr(), N, _st()), "gemm_f32")
    torch.cuda.synchronize()
    assert torch.isnan(out16[:, N:].float()).all(), "columns past N were written"
    got = out16[:, :N]
    if act == 1:       # the kernel's GELU is a polynomial fit, within 6.1e-6 of erf GELU
        err = (got.float() - F.gelu(out32).half().float()).abs()
        assert (err <= 2e-5 + 1e-3 * out32.abs()).all(), f"max abs err {err.max().item()}"
    else:
        ref = (F.relu(out32) if act == 2 else out32).half()
        assert torch.equal(got, ref)


def test_f16_epilogue_refuses_unaligned_output():
    # checked before any CUDA call, so this needs no GPU
    lib = _lib.load()
    rc = lib.samroad_op_gemm_f16(None, 64, None, 64, 128, 128, 64, None, 0, ctypes.c_void_p(8), 128, None)
    assert rc != 0 and "16-byte aligned" in _lib.last_error()
