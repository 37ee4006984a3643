"""The fp32 epilogue of the ping-pong GEMM (samroad_op_gemm_f32) at the limits the fp16 one is tested at
(test_gpu_gemm_f16_stores.py): out = acc + resid + bias + pos[m % pos_rows], summed in that order in fp32, must
equal the same sums taken in torch on the device over the kernel's own accumulators (samroad_op_gemm_f32 with no
operands), bit for bit.  Covered: an M tail, N = 96 and 800 (a last tile of one to three 32-column chunks), the
residual read in place from the output, and an output wider than N whose other columns must stay untouched.
The epilogue stores through a TMA map of the output, so an output that is not 16-byte aligned or whose row pitch is
narrower than N is refused before any launch."""
import ctypes
import math

import pytest
import torch

from sam_road_b200 import _lib

DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _operands(M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(torch.float16).to(DEV)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.float16).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    resid = torch.randn(M, N, generator=g).to(DEV)
    return A, W, bias, resid


def _f32(lib, A, W, M, N, K, bias, resid, pos, pos_rows, out, ldo):
    _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K,
                                       bias.data_ptr() if bias is not None else None,
                                       resid.data_ptr() if resid is not None else None,
                                       pos.data_ptr() if pos is not None else None, pos_rows,
                                       out.data_ptr(), ldo, _st()), "gemm_f32")


@pytest.mark.gpu
@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("use_pos", [False, True])
@pytest.mark.parametrize("N,K", [(768, 768), (800, 768), (96, 768), (800, 3072)])
def test_f32_epilogue_bit_exact(N, K, use_pos, in_place):
    lib = _lib.load()
    M = 128 * 3 + 37
    A, W, bias, resid = _operands(M, N, K, seed=N + K + 2 * use_pos + in_place)
    pos_rows = 64
    pos = torch.randn(pos_rows, N, generator=torch.Generator().manual_seed(N)).to(DEV) if use_pos else None
    acc = torch.full((M, N), float("nan"), device=DEV)
    _f32(lib, A, W, M, N, K, None, None, None, 0, acc, N)
    ldo = N + 32
    out = torch.full((M, ldo), float("nan"), device=DEV)
    if in_place:
        out[:, :N] = resid
        r = out
    else:
        r = torch.full((M, ldo), float("nan"), device=DEV)
        r[:, :N] = resid
    _f32(lib, A, W, M, N, K, bias, r, pos, pos_rows if use_pos else 0, out, ldo)
    torch.cuda.synchronize()
    assert torch.isnan(out[:, N:]).all(), "columns past N were written"
    ref = (acc + resid) + bias
    if use_pos:
        ref = ref + pos[torch.arange(M, device=DEV) % pos_rows]
    assert torch.equal(out[:, :N], ref)


# checked before any CUDA call, so these need no GPU
def test_f32_epilogue_refuses_pitch_below_n():
    lib = _lib.load()
    rc = lib.samroad_op_gemm_f32(None, 64, None, 64, 128, 256, 64, None, None, None, 0, ctypes.c_void_p(1024), 128,
                                 None)
    assert rc != 0 and "row pitch" in _lib.last_error()


def test_f32_epilogue_refuses_unaligned_output():
    lib = _lib.load()
    rc = lib.samroad_op_gemm_f32(None, 64, None, 64, 128, 128, 64, None, None, None, 0, ctypes.c_void_p(8), 128,
                                 None)
    assert rc != 0 and "16-byte aligned" in _lib.last_error()
