"""The ping-pong GEMM (gemm_pp_kernel: the two consumer warpgroups of a CTA take its 128x128 tiles in turn)
behind samroad_op_gemm_f16 / _f32, at the shapes where the alternation matters: CTAs with an odd tile
count, M / N / K tails, the in-place residual over several tiles per CTA, and launches of different
shapes back to back.  Each case is compared against the on-device SIMT checker GEMM with the epilogue
applied in torch, and a repeated call must give the same bits."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from sam_road_b200 import _lib  # noqa: E402

DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rand16(shape, scale, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.float16).to(DEV)


def _randf(shape, scale, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(M, N, K, seed):
    return _rand16((M, K), 1.0, seed), _rand16((N, K), 1.0 / math.sqrt(K), seed + 1)


def _simt(lib, A, W):
    M, K = A.shape
    N = W.shape[0]
    chk = torch.empty((M, N), dtype=torch.float32, device=DEV)
    _lib.check(lib.samroad_op_gemm_ref(A.data_ptr(), K, W.data_ptr(), K, M, N, K, chk.data_ptr(), N, _st()),
               "gemm_ref")
    return chk


def _f16(lib, A, W, bias, act):
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((M, N), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(lib.samroad_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(), act,
                                       out.data_ptr(), N, _st()), "gemm_f16")
    return out


def _f32(lib, A, W, bias, resid, pos, out):
    M, K = A.shape
    N = W.shape[0]
    _lib.check(lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K,
                                       bias.data_ptr() if bias is not None else None,
                                       resid.data_ptr() if resid is not None else None,
                                       pos.data_ptr() if pos is not None else None,
                                       pos.shape[0] if pos is not None else 0, out.data_ptr(), N, _st()),
               "gemm_f32")
    return out


def check_f16(lib, M, N, K, act, seed):
    A, W = _operands(M, N, K, seed)
    bias = _randf(N, 1.0, seed + 2)
    outs = [_f16(lib, A, W, bias, act) for _ in range(2)]
    ref = [lambda x: x, F.gelu, F.relu][act](_simt(lib, A, W) + bias)
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0].float()).all()
    err = (outs[0].float() - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), f"max abs err {err}"
    assert torch.equal(outs[0], outs[1])


def check_f32(lib, M, N, K, seed, pos_rows=0, bias=True, resid=True):
    A, W = _operands(M, N, K, seed)
    b = _randf(N, 1.0, seed + 2) if bias else None
    r = _randf((M, N), 2.0, seed + 3) if resid else None
    pos = _randf((pos_rows, N), 1.0, seed + 4) if pos_rows else None
    outs = [_f32(lib, A, W, b, r, pos, torch.full((M, N), float("nan"), device=DEV)) for _ in range(2)]
    ref = _simt(lib, A, W)
    if r is not None:
        ref = ref + r
    if b is not None:
        ref = ref + b
    if pos is not None:
        ref = ref + pos[torch.arange(M, device=DEV) % pos_rows]
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0]).all()
    err = (outs[0] - ref).abs().max().item()
    assert err < 2e-4 * max(1.0, ref.abs().max().item()), f"max abs err {err}"
    assert torch.equal(outs[0], outs[1])


# tile counts (N = 128: one tile per 128 rows) where the CTAs get 1, 2 or 3 tiles, or an odd number,
# so that one consumer runs one more tile than the other; "S" stands for the SM count
TILE_COUNTS = {"1": lambda S: 1, "2": lambda S: 2, "3": lambda S: 3, "S-1": lambda S: S - 1, "S": lambda S: S,
               "S+1": lambda S: S + 1, "2S-1": lambda S: 2 * S - 1, "2S+1": lambda S: 2 * S + 1}


def _tiles(spec):
    return TILE_COUNTS[spec](_sms())


@pytest.mark.parametrize("tiles", list(TILE_COUNTS))
def test_pingpong_tile_counts_f16(tiles):
    check_f16(_lib.load(), 128 * _tiles(tiles), 128, 256, 1, seed=10)


@pytest.mark.parametrize("tiles", list(TILE_COUNTS))
def test_pingpong_tile_counts_f32(tiles):
    check_f32(_lib.load(), 128 * _tiles(tiles), 128, 256, seed=20)


@pytest.mark.parametrize("tail", [1, 64, 127])
@pytest.mark.parametrize("N,K", [(128, 72), (384, 200), (640, 72)])
def test_pingpong_tails_f16(tail, N, K):
    check_f16(_lib.load(), 128 * 5 + tail, N, K, 2, seed=30)


@pytest.mark.parametrize("tail", [1, 64, 127])
@pytest.mark.parametrize("N,K", [(128, 200), (384, 72), (640, 200)])
def test_pingpong_tails_f32(tail, N, K):
    check_f32(_lib.load(), 128 * 7 + tail, N, K, seed=40)


def test_pingpong_inplace_shortcut():
    """out is resid (the encoder's x += proj(a)) with about six tiles per CTA."""
    lib = _lib.load()
    M, N, K = 128 * _sms() + 77, 768, 200
    A, W = _operands(M, N, K, 50)
    bias = _randf(N, 1.0, 52)
    resid = _randf((M, N), 2.0, 53)
    ref = _simt(lib, A, W) + resid + bias
    outs = []
    for _ in range(2):
        x = resid.clone()
        outs.append(_f32(lib, A, W, bias, x, None, x))
    torch.cuda.synchronize()
    assert (outs[0] - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
    assert torch.equal(outs[0], outs[1])


def test_pingpong_pos_rows_not_dividing_tile():
    """pos[m % pos_rows] with pos_rows = 100: the pos row wraps inside a tile and differs between the rows
    a thread holds."""
    check_f32(_lib.load(), 128 * 9 + 50, 256, 136, seed=60, pos_rows=100, resid=False)


def test_pingpong_plain_no_bias():
    check_f32(_lib.load(), 128 * 3 + 5, 128, 64, seed=70, bias=False, resid=False)


def test_pingpong_long_call_after_other_shape():
    """A long call right after calls of other shapes on the same stream, with no synchronisation between
    them: barrier phase state left over by one launch would corrupt the next."""
    lib = _lib.load()
    S = _sms()
    A1, W1 = _operands(128 * 3 + 1, 384, 72, 80)
    A2, W2 = _operands(128 * (3 * S + 1), 640, 768, 82)   # the checker's grid takes M < 65536
    b1, b2 = _randf(384, 1.0, 84), _randf(640, 1.0, 85)
    small = _f16(lib, A1, W1, b1, 0)
    long1 = _f16(lib, A2, W2, b2, 1)
    _f16(lib, A1, W1, b1, 0)
    long2 = _f16(lib, A2, W2, b2, 1)
    ref_small = _simt(lib, A1, W1) + b1
    ref_long = F.gelu(_simt(lib, A2, W2) + b2)
    torch.cuda.synchronize()
    assert (small.float() - ref_small).abs().max().item() <= 2e-3 * max(1.0, ref_small.abs().max().item())
    assert (long1.float() - ref_long).abs().max().item() <= 2e-3 * max(1.0, ref_long.abs().max().item())
    assert torch.equal(long1, long2)
