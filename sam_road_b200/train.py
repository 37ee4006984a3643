"""Training of the heads with a frozen encoder: the autograd bridge behind SAMRoad.training_step.

`head_losses` runs one step's forward on the device (the encoder as the inference path runs it, then the map
decoder and TopoNet in fp32, saving their activations in a workspace tensor) and returns the differentiable
0-dim fp32 (mask_loss, topo_loss).  Their backward writes one fp32 gradient per head parameter in the reference
layout, so autograd, zero_grad, gradient accumulation and GradScaler work unmodified (DESIGN.md §12).  Given image
embeddings instead, the encoder does not run and the embeddings become a differentiable input of the step.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

import torch

from . import _lib

HEAD_PREFIXES = ("map_decoder.", "topo_net.")
MAX_PAIRS = 32


def check_trainable(config, cfg_get) -> None:
    """Raises NotImplementedError naming the config key whose backward is missing (before any batch is read)."""
    if cfg_get(config, "ENCODER_LORA", False):
        raise NotImplementedError(
            "training with ENCODER_LORA needs the encoder backward, which sam_road_b200 does not implement yet; "
            "only FREEZE_ENCODER: True training of the heads is served (DESIGN.md §12)")
    if not cfg_get(config, "FREEZE_ENCODER", False):
        raise NotImplementedError(
            "training with FREEZE_ENCODER false or missing needs the encoder backward, which sam_road_b200 does "
            "not implement yet; set FREEZE_ENCODER: True to train the heads (DESIGN.md §12)")
    if cfg_get(config, "USE_SAM_DECODER", False):
        raise NotImplementedError(
            "training with USE_SAM_DECODER needs the TwoWayTransformer backward, which sam_road_b200 does not "
            "implement; only the naive map decoder is trained (DESIGN.md §12)")


def _key_table(keys: Sequence[str]):
    enc = [k.encode() for k in keys]
    arr = (C.c_char_p * len(enc))(*enc)
    return arr, enc


def _ptr_table(tensors: Sequence[torch.Tensor]):
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _as_u8(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous() if t.dtype == torch.uint8 else t.to(torch.bool).contiguous().view(torch.uint8)


def validate_batch(batch, P: int, device: torch.device):
    """The step's tensors, checked and converted for the C ABI; raises before any launch."""
    need = ("rgb", "keypoint_mask", "road_mask", "graph_points", "pairs", "valid", "connected")
    if not isinstance(batch, dict) or any(k not in batch for k in need):
        raise ValueError(f"batch must be a dict with {need}")
    rgb = batch["rgb"]
    if rgb.dim() != 4 or tuple(rgb.shape[1:]) != (P, P, 3):
        raise ValueError(f"rgb must be [B,{P},{P},3], got {tuple(rgb.shape)}")
    B = rgb.shape[0]
    pts, pairs, valid, conn = batch["graph_points"], batch["pairs"], batch["valid"], batch["connected"]
    if pts.dim() != 3 or pts.shape[0] != B or pts.shape[2] != 2:
        raise ValueError(f"graph_points must be [{B},N,2], got {tuple(pts.shape)}")
    if pairs.dim() != 4 or pairs.shape[0] != B or pairs.shape[3] != 2:
        raise ValueError(f"pairs must be [{B},Ns,Np,2], got {tuple(pairs.shape)}")
    Ns, Np = pairs.shape[1], pairs.shape[2]
    if not 1 <= Np <= MAX_PAIRS:
        raise ValueError(f"pairs per sample (MAX_NEIGHBOR_QUERIES) must be in 1..{MAX_PAIRS}, got {Np}")
    for name, t in (("valid", valid), ("connected", conn)):
        if tuple(t.shape) != (B, Ns, Np):
            raise ValueError(f"{name} must be [{B},{Ns},{Np}], got {tuple(t.shape)}")
        if t.dtype not in (torch.bool, torch.uint8):
            raise ValueError(f"{name} must be bool or uint8, got {t.dtype}")
    for name in ("keypoint_mask", "road_mask"):
        t = batch[name]
        if tuple(t.shape) != (B, P, P) or not t.is_floating_point():
            raise ValueError(f"{name} must be a float [{B},{P},{P}] tensor, got {t.dtype} {tuple(t.shape)}")
    if pts.shape[1] < 1 or Ns < 1 or B < 1:
        raise ValueError("a training batch needs B, N and N_samples >= 1")
    if rgb.dtype not in (torch.uint8, torch.float32, torch.float16, torch.bfloat16, torch.float64):
        raise ValueError(f"rgb dtype {rgb.dtype} is not supported")
    if pairs.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"pairs must be int32 or int64, got {pairs.dtype}")
    for name in need:
        if batch[name].device != device:
            raise ValueError(f"{name} is on {batch[name].device}, the trained parameters are on {device}")
    if rgb.dtype == torch.uint8:
        x, xdt = rgb.contiguous(), _lib.U8
    else:
        x, xdt = rgb.to(torch.float32).contiguous(), _lib.F32
    if pts.dtype == torch.int64:
        p, pdt = pts.contiguous(), _lib.I64
    elif pts.dtype == torch.int32:
        p, pdt = pts.contiguous(), _lib.I32
    else:
        p, pdt = pts.to(torch.float32).contiguous(), _lib.F32
    q, qdt = pairs.contiguous(), (_lib.I64 if pairs.dtype == torch.int64 else _lib.I32)
    return dict(B=B, N=pts.shape[1], Ns=Ns, Np=Np, rgb=(x, xdt), points=(p, pdt), pairs=(q, qdt),
                valid=_as_u8(valid), connected=_as_u8(conn),
                kp=batch["keypoint_mask"].to(torch.float32).contiguous(),
                road=batch["road_mask"].to(torch.float32).contiguous())


def make_args(b: Dict, focal: bool, dropout_p: float, seed: int) -> _lib.SamRoadTrainArgs:
    a = _lib.SamRoadTrainArgs()
    a.B, a.N, a.Ns, a.Np = b["B"], b["N"], b["Ns"], b["Np"]
    a.loss_kind = _lib.LOSS_FOCAL if focal else _lib.LOSS_BCE
    a.dropout_p = float(dropout_p)
    a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return a


class _HeadLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, handle, b, args, keys, emb_out, emb, *params):
        lib = _lib.load()
        dev = params[0].device
        nbytes = C.c_size_t()
        _lib.check(lib.samroad_train_workspace_bytes(handle, C.byref(args), C.byref(nbytes)),
                   "samroad_train_workspace_bytes")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        losses = torch.empty(2, dtype=torch.float32, device=dev)
        karr, kref = _key_table(keys)
        parr = _ptr_table(params)
        (x, xdt), (p, pdt), (q, qdt) = b["rgb"], b["points"], b["pairs"]
        with torch.cuda.device(dev):
            if emb is None:
                _lib.check(lib.samroad_train_forward(
                    handle, C.byref(args), karr, parr, len(params), x.data_ptr(), xdt, p.data_ptr(), pdt,
                    q.data_ptr(), qdt, b["valid"].data_ptr(), b["connected"].data_ptr(), b["kp"].data_ptr(),
                    b["road"].data_ptr(), ws.data_ptr(), nbytes.value, losses.data_ptr(), _lib.ptr(emb_out),
                    _lib.current_stream_ptr()), "samroad_train_forward")
            else:
                e32 = emb.detach().to(torch.float32).contiguous()   # fp16 / bf16 from an autocast encoder
                _lib.check(lib.samroad_train_forward_embeddings(
                    handle, C.byref(args), karr, parr, len(params), e32.data_ptr(), p.data_ptr(), pdt, q.data_ptr(),
                    qdt, b["valid"].data_ptr(), b["connected"].data_ptr(), b["kp"].data_ptr(), b["road"].data_ptr(),
                    ws.data_ptr(), nbytes.value, losses.data_ptr(), _lib.current_stream_ptr()),
                    "samroad_train_forward_embeddings")
        ctx.save_for_backward(*params)   # an in-place change before backward is reported by autograd
        ctx.handle, ctx.args, ctx.keys, ctx.ws = handle, args, keys, ws   # ws frees itself with the graph
        ctx.emb = None if emb is None else torch.empty_like(emb, device="meta")   # dtype, shape and strides
        return losses[0].clone(), losses[1].clone()

    @staticmethod
    def backward(ctx, g_mask, g_topo):
        lib = _lib.load()
        params = ctx.saved_tensors
        dev = params[0].device
        zero = torch.zeros((), dtype=torch.float32, device=dev)
        g = torch.stack([zero if g_mask is None else g_mask.to(torch.float32),
                         zero if g_topo is None else g_topo.to(torch.float32)]).contiguous()
        want_params = any(ctx.needs_input_grad[6:])
        want_emb = ctx.emb is not None and ctx.needs_input_grad[5]
        grads = [torch.empty_like(p) for p in params] if want_params or ctx.emb is None else []
        karr, kref = _key_table(ctx.keys)
        gemb = None
        with torch.cuda.device(dev):
            if ctx.emb is None:
                _lib.check(lib.samroad_train_backward(
                    ctx.handle, C.byref(ctx.args), karr, _ptr_table(params), _ptr_table(grads), len(params),
                    ctx.ws.data_ptr(), ctx.ws.numel(), g.data_ptr(), _lib.current_stream_ptr()),
                    "samroad_train_backward")
            elif want_params or want_emb:
                g32 = torch.empty(ctx.emb.shape, dtype=torch.float32, device=dev) if want_emb else None
                _lib.check(lib.samroad_train_backward_embeddings(
                    ctx.handle, C.byref(ctx.args), karr, _ptr_table(params),
                    _ptr_table(grads) if want_params else None, len(params), ctx.ws.data_ptr(), ctx.ws.numel(),
                    g.data_ptr(), _lib.ptr(g32), _lib.current_stream_ptr()),
                    "samroad_train_backward_embeddings")
                if want_emb:   # the input's dtype and layout
                    gemb = torch.empty_like(ctx.emb, device=dev).copy_(g32)
        if not grads:
            return (None, None, None, None, None, gemb) + (None,) * len(params)
        return (None, None, None, None, None, gemb) + tuple(grads)


def head_losses(handle: int, b: Dict, args: _lib.SamRoadTrainArgs, keys: List[str], params: List[torch.Tensor],
                emb_out=None, image_embeddings=None):
    """(mask_loss, topo_loss), differentiable with respect to `params` (the head parameters named by `keys`).
    With `image_embeddings` ([B,256,P/16,P/16] on the parameters' device, fp32, fp16 or bf16) the encoder does not
    run: the heads take those embeddings, which are then a differentiable input too; their gradient comes back in
    their dtype and layout (DESIGN.md §12).  Only the gradients autograd asks for are computed."""
    return _HeadLosses.apply(handle, b, args, keys, emb_out, image_embeddings, *params)


def dropout_keep(p: float, seed: int, layer: int, site: int, n: int, device) -> torch.Tensor:
    """The keep mask (bool [n]) of one TopoNet dropout site, as the training step draws it (test hook)."""
    out = torch.empty(n, dtype=torch.uint8, device=device)
    with torch.cuda.device(out.device):
        _lib.check(_lib.load().samroad_debug_train_dropout_keep(float(p), int(seed) & 0xFFFFFFFFFFFFFFFF, layer,
                                                                 site, n, out.data_ptr(), _lib.current_stream_ptr()),
                   "samroad_debug_train_dropout_keep")
    return out.bool()
