"""Drop-in `SAMRoad` for the tiled-inference hot path of htcr/sam_road, backed by libsamroad_b200.so.

Mirrors the reference's model-level interface (reference model.py):
    SAMRoad(config)                                              model.py:193
    .load_state_dict(ckpt["state_dict"], strict=True)            inferencer.py:250-252
    .forward(rgb, graph_points, pairs, valid)                    model.py:414-457
    .infer_masks_and_img_features(rgb)                           model.py:459-495
    .infer_toponet(image_embeddings, graph_points, pairs, valid) model.py:498-508
with the same state_dict key set (SURVEY.md §8b), argument meaning and output shapes/dtypes.

Host side is Python/PyTorch only as plumbing (parameters, device memory, streams); all model math
runs in the hand-written sm_90a kernels behind the C ABI (include/samroad_b200.h).  There is no
PyTorch / CPU fallback: without the shared library or a CUDA device the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from typing import Dict, Optional, Tuple

import torch
from torch import nn

from . import _lib

_VIT = {  # model.py:198-218
    "vit_b": (768, 12, 12, (2, 5, 8, 11)),
    "vit_l": (1024, 24, 16, (5, 11, 17, 23)),
    "vit_h": (1280, 32, 16, (7, 15, 23, 31)),
}
# persistent buffers (state_dict entries that are not parameters): the random-Fourier PE matrix
BUFFER_KEYS = ("prompt_encoder.pe_layer.positional_encoding_gaussian_matrix",)
_TOPO_VERSION = {"no_offset": _lib.TOPO_NO_OFFSET, "no_transformer": _lib.TOPO_NO_TRANSFORMER}


def _cfg_get(config, key, default=None):
    """Config access that tolerates addict.Dict (missing key -> empty falsy Dict, utils.py:6-9),
    plain dicts and attribute-style namespaces."""
    if isinstance(config, dict):
        v = config.get(key, default)
    else:
        v = getattr(config, key, default)
    if v is None or (isinstance(v, dict) and len(v) == 0):
        return default
    return v


def param_shapes(config) -> Dict[str, Tuple[int, ...]]:
    """The reference's parameter names and shapes for this config (SURVEY.md §8b)."""
    version = _cfg_get(config, "SAM_VERSION", "vit_b")
    assert version in _VIT, f"SAM_VERSION must be one of {sorted(_VIT)}"   # model.py:197
    D, depth, heads, glob = _VIT[version]
    P = int(_cfg_get(config, "PATCH_SIZE"))
    s, hd = P // 16, D // heads
    lora = int(_cfg_get(config, "LORA_RANK", 0)) if _cfg_get(config, "ENCODER_LORA", False) else 0
    sh: Dict[str, Tuple[int, ...]] = {}
    e = "image_encoder."
    sh[e + "pos_embed"] = (1, s, s, D)
    sh[e + "patch_embed.proj.weight"] = (D, 3, 16, 16)
    sh[e + "patch_embed.proj.bias"] = (D,)
    for i in range(depth):
        p = f"{e}blocks.{i}."
        rows = 2 * s - 1 if i in glob else 2 * 14 - 1
        sh[p + "norm1.weight"] = (D,); sh[p + "norm1.bias"] = (D,)
        sh[p + "attn.rel_pos_h"] = (rows, hd); sh[p + "attn.rel_pos_w"] = (rows, hd)
        sh[p + "attn.qkv.weight"] = (3 * D, D); sh[p + "attn.qkv.bias"] = (3 * D,)
        if lora:
            sh[p + "attn.qkv.linear_a_q.weight"] = (lora, D); sh[p + "attn.qkv.linear_b_q.weight"] = (D, lora)
            sh[p + "attn.qkv.linear_a_v.weight"] = (lora, D); sh[p + "attn.qkv.linear_b_v.weight"] = (D, lora)
        sh[p + "attn.proj.weight"] = (D, D); sh[p + "attn.proj.bias"] = (D,)
        sh[p + "norm2.weight"] = (D,); sh[p + "norm2.bias"] = (D,)
        sh[p + "mlp.lin1.weight"] = (4 * D, D); sh[p + "mlp.lin1.bias"] = (4 * D,)
        sh[p + "mlp.lin2.weight"] = (D, 4 * D); sh[p + "mlp.lin2.bias"] = (D,)
    sh[e + "neck.0.weight"] = (256, D, 1, 1)
    sh[e + "neck.1.weight"] = (256,); sh[e + "neck.1.bias"] = (256,)
    sh[e + "neck.2.weight"] = (256, 256, 3, 3)
    sh[e + "neck.3.weight"] = (256,); sh[e + "neck.3.bias"] = (256,)
    if _cfg_get(config, "USE_SAM_DECODER", False):
        # prompt_encoder (only no_mask_embed and the PE matrix are used on this path, the rest must
        # exist for strict checkpoint loading) + mask_decoder (model.py:260-282)
        pe = "prompt_encoder."
        sh[pe + BUFFER_KEYS[0][len(pe):]] = (2, 128)
        for i in range(4):
            sh[pe + f"point_embeddings.{i}.weight"] = (1, 256)
        sh[pe + "not_a_point_embed.weight"] = (1, 256)
        sh[pe + "mask_downscaling.0.weight"] = (4, 1, 2, 2); sh[pe + "mask_downscaling.0.bias"] = (4,)
        sh[pe + "mask_downscaling.1.weight"] = (4,); sh[pe + "mask_downscaling.1.bias"] = (4,)
        sh[pe + "mask_downscaling.3.weight"] = (16, 4, 2, 2); sh[pe + "mask_downscaling.3.bias"] = (16,)
        sh[pe + "mask_downscaling.4.weight"] = (16,); sh[pe + "mask_downscaling.4.bias"] = (16,)
        sh[pe + "mask_downscaling.6.weight"] = (256, 16, 1, 1); sh[pe + "mask_downscaling.6.bias"] = (256,)
        sh[pe + "no_mask_embed.weight"] = (1, 256)
        md = "mask_decoder."

        def attn(prefix, internal):
            for nm in ("q_proj", "k_proj", "v_proj"):
                sh[prefix + nm + ".weight"] = (internal, 256); sh[prefix + nm + ".bias"] = (internal,)
            sh[prefix + "out_proj.weight"] = (256, internal); sh[prefix + "out_proj.bias"] = (256,)
        for l in range(2):
            p = f"{md}transformer.layers.{l}."
            attn(p + "self_attn.", 256)
            attn(p + "cross_attn_token_to_image.", 128)
            attn(p + "cross_attn_image_to_token.", 128)
            for n in (1, 2, 3, 4):
                sh[p + f"norm{n}.weight"] = (256,); sh[p + f"norm{n}.bias"] = (256,)
            sh[p + "mlp.lin1.weight"] = (2048, 256); sh[p + "mlp.lin1.bias"] = (2048,)
            sh[p + "mlp.lin2.weight"] = (256, 2048); sh[p + "mlp.lin2.bias"] = (256,)
        attn(md + "transformer.final_attn_token_to_image.", 128)
        sh[md + "transformer.norm_final_attn.weight"] = (256,); sh[md + "transformer.norm_final_attn.bias"] = (256,)
        sh[md + "iou_token.weight"] = (1, 256); sh[md + "mask_tokens.weight"] = (3, 256)
        sh[md + "output_upscaling.0.weight"] = (256, 64, 2, 2); sh[md + "output_upscaling.0.bias"] = (64,)
        sh[md + "output_upscaling.1.weight"] = (64,); sh[md + "output_upscaling.1.bias"] = (64,)
        sh[md + "output_upscaling.3.weight"] = (64, 32, 2, 2); sh[md + "output_upscaling.3.bias"] = (32,)
        for i in range(3):
            m = f"{md}output_hypernetworks_mlps.{i}.layers."
            sh[m + "0.weight"] = (256, 256); sh[m + "0.bias"] = (256,)
            sh[m + "1.weight"] = (256, 256); sh[m + "1.bias"] = (256,)
            sh[m + "2.weight"] = (32, 256); sh[m + "2.bias"] = (32,)
        m = md + "iou_prediction_head.layers."
        sh[m + "0.weight"] = (256, 256); sh[m + "0.bias"] = (256,)
        sh[m + "1.weight"] = (256, 256); sh[m + "1.bias"] = (256,)
        sh[m + "2.weight"] = (3, 256); sh[m + "2.bias"] = (3,)
    else:
        for idx, (cin, cout) in zip((0, 3, 5, 7), ((256, 128), (128, 64), (64, 32), (32, 2))):
            sh[f"map_decoder.{idx}.weight"] = (cin, cout, 2, 2)
            sh[f"map_decoder.{idx}.bias"] = (cout,)
        sh["map_decoder.1.weight"] = (128,); sh["map_decoder.1.bias"] = (128,)
    t = "topo_net."
    sh[t + "feature_proj.weight"] = (128, 256); sh[t + "feature_proj.bias"] = (128,)
    sh[t + "pair_proj.weight"] = (128, 258); sh[t + "pair_proj.bias"] = (128,)
    if _cfg_get(config, "TOPONET_VERSION", "normal") != "no_transformer":
        for l in range(3):
            p = f"{t}transformer_encoder.layers.{l}."
            sh[p + "self_attn.in_proj_weight"] = (384, 128); sh[p + "self_attn.in_proj_bias"] = (384,)
            sh[p + "self_attn.out_proj.weight"] = (128, 128); sh[p + "self_attn.out_proj.bias"] = (128,)
            sh[p + "linear1.weight"] = (128, 128); sh[p + "linear1.bias"] = (128,)
            sh[p + "linear2.weight"] = (128, 128); sh[p + "linear2.bias"] = (128,)
            sh[p + "norm1.weight"] = (128,); sh[p + "norm1.bias"] = (128,)
            sh[p + "norm2.weight"] = (128,); sh[p + "norm2.bias"] = (128,)
    sh[t + "output_proj.weight"] = (1, 128); sh[t + "output_proj.bias"] = (1,)
    return sh


class _Node(nn.Module):
    """Parameter container; nested so that state_dict() keys equal the reference's."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container, not callable")


def _register(root: nn.Module, key: str, p: nn.Parameter) -> None:
    parts = key.split(".")
    node = root
    for name in parts[:-1]:
        if name not in node._modules:
            node.add_module(name, _Node())
        node = node._modules[name]
    node.register_parameter(parts[-1], p)


def _register_buffer(root: nn.Module, key: str, t: torch.Tensor) -> None:
    parts = key.split(".")
    node = root
    for name in parts[:-1]:
        if name not in node._modules:
            node.add_module(name, _Node())
        node = node._modules[name]
    node.register_buffer(parts[-1], t, persistent=True)


try:  # the reference derives from LightningModule (model.py:190); use it when importable
    import lightning.pytorch as _pl
    _Base = _pl.LightningModule
except Exception:  # lightning is absent in this image; inference needs nothing Lightning-specific
    _Base = nn.Module


class SAMRoad(_Base):
    """H100-native SAMRoad: inference, test, validation, and training of the heads with a frozen encoder."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        if _cfg_get(config, "NO_SAM", False):
            raise NotImplementedError(   # same behaviour as the reference (model.py:232-242)
                "This ablation experiment depends on detectron2 and is not part of the release.")
        self._shapes = param_shapes(config)
        version = _cfg_get(config, "SAM_VERSION", "vit_b")
        self._vit = _VIT[version]
        self.image_size = int(_cfg_get(config, "PATCH_SIZE"))
        gen = torch.Generator().manual_seed(0)
        for key, shape in self._shapes.items():
            if key.endswith("norm1.weight") or key.endswith("norm2.weight") or \
                    key in ("image_encoder.neck.1.weight", "image_encoder.neck.3.weight",
                            "map_decoder.1.weight"):
                init = torch.ones(shape)
            elif key.endswith(".bias") or "rel_pos" in key or key.endswith("pos_embed") or \
                    "linear_b_" in key:
                init = torch.zeros(shape)
            else:
                fan_in = 1
                for d in shape[1:]:
                    fan_in *= d
                init = (torch.rand(shape, generator=gen) * 2 - 1) / max(1.0, fan_in) ** 0.5
            if key in BUFFER_KEYS:
                _register_buffer(self, key, torch.randn(shape, generator=gen))
            else:
                _register(self, key, nn.Parameter(init, requires_grad=False))
        self.register_buffer("pixel_mean", torch.tensor([123.675, 116.28, 103.53]).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor([58.395, 57.12, 57.375]).view(-1, 1, 1), False)
        self._handles: Dict[int, _lib.Handle] = {}     # cuda device index -> samroad_handle_t
        self._weights_version = 0
        self._synced_version: Dict[int, int] = {}
        self._packed_versions: Dict[int, Dict[str, int]] = {}   # device -> key -> _version at the last pack
        self._test_curves = None               # (keypoint, road, topo) PrecisionRecallCurve, see test_step
        self.best_thresholds = None
        self.focal_loss = bool(_cfg_get(config, "FOCAL_LOSS", False))   # mask criterion, model.py:350-353
        self._val_metrics = None               # ValidationMetrics, see validation_step
        self.val_metrics = None
        self.matched_param_names = set()
        ckpt_path = _cfg_get(config, "SAM_CKPT_PATH", None)
        if ckpt_path and os.path.isfile(str(ckpt_path)):
            self._load_sam_checkpoint(str(ckpt_path))   # model.py:367-390

    # ---- weights -----------------------------------------------------------------------------
    def _load_sam_checkpoint(self, path: str) -> None:
        """Initialise from a SAM checkpoint like model.py:367-411: resize pos_embed and the global
        blocks' rel-pos tables to this tile size, then load every name+shape match (non-strict)."""
        import torch.nn.functional as F
        sd = torch.load(path, map_location="cpu")
        s = self.image_size // 16
        glob = self._vit[3]
        if "image_encoder.pos_embed" in sd and sd["image_encoder.pos_embed"].shape[1] != s:
            pe = sd["image_encoder.pos_embed"].permute(0, 3, 1, 2)
            sd["image_encoder.pos_embed"] = F.interpolate(
                pe, (s, s), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
            for i in glob:
                for ax in ("h", "w"):
                    k = f"image_encoder.blocks.{i}.attn.rel_pos_{ax}"
                    if k in sd:
                        t = sd[k][None, None]
                        sd[k] = F.interpolate(t, (2 * s - 1, t.shape[-1]), mode="bilinear",
                                              align_corners=False)[0, 0]
        own = dict(self.named_parameters())   # like the reference: parameters only (model.py:378)
        matched = {k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}
        self.matched_param_names = set(matched)
        self.load_state_dict(matched, strict=False)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._weights_version += 1
        return out

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.__dict__.pop("_heads_cache", None)   # conversions may swap the parameter objects
        self._weights_version += 1
        return out

    def mark_weights_dirty(self) -> None:
        """Call after mutating parameters in place so the packed device weights are rebuilt."""
        self._weights_version += 1

    def _handle(self, device: torch.device) -> _lib.Handle:
        if device.type != "cuda":
            raise RuntimeError(
                f"sam_road_b200.SAMRoad runs on CUDA (sm_90a) only; got input on '{device}'. "
                "There is no CPU path.")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        lib = _lib.load()
        if idx not in self._handles:
            D, depth, heads, glob = self._vit
            cfg = _lib.SamRoadCfg()
            cfg.patch_size, cfg.embed_dim, cfg.depth, cfg.num_heads = self.image_size, D, depth, heads
            cfg.window_size = 14
            for i, g in enumerate(glob):
                cfg.global_attn_indexes[i] = g
            cfg.use_sam_decoder = 1 if _cfg_get(self.config, "USE_SAM_DECODER", False) else 0
            cfg.toponet_version = _TOPO_VERSION.get(
                _cfg_get(self.config, "TOPONET_VERSION", "normal"), _lib.TOPO_NORMAL)
            cfg.lora_rank = (int(_cfg_get(self.config, "LORA_RANK", 0))
                             if _cfg_get(self.config, "ENCODER_LORA", False) else 0)
            self._handles[idx] = _lib.Handle("samroad_create", "samroad_destroy", C.byref(cfg), idx)
        # parameters that require grad (the trained heads) are watched through their autograd version
        # counter: an optimizer step changes them in place, and only those are repacked, on the device
        watched = [(k, p) for k, p in self._head_params() if p.requires_grad]
        seen = self._packed_versions.setdefault(idx, {})
        stale = [(k, p) for k, p in watched if seen.get(k) != p._version]
        if stale and self._synced_version.get(idx) == self._weights_version and any(
                p.device != device or p.dtype != torch.float32 or not p.is_contiguous() for _, p in stale):
            self._weights_version += 1     # not device-resident fp32: repack on the host
        if self._synced_version.get(idx) != self._weights_version:
            h = self._handles[idx]
            tensors = list(self.named_parameters()) + [(k, b) for k, b in self.named_buffers()
                                                        if k in BUFFER_KEYS]
            for key, p in tensors:
                t = p.detach().to(device="cpu", dtype=torch.float32).contiguous()
                shape = (C.c_int64 * t.dim())(*t.shape)
                _lib.check(lib.samroad_load_tensor(h, key.encode(), t.data_ptr(), shape, t.dim()),
                           f"samroad_load_tensor({key})")
            _lib.check(lib.samroad_finalize_weights(h), "samroad_finalize_weights")
            self._synced_version[idx] = self._weights_version
        elif stale:
            h = self._handles[idx]
            with torch.cuda.device(device):
                for key, p in stale:
                    shape = (C.c_int64 * p.dim())(*p.shape)
                    _lib.check(lib.samroad_update_tensor_device(h, key.encode(), p.data_ptr(), shape, p.dim(),
                                                                _lib.current_stream_ptr()),
                               f"samroad_update_tensor_device({key})")
        for k, p in watched:
            seen[k] = p._version
        return self._handles[idx]

    # C handles are owned by exactly one Python object: copies / unpickled objects create their own
    # on first use (copy.deepcopy of a module would otherwise destroy the same handle twice).
    def __getstate__(self):
        state = dict(self.__dict__)
        state["_handles"] = {}
        state["_synced_version"] = {}
        state["_packed_versions"] = {}
        state["_test_curves"] = None
        state["_val_metrics"] = None
        return state

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_handles", "_synced_version", "_packed_versions"):
                new.__dict__[k] = {}
            elif k in ("_test_curves", "_val_metrics"):
                new.__dict__[k] = None
            else:
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    # ---- inference entry points ----------------------------------------------------------------------
    @staticmethod
    def _prep_rgb(rgb: torch.Tensor):
        if rgb.dtype == torch.uint8:
            return rgb.contiguous(), _lib.U8
        return rgb.to(torch.float32).contiguous(), _lib.F32

    def _out_buffers(self, B, device, want_logits, out_scores, out_emb):
        P, s = self.image_size, self.image_size // 16
        if out_scores is None:
            out_scores = torch.empty((B, P, P, 2), dtype=torch.float32, device=device)
        if out_emb is None:
            out_emb = torch.empty((B, 256, s, s), dtype=torch.float32, device=device)
        for t, shape in ((out_scores, (B, P, P, 2)), (out_emb, (B, 256, s, s))):
            if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous() or \
                    t.device != device:
                raise ValueError(f"output buffer must be contiguous float32 {shape} on {device}")
        logits = torch.empty_like(out_scores) if want_logits else None
        return out_scores, logits, out_emb

    def _encode(self, rgb: torch.Tensor, want_logits: bool, out_scores=None, out_emb=None):
        if rgb.dim() != 4 or rgb.shape[-1] != 3 or rgb.shape[1] != self.image_size or \
                rgb.shape[2] != self.image_size:
            raise ValueError(f"rgb must be [B,{self.image_size},{self.image_size},3], got "
                             f"{tuple(rgb.shape)}")
        h = self._handle(rgb.device)
        B = rgb.shape[0]
        x, dt = self._prep_rgb(rgb)
        scores, logits, emb = self._out_buffers(B, rgb.device, want_logits, out_scores, out_emb)
        if B > 0:
            with torch.cuda.device(rgb.device):
                _lib.check(_lib.load().samroad_encode_masks(
                    h, x.data_ptr(), dt, B, scores.data_ptr(), _lib.ptr(logits), emb.data_ptr(),
                    _lib.current_stream_ptr()), "samroad_encode_masks")
        return scores, logits, emb

    @torch.no_grad()
    def infer_masks_and_img_features_scene(self, scene_u8: torch.Tensor, tile_xy: torch.Tensor,
                                           out_scores=None, out_emb=None):
        """`infer_masks_and_img_features` for tiles that are windows of a uint8 scene [H,W,3] already
        on the device: tile_xy = host int [B,2] origins (x0,y0).  Replaces the host crops and the float32
        upload of inferencer.py:43-58,87-96; results equal those of the cropped-tile call bit for bit."""
        if scene_u8.dtype != torch.uint8 or scene_u8.dim() != 3 or scene_u8.shape[-1] != 3 or \
                not scene_u8.is_contiguous():
            raise ValueError("scene must be a contiguous uint8 [H,W,3] tensor")
        dev = scene_u8.device
        h = self._handle(dev)
        xy_host = torch.as_tensor(tile_xy).to(device="cpu", dtype=torch.int32).reshape(-1, 2).contiguous()
        B = xy_host.shape[0]
        H, W = int(scene_u8.shape[0]), int(scene_u8.shape[1])
        P = self.image_size
        if B > 0:    # validated on the host (origins come from the host tile list): no device sync
            lo, hi = xy_host.min(dim=0).values.tolist(), xy_host.max(dim=0).values.tolist()
            if lo[0] < 0 or lo[1] < 0 or hi[0] + P > W or hi[1] + P > H:
                raise ValueError("tile origin outside the scene")
        xy = xy_host.to(dev, non_blocking=True)
        scores, _, emb = self._out_buffers(B, dev, False, out_scores, out_emb)
        if B > 0:
            with torch.cuda.device(dev):
                _lib.check(_lib.load().samroad_encode_masks_scene(
                    h, scene_u8.data_ptr(), H, W, xy.data_ptr(), B, scores.data_ptr(), None,
                    emb.data_ptr(), _lib.current_stream_ptr()), "samroad_encode_masks_scene")
        return scores, emb

    def _topo(self, image_embeddings, graph_points, pairs, valid, want_logits: bool, out_scores=None):
        dev = image_embeddings.device
        h = self._handle(dev)
        if pairs.dim() != 4 or pairs.shape[-1] != 2 or graph_points.dim() != 3 or \
                graph_points.shape[-1] != 2 or tuple(valid.shape) != tuple(pairs.shape[:3]):
            raise ValueError("expected graph_points [B,N,2], pairs [B,Ns,Np,2], valid [B,Ns,Np]; got "
                             f"{tuple(graph_points.shape)}, {tuple(pairs.shape)}, {tuple(valid.shape)}")
        B, Ns, Np = pairs.shape[0], pairs.shape[1], pairs.shape[2]
        N = graph_points.shape[1]
        s = self.image_size // 16
        if tuple(image_embeddings.shape) != (B, 256, s, s) or graph_points.shape[0] != B:
            raise ValueError(f"image_embeddings must be [{B},256,{s},{s}] and graph_points [{B},N,2]; got "
                             f"{tuple(image_embeddings.shape)}, {tuple(graph_points.shape)}")
        for name, t in (("graph_points", graph_points), ("pairs", pairs), ("valid", valid)):
            if t.device != dev:     # the reference raises a device-mismatch error here as well
                raise RuntimeError(f"{name} is on {t.device} but image_embeddings is on {dev}")
        emb = image_embeddings.to(torch.float32).contiguous()
        if graph_points.dtype == torch.int64:
            pts, pdt = graph_points.contiguous(), _lib.I64
        elif graph_points.dtype == torch.int32:
            pts, pdt = graph_points.contiguous(), _lib.I32
        else:
            pts, pdt = graph_points.to(torch.float32).contiguous(), _lib.F32
        if pairs.dtype == torch.int32:
            prs, qdt = pairs.contiguous(), _lib.I32
        else:
            prs, qdt = pairs.to(torch.int64).contiguous(), _lib.I64
        val = valid.contiguous() if valid.dtype == torch.uint8 else \
            valid.to(torch.bool).contiguous().view(torch.uint8)
        if out_scores is None:
            scores = torch.empty((B, Ns, Np, 1), dtype=torch.float32, device=dev)
        else:
            scores = out_scores
            if scores.numel() != B * Ns * Np or scores.dtype != torch.float32 or \
                    not scores.is_contiguous() or scores.device != dev:
                raise ValueError("out_scores must be a contiguous float32 buffer of B*Ns*Np elements")
        logits = torch.empty((B, Ns, Np, 1), dtype=torch.float32, device=dev) if want_logits else None
        if B * Ns * Np > 0:
            # emb / pts / prs / val stay referenced until the call returns (stream-ordered kernels
            # launched by it read them; the caching allocator reuses freed blocks only stream-ordered)
            with torch.cuda.device(dev):
                _lib.check(_lib.load().samroad_toponet(
                    h, emb.data_ptr(), pts.data_ptr(), pdt, prs.data_ptr(), qdt, val.data_ptr(), B, N,
                    Ns, Np, _lib.ptr(logits), scores.data_ptr(), _lib.current_stream_ptr()),
                    "samroad_toponet")
        return logits, scores

    @torch.no_grad()
    def forward(self, rgb, graph_points, pairs, valid):
        """(mask_logits[B,H,W,2], mask_scores[B,H,W,2], topo_logits[B,Ns,Np,1], topo_scores) --
        model.py:414-457.  Inference only: no autograd graph is produced."""
        scores, logits, emb = self._encode(rgb, True)
        t_logits, t_scores = self._topo(emb, graph_points, pairs, valid, True)
        return logits, scores, t_logits, t_scores

    @torch.no_grad()
    def infer_masks_and_img_features(self, rgb):
        """(mask_scores[B,H,W,2], image_embeddings[B,256,H/16,W/16]) -- model.py:459-495."""
        scores, _, emb = self._encode(rgb, False)
        return scores, emb

    @torch.no_grad()
    def infer_toponet(self, image_embeddings, graph_points, pairs, valid, out=None):
        """topo_scores[B,Ns,Np,1] -- model.py:498-508.  `out` (extension): a contiguous float32 buffer
        of B*Ns*Np elements the scores are written into."""
        return self._topo(image_embeddings, graph_points, pairs, valid, False, out_scores=out)[1]

    # ---- training of the heads with a frozen encoder (train.py, FREEZE_ENCODER: True) ---------------------------
    _TRAIN_LOG = dict(on_step=True, on_epoch=False, prog_bar=True)    # model.py:541-543

    def _head_params(self):
        """(key, parameter) of map_decoder.* and topo_net.*, in registration order (cached: the inference calls
        look at them on every call)."""
        heads = self.__dict__.get("_heads_cache")
        if heads is None:
            heads = [(k, p) for k, p in self.named_parameters() if k.startswith(("map_decoder.", "topo_net."))]
            self.__dict__["_heads_cache"] = heads
        return heads

    def _enable_training(self) -> None:
        """Head parameters require grad from here on (the encoder's stay frozen), so that autograd fills their
        .grad and an optimizer step is repacked on the device before the next call."""
        from .train import check_trainable
        check_trainable(self.config, _cfg_get)
        if not self.__dict__.get("_training_enabled", False):   # once: a head frozen later by the user stays so
            for _, p in self._head_params():
                p.requires_grad_(True)
            self._training_enabled = True

    def setup(self, stage: Optional[str] = None) -> None:
        """Lightning's setup hook, which runs before its DDP strategy wraps the module: for stage "fit" the head
        parameters start requiring grad here, since DistributedDataParallel only reduces (and only accepts a
        module with) parameters that require grad at wrap time.  Unsupported configurations raise here."""
        if stage == "fit":
            self._enable_training()

    def training_step(self, batch, batch_idx):
        """model.py:511-544 for FREEZE_ENCODER: True with the naive decoder: the encoder as the inference calls run
        it, then the map decoder and TopoNet (dropout 0.1 at torch's four sites when self.training) on the device,
        mask loss (BCEWithLogitsLoss, or sigmoid_focal_loss with FOCAL_LOSS) + the valid-slot topology BCE.  Returns
        the 0-dim fp32 loss, differentiable with respect to the map_decoder.* and topo_net.* parameters; its
        backward writes their .grad on the device (DESIGN.md §12).  Other configurations raise NotImplementedError
        before the batch is read.  The dropout seed is drawn from torch's default generator and, under
        torch.distributed, made per rank (ranks.rank_seed; rank 0 keeps it).  Wrapped in DistributedDataParallel
        (after setup("fit")), DDP's averaged gradients land in the heads' .grad."""
        from . import train as T
        self._enable_training()
        heads = self._head_params()
        dev = heads[0][1].device
        if dev.type != "cuda":
            raise RuntimeError(f"training runs on CUDA (sm_90a) only; the head parameters are on '{dev}'")
        b = T.validate_batch(batch, self.image_size, dev)
        h = self._handle(dev)
        dropout_p = 0.1 if self.training else 0.0
        from .ranks import draw_seed
        seed = draw_seed() if dropout_p > 0 else 0
        args = T.make_args(b, self.focal_loss, dropout_p, seed)
        mask_loss, topo_loss = T.head_losses(h, b, args, [k for k, _ in heads], [p for _, p in heads])
        loss = mask_loss + topo_loss
        if self._attached():
            self.log("train_mask_loss", mask_loss, **self._TRAIN_LOG)
            self.log("train_topo_loss", topo_loss, **self._TRAIN_LOG)
            self.log("train_loss", loss, **self._TRAIN_LOG)
        return loss

    def configure_optimizers(self):
        """model.py:637-685 for FREEZE_ENCODER: True with the naive decoder: Adam over map_decoder then topo_net,
        both at BASE_LR, and MultiStepLR(milestones=[9], gamma=0.1).  Prints the parameter count of each group as
        the reference does."""
        self._enable_training()
        lr = _cfg_get(self.config, "BASE_LR")
        groups = [{"params": [p for k, p in self._head_params() if k.startswith(prefix)], "lr": lr}
                  for prefix in ("map_decoder.", "topo_net.")]
        for i, g in enumerate(groups):
            print(f"optim param dict {i} params num: {sum(int(p.numel()) for p in g['params'])}")
        optimizer = torch.optim.Adam(groups, lr=lr)
        step_lr = torch.optim.lr_scheduler.MultiStepLR(optimizer, milestones=[9, ], gamma=0.1)
        return {"optimizer": optimizer, "lr_scheduler": step_lr}

    # ---- validation (train.py's per-epoch loop, trainer.validate) -----------------------------------
    _VAL_LOG = dict(on_step=False, on_epoch=True, prog_bar=True)    # model.py:566-568

    def _attached(self) -> bool:
        """True when a Lightning trainer drives this module (then self.log is Lightning's)."""
        return self.__dict__.get("_trainer") is not None

    @torch.no_grad()
    def validation_step(self, batch, batch_idx):
        """model.py:547-588 without autograd: the forward pass, the mask loss (BCEWithLogitsLoss, or
        sigmoid_focal_loss with FOCAL_LOSS) and the valid-slot topology BCE, and the updates of keypoint_iou,
        road_iou and topo_f1, all on the device (sam_road_b200.metrics.ValidationMetrics, DESIGN.md §11).
        batch is the reference's collated dict (masks float 0.0 / 1.0, valid / connected bool).  Returns
        {"val_mask_loss", "val_topo_loss", "val_loss"} as 0-dim float32 device tensors and, under a Lightning
        trainer, logs them with the reference's names and flags.  A step with a target other than 0 / 1
        adds nothing and makes on_validation_epoch_end raise.  Autocast is ignored, as by the inference
        calls.  The wandb image table the reference logs at batch_idx == 0 is visualisation and not served
        (DESIGN.md §7)."""
        from .metrics import VAL_LOSS_NAMES, ValidationMetrics
        rgb, valid = batch["rgb"], batch["valid"]
        scores, logits, emb = self._encode(rgb, True)
        t_logits, t_scores = self._topo(emb, batch["graph_points"], batch["pairs"], valid, True)
        if self._val_metrics is None:
            self._val_metrics = ValidationMetrics(rgb.device, focal=self.focal_loss)
        vm = self._val_metrics
        if vm.device != scores.device:
            raise RuntimeError(f"validation batches arrive on {scores.device}, the metrics were started on "
                               f"{vm.device}; call reset_validation_metrics() first")
        out = vm.update(logits, scores, batch["keypoint_mask"], batch["road_mask"], t_logits, t_scores,
                        batch["connected"], valid)
        res = dict(zip(VAL_LOSS_NAMES, out.unbind(0)))
        if self._attached():
            for name, v in res.items():
                self.log(name, v, **self._VAL_LOG)
        return res

    def on_validation_epoch_end(self):
        """model.py:591-600: keypoint_iou, road_iou and topo_f1 of the epoch (logged under a Lightning
        trainer), then the accumulator is reset.  Returns and stores in `val_metrics` a dict of the six
        numbers as Python floats: those three and the epoch means of val_mask_loss, val_topo_loss and val_loss
        (Lightning's batch-size-weighted on_epoch mean, taken exactly).  Under torch.distributed the counts of
        every rank are summed first, as torchmetrics' sync on compute does; the losses stay per rank.  Raises
        when a validation step was refused since the last report."""
        from .metrics import ValidationMetrics
        if self._val_metrics is None:
            dist = torch.distributed
            if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
                raise RuntimeError("on_validation_epoch_end: no validation_step ran since the last reset")
            # a rank without batches still joins the all-reduce of the counts
            self._val_metrics = ValidationMetrics(torch.device("cuda", torch.cuda.current_device()),
                                                  focal=self.focal_loss)
        vm = self._val_metrics
        try:
            res = vm.compute()
        finally:
            vm.reset()
        if self._attached():
            for name in ("keypoint_iou", "road_iou", "topo_f1"):
                self.log(name, torch.tensor(res[name], dtype=torch.float32, device=vm.device))
        self.val_metrics = res
        return res

    def reset_validation_metrics(self) -> None:
        """Drops the validation accumulator (its counts and loss sums) and `val_metrics`."""
        self._val_metrics = None
        self.val_metrics = None

    # ---- threshold search (test.py) ----------------------------------------------------------------
    _CURVE_NAMES = ("keypoint", "road", "topo")

    @torch.no_grad()
    def test_step(self, batch, batch_idx):
        """model.py:602-617: mask and topology scores of one evaluation batch go into three exact
        precision-recall curves (sam_road_b200.metrics).  batch is the reference's collated dict: rgb
        [B,P,P,3], keypoint_mask / road_mask [B,P,P] (float, label = int32(mask)), graph_points [B,N,2],
        pairs [B,Ns,Np,2], valid / connected [B,Ns,Np] bool.  Autocast is ignored, as by the inference
        calls: the scores are the engine's own."""
        from .metrics import PrecisionRecallCurve
        rgb, valid = batch["rgb"], batch["valid"]
        scores, _, emb = self._encode(rgb, False)
        _, topo_scores = self._topo(emb, batch["graph_points"], batch["pairs"], valid, False)
        if self._test_curves is None:
            self._test_curves = tuple(PrecisionRecallCurve(rgb.device) for _ in self._CURVE_NAMES)
        kp, road, topo = self._test_curves
        if kp.device != scores.device:
            raise RuntimeError(f"test batches arrive on {scores.device}, the curves were started on {kp.device}; "
                               "call reset_test_metrics() first")
        kp.update(scores[..., 0], batch["keypoint_mask"])
        road.update(scores[..., 1], batch["road_mask"])
        topo.update(topo_scores, batch["connected"], valid)   # valid == False is the reference's label -1

    def on_test_end(self):
        """model.py:619-634: prints the best-F1 threshold, precision, recall and F1 of each curve as
        Python floats (the form the configs record) and returns / stores them in `best_thresholds`:
        {"keypoint" | "road" | "topo": (threshold, P, R, F1)}.  Under torch.distributed (Lightning's DDP
        test loop) every rank reports the curves of the whole split: the ranks gather their entries
        (sam_road_b200.metrics), as torchmetrics' sync on compute does in the reference."""
        if self._test_curves is None:
            dist = torch.distributed
            if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
                raise RuntimeError("on_test_end: no test_step ran since the last reset_test_metrics()")
            from .metrics import PrecisionRecallCurve   # a rank without batches still joins the gathers
            dev = torch.device("cuda", torch.cuda.current_device())
            self._test_curves = tuple(PrecisionRecallCurve(dev) for _ in self._CURVE_NAMES)
        print("======= Finding best thresholds ======")
        best = {}
        for name, curve in zip(self._CURVE_NAMES, self._test_curves):
            print(f"======= {name} ======")
            thr, p, r, f1 = (t.item() for t in curve.best())
            print(f"Best threshold {thr}, P={p} R={r} F1={f1}")
            best[name] = (thr, p, r, f1)
        self.best_thresholds = best
        return best

    def reset_test_metrics(self) -> None:
        """Drops every entry of the three curves (they persist across test runs, like torchmetrics
        state, until this is called)."""
        self._test_curves = None      # the accumulators free their device memory
        self.best_thresholds = None
