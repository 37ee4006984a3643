"""Torch restatement of the heads' training loss (reference model.py:286-295, 61-148, 511-544).

The naive map decoder and TopoNet in the semantics of torch's slow path of TransformerEncoderLayer (the
path a grad-enabled call takes): post-norm, key-padding mask, all-invalid rows flipped to all-valid, padded
query rows computed like the others, dropout at four sites per layer.  Dropout is injected: `keep` maps
(layer, site) to a bool keep mask (site 0 attention probabilities [rows,4,Np,Np]; 1 dropout1, 2 the dropout
between ReLU and linear2, 3 dropout2, each [tokens,128]), survivors scaled by 1 / (1 - p).  Gradients come
from torch.autograd on the parameters passed in.  The arithmetic runs in the dtype of the embeddings and
parameters: fp32 is the reference's own, float64 gives the rounding-free yardstick the device gradients are
measured against (the dropout scale stays the fp32 value of 1 / (1 - p), which is what the reference multiplies by).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F


def _ln2d(x, w, b, eps=1e-6):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def mask_logits(p: Dict[str, torch.Tensor], emb: torch.Tensor) -> torch.Tensor:
    """map_decoder(image_embeddings) permuted to [B,P,P,2] (model.py:490-491)."""
    x = F.conv_transpose2d(emb, p["map_decoder.0.weight"], p["map_decoder.0.bias"], stride=2)
    x = F.gelu(_ln2d(x, p["map_decoder.1.weight"], p["map_decoder.1.bias"]))
    x = F.gelu(F.conv_transpose2d(x, p["map_decoder.3.weight"], p["map_decoder.3.bias"], stride=2))
    x = F.gelu(F.conv_transpose2d(x, p["map_decoder.5.weight"], p["map_decoder.5.bias"], stride=2))
    x = F.conv_transpose2d(x, p["map_decoder.7.weight"], p["map_decoder.7.bias"], stride=2)
    return x.permute(0, 2, 3, 1)


def mask_loss(logits, kp, road, focal: bool):
    gt = torch.stack([kp, road], dim=3).to(logits.dtype)
    if focal:
        from torchvision.ops import sigmoid_focal_loss
        return sigmoid_focal_loss(logits, gt, alpha=0.25, gamma=2, reduction="mean")
    return F.binary_cross_entropy_with_logits(logits, gt)


def topo_logits(p, emb, points, pairs, valid, P: int, version: str = "normal",
                keep: Optional[Dict[Tuple[int, int], torch.Tensor]] = None, dropout_p: float = 0.1):
    """TopoNet logits [B,Ns,Np] from the sampled embeddings, slow-path semantics."""
    B, Ns, Np, _ = pairs.shape
    pts = points.to(emb.dtype)
    g = (pts / P * 2.0 - 1.0).unsqueeze(2)
    feats = F.grid_sample(emb, g, mode="bilinear", align_corners=False).squeeze(-1).permute(0, 2, 1)
    pf = F.relu(F.linear(feats, p["topo_net.feature_proj.weight"], p["topo_net.feature_proj.bias"]))
    pr = pairs.reshape(B, -1, 2).long()
    bi = torch.arange(B, device=emb.device).view(-1, 1).expand(-1, Ns * Np)
    src, tgt = pf[bi, pr[:, :, 0]], pf[bi, pr[:, :, 1]]
    off = pts[bi, pr[:, :, 1]] - pts[bi, pr[:, :, 0]]
    if version == "no_offset":
        off = torch.zeros_like(off)
    x = F.relu(F.linear(torch.cat([src, tgt, off], 2), p["topo_net.pair_proj.weight"], p["topo_net.pair_proj.bias"]))
    x = x.reshape(B * Ns, Np, 128)
    v = valid.reshape(B * Ns, Np).bool()
    v = v | (v.sum(-1, keepdim=True) == 0)
    scale = torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - dropout_p)

    def drop(t, l, site):
        if keep is None:
            return t
        return t * keep[(l, site)].reshape(t.shape).to(t.dtype) * scale.to(t.device)

    if version != "no_transformer":
        R = B * Ns
        for l in range(3):
            k = f"topo_net.transformer_encoder.layers.{l}."
            qkv = F.linear(x, p[k + "self_attn.in_proj_weight"], p[k + "self_attn.in_proj_bias"])
            q, kk, vv = (t.reshape(R, Np, 4, 32).transpose(1, 2) for t in qkv.split(128, dim=-1))
            s = (q @ kk.transpose(-1, -2)) / (32 ** 0.5)
            s = s.masked_fill(~v[:, None, None, :], float("-inf"))
            a = drop(torch.softmax(s, dim=-1), l, 0)
            o = (a @ vv).transpose(1, 2).reshape(R, Np, 128)
            y = drop(F.linear(o, p[k + "self_attn.out_proj.weight"], p[k + "self_attn.out_proj.bias"]), l, 1)
            x = F.layer_norm(x + y, (128,), p[k + "norm1.weight"], p[k + "norm1.bias"], 1e-5)
            h = drop(F.relu(F.linear(x, p[k + "linear1.weight"], p[k + "linear1.bias"])), l, 2)
            y = drop(F.linear(h, p[k + "linear2.weight"], p[k + "linear2.bias"]), l, 3)
            x = F.layer_norm(x + y, (128,), p[k + "norm2.weight"], p[k + "norm2.bias"], 1e-5)
    out = F.linear(x, p["topo_net.output_proj.weight"], p["topo_net.output_proj.bias"])
    return out.reshape(B, Ns, Np)


def topo_loss(logits, connected, valid):
    m = valid.to(logits.dtype)
    t = F.binary_cross_entropy_with_logits(logits, connected.to(logits.dtype), reduction="none") * m
    return t.sum() / m.sum()


def heads_losses(p, emb, batch, P: int, focal: bool, version: str = "normal", keep=None, dropout_p: float = 0.1):
    """(mask_loss, topo_loss) of reference training_step on precomputed image embeddings."""
    ml = mask_loss(mask_logits(p, emb), batch["keypoint_mask"], batch["road_mask"], focal)
    tl = topo_loss(topo_logits(p, emb, batch["graph_points"], batch["pairs"], batch["valid"], P, version, keep,
                               dropout_p), batch["connected"], batch["valid"])
    return ml, tl
