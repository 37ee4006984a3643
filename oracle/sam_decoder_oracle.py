"""CPU oracle for the USE_SAM_DECODER: True mask head -- TEST INFRASTRUCTURE ONLY (see samroad_oracle.py).

Restates, functionally and driven by the reference state_dict, what sam_road runs when the SAM mask
decoder is enabled (model.py:260-282, 426-443, 471-488): the null-prompt PromptEncoder
(prompt_encoder.py:128-168, dense PE :62-71,171-205), MaskDecoder.predict_masks
(mask_decoder.py:112-149) with the TwoWayTransformer (transformer.py:62-106, 151-182, 185-240), and
the x4 bilinear upsampling of the two low-res masks (model.py:482-487).

Everything runs in the dtype of the inputs and the state_dict (float32 for the model oracle, float64 for
the decoder's stage tests).  `fp16=True` additionally rounds to fp16 exactly where the CUDA path stores
fp16 (csrc/sam_decoder.cu), and nowhere else:
  * the A operands of the image-side projections, fp16(keys + pe) and fp16(keys), and the fp16 weights of
    the token->image k/v projections, the image->token q and out projections and both ConvTranspose layers;
  * the image->token attention output (the A operand of its out_proj);
  * the upscaler activations u1 and u2, which are stored in fp16.
The token side (4 tokens per image) keeps its operands and weights in full precision.  With fp16=False
the functions compute exactly what they computed before the switch existed.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def _half(x: Tensor) -> Tensor:
    """x stored in fp16 (round to nearest even, as __float2half_rn) and read back in x's dtype."""
    return x.to(torch.float16).to(x.dtype)


def _keep(x: Tensor) -> Tensor:
    return x


def dense_pe(sd: Dict[str, Tensor], h: int, w: int, dtype=torch.float32) -> Tensor:
    """PromptEncoder.get_dense_pe (prompt_encoder.py:62-71,185-205) -> [1, 256, h, w] in `dtype`."""
    G = sd["prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"].to(dtype)
    grid = torch.ones((h, w), dtype=dtype, device=G.device)
    y = (grid.cumsum(dim=0) - 0.5) / h
    x = (grid.cumsum(dim=1) - 0.5) / w
    c = 2 * torch.stack([x, y], dim=-1) - 1
    c = 2 * np.pi * (c @ G)
    return torch.cat([torch.sin(c), torch.cos(c)], dim=-1).permute(2, 0, 1).unsqueeze(0)


def _attn(sd, p: str, q: Tensor, k: Tensor, v: Tensor, heads: int = 8, fp16=()) -> Tensor:
    """transformer.py:185-240: projections (possibly down-sampled internal dim), scaled dot-product
    attention with the scale applied after QK^T, out_proj.  Batch dims broadcast (token batch 1 vs B).
    The projections named in `fp16` read their operand and weight rounded to fp16 (out_proj: the
    attention output)."""
    def proj(name, x):
        wt = sd[p + name + ".weight"]
        if name in fp16:
            x, wt = _half(x), _half(wt)
        return F.linear(x, wt, sd[p + name + ".bias"])
    q, k, v = proj("q_proj", q), proj("k_proj", k), proj("v_proj", v)

    def split(x):
        b, n, c = x.shape
        return x.reshape(b, n, heads, c // heads).transpose(1, 2)
    q, k, v = split(q), split(k), split(v)
    att = (q @ k.permute(0, 1, 3, 2)) / math.sqrt(q.shape[-1])
    out = torch.softmax(att, dim=-1) @ v
    b, hds, n, c = out.shape
    out = out.transpose(1, 2).reshape(b, n, hds * c)
    return proj("out_proj", out)


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + "weight"], sd[p + "bias"], 1e-5)


def two_way_transformer(sd, src: Tensor, pos: Tensor, tokens: Tensor, fp16: bool = False):
    """TwoWayTransformer.forward (transformer.py:62-106) with depth 2; layer 0 skips the PE on its
    self-attention and REPLACES the queries (transformer.py:155-161)."""
    t = "mask_decoder.transformer."
    t2i_16 = ("k_proj", "v_proj") if fp16 else ()       # image-side K / V of token->image
    i2t_16 = ("q_proj", "out_proj") if fp16 else ()     # image-side Q and output of image->token
    keys = src.flatten(2).permute(0, 2, 1)
    key_pe = pos.flatten(2).permute(0, 2, 1)
    queries, query_pe = tokens, tokens
    for i in range(2):
        p = f"{t}layers.{i}."
        if i == 0:
            queries = _attn(sd, p + "self_attn.", queries, queries, queries)
        else:
            q = queries + query_pe
            queries = queries + _attn(sd, p + "self_attn.", q, q, queries)
        queries = _ln(queries, sd, p + "norm1.")
        q, k = queries + query_pe, keys + key_pe
        queries = _ln(queries + _attn(sd, p + "cross_attn_token_to_image.", q, k, keys, fp16=t2i_16), sd,
                      p + "norm2.")
        mlp = F.linear(F.relu(F.linear(queries, sd[p + "mlp.lin1.weight"], sd[p + "mlp.lin1.bias"])),
                       sd[p + "mlp.lin2.weight"], sd[p + "mlp.lin2.bias"])
        queries = _ln(queries + mlp, sd, p + "norm3.")
        q, k = queries + query_pe, keys + key_pe
        keys = _ln(keys + _attn(sd, p + "cross_attn_image_to_token.", k, q, queries, fp16=i2t_16), sd,
                   p + "norm4.")
    q, k = queries + query_pe, keys + key_pe
    queries = _ln(queries + _attn(sd, t + "final_attn_token_to_image.", q, k, keys, fp16=t2i_16), sd,
                  t + "norm_final_attn.")
    return queries, keys


def hypernetworks(sd, queries: Tensor) -> Tensor:
    """output_hypernetworks_mlps of the three mask tokens (mask_decoder.py:131-134): queries [B, 4, 256]
    (the transformer's output tokens) -> [B, 3, 32]."""
    hyper = []
    for i in range(3):
        x = queries[:, 1 + i, :]
        m = f"mask_decoder.output_hypernetworks_mlps.{i}.layers."
        x = F.relu(F.linear(x, sd[m + "0.weight"], sd[m + "0.bias"]))
        x = F.relu(F.linear(x, sd[m + "1.weight"], sd[m + "1.bias"]))
        hyper.append(F.linear(x, sd[m + "2.weight"], sd[m + "2.bias"]))
    return torch.stack(hyper, dim=1)


def low_res_masks(sd, keys: Tensor, hyper: Tensor, h: int, w: int, fp16: bool = False) -> Tensor:
    """output_upscaling of the keys [B, h*w, 256] and the masks hyper [B, n, 32] . upscaled
    (mask_decoder.py:129-137) -> [B, n, 4h, 4w]."""
    from .samroad_oracle import layer_norm_2d
    r = _half if fp16 else _keep
    B, C = keys.shape[0], keys.shape[2]
    up = keys.transpose(1, 2).reshape(B, C, h, w)
    u = "mask_decoder.output_upscaling."
    up = F.conv_transpose2d(r(up), r(sd[u + "0.weight"]), sd[u + "0.bias"], stride=2)
    up = r(F.gelu(layer_norm_2d(up, sd[u + "1.weight"], sd[u + "1.bias"])))
    up = r(F.gelu(F.conv_transpose2d(up, r(sd[u + "3.weight"]), sd[u + "3.bias"], stride=2)))
    b, c, hh, ww = up.shape
    return (hyper @ up.view(b, c, hh * ww)).view(b, -1, hh, ww)


def sam_low_res_masks(feat: Tensor, sd, fp16: bool = False, checkpoints: bool = False):
    """MaskDecoder.forward(multimask_output=True) on null prompts -> [B, 2, 4s, 4s]
    (mask_decoder.py:71-149; sparse prompts are empty, dense prompt = no_mask_embed broadcast,
    prompt_encoder.py:164-166).  checkpoints=True returns (queries [B, 4, 256] after norm_final_attn,
    keys [B, T, 256] after the last norm4, hyper [B, 2, 32] of mask tokens 1 and 2, low-res masks)."""
    B, C, h, w = feat.shape
    tokens = torch.cat([sd["mask_decoder.iou_token.weight"], sd["mask_decoder.mask_tokens.weight"]], 0)
    tokens = tokens.unsqueeze(0)                                         # [1, 4, 256]
    src = feat + sd["prompt_encoder.no_mask_embed.weight"].reshape(1, -1, 1, 1)
    hs, keys = two_way_transformer(sd, src, dense_pe(sd, h, w, feat.dtype), tokens, fp16)
    hyper = hypernetworks(sd, hs)                                        # [B, 3, 32]
    masks = low_res_masks(sd, keys, hyper, h, w, fp16)[:, 1:, :, :]     # multimask_output=True
    if checkpoints:
        return hs, keys, hyper[:, 1:], masks
    return masks


def upsample_masks(low: Tensor, patch_size: int) -> Tensor:
    """x4 bilinear, align_corners=False (model.py:482-487): [B, 2, 4s, 4s] -> [B, 2, P, P]."""
    return F.interpolate(low, (patch_size, patch_size), mode="bilinear", align_corners=False)


def sam_mask_logits(feat: Tensor, sd, spec, fp16: bool = False) -> Tensor:
    """mask logits [B, 2, P, P]: low-res masks upsampled x4, bilinear, align_corners=False
    (model.py:482-487)."""
    return upsample_masks(sam_low_res_masks(feat, sd, fp16), spec.patch_size)
