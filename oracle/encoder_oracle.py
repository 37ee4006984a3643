"""Staged reference of the image encoder and the naive map decoder -- TEST INFRASTRUCTURE ONLY (see
samroad_oracle.py).

The same algorithm as samroad_oracle.image_encoder / map_decoder (SAMRoad.infer_masks_and_img_features,
model.py:459-495; ImageEncoderViT.forward, image_encoder.py:106-116; map_decoder, model.py:286-295), cut
into the stages samroad_encode_masks runs as separate launches, so that a test can feed each stage the
device's own copy of the previous one (samroad_op_encoder_taps) and judge one kernel at a time.  Token
tensors are NHWC grids [B, s, s, C]; the decoder works on NCHW images as the reference does.

`EncoderRef(sd, spec, fp16=False)` computes in the given dtype (float64 for the stage tests).  With
fp16=True it also rounds to fp16 exactly where the CUDA path stores or consumes fp16 (csrc/model.cu,
kernels.cu, attention_mma.cuh, gemm_tc.cuh), and nowhere else:
  * the normalised pixels, computed as the kernel does in float32, (x - mean) * (1/std) (the A operand of
    the patch embed);
  * the packed GEMM weights: patch embed, qkv (LoRA merged first, in float32 and in the order of
    samroad_finalize_weights), proj, lin1, lin2, neck.0, neck.2 and map_decoder.0/.3/.5.  map_decoder.7,
    every bias, LayerNorm parameter, pos_embed and the rel-pos tables stay as given;
  * ln1, ln2, qkv, the attention output and GELU(lin1);
  * the window padding tokens, whose q = k = v = fp16(qkv bias);
  * the probabilities P fed to the P V product, with the softmax denominator summing the rounded P.  With
    `p_block(s, win, hd)` given, P is taken against the running maximum over key blocks of that many slots,
    as the kernel that runs the block does (attention_oracle.softmax_pv; None: P unrounded, the SIMT
    kernel); without it, against the row's global maximum;
  * fp16(X) into the neck, its two outputs n1 and feat16, and the decoder activations d1 and d2.
The image embeddings (neck output before rounding), the residual stream X, dec3 + GELU + map_decoder.7
and the logits stay in full precision.  With fp16=False the stages chained end to end are the algorithm of
samroad_oracle (tests/test_encoder_oracle_host.py).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

from . import attention_oracle as A
from .samroad_oracle import PIXEL_MEAN, PIXEL_STD, ModelSpec, layer_norm_2d, rel_pos_gather

Tensor = torch.Tensor

# score elements (windows x heads x queries x keys) of one attention chunk: bounds the float64 working set
_ATT_CHUNK = 1 << 27


def _half(x: Tensor) -> Tensor:
    """x stored in fp16 (round to nearest even, as __float2half_rn) and read back in x's dtype."""
    return x.to(torch.float16).to(x.dtype)


def _keep(x: Tensor) -> Tensor:
    return x


def quad_rows(x: Tensor, levels: int) -> Tensor:
    """NCHW image [B, C, s * 2^L, s * 2^L] -> rows [B * s * s * 4^L, C] in the order of the decoder GEMMs:
    row = ((m * 4 + d_1) * 4 + d_2) ..., m = token of the s x s grid, d_l = di_l * 2 + dj_l the sub-pixel
    of ConvTranspose level l (csrc/gemm_tc.cuh EpiDecFinal)."""
    B, C = x.shape[:2]
    s = x.shape[2] >> levels
    v = x.reshape(B, C, s, *([2] * levels), s, *([2] * levels))
    order = [0, 2, 3 + levels]
    for l in range(levels):
        order += [3 + l, 4 + levels + l]
    return v.permute(*order, 1).reshape(-1, C)


def from_quad_rows(rows: Tensor, B: int, s: int, levels: int) -> Tensor:
    """Inverse of quad_rows: rows [B * s * s * 4^L, C] -> NCHW [B, C, s * 2^L, s * 2^L]."""
    C = rows.shape[-1]
    v = rows.reshape(B, s, s, *([2, 2] * levels), C)
    # axes: 0 b, 1 i, 2 j, then (di_l, dj_l) pairs at 3 + 2l, 4 + 2l, channel last
    n = 3 + 2 * levels
    order = [0, n, 1] + [3 + 2 * l for l in range(levels)] + [2] + [4 + 2 * l for l in range(levels)]
    return v.permute(*order).reshape(B, C, s << levels, s << levels)


class EncoderRef:
    """Weights of one model prepared for the stages (rounded to fp16 where the device packs fp16)."""

    def __init__(self, sd: Dict[str, Tensor], spec: ModelSpec, fp16: bool = False, dtype=torch.float64,
                 device=None, p_block: Optional[Callable[[int, int, int], Optional[int]]] = None):
        self.spec, self.fp16, self.dtype, self.p_block = spec, fp16, dtype, p_block
        self.r = _half if fp16 else _keep
        dev = device if device is not None else next(iter(sd.values())).device
        self.device = torch.device(dev)
        t = lambda k: sd[k].to(self.device, dtype)           # noqa: E731
        w16 = lambda k: self.r(t(k))                         # noqa: E731
        W = {"pe_w": w16("image_encoder.patch_embed.proj.weight"),
             "pe_b": t("image_encoder.patch_embed.proj.bias"),
             "pos": t("image_encoder.pos_embed")}
        for i in range(spec.depth):
            p = f"image_encoder.blocks.{i}."
            W[p + "qkv_w"] = self.r(self._merged_qkv(sd, p, dtype))
            for k in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.bias",
                      "attn.proj.bias", "attn.rel_pos_h", "attn.rel_pos_w", "mlp.lin1.bias", "mlp.lin2.bias"):
                W[p + k] = t(p + k)
            for k in ("attn.proj.weight", "mlp.lin1.weight", "mlp.lin2.weight"):
                W[p + k] = w16(p + k)
        W["neck0"] = w16("image_encoder.neck.0.weight").flatten(1)
        W["neck2"] = w16("image_encoder.neck.2.weight")
        for k in ("image_encoder.neck.1.weight", "image_encoder.neck.1.bias", "image_encoder.neck.3.weight",
                  "image_encoder.neck.3.bias"):
            W[k] = t(k)
        if not spec.use_sam_decoder:
            for k in ("map_decoder.0.weight", "map_decoder.3.weight", "map_decoder.5.weight"):
                W[k] = w16(k)
            for k in ("map_decoder.0.bias", "map_decoder.1.weight", "map_decoder.1.bias", "map_decoder.3.bias",
                      "map_decoder.5.bias", "map_decoder.7.weight", "map_decoder.7.bias"):
                W[k] = t(k)
        self.W = W

    def _merged_qkv(self, sd, p: str, dtype) -> Tensor:
        """qkv weight with the LoRA updates merged (_LoRA_qkv, model.py:179-186): q rows += B_q A_q, v rows
        += B_v A_v.  Under fp16 in float32, one rank at a time, as samroad_finalize_weights packs it."""
        w = sd[p + "attn.qkv.weight"].to(self.device)
        if p + "attn.qkv.linear_a_q.weight" not in sd:
            return w.to(dtype)
        g = lambda k: sd[p + "attn.qkv." + k + ".weight"].to(self.device)   # noqa: E731
        aq, bq, av, bv = g("linear_a_q"), g("linear_b_q"), g("linear_a_v"), g("linear_b_v")
        D = w.shape[1]
        if not self.fp16:
            w = w.to(dtype).clone()
            w[:D] += bq.to(dtype) @ aq.to(dtype)
            w[2 * D:] += bv.to(dtype) @ av.to(dtype)
            return w
        w = w.float().clone()
        for j in range(aq.shape[0]):
            w[:D] += bq[:, j:j + 1].float() * aq[j:j + 1].float()
            w[2 * D:] += bv[:, j:j + 1].float() * av[j:j + 1].float()
        return w.to(dtype)

    # ---- encoder stages ---------------------------------------------------------------------------
    def patch_embed(self, rgb: Tensor) -> Tensor:
        """[B, P, P, 3] pixels 0..255 -> X [B, s, s, D]: normalisation (model.py:465-467), the 16 x 16 /
        stride 16 conv (image_encoder.py:387-395) and + pos_embed (:108-109)."""
        if self.fp16:      # the im2col kernel: float32 (x - mean) * (1 / std), stored as fp16
            mean = torch.tensor(PIXEL_MEAN, dtype=torch.float32, device=self.device)
            inv = 1.0 / torch.tensor(PIXEL_STD, dtype=torch.float32, device=self.device)
            x = _half((rgb.to(self.device, torch.float32) - mean) * inv).to(self.dtype)
        else:
            mean = torch.tensor(PIXEL_MEAN, dtype=self.dtype, device=self.device)
            std = torch.tensor(PIXEL_STD, dtype=self.dtype, device=self.device)
            x = (rgb.to(self.device, self.dtype) - mean) / std
        y = F.conv2d(x.permute(0, 3, 1, 2), self.W["pe_w"], self.W["pe_b"], stride=16)
        return y.permute(0, 2, 3, 1) + self.W["pos"]

    def ln(self, x: Tensor, i: int, which: int) -> Tensor:
        """norm1 / norm2 of block i, eps 1e-6 (image_encoder.py:168,180; model.py:250)."""
        p = f"image_encoder.blocks.{i}.norm{which}."
        return self.r(F.layer_norm(x, (x.shape[-1],), self.W[p + "weight"], self.W[p + "bias"], 1e-6))

    def qkv(self, xn: Tensor, i: int) -> Tensor:
        """the qkv linear with LoRA (image_encoder.py:227; model.py:179-186) -> [B, s, s, 3D]"""
        p = f"image_encoder.blocks.{i}."
        return self.r(F.linear(xn, self.W[p + "qkv_w"], self.W[p + "attn.qkv.bias"]))

    def attention(self, qkv: Tensor, i: int) -> Tensor:
        """softmax((q * scale) k^T + decomposed rel-pos) v of block i, windowed (zero-padded LN output, so the
        padding tokens carry the qkv bias) or global (image_encoder.py:166-176, 224-240, 243-289, 325-361)."""
        p = f"image_encoder.blocks.{i}."
        B, H, Wd, D3 = qkv.shape
        glob = i in self.spec.global_attn_indexes
        win = H if glob else self.spec.window_size
        ph, pw = (win - H % win) % win, (win - Wd % win) % win
        x = qkv
        if ph or pw:
            x = self.r(self.W[p + "attn.qkv.bias"]).expand(B, H + ph, Wd + pw, D3).clone()
            x[:, :H, :Wd] = qkv
        Hp, Wp = H + ph, Wd + pw
        wins = x.reshape(B, Hp // win, win, Wp // win, win, D3).permute(0, 1, 3, 2, 4, 5).reshape(-1, win, win, D3)
        heads = self.spec.num_heads
        per = max(1, _ATT_CHUNK // (heads * win ** 4))
        out = torch.cat([self._attention_core(wins[c:c + per], self.W[p + "attn.rel_pos_h"],
                                              self.W[p + "attn.rel_pos_w"]) for c in range(0, wins.shape[0], per)])
        out = out.view(B, Hp // win, Wp // win, win, win, -1).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, -1)
        return out[:, :H, :Wd].contiguous()

    def _attention_core(self, wins: Tensor, rel_h: Tensor, rel_w: Tensor) -> Tensor:
        n, win, _, D3 = wins.shape
        heads, D, L = self.spec.num_heads, D3 // 3, win * win
        hd = D // heads
        q, k, v = wins.reshape(n, L, 3, heads, hd).permute(2, 0, 3, 1, 4).unbind(0)   # [n, heads, L, hd]
        scores = (q * hd ** -0.5) @ k.transpose(-2, -1)                                # :231
        qg = q.reshape(n, heads, win, win, hd)                                         # UNscaled q (:354-355)
        rh = torch.einsum("nahwc,hkc->nahwk", qg, rel_pos_gather(win, win, rel_h))
        rw = torch.einsum("nahwc,wkc->nahwk", qg, rel_pos_gather(win, win, rel_w))
        scores = (scores.view(n, heads, win, win, win, win) + rh[..., :, None] + rw[..., None, :]).view(n, heads, L, L)
        if self.fp16:
            block = self.p_block(self.spec.grid, win, hd) if self.p_block else win * A.win_pitch(win)
            o = A.softmax_pv(scores, v, A.key_blocks(win, block, scores.device))
        else:
            o = scores.softmax(-1) @ v
        return self.r(o.permute(0, 2, 1, 3).reshape(n, win, win, D))

    def proj(self, att: Tensor, x: Tensor, i: int) -> Tensor:
        """X + proj(att) (image_encoder.py:176,239)"""
        p = f"image_encoder.blocks.{i}."
        return x + F.linear(att, self.W[p + "attn.proj.weight"], self.W[p + "attn.proj.bias"])

    def lin1(self, xn: Tensor, i: int) -> Tensor:
        """GELU(lin1(norm2 output)), exact erf GELU (common.py:13-18)"""
        p = f"image_encoder.blocks.{i}."
        return self.r(F.gelu(F.linear(xn, self.W[p + "mlp.lin1.weight"], self.W[p + "mlp.lin1.bias"])))

    def lin2(self, h: Tensor, x: Tensor, i: int) -> Tensor:
        """X + lin2(h) (image_encoder.py:180)"""
        p = f"image_encoder.blocks.{i}."
        return x + F.linear(h, self.W[p + "mlp.lin2.weight"], self.W[p + "mlp.lin2.bias"])

    def block(self, x: Tensor, i: int, taps: Optional[dict] = None) -> Tensor:
        """Block i from its input X (image_encoder.py:166-182); `taps` receives every operand."""
        t = {"ln1": self.ln(x, i, 1)}
        t["qkv"] = self.qkv(t["ln1"], i)
        t["att"] = self.attention(t["qkv"], i)
        t["x_attn"] = self.proj(t["att"], x, i)
        t["ln2"] = self.ln(t["x_attn"], i, 2)
        t["h"] = self.lin1(t["ln2"], i)
        t["x"] = self.lin2(t["h"], t["x_attn"], i)
        if taps is not None:
            taps.update(t)
        return t["x"]

    def neck1(self, x: Tensor) -> Tensor:
        """1 x 1 conv (no bias) + LayerNorm2d on fp16(X) (image_encoder.py:88-95) -> n1 [B, s, s, 256]"""
        y = F.linear(self.r(x), self.W["neck0"])
        return self.r(F.layer_norm(y, (256,), self.W["image_encoder.neck.1.weight"],
                                   self.W["image_encoder.neck.1.bias"], 1e-6))

    def neck2(self, n1: Tensor):
        """3 x 3 conv (pad 1, no bias) + LayerNorm2d (image_encoder.py:96-103) -> (image embeddings NCHW
        [B, 256, s, s], feat16 NHWC [B, s, s, 256] = what the map decoder reads)"""
        y = F.conv2d(n1.permute(0, 3, 1, 2), self.W["neck2"], padding=1)
        emb = layer_norm_2d(y, self.W["image_encoder.neck.3.weight"], self.W["image_encoder.neck.3.bias"])
        return emb, self.r(emb).permute(0, 2, 3, 1)

    # ---- naive map decoder (model.py:286-295) -------------------------------------------------------
    def dec1(self, feat: Tensor) -> Tensor:
        """ConvT(256->128, k2 s2) + LayerNorm2d + GELU on NCHW [B, 256, s, s] -> d1 [B, 128, 2s, 2s]"""
        y = F.conv_transpose2d(feat, self.W["map_decoder.0.weight"], self.W["map_decoder.0.bias"], stride=2)
        return self.r(F.gelu(layer_norm_2d(y, self.W["map_decoder.1.weight"], self.W["map_decoder.1.bias"])))

    def dec2(self, d1: Tensor) -> Tensor:
        """ConvT(128->64) + GELU -> d2 [B, 64, 4s, 4s]"""
        return self.r(F.gelu(F.conv_transpose2d(d1, self.W["map_decoder.3.weight"], self.W["map_decoder.3.bias"],
                                                stride=2)))

    def dec3(self, d2: Tensor) -> Tensor:
        """ConvT(64->32) + GELU, ConvT(32->2) -> mask logits NCHW [B, 2, P, P]"""
        h = F.gelu(F.conv_transpose2d(d2, self.W["map_decoder.5.weight"], self.W["map_decoder.5.bias"], stride=2))
        return F.conv_transpose2d(h, self.W["map_decoder.7.weight"], self.W["map_decoder.7.bias"], stride=2)

    # ---- the stages chained ---------------------------------------------------------------------------
    def encoder(self, rgb: Tensor, taps: Optional[dict] = None):
        """-> (image embeddings NCHW, feat16 NHWC); `taps` receives tokens0, block{i}, n1."""
        x = self.patch_embed(rgb)
        if taps is not None:
            taps["tokens0"] = x
        for i in range(self.spec.depth):
            x = self.block(x, i)
            if taps is not None:
                taps[f"block{i}"] = x
        n1 = self.neck1(x)
        if taps is not None:
            taps["n1"] = n1
        return self.neck2(n1)

    def map_decoder(self, feat16: Tensor) -> Tensor:
        """feat16 NHWC -> mask logits NCHW [B, 2, P, P]"""
        return self.dec3(self.dec2(self.dec1(feat16.permute(0, 3, 1, 2))))
