"""CPU oracle of the validation loop -- TEST INFRASTRUCTURE ONLY.

A NumPy restatement of what SAMRoad.validation_step / on_validation_epoch_end compute (reference
model.py:349-359, 547-600) with the sums made exact:
  - per-element loss terms in float32, one rounding per torch op: BCEWithLogits
    (1 - y) * x - log_sigmoid(x) with log_sigmoid(x) = min(0, x) - log1p(exp(-|x|)), and torchvision's
    sigmoid_focal_loss(alpha=0.25, gamma=2) built on it.  exp and log1p are float64 rounded once to
    float32.  Libms differ from one another by an ulp or two there, and the expressions cancel (BCE
    where y = 0 and x < 0, focal's 1 - p_t where p_t is near 1), which magnifies that in the term; the
    one-op functions can be swapped for another library's to compare the expressions alone;
  - a mean is the exact sum (math.fsum) over the count, rounded to float32 once; the topology mean runs over
    the valid slots only and is NaN without one;
  - confusion counts as Python ints, a prediction positive when score > 0.5;
  - IoU = tp / ((fp + fn) + tp) and F1 = 2 tp / ((2 tp + fn) + fp) in float32 from float32 counts, 0 when
    the denominator is 0 (torchmetrics' _jaccard_index_reduce / _fbeta_reduce with _safe_divide);
  - the epoch mean of a logged step value is f32(sum(f64(value) * B) / sum(B)).
torchmetrics is not installed where these tests run; tests/test_val_host.py pins this file against
torch.nn.functional, torchvision.ops.sigmoid_focal_loss and sklearn.metrics instead.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import numpy as np
import torch

F32 = np.float32


def _exp(x):
    """float32 exp, correctly rounded in practice (float64 exp rounded once; overflows to inf)."""
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(x, F32).astype(np.float64)).astype(F32)


def _log1p(x):
    return np.log1p(np.asarray(x, F32).astype(np.float64)).astype(F32)


def log_sigmoid(x):
    """torch's float32 form: min(0, x) - log1p(exp(-|x|))."""
    x = np.asarray(x, F32)
    return (np.minimum(F32(0), x) - _log1p(_exp(-np.abs(x)))).astype(F32)


def sigmoid(x):
    """torch's float32 form: 1 / (1 + exp(-x)) (0 where exp(-x) overflows)."""
    x = np.asarray(x, F32)
    return (F32(1) / (F32(1) + _exp(-x))).astype(F32)


def bce_terms(x, y, log_sigmoid=log_sigmoid):
    """F.binary_cross_entropy_with_logits(x, y, reduction='none') in float32.  `log_sigmoid` may be
    replaced by another implementation of that one op (e.g. torch's, to compare the expression alone)."""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    return ((F32(1) - y) * x - np.asarray(log_sigmoid(x), F32)).astype(F32)


def focal_terms(x, y, alpha: float = 0.25, sigmoid=sigmoid, log_sigmoid=log_sigmoid):
    """torchvision.ops.sigmoid_focal_loss(x, y, alpha, gamma=2, reduction='none') in float32."""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    p = np.asarray(sigmoid(x), F32)
    ce = bce_terms(x, y, log_sigmoid)
    p_t = p * y + (F32(1) - p) * (F32(1) - y)
    m = F32(1) - p_t
    loss = ce * (m * m)
    alpha_t = F32(alpha) * y + F32(1 - alpha) * (F32(1) - y)
    return (alpha_t * loss).astype(F32)


def exact_mean(terms) -> np.float32:
    """f32(fsum(terms) / n); NaN when there are no terms."""
    t = np.asarray(terms, np.float64).ravel()
    if t.size == 0:
        return F32(np.nan)
    return F32(math.fsum(t) / t.size)


def counts(scores, labels, keep=None):
    """(tp, fp, fn, tn) as ints: prediction positive when score > 0.5, label 1 positive."""
    s = np.asarray(scores, F32).ravel()
    y = np.asarray(labels).ravel().astype(bool)
    if keep is not None:
        k = np.asarray(keep).ravel().astype(bool)
        s, y = s[k], y[k]
    pred = s > F32(0.5)
    return (int((pred & y).sum()), int((pred & ~y).sum()), int((~pred & y).sum()), int((~pred & ~y).sum()))


def _safe_divide(num, den):
    with np.errstate(divide="ignore", invalid="ignore"):
        return F32(num / den) if den != 0 else F32(0)


def iou(tp: int, fp: int, fn: int) -> np.float32:
    return _safe_divide(F32(tp), (F32(fp) + F32(fn)) + F32(tp))


def f1(tp: int, fp: int, fn: int) -> np.float32:
    num = F32(2) * F32(tp)
    return _safe_divide(num, (num + F32(fn)) + F32(fp))


def validation_step_targets(batch):
    """The reference's targets (model.py:555-588): the float masks for the mask loss and the IoUs,
    connected as float for the topology BCE, and the F1 label connected / -1 where valid is False."""
    valid = batch["valid"].to(torch.int32)
    topo_gt = batch["connected"].to(torch.int32)
    f1_gt = (1 - valid) * -1 + valid * topo_gt
    return (batch["keypoint_mask"].to(torch.float32), batch["road_mask"].to(torch.float32),
            topo_gt.to(torch.float32), valid.to(torch.bool), f1_gt)


def step_values(mask_logits, kp_mask, road_mask, topo_logits, connected, valid, focal: bool = False):
    """(mask_loss, topo_loss, loss) float32 of one step; mask_logits [B,P,P,2]."""
    ml = np.asarray(mask_logits, F32)
    y = np.stack([np.asarray(kp_mask, F32), np.asarray(road_mask, F32)], -1)
    terms = (focal_terms if focal else bce_terms)(ml, y)
    v = np.asarray(valid).ravel().astype(bool)
    tt = bce_terms(np.asarray(topo_logits, F32).ravel()[v], np.asarray(connected, F32).ravel()[v])
    m, t = exact_mean(terms), exact_mean(tt)
    return m, t, F32(m + t)


def step_counts(mask_scores, kp_mask, road_mask, topo_scores, connected, valid) -> Dict[str, int]:
    ms = np.asarray(mask_scores, F32)
    out = {}
    for name, c, m in (("keypoint", 0, kp_mask), ("road", 1, road_mask)):
        tp, fp, fn, tn = counts(ms[..., c], m)
        out.update({f"{name}_tp": tp, f"{name}_fp": fp, f"{name}_fn": fn, f"{name}_tn": tn})
    tp, fp, fn, _ = counts(topo_scores, connected, valid)
    out.update(topo_tp=tp, topo_fp=fp, topo_fn=fn)
    return out


def epoch_mean(values: Sequence[float], batch_sizes: Sequence[int]) -> np.float32:
    """Lightning's on_epoch mean weighted by batch size, exact: f32(sum(f64(v) * B) / sum(B))."""
    num = math.fsum(float(F32(v)) * int(b) for v, b in zip(values, batch_sizes))
    return F32(num / sum(int(b) for b in batch_sizes))


def epoch_metrics(c: Dict[str, int]) -> Dict[str, np.float32]:
    return {"keypoint_iou": iou(c["keypoint_tp"], c["keypoint_fp"], c["keypoint_fn"]),
            "road_iou": iou(c["road_tp"], c["road_fp"], c["road_fn"]),
            "topo_f1": f1(c["topo_tp"], c["topo_fp"], c["topo_fn"])}
