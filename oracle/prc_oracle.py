"""CPU oracle of the threshold search in test.py -- TEST INFRASTRUCTURE ONLY.

A NumPy restatement of what SAMRoad.test_step / on_test_end compute (reference model.py:361-363,
602-634) through torchmetrics' BinaryPrecisionRecallCurve(thresholds=None, ignore_index=-1), with the
counting made exact:
  - entries whose label is ignore_index are dropped; labels must then be 0 or 1 and scores in [0, 1]
    (torchmetrics raises on other labels and would sigmoid the batch on out-of-range scores; both are
    refused here as in sam_road_b200.metrics);
  - one threshold per distinct score, ascending; tps / fps count the positives / negatives with
    score >= threshold as int64 (a scan from the highest score down);
  - precision = tps / (tps + fps), recall = tps / tps_total in float32 with tps, fps rounded to float32
    first, then the final point (1, 0) -- torchmetrics' layout, without its optional truncation after
    full recall;
  - find_best_threshold: F1 = 2 * (P * R) / (P + R) in float32 and torch.argmax's choice (first maximum,
    NaN above every number).
torchmetrics is not installed where these tests run; tests/test_prc_host.py pins this file against
sklearn.metrics.precision_recall_curve and a brute-force threshold sweep instead.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch


def test_step_targets(batch) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Label tensors test_step hands to the three curves (model.py:609-617): int32(keypoint_mask),
    int32(road_mask), and connected with -1 where valid is False."""
    valid = batch["valid"].to(torch.int32)
    topo_gt = batch["connected"].to(torch.int32)
    topo_gt = (1 - valid) * -1 + valid * topo_gt
    return (batch["keypoint_mask"].to(torch.int32), batch["road_mask"].to(torch.int32),
            topo_gt.unsqueeze(-1).to(torch.int32))


def binary_pr_curve(preds, target, ignore_index: int = -1, return_counts: bool = False):
    """(precision [T+1], recall [T+1], thresholds [T]) float32, thresholds ascending; with return_counts
    the int64 tps and fps [T] follow."""
    preds = np.asarray(preds, dtype=np.float32).ravel()
    target = np.asarray(target).ravel().astype(np.int64)
    if preds.shape != target.shape:
        raise ValueError(f"preds and target differ in size: {preds.shape} vs {target.shape}")
    keep = target != ignore_index
    preds, target = preds[keep], target[keep]
    if preds.size == 0:
        raise ValueError("no entries")
    if not np.all((preds >= 0) & (preds <= 1)):
        raise ValueError("a prediction is NaN or outside [0, 1]")
    if not np.all((target == 0) | (target == 1)):
        raise ValueError("a target is not 0 or 1")
    preds = np.where(preds == 0, np.float32(0), preds)         # -0.0 and 0.0 are one threshold
    thresholds, inverse = np.unique(preds, return_inverse=True)
    T = thresholds.size
    count = np.bincount(inverse, minlength=T).astype(np.int64)
    pos = np.bincount(inverse, weights=target, minlength=T).astype(np.int64)
    tps = np.cumsum(pos[::-1])[::-1]
    fps = np.cumsum(count[::-1])[::-1] - tps
    tf, ff = tps.astype(np.float32), fps.astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        precision = tf / (tf + ff)
        recall = tf / np.float32(tps[0])
    precision = np.concatenate([precision, np.ones(1, np.float32)])
    recall = np.concatenate([recall, np.zeros(1, np.float32)])
    if return_counts:
        return precision, recall, thresholds, tps, fps
    return precision, recall, thresholds


def find_best_threshold(precision, recall, thresholds):
    """on_test_end's pick (model.py:621-629): (index, threshold, P, R, F1) at torch.argmax(F1)."""
    p = np.asarray(precision, np.float32)
    r = np.asarray(recall, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        f1 = np.float32(2) * (p * r) / (p + r)
    nan = np.isnan(f1)
    i = int(np.argmax(nan)) if nan.any() else int(np.argmax(f1))
    return i, thresholds[i], p[i], r[i], f1[i]
