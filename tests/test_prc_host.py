"""CPU: the precision-recall oracle (oracle/prc_oracle.py) against sklearn and a brute-force threshold
sweep, its argmax rule in the NaN and no-positive cases, the test_step label mapping, and the C ABI of
the accumulator."""
import os
import re

import numpy as np
import pytest
import torch
from sklearn.metrics import precision_recall_curve

from oracle import prc_oracle as PO
from sam_road_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tied_scores(rng, n):
    """uint8-quantised scores (k/255) with exact 0.0 and 1.0 over-represented: heavy ties."""
    k = rng.integers(0, 256, n)
    k[rng.random(n) < 0.1] = 0
    k[rng.random(n) < 0.1] = 255
    return (k.astype(np.float32) / np.float32(255)).astype(np.float32)


def _brute_force(preds, target):
    thr = np.unique(preds)
    tps = np.array([int(((preds >= t) & (target == 1)).sum()) for t in thr], np.int64)
    fps = np.array([int(((preds >= t) & (target == 0)).sum()) for t in thr], np.int64)
    return thr, tps, fps


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_brute_force_sweep(seed):
    rng = np.random.default_rng(seed)
    n = 3000
    preds = _tied_scores(rng, n)
    target = (rng.random(n) < 0.3).astype(np.int64)
    target[rng.random(n) < 0.2] = -1
    keep = target != -1
    prec, rec, thr, tps, fps = PO.binary_pr_curve(preds, target, return_counts=True)
    bthr, btps, bfps = _brute_force(preds[keep], target[keep])
    np.testing.assert_array_equal(thr, bthr)
    np.testing.assert_array_equal(tps, btps)
    np.testing.assert_array_equal(fps, bfps)
    tf, ff = btps.astype(np.float32), bfps.astype(np.float32)
    np.testing.assert_array_equal(prec[:-1].view(np.uint32), (tf / (tf + ff)).view(np.uint32))
    np.testing.assert_array_equal(rec[:-1].view(np.uint32), (tf / np.float32(btps[0])).view(np.uint32))
    assert prec[-1] == 1 and rec[-1] == 0 and prec.dtype == rec.dtype == np.float32


@pytest.mark.parametrize("seed", [3, 4])
def test_oracle_matches_sklearn(seed):
    rng = np.random.default_rng(seed)
    n = 5000
    preds = np.concatenate([_tied_scores(rng, n // 2), rng.random(n // 2).astype(np.float32)])
    target = (rng.random(n) < preds * 0.8).astype(np.int64)
    prec, rec, thr = PO.binary_pr_curve(preds, target)
    sp, sr, st = precision_recall_curve(target, preds.astype(np.float64))
    # sklearn keeps every threshold up to full recall; compare on its points (all of them here)
    idx = np.searchsorted(thr, st.astype(np.float32))
    np.testing.assert_array_equal(thr[idx], st.astype(np.float32))
    np.testing.assert_allclose(prec[idx], sp[:-1], rtol=1e-6)
    np.testing.assert_allclose(rec[idx], sr[:-1], rtol=1e-6)
    assert len(st) <= len(thr)


def test_best_point_nan_rule_top_scores_negative():
    # the highest scores are negatives: P = R = 0 there, F1 = NaN, and torch.argmax picks the first NaN
    preds = np.array([0.1, 0.2, 0.3, 0.8, 0.9], np.float32)
    target = np.array([1, 0, 1, 0, 0])
    prec, rec, thr = PO.binary_pr_curve(preds, target)
    i, t, p, r, f1 = PO.find_best_threshold(prec, rec, thr)
    assert np.isnan(f1) and i == 3 and t == np.float32(0.8) and p == 0 and r == 0
    # torch.argmax agrees on the same float32 F1 array
    f1t = 2 * (torch.from_numpy(prec) * torch.from_numpy(rec)) / (torch.from_numpy(prec) + torch.from_numpy(rec))
    assert int(torch.argmax(f1t)) == i


def test_best_point_without_positives():
    preds = np.array([0.5, 0.25, 0.75], np.float32)
    prec, rec, thr = PO.binary_pr_curve(preds, np.zeros(3, np.int64))
    assert np.isnan(rec[:-1]).all()
    i, t, p, r, f1 = PO.find_best_threshold(prec, rec, thr)
    assert i == 0 and t == np.float32(0.25) and np.isnan(f1)


def test_best_point_first_maximum():
    preds = np.array([0.2, 0.4, 0.6, 0.8], np.float32)
    target = np.array([0, 1, 0, 1])
    prec, rec, thr = PO.binary_pr_curve(preds, target)
    i, t, p, r, f1 = PO.find_best_threshold(prec, rec, thr)
    f1s = np.float32(2) * (prec * rec) / (prec + rec)
    assert f1 == f1s.max() and i == int(np.flatnonzero(f1s == f1s.max())[0])


def test_oracle_refuses_what_torchmetrics_would_not_count():
    with pytest.raises(ValueError, match="prediction"):
        PO.binary_pr_curve(np.array([0.5, 1.5], np.float32), np.array([0, 1]))
    with pytest.raises(ValueError, match="prediction"):
        PO.binary_pr_curve(np.array([0.5, np.nan], np.float32), np.array([0, 1]))
    with pytest.raises(ValueError, match="target"):
        PO.binary_pr_curve(np.array([0.5, 0.5], np.float32), np.array([0, 2]))
    # an ignored entry is neither counted nor checked
    prec, rec, thr = PO.binary_pr_curve(np.array([0.5, 0.25], np.float32), np.array([1, -1]))
    assert thr.tolist() == [0.5]


def test_test_step_targets_mapping():
    k = torch.arange(256, dtype=torch.float32).view(1, 16, 16) / 255.0
    valid = torch.tensor([[[True, False, True]]])
    connected = torch.tensor([[[True, True, False]]])
    kp, road, topo = PO.test_step_targets(dict(keypoint_mask=k, road_mask=k, valid=valid, connected=connected))
    assert kp.dtype == torch.int32 and int(kp.sum()) == 1 and int(kp.view(-1)[255]) == 1   # only 255/255
    assert topo.view(-1).tolist() == [1, -1, 0]


def test_prc_abi_version_and_symbols():
    src = open(os.path.join(ROOT, "include", "samroad_b200.h")).read()
    assert int(re.search(r"#define SAMROAD_ABI_VERSION (\d+)", src).group(1)) == _lib.ABI_VERSION == 5
    lib = _lib.load()
    assert lib.samroad_abi_version() == 5
    for name in ("create", "destroy", "reset", "update", "compute", "read_curve"):
        assert f"samroad_prc_{name}" in _lib.SIGNATURES


def test_prc_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    # argument checks come before any CUDA call
    assert lib.samroad_prc_update(None, None, 1, None, 0, None, 4, None) != 0
    assert lib.samroad_prc_read_curve(None, None, None, None, None, None, None) != 0
    assert lib.samroad_prc_compute(None, None, None, None) != 0
    assert lib.samroad_prc_destroy(None) == 0
