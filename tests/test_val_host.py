"""CPU: the validation oracle (oracle/val_oracle.py) against torch.nn.functional, torchvision's
sigmoid_focal_loss and sklearn's jaccard / F1 scores, its exact means, the validation_step label mapping,
and the argument checks of the samroad_val_* calls."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from sklearn.metrics import f1_score, jaccard_score

from oracle import val_oracle as VO
from sam_road_b200 import _lib
from sam_road_b200.metrics import f1_from_counts, iou_from_counts


def _logits(seed, n=20000):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) * 6).astype(np.float32)
    x[:12] = [0.0, -0.0, 20.0, -20.0, 90.0, -90.0, 1e-8, -1e-8, 17.5, -17.5, 0.5, -0.5]
    y = (rng.random(n) < 0.4).astype(np.float32)
    return x, y


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def _torch_op(fn):
    return lambda x: fn(torch.from_numpy(np.asarray(x, np.float32))).numpy()


@pytest.mark.parametrize("seed", [0, 1])
def test_bce_terms_match_torch(seed):
    x, y = _logits(seed)
    ref = F.binary_cross_entropy_with_logits(torch.from_numpy(x), torch.from_numpy(y), reduction="none").numpy()
    # the expression, with torch's log_sigmoid
    assert _ulps(VO.bce_terms(x, y, _torch_op(F.logsigmoid)), ref).max() <= 1
    # the decomposition the kernels use is torch's, bit for bit on the CPU
    dec = ((1 - torch.from_numpy(y)) * torch.from_numpy(x) - F.logsigmoid(torch.from_numpy(x))).numpy()
    np.testing.assert_array_equal(ref.view(np.uint32), dec.view(np.uint32))
    # the oracle's own log_sigmoid is within 2 ulps of torch's CPU one; in the term that error is bounded
    # at the scale of the operands (the expression cancels for y = 0, x < 0)
    ls = VO.log_sigmoid(x)
    assert _ulps(ls, F.logsigmoid(torch.from_numpy(x)).numpy()).max() <= 2
    scale = np.maximum(np.abs((1 - y) * x), np.abs(ls))
    assert (np.abs(VO.bce_terms(x, y) - ref) <= 4 * np.spacing(scale)).all()


@pytest.mark.parametrize("seed", [2, 3])
def test_focal_terms_match_torchvision(seed):
    from torchvision.ops import sigmoid_focal_loss
    x, y = _logits(seed)
    ref = sigmoid_focal_loss(torch.from_numpy(x), torch.from_numpy(y), alpha=0.25, gamma=2, reduction="none").numpy()
    got = VO.focal_terms(x, y, sigmoid=_torch_op(torch.sigmoid), log_sigmoid=_torch_op(F.logsigmoid))
    assert _ulps(got, ref).max() <= 1
    assert _ulps(VO.sigmoid(x), torch.sigmoid(torch.from_numpy(x)).numpy()).max() <= 2


def test_means_are_exact_and_rounded_once():
    x, y = _logits(4, 5000)
    t = VO.bce_terms(x, y)
    exact = sum(Fraction(float(v)) for v in t) / len(t)
    assert VO.exact_mean(t) == np.float32(float(exact))
    assert VO.exact_mean(t) == np.float32(math.fsum(t.astype(np.float64)) / t.size)
    assert np.isnan(VO.exact_mean(np.zeros(0, np.float32)))
    # the weighted epoch mean
    vals, bs = [np.float32(0.25), np.float32(1.0 / 3.0), np.float32(7.5)], [2, 3, 1]
    exact = sum(Fraction(float(v)) * b for v, b in zip(vals, bs)) / sum(bs)
    assert VO.epoch_mean(vals, bs) == np.float32(float(exact))


@pytest.mark.parametrize("seed", [5, 6, 7])
def test_iou_and_f1_match_sklearn(seed):
    rng = np.random.default_rng(seed)
    n = 4000
    s = rng.random(n).astype(np.float32)
    s[:50] = 0.5                          # exact ties at the threshold count as negative
    y = rng.random(n) < 0.3
    tp, fp, fn, _ = VO.counts(s, y)
    pred = s > 0.5
    assert VO.iou(tp, fp, fn) == pytest.approx(jaccard_score(y, pred), rel=2 ** -23)
    assert VO.f1(tp, fp, fn) == pytest.approx(f1_score(y, pred), rel=2 ** -22)
    assert iou_from_counts(tp, fp, fn).item() == float(VO.iou(tp, fp, fn))
    assert f1_from_counts(tp, fp, fn).item() == float(VO.f1(tp, fp, fn))


def test_zero_denominators():
    y = np.zeros(10, bool)
    pred = np.zeros(10, bool)
    assert VO.iou(0, 0, 0) == 0 == jaccard_score(y, pred, zero_division=0)
    assert VO.f1(0, 0, 0) == 0 == f1_score(y, pred, zero_division=0)
    assert iou_from_counts(0, 0, 0).item() == 0.0 and f1_from_counts(0, 0, 0).item() == 0.0


def test_counts_past_2_24_round_as_torchmetrics():
    tp, fp, fn = 2 ** 24 + 1, 3, 2 ** 24 + 3
    # (f32(fp) + f32(fn)) + f32(tp), not f32(tp + fp + fn)
    expect = np.float32(2 ** 24) / ((np.float32(3) + np.float32(2 ** 24 + 4)) + np.float32(2 ** 24))
    assert VO.iou(tp, fp, fn) == expect == np.float32(iou_from_counts(tp, fp, fn).item())


def test_all_invalid_topology_gives_nan_topo_loss():
    ml = np.zeros((1, 4, 4, 2), np.float32)
    m = np.ones((1, 4, 4), np.float32)
    mask_loss, topo_loss, loss = VO.step_values(ml, m, m, np.zeros(6, np.float32), np.ones(6), np.zeros(6))
    assert mask_loss == np.float32(math.log(2)) and np.isnan(topo_loss) and np.isnan(loss)
    # torch on the same data, the reference's expression
    tl = F.binary_cross_entropy_with_logits(torch.zeros(6), torch.ones(6), reduction="none")
    assert torch.isnan((tl * torch.zeros(6)).sum() / torch.zeros(6).sum())
    c = VO.step_counts(np.full((1, 4, 4, 2), 0.5, np.float32), m, m, np.ones(6, np.float32), np.ones(6), np.zeros(6))
    assert (c["topo_tp"], c["topo_fp"], c["topo_fn"]) == (0, 0, 0) and VO.f1(0, 0, 0) == 0


def test_validation_step_targets_mapping():
    valid = torch.tensor([[[True, False, True]]])
    connected = torch.tensor([[[True, True, False]]])
    m = torch.ones(1, 2, 2)
    kp, road, topo, val, f1_gt = VO.validation_step_targets(
        dict(keypoint_mask=m, road_mask=m, valid=valid, connected=connected))
    assert topo.view(-1).tolist() == [1.0, 1.0, 0.0] and val.view(-1).tolist() == [True, False, True]
    assert f1_gt.view(-1).tolist() == [1, -1, 0]


def test_val_symbols_bound_and_reject_bad_arguments_without_gpu():
    lib = _lib.load()
    for name in ("create", "destroy", "reset", "update", "read"):
        assert f"samroad_val_{name}" in _lib.SIGNATURES
    # argument checks come before any CUDA call
    assert lib.samroad_val_create(0, None) != 0
    assert lib.samroad_val_reset(None, None) != 0
    assert lib.samroad_val_update(None, *([None] * 8), 1, 16, 1, 1, 0, None, None) != 0
    assert lib.samroad_val_read(None, None, None, None, None) != 0
    assert lib.samroad_val_destroy(None) == 0
