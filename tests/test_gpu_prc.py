"""GPU: the exact precision-recall curves of sam_road_b200.metrics and SAMRoad.test_step / on_test_end,
bit for bit against the NumPy oracle (oracle/prc_oracle.py)."""
import re

import numpy as np
import pytest
import torch

from oracle import prc_oracle as PO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200.metrics import PrecisionRecallCurve

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _same_bits(a, b):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    assert a.shape == b.shape, (a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    np.testing.assert_array_equal(na, nb)
    np.testing.assert_array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _check(curve, preds, target):
    """curve's result equals the oracle's on (preds, target with -1 = ignored), float32 bits."""
    prec, rec, thr, tps, fps = (t.cpu().numpy() for t in curve.compute(with_counts=True))
    oprec, orec, othr, otps, ofps = PO.binary_pr_curve(preds, target, return_counts=True)
    _same_bits(thr, othr)
    _same_bits(prec, oprec)
    _same_bits(rec, orec)
    np.testing.assert_array_equal(tps, otps)
    np.testing.assert_array_equal(fps, ofps)
    i, t, p, r, f1 = PO.find_best_threshold(oprec, orec, othr)
    _same_bits([x.item() for x in curve.best()], [t, p, r, f1])
    return prec, rec, thr


def _tied(gen, shape):
    k = torch.randint(0, 256, shape, generator=gen)
    k[torch.rand(shape, generator=gen) < 0.1] = 0
    k[torch.rand(shape, generator=gen) < 0.1] = 255
    return k.float() / 255.0


def test_strided_channel_views_and_float_targets():
    gen = torch.Generator().manual_seed(0)
    B, P = 3, 64
    scores = torch.stack([_tied(gen, (B, P, P)), torch.rand((B, P, P), generator=gen)], -1).to(DEV)
    assert not scores[..., 0].is_contiguous()
    # dataset-style targets mask / 255: only 255 / 255 truncates to 1
    masks = [torch.randint(0, 256, (B, P, P), generator=gen).float() for _ in range(2)]
    for m in masks:
        m[torch.rand((B, P, P), generator=gen) < 0.3] = 255.0
    for c in range(2):
        curve = PrecisionRecallCurve(DEV)
        tgt = (masks[c] / 255.0).to(DEV)
        curve.update(scores[..., c], tgt)
        _check(curve, scores[..., c].cpu().numpy(), (masks[c] / 255.0).to(torch.int32).numpy())


def test_byte_targets_with_valid():
    gen = torch.Generator().manual_seed(1)
    shape = (4, 40, 16, 1)
    preds = _tied(gen, shape).to(DEV)
    connected = torch.rand(shape[:3], generator=gen) < 0.4
    valid = torch.rand(shape[:3], generator=gen) < 0.7
    curve = PrecisionRecallCurve(DEV)
    curve.update(preds, connected.to(DEV), valid.to(DEV))
    target = torch.where(valid, connected.to(torch.int64), torch.full_like(connected, -1, dtype=torch.int64))
    _check(curve, preds.cpu().numpy(), target.numpy())


def test_split_and_permutation_invariance():
    gen = torch.Generator().manual_seed(2)
    n = 200_000
    preds = torch.cat([_tied(gen, (n // 2,)), torch.rand(n // 2, generator=gen)])
    target = (torch.rand(n, generator=gen) < preds * 0.7).to(torch.uint8)
    whole = PrecisionRecallCurve(DEV)
    whole.update(preds.to(DEV), target.to(DEV))
    ref = _check(whole, preds.numpy(), target.numpy())
    perm = torch.randperm(n, generator=gen)
    split = PrecisionRecallCurve(DEV)
    bounds = [0, 1, 77, 5000, 120_000, n]
    for a, b in zip(bounds[:-1], bounds[1:]):
        idx = perm[a:b]
        split.update(preds[idx].to(DEV), target[idx].to(DEV))
    for x, y in zip(ref, split.compute()):
        _same_bits(x, y.cpu().numpy())
    # state persists across compute calls and is dropped by reset
    split.update(preds[:10].to(DEV), target[:10].to(DEV))
    _check(split, torch.cat([preds, preds[:10]]).numpy(), torch.cat([target, target[:10]]).numpy())
    split.reset()
    split.update(preds[:1000].to(DEV), target[:1000].to(DEV))
    _check(split, preds[:1000].numpy(), target[:1000].numpy())


@pytest.mark.parametrize("n", [1, 4095, 4096, 4097, 65_537])
def test_entry_counts_around_one_scan_tile(n):
    """One and two 4096-key sort chunks and curve tiles, and 17 chunks, whose 256 x 17 histogram is scanned in
    more than one tile."""
    gen = torch.Generator().manual_seed(n)
    preds = _tied(gen, (n,))
    target = (torch.rand(n, generator=gen) < preds * 0.7).to(torch.uint8)
    curve = PrecisionRecallCurve(DEV)
    curve.update(preds.to(DEV), target.to(DEV))
    _check(curve, preds.numpy(), target.numpy())


def test_exact_counts_past_2_24():
    # 3e7 entries, ~1.8e7 positives: float32 partial sums would round above 2^24
    n = 30_000_000
    g = torch.Generator(device=DEV).manual_seed(3)
    preds = torch.randint(0, 1001, (n,), generator=g, device=DEV).float() / 1000.0
    target = (torch.rand(n, generator=g, device=DEV) < 0.6).to(torch.uint8)
    curve = PrecisionRecallCurve(DEV)
    for part in range(3):   # three updates make the key buffer grow
        sl = slice(part * n // 3, (part + 1) * n // 3)
        curve.update(preds[sl], target[sl])
    prec, rec, thr, tps, fps = (t.cpu().numpy() for t in curve.compute(with_counts=True))
    p_host, t_host = preds.cpu().numpy(), target.cpu().numpy()
    vals, count = np.unique(p_host, return_counts=True)
    pos = np.zeros_like(count)
    pv, pc = np.unique(p_host[t_host == 1], return_counts=True)
    pos[np.searchsorted(vals, pv)] = pc
    exp_tps = np.cumsum(pos[::-1])[::-1]
    exp_fps = np.cumsum(count[::-1])[::-1] - exp_tps
    assert exp_tps[0] > 2 ** 24 and exp_fps[0] > 2 ** 23
    _same_bits(thr, vals)
    np.testing.assert_array_equal(tps, exp_tps)
    np.testing.assert_array_equal(fps, exp_fps)
    tf, ff = exp_tps.astype(np.float32), exp_fps.astype(np.float32)
    _same_bits(prec[:-1], tf / (tf + ff))
    _same_bits(rec[:-1], tf / np.float32(exp_tps[0]))


@pytest.mark.parametrize("bad", ["score_1.5", "score_nan", "target_2"])
def test_rejected_update_adds_nothing(bad):
    gen = torch.Generator().manual_seed(4)
    good_p = _tied(gen, (5000,))
    good_t = (torch.rand(5000, generator=gen) < 0.5).float()
    bad_p, bad_t = good_p[:100].clone(), good_t[:100].clone()
    if bad == "score_1.5":
        bad_p[37] = 1.5
    elif bad == "score_nan":
        bad_p[37] = float("nan")
    else:
        bad_t[37] = 2.0
    curve = PrecisionRecallCurve(DEV)
    curve.update(good_p[:2500].to(DEV), good_t[:2500].to(DEV))
    curve.update(bad_p.to(DEV), bad_t.to(DEV))
    with pytest.raises(RuntimeError, match=r"code 3.* 1 update\(s\) .*refused.*update #1 .*element 37: a (prediction|target)"):
        curve.compute()
    _check(curve, good_p[:2500].numpy(), good_t[:2500].to(torch.int32).numpy())
    curve.update(good_p[2500:].to(DEV), good_t[2500:].to(DEV))
    _check(curve, good_p.numpy(), good_t.to(torch.int32).numpy())


def test_every_refused_update_is_reported():
    gen = torch.Generator().manual_seed(6)
    p = _tied(gen, (3000,))
    t = (torch.rand(3000, generator=gen) < 0.5).to(torch.uint8)
    bad = p[:50].clone()
    bad[3] = -0.5
    curve = PrecisionRecallCurve(DEV)
    for k in range(6):    # updates #1 and #4 are refused
        sl = slice(k * 500, (k + 1) * 500)
        if k in (1, 4):
            curve.update(bad.to(DEV), t[:50].to(DEV))
        else:
            curve.update(p[sl].to(DEV), t[sl].to(DEV))
    with pytest.raises(RuntimeError, match=r" 2 update\(s\) .*update #1 .*element 3"):
        curve.compute()
    keep = torch.cat([torch.arange(k * 500, (k + 1) * 500) for k in (0, 2, 3, 5)])
    _check(curve, p[keep].numpy(), t[keep].numpy())      # both were reported, nothing is missing silently
    curve.update(bad.to(DEV), t[:50].to(DEV))            # a refusal after the report is reported again
    with pytest.raises(RuntimeError, match=r" 1 update\(s\) .*update #6 "):
        curve.compute()
    _check(curve, p[keep].numpy(), t[keep].numpy())


def test_no_positives_and_nan_best_point():
    curve = PrecisionRecallCurve(DEV)
    preds = torch.tensor([0.5, 0.25, 0.75, 0.25])
    curve.update(preds.to(DEV), torch.zeros(4, dtype=torch.uint8, device=DEV))
    _check(curve, preds.numpy(), np.zeros(4, np.int64))
    thr, p, r, f1 = (x.item() for x in curve.best())
    assert thr == 0.25 and np.isnan(r) and np.isnan(f1)
    curve = PrecisionRecallCurve(DEV)
    preds = torch.tensor([0.1, 0.2, 0.3, 0.8, 0.9])
    curve.update(preds.to(DEV), torch.tensor([1, 0, 1, 0, 0], dtype=torch.uint8, device=DEV))
    _check(curve, preds.numpy(), np.array([1, 0, 1, 0, 0]))
    assert curve.best()[0].item() == np.float32(0.8)


_LINE = re.compile(r"^Best threshold (\S+), P=(\S+) R=(\S+) F1=(\S+)$")


@pytest.mark.parametrize("P,n_points,n_samples", [(256, 40, 24), (512, 90, 50)])
def test_test_step_matches_oracle_on_device_scores(P, n_points, n_samples, capsys):
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=P, USE_SAM_DECODER=False, ENCODER_LORA=False,
               TOPONET_VERSION="normal", NO_SAM=False)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=8.0), strict=True)
    net.eval().to(DEV)
    gen = torch.Generator().manual_seed(5)
    labels = {k: [] for k in ("keypoint", "road", "topo")}
    scores = {k: [] for k in ("keypoint", "road", "topo")}
    for step in range(3):
        B = 2
        rgb = synth.make_tiles(B, P, seed=10 + step, dtype=torch.float32)
        pts, prs, val = synth.make_topo_inputs(B, P, n_points, seed=20 + step)
        # TOPO_SAMPLE_NUM-style: Ns sampled source points out of N
        prs, val = prs[:, :n_samples], val[:, :n_samples]
        masks = [torch.randint(0, 256, (B, P, P), generator=gen).float() for _ in range(2)]
        for m in masks:
            m[torch.rand((B, P, P), generator=gen) < 0.2] = 255.0
        batch = {
            "rgb": rgb, "keypoint_mask": masks[0] / 255.0, "road_mask": masks[1] / 255.0,
            "graph_points": pts.float(), "pairs": prs.to(torch.int32),
            "connected": torch.rand(val.shape, generator=gen) < 0.5, "valid": val,
        }
        batch = {k: v.to(DEV) for k, v in batch.items()}
        net.test_step(batch, step)
        # the same device calls test_step makes, for the oracle
        ms, emb = net.infer_masks_and_img_features(batch["rgb"])
        ts = net.infer_toponet(emb, batch["graph_points"], batch["pairs"], batch["valid"])
        kp, road, topo = PO.test_step_targets({k: v.cpu() for k, v in batch.items()})
        for name, s, t in (("keypoint", ms[..., 0], kp), ("road", ms[..., 1], road), ("topo", ts, topo)):
            scores[name].append(s.cpu().numpy().ravel())
            labels[name].append(t.numpy().ravel())
    best = net.on_test_end()
    out = capsys.readouterr().out.strip().splitlines()
    assert out[0] == "======= Finding best thresholds ======"
    for k, name in enumerate(("keypoint", "road", "topo")):
        s, t = np.concatenate(scores[name]), np.concatenate(labels[name])
        _check(net._test_curves[k], s, t)
        i, thr, p, r, f1 = PO.find_best_threshold(*PO.binary_pr_curve(s, t))
        assert out[1 + 2 * k] == f"======= {name} ======"
        m = _LINE.match(out[2 + 2 * k])
        assert m, out[2 + 2 * k]
        expect = tuple(str(float(v)) for v in (thr, p, r, f1))    # str: an F1 of NaN prints as nan
        assert m.groups() == expect
        assert tuple(map(str, best[name])) == expect and net.best_thresholds is best
    net.reset_test_metrics()
    with pytest.raises(RuntimeError, match="no test_step"):
        net.on_test_end()
