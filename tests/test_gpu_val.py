"""GPU: the validation losses and metrics of sam_road_b200.metrics.ValidationMetrics and SAMRoad.validation_step
/ on_validation_epoch_end, against torch on the same device tensors and the NumPy oracle
(oracle/val_oracle.py)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import val_oracle as VO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200.metrics import VAL_COUNT_NAMES, ValidationMetrics

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SPECIAL = [0.0, -0.0, 20.0, -20.0, 90.0, -90.0]


def _ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    if np.isnan(a) or np.isnan(b):
        return 0 if (np.isnan(a) and np.isnan(b)) else 1 << 31
    ia, ib = int(np.array(a).view(np.int32)), int(np.array(b).view(np.int32))
    ia = -(ia & 0x7FFFFFFF) if ia < 0 else ia
    ib = -(ib & 0x7FFFFFFF) if ib < 0 else ib
    return abs(ia - ib)


def _f32_mean(terms):
    t = terms.double().cpu().numpy().ravel()
    return np.float32(math.fsum(t) / t.size) if t.size else np.float32(np.nan)


def _torch_terms(x, y, focal):
    if focal:
        from torchvision.ops import sigmoid_focal_loss
        return sigmoid_focal_loss(x, y, alpha=0.25, gamma=2, reduction="none")
    return F.binary_cross_entropy_with_logits(x, y, reduction="none")


def _inputs(B, P, Ns, Np, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ml = torch.randn((B, P, P, 2), generator=g, device=DEV) * 6
    flat = ml.view(-1)
    flat[: 8 * len(SPECIAL)] = torch.tensor(SPECIAL * 8, device=DEV)     # ±0 give scores of exactly 0.5
    kp = (torch.rand((B, P, P), generator=g, device=DEV) < 0.3).float()
    road = (torch.rand((B, P, P), generator=g, device=DEV) < 0.5).float()
    tl = torch.randn((B, Ns, Np, 1), generator=g, device=DEV) * 5
    tl.view(-1)[: len(SPECIAL)] = torch.tensor(SPECIAL, device=DEV)
    connected = torch.rand((B, Ns, Np), generator=g, device=DEV) < 0.4
    valid = torch.rand((B, Ns, Np), generator=g, device=DEV) < 0.7
    return ml, torch.sigmoid(ml), kp, road, tl, torch.sigmoid(tl), connected, valid


def _torch_step(ml, ms, kp, road, tl, ts, connected, valid, focal):
    """Reference formulas on the device: (mask_loss, topo_loss, loss) to check within 1 ulp, and the counts."""
    gt = torch.stack([kp, road], 3)
    m = _f32_mean(_torch_terms(ml, gt, focal))
    tt = F.binary_cross_entropy_with_logits(tl[..., 0], connected.float(), reduction="none")[valid]
    t = _f32_mean(tt)
    c = {}
    for name, ch, y in (("keypoint", 0, kp), ("road", 1, road)):
        pred, lab = ms[..., ch] > 0.5, y == 1
        c.update({f"{name}_tp": int((pred & lab).sum()), f"{name}_fp": int((pred & ~lab).sum()),
                  f"{name}_fn": int((~pred & lab).sum()), f"{name}_tn": int((~pred & ~lab).sum())})
    pred, lab = ts[..., 0][valid] > 0.5, connected[valid]
    c.update(topo_tp=int((pred & lab).sum()), topo_fp=int((pred & ~lab).sum()), topo_fn=int((~pred & lab).sum()))
    return (m, t, np.float32(m + t)), c


@pytest.mark.parametrize("focal", [False, True])
@pytest.mark.parametrize("B,P,Ns,Np", [(3, 256, 40, 7), (2, 512, 50, 16), (3, 256, 24, 32)])
def test_step_against_torch(B, P, Ns, Np, focal):
    args = _inputs(B, P, Ns, Np, seed=B * 1000 + P + Np)
    assert int((args[1] == 0.5).sum()) >= 16            # exact ties at the threshold
    vm = ValidationMetrics(DEV, focal=focal)
    out = vm.update(*args).cpu().numpy()
    expect, counts = _torch_step(*args, focal=focal)
    for got, want in zip(out, expect):
        assert _ulps(got, want) <= 1, (out, expect)
    c, means, totals = vm.read()
    assert c == counts
    assert totals == (1, B)
    for got, want in zip(means, out):          # one step: the epoch mean is the step value
        assert np.float32(got) == want


def test_terms_one_by_one_against_torch():
    """Every term on its own (a 1x1 tile with both channels equal, one valid pair slot): the kernels' float32
    expressions against torch's on the same device."""
    x = torch.cat([torch.tensor(SPECIAL), torch.linspace(-30, 30, 121), torch.randn(60) * 8]).to(DEV)
    worst = {"bce": 0, "focal": 0, "topo": 0}
    vms = {False: ValidationMetrics(DEV, focal=False), True: ValidationMetrics(DEV, focal=True)}
    one = torch.ones((1, 1, 1), dtype=torch.bool, device=DEV)
    for y in (0.0, 1.0):
        for focal in (False, True):
            ref = _torch_terms(x, torch.full_like(x, y), focal).cpu().numpy()
            for i in range(x.numel()):
                ml = x[i].view(1, 1, 1, 1).expand(1, 1, 1, 2).contiguous()
                m = torch.full((1, 1, 1), y, device=DEV)
                out = vms[focal].update(ml, torch.sigmoid(ml), m, m, ml[..., :1], torch.sigmoid(ml[..., :1]),
                                        one if y else ~one, one).cpu().numpy()
                worst["focal" if focal else "bce"] = max(worst["focal" if focal else "bce"], _ulps(out[0], ref[i]))
                if not focal:
                    worst["topo"] = max(worst["topo"], _ulps(out[1], ref[i]))
    print(f"largest term-wise difference to torch, in ulps: {worst}")
    assert max(worst.values()) <= 1, worst


def test_counts_past_2_24():
    B, P = 1, 4200                                     # 1.76e7 pixels, ~1.7e7 keypoint positives
    g = torch.Generator(device=DEV).manual_seed(7)
    ml = torch.randn((B, P, P, 2), generator=g, device=DEV) + 3
    ms = torch.sigmoid(ml)
    kp = (torch.rand((B, P, P), generator=g, device=DEV) < 0.97).float()
    road = (torch.rand((B, P, P), generator=g, device=DEV) < 0.5).float()
    Ns, Np = 8, 4
    tl = torch.randn((B, Ns, Np, 1), generator=g, device=DEV)
    con = torch.ones((B, Ns, Np), dtype=torch.bool, device=DEV)
    vm = ValidationMetrics(DEV)
    vm.update(ml, ms, kp, road, tl, torch.sigmoid(tl), con, con)
    c, _, _ = vm.read()
    pred, lab = ms[..., 0] > 0.5, kp == 1
    tp = int((pred & lab).sum(dtype=torch.int64))
    fp, fn = int((pred & ~lab).sum(dtype=torch.int64)), int((~pred & lab).sum(dtype=torch.int64))
    assert tp > 2 ** 24 and (c["keypoint_tp"], c["keypoint_fp"], c["keypoint_fn"]) == (tp, fp, fn)
    assert c["keypoint_tn"] == B * P * P - tp - fp - fn
    vm.update(ml, ms, kp, road, tl, torch.sigmoid(tl), con, con)
    res = vm.compute()
    assert np.float32(res["keypoint_iou"]) == VO.iou(2 * tp, 2 * fp, 2 * fn)


def test_determinism_and_split_invariance():
    args = _inputs(4, 256, 30, 16, seed=11)
    a, b = ValidationMetrics(DEV), ValidationMetrics(DEV)
    o1, o2 = a.update(*args).cpu(), b.update(*args).cpu()
    assert torch.equal(o1.view(torch.int32), o2.view(torch.int32))
    whole, _, _ = a.read()
    split = ValidationMetrics(DEV)
    for lo, hi in ((0, 1), (1, 3), (3, 4)):
        split.update(*(t[lo:hi] for t in args))
    c, _, totals = split.read()
    assert c == whole and totals == (3, 4)


def _net(focal=False):
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False, ENCODER_LORA=False,
               TOPONET_VERSION="normal", NO_SAM=False, FOCAL_LOSS=focal)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=8.0), strict=True)
    return net.eval().to(DEV)


def _batch(B, seed, n_points=40, n_samples=24):
    gen = torch.Generator().manual_seed(seed)
    pts, prs, val = synth.make_topo_inputs(B, 256, n_points, seed=seed + 1)
    prs, val = prs[:, :n_samples], val[:, :n_samples]
    batch = {"rgb": synth.make_tiles(B, 256, seed=seed + 2, dtype=torch.float32),
             "keypoint_mask": (torch.rand((B, 256, 256), generator=gen) < 0.2).float(),
             "road_mask": (torch.rand((B, 256, 256), generator=gen) < 0.4).float(),
             "graph_points": pts.float(), "pairs": prs.to(torch.int32),
             "connected": torch.rand(val.shape, generator=gen) < 0.5, "valid": val}
    return {k: v.to(DEV) for k, v in batch.items()}


@pytest.mark.parametrize("focal", [False, True])
def test_validation_step_and_epoch_end(focal):
    net = _net(focal)
    assert net.focal_loss is focal
    steps, bs, totals = [], [], {k: 0 for k in VAL_COUNT_NAMES}
    for i, B in enumerate((2, 3, 1)):
        batch = _batch(B, seed=50 + 10 * i)
        res = net.validation_step(batch, i)
        assert set(res) == {"val_mask_loss", "val_topo_loss", "val_loss"}
        assert all(v.dim() == 0 and v.device == DEV for v in res.values())
        ml, ms, tl, ts = net(batch["rgb"], batch["graph_points"], batch["pairs"], batch["valid"])
        expect, counts = _torch_step(ml, ms, batch["keypoint_mask"], batch["road_mask"], tl, ts,
                                     batch["connected"], batch["valid"], focal)
        got = [res[k].item() for k in ("val_mask_loss", "val_topo_loss", "val_loss")]
        for g_, e_ in zip(got, expect):
            assert _ulps(g_, e_) <= 1, (got, expect)
        # the oracle's counts on the same scores
        oc = VO.step_counts(ms.cpu().numpy(), batch["keypoint_mask"].cpu().numpy(),
                            batch["road_mask"].cpu().numpy(), ts.cpu().numpy(), batch["connected"].cpu().numpy(),
                            batch["valid"].cpu().numpy())
        assert oc == counts
        for k in totals:
            totals[k] += oc[k]
        steps.append(got)
        bs.append(B)
    out = net.on_validation_epoch_end()
    assert net.val_metrics is out
    for k, name in enumerate(("val_mask_loss", "val_topo_loss", "val_loss")):
        assert np.float32(out[name]) == VO.epoch_mean([s[k] for s in steps], bs)
    for name, v in VO.epoch_metrics(totals).items():
        assert np.array(np.float32(out[name])).view(np.uint32) == np.array(v).view(np.uint32), (name, out[name], v)
    # the epoch end reset the accumulator
    assert net._val_metrics.read()[2] == (0, 0)


def test_refused_step_and_next_epoch():
    net = _net()
    good = _batch(2, seed=90)
    bad = dict(good)
    km = good["keypoint_mask"].clone()
    km[1, 5, 7] = 0.5
    bad["keypoint_mask"] = km
    net.validation_step(good, 0)
    res = net.validation_step(bad, 1)
    assert all(math.isnan(v.item()) for v in res.values())
    P = 256
    with pytest.raises(RuntimeError, match=r"code 3.* 1 update\(s\) .*update #1 .*element "
                                           rf"{2 * ((1 * P + 5) * P + 7)}: a mask target"):
        net.on_validation_epoch_end()
    r0 = net.validation_step(good, 0)
    out = net.on_validation_epoch_end()
    assert out["val_loss"] == r0["val_loss"].item()


def test_lightning_logging_names_and_flags():
    net = _net()
    calls = []
    net.log = lambda name, value, **kw: calls.append((name, kw, value))
    net.validation_step(_batch(2, seed=120), 0)
    assert calls == []                                  # no trainer attached: nothing is logged
    net._trainer = object()
    net.validation_step(_batch(2, seed=130), 1)
    assert [(n, kw) for n, kw, _ in calls] == [(n, dict(on_step=False, on_epoch=True, prog_bar=True))
                                               for n in ("val_mask_loss", "val_topo_loss", "val_loss")]
    calls.clear()
    out = net.on_validation_epoch_end()
    assert [(n, kw) for n, kw, _ in calls] == [(n, {}) for n in ("keypoint_iou", "road_iou", "topo_f1")]
    assert all(v.item() == np.float32(out[n]) for n, _, v in calls)
    import copy
    assert net._val_metrics is not None and copy.deepcopy(net)._val_metrics is None
    assert net.__getstate__()["_val_metrics"] is None
    net.reset_validation_metrics()
    assert net.val_metrics is None and net._val_metrics is None
    with pytest.raises(NotImplementedError):
        net.training_step(None, 0)
