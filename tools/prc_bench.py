"""Threshold search at the CityScale test size: the exact precision-recall curves of sam_road_b200.metrics
against torch.sort + cumsum computing the same curve, on the same card, alternating round by round.

Workload: 432 evaluation patches of 512^2 (27 scenes x 16 patches), mask scores [432,512,512,2] read as
strided channel views in batches of --batch patches (what test_step hands over), float targets 0.0 / 1.0;
topology: 432 x 512 samples x 16 pairs with a valid mask.  Scores are sigmoid(logits) in float32, so most
scores are distinct, as a model's are.

torch leg: torchmetrics' _binary_clf_curve on the concatenated scores (argsort descending, stable; float32
cumsum of the labels at the last index of every distinct score; precision, recall), started from contiguous
flat tensors (the concatenation torchmetrics does first is not timed).  Agreement is checked against the
same torch pipeline with an int64 cumsum (exact), and the largest deviation of the float32-cumsum curve is
reported.  Prints one JSON object.

    python tools/prc_bench.py [--rounds 3] [--batch 16] [--patches 432]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200.metrics import PrecisionRecallCurve  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def torch_curve(preds, target, exact=False):
    """torchmetrics _binary_clf_curve + _binary_precision_recall_curve_compute (no truncation), ascending."""
    order = torch.argsort(preds, descending=True, stable=True)
    p, t = preds[order], target[order]
    distinct = torch.where(p[1:] - p[:-1])[0]
    idx = torch.cat([distinct, torch.tensor([p.numel() - 1], device=p.device)])
    if exact:
        tps_i = torch.cumsum(t.to(torch.int64), 0)[idx]
        tps, fps = tps_i.to(torch.float32), (1 + idx - tps_i).to(torch.float32)
    else:
        tps = torch.cumsum(t, 0)[idx]
        fps = 1 + idx - tps
    prec = tps / (tps + fps)
    rec = tps / tps[-1]
    one, zero = torch.ones(1, device=p.device), torch.zeros(1, device=p.device)
    return torch.cat([prec.flip(0), one]), torch.cat([rec.flip(0), zero]), p[idx].flip(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--patches", type=int, default=432)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    n_p, P, S, K = a.patches, 512, 512, 16
    scores = torch.sigmoid(2.5 * torch.randn((n_p, P, P, 2), generator=g, device=dev) - 1.0)
    # 0/1 float labels correlated with the scores (a 0/255 mask divided by 255)
    masks = [(torch.rand((n_p, P, P), generator=g, device=dev) < scores[..., c] ** 2).float() for c in range(2)]
    topo = torch.sigmoid(3.0 * torch.randn((n_p, S, K, 1), generator=g, device=dev))
    connected = torch.rand((n_p, S, K), generator=g, device=dev) < topo[..., 0]
    valid = torch.rand((n_p, S, K), generator=g, device=dev) < 0.6
    curves = [PrecisionRecallCurve(dev) for _ in range(3)]

    def ours_update():
        for c in curves:
            c.reset()
        for b0 in range(0, n_p, a.batch):
            b1 = min(n_p, b0 + a.batch)
            curves[0].update(scores[b0:b1, ..., 0], masks[0][b0:b1])
            curves[1].update(scores[b0:b1, ..., 1], masks[1][b0:b1])
            curves[2].update(topo[b0:b1], connected[b0:b1], valid[b0:b1])

    flat = [(scores[..., c].reshape(-1).contiguous(), masks[c].reshape(-1).contiguous()) for c in range(2)]
    keep = valid.reshape(-1)
    flat.append((topo.reshape(-1)[keep].contiguous(), connected.reshape(-1)[keep].float().contiguous()))
    names = ("keypoint", "road", "topo")
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        e[0].record()
        out = fn()
        e[1].record()
        e[1].synchronize()
        return e[0].elapsed_time(e[1]), out

    t_upd, t_cmp = [], {k: [] for k in names}
    t_torch = {k: [] for k in names}
    for r in range(a.rounds + 1):           # round 0 warms every shape up and is not counted
        ms_u, _ = timed(ours_update)
        ms_c = [timed(c.compute)[0] for c in curves]
        ms_t = [timed(lambda f=f: torch_curve(*f))[0] for f in flat]
        if r:
            t_upd.append(ms_u)
            for k, mc, mt in zip(names, ms_c, ms_t):
                t_cmp[k].append(mc)
                t_torch[k].append(mt)
    res = {"card": _card(), "patches": n_p, "patch": P, "topo": [S, K], "batch": a.batch, "rounds": a.rounds,
           "update_ms_all_three": {"min": min(t_upd), "max": max(t_upd)}, "curves": {}}
    for k, c, f in zip(names, curves, flat):
        prec, rec, thr = c.compute()
        (n, n_pos, T, _), best = c._best
        ep, er, et = torch_curve(*f, exact=True)
        fp, fr, _ = torch_curve(*f)
        agree = bool(torch.equal(thr, et) and torch.equal(prec.view(torch.int32), ep.view(torch.int32))
                     and torch.equal(rec.view(torch.int32), er.view(torch.int32)))
        res["curves"][k] = {
            "entries": n, "positives": n_pos, "thresholds": T,
            "compute_ms": {"min": min(t_cmp[k]), "max": max(t_cmp[k])},
            "torch_sort_cumsum_ms": {"min": min(t_torch[k]), "max": max(t_torch[k])},
            "bit_equal_to_torch_int64_cumsum": agree,
            "float32_cumsum_max_abs_dev": {"precision": float((fp - prec).abs().max()),
                                           "recall": float((fr - rec).abs().max())},
            "best": list(best),
        }
        assert agree, f"{k}: curves differ"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
