"""One validation step at the training batch size: sam_road_b200.metrics.ValidationMetrics.update against the
torch composition of the reference's ops, on the same card, alternating round by round.

Workload: B = 64 tiles of 512^2 (mask logits and scores [64,512,512,2], float 0.0 / 1.0 masks) and
Ns = 512 (TOPO_SAMPLE_NUM) x Np = 16 pair slots per tile.

torch leg (validation_step, model.py:555-588): torch.stack of the two masks, BCEWithLogitsLoss (mean), the
masked topology BCE sum / valid.sum(), and for each of the three metrics the comparisons against 0.5 reduced
with .sum() (standing in for the torchmetrics updates, which do more).

Reports the update's time against the bytes it must read (both passes) and the share of the 3.35 TB/s
data-sheet HBM3 bound, and, next to the forward pass, the share of a whole SAMRoad.validation_step (ViT-B
with synthetic weights) the update takes.  Prints one JSON object.

    python tools/val_bench.py [--rounds 5] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import SAMRoad, synth  # noqa: E402
from sam_road_b200.metrics import ValidationMetrics  # noqa: E402

HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def torch_step(ml, ms, kp, road, tl, ts, connected, valid):
    gt = torch.stack([kp, road], 3)
    mask_loss = F.binary_cross_entropy_with_logits(ml, gt)
    vf = valid.to(torch.float32)
    topo = F.binary_cross_entropy_with_logits(tl, connected.to(torch.float32).unsqueeze(-1), reduction="none")
    topo_loss = (topo * vf.unsqueeze(-1)).sum() / vf.sum()
    stats = []
    for c, y in ((0, kp), (1, road)):
        pred, lab = ms[..., c] > 0.5, y == 1
        stats += [(pred & lab).sum(), (pred & ~lab).sum(), (~pred & lab).sum()]
    pred, lab = ts[..., 0] > 0.5, connected & valid
    stats += [(pred & lab).sum(), (pred & ~lab & valid).sum(), (~pred & lab).sum()]
    return torch.stack([mask_loss, topo_loss, mask_loss + topo_loss]), stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    B, P, Ns, Np = a.batch, 512, 512, 16
    g = torch.Generator(device=dev).manual_seed(0)
    ml = torch.randn((B, P, P, 2), generator=g, device=dev) * 4
    ms = torch.sigmoid(ml)
    kp = (torch.rand((B, P, P), generator=g, device=dev) < 0.1).float()
    road = (torch.rand((B, P, P), generator=g, device=dev) < 0.2).float()
    tl = torch.randn((B, Ns, Np, 1), generator=g, device=dev) * 3
    ts = torch.sigmoid(tl)
    connected = torch.rand((B, Ns, Np), generator=g, device=dev) < 0.3
    valid = torch.rand((B, Ns, Np), generator=g, device=dev) < 0.6
    args = (ml, ms, kp, road, tl, ts, connected, valid)
    vm = ValidationMetrics(dev)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn, n):
        fn()
        e[0].record()
        for _ in range(n):
            fn()
        e[1].record()
        e[1].synchronize()
        return e[0].elapsed_time(e[1]) / n

    ours, ref = [], []
    for _ in range(a.rounds):
        ours.append(timed(lambda: vm.update(*args), a.iters))
        ref.append(timed(lambda: torch_step(*args), a.iters))
    vm.reset()
    out = vm.update(*args)
    tout, _ = torch_step(*args)
    n_pix, n_slot = B * P * P, B * Ns * Np
    bytes_read = n_pix * (8 + 8 + 4 + 4) + n_slot * (4 + 4 + 1 + 1)

    # a whole validation_step next to its forward pass
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=P, USE_SAM_DECODER=False, ENCODER_LORA=False,
               TOPONET_VERSION="normal", NO_SAM=False)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=8.0), strict=True)
    net.eval().to(dev)
    pts, prs, val = synth.make_topo_inputs(B, P, Ns, seed=1)
    batch = {"rgb": synth.make_tiles(B, P, seed=2, dtype=torch.float32), "keypoint_mask": kp.cpu(),
             "road_mask": road.cpu(), "graph_points": pts.float(), "pairs": prs.to(torch.int32),
             "connected": torch.rand(val.shape) < 0.3, "valid": val}
    batch = {k: v.to(dev) for k, v in batch.items()}
    step_ms, fwd_ms = [], []
    for _ in range(max(2, a.rounds // 2)):
        step_ms.append(timed(lambda: net.validation_step(batch, 1), 3))
        fwd_ms.append(timed(lambda: net(batch["rgb"], batch["graph_points"], batch["pairs"], batch["valid"]), 3))
    net.reset_validation_metrics()
    upd = min(ours)
    res = {
        "card": _card(), "B": B, "patch": P, "Ns": Ns, "Np": Np, "rounds": a.rounds, "iters": a.iters,
        "update_ms": {"min": min(ours), "max": max(ours)},
        "torch_composition_ms": {"min": min(ref), "max": max(ref)},
        "update_bytes_read": bytes_read,
        "update_GB_per_s": bytes_read / (upd * 1e-3) / 1e9,
        "share_of_3.35TB_per_s_bound": bytes_read / HBM_BYTES_PER_S / (upd * 1e-3),
        "validation_step_ms": {"min": min(step_ms), "max": max(step_ms)},
        "forward_ms": {"min": min(fwd_ms), "max": max(fwd_ms)},
        "update_share_of_validation_step": upd / min(step_ms),
        "ours_step_values": out.tolist(), "torch_step_values": tout.tolist(),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
