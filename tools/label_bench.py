"""Device time of one training batch of sam_road_b200.dataset (csrc/labels.cu) next to a training step.

Synthetic cityscale-like scenes (2048 x 2048, a street grid every 48 pixels with overpasses) are written to a
temporary directory; batches of B=16 @512 with TOPO_SAMPLE_NUM 512 and MAX_NEIGHBOR_QUERIES 16 are generated
on the device and timed with CUDA events, alternating with SAMRoad.training_step + backward (ViT-B, frozen
encoder) in the same run.  The numpy oracle's CPU time per sample (oracle/label_oracle.py, the reference's
algorithm with the same draws) is reported as a stand-in for the reference's sample_patch, whose libraries are
not installed here.  The card's name and power limit are read in the same run.

    python tools/label_bench.py [--steps 20] [--warmup 3] [--out path.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import label_oracle as LO  # noqa: E402
from sam_road_b200 import SAMRoad, synth  # noqa: E402
from sam_road_b200 import dataset as D  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--patch", type=int, default=512)
    ap.add_argument("--oracle-samples", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "label_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    cfg = dict(DATASET="cityscale", PATCH_SIZE=a.patch, TOPO_SAMPLE_NUM=512, MAX_NEIGHBOR_QUERIES=16,
               NEIGHBOR_RADIUS=64, ROAD_NMS_RADIUS=16, SAM_VERSION="vit_b", FREEZE_ENCODER=True, BASE_LR=1e-3,
               TOPONET_VERSION="normal", FOCAL_LOSS=False)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_label_scenes(tmp, "cityscale", (0, 1, 2, 3), 2048, seed=1, extent=2032)
        os.chdir(tmp)
        try:
            t0 = time.perf_counter()
            ds = D.SatMapDataset(cfg, is_train=True, dev_run=True, device=dev)
            t_build = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0))
    net = net.to(dev)
    opt = net.configure_optimizers()["optimizer"]
    torch.manual_seed(0)
    t_batch, t_step, t_wall = [], [], []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for it in range(a.warmup + a.steps):
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        ev[0].record()
        batch = ds.batch(a.batch)
        ev[1].record()
        w1 = time.perf_counter()
        loss = net.training_step(batch, it)
        opt.zero_grad()
        loss.backward()
        opt.step()
        ev[2].record()
        torch.cuda.synchronize()
        if it >= a.warmup:
            t_batch.append(ev[0].elapsed_time(ev[1]))
            t_step.append(ev[1].elapsed_time(ev[2]))
            t_wall.append((w1 - w0) * 1e3)
    # oracle CPU time per sample on the device's own draws
    batch, draws = ds._scenes.batch(a.batch, export_draws=True)
    d = {k: v.cpu().numpy() for k, v in draws.items()}
    t_or, n_or = 0.0, 0
    for i in range(a.batch):
        if n_or >= a.oracle_samples:
            break
        scene, x0, y0, rot = (int(v) for v in d["patches"][i])
        sc = ds.scenes[scene]
        m = LO.candidates(sc.points, sc.excluded, x0, y0, a.patch, "index").shape[0]
        if m == 0:
            continue
        t0 = time.perf_counter()
        LO.sample_patch(sc, x0, y0, rot, ds.lc, dict(score=0.9 + (1.0 - 0.9) * d["score_u"][i][:m],
                                                     source_u=d["source_u"][i], noise=d["noise"][i]))
        t_or += time.perf_counter() - t0
        n_or += 1
    name, power = card()
    med = lambda v: float(np.median(v))  # noqa: E731
    res = {"card": name, "power_limit": power, "B": a.batch, "patch": a.patch, "topo_sample_num": 512,
           "max_neighbor_queries": 16, "scenes": len(ds.scenes), "max_patch_points": ds._scenes.cap,
           "scene_points": [int(s.points.shape[0]) for s in ds.scenes], "dataset_build_s": round(t_build, 2),
           "batch_ms_median": med(t_batch), "batch_ms_min": min(t_batch), "batch_ms_max": max(t_batch),
           "batch_wall_ms_median": med(t_wall), "train_step_ms_median": med(t_step), "train_step_ms_min": min(t_step),
           "batch_share_of_step": med(t_batch) / med(t_step), "steps": a.steps,
           "oracle_cpu_ms_per_sample": 1e3 * t_or / max(n_or, 1), "oracle_samples": n_or,
           "points_per_batch": int(batch["graph_points"].shape[1])}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
