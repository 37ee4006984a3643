"""Wall time of the three evaluation commands on a synthetic CityScale split at the launcher's world size: `python -m
sam_road_b200.inferencer`, `topo_metric` and `apls_metric`, each called as its `main()` in this process.

    python tools/eval_bench.py                                   # one GPU
    torchrun --nproc-per-node N tools/eval_bench.py              # N GPUs, one rank each

The split is the 27 CityScale test scenes at 2048², random RGB, with the ViT-B @512 inference grid of the reference's
CityScale config (16 x 16 tiles, margin 64) and synthetic weights; the keypoint and road thresholds come from the
fused masks of one scene, as bench.py sets them.  Under random weights the predicted graphs are not road networks, so
the two metrics score `synth.city_tile` pairs instead (the 2048² street-grid tile of tools/topo_bench.py and
tools/apls_bench.py, one seed per scene).  Every command is timed on rank 0 from a barrier to its return; each ends
with the status all-reduce every rank takes part in, so the time covers the slowest rank, and includes loading the
model (inferencer) and the summary rank 0 writes (metrics).  The files go to a temporary directory, removed at the end.
Rank 0 prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sam_road_b200 import SAMRoad, apls_metric, inferencer, ranks, synth, topo_metric  # noqa: E402

CITY_IDS = [x for x in range(180) if x % 10 == 9 or x % 20 == 8]
CFG = dict(DATASET="cityscale", SAM_VERSION="vit_b", PATCH_SIZE=512, USE_SAM_DECODER=False, ENCODER_LORA=False,
           TOPONET_VERSION="normal", NO_SAM=False, INFER_BATCH_SIZE=64, SAMPLE_MARGIN=64, INFER_PATCHES_PER_EDGE=16,
           TOPO_THRESHOLD=0.5, ITSC_NMS_RADIUS=8, ROAD_NMS_RADIUS=16, NEIGHBOR_RADIUS=64, MAX_NEIGHBOR_QUERIES=16)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def _scene(k, size):
    return np.random.RandomState(5000 + k).randint(0, 256, (size, size, 3)).astype(np.uint8)


def prepare(box, n, size):
    """Scenes, ground truth and metric proposals, checkpoint (written by rank 0)."""
    import cv2
    os.makedirs(os.path.join(box, "cityscale", "20cities"))
    os.makedirs(os.path.join(box, "save", "metrics", "graph"))
    for k, t in enumerate(CITY_IDS[:n]):
        cv2.imwrite(os.path.join(box, "cityscale", "20cities", f"region_{t}_sat.png"), _scene(k, size)[:, :, ::-1])
        gt, prop = synth.city_tile(size, seed=k)
        with open(topo_metric.gt_path("cityscale", os.path.join(box, "cityscale"), t), "wb") as f:
            pickle.dump(gt, f)
        with open(os.path.join(box, "save", "metrics", "graph", f"{t}.p"), "wb") as f:
            pickle.dump(prop, f)
    torch.save({"state_dict": synth.make_state_dict(CFG, seed=0, logit_gain=6.0)}, os.path.join(box, "ckpt.pt"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=len(CITY_IDS), help="the first N CityScale test scenes")
    ap.add_argument("--size", type=int, default=2048)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_bench: needs a CUDA device")
    if not 1 <= a.scenes <= len(CITY_IDS):
        sys.exit(f"eval_bench: --scenes must be in [1, {len(CITY_IDS)}]")
    with ranks.process_group() as (rank, world):
        dev = torch.device("cuda", ranks.local_gpu() if world > 1 else 0)
        box = None
        if rank == 0:
            box = tempfile.mkdtemp(prefix="eval_bench_")
            prepare(box, a.scenes, a.size)
        box = ranks.broadcast(box)      # the others continue once rank 0 has written the split
        cwd = os.getcwd()
        os.chdir(box)
        try:
            # thresholds from one scene's fused masks (every rank computes the same; this also warms the GPU up)
            cfg = dict(CFG, ITSC_THRESHOLD=2.0, ROAD_THRESHOLD=2.0)
            net = SAMRoad(cfg)
            net.load_state_dict(torch.load("ckpt.pt")["state_dict"], strict=True)
            net.eval().to(dev)
            _, _, kp, road = inferencer.infer_one_img(net, _scene(0, a.size), cfg, device=dev)
            cfg.update(ITSC_THRESHOLD=float(np.quantile(kp, 0.996)) / 255,
                       ROAD_THRESHOLD=float(np.quantile(road, 0.95)) / 255)
            del net
            torch.cuda.empty_cache()
            if rank == 0:
                import yaml
                with open("cityscale.yaml", "w") as f:
                    yaml.safe_dump(cfg, f)
            ranks.broadcast(None)
            commands = {
                "inferencer": (inferencer.main, ["--checkpoint", "ckpt.pt", "--config", "cityscale.yaml",
                                                 "--output_dir", "bench"]),
                "topo_metric": (topo_metric.main, ["--savedir", "save/metrics", "--dataset", "cityscale"]),
                "apls_metric": (apls_metric.main, ["--savedir", "save/metrics", "--dataset", "cityscale"]),
            }
            wall = {}
            for name, (fn, argv) in commands.items():
                ranks.broadcast(None)
                t0 = time.perf_counter()
                fn(argv)
                wall[name] = time.perf_counter() - t0
            if rank == 0:
                loop = open(os.path.join("save", "bench", "inference_time.txt")).read().split(" in ")[-1].split()[0]
                topo = json.load(open(os.path.join("save", "metrics", "score", "topo.json")))["mean topo"]
                apls = json.load(open(os.path.join("save", "metrics", "score", "apls.json")))["final_APLS"]
                print(json.dumps({"card": _card(), "world": world, "scenes": a.scenes, "size": a.size,
                                  "wall_s": wall, "inference_loop_s": float(loop),
                                  "per_scene_s": {k: v / a.scenes for k, v in wall.items()},
                                  "topo": topo, "apls": apls}))
            ranks.broadcast(None)
        finally:
            os.chdir(cwd)
            if rank == 0:
                shutil.rmtree(box, ignore_errors=True)


if __name__ == "__main__":
    main()
