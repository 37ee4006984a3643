"""TopoNet time per call at n_pairs 16 (fused kernel), 31 (layered path) and 32 (fused kernel) on the C2
TopoNet shape (B = 64 tiles of 512 px, 256 keypoints per tile, Ns = N), and infer_one_img on a 2048^2
scene at MAX_NEIGHBOR_QUERIES 16 and 32.  CUDA events around the calls, after warm-up; the n_pairs
are interleaved round by round so that clock drift hits all of them alike.  Prints one JSON object.

    python tools/toponet_npairs_bench.py [--rounds 7] [--calls 20] [--no-scene]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import SAMRoad, synth  # noqa: E402
from sam_road_b200.inferencer import infer_one_img  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--scene-runs", type=int, default=3)
    ap.add_argument("--no-scene", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=512, USE_SAM_DECODER=False, ENCODER_LORA=False, LORA_RANK=0,
               TOPONET_VERSION="normal", NO_SAM=False, INFER_BATCH_SIZE=64, SAMPLE_MARGIN=64,
               INFER_PATCHES_PER_EDGE=16, TOPO_THRESHOLD=0.5, ITSC_NMS_RADIUS=8, ROAD_NMS_RADIUS=16,
               NEIGHBOR_RADIUS=64, MAX_NEIGHBOR_QUERIES=16, ITSC_THRESHOLD=2.0, ROAD_THRESHOLD=2.0)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=6.0), strict=True)
    net.eval().to(dev)
    B, N = 64, 256
    feat = torch.randn(B, 256, 32, 32, generator=torch.Generator().manual_seed(0)).to(dev)
    inputs = {}
    for npairs in (16, 31, 32):
        pts, prs, val = synth.make_topo_inputs(B, 512, N, seed=npairs, max_nbr=npairs, ragged=False)
        inputs[npairs] = (pts.to(dev), prs.to(dev), val.to(dev), torch.empty(B * N * npairs, device=dev))
    res = {"card": _card(), "shape": {"B": B, "N": N, "Ns": N}, "toponet": {}}
    with torch.no_grad():
        for npairs, (pts, prs, val, out) in inputs.items():        # warm-up of every shape
            for _ in range(5):
                net.infer_toponet(feat, pts, prs, val, out=out)
        torch.cuda.synchronize()
        times = {k: [] for k in inputs}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for npairs, (pts, prs, val, out) in inputs.items():
                e0.record()
                for _ in range(a.calls):
                    net.infer_toponet(feat, pts, prs, val, out=out)
                e1.record()
                e1.synchronize()
                times[npairs].append(e0.elapsed_time(e1) / a.calls)
    for npairs, t in times.items():
        ms = float(np.median(t))
        res["toponet"][f"np{npairs}"] = {
            "path": "fused" if npairs in (16, 32) else "layered", "ms_per_call_median": ms,
            "ms_per_call_min": float(np.min(t)), "ms_per_call_max": float(np.max(t)),
            "ns_per_pair_token": ms * 1e6 / (B * N * npairs)}
    if not a.no_scene:
        img = np.random.RandomState(17).randint(0, 256, size=(2048, 2048, 3)).astype(np.uint8)
        _, _, kp, road = infer_one_img(net, img, cfg, device=dev)
        cfg.update(ITSC_THRESHOLD=float(np.quantile(kp, 0.996)) / 255,
                   ROAD_THRESHOLD=float(np.quantile(road, 0.95)) / 255)
        res["scene"] = {}
        runs = {16: [], 32: []}
        for K in runs:                                             # warm-up
            infer_one_img(net, img, dict(cfg, MAX_NEIGHBOR_QUERIES=K), device=dev)
        for _ in range(a.scene_runs):
            for K in runs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                nodes, edges, _, _ = infer_one_img(net, img, dict(cfg, MAX_NEIGHBOR_QUERIES=K), device=dev)
                torch.cuda.synchronize()
                runs[K].append((time.perf_counter() - t0) * 1e3)
        for K, t in runs.items():
            tm = {}
            nodes, edges, _, _ = infer_one_img(net, img, dict(cfg, MAX_NEIGHBOR_QUERIES=K), device=dev, timings=tm)
            res["scene"][f"K{K}"] = {"ms_median": float(np.median(t)), "ms_all": t, "n_points": int(nodes.shape[0]),
                                     "n_edges": int(edges.shape[0]),
                                     "toponet_ms": 1e3 * tm["toponet_s"], "pair_queries_ms": 1e3 * tm["pair_queries_s"],
                                     "edges_ms": 1e3 * tm["edges_s"], "topo_samples": tm["topo_samples"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
