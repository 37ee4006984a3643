"""Throughput of the other BASELINE.json configurations (not bench.py lines; for the record):
C1/C3 tile shape (ViT-B @256), C4 (ViT-B @512, dense TopoNet: 1024 keypoints x 16 pairs per tile) and
C5 (ViT-H @256, encoder + mask head).  Device-resident inputs, CUDA events, seeded random weights.

    python tools/bench_configs.py [--steps 5] > other_configs.json
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sam_road_b200 import SAMRoad, synth  # noqa: E402


def cfg(patch, version="vit_b"):
    return dict(SAM_VERSION=version, PATCH_SIZE=patch, USE_SAM_DECODER=False, ENCODER_LORA=False,
                TOPONET_VERSION="normal", NO_SAM=False)


def run(name, c, B, n_points, steps, warmup=2):
    dev = torch.device("cuda:0")
    net = SAMRoad(c)
    net.load_state_dict(synth.make_state_dict(c, seed=0), strict=True)
    net.eval().to(dev)
    P = c["PATCH_SIZE"]
    rgb = synth.make_tiles(B, P, seed=3).to(dev)
    topo = None
    if n_points:
        topo = [t.to(dev) for t in synth.make_topo_inputs(B, P, n_points, seed=4, ragged=False)]

    def step():
        scores, feat = net.infer_masks_and_img_features(rgb)
        if topo:
            net.infer_toponet(feat, *topo)

    for _ in range(warmup):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"config": name, "tiles_per_step": B, "patch": P, "points_per_tile": n_points,
            "ms_per_step": ms, "tiles_per_s": B / ms * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    out = [run("vitb_256 (C1/C3 tile shape) + TopoNet 64 keypoints", cfg(256), 256, 64, a.steps),
           run("vitb_512 dense TopoNet (C4: 1024 keypoints x 16 pairs)", cfg(512), 64, 1024, a.steps),
           run("vith_256 encoder + mask head (C5; head_dim 80 tensor-core attention)",
               cfg(256, "vit_h"), 64, 0, a.steps)]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
