"""Run-to-run determinism of the encoder + mask head at several batch sizes, by default, with every
LayerNorm walking its rows ascending, and with the SIMT attention kernel: which switch makes two
identical calls return identical bits tells which kernel family has a schedule-dependent result.
    python tools/determinism_probe.py [--patch 256]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patch", type=int, default=256)
    a = ap.parse_args()
    dev = "cuda:0"
    lib = _lib.load()
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=a.patch, USE_SAM_DECODER=False, ENCODER_LORA=False,
               TOPONET_VERSION="normal", NO_SAM=False)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=6.0), strict=True)
    net.eval().to(dev)
    out = {}
    for B in (4, 16, 32, 64):
        rgb = synth.make_tiles(B, a.patch, seed=3).to(dev)
        for tag, gemm_mode, att_mode in (("default", 0, 0), ("no_snake", 16, 0), ("simt_attention", 0, 1)):
            lib.samroad_debug_disable_2cta_gemm(gemm_mode)
            lib.samroad_debug_force_simt_attention(att_mode)
            runs = []
            for _ in range(4):
                s, f = net.infer_masks_and_img_features(rgb)
                runs.append((s.clone(), f.clone()))
            torch.cuda.synchronize()
            ndiff_f = [int((runs[0][1] != r[1]).sum().item()) for r in runs[1:]]
            ndiff_s = [int((runs[0][0] != r[0]).sum().item()) for r in runs[1:]]
            mx = max(float((runs[0][1] - r[1]).abs().max().item()) for r in runs[1:])
            out[f"B{B}:{tag}"] = {"feat_elems_differing": ndiff_f, "score_elems_differing": ndiff_s, "feat_maxabs": mx,
                                  "tiles_differing": sorted({int(i) for r in runs[1:] for i in
                                                             (runs[0][1] != r[1]).flatten(1).any(1).nonzero().flatten().tolist()})[:16]}
            print(f"B{B}:{tag}", out[f"B{B}:{tag}"], flush=True)
    lib.samroad_debug_disable_2cta_gemm(0)
    lib.samroad_debug_force_simt_attention(0)
    json.dump(out, open("gpurun_out/determinism_probe.json", "w"), indent=1)


if __name__ == "__main__":
    main()
