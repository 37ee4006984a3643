"""One FREEZE_ENCODER training step at the reference's training shape, split by phase, next to the same heads in
torch autograd (the fp32 oracle, oracle/train_oracle.py, in fp32 and under autocast fp16) fed by the engine's
embeddings, alternating round by round.

Workload: ViT-B, B = 16 tiles of 512^2, Ns = 512 samples x Np = 16 pairs per tile, BCE, dropout on (train mode).
Phases (CUDA events, each ends in a synchronise): encoder (samroad_encode_masks, embeddings only), heads forward
(training forward minus the encoder), backward, Adam step, refresh of the packed weights.  Prints one JSON object
with the card name and power limit.

    python tools/train_bench.py [--rounds 3] [--batch 16]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import train_oracle as TO  # noqa: E402
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    B, P, Ns, Np = a.batch, 512, 512, 16
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=P, FREEZE_ENCODER=True, BASE_LR=1e-4, TOPONET_VERSION="normal")
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=4.0))
    net = net.to(dev).train()
    pts, pairs, valid = synth.make_topo_inputs(B, P, Ns, seed=1, max_nbr=Np)
    g = torch.Generator().manual_seed(0)
    batch = {"rgb": synth.make_tiles(B, P, seed=2), "graph_points": pts, "pairs": pairs, "valid": valid,
             "connected": torch.rand(valid.shape, generator=g) < 0.3,
             "keypoint_mask": (torch.rand((B, P, P), generator=g) < 0.1).float(),
             "road_mask": (torch.rand((B, P, P), generator=g) < 0.2).float()}
    batch = {k: v.to(dev) for k, v in batch.items()}
    opt = net.configure_optimizers()["optimizer"]
    lib = _lib.load()
    s = P // 16
    emb = torch.empty((B, 256, s, s), device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]

    def engine_step():
        ev[0].record()
        h = net._handle(dev)
        _lib.check(lib.samroad_encode_masks(h, batch["rgb"].data_ptr(), _lib.U8, B, None, None, emb.data_ptr(),
                                            _lib.current_stream_ptr()), "samroad_encode_masks")
        ev[1].record()
        loss = net.training_step(batch, 0)
        ev[2].record()
        loss.backward()
        ev[3].record()
        opt.step()
        opt.zero_grad()
        ev[4].record()
        net._handle(dev)           # refresh of the packed head weights
        ev[5].record()
        ev[5].synchronize()
        t = [ev[i].elapsed_time(ev[i + 1]) for i in range(5)]
        # training_step runs the encoder again: its forward minus the encoder is the heads' forward
        return {"encoder": t[0], "heads_forward": t[1] - t[0], "backward": t[2], "optimizer": t[3],
                "refresh": t[4], "step_with_encoder_once": t[1] + t[2] + t[3] + t[4]}

    params = {k: p.detach().clone().requires_grad_(True) for k, p in net._head_params()}
    topt = torch.optim.Adam(list(params.values()), lr=1e-4)

    def torch_step(autocast):
        ev[0].record()
        with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
            ml, tl = TO.heads_losses(params, emb, batch, P, False, "normal", None, 0.1)
            loss = ml + tl
        ev[1].record()
        loss.backward()
        ev[2].record()
        topt.step()
        topt.zero_grad()
        ev[3].record()
        ev[3].synchronize()
        return {"heads_forward": ev[0].elapsed_time(ev[1]), "backward": ev[1].elapsed_time(ev[2]),
                "optimizer": ev[2].elapsed_time(ev[3])}

    engine_step()
    torch_step(False)
    torch_step(True)
    rounds = {"engine": [], "torch_fp32": [], "torch_autocast_fp16": []}
    for _ in range(a.rounds):
        rounds["engine"].append(engine_step())
        rounds["torch_fp32"].append(torch_step(False))
        rounds["torch_autocast_fp16"].append(torch_step(True))
    summary = {name: {k: [min(r[k] for r in rs), max(r[k] for r in rs)] for k in rs[0]} for name, rs in rounds.items()}
    import ctypes as C
    from sam_road_b200 import train as T
    targs = T.make_args(T.validate_batch(batch, P, dev), False, 0.1, 0)
    nbytes = C.c_size_t()
    _lib.check(lib.samroad_train_workspace_bytes(net._handle(dev), C.byref(targs), C.byref(nbytes)), "workspace")
    print(json.dumps({"card": _card(), "B": B, "patch": P, "Ns": Ns, "Np": Np, "rounds": a.rounds,
                      "workspace_GB": nbytes.value / 1e9, "ms_min_max": summary,
                      "peak_memory_GB": torch.cuda.max_memory_allocated(dev) / 1e9}))


if __name__ == "__main__":
    main()
