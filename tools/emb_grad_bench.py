"""Time the gradient of the heads' losses with respect to the image embeddings at the benched training shape:
ViT-B, B=16 @512, Ns=512, Np=16, training mode (dropout 0.1).

Times, as min / median / max over --rounds of CUDA events:
  forward            samroad_train_forward_embeddings (the heads from the given embeddings and both losses)
  backward_weights   samroad_train_backward_embeddings with the weight gradients only (training_step's backward)
  backward_both      ... with the weight gradients and the embeddings gradient
  backward_emb_only  ... with the embeddings gradient only (frozen heads)
  torch_*            torch autograd on the fp32 oracle heads (oracle/train_oracle.py), forward and backward with
                     respect to the embeddings and the head parameters
and prints one JSON line with the card name, its power limit and its SM clock.

    python tools/emb_grad_bench.py [--rounds 20]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import train_oracle as TO  # noqa: E402
from sam_road_b200 import SAMRoad, _lib, synth  # noqa: E402
from sam_road_b200 import train as T  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        lines = q.stdout.strip().splitlines()
        return lines[0] if lines else "unknown"
    except Exception as e:      # the card name is part of the number; report why it is missing
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    B, P, N, Ns, Np = 16, 512, 512, 512, 16
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=P, FREEZE_ENCODER=False, TOPONET_VERSION="normal")
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=4.0))
    net = net.to(dev).train()
    pts, pairs, valid = synth.make_topo_inputs(B, P, N, seed=1, max_nbr=Np)
    g = torch.Generator().manual_seed(0)
    batch = {"rgb": synth.make_tiles(B, P, seed=2), "graph_points": pts, "pairs": pairs[:, :Ns],
             "valid": valid[:, :Ns], "connected": torch.rand(valid[:, :Ns].shape, generator=g) < 0.3,
             "keypoint_mask": (torch.rand((B, P, P), generator=g) < 0.1).float(),
             "road_mask": (torch.rand((B, P, P), generator=g) < 0.2).float()}
    batch = {k: v.to(dev) for k, v in batch.items()}
    s = P // 16
    emb = torch.randn((B, 256, s, s), generator=torch.Generator(device=dev).manual_seed(3), device=dev) * 0.5

    lib = _lib.load()
    h = net._handle(dev)
    heads = net._head_params()
    keys = [k for k, _ in heads]
    params = [p.detach() for _, p in heads]
    b = T.validate_batch(batch, P, dev)
    args = T.make_args(b, False, 0.1, 1234)
    nbytes = C.c_size_t()
    _lib.check(lib.samroad_train_workspace_bytes(h, C.byref(args), C.byref(nbytes)), "workspace")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    losses = torch.empty(2, dtype=torch.float32, device=dev)
    grads = [torch.empty_like(p) for p in params]
    gemb = torch.empty_like(emb)
    gin = torch.ones(2, dtype=torch.float32, device=dev)
    karr = (C.c_char_p * len(keys))(*[k.encode() for k in keys])
    parr = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
    garr = (C.c_void_p * len(grads))(*[x.data_ptr() for x in grads])
    (p_, pdt), (q_, qdt) = b["points"], b["pairs"]
    st = _lib.current_stream_ptr()

    def forward():
        _lib.check(lib.samroad_train_forward_embeddings(
            h, C.byref(args), karr, parr, len(params), emb.data_ptr(), p_.data_ptr(), pdt, q_.data_ptr(), qdt,
            b["valid"].data_ptr(), b["connected"].data_ptr(), b["kp"].data_ptr(), b["road"].data_ptr(),
            ws.data_ptr(), nbytes.value, losses.data_ptr(), st), "forward")

    def backward(weights, embeddings):
        _lib.check(lib.samroad_train_backward_embeddings(
            h, C.byref(args), karr, parr, garr if weights else None, len(params), ws.data_ptr(), nbytes.value,
            gin.data_ptr(), gemb.data_ptr() if embeddings else None, st), "backward")

    tp = {k: p.clone().requires_grad_(True) for k, p in zip(keys, params)}
    te = emb.clone().requires_grad_(True)
    keep = {}
    rows, tok = B * Ns, B * Ns * Np
    for l in range(3):
        keep[(l, 0)] = T.dropout_keep(0.1, 1234, l, 0, rows * 4 * Np * Np, dev).view(rows, 4, Np, Np)
        for site in (1, 2, 3):
            keep[(l, site)] = T.dropout_keep(0.1, 1234, l, site, tok * 128, dev).view(rows, Np, 128)
    holder = {}

    def torch_forward():
        holder["loss"] = sum(TO.heads_losses(tp, te, batch, P, False, "normal", keep, 0.1))

    def torch_backward():
        torch.autograd.grad(holder.pop("loss"), [te] + list(tp.values()))

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        ev[0].record()
        fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    runs = {k: [] for k in ("forward", "backward_weights", "backward_both", "backward_emb_only", "torch_forward",
                            "torch_backward")}
    for r in range(a.rounds + 2):          # two untimed rounds first
        t = {"forward": timed(forward),
             "backward_weights": timed(lambda: backward(True, False)),
             "backward_both": timed(lambda: backward(True, True)),
             "backward_emb_only": timed(lambda: backward(False, True)),
             "torch_forward": timed(torch_forward),
             "torch_backward": timed(torch_backward)}
        if r >= 2:
            for k, v in t.items():
                runs[k].append(v)
    summary = {k: {"min": min(v), "median": statistics.median(v), "max": max(v)} for k, v in runs.items()}
    print(json.dumps({"card": _card(), "B": B, "patch": P, "N": N, "Ns": Ns, "Np": Np, "dropout": 0.1,
                      "rounds": a.rounds, "workspace_GB": nbytes.value / 1e9, "ms": summary}))


if __name__ == "__main__":
    main()
