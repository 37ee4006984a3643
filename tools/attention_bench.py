"""Times the encoder attention op (`samroad_op_attention`) with CUDA events at the shapes the benchmark
workloads run, and checks it against the fp32 SIMT kernel of the same library.

    python tools/attention_bench.py [--lib-b PATH] [--rounds 5] [--iters 20] [--out FILE]

Per shape it reports ms per call, algorithmic TFLOP/s (real queries x real keys, the count model.cu
gives the timing hook), the executed / needed score ratio of this tree's tensor-core kernel, and the
max-abs difference against the SIMT kernel.  With --lib-b a second build of the library (for example
one of another commit) is loaded through ctypes and timed on the same inputs, the two alternating
round by round; the max-abs difference between the two outputs is reported too.  The card name,
power limit and max SM clock are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import _lib  # noqa: E402

DEV = "cuda:0"
# (name, B, s, win, heads, hd): c2/c4 ViT-B @512 (s 32), c1/c3 ViT-B @256 (s 16), c5 ViT-H @256,
# and a 1024 tile's global unit (s 64)
SHAPES = [
    ("vitb_s32_win14", 64, 32, 14, 12, 64),
    ("vitb_s32_global", 64, 32, 32, 12, 64),
    ("vitb_s16_win14", 64, 16, 14, 12, 64),
    ("vitb_s16_global", 64, 16, 16, 12, 64),
    ("vith_s16_win14", 64, 16, 14, 16, 80),
    ("vith_s16_global", 64, 16, 16, 16, 80),
    ("vitb_s64_global", 8, 64, 64, 12, 64),
]


def windows(s, win):
    nw = (s + win - 1) // win
    for wy in range(nw):
        for wx in range(nw):
            yield min(win, s - wy * win), min(win, s - wx * win)


def att_flops(B, s, win, heads, hd):
    return 4.0 * hd * B * heads * sum((ry * rx) ** 2 for ry, rx in windows(s, win))


def score_ratio(s, win):
    """Executed / needed scores of attention_mma.cuh: 16-row tiles of the real queries against
    whole 64-slot chunks of win x winP key slots (an upper half with no key skipped)."""
    winp = 8
    while winp < win:
        winp *= 2
    slots = win * winp
    executed_keys = (slots // 64) * 64 + (0 if slots % 64 == 0 else (32 if slots % 64 <= 32 else 64))
    executed = needed = 0
    for ry, rx in windows(s, win):
        executed += math.ceil(ry * rx / 16) * 16 * executed_keys
        needed += ry * rx * win * win
    return executed / needed


def load_lib(path):
    lib = C.CDLL(path)
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-b", default=None, help="a second libsamroad_b200.so to time against this tree's")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="calls per timed window")
    ap.add_argument("--out", default=None, help="write the results as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "attention_bench needs a CUDA device"

    libs = {"a": _lib.load()}
    if args.lib_b:
        libs["b"] = load_lib(args.lib_b)
    st = torch.cuda.current_stream().cuda_stream
    result = {"card": card_info(), "lib_b": args.lib_b, "shapes": {}}
    for name, B, s, win, heads, hd in SHAPES:
        D = heads * hd
        g = torch.Generator().manual_seed(11)
        qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
        bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
        rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
        rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)

        def call(lib, out):
            rc = lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                          B, s, win, heads, hd, out.data_ptr(), st)
            if rc != 0:
                raise RuntimeError(f"attention failed (code {rc}): {lib.samroad_last_error().decode()}")

        outs = {}
        for key, lib in libs.items():
            outs[key] = torch.zeros(B * s * s, D, dtype=torch.float16, device=DEV)
            for _ in range(3):
                call(lib, outs[key])
        simt = torch.zeros_like(outs["a"])
        libs["a"].samroad_debug_force_simt_attention(1)
        try:
            call(libs["a"], simt)
        finally:
            libs["a"].samroad_debug_force_simt_attention(0)
        torch.cuda.synchronize()

        times = {k: [] for k in libs}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for key, lib in libs.items():
                ev0.record()
                for _ in range(args.iters):
                    call(lib, outs[key])
                ev1.record()
                torch.cuda.synchronize()
                times[key].append(ev0.elapsed_time(ev1) / args.iters)
        flops = att_flops(B, s, win, heads, hd)
        row = {"B": B, "s": s, "win": win, "heads": heads, "hd": hd, "score_ratio_a": round(score_ratio(s, win), 3),
               "maxabs_a_vs_simt": float((outs["a"].float() - simt.float()).abs().max())}
        for key in libs:
            ms = sorted(times[key])[len(times[key]) // 2]
            row[f"ms_{key}"] = round(ms, 4)
            row[f"ms_{key}_rounds"] = [round(t, 4) for t in times[key]]
            row[f"tflops_{key}"] = round(flops / (ms * 1e-3) / 1e12, 2)
        if "b" in libs:
            row["maxabs_a_vs_b"] = float((outs["a"].float() - outs["b"].float()).abs().max())
            row["speedup_b_over_a"] = round(row["ms_b"] / row["ms_a"], 3)
        result["shapes"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result["card"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
