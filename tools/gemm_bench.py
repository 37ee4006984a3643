"""Times the encoder GEMMs (`samroad_op_gemm_f16` / `samroad_op_gemm_f32`) with CUDA events at the shapes of
the c2 (ViT-B @512, 64 tiles) and c5 (ViT-H @256, 64 tiles) encoder blocks.

    python tools/gemm_bench.py [--lib-b PATH] [--rounds 5] [--iters 20] [--out FILE]

Per shape it reports ms per call (median over the rounds) and TFLOP/s of the algorithmic work 2*M*N*K.
With --lib-b a second build of the library (for example one of another commit) is loaded through ctypes
and timed on the same inputs, the two alternating round by round; whether the two outputs are
bit-identical is reported too.  The card name, power limit and max SM clock are read in the same run."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import _lib  # noqa: E402
from tools.attention_bench import card_info, load_lib  # noqa: E402

DEV = "cuda:0"
# (name, M, N, K, epilogue): "f16" = bias, "gelu" = bias + GELU, "resid" = in-place shortcut + bias,
# "pos" = bias + pos_embed (pos rows = tokens per image)
SHAPES = [
    ("c2_qkv", 65536, 2304, 768, "f16"),
    ("c2_proj", 65536, 768, 768, "resid"),
    ("c2_lin1", 65536, 3072, 768, "gelu"),
    ("c2_lin2", 65536, 768, 3072, "resid"),
    ("c2_patch_embed", 65536, 768, 768, "pos"),
    ("c5_qkv", 16384, 3840, 1280, "f16"),
    ("c5_proj", 16384, 1280, 1280, "resid"),
    ("c5_lin1", 16384, 5120, 1280, "gelu"),
    ("c5_lin2", 16384, 1280, 5120, "resid"),
    ("c5_patch_embed", 16384, 1280, 768, "pos"),
]
POS_ROWS = {65536: 1024, 16384: 256}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-b", default=None, help="a second libsamroad_b200.so to time against this tree's")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="calls per timed window")
    ap.add_argument("--out", default=None, help="write the results as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_bench needs a CUDA device"

    libs = {"a": _lib.load()}
    if args.lib_b:
        libs["b"] = load_lib(args.lib_b)
    st = torch.cuda.current_stream().cuda_stream
    result = {"card": card_info(), "lib_b": args.lib_b, "shapes": {}}
    for name, M, N, K, epi in SHAPES:
        g = torch.Generator().manual_seed(5)
        A = torch.randn(M, K, generator=g).to(torch.float16).to(DEV)
        W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.float16).to(DEV)
        bias = torch.randn(N, generator=g).to(DEV)
        x0 = torch.randn(M, N, generator=g).to(DEV) if epi == "resid" else None
        pos = torch.randn(POS_ROWS[M], N, generator=g).to(DEV) if epi == "pos" else None

        def call(lib, out):
            if epi in ("f16", "gelu"):
                rc = lib.samroad_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                             1 if epi == "gelu" else 0, out.data_ptr(), N, st)
            else:
                rc = lib.samroad_op_gemm_f32(A.data_ptr(), K, W.data_ptr(), K, M, N, K, bias.data_ptr(),
                                             out.data_ptr() if epi == "resid" else None,
                                             pos.data_ptr() if pos is not None else None,
                                             POS_ROWS[M] if pos is not None else 0, out.data_ptr(), N, st)
            if rc != 0:
                raise RuntimeError(f"gemm failed (code {rc}): {lib.samroad_last_error().decode()}")

        def fresh():
            if epi in ("f16", "gelu"):
                return torch.zeros(M, N, dtype=torch.float16, device=DEV)
            return x0.clone() if x0 is not None else torch.zeros(M, N, device=DEV)

        first = {}
        for key, lib in libs.items():       # one call on fresh buffers: the outputs compared below
            first[key] = fresh()
            call(lib, first[key])
        outs = {key: fresh() for key in libs}
        for key, lib in libs.items():
            for _ in range(3):
                call(lib, outs[key])
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
        flops = 2.0 * M * N * K
        row = {"M": M, "N": N, "K": K, "epilogue": epi}
        for key in libs:
            ms = sorted(times[key])[len(times[key]) // 2]
            row[f"ms_{key}"] = round(ms, 4)
            row[f"ms_{key}_rounds"] = [round(t, 4) for t in times[key]]
            row[f"tflops_{key}"] = round(flops / (ms * 1e-3) / 1e12, 1)
        if "b" in libs:
            row["bit_identical_a_b"] = bool(torch.equal(first["a"], first["b"]))
            row["maxabs_a_vs_b"] = float((first["a"].float() - first["b"].float()).abs().max())
            row["speedup_a_over_b"] = round(row["ms_b"] / row["ms_a"], 3)
        result["shapes"][name] = row
        print(name, json.dumps(row), flush=True)
        del A, W, x0, pos, outs, first
        torch.cuda.empty_cache()
    print(json.dumps(result["card"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
