"""Per-tile phase trace of the ping-pong GEMM (`gemm_pp_kernel`) at the c2 and c5 encoder shapes.

    python tools/gemm_trace.py [--lib PATH] [--no-store] [--shapes c2_qkv,c2_lin1] [--out FILE]

The trace is compiled in only with -DSRB_GEMM_TRACE.  Without --lib, this tool compiles gemm_ops.cu with it into a
temporary directory and links it with the other objects of this tree's build (`python -m sam_road_b200.build`
first).  Each GEMM runs a few times untraced, then once with every CTA stamping `clock64` at the phases of each of
its tiles (see the TR_* events in gemm_tc.cuh).  Per shape it prints the medians, in SM clocks, over all traced
tiles:

  mainloop      first full_bar wait passed -> last k-block's MMAs issued (ideal: num_k * 512 clocks, the
                tensor-core time of 8 wgmma m64n128k16 per k-block at 4096 FLOP per clock)
  first_full    order_bar passed -> first full_bar wait passed (the tile's first stage not yet loaded)
  drain         last MMAs issued -> wgmma_wait<0> returned
  epilogue      wgmma_wait<0> returned -> last store of the epilogue issued, in three parts:
    epi_loads   wgmma_wait<0> returned -> the epilogue's first operands (bias, residual) in registers
    epi_math    -> the tile's last values computed and packed (staged in shared memory, where it is)
    epi_stores  -> last store issued
  order_wait    epilogue done -> the other consumer has issued its mainloop (this consumer idles)
  tensor_idle   max(0, first MMA of tile i - tile i-1's MMAs complete): tensor cores idle at the handoff
  producer_stall  clocks the producer waited on empty_bar for the tile's k-blocks
  period        between the last MMA issues of consecutive tiles of a CTA (the CTA's time per tile)

With --no-store the library is built with -DSRB_GEMM_TRACE_NOSTORE as well: the epilogues compute everything but
issue no global stores (the output is not written), which gives the length of their loads and math alone.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import build as B  # noqa: E402
from tools.attention_bench import card_info, load_lib  # noqa: E402
from tools.gemm_bench import POS_ROWS, SHAPES  # noqa: E402

DEV = "cuda:0"
EVENTS = 10                    # kGemmTraceEvents
ORDER_WAIT, ORDER_DONE, FIRST_FULL, LAST_ISSUE, DRAINED, EPI_DONE, EMPTY_WAIT, EPI_LOADED, EPI_STAGED = range(9)
MAX_TILES = 128                # local tiles traced per CTA


def build_traced(out_dir, no_store=False):
    """gemm_ops.cu with -DSRB_GEMM_TRACE, linked with the tree's other objects, as out_dir/libsamroad_b200_trace.so."""
    B.build()
    nvcc = B._nvcc()
    obj = os.path.join(out_dir, "gemm_ops_trace.o")
    lib = os.path.join(out_dir, "libsamroad_b200_trace.so")
    defs = ["-DSRB_GEMM_TRACE"] + (["-DSRB_GEMM_TRACE_NOSTORE"] if no_store else [])
    subprocess.run([nvcc, *B.NVCC_FLAGS, *defs, "-c", str(B.CSRC / "gemm_ops.cu"), "-o", obj], check=True)
    objs = [obj if s == "gemm_ops.cu" else str(B.OBJ_DIR / (s + ".o")) for s in B.SOURCES]
    subprocess.run([nvcc, "-shared", "-o", lib, *objs, "-lcudart"], check=True)
    return lib


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if xs else float("nan")


def phases(tr, num_k):
    """Medians of the phase durations over tr [ctas, tiles, EVENTS] (int64 clocks, zero = not reached)."""
    q = {k: [] for k in ("mainloop", "first_full", "drain", "epilogue", "epi_loads", "epi_math", "epi_stores",
                         "order_wait", "tensor_idle", "producer_stall", "period")}
    for cta in tr.tolist():
        n = sum(1 for t in cta if t[EPI_DONE] != 0)
        for i in range(n):
            t = cta[i]
            q["mainloop"].append(t[LAST_ISSUE] - t[FIRST_FULL])
            q["first_full"].append(t[FIRST_FULL] - t[ORDER_DONE])
            q["drain"].append(t[DRAINED] - t[LAST_ISSUE])
            q["epilogue"].append(t[EPI_DONE] - t[DRAINED])
            q["epi_loads"].append(t[EPI_LOADED] - t[DRAINED])
            q["epi_math"].append(t[EPI_STAGED] - t[EPI_LOADED])
            q["epi_stores"].append(t[EPI_DONE] - t[EPI_STAGED])
            q["producer_stall"].append(t[EMPTY_WAIT])
            if i >= 1:
                p = cta[i - 1]
                q["tensor_idle"].append(max(0, t[FIRST_FULL] - p[DRAINED]))
                q["period"].append(t[LAST_ISSUE] - p[LAST_ISSUE])
            if i >= 2:
                q["order_wait"].append(t[ORDER_DONE] - t[ORDER_WAIT])
    row = {k: median(v) for k, v in q.items()}
    row["ideal_mainloop"] = num_k * 8 * 64
    row["tiles_traced"] = len(q["mainloop"])
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a library built with -DSRB_GEMM_TRACE (default: build one)")
    ap.add_argument("--no-store", action="store_true", help="build without the epilogues' global stores")
    ap.add_argument("--shapes", default="c2_qkv,c2_proj,c2_lin1,c2_lin2,c2_patch_embed,c5_qkv,c5_lin1")
    ap.add_argument("--out", default=None, help="write the results as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_trace needs a CUDA device"

    with tempfile.TemporaryDirectory() as tmp:
        path = args.lib or build_traced(tmp, args.no_store)
        lib = load_lib(path)
        lib.samroad_debug_gemm_trace.restype = C.c_int
        lib.samroad_debug_gemm_trace.argtypes = [C.c_void_p, C.c_int, C.c_int]
        st = torch.cuda.current_stream().cuda_stream
        ctas = torch.cuda.get_device_properties(0).multi_processor_count
        buf = torch.zeros(ctas, MAX_TILES, EVENTS, dtype=torch.int64, device=DEV)
        result = {"card": card_info(), "lib": args.lib, "no_store": args.no_store, "unit": "SM clocks", "shapes": {}}
        wanted = args.shapes.split(",")
        for name, M, N, K, epi in SHAPES:
            if name not in wanted:
                continue
            g = torch.Generator().manual_seed(5)
            A = torch.randn(M, K, generator=g).to(torch.float16).to(DEV)
            W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.float16).to(DEV)
            bias = torch.randn(N, generator=g).to(DEV)
            pos = torch.randn(POS_ROWS[M], N, generator=g).to(DEV) if epi == "pos" else None
            out = (torch.zeros(M, N, dtype=torch.float16, device=DEV) if epi in ("f16", "gelu")
                   else torch.randn(M, N, generator=g).to(DEV))

            def call():
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

            for _ in range(5):
                call()
            buf.zero_()
            torch.cuda.synchronize()
            assert lib.samroad_debug_gemm_trace(buf.data_ptr(), ctas, MAX_TILES) == 0
            call()
            torch.cuda.synchronize()
            assert lib.samroad_debug_gemm_trace(None, 0, 0) == 0
            row = {"M": M, "N": N, "K": K, "epilogue": epi, **phases(buf.cpu(), (K + 63) // 64)}
            result["shapes"][name] = row
            print(name, json.dumps(row), flush=True)
            del A, W, bias, pos, out
            torch.cuda.empty_cache()
    print(json.dumps(result["card"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
