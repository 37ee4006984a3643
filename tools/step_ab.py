"""Whole-step A/B of two trees of this project in one run on one GPU: bench.py as a subprocess, alternately from a
copy of another commit (its library built beforehand) and from this tree.

    python tools/step_ab.py --parent parent_tree [--runs 3] [--workload c2] [--out DIR] [-- extra bench.py args]

Per run it prints `value` (tiles/s), `ms_per_step`, the attention and GEMM entries of `kernels` and `clocks`; at the end the
fastest and slowest run of each tree.  With --out the first run of each tree also dumps its outputs
(bench.py --dump-outputs) and the max-abs differences of mask_scores, img_features and topo_scores are printed.
The card name, power limit and max SM clock are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bench(tree, workload, extra):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--no-cpu-baseline", "--steps", "20", "--warmup", "3",
           "--workload", workload, *extra]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"bench.py failed in {tree}:\n{r.stderr[-2000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="directory holding the other tree, library built")
    ap.add_argument("--runs", type=int, default=3, help="runs per tree")
    ap.add_argument("--workload", default="c2")
    ap.add_argument("--out", default=None, help="directory for the output dumps and the JSON summary")
    ap.add_argument("extra", nargs="*", help="further bench.py arguments, after --")
    args = ap.parse_args()
    trees = {"parent": os.path.abspath(args.parent), "new": ROOT}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)

    rows = {k: [] for k in trees}
    for i in range(args.runs):
        for key, tree in trees.items():
            extra = list(args.extra)
            if args.out and i == 0:
                extra += ["--dump-outputs", os.path.join(os.path.abspath(args.out), f"dump_{args.workload}_{key}")]
            line = bench(tree, args.workload, extra)
            row = {"value": line["value"], "ms_per_step": line["ms_per_step"], "clocks": line["clocks"],
                   "attention": {k: round(v["ms_per_step"], 3) for k, v in line["kernels"].items() if "attention" in k},
                   "gemm": {k: round(v["ms_per_step"], 3) for k, v in line["kernels"].items() if k.startswith("gemm_")}}
            rows[key].append(row)
            print(args.workload, key, i, json.dumps(row), flush=True)
    summary = {"workload": args.workload, "card": q.stdout.strip(), "runs": rows}
    for key in trees:
        v = [r["value"] for r in rows[key]]
        summary[key] = {"min": min(v), "max": max(v)}
        print(f"{args.workload} {key}: {min(v):.1f} .. {max(v):.1f} tiles/s", flush=True)
    if args.out:
        import numpy as np
        diffs = {}
        for name in ("mask_scores", "img_features", "topo_scores"):
            a, b = (os.path.join(args.out, f"dump_{args.workload}_{k}", name + ".npy") for k in trees)
            if os.path.exists(a) and os.path.exists(b):
                diffs[name] = float(np.abs(np.load(a) - np.load(b)).max())
        summary["maxabs_parent_vs_new"] = diffs
        print("max-abs parent vs new:", json.dumps(diffs), flush=True)
        with open(os.path.join(args.out, f"step_ab_{args.workload}.json"), "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
