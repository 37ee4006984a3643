"""TOPO metric on one synthetic 2048 x 2048 city tile: device time of the per-pair work and of the whole tile, and,
where the reference checkout exists, the reference's CPU time for the same tile through tools/make_golden.py's
shims.  Prints one JSON line with the card name and power limit.

    python tools/topo_bench.py [--reps 3] [--reference]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sam_road_b200 import topo_metric as TM  # noqa: E402
from sam_road_b200.synth import city_tile  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reference", action="store_true", help="also time the reference (needs its checkout)")
    a = ap.parse_args()
    gt, prop = city_tile()
    res = dict(tile="2048x2048 synthetic city", gt_nodes=len(gt), prop_nodes=len(prop))
    if not a.reference:
        import torch
        dev = TM.TopoDevice(0)
        inner = []

        def timed(gtg, propg):
            score = TM.device_scorer(dev, gtg, propg)

            def f(pn, pd, r, step, thr):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = score(pn, pd, r, step, thr)
                inner.append(time.perf_counter() - t0)
                return out
            return f

        walls = []
        for _ in range(a.reps + 1):
            t0 = time.perf_counter()
            p, r, d = TM.topo_tile(gt, prop, TM.TopoState(), "cityscale", scorer=timed)
            walls.append(time.perf_counter() - t0)
        dev.close()
        res.update(gpu=gpu_info(), pairs=int(d.counts.shape[0]), r=d.r, precision=p, recall=r,
                   max_marbles=int(d.counts[:, :3].max()) if d.counts.size else 0,
                   device_pairs_s=sorted(inner[1:]), tile_total_s=sorted(walls[1:]))
    else:
        from tools import make_golden as MG
        with tempfile.TemporaryDirectory() as wd:
            t0 = time.perf_counter()
            rec = MG._reference_topo_run([(gt, prop)], "cityscale", wd)[0]
            res.update(reference_cpu_s=time.perf_counter() - t0, pairs=len(rec["lmap"]),
                       last_line=rec["text"].splitlines()[-1])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
