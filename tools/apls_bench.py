"""APLS on one synthetic 2048² city tile (synth.city_tile), both directions: the device calls (candidates, shortest
paths and pair score, each a synchronous call into csrc/apls_metric.cu), the host stages around them, and the
oracle's time for the same tile, after a warm-up run.

    python tools/apls_bench.py [--reps 5] [--out DIR] [--heapq-oracle]

The oracle runs with scipy's Dijkstra and a vectorised nearest-node search (oracle.apls_oracle.scipy_scorer);
`--heapq-oracle` times its pure-Python heapq Dijkstra instead (minutes per tile).  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import apls_oracle as O  # noqa: E402
from sam_road_b200 import apls_metric as AM  # noqa: E402
from sam_road_b200 import synth  # noqa: E402


class Timed(AM.AplsDevice):
    """An AplsDevice that adds the wall time of every synchronous library call to `self.t`."""

    t = 0.0

    def _timed(self, f, *a, **k):
        t0 = time.perf_counter()
        try:
            return f(*a, **k)
        finally:
            self.t += time.perf_counter() - t0

    def upload_csr(self, *a, **k):
        return self._timed(super().upload_csr, *a, **k)

    def candidates(self, *a, **k):
        return self._timed(super().candidates, *a, **k)

    def one_way(self, *a, **k):
        return self._timed(super().one_way, *a, **k)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--heapq-oracle", action="store_true")
    a = ap.parse_args()
    gt, prop = synth.city_tile()
    dev = Timed(0)
    try:
        AM.apls_tile(gt, prop, "cityscale", device=dev)            # warm-up: module load, buffer growth
        dev_t, tot_t, res = [], [], None
        for _ in range(a.reps):
            dev.t = 0.0
            t0 = time.perf_counter()
            res = AM.apls_tile(gt, prop, "cityscale", device=dev)
            tot_t.append(time.perf_counter() - t0)
            dev_t.append(dev.t)
    finally:
        dev.close()
    d = res[3]
    t0 = time.perf_counter()
    o = AM.apls_tile(gt, prop, "cityscale", scorer=O.scorer if a.heapq_oracle else O.scipy_scorer)
    oracle_t = time.perf_counter() - t0
    assert o[3].line == d.line, (o[3].line, d.line)
    out = dict(gpu=gpu_info(), tile="synth.city_tile()", line=d.line.strip(),
               gt_nodes=len(d.gt.nodes), prop_nodes=len(d.prop.nodes),
               control_points=[len(d.gt_way.control_points), len(d.prop_way.control_points)],
               scored_pairs=[d.gt_way.result["scored"], d.prop_way.result["scored"]],
               terminals=[list(d.gt_way.result["terminals"]), list(d.prop_way.result["terminals"])],
               device_call_s=[round(x, 4) for x in dev_t], tile_s=[round(x, 4) for x in tot_t],
               host_s=[round(t - x, 4) for t, x in zip(tot_t, dev_t)],
               oracle="heapq" if a.heapq_oracle else "scipy", oracle_s=round(oracle_t, 3))
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "apls_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
