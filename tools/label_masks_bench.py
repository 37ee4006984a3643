"""Time of the label masks of a whole dataset (sam_road_b200.label_masks, csrc/label_masks.cu) next to the loop the
reference's generate_labels.py scripts run (networkx graph + cv2.circle / cv2.line per tile).

Workloads: 180 CityScale-like 2048^2 tiles (synth.city_tile graphs: streets every 128 px, nodes every 16 px,
diagonals) and 2,500 SpaceNet-like 400^2 tiles (synth.make_road_graph), the tile counts of the two datasets.
Reported per workload: the host parse (tile_arrays), the device time in CUDA events of one draw_masks call with the
upload of the arrays included, the cv2 + networkx loop (skipped with a note when either module is absent), and
the PNG writing of the command (cv2.imwrite of both masks of every tile into a temporary directory).  The card's
name and power limit are read in the same run.

    python tools/label_masks_bench.py [--steps 5] [--warmup 2] [--out path.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sam_road_b200 import label_masks as L  # noqa: E402
from sam_road_b200 import synth  # noqa: E402
from tools.label_bench import card  # noqa: E402


def workloads():
    city = [synth.city_tile(2048, seed=s)[s % 2] for s in range(6)]
    space = [synth.make_road_graph(400 - 16 * (s % 3), seed=s, spacing=40 + 4 * (s % 4)) for s in range(50)]
    return {"cityscale": [city[t % len(city)] for t in range(180)],
            "spacenet": [space[t % len(space)] for t in range(2500)]}


def reference_loop(adjs, dataset):
    """What generate_labels.py does per tile, minus the file I/O."""
    import cv2
    import networkx as nx
    size = L.IMAGE_SIZE[dataset]
    for adj in adjs:
        g = nx.Graph()
        for n, neis in adj.items():
            for nei in neis:
                if dataset == "cityscale":
                    g.add_edge((int(n[1]), int(n[0])), (int(nei[1]), int(nei[0])))
                else:
                    g.add_edge((int(n[1]), size - int(n[0])), (int(nei[1]), size - int(nei[0])))
        kp = np.zeros((size, size), np.uint8)
        for node, degree in g.degree():
            if degree != 2:
                cv2.circle(kp, node, 3, 255, -1)
        road = np.zeros((size, size), np.uint8)
        for (p, q) in g.edges():
            cv2.line(road, p, q, 255, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power = card()
    res = {"gpu": name, "power_limit": power}
    for dataset, adjs in workloads().items():
        t0 = time.perf_counter()
        arrays = [L.tile_arrays(a, dataset) for a in adjs]
        parse_s = time.perf_counter() - t0
        kps, edges = [a[0] for a in arrays], [a[1] for a in arrays]
        size = L.IMAGE_SIZE[dataset]
        for _ in range(args.warmup):
            L.draw_masks(kps, edges, size, dev)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.steps):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            kp, road = L.draw_masks(kps, edges, size, dev)
            stop.record()
            torch.cuda.synchronize()
            times.append(start.elapsed_time(stop))
            del kp, road
        kp, road = L.draw_masks(kps, edges, size, dev)
        kp, road = kp.cpu().numpy(), road.cpu().numpy()
        r = {"tiles": len(adjs), "edges": int(sum(len(e) for e in edges)), "keypoints": int(sum(len(k) for k in kps)),
             "parse_ms": 1e3 * parse_s, "device_ms_median": float(np.median(times)),
             "device_ms_min": float(np.min(times)), "output_bytes": int(kp.nbytes + road.nbytes)}
        try:
            import cv2  # noqa: F401
            import networkx  # noqa: F401
            t0 = time.perf_counter()
            reference_loop(adjs, dataset)
            r["cv2_networkx_ms"] = 1e3 * (time.perf_counter() - t0)
        except ImportError as e:
            r["cv2_networkx_ms"] = None
            r["note"] = f"reference loop skipped: {e}"
        try:
            import cv2
            with tempfile.TemporaryDirectory() as tmp:
                t0 = time.perf_counter()
                for t in range(len(adjs)):
                    cv2.imwrite(os.path.join(tmp, f"keypoint_mask_{t}.png"), kp[t])
                    cv2.imwrite(os.path.join(tmp, f"road_mask_{t}.png"), road[t])
                r["png_write_ms"] = 1e3 * (time.perf_counter() - t0)
        except ImportError:
            r["png_write_ms"] = None
        res[dataset] = r
        print(f"{dataset}: {json.dumps(r)}", flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
