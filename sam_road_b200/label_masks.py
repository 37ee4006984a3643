"""The label masks of the datasets on the device: cityscale/generate_labels.py and spacenet/generate_labels.py.

    python -m sam_road_b200.label_masks --dataset cityscale|spacenet [--root DIR]

reads every ground-truth graph pickle of the dataset under DIR (default ./cityscale or ./spacenet, the layout
SatMapDataset reads) and writes processed/keypoint_mask_<tile>.png and processed/road_mask_<tile>.png: a filled
disc of radius 3 at every node whose degree is not 2 and a 3-pixel cv2.line for every edge, pixel-identical to the
masks the reference scripts draw with OpenCV (DESIGN.md §16).  The reference scripts delete and recreate
processed/ first; this command only creates the directory when it is missing and overwrites the two files of each
tile, so anything else a user keeps there stays.

`tile_arrays` turns one adjacency dict into the keypoints and edges the scripts derive through networkx;
`masks_from_graphs` rasterises a list of them in one call of csrc/label_masks.cu."""
from __future__ import annotations

import argparse
import json
import os
import pickle
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import _lib

KEYPOINT_RADIUS = 3
ROAD_WIDTH = 3
SPACENET_SIZE = 400
IMAGE_SIZE = {"cityscale": 2048, "spacenet": SPACENET_SIZE}
CHUNK_BYTES = 1 << 28          # device bytes of the two masks of one chunk of tiles


def _node_key(dataset: str):
    if dataset == "cityscale":
        return lambda n: (int(n[1]), int(n[0]))
    if dataset == "spacenet":
        return lambda n: (int(n[1]), SPACENET_SIZE - int(n[0]))
    raise ValueError(f"dataset must be 'cityscale' or 'spacenet' (got {dataset!r})")


def tile_arrays(adj: Dict, dataset: str) -> Tuple[np.ndarray, np.ndarray]:
    """(keypoints [k, 2], edges [m, 4]) int32 of one ground-truth graph {(row, col): [(row, col), ...]}, as the
    scripts build them: node (int(col), int(row)) for CityScale and (int(col), 400 - int(row)) for SpaceNet (int
    truncates, so nearby float nodes merge); an undirected simple graph in which repeated and one-way entries
    collapse and nodes exist only through edges; keypoints are the nodes of degree != 2, a self-loop counting 2.
    Edges (x0, y0, x1, y1) are unique with (x0, y0) <= (x1, y1); both arrays are sorted."""
    key = _node_key(dataset)
    pairs = [key(n) + key(m) for n, neis in adj.items() for m in neis]
    if not pairs:
        return np.zeros((0, 2), np.int32), np.zeros((0, 4), np.int32)
    e = np.array(pairs, dtype=np.int64)
    if e.min() < np.iinfo(np.int32).min or e.max() > np.iinfo(np.int32).max:
        raise ValueError("a graph coordinate does not fit in int32")
    a, b = e[:, :2], e[:, 2:]
    swap = (a[:, 0] > b[:, 0]) | ((a[:, 0] == b[:, 0]) & (a[:, 1] > b[:, 1]))
    e = np.unique(np.where(swap[:, None], np.concatenate([b, a], 1), e), axis=0)
    nodes, inv = np.unique(np.concatenate([e[:, :2], e[:, 2:]]), axis=0, return_inverse=True)
    degree = np.bincount(inv.ravel(), minlength=len(nodes))
    return nodes[degree != 2].astype(np.int32), e.astype(np.int32)


def _csr(arrays: Sequence[np.ndarray], cols: int):
    off = np.zeros(len(arrays) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in arrays])
    flat = np.concatenate([np.asarray(x, np.int32).reshape(-1, cols) for x in arrays] + [np.zeros((1, cols), np.int32)])
    return flat, off       # one padding row: a zero-length device array has no address


def draw_masks(keypoints: Sequence[np.ndarray], edges: Sequence[np.ndarray], size: int, device="cuda",
               keypoint_radius: int = KEYPOINT_RADIUS, road_width: int = ROAD_WIDTH):
    """Device uint8 (keypoint [T, size, size], road [T, size, size]) of 0 / 255 for T tiles: cv2.circle(kp, p,
    keypoint_radius, 255, -1) at every keypoints[t] row (x, y) and cv2.line(road, p0, p1, 255, road_width) for
    every edges[t] row (x0, y0, x1, y1).  Asynchronous on the device's current stream."""
    import torch
    if len(keypoints) != len(edges):
        raise ValueError(f"{len(keypoints)} keypoint arrays but {len(edges)} edge arrays")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"label masks are drawn on a CUDA device (got {dev})")
    T = len(keypoints)
    nodes, node_off = _csr(keypoints, 2)
    segs, edge_off = _csr(edges, 4)
    up = [torch.from_numpy(x).to(dev) for x in (nodes, node_off, segs, edge_off)]
    kp = torch.empty((T, size, size), dtype=torch.uint8, device=dev)
    road = torch.empty((T, size, size), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.load().samroad_label_masks(T, size, *(_lib.ptr(t) for t in up), keypoint_radius, road_width,
                                               _lib.ptr(kp), _lib.ptr(road), stream), "samroad_label_masks")
    return kp, road


def masks_from_graphs(adjs: Sequence[Dict], dataset: str, device="cuda"):
    """Device uint8 (keypoint [T, S, S], road [T, S, S]) of the T ground-truth graphs `adjs` of `dataset`
    (S = 2048 for CityScale, 400 for SpaceNet), equal to what generate_labels.py writes for them."""
    arrays = [tile_arrays(adj, dataset) for adj in adjs]
    return draw_masks([a[0] for a in arrays], [a[1] for a in arrays], IMAGE_SIZE[dataset], device)


def tile_list(dataset: str, root: str) -> List:
    """The tiles generate_labels.py processes, in its order, with the path of each ground-truth pickle."""
    if dataset == "cityscale":
        return [(i, os.path.join(root, "20cities", f"region_{i}_refine_gt_graph.p")) for i in range(180)]
    if dataset == "spacenet":
        with open(os.path.join(root, "data_split.json")) as f:
            split = json.load(f)
        return [(t, os.path.join(root, "RGB_1.0_meter", f"{t}__gt_graph.p"))
                for t in split["test"] + split["validation"] + split["train"]]
    raise ValueError(f"dataset must be 'cityscale' or 'spacenet' (got {dataset!r})")


def write_dataset_masks(dataset: str, root: str, device="cuda") -> int:
    """Writes processed/{keypoint,road}_mask_<tile>.png under root for every tile; returns the tile count."""
    import cv2
    tiles = tile_list(dataset, root)
    for _, path in tiles:
        if not os.path.isfile(path):
            raise FileNotFoundError(f"ground-truth graph {path} is missing")
    out_dir = os.path.join(root, "processed")
    os.makedirs(out_dir, exist_ok=True)
    size = IMAGE_SIZE[dataset]
    chunk = max(1, CHUNK_BYTES // (2 * size * size))
    for first in range(0, len(tiles), chunk):
        part = tiles[first:first + chunk]
        adjs = []
        for _, path in part:
            with open(path, "rb") as f:
                adjs.append(pickle.load(f))
        kp, road = masks_from_graphs(adjs, dataset, device)
        kp, road = kp.cpu().numpy(), road.cpu().numpy()     # synchronises
        for k, (tile, _) in enumerate(part):
            for name, mask in (("keypoint", kp[k]), ("road", road[k])):
                png = os.path.join(out_dir, f"{name}_mask_{tile}.png")
                if not cv2.imwrite(png, mask):
                    raise OSError(f"cv2.imwrite could not write {png}")
        print(f"{dataset}: tiles {first}..{first + len(part) - 1} of {len(tiles)} written to {out_dir}")
    return len(tiles)


def main(argv=None) -> None:
    p = argparse.ArgumentParser(description="Write the keypoint and road label masks of a dataset (the "
                                            "reference's generate_labels.py) on the GPU.")
    p.add_argument("--dataset", required=True, choices=("cityscale", "spacenet"))
    p.add_argument("--root", default=None, help="dataset directory (default ./cityscale or ./spacenet)")
    args = p.parse_args(argv)
    write_dataset_masks(args.dataset, args.root or os.path.join(".", args.dataset))


if __name__ == "__main__":
    main()
