"""Deterministic synthetic weights and inputs for benchmarks and tests.

No SAM / sam_road checkpoint exists offline (SURVEY.md §7), so parity and throughput are measured
on seeded random weights carrying the reference's exact state_dict key set and shapes
(`model.param_shapes`, SURVEY.md §8b).  pos_embed and the rel-pos tables are randomised: the
reference zero-initialises them (image_encoder.py:68-70,221-222), which would hide rel-pos bugs.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch

from .model import param_shapes

_NORM_WEIGHTS = ("image_encoder.neck.1.weight", "image_encoder.neck.3.weight", "map_decoder.1.weight",
                 "mask_decoder.output_upscaling.1.weight", "prompt_encoder.mask_downscaling.1.weight",
                 "prompt_encoder.mask_downscaling.4.weight")


def _is_norm(key: str) -> bool:
    stem = key.rsplit(".", 1)[0]
    last = stem.rsplit(".", 1)[-1]
    return last in ("norm1", "norm2", "norm3", "norm4", "norm_final_attn") or \
        (stem + ".weight") in _NORM_WEIGHTS


def make_state_dict(config, seed: int = 0, logit_gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Reference-layout state_dict (fp32, CPU).  `logit_gain` scales the last decoder layer and
    TopoNet's output_proj so logits span a wider range than default-scale init gives (+-0.5)."""
    gen = torch.Generator().manual_seed(seed)
    shapes = param_shapes(config)
    sd: Dict[str, torch.Tensor] = {}

    def uniform(shape, bound):
        return (torch.rand(shape, generator=gen, dtype=torch.float32) * 2.0 - 1.0) * bound

    for key, shape in shapes.items():
        leaf = key.rsplit(".", 1)[1]
        if key.endswith("positional_encoding_gaussian_matrix"):
            t = torch.randn(shape, generator=gen)           # PositionEmbeddingRandom, scale 1.0
        elif key.endswith("pos_embed") or "rel_pos" in key:
            t = 0.02 * torch.randn(shape, generator=gen)
        elif _is_norm(key):
            t = (1.0 + 0.1 * torch.randn(shape, generator=gen)) if leaf == "weight" \
                else 0.05 * torch.randn(shape, generator=gen)
        elif leaf == "in_proj_weight":
            t = uniform(shape, math.sqrt(6.0 / (shape[0] + shape[1])))
        elif leaf == "in_proj_bias":
            t = 0.02 * torch.randn(shape, generator=gen)
        elif "linear_b_" in key:
            t = uniform(shape, 0.3 / math.sqrt(shape[1]))
        elif leaf == "weight":
            fan_in = int(np.prod(shape[1:])) if len(shape) > 1 else shape[0]
            t = uniform(shape, 1.0 / math.sqrt(fan_in))
        else:   # bias of a linear / conv: bound from the matching weight's fan-in
            wshape = shapes[key.rsplit(".", 1)[0] + ".weight"]
            t = uniform(shape, 1.0 / math.sqrt(int(np.prod(wshape[1:]))))
        sd[key] = t
    for key in ("map_decoder.7.weight", "map_decoder.7.bias", "topo_net.output_proj.weight",
                "topo_net.output_proj.bias", "mask_decoder.output_hypernetworks_mlps.1.layers.2.weight",
                "mask_decoder.output_hypernetworks_mlps.2.layers.2.weight"):
        if key in sd:
            sd[key] = sd[key] * logit_gain
    return sd


def make_tiles(batch: int, patch_size: int, seed: int = 0, dtype=torch.uint8) -> torch.Tensor:
    """Uniform random RGB tiles [B,P,P,3] (SURVEY.md §8d synthetic inputs)."""
    gen = torch.Generator().manual_seed(1000 + seed)
    t = torch.randint(0, 256, (batch, patch_size, patch_size, 3), generator=gen, dtype=torch.uint8)
    return t if dtype == torch.uint8 else t.to(dtype)


def make_topo_inputs(batch: int, patch_size: int, n_points: int, seed: int = 0, max_nbr: int = 16,
                     radius: float = 64.0, ragged: bool = True):
    """Keypoints on a jittered lattice per tile and kNN pair queries built the way
    inferencer.py:156-176 builds them (neighbours sorted by distance => prefix-valid masks; invalid
    slots point back at the source), padded to the batch maximum (inferencer.py:179-185).
    Returns int64 points [B,N,2] (x,y), int64 pairs [B,N,K,2], bool valid [B,N,K]."""
    import scipy.spatial
    rng = np.random.RandomState(2000 + seed)
    side = int(math.ceil(math.sqrt(n_points)))
    step = patch_size / side
    pts_l, pairs_l, valid_l = [], [], []
    for b in range(batch):
        n = n_points if not ragged else max(1, n_points - (b * 7) % max(1, n_points // 3))
        gy, gx = np.divmod(rng.permutation(side * side)[:n], side)
        jit = rng.uniform(-0.35, 0.35, size=(n, 2)) * step
        xy = np.stack([(gx + 0.5) * step, (gy + 0.5) * step], 1) + jit
        xy = np.clip(np.round(xy), 0, patch_size).astype(np.int64)
        tree = scipy.spatial.KDTree(xy)
        k = min(max_nbr + 1, max(2, n))
        _, knn = tree.query(xy, k=k, distance_upper_bound=radius)
        knn = knn.reshape(n, -1)[:, 1:]
        if knn.shape[1] < max_nbr:
            knn = np.pad(knn, [(0, 0), (0, max_nbr - knn.shape[1])], constant_values=n)
        src = np.tile(np.arange(n)[:, None], (1, max_nbr))
        valid = knn < n
        tgt = np.where(valid, knn, src)
        pts_l.append(xy)
        pairs_l.append(np.stack([src, tgt], -1))
        valid_l.append(valid)
    nmax = max(p.shape[0] for p in pts_l)
    pad = lambda a: np.pad(a, [(0, nmax - a.shape[0])] + [(0, 0)] * (a.ndim - 1))  # noqa: E731
    return (torch.tensor(np.stack([pad(p) for p in pts_l])),
            torch.tensor(np.stack([pad(p) for p in pairs_l])),
            torch.tensor(np.stack([pad(v) for v in valid_l])))


def make_road_graph(extent: int, seed: int = 0, spacing: int = 48, lo: int = 16):
    """Sat2graph adjacency dict {(row, col): [(row, col), ...]} of a synthetic road network inside
    [lo, extent]^2: an axis-aligned street grid with nodes every `spacing` pixels and intermediate nodes (equal
    distances along axis-aligned runs), a few missing grid edges (degree-3 intersections), dead-end spurs, and two
    diagonal overpasses that cross grid edges without sharing a node (crossovers)."""
    rng = np.random.RandomState(3000 + seed)
    adj: Dict = {}

    def link(a, b):
        adj.setdefault(a, [])
        adj.setdefault(b, [])
        if b not in adj[a]:
            adj[a].append(b)
            adj[b].append(a)

    lines = list(range(lo, extent + 1, spacing))
    for r in lines:
        for i, c in enumerate(lines[:-1]):
            c2 = lines[i + 1]
            if rng.rand() < 0.12:
                continue
            mid = (r, c + (c2 - c) // 2)
            link((r, c), mid)
            link(mid, (r, c2))
    for c in lines:
        for i, r in enumerate(lines[:-1]):
            r2 = lines[i + 1]
            if rng.rand() < 0.12:
                continue
            link((r, c), (r2, c))
    for _ in range(max(2, len(lines))):       # dead ends
        r, c = lines[rng.randint(len(lines))], lines[rng.randint(len(lines))]
        link((r, c), (r + int(rng.randint(9, spacing // 2)), c + int(rng.randint(5, spacing // 2))))
    for k in range(2):                          # overpasses: off-grid nodes only
        a = (lo + 7 + 11 * k, lo + 5 + 3 * k)
        m = (lo + (extent - lo) // 2 + 5 + 2 * k, lo + (extent - lo) // 2 + 9 - 4 * k)
        b = (extent - 3 - 7 * k, extent - 13 + 5 * k)
        if k:
            a, b = (a[0], b[1]), (b[0], a[1])
            m = (m[0] + 3, m[1] - 6)
        link(a, m)
        link(m, b)
    return adj


def write_label_scenes(root: str, dataset: str, tiles, size: int, seed: int = 0, extent: int = None,
                       empty=(), spacing: int = 48) -> None:
    """Scene files of `tiles` in the reference's cityscale / spacenet layout under root (dataset.py:311-340):
    a seeded RGB PNG, binary keypoint / road mask PNGs (0 / 255) and the pickled ground-truth graph (an empty
    dict for the tiles in `empty`).  Graph coordinates are (row, col) for cityscale and the spacenet convention
    (x = col, y = 400 - row) is applied by the dataset.  `spacing` is the street grid's (make_road_graph)."""
    import os
    import pickle

    import cv2
    pat = {"cityscale": ("cityscale/20cities/region_{}_sat.png", "cityscale/processed/keypoint_mask_{}.png",
                         "cityscale/processed/road_mask_{}.png", "cityscale/20cities/region_{}_refine_gt_graph.p"),
           "spacenet": ("spacenet/RGB_1.0_meter/{}__rgb.png", "spacenet/processed/keypoint_mask_{}.png",
                        "spacenet/processed/road_mask_{}.png", "spacenet/RGB_1.0_meter/{}__gt_graph.p")}[dataset]
    for p in pat:
        os.makedirs(os.path.join(root, os.path.dirname(p)), exist_ok=True)
    for k, t in enumerate(tiles):
        rng = np.random.RandomState(4000 + 97 * seed + k)
        rgb = rng.randint(0, 256, (size, size, 3)).astype(np.uint8)
        kp = ((rng.rand(size, size) < 0.1) * 255).astype(np.uint8)
        road = ((rng.rand(size, size) < 0.3) * 255).astype(np.uint8)
        cv2.imwrite(os.path.join(root, pat[0].format(t)), rgb[:, :, ::-1])
        cv2.imwrite(os.path.join(root, pat[1].format(t)), kp)
        cv2.imwrite(os.path.join(root, pat[2].format(t)), road)
        adj = {} if t in empty else make_road_graph(extent or size - 16, seed=seed + k, spacing=spacing)
        with open(os.path.join(root, pat[3].format(t)), "wb") as f:
            pickle.dump(adj, f)
