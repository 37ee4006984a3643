"""Tile-loop driver: drop-in for the reference's `inferencer.infer_one_img` / CLI (inferencer.py:61-349).

    pred_nodes, pred_edges, keypoint_mask, road_mask = infer_one_img(net, img, config)

Same signature, argument meaning and return values as the reference (SURVEY.md §8b).  What changes is
where the work happens -- everything between the uint8 scene going up and the graph coming down runs
on the GPU (SURVEY.md §7 steps 8-9, §8f rows 1-3):
  * the uint8 scene is uploaded once; tiles are windows of it, cropped on the device and fed to the
    encoder as uint8 (the reference converts every crop to float32 on the CPU and copies it
    synchronously, inferencer.py:52-58,94);
  * mask fusion (inferencer.py:79-110) is one kernel that adds the tiles in tile-list order, so the
    uint8 masks are bit-identical to the reference's accumulation for identical scores;
  * keypoint extraction (graph_extraction.py:130-139, graph_utils.py:572-591), the per-tile box query
    + kNN pair construction (inferencer.py:126-197) and the edge aggregation (inferencer.py:206-230)
    are device kernels behind `sam_road_b200.graph.SceneGraph` (csrc/graph.cu): exact greedy NMS in the
    reference's visiting order, exact kNN, float32 sums in the reference's (tile, sample, pair) order;
  * with torch.distributed initialised, tiles are sharded over ranks in contiguous blocks, the
    per-tile mask scores are all-gathered once (by the copy engines over NVLink peer memory, batch by
    batch under the next batch's compute: sam_road_b200/exchange.py), the topology scores with one
    all-reduce of a disjointly-written buffer, and every rank fuses / aggregates in global tile order
    -> identical masks and graph on all ranks and at any world size (SURVEY.md §8e).
There is no CPU path: without the CUDA library every stage raises.
"""
from __future__ import annotations

import os
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .graph import SceneGraph
from .model import _cfg_get

TileInfo = Tuple[int, Tuple[int, int], Tuple[int, int]]


def get_patch_info_one_img(image_index: int, image_size: int, sample_margin: int, patch_size: int,
                           patches_per_edge: int) -> List[TileInfo]:
    """Tile grid: round(linspace(margin, size-(P+margin), n)), x outer / y inner (dataset.py:56-67)."""
    lo, hi = sample_margin, image_size - (patch_size + sample_margin)
    origins = [round(v) for v in np.linspace(start=lo, stop=hi, num=patches_per_edge)]
    return [(image_index, (x, y), (x + patch_size, y + patch_size)) for x in origins for y in origins]


def _shard(n_items: int, rank: int, world: int) -> Tuple[int, int, int]:
    """Contiguous block of items owned by `rank`; returns (begin, end, per_rank)."""
    per = (n_items + world - 1) // world
    b = min(n_items, rank * per)
    return b, min(n_items, b + per), per


def batch_plan(n_tiles: int, batch_size: int, world: int) -> List[Tuple[int, int, int]]:
    """Every rank's batches as (rank, first_tile, n) in global tile order.  All ranks compute the same
    list, which fixes the layout of the exchanged topology-score buffer."""
    out = []
    for r in range(world):
        lo, hi, _ = _shard(n_tiles, r, world)
        for b0 in range(lo, hi, batch_size):
            out.append((r, b0, min(batch_size, hi - b0)))
    return out


def fuse_masks_device(scores: torch.Tensor, tiles: Sequence[TileInfo], H: int, W: int):
    """scores [n_tiles,P,P,2] fp32 (device, tile-list order) -> uint8 keypoint / road masks [H,W]."""
    dev = scores.device
    P = scores.shape[1]
    x0 = torch.tensor([t[1][0] for t in tiles], dtype=torch.int32).to(dev)
    y0 = torch.tensor([t[1][1] for t in tiles], dtype=torch.int32).to(dev)
    kp = torch.empty((H, W), dtype=torch.uint8, device=dev)
    road = torch.empty((H, W), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().samroad_fuse_masks(scores.data_ptr(), len(tiles), P, x0.data_ptr(),
                                                  y0.data_ptr(), H, W, kp.data_ptr(), road.data_ptr(),
                                                  _lib.current_stream_ptr()), "samroad_fuse_masks")
    return kp, road


_GRAPHS: Dict[int, SceneGraph] = {}
_EXCHANGES: Dict[tuple, "object"] = {}


def _exchange(rows_per_rank: int, P: int, device: torch.device, group, world: int):
    """Cached gather buffers of the mask-score exchange (allocating symmetric memory is a collective)."""
    from .exchange import TileExchange
    key = (rows_per_rank, P, device.index, id(group), world)
    if key not in _EXCHANGES:
        _EXCHANGES.clear()
        _EXCHANGES[key] = TileExchange(rows_per_rank, (P, P, 2), torch.float32, device, group=group, slots=1)
    return _EXCHANGES[key]
_PINNED: Dict[Tuple[int, int, int], Tuple[torch.Tensor, torch.Tensor]] = {}


def _pinned_masks(H: int, W: int, slot: int = 0):
    """Page-locked staging for the two uint8 masks (allocated once per scene size and pipeline slot; the
    caller gets copies)."""
    if (H, W, slot) not in _PINNED:
        for k in [k for k in _PINNED if k[:2] != (H, W)]:
            del _PINNED[k]
        _PINNED[(H, W, slot)] = (torch.empty((H, W), dtype=torch.uint8).pin_memory(),
                                 torch.empty((H, W), dtype=torch.uint8).pin_memory())
    return _PINNED[(H, W, slot)]


def _scene_graph(device: torch.device) -> SceneGraph:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _GRAPHS:
        _GRAPHS[idx] = SceneGraph(torch.device("cuda", idx))
    return _GRAPHS[idx]


class _SceneJob:
    """State of one scene between its two halves (pass 1 enqueued -> graph stage / pass 2)."""
    pass


def _scene_start(net, img: np.ndarray, config, device: torch.device, group, shard: bool, slot: int = 0) -> _SceneJob:
    """First half of infer_one_img (inferencer.py:61-110), enqueue only: scene upload, pass 1 over the
    tiles this rank owns, the mask-score exchange, fusion and the start of the mask download -- all on the
    current stream, no host synchronisation."""
    import torch.distributed as dist
    j = _SceneJob()
    distributed = shard and dist.is_available() and dist.is_initialized()
    j.group = group
    j.rank = rank = dist.get_rank(group) if distributed else 0
    j.world = world = dist.get_world_size(group) if distributed else 1
    j.device, j.net, j.config = device, net, config
    j.t_start = time.perf_counter()
    H, W = int(img.shape[0]), int(img.shape[1])
    j.P = P = int(_cfg_get(config, "PATCH_SIZE"))
    s = P // 16
    j.bs = bs = int(_cfg_get(config, "INFER_BATCH_SIZE"))
    tiles = get_patch_info_one_img(0, H, int(_cfg_get(config, "SAMPLE_MARGIN")), P,
                                   int(_cfg_get(config, "INFER_PATCHES_PER_EDGE")))
    j.n_tiles = n_tiles = len(tiles)
    j.tile_xy = tile_xy = np.array([t[1] for t in tiles], dtype=np.int32).reshape(-1, 2)
    lo, hi, per = _shard(n_tiles, rank, world)
    j.lo, n_mine = lo, hi - lo

    # ---- pass 1: masks + image features of the tiles this rank owns -------------------------------
    img_d = torch.as_tensor(np.ascontiguousarray(img)).to(device)               # one H2D of the scene
    ex = None
    if world > 1:   # the exchange step (SURVEY.md §8e): every rank's per-tile mask scores to every rank
        ex = _exchange(per, P, device, group, world)
        ex.wait(0)
        scores_all, my_scores = ex.gathered(0), ex.local_block(0)
    else:
        scores_all = torch.empty((per, P, P, 2), dtype=torch.float32, device=device)
        my_scores = scores_all
    j.feats = feats = torch.empty((max(n_mine, 1), 256, s, s), dtype=torch.float32, device=device)
    j.scene_call = scene_call = getattr(net, "infer_masks_and_img_features_scene", None)
    n_batches = (n_mine + bs - 1) // bs
    for bi, b0 in enumerate(range(0, n_mine, bs)):
        nb = min(bs, n_mine - b0)
        if scene_call is not None:
            scene_call(img_d, tile_xy[lo + b0: lo + b0 + nb], out_scores=my_scores[b0:b0 + nb],
                       out_emb=feats[b0:b0 + nb])
        else:    # any object with the reference's model interface
            rgb = torch.stack([img_d[y0:y1, x0:x1, :] for _, (x0, y0), (x1, y1) in tiles[lo + b0: lo + b0 + nb]], 0)
            sc, ft = net.infer_masks_and_img_features(rgb)
            my_scores[b0:b0 + nb].copy_(sc)
            feats[b0:b0 + nb].copy_(ft)
        if ex is not None:      # a batch's scores leave while the next batch computes
            ex.publish(0, b0, b0 + nb, first=bi == 0, last=bi == n_batches - 1)
    if ex is not None:
        if n_batches == 0:      # more ranks than tiles: still part of the round
            ex.publish(0, 0, 0, first=True, last=True)
        ex.wait(0)
    j.kp_d, j.road_d = fuse_masks_device(scores_all[:n_tiles], tiles, H, W)
    # the masks are return values: start their download now, it overlaps the graph stage
    j.kp_h, j.road_h = _pinned_masks(H, W, slot)
    j.kp_h.copy_(j.kp_d, non_blocking=True)
    j.road_h.copy_(j.road_d, non_blocking=True)
    j.masks_done = torch.cuda.Event()
    j.masks_done.record()
    return j


def _scene_finish(j: _SceneJob, nms_tie_order: Optional[str], timings: Optional[dict]):
    """Second half of infer_one_img (inferencer.py:112-234) on the current stream: keypoints, pair
    queries, TopoNet on the stored features, edge aggregation, downloads."""
    import torch.distributed as dist
    device, net, config, world, rank, group = j.device, j.net, j.config, j.world, j.rank, j.group
    n_tiles, tile_xy, P, bs, lo, feats, scene_call = j.n_tiles, j.tile_xy, j.P, j.bs, j.lo, j.feats, j.scene_call
    kp_h, road_h, masks_done, t_start = j.kp_h, j.road_h, j.masks_done, j.t_start
    if timings is not None:
        torch.cuda.synchronize(device)
    t_pass1 = time.perf_counter()

    # ---- keypoints (device) ------------------------------------------------------------------------------
    gx = _scene_graph(device)
    points_d = gx.extract_graph_points(j.kp_d, j.road_d, _cfg_get(config, "ITSC_THRESHOLD"),
                                       _cfg_get(config, "ROAD_THRESHOLD"),
                                       _cfg_get(config, "ITSC_NMS_RADIUS"),
                                       _cfg_get(config, "ROAD_NMS_RADIUS"), tie_order=nms_tie_order)
    n_points = int(points_d.shape[0])
    t_points = time.perf_counter()
    if n_points == 0:    # inferencer.py:123-124
        masks_done.synchronize()
        if timings is not None:
            timings.update(pass1_s=t_pass1 - t_start, keypoints_s=t_points - t_pass1, pass2_s=0.0,
                           total_s=time.perf_counter() - t_start, n_tiles=n_tiles, n_points=0,
                           graph_stats=dict(gx.stats))
        return (np.zeros((0, 2), dtype=np.int64), np.zeros((0, 2), dtype=np.int32), kp_h.numpy().copy(),
                road_h.numpy().copy())

    # ---- pass 2: TopoNet on the stored features -------------------------------------------------------
    K = int(_cfg_get(config, "MAX_NEIGHBOR_QUERIES"))
    R = float(_cfg_get(config, "NEIGHBOR_RADIUS"))

    def _mark():
        if timings is not None:
            torch.cuda.synchronize(device)
        return time.perf_counter()
    counts = gx.plan_pair_queries(points_d, tile_xy, P, R)
    t_plan = _mark()
    # layout of the scene-wide score buffer: per batch [n, nmax_of_the_batch, K] (inferencer.py:179-185
    # pads every batch to its own maximum); batches with no point at all are skipped (188-189)
    plan = batch_plan(n_tiles, bs, world)
    tile_off = np.full(n_tiles, -1, dtype=np.int64)
    batch_nmax, cursor = [], 0
    for (_, b0, nb) in plan:
        nmax = int(counts[b0:b0 + nb].max()) if nb > 0 else 0
        batch_nmax.append(nmax)
        if nmax > 0:
            tile_off[b0:b0 + nb] = cursor + np.arange(nb, dtype=np.int64) * (nmax * K)
            cursor += nb * nmax * K
    topo_flat = torch.zeros((max(cursor, 1),), dtype=torch.float32, device=device)
    for (r, b0, nb), nmax in zip(plan, batch_nmax):
        if r != rank or nmax == 0:
            continue
        pts, prs, val = gx.fill_batch(b0, nb, nmax, K)
        out = topo_flat[int(tile_off[b0]): int(tile_off[b0]) + nb * nmax * K]
        if scene_call is not None:
            net.infer_toponet(feats[b0 - lo: b0 - lo + nb], pts, prs, val, out=out)
        else:
            out.copy_(net.infer_toponet(feats[b0 - lo: b0 - lo + nb], pts, prs, val).reshape(-1))
    if world > 1:   # every element is written by exactly one rank (zeros elsewhere): the sum is exact
        dist.all_reduce(topo_flat, op=dist.ReduceOp.SUM, group=group)
    t_topo = _mark()
    edges_d = gx.aggregate_edges(topo_flat, tile_off, K, float(_cfg_get(config, "TOPO_THRESHOLD")))
    t_agg = _mark()
    graph_points = points_d.cpu().numpy()
    pred_edges = edges_d.cpu().numpy()
    if pred_edges.shape[0] == 0:
        pred_edges = np.array([]).reshape(-1, 2)          # what np.array([]).reshape(-1, 2) gives the reference
    pred_nodes = graph_points[:, ::-1]   # to (r, c), inferencer.py:230
    masks_done.synchronize()
    if timings is not None:
        t_end = time.perf_counter()
        timings.update(pass1_s=t_pass1 - t_start, keypoints_s=t_points - t_pass1,
                       pass2_s=t_end - t_points, pair_queries_s=t_plan - t_points, toponet_s=t_topo - t_plan,
                       edges_s=t_agg - t_topo, download_s=t_end - t_agg, total_s=t_end - t_start,
                       n_tiles=n_tiles, n_points=n_points, n_edges=int(pred_edges.shape[0]),
                       graph_stats=dict(gx.stats),
                       topo_samples=int(sum(nb * nm for (_, _, nb), nm in zip(plan, batch_nmax))))
    return pred_nodes, pred_edges, kp_h.numpy().copy(), road_h.numpy().copy()


def _resolve_device(net, device) -> torch.device:
    if device is None:
        device = next(net.parameters()).device
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"sam_road_b200 scene inference runs on CUDA only, got '{device}'")
    return device


def infer_one_img(net, img: np.ndarray, config, device: Optional[torch.device] = None,
                  group=None, timings: Optional[dict] = None, shard: bool = True,
                  nms_tie_order: Optional[str] = None):
    """Whole-scene inference (inferencer.py:61-234).

    img: uint8 [H,W,3] RGB.  Returns (pred_nodes int64 [N,2] (r,c), pred_edges int64 [E,2],
    fused_keypoint_mask uint8 [H,W], fused_road_mask uint8 [H,W]) -- identical on every rank when run
    distributed.  `shard=False` makes a rank process the whole scene alone even if torch.distributed
    is up.  `nms_tie_order`: "numpy" (default; this host's np.argsort decides ties like the reference)
    or "stable" (device-only sort), see sam_road_b200.graph."""
    device = _resolve_device(net, device)
    job = _scene_start(net, img, config, device, group, shard)
    return _scene_finish(job, nms_tie_order, timings)


def infer_scenes(net, images, config, device: Optional[torch.device] = None,
                 nms_tie_order: Optional[str] = None, prefetch: int = 2):
    """Generator over `infer_one_img(net, img, config)` for a sequence of scenes (the reference loops
    `for img_id in test_img_indices` and reads each image right before it is needed, inferencer.py:271-281):
    a background thread pulls the next images from the `images` iterable -- file reads and PNG decoding in the
    CLI -- while the GPU works on the current scene.  Results are infer_one_img's, in order.

    The scenes themselves run back to back on one stream.  The next scene's encoder pass is not enqueued on a
    second stream under the current scene's graph stage: the encoder GEMMs are persistent (one CTA per SM), so
    the ~60 small kernels and the read-backs of the graph stage would queue behind them."""
    import queue
    import threading
    device = _resolve_device(net, device)
    q: "queue.Queue" = queue.Queue(maxsize=max(1, prefetch))
    _END = object()

    def _loader():
        try:
            for im in images:
                q.put(im)
            q.put(_END)
        except BaseException as e:      # surface loader errors in the consumer
            q.put(e)

    threading.Thread(target=_loader, daemon=True).start()
    while True:
        item = q.get()
        if isinstance(item, BaseException):
            raise item
        if item is _END:
            return
        yield infer_one_img(net, item, config, device=device, shard=False, nms_tie_order=nms_tie_order)


# --------------------------------------------------------------------------------------------------
# CLI (inferencer.py:24-35, 239-349): same flags, same output tree
# --------------------------------------------------------------------------------------------------
class _Cfg(dict):
    """addict.Dict-like: attribute access, missing keys read as an empty (falsy) _Cfg (utils.py:6-9)."""

    def __getattr__(self, k):
        return self[k] if k in self else _Cfg()


def load_config(path: str) -> _Cfg:
    import yaml
    with open(path) as f:
        return _Cfg(yaml.safe_load(f))


def convert_to_sat2graph_format(nodes: np.ndarray, edges: np.ndarray) -> dict:
    """{(r,c): [(r,c) neighbours]} with reverse edges added (graph_utils.py:383-405)."""
    int_nodes = [(round(float(x)), round(float(y))) for x, y in nodes]
    adj: List[list] = [[] for _ in int_nodes]
    for a, b in list(edges) + [e[::-1] for e in edges]:
        if int(b) not in adj[int(a)]:
            adj[int(a)].append(int(b))
    return {int_nodes[i]: [int_nodes[j] for j in nbrs] for i, nbrs in enumerate(adj)}


def main(argv=None):
    import pickle
    from argparse import ArgumentParser

    import cv2
    from .model import SAMRoad
    ap = ArgumentParser()
    ap.add_argument("--checkpoint", default=None, help="checkpoint of the model to test.")
    ap.add_argument("--config", default=None, help="model config.")
    ap.add_argument("--output_dir", default=None, help="Name of the output dir under ./save/")
    ap.add_argument("--device", default="cuda", help="device to use")
    args = ap.parse_args(argv)
    config = load_config(args.config)
    device = torch.device(args.device)
    net = SAMRoad(config)
    ckpt = torch.load(args.checkpoint, map_location="cpu")
    print(f"##### Loading Trained CKPT {args.checkpoint} #####")
    net.load_state_dict(ckpt["state_dict"], strict=True)
    net.eval().to(device)

    if config.DATASET == "cityscale":
        test_ids = [x for x in range(180) if x % 10 == 9 or x % 20 == 8]       # dataset.py:21-41
        rgb_pattern = "./cityscale/20cities/region_{}_sat.png"
    elif config.DATASET == "spacenet":
        import json
        test_ids = json.load(open("./spacenet/data_split.json"))["test"]        # dataset.py:44-53
        rgb_pattern = "./spacenet/RGB_1.0_meter/{}__rgb.png"
    else:
        raise SystemExit(f"config.DATASET must be 'cityscale' or 'spacenet', got {config.DATASET!r}")
    out_dir = f"./save/{args.output_dir}" if args.output_dir else \
        "./save/infer_" + time.strftime("%Y%m%d_%H%M%S")
    for sub in ("mask", "viz", "graph"):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    loaded = {}

    def read_all():      # runs on infer_scenes' loader thread: decoding overlaps the GPU work of earlier scenes
        for i in test_ids:
            im = cv2.cvtColor(cv2.imread(rgb_pattern.format(i)), cv2.COLOR_BGR2RGB)
            loaded[i] = im
            yield im

    t0 = time.time()
    results = infer_scenes(net, read_all(), config, device=device)
    for img_id, (nodes, edges, itsc_mask, road_mask) in zip(test_ids, results):
        print(f"Processing {img_id}")
        img = loaded.pop(img_id)
        cv2.imwrite(os.path.join(out_dir, "mask", f"{img_id}_road.png"), road_mask)
        cv2.imwrite(os.path.join(out_dir, "mask", f"{img_id}_itsc.png"), itsc_mask)
        viz = cv2.cvtColor(img.copy(), cv2.COLOR_RGB2BGR)
        for a, b in edges:
            cv2.line(viz, (int(nodes[a][1]), int(nodes[a][0])), (int(nodes[b][1]), int(nodes[b][0])),
                     (15, 160, 253), 4)
        for r, c in nodes:
            cv2.circle(viz, (int(c), int(r)), 4, (0, 255, 255), -1)
        cv2.imwrite(os.path.join(out_dir, "viz", f"{img_id}.png"), viz)
        if config.DATASET == "spacenet":    # r, c -> sat2graph convention (inferencer.py:332-334)
            nodes = np.stack([400 - nodes[:, 0], nodes[:, 1]], axis=1)
        with open(os.path.join(out_dir, "graph", f"{img_id}.p"), "wb") as f:
            pickle.dump(convert_to_sat2graph_format(nodes, np.asarray(edges).reshape(-1, 2)), f)
        print(f"Done for {img_id}.")
    total = time.time() - t0      # wall time of the whole (pipelined) loop, output writing included
    msg = f"Inference completed for {args.config} in {total} seconds."
    print(msg)
    with open(os.path.join(out_dir, "inference_time.txt"), "w") as f:
        f.write(msg)


if __name__ == "__main__":
    main()
