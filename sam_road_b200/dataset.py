"""Training and evaluation batches on the device: SatMapDataset and GraphLabelGenerator.sample_patch
(dataset.py:56-445 of the reference), DESIGN.md §13.

Per scene, once, on the host (numpy / scipy, no igraph / rtree / shapely): the ground-truth graph as
GraphLabelGenerator.__init__ (dataset.py:71-125) builds it -- de-duplicated edges, crossover points,
the graph subdivided at resolution 4, the points excluded near crossovers, the NMS immunity of points
whose subdivided degree is not 2, the sampling weights and a CSR adjacency.  That and the scene's uint8
RGB and masks go to the device once.  Per batch, on the device (csrc/labels.cu): patch draws, crop and
rot90, box query, NMS, source sampling, kNN, BFS labels, point transform and collation.

    ds = SatMapDataset(config, is_train=True)
    for batch in ds.loader(config.BATCH_SIZE):     # dicts of device tensors, graph_collate_fn's layout
        loss = net.training_step(batch, i)

Randomness is Philox on the device keyed by a 62-bit seed drawn from torch's default generator per
batch, so torch.manual_seed reproduces a batch bit for bit.  NumPy's streams are not reproduced.  Under
torch.distributed the drawn seed is made per rank and each rank's loader serves its share (BatchLoader).
"""
from __future__ import annotations

import ctypes as C
import json
import math
import pickle
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

SUBDIVIDE_RESOLUTION = 4      # dataset.py:81
CROSSOVER_EXCLUDE_RADIUS = 4  # dataset.py:96
INTERESTING_RADIUS = 32       # dataset.py:115
EXCLUDED, IMMUNE = 1, 2       # flag bits of the device upload (include/samroad_b200.h)


# ---- per-scene precompute (GraphLabelGenerator.__init__) ------------------------------------------------------

def graph_from_adj_dict(graph: dict, coord_transform: Callable) -> Tuple[np.ndarray, List[Tuple[int, int]]]:
    """(nodes [n,2] after coord_transform, edges) of a sat2graph adjacency dict (graph_utils.py:408-474).
    Node ids follow first appearance over the keys and then their neighbour lists; edges are de-duplicated as
    (min, max) pairs in the iteration order of the Python set that de-duplicates them, as the reference builds
    its igraph from that set."""
    node_id: Dict = {}
    for node, nbrs in graph.items():
        node_id.setdefault(node, len(node_id))
        for nb in nbrs:
            node_id.setdefault(nb, len(node_id))
    pairs = set()
    for node, nbrs in graph.items():
        a = node_id[node]
        for nb in nbrs:
            b = node_id[nb]
            pairs.add((min(a, b), max(a, b)))
    nodes = [None] * len(node_id)
    for node, i in node_id.items():
        nodes[i] = node
    arr = np.array(nodes) if nodes else np.zeros((0, 2))
    return np.asarray(coord_transform(arr)), list(pairs)


def segment_crossings(p1: np.ndarray, p2: np.ndarray, p3: np.ndarray, p4: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Proper crossings of segments p1p2 and p3p4 (arrays [k,2]): (mask [k], points [k,2]).  A crossing is a
    single intersection point that is an endpoint of neither segment; parallel and collinear pairs never
    cross.  The endpoint test is made on the exact cross-product numerators (integer coordinates stay exact
    in float64), the point is p1 + t (p2 - p1)."""
    d1, d2, q = p2 - p1, p4 - p3, p3 - p1
    den = d1[:, 0] * d2[:, 1] - d1[:, 1] * d2[:, 0]
    tn = q[:, 0] * d2[:, 1] - q[:, 1] * d2[:, 0]
    un = q[:, 0] * d1[:, 1] - q[:, 1] * d1[:, 0]
    s = np.sign(den)
    den_a, tn_s, un_s = np.abs(den), tn * s, un * s
    hit = (den != 0) & (tn_s > 0) & (tn_s < den_a) & (un_s > 0) & (un_s < den_a)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(den != 0, tn / np.where(den != 0, den, 1.0), 0.0)
    pts = p1 + t[:, None] * d1
    for e in (p1, p2, p3, p4):
        hit &= ~np.all(pts == e, axis=1)
    return hit, pts


def crossover_points(points: np.ndarray, edges: np.ndarray) -> np.ndarray:
    """Points where two edges of the graph cross (graph_utils.py:516-544), one per crossing pair of edges."""
    import scipy.spatial
    if edges.shape[0] < 2:
        return np.zeros((0, 2))
    a, b = points[edges[:, 0]].astype(np.float64), points[edges[:, 1]].astype(np.float64)
    mid, half = 0.5 * (a + b), 0.5 * np.linalg.norm(b - a, axis=1)
    # two segments can only meet when their midpoints are within the sum of their half lengths
    cand = scipy.spatial.cKDTree(mid).query_pairs(2.0 * float(half.max()) + 1.0, output_type="ndarray")
    if cand.shape[0] == 0:
        return np.zeros((0, 2))
    i, j = cand[:, 0], cand[:, 1]
    hit, pts = segment_crossings(a[i], b[i], a[j], b[j])
    return pts[hit]


def subdivide(points: np.ndarray, edges: np.ndarray, resolution: float) -> Tuple[np.ndarray, np.ndarray]:
    """Subdivided graph (graph_utils.py:546-570): original nodes first, then the new points edge by edge;
    each edge of length L becomes max(1, int(L / resolution)) pieces at np.linspace(0, 1) fractions."""
    new_pts = [np.asarray(points, dtype=np.float64).reshape(-1, 2)]
    new_edges = []
    nxt = points.shape[0]
    for s, t in edges:
        p0, p1 = points[s], points[t]
        d = p1 - p0
        pieces = max(1, int(np.linalg.norm(d) / resolution))
        frac = np.linspace(0.0, 1.0, pieces + 1, endpoint=True)
        inner = (np.expand_dims(np.array(p0), 0) + np.expand_dims(frac, 1) @ np.expand_dims(d, 0))[1:-1]
        ids = list(range(nxt, nxt + inner.shape[0]))
        nxt += inner.shape[0]
        new_pts.append(inner.astype(np.float64))
        chain = [int(s)] + ids + [int(t)]
        new_edges.extend(zip(chain[:-1], chain[1:]))
    e = np.array(new_edges, dtype=np.int64).reshape(-1, 2)
    return np.concatenate(new_pts, axis=0), e


@dataclass
class SceneLabels:
    """What GraphLabelGenerator.__init__ holds for one scene, as arrays over the subdivided points."""
    points: np.ndarray          # [n, 2] float64 (x, y)
    edges: np.ndarray           # [m, 2] int64 subdivided edges
    crossovers: np.ndarray      # [c, 2] float64
    excluded: np.ndarray        # [n] bool: within CROSSOVER_EXCLUDE_RADIUS of a crossover, inclusive
    nms_override: np.ndarray    # [n] float32: 2.0 where the subdivided degree is not 2
    weights: np.ndarray         # [n] float32: 0.9 within INTERESTING_RADIUS of an intersection / crossover
    adj_start: np.ndarray       # [n + 1] int32 CSR offsets
    adj: np.ndarray             # [2m] int32 neighbours

    @property
    def flags(self) -> np.ndarray:
        return (self.excluded.astype(np.uint8) * EXCLUDED) | ((self.nms_override > 1.0).astype(np.uint8) * IMMUNE)


def _ball_union(tree, centres: np.ndarray, r: float, n: int) -> np.ndarray:
    out = np.zeros(n, dtype=bool)
    if len(centres) == 0:
        return out
    for lst in tree.query_ball_point(np.asarray(centres, dtype=np.float64).reshape(-1, 2), r):
        out[lst] = True
    return out


def precompute_scene(adj_dict: dict, coord_transform: Callable) -> SceneLabels:
    """GraphLabelGenerator.__init__ (dataset.py:71-125) for one non-empty sat2graph adjacency dict."""
    import scipy.spatial
    nodes, edge_list = graph_from_adj_dict(adj_dict, coord_transform)
    edges = np.array(edge_list, dtype=np.int64).reshape(-1, 2)
    cross = crossover_points(nodes, edges)
    pts, sub_edges = subdivide(nodes, edges, SUBDIVIDE_RESOLUTION)
    n = pts.shape[0]
    tree = scipy.spatial.cKDTree(pts)
    excluded = _ball_union(tree, cross, CROSSOVER_EXCLUDE_RADIUS, n)
    degree = np.bincount(sub_edges.reshape(-1), minlength=n)
    override = np.where(degree != 2, 2.0, 0.0).astype(np.float32)
    interesting = _ball_union(tree, pts[degree != 2], INTERESTING_RADIUS, n) | \
        _ball_union(tree, cross, INTERESTING_RADIUS, n)
    weights = np.where(interesting, 0.9, 0.1).astype(np.float32)
    src = np.concatenate([sub_edges[:, 0], sub_edges[:, 1]])
    dst = np.concatenate([sub_edges[:, 1], sub_edges[:, 0]])
    order = np.argsort(src, kind="stable")
    adj_start = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=adj_start[1:])
    if n >= 2 ** 31 - 1 or adj_start[-1] >= 2 ** 31:
        raise ValueError(f"scene graph too large for int32 indexing ({n} points)")
    return SceneLabels(points=pts, edges=sub_edges, crossovers=cross, excluded=excluded, nms_override=override,
                       weights=weights, adj_start=adj_start.astype(np.int32), adj=dst[order].astype(np.int32))


def max_window_points(points: np.ndarray, keep: np.ndarray, lo: int, hi: int, patch: int) -> int:
    """Most points (where keep) inside any inclusive window [x0, x0 + patch] x [y0, y0 + patch] with integer
    origins x0, y0 in [lo, hi]: the candidate capacity of a patch."""
    if hi < lo:
        return 0
    p = points[keep]
    # a point counts for the origins ceil(v - patch) .. floor(v) on each axis
    ax0, ax1 = np.ceil(p[:, 0] - patch), np.floor(p[:, 0])
    ay0, ay1 = np.ceil(p[:, 1] - patch), np.floor(p[:, 1])
    ax0, ay0 = np.maximum(ax0, lo), np.maximum(ay0, lo)
    ax1, ay1 = np.minimum(ax1, hi), np.minimum(ay1, hi)
    ok = (ax0 <= ax1) & (ay0 <= ay1)
    if not ok.any():
        return 0
    n = hi - lo + 2
    grid = np.zeros((n, n), dtype=np.int64)
    x0, x1 = (ax0[ok] - lo).astype(np.int64), (ax1[ok] - lo + 1).astype(np.int64)
    y0, y1 = (ay0[ok] - lo).astype(np.int64), (ay1[ok] - lo + 1).astype(np.int64)
    np.add.at(grid, (y0, x0), 1)
    np.add.at(grid, (y0, x1), -1)
    np.add.at(grid, (y1, x0), -1)
    np.add.at(grid, (y1, x1), 1)
    return int(grid.cumsum(0).cumsum(1).max())


# ---- dataset layout (dataset.py:21-67, 306-400) ---------------------------------------------------------------

def cityscale_data_partition():
    train, test, val = [], [], []
    for x in range(180):
        if x % 10 < 8:
            train.append(x)
        if x % 10 == 9:
            test.append(x)
        if x % 20 == 18:
            val.append(x)
        if x % 20 == 8:
            test.append(x)
    return train, val, test


def spacenet_data_partition():
    with open("./spacenet/data_split.json", "r") as jf:
        split = json.load(jf)
    return split["train"], split["validation"], split["test"]


def get_patch_info_one_img(image_index, image_size, sample_margin, patch_size, patches_per_edge):
    """[(image_index, (x0, y0), (x1, y1))] of the evaluation grid (dataset.py:56-67)."""
    grid = [round(x) for x in np.linspace(sample_margin, image_size - (patch_size + sample_margin),
                                          num=patches_per_edge)]
    return [(image_index, (x, y), (x + patch_size, y + patch_size)) for x in grid for y in grid]


def cityscale_transform(v):
    return v[:, ::-1]


def spacenet_transform(v):
    return np.stack([v[:, 1], 400 - v[:, 0]], axis=1)


LAYOUTS = {
    "cityscale": dict(image_size=2048, margin=64, partition=cityscale_data_partition, transform=cityscale_transform,
                      rgb="./cityscale/20cities/region_{}_sat.png",
                      keypoint="./cityscale/processed/keypoint_mask_{}.png",
                      road="./cityscale/processed/road_mask_{}.png",
                      graph="./cityscale/20cities/region_{}_refine_gt_graph.p"),
    "spacenet": dict(image_size=400, margin=0, partition=spacenet_data_partition, transform=spacenet_transform,
                     rgb="./spacenet/RGB_1.0_meter/{}__rgb.png",
                     keypoint="./spacenet/processed/keypoint_mask_{}.png",
                     road="./spacenet/processed/road_mask_{}.png",
                     graph="./spacenet/RGB_1.0_meter/{}__gt_graph.p"),
}


def _cfg(config, key):
    v = config.get(key) if isinstance(config, dict) else getattr(config, key, None)
    if v is None or (isinstance(v, dict) and len(v) == 0):
        raise ValueError(f"config has no {key}")
    return v


def _positive_int(config, key, lo=1, hi=None) -> int:
    v = _cfg(config, key)
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        raise ValueError(f"{key} must be an integer in [{lo}, {hi if hi is not None else 'inf'}] (got {v!r})")
    return int(v)


def _positive_float(config, key) -> float:
    v = _cfg(config, key)
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(v) \
            or v <= 0:
        raise ValueError(f"{key} must be a positive number (got {v!r})")
    return float(v)


def label_config(config, image_size: int, margin: int) -> Dict:
    """The configuration keys the batches use, checked: PATCH_SIZE, TOPO_SAMPLE_NUM, MAX_NEIGHBOR_QUERIES
    (1..32), ROAD_NMS_RADIUS, NEIGHBOR_RADIUS (its BFS depth NEIGHBOR_RADIUS // 4 must fit an int32).  Raises
    ValueError without touching a GPU."""
    c = dict(P=_positive_int(config, "PATCH_SIZE"), S=_positive_int(config, "TOPO_SAMPLE_NUM"),
             Np=_positive_int(config, "MAX_NEIGHBOR_QUERIES", 1, 32),
             r_nms=_positive_float(config, "ROAD_NMS_RADIUS"), r_nbr=_positive_float(config, "NEIGHBOR_RADIUS"))
    if c["r_nbr"] // SUBDIVIDE_RESOLUTION > 2 ** 31 - 1:
        raise ValueError(f"NEIGHBOR_RADIUS {c['r_nbr']!r} gives a BFS depth NEIGHBOR_RADIUS // "
                         f"{SUBDIVIDE_RESOLUTION} beyond 2**31 - 1")
    if c["P"] + 2 * margin > image_size:
        raise ValueError(f"PATCH_SIZE {c['P']} with margin {margin} does not fit a {image_size}-pixel scene")
    return c


def _read_rgb(path):
    import cv2
    bgr = cv2.imread(path)
    if bgr is None:
        raise FileNotFoundError(path)
    return cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)


def _read_gray(path):
    import cv2
    img = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
    if img is None:
        raise FileNotFoundError(path)
    return img


class LabelScenes:
    """The device side of a dataset: a samroad_labels object holding every scene (include/samroad_b200.h)."""

    def __init__(self, lc: Dict, image_size: int, margin: int, max_patch_points: int, device):
        from . import _lib
        import torch
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise RuntimeError(f"batches are generated on CUDA (sm_90a) only; got '{self.device}'")
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        self.lc, self.image_size, self.margin, self.cap = lc, image_size, margin, max(1, int(max_patch_points))
        cfg = _lib.SamRoadLabelCfg(lc["P"], image_size, margin, lc["S"], lc["Np"], self.cap, lc["r_nms"],
                                   lc["r_nbr"])
        self._h = _lib.Handle("samroad_labels_create", "samroad_labels_destroy", idx, C.byref(cfg))
        self.n_scenes = 0

    def __getstate__(self):
        raise TypeError("LabelScenes holds device state and cannot be copied or pickled")

    def close(self) -> None:
        self._h.close()

    def upload(self, scene: SceneLabels, rgb: np.ndarray, keypoint_mask: np.ndarray, road_mask: np.ndarray) -> int:
        from . import _lib
        S = self.image_size
        if rgb.shape != (S, S, 3) or keypoint_mask.shape != (S, S) or road_mask.shape != (S, S):
            raise ValueError(f"scene images must be [{S},{S},3] / [{S},{S}] (got {rgb.shape}, "
                             f"{keypoint_mask.shape}, {road_mask.shape})")
        arrs = [np.ascontiguousarray(a, dtype=t) for a, t in (
            (rgb, np.uint8), (keypoint_mask, np.uint8), (road_mask, np.uint8), (scene.points, np.float64),
            (scene.flags, np.uint8), (scene.weights, np.float32), (scene.adj_start, np.int32), (scene.adj, np.int32))]
        ptrs = [a.ctypes.data_as(C.c_void_p) for a in arrs]
        out = C.c_int32()
        _lib.check(_lib.load().samroad_labels_upload(self._h, ptrs[0], ptrs[1], ptrs[2], int(scene.points.shape[0]),
                                                     ptrs[3], ptrs[4], ptrs[5], ptrs[6], ptrs[7], C.byref(out)),
                   "samroad_labels_upload")
        self.n_scenes += 1
        return out.value

    def batch(self, B: int, patches=None, seed: Optional[int] = None, draws: Optional[Dict] = None,
              export_draws: bool = False):
        """One collated batch of B patches (dict of device tensors, graph_collate_fn's layout).  patches: [B,4]
        int32 (scene, x0, y0, rot) or None to draw them; seed: 62-bit Philox key (None: from torch's default
        generator).  Test hooks: draws = {"patches", "score_u", "source_u", "noise"} arrays are used instead of
        drawing; export_draws=True draws everything and returns (batch, draws).  A drawn seed is made per rank
        under torch.distributed (ranks.rank_seed; rank 0 keeps it)."""
        import torch
        from . import _lib
        lc, dev = self.lc, self.device
        P, S, Np = lc["P"], lc["S"], lc["Np"]
        f32 = dict(dtype=torch.float32, device=dev)
        rgb = torch.empty((B, P, P, 3), **f32)
        kp = torch.empty((B, P, P), **f32)
        road = torch.empty((B, P, P), **f32)
        pts = torch.empty((B * self.cap * 2,), **f32)
        pairs = torch.empty((B, S, Np, 2), dtype=torch.int32, device=dev)
        conn = torch.empty((B, S, Np), dtype=torch.bool, device=dev)
        valid = torch.empty((B, S, Np), dtype=torch.bool, device=dev)
        n_out = C.c_int32()
        outs = (rgb.data_ptr(), kp.data_ptr(), road.data_ptr(), pts.data_ptr(), pairs.data_ptr(), conn.data_ptr(),
                valid.data_ptr(), C.byref(n_out))
        want = {"patches": ((B, 4), torch.int32), "score_u": ((B, self.cap), torch.float64),
                "source_u": ((B, S), torch.float64), "noise": ((B, self.cap, 2), torch.float64)}
        if seed is None:
            from .ranks import draw_seed
            seed = draw_seed()
        seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        lib = _lib.load()
        with torch.cuda.device(dev):
            stream = _lib.current_stream_ptr()
            if draws is not None or export_draws:
                if draws is not None:
                    d = {k: torch.as_tensor(np.ascontiguousarray(v)).to(dev) for k, v in draws.items()}
                    for k, (shape, dt) in want.items():
                        if k not in d or tuple(d[k].shape) != shape or d[k].dtype != dt:
                            raise ValueError(f"draws[{k!r}] must be {dt} {shape}")
                else:
                    d = {k: torch.empty(shape, dtype=dt, device=dev) for k, (shape, dt) in want.items()}
                _lib.check(lib.samroad_debug_labels_batch_draws(
                    self._h, B, 0 if draws is not None else 1, seed, d["patches"].data_ptr(), d["score_u"].data_ptr(),
                    d["source_u"].data_ptr(), d["noise"].data_ptr(), *outs, stream), "samroad_debug_labels_batch_draws")
            else:
                pt = None
                if patches is not None:
                    pt = torch.as_tensor(np.ascontiguousarray(patches, dtype=np.int32)).reshape(B, 4).to(dev)
                _lib.check(lib.samroad_labels_batch(self._h, B, seed, None if pt is None else pt.data_ptr(), *outs,
                                                    stream), "samroad_labels_batch")
        N = n_out.value
        out = {"rgb": rgb, "keypoint_mask": kp, "road_mask": road, "graph_points": pts[:B * N * 2].view(B, N, 2),
               "pairs": pairs, "connected": conn, "valid": valid}
        return (out, d) if export_draws else out


class SatMapDataset:
    """SatMapDataset(config, is_train, dev_run=False) of dataset.py:306-400 whose batches are generated on the
    device: same file layout, partitions, coordinate transforms, IMAGE_SIZE / SAMPLE_MARGIN, dev_run slicing,
    eval patches and __len__.  Iterate `ds.loader(batch_size)`; samples are not served one by one."""

    def __init__(self, config, is_train, dev_run=False, device=None):
        self.config = config
        dataset = _cfg(config, "DATASET")
        if dataset not in LAYOUTS:
            raise ValueError(f"DATASET must be 'cityscale' or 'spacenet' (got {dataset!r})")
        lay = LAYOUTS[dataset]
        self.dataset = dataset
        self.IMAGE_SIZE, self.SAMPLE_MARGIN = lay["image_size"], lay["margin"]
        self.lc = label_config(config, self.IMAGE_SIZE, self.SAMPLE_MARGIN)
        self.is_train = bool(is_train)
        train, val, test = lay["partition"]()
        tile_indices = (train + val) if self.is_train else test
        self.tile_indices = tile_indices
        if dev_run:
            tile_indices = tile_indices[:4]
        self.sample_min = self.SAMPLE_MARGIN
        self.sample_max = self.IMAGE_SIZE - (self.lc["P"] + self.SAMPLE_MARGIN)
        scenes, images = [], []
        for tile_idx in tile_indices:
            print(f"loading tile {tile_idx}")
            with open(lay["graph"].format(tile_idx), "rb") as f:
                adj = pickle.load(f)
            if len(adj) == 0:
                print(f"===== skipped empty tile {tile_idx} =====")
                continue
            images.append((_read_rgb(lay["rgb"].format(tile_idx)), _read_gray(lay["keypoint"].format(tile_idx)),
                           _read_gray(lay["road"].format(tile_idx))))
            scenes.append(precompute_scene(adj, lay["transform"]))
        if not scenes:
            raise ValueError("no scene with a non-empty ground-truth graph")
        cap = max(max_window_points(s.points, ~s.excluded, self.sample_min, self.sample_max, self.lc["P"])
                  for s in scenes)
        self._scenes = LabelScenes(self.lc, self.IMAGE_SIZE, self.SAMPLE_MARGIN, cap, device)
        for s, (rgb, kp, road) in zip(scenes, images):
            self._scenes.upload(s, rgb, kp, road)
        self.scenes = scenes
        if not self.is_train:
            per_edge = math.ceil((self.IMAGE_SIZE - 2 * self.SAMPLE_MARGIN) / self.lc["P"])
            self.eval_patches = []
            for i in range(len(tile_indices)):   # as dataset.py:387-390: indices over the tiles, skipped or not
                self.eval_patches += get_patch_info_one_img(i, self.IMAGE_SIZE, self.SAMPLE_MARGIN, self.lc["P"],
                                                            per_edge)

    @property
    def device(self):
        return self._scenes.device

    def __len__(self):
        if self.is_train:
            if self.dataset == "cityscale":
                return max(1, int(self.IMAGE_SIZE / self.lc["P"])) ** 2 * 2500
            return 84667
        return len(self.eval_patches)

    def __getitem__(self, idx):
        import torch.utils.data
        where = "a DataLoader worker" if torch.utils.data.get_worker_info() is not None else "__getitem__"
        raise RuntimeError(f"sam_road_b200.dataset.SatMapDataset builds whole batches on the GPU and cannot serve "
                           f"single samples to {where}; iterate `ds.loader(batch_size)` instead of wrapping the "
                           f"dataset in a torch DataLoader")

    def __getstate__(self):
        raise TypeError("sam_road_b200.dataset.SatMapDataset holds device state and cannot be pickled (e.g. into "
                        "DataLoader worker processes); iterate `ds.loader(batch_size)` instead")

    def patches(self, first: int, count: int) -> np.ndarray:
        """[count, 4] int32 (scene, x0, y0, rot 0) of eval patches first .. first + count - 1."""
        return self.patches_at(range(first, first + count))

    def patches_at(self, indices) -> np.ndarray:
        """[len(indices), 4] int32 (scene, x0, y0, rot 0) of the eval patches at `indices`."""
        out = np.zeros((len(indices), 4), dtype=np.int32)
        for k, i in enumerate(indices):
            img, (x0, y0), _ = self.eval_patches[i]
            out[k, :3] = (img, x0, y0)
        return out

    def batch(self, batch_size: int, first: int = 0, seed: Optional[int] = None) -> Dict:
        """One batch: training draws its patches; evaluation takes eval patches first .. first + batch_size - 1."""
        if self.is_train:
            return self._scenes.batch(batch_size, seed=seed)
        return self._scenes.batch(batch_size, patches=self.patches(first, batch_size), seed=seed)

    def loader(self, batch_size: int) -> "BatchLoader":
        return BatchLoader(self, batch_size)


def eval_shard(n: int, rank: int, world: int) -> np.ndarray:
    """Indices of rank `rank` of `world` into n samples, as DistributedSampler(shuffle=False, drop_last=False)
    gives them: the list 0 .. n-1 is padded to ceil(n / world) * world by repeating it from its start, and the
    rank takes every world-th index from `rank` on."""
    if not 0 <= rank < world:
        raise ValueError(f"rank {rank} is not in [0, {world})")
    per_rank = -(-n // world)
    return np.resize(np.arange(n, dtype=np.int64), per_rank * world)[rank::world]


class BatchLoader:
    """Re-iterable batches of a SatMapDataset, already collated on the device.  The last batch is short when B
    does not divide the sample count, as DataLoader(drop_last=False) makes it.

    In one process len() is ceil(len(ds) / B).  Under torch.distributed each rank gets what Lightning's
    DistributedSampler would give it: ceil(len(ds) / world) samples, so len() is ceil(ceil(len(ds) / world) / B);
    evaluation takes this rank's eval_shard of the patch list, in order; training draws its own patches (the
    seeds differ per rank, LabelScenes.batch)."""

    def __init__(self, ds: SatMapDataset, batch_size: int):
        if isinstance(batch_size, bool) or not isinstance(batch_size, (int, np.integer)) or batch_size < 1:
            raise ValueError(f"batch_size must be a positive integer (got {batch_size!r})")
        self.ds, self.batch_size = ds, int(batch_size)

    def _samples(self) -> int:
        from .ranks import rank_and_world
        return -(-len(self.ds) // rank_and_world()[1])

    def __len__(self):
        return (self._samples() + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        from .ranks import rank_and_world
        B = self.batch_size
        if self.ds.is_train:
            n = self._samples()
            for first in range(0, n, B):
                yield self.ds.batch(min(B, n - first))
            return
        idx = eval_shard(len(self.ds), *rank_and_world())
        for first in range(0, len(idx), B):
            rows = self.ds.patches_at(idx[first:first + B])
            yield self.ds._scenes.batch(rows.shape[0], patches=rows)
