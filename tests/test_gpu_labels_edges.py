"""GPU: batch generation (csrc/labels.cu) at its limits, against the numpy oracle (oracle/label_oracle.py,
ties="index") on hand-built scenes with injected draws: window capacity at the shared-memory limit, PATCH_SIZE 1024,
non-default radii, odd sample counts, draw boundaries, the BFS size limit, coincident survivors, one object across
batch sizes and the upload refusals.  Each case's docstring names the labels.cu path it reaches."""
import math
import os

import cv2
import numpy as np
import pytest
import torch

from oracle import label_oracle as LO
from sam_road_b200 import synth
from sam_road_b200 import dataset as D

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


# ---- helpers ----------------------------------------------------------------------------------------------------

def _lc(P=256, S=5, Np=4, r_nms=16.0, r_nbr=64.0):
    return dict(P=P, S=S, Np=Np, r_nms=float(r_nms), r_nbr=float(r_nbr))


def _scene(points, immune=None, excluded=None, weights=None, adj=None) -> D.SceneLabels:
    """A SceneLabels from explicit points [n,2], flags, weights (default 0.1) and adjacency lists (default none)."""
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 2)
    n = pts.shape[0]
    immune = np.zeros(n, bool) if immune is None else np.asarray(immune, bool)
    excluded = np.zeros(n, bool) if excluded is None else np.asarray(excluded, bool)
    weights = np.full(n, 0.1, np.float32) if weights is None else np.asarray(weights, np.float32)
    adj = [[] for _ in range(n)] if adj is None else adj
    start = np.zeros(n + 1, np.int32)
    start[1:] = np.cumsum([len(a) for a in adj])
    flat = np.array([v for a in adj for v in a], dtype=np.int32)
    edges = np.array([(u, v) for u, a in enumerate(adj) for v in a if u <= v], dtype=np.int64).reshape(-1, 2)
    return D.SceneLabels(points=pts, edges=edges, crossovers=np.zeros((0, 2)), excluded=excluded,
                         nms_override=np.where(immune, 2.0, 0.0).astype(np.float32), weights=weights,
                         adj_start=start, adj=flat)


def _link(adj, a, b):
    adj[a].append(b)
    adj[b].append(a)


def _images(size, seed):
    rng = np.random.RandomState(seed)
    return (rng.randint(0, 256, (size, size, 3)).astype(np.uint8), rng.randint(0, 256, (size, size)).astype(np.uint8),
            rng.randint(0, 256, (size, size)).astype(np.uint8))


class Labels:
    """A LabelScenes with the host copies the oracle needs."""

    def __init__(self, lc, size, margin, cap, scenes, images=None):
        self.lc, self.size, self.margin = lc, size, margin
        self.ls = D.LabelScenes(lc, size, margin, cap, DEV)
        self.scenes, self.images = [], []
        for k, sc in enumerate(scenes):
            self.upload(sc, images[k] if images is not None else _images(size, 50 + k))

    def upload(self, sc, imgs):
        idx = self.ls.upload(sc, *imgs)
        assert idx == len(self.scenes)
        self.scenes.append(sc)
        self.images.append(imgs)

    def candidates(self, patch):
        scene, x0, y0, _ = (int(v) for v in patch)
        sc = self.scenes[scene]
        return LO.candidates(sc.points, sc.excluded, x0, y0, self.lc["P"], "index")

    def draws(self, patches, seed=0, score_u=None, source_u=None):
        """Random draws for patches [B,4]; score_u / source_u: per-patch callables (rows) overriding them."""
        rng = np.random.RandomState(seed)
        patches = np.asarray(patches, np.int32).reshape(-1, 4)
        B, cap, S = patches.shape[0], self.ls.cap, self.lc["S"]
        d = dict(patches=patches, score_u=rng.rand(B, cap), source_u=rng.rand(B, S), noise=rng.randn(B, cap, 2))
        for i in range(B):
            if score_u is not None:
                score_u(i, d["score_u"][i])
            if source_u is not None:
                source_u(i, d["source_u"][i])
        return d

    def oracle(self, patch, score_u, source_u, noise):
        scene, x0, y0, rot = (int(v) for v in patch)
        m = self.candidates(patch).shape[0]
        draws = dict(score=0.9 + (1.0 - 0.9) * np.asarray(score_u[:m]), source_u=source_u, noise=noise)
        return LO.sample_patch(self.scenes[scene], x0, y0, rot, self.lc, draws, ties="index")

    def run(self, draws):
        return self.ls.batch(np.asarray(draws["patches"]).shape[0], draws=draws)

    def check(self, draws, batch=None):
        """Device batch == oracle on the same draws: points bit for bit, pairs / valid / connected, crops."""
        batch = self.run(draws) if batch is None else batch
        b = {k: v.cpu().numpy() for k, v in batch.items()}
        B, N = b["graph_points"].shape[:2]
        P, outs = self.lc["P"], []
        for i in range(B):
            o = self.oracle(draws["patches"][i], draws["score_u"][i], draws["source_u"][i], draws["noise"][i])
            n = o["points"].shape[0]
            assert n <= N
            assert np.array_equal(b["graph_points"][i, :n].view(np.uint32), o["points"].view(np.uint32)), i
            assert not b["graph_points"][i, n:].any()
            for k in ("pairs", "valid", "connected"):
                assert np.array_equal(b[k][i], o[k]), (i, k)
            scene, x0, y0, rot = (int(v) for v in draws["patches"][i])
            rgb, kp, road = self.images[scene]
            assert np.array_equal(b["rgb"][i], LO.crop(rgb, x0, y0, P, rot).astype(np.float32)), i
            assert np.array_equal(b["keypoint_mask"][i], LO.crop(kp, x0, y0, P, rot).astype(np.float32) / np.float32(255))
            assert np.array_equal(b["road_mask"][i], LO.crop(road, x0, y0, P, rot).astype(np.float32) / np.float32(255))
            outs.append(o)
        assert N == max(o["points"].shape[0] for o in outs)
        return batch, outs


def _source_u_for(weights, want):
    """source_u picking survivor indices `want` (midpoints of their running-sum intervals)."""
    cdf = np.cumsum(np.asarray(weights, np.float64))
    lo = np.concatenate([[0.0], cdf[:-1]])
    return np.array([(lo[i] + cdf[i]) / 2.0 / cdf[-1] for i in want])


def _road_scene(extent, seed=0, spacing=48):
    return D.precompute_scene(synth.make_road_graph(extent, seed=seed, spacing=spacing), D.cityscale_transform)


# ---- 1. window capacity at the shared-memory limit -------------------------------------------------------------

def test_window_capacity_at_shared_memory_limit():
    """patch_kernel with max_patch_points = 8192, the most the H100's opt-in shared memory admits
    (patch_smem_bytes(8192) = 221 712 B): a window with 8192 non-excluded candidates runs the full 8192-slot
    bitonic sort and the 33 x 33 cell grid (cell = P/32 = 8 > ROAD_NMS_RADIUS) and equals the oracle.  8193
    (287 258 B) is refused by samroad_labels_create before any batch."""
    with pytest.raises(RuntimeError, match=r"holds up to 8193 labelled points.*shared memory"):
        D.LabelScenes(_lc(), 320, 0, 8193, DEV)
    rng = np.random.RandomState(1)
    x0 = y0 = 32
    gx, gy = np.meshgrid(np.arange(128) * 2.0 + 1.0, np.arange(64) * 4.0 + 2.0)
    pts = np.stack([gx.ravel(), gy.ravel()], 1) + rng.uniform(-0.7, 0.7, (8192, 2)) + [x0, y0]
    pts[:, 0] = np.clip(pts[:, 0], x0, x0 + 256)
    pts[:, 1] = np.clip(pts[:, 1], y0, y0 + 256)
    extra = np.array([[5.0, 5.0], [300.0, 310.0], [x0 - 0.5, y0 + 3]])          # outside the window
    pts = np.concatenate([pts, extra])
    n = pts.shape[0]
    adj = [[] for _ in range(n)]
    for r in range(64):                                                          # rows are paths
        for c in range(127):
            _link(adj, r * 128 + c, r * 128 + c + 1)
    immune = rng.rand(n) < 0.05
    lab = Labels(_lc(S=64, Np=16, r_nms=1.5, r_nbr=9.0), 320, 0, 8192,
                 [_scene(pts, immune=immune, weights=rng.choice([0.1, 0.9], n), adj=adj)])
    d = lab.draws([[0, x0, y0, 1]], seed=2)
    assert lab.candidates(d["patches"][0]).shape[0] == 8192
    _, outs = lab.check(d)
    assert 2000 < outs[0]["survivors"].shape[0] < 8192 and outs[0]["connected"].any()


# ---- 2. PATCH_SIZE 1024 ----------------------------------------------------------------------------------------

CFG_1024 = dict(DATASET="cityscale", PATCH_SIZE=1024, TOPO_SAMPLE_NUM=512, MAX_NEIGHBOR_QUERIES=16,
                NEIGHBOR_RADIUS=64, ROAD_NMS_RADIUS=16)


def test_patch_size_1024(tmp_path, monkeypatch):
    """toponet_vitb_1024's settings (S 512, Np 16, radii 16 / 64) on cityscale scenes with a street every 80
    pixels: P/32 = 32 is the NMS cell (wider than the radius), origins span [64, 960], rot 0-3 and the crops.  The
    bench's 48-pixel grid holds more candidates in its densest window than the shared memory admits: refused."""
    synth.write_label_scenes(str(tmp_path), "cityscale", (0, 1, 2, 3), 2048, seed=3, spacing=80)
    monkeypatch.chdir(tmp_path)
    ds = D.SatMapDataset(CFG_1024, is_train=True, dev_run=True, device=DEV)
    assert (ds.sample_min, ds.sample_max) == (64, 960) and ds._scenes.cap <= 8192
    lab = Labels.__new__(Labels)
    lab.lc, lab.ls, lab.scenes = ds.lc, ds._scenes, ds.scenes
    lab.images = []
    for t in (0, 1, 2, 3):
        p = lambda k: os.path.join(str(tmp_path), D.LAYOUTS["cityscale"][k].format(t))  # noqa: E731
        lab.images.append((cv2.cvtColor(cv2.imread(p("rgb")), cv2.COLOR_BGR2RGB),
                           cv2.imread(p("keypoint"), cv2.IMREAD_GRAYSCALE), cv2.imread(p("road"), cv2.IMREAD_GRAYSCALE)))
    d = lab.draws([[0, 64, 64, 0], [1, 960, 960, 1], [2, 64, 960, 2], [3, 517, 300, 3]], seed=4)
    _, outs = lab.check(d)
    assert min(o["survivors"].shape[0] for o in outs) > 200 and all(o["connected"].any() for o in outs)
    torch.manual_seed(5)
    batch, draws = ds._scenes.batch(2, export_draws=True)
    lab.check({k: v.cpu().numpy() for k, v in draws.items()}, batch)
    dense = _road_scene(2032, seed=0, spacing=48)
    cap = D.max_window_points(dense.points, ~dense.excluded, 64, 960, 1024)
    assert cap > 8192, cap
    with pytest.raises(RuntimeError, match=f"holds up to {cap} labelled points"):
        D.LabelScenes(ds.lc, 2048, 64, cap, DEV)


# ---- 3. non-default radii --------------------------------------------------------------------------------------

def _nms_scene(r, x0, y0, P):
    """Non-immune pairs at exactly r (3-4-5 offsets) and one float64 ulp inside / outside it, across a cell
    boundary, inside a cell, on the window's right edge x = x0 + P and bottom edge y = y0 + P; a chain A - B - C with
    |AB| = r, |BC| = 0.9 r, |AC| = 1.9 r.  prio: score_u per point (the first of each pair is visited first)."""
    cell = max(r, P / 32.0)
    pts, prio = [], []
    dx, dy = 0.6 * r, 0.8 * r
    assert dx * dx + dy * dy == r * r
    rows = (y0 + 20.0, y0 + 60.0, y0 + 100.0)
    for row, nudge in zip(rows, (0, 1, -1)):
        for ax in (x0 + 2 * cell - 3.0, x0 + 7 * cell + 0.5, x0 + P - dx):
            bx = ax + dx
            bx = bx if nudge == 0 else np.nextafter(bx, np.inf if nudge > 0 else -np.inf)
            pts += [(ax, row), (bx, row + dy)]
            prio += [0.99, 0.1]
    for ax in (x0 + 40.0, x0 + 100.0):                   # bottom edge
        pts += [(ax, y0 + P - dy), (ax + dx, y0 + P)]
        prio += [0.99, 0.1]
    cx, cy = x0 + 150.0, y0 + 150.0                     # chain
    pts += [(cx, cy), (cx + r, cy), (cx + 1.9 * r, cy)]
    prio += [0.99, 0.98, 0.97]
    rng = np.random.RandomState(int(r * 8))
    lone = rng.uniform(10, P - 10, (12, 2)) + [x0, y0]   # a few more, around y0 + 200
    lone[:, 1] = y0 + 190 + rng.uniform(0, 40, 12)
    pts += [tuple(v) for v in lone]
    prio += rng.uniform(0, 0.9, 12).tolist()
    return np.array(pts), np.array(prio)


def _knn_scene(r, x0, y0, P):
    """Immune survivors around a source S at the window centre: at exactly NEIGHBOR_RADIUS (out, strict), one ulp
    inside (in) and one ulp outside; 3-4-5 offsets where 0.6 r and 0.8 r are exact.  Targets in range are joined
    to S by paths of `depth` hops (reached) and `depth + 1` hops (not reached) through excluded points.  A second
    source far from everything has no target in range."""
    depth = int(r // 4)
    sx, sy = x0 + P / 2.0, y0 + P / 2.0
    pts = [(sx, sy), (sx + r, sy), (sx, np.nextafter(sy + r, -np.inf)), (np.nextafter(sx - r, -np.inf), sy),
           (sx - 0.7 * r, sy - 0.7 * r)]
    if (0.6 * r) ** 2 + (0.8 * r) ** 2 == r * r:
        pts += [(sx - 0.6 * r, sy + 0.8 * r), (sx + 0.6 * r, np.nextafter(sy + 0.8 * r, -np.inf))]
    pts.append((x0 + 3.0, y0 + 3.0))                     # lone source
    n0 = len(pts)
    adj = [[] for _ in range(n0)]
    excluded = [False] * n0

    def path(a, b, hops):
        prev = a
        for h in range(1, hops):
            pts.append((x0 + 1.0 + h, y0 + P - 1.0))
            adj.append([])
            excluded.append(True)
            _link(adj, prev, len(pts) - 1)
            prev = len(pts) - 1
        _link(adj, prev, b)

    path(0, 2, max(depth, 1))          # one ulp inside: reached (at depth 0 it is adjacent but not reached)
    path(0, 4, depth + 1)              # inside, one hop too far
    if n0 == 8:
        path(0, 6, max(depth, 1))
    n = len(pts)
    return _scene(pts, immune=[i < n0 for i in range(n)], excluded=excluded,
                  weights=np.linspace(0.2, 1.0, n), adj=adj), n0


@pytest.mark.parametrize("r_nms,r_nbr", [(16.0, 30.0), (16.0, 4.0), (16.0, 3.0), (10.0, 64.0), (12.5, 64.0)])
def test_non_default_radii(r_nms, r_nbr):
    """patch_kernel's NMS with the cell equal to ROAD_NMS_RADIUS (10, 12.5: floor((x - x0) / cell) inexact) and the
    clamped last cell row / column; pairs_kernel's strict kNN test `d < r_nbr2` and the BFS depth floor(r / 4) at
    NEIGHBOR_RADIUS 30 (depth 7), 4 (depth 1) and 3 (depth 0: nothing is expanded); Np 4, S 5 (the tail warp of
    the last pairs_kernel block returns)."""
    P, x0, y0 = 256, 32, 32
    lc = _lc(P=P, S=5, Np=4, r_nms=r_nms, r_nbr=r_nbr)
    npts, prio = _nms_scene(r_nms, x0, y0, P)
    knn_scene, n0 = _knn_scene(r_nbr, x0, y0, P)
    lab = Labels(lc, 320, 16, 64, [_scene(npts, weights=np.full(len(npts), 0.5)), knn_scene])
    patches = [[0, x0, y0, 0], [1, x0, y0, 1], [0, x0, y0, 2], [1, x0, y0, 3]]

    cand0 = lab.candidates(patches[0])

    def score(i, row):
        if patches[i][0] == 0:
            row[:cand0.shape[0]] = prio[cand0]           # candidates are in ascending id

    # scene 1: sources S, S, the lone point, the one-ulp-inside point, S (survivors are the immune points in id order)
    want = [0, 0, n0 - 1, 2, 0]
    w1 = knn_scene.weights[:n0]

    def source(i, row):
        if patches[i][0] == 1:
            row[:] = _source_u_for(w1, want)

    d = lab.draws(patches, seed=int(r_nms + r_nbr), score_u=score, source_u=source)
    assert cand0.shape[0] == len(npts) - 1               # the right-edge point nudged one ulp out
    _, outs = lab.check(d)
    o0, o1 = outs[0], outs[1]
    kept = set(o0["survivors"].tolist())
    assert 0 in kept and 1 not in kept                  # exactly at ROAD_NMS_RADIUS: suppressed (inclusive)
    c = len(npts) - 15
    assert {c, c + 2} <= kept and c + 1 not in kept     # chain: C survives because B was suppressed
    assert np.array_equal(o1["sources"], want)
    tgt = {int(t) for t in o1["pairs"][0, o1["valid"][0], 1]}
    assert 1 not in tgt and 3 not in tgt and 2 in tgt   # at the radius: out; one ulp inside: in
    conn = dict(zip(o1["pairs"][0, :, 1].tolist(), o1["connected"][0].tolist()))
    assert conn[2] == (r_nbr >= 4) and not conn.get(4, False)
    assert not o1["valid"][2].any() and (o1["pairs"][2] == n0 - 1).all()   # lone source: all padding


# ---- 4. odd sample counts and tiny patches ---------------------------------------------------------------------

@pytest.mark.parametrize("S", [1, 3, 5, 513])
def test_odd_sample_counts_and_tiny_patches(S):
    """pairs_kernel with S not a multiple of kPairWarps (the last block's tail warps return), Np 32: a road-graph
    window, a one-point scene (every pair is (src, src) padding; its adjacency is empty, the upload's m == 0
    path), a window with fewer survivors than Np + 1, an empty window; then an all-empty batch, whose graph_points
    is [B, 1, 2] of zeros."""
    lc = _lc(P=128, S=S, Np=32, r_nms=16, r_nbr=64)
    road = _road_scene(200, seed=1)                      # spurs end before 248: the last window is empty
    few = _scene([(60.0, 60.0), (70.0, 60.0), (60.0, 75.0), (90.0, 90.0), (100.0, 40.0)], immune=[True] * 5,
                 weights=[0.3, 0.2, 0.9, 0.5, 0.1], adj=[[1], [0, 2], [1], [], []])
    one = _scene([(64.0, 64.0)], immune=[True], weights=[0.7])
    lab = Labels(lc, 384, 8, max(D.max_window_points(road.points, ~road.excluded, 8, 248, 128), 5),
                 [road, one, few])
    patches = [[0, 40, 60, 1], [1, 8, 8, 2], [2, 20, 20, 3], [0, 248, 248, 0]]
    d = lab.draws(patches, seed=S)
    batch, outs = lab.check(d)
    assert outs[0]["valid"].any() and outs[0]["connected"].any()
    assert outs[1]["survivors"].shape[0] == 1 and not outs[1]["valid"].any() and not outs[1]["pairs"].any()
    assert 1 < outs[2]["survivors"].shape[0] < 33 and outs[2]["valid"].sum(1).max() == 4
    assert outs[3]["survivors"].shape[0] == 0
    empty = lab.run(lab.draws([[0, 248, 248, 1], [2, 200, 200, 0]], seed=S + 1))
    assert empty["graph_points"].shape == (2, 1, 2) and not empty["graph_points"].any()
    assert not empty["valid"].any() and not empty["connected"].any() and not empty["pairs"].any()


# ---- 5. draw boundaries ----------------------------------------------------------------------------------------

def test_draw_boundaries():
    """patch_kernel step 6, `cdf[mid] > v`: power-of-two weights make the running sums exact, and source_u is
    exactly cdf[i] / total (the next survivor is chosen), 0 and nextafter(1, 0).  The sort key tie `ia < ib`:
    non-immune points with equal scores (all score_u equal, and u / nextafter(u) that round to one score) are
    visited by id, which decides who suppresses whom; and 300 immune points (score 2.0) in one window."""
    x0 = y0 = 16
    w = np.array([0.25, 0.5, 1.0, 0.25, 1.0, 0.5, 0.25, 0.25])        # sums to 4: u * total is exact
    ring = [(x0 + 20.0 + 25 * k, y0 + 20.0) for k in range(8)]
    # a shuffled chain of non-immune points 0.6 r apart (ids not in spatial order)
    rng = np.random.RandomState(7)
    order = rng.permutation(20)
    chain = [(x0 + 20.0 + 9.6 * order[k], y0 + 80.0) for k in range(20)]
    cluster = [(x0 + 10.0 + 11.0 * (k % 20), y0 + 120.0 + 11.0 * (k // 20)) for k in range(300)]
    pts = ring + chain + cluster
    immune = [True] * 8 + [False] * 20 + [True] * 300
    weights = np.concatenate([w, np.full(20, 0.5), np.full(300, 0.125)])
    lab = Labels(_lc(P=256, S=11, Np=4, r_nms=16, r_nbr=30), 300, 16, len(pts),
                 [_scene(pts, immune=immune, weights=weights), _scene(ring, immune=[True] * 8, weights=w)])
    cdf = np.cumsum(w)
    src_u = np.concatenate([[0.0], cdf[:-1] / 4.0, [np.nextafter(1.0, 0.0), 0.5, 0.25]])
    assert np.array_equal(src_u[1:8] * 4.0, cdf[:-1])
    u = 0.375
    k = 1.0 - 0.9
    assert 0.9 + k * u == 0.9 + k * np.nextafter(u, 1.0)                  # one score for both draws

    def score(i, row):
        if i == 0:
            row[:] = 0.5                                 # every score equal
        elif i == 1:
            row[:] = np.where(np.arange(row.shape[0]) % 2, np.nextafter(u, 1.0), u)

    def source(i, row):
        row[:] = src_u

    d = lab.draws([[0, x0, y0, 0], [0, x0, y0, 3], [1, x0, y0, 1]], seed=3, score_u=score, source_u=source)
    _, outs = lab.check(d)
    assert outs[2]["sources"].tolist() == [0, 1, 2, 3, 4, 5, 6, 7, 7, 4, 2]   # 0.5 * 4 = cdf[3]: the next one
    chain_kept = [i for i in outs[0]["survivors"].tolist() if 8 <= i < 28]
    assert chain_kept and chain_kept == sorted(chain_kept)          # visited, and kept, by ascending id
    assert outs[0]["survivors"].shape[0] == outs[1]["survivors"].shape[0]


# ---- 6. BFS at its size limit ----------------------------------------------------------------------------------

def _hub_scene(spokes, x0, y0, P, targets=True):
    """An immune hub at the window centre whose `spokes` neighbours lie outside the window, plus (targets) an
    immune target adjacent to it (counted among the spokes) and one that is not."""
    hx, hy = x0 + P / 2.0, y0 + P / 2.0
    pts = [(hx, hy)]
    adj = [[]]
    if targets:
        pts += [(hx + 10.0, hy), (hx, hy + 20.0)]
        adj += [[], []]
        _link(adj, 0, 1)
    outside = spokes - (1 if targets else 0)
    for k in range(outside):
        pts.append((x0 - 50.0 - (k % 40), y0 + (k // 40) * 3.0))
        adj.append([])
        _link(adj, 0, len(pts) - 1)
    n = len(pts)
    return _scene(pts, immune=[True] * n, adj=adj)


def test_bfs_size_limit_and_recovery():
    """pairs_kernel's BFS list (kBfsList = 1024): a hub with 1023 neighbours reaches exactly 1024 nodes and equals
    the oracle; with 1024 it is refused with the overflow message (labels.cu:677).  After that refusal and after a
    bad-patch refusal the next batch on the same object is correct.  A lone hub with 2000 neighbours and no target
    in range gives all-padding samples without walking.  Self-loops, duplicate adjacency entries, a degree-0 point
    and a one-point scene (empty adjacency, the upload's m == 0 path) equal the oracle."""
    P, x0, y0 = 128, 64, 64
    lc = _lc(P=P, S=6, Np=4, r_nms=4, r_nbr=64)
    small = [(100.0, 100.0), (104.0, 100.0), (108.0, 100.0), (112.0, 100.0), (100.0, 120.0), (130.0, 130.0)]
    adj = [[0, 1, 1], [0, 2, 0], [1, 3, 3, 2], [2, 2], [], [5]]     # self-loops, duplicates, degree 0
    loops = _scene(small, immune=[True] * 6, weights=[0.5, 0.25, 1.0, 0.5, 0.75, 0.1], adj=adj)
    lab = Labels(lc, 320, 64, 8, [_hub_scene(1023, x0, y0, P), _hub_scene(1024, x0, y0, P),
                                  _hub_scene(2000, x0, y0, P, targets=False), loops,
                                  _scene([(100.0, 100.0)], immune=[True], weights=[1.0])])
    zero = lambda i, row: row.__setitem__(slice(None), 0.0)  # noqa: E731  every source is survivor 0, the hub
    good = lab.draws([[0, x0, y0, 0], [2, x0, y0, 1], [3, x0, y0, 2], [4, x0, y0, 3]], seed=1, source_u=zero)
    good["source_u"][2] = np.random.RandomState(2).rand(6)
    ref, outs = lab.check(good)
    assert outs[0]["connected"][:, 0].all() and not outs[0]["connected"][:, 1].any()
    assert LO.bfs_reached(lab.scenes[0].adj_start, lab.scenes[0].adj, 0, [1, 2], 16).__len__() == 1024
    assert not outs[1]["valid"].any()                    # lone hub: padding, no walk
    assert outs[2]["connected"].any()
    with pytest.raises(RuntimeError, match=r"BFS reached more than 1024 nodes within NEIGHBOR_RADIUS // 4 = 16"):
        lab.run(lab.draws([[1, x0, y0, 0]], seed=1, source_u=zero))
    again = lab.run(good)
    for k in ref:
        assert torch.equal(ref[k], again[k]), k
    bad = lab.draws([[0, x0, y0, 0], [5, x0, y0, 0]], seed=1)
    with pytest.raises(RuntimeError, match="missing scene"):
        lab.run(bad)
    lab.check(good)


# ---- 7. coincident survivors -----------------------------------------------------------------------------------

def test_coincident_survivors():
    """pairs_kernel's kNN tie rule (distance, survivor index) at d = 0: two immune points at identical coordinates.
    From the twin with the larger survivor index, the nearest (dropped) is the other twin, so the source becomes a
    target of itself: a valid (src, src) pair, connected because the source is always reached."""
    pts = [(100.0, 100.0), (100.0, 100.0), (110.0, 100.0), (100.0, 130.0), (100.0, 100.0)]
    adj = [[2], [], [0, 3], [2], []]
    sc = _scene(pts, immune=[True, True, True, True, False], weights=[0.5, 0.5, 0.5, 0.5, 0.5], adj=adj)
    lab = Labels(_lc(P=128, S=5, Np=4, r_nms=8, r_nbr=64), 256, 0, 8, [sc])
    d = lab.draws([[0, 40, 40, 0], [0, 40, 40, 2]], seed=9,
                  source_u=lambda i, row: row.__setitem__(slice(None), _source_u_for(sc.weights[:4], [0, 1, 2, 1, 3])))
    _, outs = lab.check(d)
    o = outs[0]
    assert o["survivors"].tolist() == [0, 1, 2, 3]       # the non-immune twin is suppressed
    assert o["pairs"][1, 0].tolist() == [1, 1] and o["valid"][1, 0] and o["connected"][1, 0]
    assert o["pairs"][0, 0].tolist() == [0, 1] and o["valid"][0, 0] and not o["connected"][0, 0]


# ---- 8. one object across batch sizes --------------------------------------------------------------------------

def test_one_object_across_batch_sizes():
    """The work area: B = 2, 40, 5, 1 on one LabelScenes re-grows the work buffers and the pinned read-back once and
    then reuses them.  The status word is read with the survivor counts for every B up to the allocated one; each
    batch equals the oracle and a fresh object's batch, and a bad patch in a smaller batch is still refused."""
    lc = _lc(P=128, S=7, Np=8, r_nms=16, r_nbr=64)
    scenes = [_road_scene(300, seed=2), _road_scene(300, seed=3)]
    cap = max(D.max_window_points(s.points, ~s.excluded, 0, 172, 128) for s in scenes)
    lab = Labels(lc, 300, 0, cap, scenes)
    rng = np.random.RandomState(4)
    for B in (2, 40, 5, 1):
        patches = np.stack([rng.randint(0, 2, B), rng.randint(0, 173, B), rng.randint(0, 173, B),
                            rng.randint(0, 4, B)], 1)
        if B == 40:   # the counts after the first 5 / 1 patches are odd: a stale count read as status would refuse
            patches[5] = patches[1] = [0, 20, 20, 0]
            assert lab.candidates(patches[5]).shape[0] > 0
        d = lab.draws(patches, seed=B)
        got, outs = lab.check(d)
        if B == 40:
            n = outs[5]["survivors"].shape[0]
            assert n & (1 | 2 | 4), n
        fresh = Labels(lc, 300, 0, cap, scenes, lab.images)
        want = fresh.run(d)
        for k in want:
            assert torch.equal(got[k], want[k]), (B, k)
    with pytest.raises(RuntimeError, match="missing scene"):
        lab.run(lab.draws([[0, 0, 0, 0], [0, 1, 1, 1], [7, 0, 0, 0]], seed=1))
    lab.check(lab.draws([[1, 3, 4, 1]], seed=2))


# ---- 9. upload refusals ----------------------------------------------------------------------------------------

def _corrupt(sc, what):
    pts, w = sc.points.copy(), sc.weights.copy()
    start, adj = sc.adj_start.copy(), sc.adj.copy()
    n = pts.shape[0]
    if what == "negative weight":
        w[3] = -0.5
    elif what == "zero weights":
        w[:] = 0.0
    elif what == "nan point":
        pts[2, 1] = np.nan
    elif what == "start":
        start = start + 1
    elif what == "decreasing":
        start[2], start[3] = start[3], start[2]
        start[2] += 1
    elif what == "neighbour":
        adj[1] = n
    elif what == "empty":
        return D.SceneLabels(points=np.zeros((0, 2)), edges=np.zeros((0, 2), np.int64), crossovers=np.zeros((0, 2)),
                             excluded=np.zeros(0, bool), nms_override=np.zeros(0, np.float32),
                             weights=np.zeros(0, np.float32), adj_start=np.zeros(1, np.int32),
                             adj=np.zeros(0, np.int32))
    return D.SceneLabels(points=pts, edges=sc.edges, crossovers=sc.crossovers, excluded=sc.excluded,
                         nms_override=sc.nms_override, weights=w, adj_start=start, adj=adj)


@pytest.mark.parametrize("what,msg", [("negative weight", "weight 3 is not a positive finite number"),
                                      ("zero weights", "weight 0 is not a positive finite number"),
                                      ("nan point", "point 2 is not finite"),
                                      ("start", "offsets must start at 0"),
                                      ("decreasing", "offsets decrease at 2"),
                                      ("neighbour", "out of range"),
                                      ("empty", "at least one graph point")])
def test_upload_refusals(what, msg):
    """samroad_labels_upload's refusals (labels.cu:726-739), including the non-positive weights that would let the
    running sum pick the last survivor where the reference's np.random.choice raises: each names the defect,
    leaves n_scenes unchanged and the next batch equal to the one before."""
    sc = _road_scene(200, seed=4)
    lab = Labels(_lc(P=128, S=5, Np=4), 200, 0, D.max_window_points(sc.points, ~sc.excluded, 0, 72, 128), [sc])
    d = lab.draws([[0, 30, 40, 1], [0, 72, 0, 2]], seed=6)
    before, _ = lab.check(d)
    with pytest.raises(RuntimeError, match=msg):
        lab.ls.upload(_corrupt(sc, what), *lab.images[0])
    assert lab.ls.n_scenes == 1
    after = lab.run(d)
    for k in before:
        assert torch.equal(before[k], after[k]), k
    with pytest.raises(RuntimeError, match="missing scene"):
        lab.run(lab.draws([[1, 0, 0, 0]], seed=1))


# ---- the point transform where the reference's inverse is inexact ----------------------------------------------

def test_point_transform_at_inexact_patch_size():
    """points_kernel at P = 1488, where np.linalg.inv of the reference's float32 centring matrix is inexact
    (DESIGN.md §13): within one float32 ulp of the oracle, which uses the reference's matrix product."""
    P = 1488
    rng = np.random.RandomState(8)
    pts = rng.uniform(0, P, (900, 2)) + 8
    lab = Labels(_lc(P=P, S=3, Np=4, r_nms=1e-3, r_nbr=8), P + 16, 8, 900,
                 [_scene(pts, immune=np.ones(900, bool), weights=np.full(900, 0.5))],
                 [tuple(np.zeros(s, np.uint8) for s in ((P + 16, P + 16, 3), (P + 16, P + 16), (P + 16, P + 16)))])
    d = lab.draws([[0, 8, 8, r] for r in range(4)], seed=3)
    b = lab.run(d)
    got = b["graph_points"].cpu().numpy()
    for i in range(4):
        o = lab.oracle(d["patches"][i], d["score_u"][i], d["source_u"][i], d["noise"][i])
        n = o["points"].shape[0]
        assert n == 900
        a, e = got[i, :n], o["points"]
        assert (np.abs(a - e) <= np.spacing(np.maximum(np.abs(a), np.abs(e)))).all(), i
        for k in ("pairs", "valid", "connected"):
            assert np.array_equal(b[k][i].cpu().numpy(), o[k]), (i, k)
    assert math.isclose(float(np.abs(got).max()), P, rel_tol=0.01)
