"""NumPy restatement of GraphLabelGenerator.sample_patch (dataset.py:127-231) and the crop / rot90 of
SatMapDataset.__getitem__ (dataset.py:402-445) with injected draws: the checker of csrc/labels.cu.

The reference draws from NumPy's global generator; here every draw is an argument:
  score      U(0.9, 1) per candidate, in the candidate order of the mode (see `candidates`)
  source_index / source_u
             the sources as indices into the NMS survivors (what np.random.choice returned), or one U[0,1)
             each, turned into an index by the device's rule: the first survivor whose running weight sum
             exceeds u * total (float64, summed in survivor order)
  noise      [N, 2] N(0, 1), added to the transformed points

ties="scipy" is the reference verbatim: candidates in `list(set)` order, NMS visit order from
`np.argsort(scores)[::-1]`, scipy's ball query and kNN (cKDTree's order among equidistant neighbours).
ties="index" pins what the reference leaves open, as the device does: candidates in ascending id, visit by
(score descending, candidate position ascending), neighbours by (distance, survivor index)."""
from __future__ import annotations

from collections import deque
from typing import Dict, Optional

import numpy as np

SUBDIVIDE_RESOLUTION = 4


def candidates(points: np.ndarray, excluded: np.ndarray, x0: int, y0: int, patch: int, ties: str) -> np.ndarray:
    """Subdivided-point ids inside the inclusive box [x0, x0+P] x [y0, y0+P] that are not excluded."""
    x, y = points[:, 0], points[:, 1]
    ids = np.nonzero((x >= x0) & (x <= x0 + patch) & (y >= y0) & (y <= y0 + patch))[0]
    if ties == "scipy":   # the reference's set difference and list(set) order (dataset.py:130-134)
        return np.array(list(set(ids.tolist()) - set(np.nonzero(excluded)[0].tolist())), dtype=np.int64)
    return ids[~excluded[ids]]


def nms(pts: np.ndarray, scores: np.ndarray, radius: float, ties: str) -> np.ndarray:
    """Indices into pts of the survivors in visiting order (graph_utils.py:572-591): a visited survivor
    suppresses every point within radius (inclusive) whose score is not above 1."""
    n = pts.shape[0]
    if ties == "scipy":
        import scipy.spatial
        order = np.argsort(scores)[::-1]
        sp = pts[order]
        tree = scipy.spatial.KDTree(sp)
        kept = np.ones(n, dtype=bool)
        for i in range(n):
            if not kept[i]:
                continue
            nb = tree.query_ball_point(sp[i], r=radius)
            kept[nb] = scores[order][nb] > 1.0
            kept[i] = True
        return order[kept]
    order = np.lexsort((np.arange(n), -scores))
    sp, ss = pts[order], scores[order]
    kept = np.ones(n, dtype=bool)
    r2 = float(radius) * float(radius)
    for i in range(n):
        if not kept[i]:
            continue
        d2 = (sp[:, 0] - sp[i, 0]) ** 2 + (sp[:, 1] - sp[i, 1]) ** 2
        sup = (d2 <= r2) & (ss <= 1.0)
        sup[:i + 1] = False
        kept[sup] = False
    return order[kept]


def choose_sources(weights: np.ndarray, draws: Dict) -> np.ndarray:
    if "source_index" in draws:
        return np.asarray(draws["source_index"], dtype=np.int64)
    cdf = np.cumsum(weights.astype(np.float64))
    v = np.asarray(draws["source_u"], dtype=np.float64) * cdf[-1]
    return np.minimum(np.searchsorted(cdf, v, side="right"), weights.shape[0] - 1)


def knn(pts: np.ndarray, queries: np.ndarray, k: int, radius: float, ties: str) -> np.ndarray:
    """[len(queries), k] indices into pts of the k nearest strictly inside radius, ascending; pts.shape[0]
    where fewer exist (scipy's convention)."""
    n = pts.shape[0]
    if ties == "scipy":
        import scipy.spatial
        _, idx = scipy.spatial.KDTree(pts).query(queries, k=k, distance_upper_bound=radius)
        return np.asarray(idx).reshape(len(queries), k)
    out = np.full((len(queries), k), n, dtype=np.int64)
    r2 = float(radius) * float(radius)
    for q in range(len(queries)):
        d2 = (pts[:, 0] - queries[q, 0]) ** 2 + (pts[:, 1] - queries[q, 1]) ** 2
        cand = np.nonzero(d2 < r2)[0]
        cand = cand[np.lexsort((cand, d2[cand]))][:k]
        out[q, :cand.shape[0]] = cand
    return out


def bfs_reached(adj_start: np.ndarray, adj: np.ndarray, source: int, stops, max_depth) -> set:
    """Nodes a breadth-first walk from source visits when it expands no stop node and nothing at depth
    max_depth (graph_utils.py:594-630)."""
    stops = set(stops)
    seen = {source}
    queue = deque([(source, 0)])
    while queue:
        u, d = queue.popleft()
        if u in stops or d >= max_depth:
            continue
        for v in adj[adj_start[u]:adj_start[u + 1]].tolist():
            if v not in seen:
                seen.add(v)
                queue.append((v, d + 1))
    return seen


def transform_points(pts: np.ndarray, x0: int, y0: int, patch: int, rot: int, noise: np.ndarray) -> np.ndarray:
    """Patch coordinates, rot90 about the patch centre (dataset.py:207-229), plus noise, in float64."""
    p = pts - np.array([x0, y0])[np.newaxis, :]
    p = np.concatenate([p, np.ones((p.shape[0], 1), dtype=p.dtype)], axis=1)
    trans = np.array([[1, 0, -0.5 * patch], [0, 1, -0.5 * patch], [0, 0, 1]], dtype=np.float32)
    rotm = np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1]], dtype=np.float32)
    p = p @ trans.T @ np.linalg.matrix_power(rotm.T, rot) @ np.linalg.inv(trans.T)
    return p[:, :2] + noise


def sample_patch(scene, x0: int, y0: int, rot: int, cfg: Dict, draws: Dict, ties: str = "index") -> Dict:
    """One sample of GraphLabelGenerator.sample_patch.  scene: sam_road_b200.dataset.SceneLabels (or anything
    with points / excluded / nms_override / weights / adj_start / adj).  cfg: P, S, Np, r_nms, r_nbr.
    Returns points [N,2] float32, pairs [S,Np,2] int32, connected / valid [S,Np] bool, and for inspection the
    candidate ids, the survivors' ids in visiting order and the source indices."""
    P, S, Np = cfg["P"], cfg["S"], cfg["Np"]
    cand = candidates(scene.points, scene.excluded, x0, y0, P, ties)
    if cand.shape[0] == 0:
        return dict(points=np.zeros((1, 2), np.float32), pairs=np.zeros((S, Np, 2), np.int32),
                    connected=np.zeros((S, Np), bool), valid=np.zeros((S, Np), bool), candidates=cand,
                    survivors=np.zeros(0, np.int64), sources=np.zeros(0, np.int64))
    scores = np.maximum(np.asarray(draws["score"], dtype=np.float64)[:cand.shape[0]],
                        scene.nms_override[cand])
    keep = nms(scene.points[cand], scores, cfg["r_nms"], ties)
    surv = cand[keep]
    spts = scene.points[surv]
    src = choose_sources(scene.weights[surv], draws)
    nbr = knn(spts, spts[src], Np + 1, cfg["r_nbr"], ties)
    depth = cfg["r_nbr"] // SUBDIVIDE_RESOLUTION
    pairs = np.zeros((S, Np, 2), np.int32)
    conn = np.zeros((S, Np), bool)
    valid = np.zeros((S, Np), bool)
    for s in range(S):
        row = nbr[s][nbr[s] < surv.shape[0]][1:]
        reached = bfs_reached(scene.adj_start, scene.adj, int(surv[src[s]]), surv[row].tolist(), depth)
        pairs[s, :, 0] = src[s]
        pairs[s, :, 1] = src[s]
        pairs[s, :row.shape[0], 1] = row
        valid[s, :row.shape[0]] = True
        conn[s, :row.shape[0]] = [int(t) in reached for t in surv[row]]
    noise = np.asarray(draws["noise"], dtype=np.float64)[:surv.shape[0]]
    points = transform_points(spts, x0, y0, P, rot, noise).astype(np.float32)
    return dict(points=points, pairs=pairs, connected=conn, valid=valid, candidates=cand, survivors=surv,
                sources=src)


def crop(img: np.ndarray, x0: int, y0: int, patch: int, rot: int) -> np.ndarray:
    """np.rot90 of the crop (dataset.py:414-425)."""
    return np.rot90(img[y0:y0 + patch, x0:x0 + patch], rot, (0, 1)).copy()
