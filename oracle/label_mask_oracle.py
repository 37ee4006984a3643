"""Pure Python restatement of the label masks that cityscale/generate_labels.py and spacenet/generate_labels.py
write: the checker of csrc/label_masks.cu.

Graph semantics (what the scripts get from networkx): every adjacency entry (n, nei) adds the undirected edge
{key(n), key(nei)} with key (int(col), int(row)) for CityScale and (int(col), 400 - int(row)) for SpaceNet; repeated
and one-way entries collapse, nodes exist only through edges, and a self-loop adds 2 to its node's degree.

Drawing (OpenCV 4.x drawing.cpp, restated as its loops run, for an 8-bit one-channel image):
  circle(img, c, r, 255, -1)    -> Circle(img, c, r, fill=1)          integer midpoint spans
  line(img, p0, p1, 255, t > 1) -> clipLine of the segment to the image grown by t pixels on every side, then
                                   ThickLine: the quad p0 +- d, p1 -+ d in 16-bit fixed point filled by
                                   FillConvexPoly(LINE_8, shift 16) (outline by Line2, then scanline spans), and
                                   Circle(p, (t + 1) // 2, fill=1) at both ends
The scanline walk below accumulates x += dx row by row as OpenCV does; the device computes every row in closed
form, so the two are independent."""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
SPACENET_SIZE = 400


def _tdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def _hline(img: np.ndarray, y: int, x1: int, x2: int) -> None:
    img[y, x1:x2 + 1] = 255


def circle_fill(img: np.ndarray, cx: int, cy: int, radius: int) -> None:
    """Circle(img, center, radius, color, fill=1): spans of the midpoint walk, clipped to the image."""
    h, w = img.shape
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    while dx >= dy:
        for (y1, y2, xa, xb) in ((cy - dy, cy + dy, cx - dx, cx + dx), (cy - dx, cy + dx, cx - dy, cx + dy)):
            if xa < w and xb >= 0:
                xa, xb = max(xa, 0), min(xb, w - 1)
                for y in (y1, y2):
                    if 0 <= y < h:
                        _hline(img, y, xa, xb)
        dy += 1
        err += plus
        plus += 2
        mask = (err <= 0) - 1
        err -= minus & mask
        dx += mask
        minus -= mask & 2


def clip_line(w: int, h: int, p1: List[int], p2: List[int]) -> bool:
    """clipLine(Size2l, Point2l&, Point2l&): Cohen-Sutherland with double-precision intersections."""
    right, bottom = w - 1, h - 1
    x1, y1 = p1
    x2, y2 = p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    p1[:] = [x1, y1]
    p2[:] = [x2, y2]
    return (c1 | c2) == 0


def line2(img: np.ndarray, pt1: Tuple[int, int], pt2: Tuple[int, int]) -> None:
    """Line2: the 8-connected fixed-point DDA FillConvexPoly outlines a polygon with."""
    h, w = img.shape
    p1, p2 = list(pt1), list(pt2)
    if not clip_line(w << XY_SHIFT, h << XY_SHIFT, p1, p2):
        return
    dx, dy = p2[0] - p1[0], p2[1] - p1[1]
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            dy = -dy
            p1, p2 = p2, p1
        x_step, y_step = XY_ONE, _tdiv(dy << XY_SHIFT, ax | 1)
        ecount = (p2[0] - p1[0]) >> XY_SHIFT
    else:
        if dy < 0:
            dx = -dx
            p1, p2 = p2, p1
        x_step, y_step = _tdiv(dx << XY_SHIFT, ay | 1), XY_ONE
        ecount = (p2[1] - p1[1]) >> XY_SHIFT
    x, y = p1[0] + (XY_ONE >> 1), p1[1] + (XY_ONE >> 1)

    def put(px, py):
        if 0 <= px < w and 0 <= py < h:
            img[py, px] = 255

    put((p2[0] + (XY_ONE >> 1)) >> XY_SHIFT, (p2[1] + (XY_ONE >> 1)) >> XY_SHIFT)
    if ax > ay:
        x >>= XY_SHIFT
        while ecount >= 0:
            put(x, y >> XY_SHIFT)
            x += 1
            y += y_step
            ecount -= 1
    else:
        y >>= XY_SHIFT
        while ecount >= 0:
            put(x >> XY_SHIFT, y)
            x += x_step
            y += 1
            ecount -= 1


def fill_convex_poly(img: np.ndarray, v: List[Tuple[int, int]]) -> None:
    """FillConvexPoly(img, v, npts, color, LINE_8, shift=XY_SHIFT)."""
    h, w = img.shape
    npts = len(v)
    delta = XY_ONE >> 1
    imin = 0
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    p0 = v[npts - 1]
    for i in range(npts):
        p = v[i]
        if p[1] < ymin:
            ymin, imin = p[1], i
        ymax, xmax, xmin = max(ymax, p[1]), max(xmax, p[0]), min(xmin, p[0])
        line2(img, p0, p)
        p0 = p
    xmin, xmax = (xmin + delta) >> XY_SHIFT, (xmax + delta) >> XY_SHIFT
    ymin, ymax = (ymin + delta) >> XY_SHIFT, (ymax + delta) >> XY_SHIFT
    if npts < 3 or xmax < 0 or ymax < 0 or xmin >= w or ymin >= h:
        return
    ymax = min(ymax, h - 1)
    edges = npts
    idx_ = [imin, imin]
    di = [1, npts - 1]
    ye = [ymin, ymin]
    ex = [-XY_ONE, -XY_ONE]
    edx = [0, 0]
    y = ymin
    while True:
        for i in range(2):
            if y >= ye[i]:
                idx0 = idx_[i]
                idx = (idx0 + di[i]) % npts
                while True:
                    go = edges > 0
                    edges -= 1
                    if not go:
                        break
                    ty = (v[idx][1] + delta) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        ye[i] = ty
                        edx[i] = _tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        ex[i] = xs
                        idx_[i] = idx
                        break
                    idx0 = idx
                    idx = (idx + di[i]) % npts
        if edges < 0:
            break
        if y >= 0:
            left, right = (1, 0) if ex[0] > ex[1] else (0, 1)
            xx1 = (ex[left] + delta) >> XY_SHIFT
            xx2 = (ex[right] + delta) >> XY_SHIFT
            if xx2 >= 0 and xx1 < w:
                _hline(img, y, max(xx1, 0), min(xx2, w - 1))
        ex[0] += edx[0]
        ex[1] += edx[1]
        y += 1
        if y > ymax:
            break


def thick_line(img: np.ndarray, p0: Tuple[int, int], p1: Tuple[int, int], thickness: int) -> None:
    """cv2.line(img, p0, p1, 255, thickness) for thickness >= 2: the segment clipped in whole pixels to the image
    grown by `thickness` on every side, then ThickLine with LINE_8, shift 0."""
    assert thickness >= 2
    h, w = img.shape
    a, b = [p0[0] + thickness, p0[1] + thickness], [p1[0] + thickness, p1[1] + thickness]
    if not clip_line(w + 2 * thickness, h + 2 * thickness, a, b):
        return
    p0, p1 = (a[0] - thickness, a[1] - thickness), (b[0] - thickness, b[1] - thickness)
    a = (p0[0] << XY_SHIFT, p0[1] << XY_SHIFT)
    b = (p1[0] << XY_SHIFT, p1[1] << XY_SHIFT)
    dx = (a[0] - b[0]) / XY_ONE
    dy = (b[1] - a[1]) / XY_ONE
    r = dx * dx + dy * dy
    odd = thickness & 1
    t = thickness << (XY_SHIFT - 1)
    if abs(r) > np.finfo(np.float64).eps:
        r = (t + odd * XY_ONE * 0.5) / math.sqrt(r)
        dpx, dpy = round(dy * r), round(dx * r)          # cvRound: nearest, ties to even
        fill_convex_poly(img, [(a[0] + dpx, a[1] + dpy), (a[0] - dpx, a[1] - dpy),
                               (b[0] - dpx, b[1] - dpy), (b[0] + dpx, b[1] + dpy)])
    cap = (t + (XY_ONE >> 1)) >> XY_SHIFT
    for p in (p0, p1):
        circle_fill(img, p[0], p[1], cap)


def node_key(n, dataset: str) -> Tuple[int, int]:
    if dataset == "cityscale":
        return (int(n[1]), int(n[0]))
    if dataset == "spacenet":
        return (int(n[1]), SPACENET_SIZE - int(n[0]))
    raise ValueError(f"unknown dataset {dataset!r}")


def tile_graph(adj: Dict, dataset: str):
    """(keypoints, edges) as generate_labels.py derives them from a networkx Graph: keypoints are the nodes of
    degree != 2 (a self-loop counts 2), edges the unique undirected pairs, self-loops included."""
    nbrs: Dict[Tuple[int, int], set] = {}
    for n, neis in adj.items():
        for nei in neis:
            u, v = node_key(n, dataset), node_key(nei, dataset)
            nbrs.setdefault(u, set()).add(v)
            nbrs.setdefault(v, set()).add(u)
    deg = {u: len(s) + (u in s) for u, s in nbrs.items()}
    keypoints = sorted(u for u, d in deg.items() if d != 2)
    edges = sorted({(min(u, v), max(u, v)) for u, s in nbrs.items() for v in s})
    return keypoints, edges


def draw_masks(keypoints, edges, size: int, keypoint_radius: int = 3, road_width: int = 3):
    """uint8 (keypoint_mask, road_mask) [size, size] of 0 / 255."""
    kp = np.zeros((size, size), np.uint8)
    road = np.zeros((size, size), np.uint8)
    for (x, y) in keypoints:
        circle_fill(kp, x, y, keypoint_radius)
    for (p, q) in edges:
        thick_line(road, p, q, road_width)
    return kp, road


def tile_masks(adj: Dict, dataset: str, size: int):
    kps, edges = tile_graph(adj, dataset)
    return draw_masks(kps, edges, size)
