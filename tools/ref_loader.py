"""Import the UNMODIFIED reference (htcr/sam_road) from /root/reference for oracle validation.

Only usable where /root/reference exists (the build container); nothing under tests -m gpu, smoke()
or bench.py depends on it.  The reference's model.py needs `lightning`, `torchmetrics` and
`matplotlib`, which are absent here, so three stub modules are injected into sys.modules
(SURVEY.md §8c) -- the reference's own source files are imported as they lie, never copied.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

REF_ROOT = os.environ.get("SAMROAD_REFERENCE", "/root/reference")


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "model.py"))


def _install_stubs():
    import torch.nn as nn
    if "lightning" not in sys.modules:
        lightning = types.ModuleType("lightning")
        pl = types.ModuleType("lightning.pytorch")

        class LightningModule(nn.Module):
            def log(self, *a, **k):
                pass

            def log_dict(self, *a, **k):
                pass

        pl.LightningModule = LightningModule
        lightning.pytorch = pl
        sys.modules["lightning"] = lightning
        sys.modules["lightning.pytorch"] = pl
    if "torchmetrics" not in sys.modules:
        tm = types.ModuleType("torchmetrics")
        tmc = types.ModuleType("torchmetrics.classification")

        class _Metric(nn.Module):
            def __init__(self, *a, **k):
                super().__init__()

        tmc.BinaryJaccardIndex = _Metric
        tmc.F1Score = _Metric
        tmc.BinaryPrecisionRecallCurve = _Metric
        tm.classification = tmc
        sys.modules["torchmetrics"] = tm
        sys.modules["torchmetrics.classification"] = tmc
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"] = mpl
        sys.modules["matplotlib.pyplot"] = plt
    os.environ.setdefault("WANDB_MODE", "disabled")


def _install_graph_shims():
    """Import shims for what the reference's dataset.py / graph_utils.py import and this machine lacks:
    igraph, rtree, shapely, matplotlib.colors and addict.  Each is installed only where the real module is
    missing.  They restate the libraries' documented semantics for the calls the reference makes -- they are
    not the libraries: a fixture made with them pins the reference's logic, not GEOS's floating point.
      igraph   Graph(n, edges) undirected; vs['attr'] get / set per vertex; es with .source / .target (the
               smaller / larger vertex id, as igraph reports undirected edges); degree(i) counts a self-loop
               twice; neighbors(i, mode='all').
      rtree    index.Index with insert(id, (minx, miny, maxx, maxy)) and intersection(box): the ids whose boxes
               meet the query box, bounds inclusive, in ascending id.
      shapely  LineString([p, q]).intersection(other) for two segments: empty, a Point (exactly the shared
               endpoint when they meet there) or a LineString for a collinear overlap; Point.equals compares
               coordinates.  shapely.strtree.STRtree is imported only.
    """
    if "igraph" not in sys.modules and not _has("igraph"):
        ig = types.ModuleType("igraph")

        class _Edge:
            def __init__(self, s, t):
                self.source, self.target = min(s, t), max(s, t)

        class _VertexSeq:
            def __init__(self, n):
                self._n, self._attrs = n, {}

            def __len__(self):
                return self._n

            def __getitem__(self, key):
                return list(self._attrs[key])

            def __setitem__(self, key, values):
                vals = list(values)
                if len(vals) != self._n:
                    raise ValueError("attribute list length must match the vertex count")
                self._attrs[key] = vals

        class Graph:
            def __init__(self, n=0, edges=None):
                self.vs = _VertexSeq(int(n))
                self.es = [_Edge(int(a), int(b)) for a, b in (edges or [])]
                self._nbrs = [[] for _ in range(int(n))]
                for e in self.es:
                    self._nbrs[e.source].append(e.target)
                    self._nbrs[e.target].append(e.source)

            def degree(self, i):
                return len(self._nbrs[i])

            def neighbors(self, i, mode="all"):
                return sorted(self._nbrs[i])

        ig.Graph = Graph
        sys.modules["igraph"] = ig
    if "rtree" not in sys.modules and not _has("rtree"):
        rtree = types.ModuleType("rtree")
        index = types.ModuleType("rtree.index")

        class Index:
            def __init__(self):
                self._ids, self._boxes = [], []

            def insert(self, i, box):
                self._ids.append(i)
                self._boxes.append(tuple(float(v) for v in box))

            def intersection(self, box):
                x0, y0, x1, y1 = (float(v) for v in box)
                return sorted(i for i, (a, b, c, d) in zip(self._ids, self._boxes)
                              if a <= x1 and c >= x0 and b <= y1 and d >= y0)

        index.Index = Index
        rtree.index = index
        sys.modules["rtree"] = rtree
        sys.modules["rtree.index"] = index
    if "shapely" not in sys.modules and not _has("shapely"):
        shapely = types.ModuleType("shapely")
        geometry = types.ModuleType("shapely.geometry")
        strtree = types.ModuleType("shapely.strtree")

        class Point:
            geom_type = "Point"
            is_empty = False

            def __init__(self, x, y=None):
                if y is None:
                    x, y = x
                self.x, self.y = float(x), float(y)

            def equals(self, other):
                return self.x == other.x and self.y == other.y

        class _Empty:
            geom_type = "GeometryCollection"
            is_empty = True

        class LineString:
            geom_type = "LineString"
            is_empty = False

            def __init__(self, coords):
                (self.p, self.q) = [tuple(float(v) for v in c) for c in coords]

            def intersection(self, other):
                (x1, y1), (x2, y2), (x3, y3), (x4, y4) = self.p, self.q, other.p, other.q
                d1x, d1y, d2x, d2y, qx, qy = x2 - x1, y2 - y1, x4 - x3, y4 - y3, x3 - x1, y3 - y1
                den = d1x * d2y - d1y * d2x
                tn, un = qx * d2y - qy * d2x, qx * d1y - qy * d1x
                if den == 0:
                    if tn != 0:                       # parallel, not collinear
                        return _Empty()
                    # collinear: the overlap along the first segment's direction
                    ll = d1x * d1x + d1y * d1y
                    if ll == 0:
                        return _Empty()
                    ta = (qx * d1x + qy * d1y) / ll
                    tb = ((x4 - x1) * d1x + (y4 - y1) * d1y) / ll
                    lo, hi = max(0.0, min(ta, tb)), min(1.0, max(ta, tb))
                    if lo > hi:
                        return _Empty()
                    if lo == hi:
                        pts = [p for p in (self.p, self.q, other.p, other.q)
                               if (p[0] - x1) * d1x + (p[1] - y1) * d1y == lo * ll]
                        return Point(*pts[0]) if pts else Point(x1 + lo * d1x, y1 + lo * d1y)
                    ls = LineString([(x1 + lo * d1x, y1 + lo * d1y), (x1 + hi * d1x, y1 + hi * d1y)])
                    return ls
                s = 1.0 if den > 0 else -1.0
                if not (0 <= tn * s <= abs(den) and 0 <= un * s <= abs(den)):
                    return _Empty()
                for num, pt in ((tn, self.p), (tn - den, self.q), (un, other.p), (un - den, other.q)):
                    if num == 0:
                        return Point(*pt)
                t = tn / den
                return Point(x1 + t * d1x, y1 + t * d1y)

        class STRtree:
            def __init__(self, *a, **k):
                raise NotImplementedError("shapely.strtree.STRtree is not shimmed")

        geometry.Point, geometry.LineString = Point, LineString
        strtree.STRtree = STRtree
        shapely.geometry, shapely.strtree = geometry, strtree
        sys.modules.update({"shapely": shapely, "shapely.geometry": geometry, "shapely.strtree": strtree})
    if not _has("matplotlib"):
        mpl = sys.modules.get("matplotlib") or types.ModuleType("matplotlib")
        if not hasattr(mpl, "pyplot"):
            mpl.pyplot = types.ModuleType("matplotlib.pyplot")
            sys.modules["matplotlib.pyplot"] = mpl.pyplot
        colors = types.ModuleType("matplotlib.colors")
        colors.ListedColormap = type("ListedColormap", (), {"__init__": lambda self, *a, **k: None})
        mpl.colors = colors
        sys.modules["matplotlib"] = mpl
        sys.modules["matplotlib.colors"] = colors
    if "addict" not in sys.modules and not _has("addict"):
        addict = types.ModuleType("addict")
        addict.Dict = AttrDict
        sys.modules["addict"] = addict


def _has(name: str) -> bool:
    import importlib.util
    try:
        return importlib.util.find_spec(name) is not None
    except (ImportError, ValueError):
        return False


def load_reference_dataset():
    """The reference's dataset.py module (GraphLabelGenerator, sample_patch) as it lies, with the import shims of
    _install_graph_shims where the real libraries are missing."""
    assert available(), f"reference not found under {REF_ROOT}"
    _install_graph_shims()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import dataset as ref_dataset  # noqa: the reference's dataset.py
    return ref_dataset


class AttrDict(dict):
    """addict.Dict-like config: missing keys read as an empty (falsy) AttrDict (utils.py:6-9)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            return AttrDict()

    def __setattr__(self, k, v):
        self[k] = v


def load_reference_model(config: dict):
    """Instantiate the reference SAMRoad (eval mode, CPU) with a synthetic SAM_CKPT_PATH that only
    holds a correctly sized pos_embed (model.py:367-396 loads it unconditionally)."""
    import contextlib
    import io

    import torch
    assert available(), f"reference not found under {REF_ROOT}"
    _install_stubs()
    for p in (REF_ROOT, os.path.join(REF_ROOT, "sam")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import model as ref_model  # noqa: the reference's model.py

    cfg = AttrDict(config)
    from oracle.samroad_oracle import ModelSpec
    spec = ModelSpec.from_config(cfg)
    with tempfile.NamedTemporaryFile(suffix=".pth", delete=False) as f:
        torch.save({"image_encoder.pos_embed": torch.zeros(1, spec.grid, spec.grid, spec.embed_dim)}, f)
        cfg["SAM_CKPT_PATH"] = f.name
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            net = ref_model.SAMRoad(cfg)
    finally:
        os.unlink(cfg["SAM_CKPT_PATH"])
    net.eval()
    return net
