"""Host mirror of the device-side graph stage of `inferencer.infer_one_img`.

The reference runs three pieces of host code between and after its two model passes:
    graph_extraction.extract_graph_points   graph_extraction.py:130-139 (+ graph_utils.nms_points 572-591)
    pair-query construction                 inferencer.py:126-197 (rtree box query + KDTree kNN per tile)
    edge aggregation                        inferencer.py:206-230 (Python triple loop over dicts)
`SceneGraph` binds the C-ABI entry points that run them on the GPU (include/samroad_b200.h,
csrc/graph.cu).  All three are integer / index work plus one ordered float32 sum: results are exact.

Tie order.  `nms_points` visits candidates in `np.argsort(scores)[::-1]` order; how NumPy's unstable
sort orders EQUAL scores depends on the NumPy build and the CPU (AVX-512 / AVX2 / generic paths give
different permutations), and mask scores are uint8, so ties are the rule.  `tie_order="numpy"` (default)
asks this host's NumPy for the permutation through a callback -- bit-exact with the reference run on
the same machine; `tie_order="stable"` sorts on the device as `argsort(kind="stable")[::-1]` would.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

TIE_ORDERS = ("numpy", "stable")


def default_tie_order() -> str:
    v = os.environ.get("SAMROAD_NMS_TIE_ORDER", "numpy").lower()
    if v not in TIE_ORDERS:
        raise ValueError(f"SAMROAD_NMS_TIE_ORDER must be one of {TIE_ORDERS}, got {v!r}")
    return v


def _numpy_argsort(keys, key_dtype, n, order_out, user):      # samroad_argsort_fn
    try:
        ctype = C.c_uint8 if key_dtype == _lib.U8 else C.c_double
        if key_dtype not in (_lib.U8, _lib.F64):
            return 2
        a = np.ctypeslib.as_array(C.cast(keys, C.POINTER(ctype)), shape=(n,))
        np.ctypeslib.as_array(order_out, shape=(n,))[:] = np.argsort(a)   # graph_utils.py:574
        return 0
    except Exception:       # never let an exception cross the C boundary
        return 1


_NUMPY_ARGSORT_CB = _lib.ARGSORT_FN(_numpy_argsort)
_NULL_CB = C.cast(None, _lib.ARGSORT_FN)


class SceneGraph:
    """Scratch owner + bindings for one device.  Not thread-safe; calls are ordered on the current
    torch CUDA stream (each of the three stages synchronises it to read a few counts back)."""

    def __init__(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"SceneGraph runs on CUDA only, got '{device}' (there is no CPU path)")
        self.device = device
        self._idx = device.index if device.index is not None else torch.cuda.current_device()
        self._h = _lib.Handle("samroad_graph_create", "samroad_graph_destroy", self._idx)
        self._points_buf: Optional[torch.Tensor] = None
        self._edges_buf: Optional[torch.Tensor] = None
        self._counts: Optional[np.ndarray] = None
        self.stats: dict = {}

    __getstate__ = _lib.refuse_copy

    def close(self) -> None:
        self._h.close()

    # ---- keypoints ----------------------------------------------------------------------------------
    def extract_graph_points(self, keypoint_mask: torch.Tensor, road_mask: torch.Tensor, itsc_threshold,
                             road_threshold, itsc_nms_radius, road_nms_radius,
                             tie_order: Optional[str] = None) -> torch.Tensor:
        """graph_extraction.extract_graph_points on device uint8 masks [H,W] -> int64 [N,2] (x,y) device
        tensor in the reference's order.  Thresholds are the config's 0..1 values (scaled by 255 here,
        graph_extraction.py:131,133)."""
        tie_order = tie_order or default_tie_order()
        if tie_order not in TIE_ORDERS:
            raise ValueError(f"tie_order must be one of {TIE_ORDERS}")
        for m in (keypoint_mask, road_mask):
            if m.dtype != torch.uint8 or m.dim() != 2 or not m.is_contiguous() or m.device != self.device:
                raise ValueError("masks must be contiguous uint8 [H,W] tensors on the graph's device")
        H, W = int(keypoint_mask.shape[0]), int(keypoint_mask.shape[1])
        if tuple(road_mask.shape) != (H, W):
            raise ValueError("mask shapes differ")
        cap = H * W
        if self._points_buf is None or self._points_buf.shape[0] < cap:
            self._points_buf = torch.empty((cap, 2), dtype=torch.int64, device=self.device)
        n = C.c_int(0)
        stats = (C.c_int32 * 16)()
        cb = _NUMPY_ARGSORT_CB if tie_order == "numpy" else _NULL_CB
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_extract_graph_points(
                self._h, keypoint_mask.data_ptr(), road_mask.data_ptr(), H, W,
                float(itsc_threshold) * 255, float(road_threshold) * 255, float(itsc_nms_radius),
                float(road_nms_radius), cb, None, self._points_buf.data_ptr(), cap, C.byref(n), stats,
                _lib.current_stream_ptr()), "samroad_extract_graph_points")
        self.stats.update(candidates=(stats[0], stats[1]), pass_survivors=(stats[2], stats[3]),
                          nms_rounds=(stats[4], stats[5], stats[6]), n_points=n.value, tie_order=tie_order,
                          us=dict(candidates=stats[8], order=(stats[9], stats[10], stats[11]),
                                  nms=(stats[12], stats[13], stats[14]), total=stats[15]))
        return self._points_buf[: n.value].clone()

    # ---- pair queries -------------------------------------------------------------------------------
    def plan_pair_queries(self, points_xy: torch.Tensor, tile_xy: np.ndarray, patch_size: int,
                          neighbor_radius: float, max_nbr: int = 16) -> np.ndarray:
        """Box query + kNN for every tile (inferencer.py:148-176).  points_xy: int64 [N,2] on the device;
        tile_xy: host int [n_tiles,2] origins in tile-list order; max_nbr: MAX_NEIGHBOR_QUERIES (1..32),
        the largest K fill_batch / aggregate_edges may then use.  Returns the per-tile point counts."""
        if points_xy.dtype != torch.int64 or points_xy.dim() != 2 or points_xy.shape[1] != 2 or \
                points_xy.device != self.device:
            raise ValueError("points_xy must be an int64 [N,2] tensor on the graph's device")
        pts = points_xy.contiguous()
        txy = np.ascontiguousarray(tile_xy, dtype=np.int32).reshape(-1, 2)
        counts = np.zeros(txy.shape[0], dtype=np.int32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_pair_queries_plan_k(
                self._h, pts.data_ptr(), int(pts.shape[0]), txy.ctypes.data, int(txy.shape[0]),
                int(patch_size), float(neighbor_radius), int(max_nbr), counts.ctypes.data,
                _lib.current_stream_ptr()), "samroad_pair_queries_plan")
        self._counts = counts
        return counts

    def fill_batch(self, tile_begin: int, n_tiles: int, nmax: int, max_nbr: int
                   ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Padded TopoNet inputs of tiles [tile_begin, tile_begin + n_tiles) (inferencer.py:164-197):
        points int32 [B,nmax,2], pairs int32 [B,nmax,K,2], valid bool [B,nmax,K]."""
        pts = torch.empty((n_tiles, nmax, 2), dtype=torch.int32, device=self.device)
        prs = torch.empty((n_tiles, nmax, max_nbr, 2), dtype=torch.int32, device=self.device)
        val = torch.empty((n_tiles, nmax, max_nbr), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_pair_queries_fill(
                self._h, int(tile_begin), int(n_tiles), int(nmax), int(max_nbr), pts.data_ptr(),
                prs.data_ptr(), val.data_ptr(), _lib.current_stream_ptr()), "samroad_pair_queries_fill")
        return pts, prs, val.view(torch.bool)

    # ---- edges --------------------------------------------------------------------------------------
    def aggregate_edges(self, topo_scores: torch.Tensor, tile_score_offsets: Sequence[int], max_nbr: int,
                        topo_threshold: float) -> torch.Tensor:
        """inferencer.py:206-230 over the planned tiles.  topo_scores: flat float32 device buffer; tile t's
        [nmax_of_its_batch, K] block starts at element tile_score_offsets[t] (negative = batch skipped).
        Returns int64 [E,2] (src,tgt) global point indices on the device, in the reference's edge order.
        Raises AssertionError when a score lies outside [0,1], like the reference (inferencer.py:219)."""
        assert self._counts is not None, "plan_pair_queries first"
        total = int(self._counts.sum())
        cap = max(1, total * int(max_nbr))
        if self._edges_buf is None or self._edges_buf.shape[0] < cap:
            self._edges_buf = torch.empty((cap, 2), dtype=torch.int64, device=self.device)
        offs = np.ascontiguousarray(tile_score_offsets, dtype=np.int64)
        assert offs.shape[0] == self._counts.shape[0]
        sc = topo_scores.contiguous()
        assert sc.dtype == torch.float32 and sc.device == self.device
        n, bad = C.c_int(0), C.c_int(0)
        # threshold as float32: `np.float32 mean > python float` compares in float32 (NEP 50)
        thr = float(np.float32(topo_threshold))
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_aggregate_edges(
                self._h, sc.data_ptr(), offs.ctypes.data, int(max_nbr), thr, self._edges_buf.data_ptr(),
                cap, C.byref(n), C.byref(bad), _lib.current_stream_ptr()), "samroad_aggregate_edges")
        assert bad.value == 0, "topology score outside [0,1]"      # inferencer.py:219
        return self._edges_buf[: n.value].clone()
