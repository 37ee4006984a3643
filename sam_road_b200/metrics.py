"""Exact binary precision-recall curves on the device (the threshold search of the reference's test.py).

`PrecisionRecallCurve` stands for one torchmetrics `BinaryPrecisionRecallCurve(ignore_index=-1)` of
SAMRoad (reference model.py:361-363): `update` appends scores and labels on the device without a host
synchronisation, `compute` returns the exact curve in torchmetrics' layout.  Under torch.distributed
(world size > 1) `compute` is the curve of every rank's entries, as torchmetrics' sync on compute gives:
the ranks all-gather their packed keys, and since the curve depends only on the multiset of keys the
result is exact and the same on every rank.  The work runs in the
`samroad_prc_*` kernels of libsamroad_b200.so (include/samroad_b200.h); DESIGN.md §10 states where the
result differs from torchmetrics' (integer counts, no sigmoid of out-of-range scores).

`ValidationMetrics` stands for the criteria and the BinaryJaccardIndex / F1Score metrics validation_step feeds
(reference model.py:349-359, 547-600), in the `samroad_val_*` kernels; DESIGN.md §11 states its contract.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib


class PrecisionRecallCurve:
    """Accumulates (score, label) pairs on one CUDA device; state persists until `reset()`."""

    def __init__(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"PrecisionRecallCurve runs on CUDA only; got '{device}'. There is no CPU path.")
        self.device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
        self._h = _lib.Handle("samroad_prc_create", "samroad_prc_destroy", self.device.index)
        self._curve_h = self._h     # the handle the last compute ran on (a gathered one under distributed)
        self._best = None

    __getstate__ = _lib.refuse_copy

    def close(self) -> None:
        self._drop_gathered()
        self._h.close()

    def _drop_gathered(self):
        if self._curve_h is not self._h:
            self._curve_h.close()
        self._curve_h = self._h

    def reset(self) -> None:
        with torch.cuda.device(self.device):
            self._drop_gathered()
            _lib.check(_lib.load().samroad_prc_reset(self._h, _lib.current_stream_ptr()), "samroad_prc_reset")
        self._best = None

    def update(self, preds: torch.Tensor, target: torch.Tensor, valid: Optional[torch.Tensor] = None) -> None:
        """preds: float32 scores in [0, 1], any view whose elements sit at one common stride (such as
        mask_scores[..., c]) is read in place.  target: float (label = int32(target)) or bool / uint8
        labels of the same number of elements.  valid: optional bool / uint8 mask, False = ignored.
        Asynchronous: an update with a NaN or out-of-range score or a label other than 0 / 1 adds nothing
        and is reported by the next `compute()`."""
        n = preds.numel()
        if target.numel() != n or (valid is not None and valid.numel() != n):
            raise ValueError(f"preds, target and valid must have the same number of elements; got {n}, "
                             f"{target.numel()}, {None if valid is None else valid.numel()}")
        for name, t in (("preds", preds), ("target", target), ("valid", valid)):
            if t is not None and t.device != self.device:
                raise RuntimeError(f"{name} is on {t.device}, the accumulator on {self.device}")
        if preds.dtype != torch.float32:
            raise TypeError(f"preds must be float32, got {preds.dtype}")
        flat = preds.reshape(-1)            # a view whenever the elements share one stride
        stride = flat.stride(0) if n > 1 else 1
        if target.dtype in (torch.bool, torch.uint8):
            tgt, tdt = target.reshape(-1).contiguous().view(torch.uint8), _lib.U8
        elif target.dtype == torch.float32:
            tgt, tdt = target.reshape(-1).contiguous(), _lib.F32
        else:
            raise TypeError(f"target must be float32, bool or uint8, got {target.dtype}")
        val = None
        if valid is not None:
            if valid.dtype not in (torch.bool, torch.uint8):
                raise TypeError(f"valid must be bool or uint8, got {valid.dtype}")
            val = valid.reshape(-1).contiguous().view(torch.uint8)
        self._best = None
        if n == 0:
            return
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_prc_update(
                self._h, flat.data_ptr(), stride, tgt.data_ptr(), tdt, _lib.ptr(val), n,
                _lib.current_stream_ptr()), "samroad_prc_update")

    def _gathered_handle(self, dist) -> _lib.Handle:
        """A new accumulator holding the accepted keys of every rank.  Every rank takes part in the same
        collectives even when one of them fails, so a refusal on one rank raises on all of them instead of
        leaving the others waiting."""
        lib, stream = _lib.load(), _lib.current_stream_ptr()
        world = dist.get_world_size()
        comm_dev = self.device if dist.get_backend() == "nccl" else torch.device("cpu")
        n = C.c_int64(0)
        rc = lib.samroad_prc_export_keys(self._h, None, 0, C.byref(n), stream)
        err = _lib.last_error() if rc else ""
        mine = torch.tensor([n.value if rc == 0 else -1], dtype=torch.int64, device=comm_dev)
        counts = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(counts, mine)
        counts = [int(c) for c in counts]
        if rc:
            raise RuntimeError(f"samroad_prc_export_keys failed (code {rc}): {err}")
        if min(counts) < 0:
            raise RuntimeError(f"rank {counts.index(-1)} could not contribute its entries to the curve "
                               "(its own error names the cause)")
        m = max(max(counts), 1)
        local = torch.zeros(m, dtype=torch.int32, device=self.device)    # packed uint32 keys, as int32
        _lib.check(lib.samroad_prc_export_keys(self._h, local.data_ptr(), m, C.byref(n), stream),
                   "samroad_prc_export_keys")
        send = local.to(comm_dev)
        parts = [torch.empty(m, dtype=torch.int32, device=comm_dev) for _ in range(world)]
        dist.all_gather(parts, send)
        h = _lib.Handle("samroad_prc_create", "samroad_prc_destroy", self.device.index)
        try:
            for part, c in zip(parts, counts):
                part = part[:c].to(self.device)
                _lib.check(lib.samroad_prc_append_keys(h, part.data_ptr(), c, stream), "samroad_prc_append_keys")
            torch.cuda.current_stream().synchronize()    # `parts` are freed on return
        except Exception:
            h.close()
            raise
        return h

    def _compute(self):
        counts = (C.c_int64 * 4)()
        best = (C.c_float * 4)()
        with torch.cuda.device(self.device):
            self._drop_gathered()
            dist = torch.distributed
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                self._curve_h = self._gathered_handle(dist)
            _lib.check(_lib.load().samroad_prc_compute(self._curve_h, counts, best, _lib.current_stream_ptr()),
                       "samroad_prc_compute")
        self._best = (tuple(counts), tuple(best))
        return self._best

    def compute(self, with_counts: bool = False):
        """(precision [T+1], recall [T+1], thresholds [T]) as device float32 tensors, thresholds ascending
        and the curve ending with the point (1, 0) like torchmetrics'.  With `with_counts` the int64
        true / false positive counts [T] at each threshold follow."""
        (n, n_pos, T, _), _ = self._compute()
        dev = self.device
        thr = torch.empty(T, dtype=torch.float32, device=dev)
        prec = torch.empty(T + 1, dtype=torch.float32, device=dev)
        rec = torch.empty(T + 1, dtype=torch.float32, device=dev)
        tps = torch.empty(T, dtype=torch.int64, device=dev) if with_counts else None
        fps = torch.empty(T, dtype=torch.int64, device=dev) if with_counts else None
        with torch.cuda.device(dev):
            _lib.check(_lib.load().samroad_prc_read_curve(
                self._curve_h, thr.data_ptr(), prec.data_ptr(), rec.data_ptr(), _lib.ptr(tps), _lib.ptr(fps),
                _lib.current_stream_ptr()), "samroad_prc_read_curve")
        return (prec, rec, thr, tps, fps) if with_counts else (prec, rec, thr)

    def best(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """0-dim float32 device tensors (threshold, precision, recall, F1) at torch.argmax of
        F1 = 2*(P*R)/(P+R) over the curve: the first maximum, a NaN counting as the largest value."""
        if self._best is None:
            self._compute()
        _, vals = self._best
        return tuple(torch.tensor(v, dtype=torch.float32, device=self.device) for v in vals)


# order of the int64 counts samroad_val_read returns
VAL_COUNT_NAMES = ("keypoint_tp", "keypoint_fp", "keypoint_fn", "keypoint_tn",
                   "road_tp", "road_fp", "road_fn", "road_tn",
                   "topo_tp", "topo_fp", "topo_fn")
VAL_LOSS_NAMES = ("val_mask_loss", "val_topo_loss", "val_loss")


def _f32(x: int) -> torch.Tensor:
    return torch.tensor(x, dtype=torch.int64).to(torch.float32)


def iou_from_counts(tp: int, fp: int, fn: int) -> torch.Tensor:
    """BinaryJaccardIndex's value from exact counts, torchmetrics 1.4.0 `_jaccard_index_reduce(average=
    "binary")`: the confusion matrix converted to float32, then tp / ((fp + fn) + tp), 0 when the
    denominator is 0 (`_safe_divide`)."""
    tpf, fpf, fnf = _f32(tp), _f32(fp), _f32(fn)
    den = fpf + fnf + tpf
    return torch.where(den != 0, tpf / den, torch.zeros((), dtype=torch.float32))


def f1_from_counts(tp: int, fp: int, fn: int) -> torch.Tensor:
    """Binary F1Score's value from exact counts, torchmetrics 1.4.0 `_fbeta_reduce(beta=1.0, average=
    "binary")`: 2 * tp / ((2 * tp + fn) + fp) in float32, 0 when the denominator is 0 (`_safe_divide`)."""
    tpf, fpf, fnf = _f32(tp), _f32(fp), _f32(fn)
    num = 2.0 * tpf
    den = num + 1.0 * fnf + fpf
    return torch.where(den != 0, num / den, torch.zeros((), dtype=torch.float32))


class ValidationMetrics:
    """The criteria and metrics validation_step feeds (reference model.py:349-359, 547-600) on one CUDA
    device: per step the (mask_loss, topo_loss, loss) triple, over the epoch the batch-size-weighted mean of
    each (Lightning's on_epoch mean, taken exactly) and the exact confusion counts behind keypoint_iou,
    road_iou and topo_f1.  `focal` selects torchvision's sigmoid_focal_loss (FOCAL_LOSS) for the masks.
    State persists until `reset()`."""

    def __init__(self, device, focal: bool = False):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"ValidationMetrics runs on CUDA only; got '{device}'. There is no CPU path.")
        self.device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
        self.loss_kind = _lib.LOSS_FOCAL if focal else _lib.LOSS_BCE
        self._h = _lib.Handle("samroad_val_create", "samroad_val_destroy", self.device.index)

    __getstate__ = _lib.refuse_copy

    def close(self) -> None:
        self._h.close()

    def reset(self) -> None:
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_val_reset(self._h, _lib.current_stream_ptr()), "samroad_val_reset")

    def _on_device(self, name, t, dtype):
        if t.device != self.device:
            raise RuntimeError(f"{name} is on {t.device}, the accumulator on {self.device}")
        if dtype == torch.uint8:
            if t.dtype not in (torch.bool, torch.uint8):
                raise TypeError(f"{name} must be bool or uint8, got {t.dtype}")
            return t.contiguous().view(torch.uint8)
        return t.to(torch.float32).contiguous()

    def update(self, mask_logits, mask_scores, keypoint_mask, road_mask, topo_logits, topo_scores,
               connected, valid) -> torch.Tensor:
        """One validation step.  mask_logits / mask_scores [B,P,P,2] float32 (as SAMRoad's encoder writes
        them), keypoint_mask / road_mask [B,P,P] float targets 0.0 / 1.0 (read in place when contiguous
        float32), topo_logits / topo_scores [B,Ns,Np(,1)], connected / valid [B,Ns,Np] bool.  Returns the
        step's (mask_loss, topo_loss, loss) as a float32 [3] device tensor; asynchronous.  A step with a
        target other than 0 / 1 or a NaN / out-of-range score adds nothing (its values are NaN) and is
        reported by the next `compute()` / `read()`."""
        if mask_logits.dim() != 4 or mask_logits.shape[-1] != 2 or mask_logits.shape[1] != mask_logits.shape[2]:
            raise ValueError(f"mask_logits must be [B,P,P,2], got {tuple(mask_logits.shape)}")
        B, P = int(mask_logits.shape[0]), int(mask_logits.shape[1])
        if B < 1:
            raise ValueError("a validation step needs at least one tile")
        if tuple(mask_scores.shape) != tuple(mask_logits.shape):
            raise ValueError(f"mask_scores {tuple(mask_scores.shape)} differs from mask_logits {tuple(mask_logits.shape)}")
        for name, m in (("keypoint_mask", keypoint_mask), ("road_mask", road_mask)):
            if tuple(m.shape) != (B, P, P):
                raise ValueError(f"{name} must be [{B},{P},{P}], got {tuple(m.shape)}")
        if connected.dim() != 3 or connected.shape[0] != B or tuple(valid.shape) != tuple(connected.shape):
            raise ValueError(f"connected / valid must be [{B},Ns,Np]; got {tuple(connected.shape)}, {tuple(valid.shape)}")
        Ns, Np = int(connected.shape[1]), int(connected.shape[2])
        n = B * Ns * Np
        if topo_logits.numel() != n or topo_scores.numel() != n:
            raise ValueError(f"topo_logits / topo_scores must hold B*Ns*Np = {n} elements; got "
                             f"{topo_logits.numel()}, {topo_scores.numel()}")
        ml, ms = (self._on_device(k, t, torch.float32) for k, t in (("mask_logits", mask_logits),
                                                                     ("mask_scores", mask_scores)))
        kp, road = (self._on_device(k, t, torch.float32) for k, t in (("keypoint_mask", keypoint_mask),
                                                                       ("road_mask", road_mask)))
        tl, ts = (self._on_device(k, t, torch.float32) for k, t in (("topo_logits", topo_logits),
                                                                     ("topo_scores", topo_scores)))
        con, val = (self._on_device(k, t, torch.uint8) for k, t in (("connected", connected), ("valid", valid)))
        out = torch.empty(3, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().samroad_val_update(
                self._h, ml.data_ptr(), ms.data_ptr(), kp.data_ptr(), road.data_ptr(), tl.data_ptr(), ts.data_ptr(),
                con.data_ptr(), val.data_ptr(), B, P, Ns, Np, self.loss_kind, out.data_ptr(),
                _lib.current_stream_ptr()), "samroad_val_update")
        return out

    def _read(self):
        """(rc, error, counts [11], means [3], totals [2]) of this rank; synchronises."""
        counts, means, totals = (C.c_int64 * 11)(), (C.c_float * 3)(), (C.c_int64 * 2)()
        with torch.cuda.device(self.device):
            rc = _lib.load().samroad_val_read(self._h, counts, means, totals, _lib.current_stream_ptr())
        return rc, (_lib.last_error() if rc else ""), list(counts), list(means), list(totals)

    def read(self):
        """This rank's state: ({count name: int}, (epoch mean mask_loss, topo_loss, loss) as Python floats,
        (accepted steps, sum of B)).  Synchronises; raises when a step was refused since the last report."""
        rc, err, counts, means, totals = self._read()
        if rc:
            raise RuntimeError(f"samroad_val_read failed (code {rc}): {err}")
        return dict(zip(VAL_COUNT_NAMES, counts)), tuple(means), tuple(totals)

    def compute(self) -> dict:
        """{"val_mask_loss", "val_topo_loss", "val_loss", "keypoint_iou", "road_iou", "topo_f1"} as Python
        floats.  The losses are this rank's epoch means (the reference logs them without sync_dist).  Under
        torch.distributed with more than one rank the counts are summed over every rank first, as
        torchmetrics' sync on compute does; every rank takes part even when it refused a step or ran none,
        and a refusal on any rank raises on all of them."""
        rc, err, counts, means, _ = self._read()
        dist = torch.distributed
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            comm_dev = self.device if dist.get_backend() == "nccl" else torch.device("cpu")
            vec = torch.tensor([1 if rc else 0] + ([0] * 11 if rc else counts), dtype=torch.int64, device=comm_dev)
            dist.all_reduce(vec)
            vec = vec.cpu().tolist()
            if rc:
                raise RuntimeError(f"samroad_val_read failed (code {rc}): {err}")
            if vec[0]:
                raise RuntimeError(f"{vec[0]} other rank(s) refused a validation step or could not report "
                                   "their counts (their own errors name the cause)")
            counts = vec[1:]
        elif rc:
            raise RuntimeError(f"samroad_val_read failed (code {rc}): {err}")
        c = dict(zip(VAL_COUNT_NAMES, counts))
        res = dict(zip(VAL_LOSS_NAMES, means))
        for name in ("keypoint", "road"):
            res[f"{name}_iou"] = iou_from_counts(c[f"{name}_tp"], c[f"{name}_fp"], c[f"{name}_fn"]).item()
        res["topo_f1"] = f1_from_counts(c["topo_tp"], c["topo_fp"], c["topo_fn"]).item()
        return res
