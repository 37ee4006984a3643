"""The visiting-order checks of the keypoint NMS passes (csrc/graph.cu), reached through wrong host
argsort callbacks.

`samroad_extract_graph_points` takes the visiting order of each of its three NMS passes from a host
callback (`samroad_argsort_fn`) and checks it on the device before using it: every index in range
(code 1) and the order non-increasing in the pass's key (code 2).  Each case hands it one wrong callback,
then makes a correct call on the same SceneGraph, which must still give the oracle's keypoints.  The
order made on the device without a callback (tie order "stable") is covered by test_gpu_graph.py."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200 import _lib  # noqa: E402
from sam_road_b200.graph import SceneGraph  # noqa: E402

DEV = "cuda:0"
RADII = (8.0, 16.0)
# thresholds >= 2/255 make every candidate immune: the three argsorts then run up front, side by side.
# Below that, each pass asks for its argsort when it starts.
THRESHOLDS = {"presorted": (0.9, 0.8), "per_pass": (0.5 / 255, 0.5 / 255)}


@pytest.fixture(scope="module")
def gx():
    return SceneGraph(DEV)


def _masks(regime):
    rng = np.random.RandomState(5)
    hi = 256 if regime == "presorted" else 4
    kp = rng.randint(0, hi, size=(96, 128)).astype(np.uint8)
    road = rng.randint(0, hi - 1, size=(96, 128)).astype(np.uint8)
    return kp, road


def _argsort_cb(tamper):
    """np.argsort as a samroad_argsort_fn; `tamper(key_dtype, asc)` may then edit `asc` and returns the status."""
    def cb(keys, key_dtype, n, order_out, user):
        try:
            ctype = C.c_uint8 if key_dtype == _lib.U8 else C.c_double
            asc = np.ctypeslib.as_array(order_out, shape=(n,))
            asc[:] = np.argsort(np.ctypeslib.as_array(C.cast(keys, C.POINTER(ctype)), shape=(n,)))
            return tamper(key_dtype, asc)
        except Exception:
            return 1
    return _lib.ARGSORT_FN(cb)


def _float64_identity(key_dtype, asc):
    # pass 3 sorts [1.0]*m0 + [0.0]*m1: the identity puts the road-mask entries first in the visit
    if key_dtype == _lib.F64:
        asc[:] = np.arange(asc.shape[0])
    return 0


def _out_of_range_for(n_road):
    def tamper(key_dtype, asc):
        if key_dtype == _lib.U8 and asc.shape[0] == n_road:
            asc[asc == 0] = n_road      # out of range, and the order stays non-increasing: code 1 only
        return 0
    return tamper


@pytest.mark.parametrize("regime", sorted(THRESHOLDS))
@pytest.mark.parametrize("case", ["float64_identity", "road_index_out_of_range", "failed_status",
                                  "float64_failed_status"])
def test_wrong_argsort_callback(gx, regime, case):
    kp, road = _masks(regime)
    thr = THRESHOLDS[regime]
    n_kp, n_road = int((kp > thr[0] * 255).sum()), int((road > thr[1] * 255).sum())
    assert n_kp != n_road            # the callback tells the two masks apart by their sizes
    tamper, want = {
        "float64_identity": (_float64_identity, "invalid permutation (code 2) for the merged pass"),
        "road_index_out_of_range": (_out_of_range_for(n_road), "invalid permutation (code 1) for mask 1"),
        "failed_status": (lambda key_dtype, asc: 3, "argsort callback failed"),
        # fails the merged pass only: its own message, or the third status of the up-front sorts
        "float64_failed_status": (lambda key_dtype, asc: 3 if key_dtype == _lib.F64 else 0,
                                  "argsort callback failed (float64 priorities)" if regime == "per_pass"
                                  else "argsort callback failed (0 0 3)"),
    }[case]
    cb = _argsort_cb(tamper)
    kp_d, road_d = torch.as_tensor(kp).to(DEV), torch.as_tensor(road).to(DEV)
    H, W = kp.shape
    out = torch.empty((H * W, 2), dtype=torch.int64, device=DEV)
    n = C.c_int(0)
    stats = (C.c_int32 * 16)()
    with torch.cuda.device(gx.device):
        rc = _lib.load().samroad_extract_graph_points(
            gx._h, kp_d.data_ptr(), road_d.data_ptr(), H, W, thr[0] * 255, thr[1] * 255, RADII[0], RADII[1], cb,
            None, out.data_ptr(), H * W, C.byref(n), stats, _lib.current_stream_ptr())
    assert rc != 0 and want in _lib.last_error(), (rc, _lib.last_error())

    mine = gx.extract_graph_points(kp_d, road_d, thr[0], thr[1], RADII[0], RADII[1], tie_order="numpy")
    ref = O.extract_graph_points(kp, road, thr[0], thr[1], RADII[0], RADII[1], "numpy")
    assert np.array_equal(mine.cpu().numpy(), ref)
    assert min(gx.stats["pass_survivors"]) > 0       # pass 3 holds entries of both classes
