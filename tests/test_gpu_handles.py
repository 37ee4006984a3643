"""Native handle ownership: an allocation the device cannot satisfy is refused with an error naming the call and
leaves the handle usable, and every Python owner of a handle refuses copies, closes idempotently, refuses calls
once closed and releases the handle when it is collected."""
import copy
import ctypes as C
import gc
import pickle

import numpy as np
import pytest
import torch

from sam_road_b200 import _lib
from sam_road_b200 import apls_metric as AM
from sam_road_b200 import dataset as D
from sam_road_b200 import topo_metric as TM
from sam_road_b200.graph import SceneGraph
from sam_road_b200.metrics import PrecisionRecallCurve, ValidationMetrics
from test_gpu_labels_edges import _lc, _road_scene
from test_gpu_topo_limits import D as STEP, meridian, score

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _labels(cap=4096):
    ls = D.LabelScenes(_lc(P=128), 200, 0, cap, DEV)
    rng = np.random.RandomState(0)
    ls.upload(_road_scene(200, seed=4), rng.randint(0, 256, (200, 200, 3)).astype(np.uint8),
              rng.randint(0, 256, (200, 200)).astype(np.uint8), rng.randint(0, 256, (200, 200)).astype(np.uint8))
    return ls


def test_labels_batch_beyond_device_memory_then_a_normal_batch():
    # 2^30 patches of up to 4096 points need about 2^30 * 4096 * 64 bytes of work area: refused before any launch,
    # so the small dummy outputs are never touched
    ls = _labels()
    small = torch.zeros(64, dtype=torch.float32, device=DEV)
    n = C.c_int32()
    lib = _lib.load()
    launches = lib.samroad_launch_count(0)
    with torch.cuda.device(DEV):
        rc = lib.samroad_labels_batch(ls._h, 2 ** 30, 7, None, *([small.data_ptr()] * 7), C.byref(n),
                                      _lib.current_stream_ptr())
    assert rc != 0
    msg = _lib.last_error()
    assert "samroad_labels_batch" in msg and "out of device memory" in msg, msg
    assert lib.samroad_launch_count(0) == launches
    got = ls.batch(2, seed=11)
    want = _labels().batch(2, seed=11)
    for k in want:
        assert torch.equal(got[k], want[k]), k


def test_topo_run_beyond_device_memory_then_a_small_run():
    # 2^28 candidate edges per matching: 2 GB of match workspace per pair slot, so 1024 slots cannot fit
    d = TM.TopoDevice(0, max_candidates=2 ** 28, slots=1024)
    try:
        g = meridian(40)
        h = STEP / 2
        d.upload(0, g)
        d.upload(1, g)
        pn = np.array([[19, 20, 19, 20]] * 1024, dtype=np.int32)
        pd = np.full((1024, 4), h)
        with pytest.raises(RuntimeError, match="samroad_topo_run: out of device memory.*lower the slot count"):
            d.run(pn, pd, 12 * STEP, STEP / 4, STEP / 4)
        score(d, g, g, [[19, 20, 19, 20], [38, 39, 37, 38]], [[h] * 4] * 2, 12 * STEP, STEP / 4, STEP / 4)
    finally:
        d.close()


def _call_scene_graph(o):
    m = torch.zeros((32, 32), dtype=torch.uint8, device=DEV)
    o.extract_graph_points(m, m, 0.5, 0.5, 4, 4)


def _call_topo(o):
    o.upload(0, meridian(4))


def _call_apls(o):
    o.upload_csr(0, [(40.0, -70.0), (40.001, -70.0)], [0, 1, 2], [1, 0], [100, 100])


OWNERS = {
    "SceneGraph": (lambda: SceneGraph(DEV), _call_scene_graph),
    "TopoDevice": (lambda: TM.TopoDevice(0), _call_topo),
    "AplsDevice": (lambda: AM.AplsDevice(0), _call_apls),
    "LabelScenes": (lambda: _labels(), lambda o: o.batch(1, seed=0)),
    "PrecisionRecallCurve": (lambda: PrecisionRecallCurve(DEV), lambda o: o.reset()),
    "ValidationMetrics": (lambda: ValidationMetrics(DEV), lambda o: o.reset()),
}


@pytest.mark.parametrize("name", sorted(OWNERS))
def test_owner_refuses_copies(name):
    make, _ = OWNERS[name]
    o = make()
    try:
        for dup in (copy.copy, copy.deepcopy, pickle.dumps):
            with pytest.raises(TypeError):
                dup(o)
        with pytest.raises(TypeError):
            copy.copy(o._h)
    finally:
        o.close()


@pytest.mark.parametrize("name", sorted(OWNERS))
def test_owner_close_twice_then_a_call_is_refused(name):
    make, call = OWNERS[name]
    o = make()
    call(o)
    o.close()
    o.close()
    with pytest.raises(RuntimeError):
        call(o)


@pytest.mark.parametrize("name", sorted(OWNERS))
def test_owner_releases_its_handle_when_collected(name):
    make, _ = OWNERS[name]
    o = make()
    fin = o._h._finalizer
    assert fin.alive
    del o
    gc.collect()
    assert not fin.alive
