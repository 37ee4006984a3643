"""CPU: the embeddings-gradient entry points are bound and refuse bad arguments before touching a GPU, and the
oracle's d(loss)/d(image embeddings) is the unmodified reference's (tests/golden/emb_grad_vitb_256.npz, written by
tools/make_golden.py --emb-grad from the reference's training_step + loss.backward())."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import samroad_oracle as O
from oracle import train_oracle as TO
from sam_road_b200 import SAMRoad, _lib, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emb_grad_vitb_256.npz")


def _cfg(**kw):
    c = {"SAM_VERSION": "vit_b", "PATCH_SIZE": 256, "FREEZE_ENCODER": False, "TOPONET_VERSION": "normal"}
    c.update(kw)
    return c


def test_symbols_bound_and_refuse_without_gpu():
    lib = _lib.load()
    assert lib.samroad_abi_version() == 5
    a = _lib.SamRoadTrainArgs()
    assert lib.samroad_train_forward_embeddings(None, C.byref(a), None, None, 0, None, None, 0, None, 0, None, None,
                                                None, None, None, 0, None, None) != 0
    assert "null handle" in _lib.last_error()
    buf = (C.c_float * 4)()
    assert lib.samroad_train_backward_embeddings(None, C.byref(a), None, None, None, 0, None, 0, None,
                                                 C.addressof(buf), None) != 0
    assert "null handle" in _lib.last_error()
    # neither the weight gradients nor the embeddings gradient: refused before the handle is looked at
    assert lib.samroad_train_backward_embeddings(None, C.byref(a), None, None, None, 0, None, 0, None, None,
                                                 None) != 0
    assert "no gradient requested" in _lib.last_error()


def _batch():
    from tools.make_golden import train_heads_batch
    return train_heads_batch()


def test_head_losses_refuses_on_the_host():
    net = SAMRoad(_cfg())
    b = _batch()
    emb = torch.zeros(2, 256, 16, 16)
    with pytest.raises(RuntimeError, match="CUDA"):     # CPU heads: no CPU path
        net.head_losses(b, emb)
    with pytest.raises(NotImplementedError, match="USE_SAM_DECODER"):
        SAMRoad(_cfg(USE_SAM_DECODER=True)).head_losses(b, emb)


def _oracle_grads(tag, dtype):
    cfg = dict(_cfg(), FOCAL_LOSS=tag == "focal", USE_SAM_DECODER=False, ENCODER_LORA=False, NO_SAM=False)
    sd = synth.make_state_dict(cfg, seed=12, logit_gain=4.0)
    b = _batch()
    with torch.no_grad():
        emb = O.infer_masks_and_img_features(sd, O.ModelSpec.from_config(cfg), b["rgb"])[1]
    params = {k: v.to(dtype) for k, v in sd.items() if k.startswith(("map_decoder.", "topo_net."))}
    e = emb.to(dtype).requires_grad_(True)
    ml, tl = TO.heads_losses(params, e, b, 256, tag == "focal", "normal", None, 0.0)
    gm, = torch.autograd.grad(ml, e, retain_graph=True)
    g, = torch.autograd.grad(ml + tl, e)
    return emb, g, gm


@pytest.mark.parametrize("focal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_embeddings_gradient_is_the_references(focal, dtype):
    """The embeddings are recomputed by the fp32 encoder oracle, which agrees with the reference's within 2e-5
    (tests/test_oracle_golden.py); that difference bounds the match."""
    z = np.load(GOLDEN)
    tag = "focal" if focal else "bce"
    emb, g, gm = _oracle_grads(tag, dtype)
    d = emb.double()
    np.testing.assert_allclose([d.sum().item(), d.abs().sum().item(), (d * d).sum().item()], z[f"{tag}/emb_stats"],
                               rtol=1e-5)
    for grad, pre in ((g.double(), ""), (gm.double(), "mask_")):
        norm, mx = z[f"{tag}/{pre}norm_maxabs"]
        assert abs(grad.norm().item() - norm) <= 1e-4 * norm, (pre, grad.norm().item(), norm)
        assert abs(grad.abs().max().item() - mx) <= 1e-4 * mx, (pre, grad.abs().max().item(), mx)
        ts = grad.sum(1).numpy()
        ref = z[f"{tag}/{pre}texel_sum"]
        assert np.abs(ts - ref).max() <= 1e-4 * np.abs(ref).max(), pre
    mx = z[f"{tag}/norm_maxabs"][1]
    idx = torch.from_numpy(z[f"{tag}/idx"].astype(np.int64))
    assert np.abs(g.reshape(-1)[idx].double().numpy() - z[f"{tag}/val"]).max() <= 1e-4 * mx
    cs = g.double().sum((2, 3)).numpy()
    assert np.abs(cs - z[f"{tag}/channel_sum"]).max() <= 1e-4 * np.abs(z[f"{tag}/channel_sum"]).max()
