"""GPU: samroad_finalize_weights and samroad_update_tensor_device pack through one list of regions and one kernel
(csrc/model.cu, packed_regions / pack_kernel).

A device refresh of every head tensor must give the bytes a fresh pack of the same values gives, for each TopoNet
version (both sides run the same packing kernel, so this checks which regions and offsets a key reaches, not the
layouts themselves: the golden and oracle tests check those); a refused refresh launches nothing; a failed finalize returns 3 and leaves the handle without weights,
also when it follows a successful one."""
import ctypes

import pytest
import torch

from sam_road_b200 import SAMRoad, _lib, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
P = 256


def _cfg(version="normal", sam_decoder=False):
    return dict(SAM_VERSION="vit_b", PATCH_SIZE=P, USE_SAM_DECODER=sam_decoder, ENCODER_LORA=False,
                TOPONET_VERSION=version, NO_SAM=False)


def _is_head(key):
    return key.startswith(("map_decoder.", "topo_net."))


def _net(cfg, sd):
    net = SAMRoad(cfg)
    net.load_state_dict(sd)
    return net.eval().to(DEV)


def _outputs(net):
    rgb = synth.make_tiles(2, P, seed=3).to(DEV)
    pts, pairs, valid = synth.make_topo_inputs(2, P, 40, seed=4)
    scores, emb = net.infer_masks_and_img_features(rgb)
    topo = net.infer_toponet(emb, pts.to(DEV), pairs.to(DEV), valid.to(DEV))
    return scores, emb, topo


def _update(h, key, t):
    shape = (ctypes.c_int64 * t.dim())(*t.shape)
    return _lib.load().samroad_update_tensor_device(h, key.encode(), t.data_ptr(), shape, t.dim(),
                                                    _lib.current_stream_ptr())


@pytest.mark.parametrize("version", ["normal", "no_offset", "no_transformer"])
def test_refresh_equals_fresh_pack(version):
    cfg = _cfg(version)
    sd_a = synth.make_state_dict(cfg, seed=0, logit_gain=4.0)
    heads_b = {k: v for k, v in synth.make_state_dict(cfg, seed=1, logit_gain=4.0).items() if _is_head(k)}
    a, b = _net(cfg, sd_a), _net(cfg, {**sd_a, **heads_b})   # same encoder, other heads
    before = _outputs(a)
    h = a._handle(DEV)
    keys = [k for k, _ in a._head_params()]
    assert sorted(keys) == sorted(heads_b)
    assert not any(p.requires_grad for _, p in a._head_params())   # so a's calls do not repack its own values
    for k in keys:
        _lib.check(_update(h, k, heads_b[k].to(DEV)), k)
    got, want = _outputs(a), _outputs(b)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert not torch.equal(before[0], want[0]) and not torch.equal(before[2], want[2])


def test_refusals_launch_nothing():
    lib = _lib.load()
    sd = synth.make_state_dict(_cfg(), seed=0)
    h = _net(_cfg(), sd)._handle(DEV)
    cfg_nt = _cfg("no_transformer")
    h_nt = _net(cfg_nt, synth.make_state_dict(cfg_nt, seed=0))._handle(DEV)
    cfg_sam = _cfg(sam_decoder=True)
    h_sam = _net(cfg_sam, synth.make_state_dict(cfg_sam, seed=0))._handle(DEV)
    layer = "topo_net.transformer_encoder.layers.0.linear1.weight"
    cases = [
        (h, "image_encoder.neck.1.weight", sd["image_encoder.neck.1.weight"],
         "'image_encoder.neck.1.weight' is not a head tensor of this configuration"),
        (h, "topo_net.no_such.weight", torch.zeros(128),
         "'topo_net.no_such.weight' is not a head tensor of this configuration"),
        (h, "topo_net.transformer_encoder.layers.3.linear1.weight", torch.zeros(128, 128),
         "'topo_net.transformer_encoder.layers.3.linear1.weight' is not a head tensor of this configuration"),
        (h, "map_decoder.1.weight", torch.zeros(64), "'map_decoder.1.weight' has the wrong shape"),
        (h, "topo_net.pair_proj.weight", torch.zeros(128, 256), "'topo_net.pair_proj.weight' has the wrong shape"),
        (h_nt, layer, sd[layer], f"'{layer}' is not a head tensor of this configuration"),
        (h_sam, "topo_net.feature_proj.bias", sd["topo_net.feature_proj.bias"],
         "the SAM mask decoder is repacked on the host only"),
    ]
    for handle, key, t, msg in cases:
        torch.cuda.synchronize()
        n0 = lib.samroad_launch_count(0)
        rc = _update(handle, key, t.to(DEV).contiguous())
        assert rc != 0 and msg in _lib.last_error(), (key, rc, _lib.last_error())
        assert lib.samroad_launch_count(0) == n0, key


def _raw_handle():
    """A ViT-B handle at PATCH_SIZE 256 with nothing loaded."""
    cfg = _lib.SamRoadCfg()
    cfg.patch_size, cfg.embed_dim, cfg.depth, cfg.num_heads, cfg.window_size = P, 768, 12, 12, 14
    for i, g in enumerate((2, 5, 8, 11)):
        cfg.global_attn_indexes[i] = g
    return _lib.Handle("samroad_create", "samroad_destroy", ctypes.byref(cfg), 0)


def _load(h, sd):
    lib = _lib.load()
    for k, v in sd.items():
        t = v.to(torch.float32).contiguous()
        shape = (ctypes.c_int64 * t.dim())(*t.shape)
        _lib.check(lib.samroad_load_tensor(h, k.encode(), t.data_ptr(), shape, t.dim()), k)


def _encode(h):
    rgb = synth.make_tiles(1, P, seed=5).to(DEV)
    emb = torch.empty((1, 256, P // 16, P // 16), device=DEV)
    rc = _lib.load().samroad_encode_masks(h, rgb.data_ptr(), _lib.U8, 1, None, None, emb.data_ptr(),
                                          _lib.current_stream_ptr())
    torch.cuda.synchronize()
    return rc


def _finalize_fails(h, msg):
    rc = _lib.load().samroad_finalize_weights(h)
    assert rc == 3 and msg in _lib.last_error(), (rc, _lib.last_error())
    assert _encode(h) != 0 and "weights not finalized" in _lib.last_error()


def test_finalize_errors():
    sd = synth.make_state_dict(_cfg(), seed=0)
    h = _raw_handle()
    _load(h, {k: v for k, v in sd.items() if k != "map_decoder.3.weight"})
    _finalize_fails(h, "missing state_dict key 'map_decoder.3.weight'")
    _load(h, {"map_decoder.3.weight": sd["map_decoder.3.weight"][:, :32]})
    _finalize_fails(h, "state_dict key 'map_decoder.3.weight' has shape [128,32,2,2,] but [128,64,2,2,] is required")
    _load(h, {"map_decoder.3.weight": sd["map_decoder.3.weight"]})
    _lib.check(_lib.load().samroad_finalize_weights(h), "samroad_finalize_weights")
    assert _encode(h) == 0, _lib.last_error()
    h.close()


def test_second_finalize_without_loads_unfinalizes():
    """A finalize empties the staged tensors, so a second one fails; it must not leave the handle marked
    finalized with its weights freed."""
    h = _raw_handle()
    _load(h, synth.make_state_dict(_cfg(), seed=0))
    _lib.check(_lib.load().samroad_finalize_weights(h), "samroad_finalize_weights")
    assert _encode(h) == 0, _lib.last_error()
    _finalize_fails(h, "missing state_dict key")
    h.close()
