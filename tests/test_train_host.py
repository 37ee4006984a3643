"""CPU: the heads' training oracle (oracle/train_oracle.py) against torch's own modules, configure_optimizers,
the refusal of configurations without a backward, and the argument checks of the samroad_train_* calls."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
from torch import nn

from oracle import train_oracle as TO
from sam_road_b200 import SAMRoad, _lib, synth
from sam_road_b200.train import dropout_keep  # noqa: F401  (import check: the module loads without a GPU)

P = 64


def _cfg(**kw):
    c = {"SAM_VERSION": "vit_b", "PATCH_SIZE": P, "FREEZE_ENCODER": True, "BASE_LR": 1e-3,
         "TOPONET_VERSION": "normal"}
    c.update(kw)
    return c


class _LayerNorm2d(nn.Module):   # segment_anything's LayerNorm2d
    def __init__(self, c):
        super().__init__()
        self.weight, self.bias = nn.Parameter(torch.ones(c)), nn.Parameter(torch.zeros(c))

    def forward(self, x):
        u = x.mean(1, keepdim=True)
        s = (x - u).pow(2).mean(1, keepdim=True)
        x = (x - u) / torch.sqrt(s + 1e-6)
        return self.weight[:, None, None] * x + self.bias[:, None, None]


class _Heads(nn.Module):
    """The reference's map_decoder and TopoNet built from torch modules (model.py:61-148, 286-295)."""

    def __init__(self, version):
        super().__init__()
        self.version = version
        self.map_decoder = nn.Sequential(nn.ConvTranspose2d(256, 128, 2, 2), _LayerNorm2d(128), nn.GELU(),
                                         nn.ConvTranspose2d(128, 64, 2, 2), nn.GELU(),
                                         nn.ConvTranspose2d(64, 32, 2, 2), nn.GELU(), nn.ConvTranspose2d(32, 2, 2, 2))
        t = nn.Module()
        t.feature_proj, t.pair_proj = nn.Linear(256, 128), nn.Linear(258, 128)
        if version != "no_transformer":
            layer = nn.TransformerEncoderLayer(128, 4, 128, 0.1, "relu", batch_first=True)
            t.transformer_encoder = nn.TransformerEncoder(layer, 3)
        t.output_proj = nn.Linear(128, 1)
        self.topo_net = t

    def losses(self, emb, b, focal):
        ml = TO.mask_loss(self.map_decoder(emb).permute(0, 2, 3, 1), b["keypoint_mask"], b["road_mask"], focal)
        pts = b["graph_points"].float()
        B, Ns, Np, _ = b["pairs"].shape
        f = torch.nn.functional.grid_sample(emb, (pts / P * 2 - 1).unsqueeze(2), align_corners=False)
        pf = torch.relu(self.topo_net.feature_proj(f.squeeze(-1).permute(0, 2, 1)))
        pr = b["pairs"].view(B, -1, 2)
        bi = torch.arange(B).view(-1, 1).expand(-1, Ns * Np)
        off = pts[bi, pr[:, :, 1]] - pts[bi, pr[:, :, 0]]
        if self.version == "no_offset":
            off = torch.zeros_like(off)
        x = torch.relu(self.topo_net.pair_proj(torch.cat([pf[bi, pr[:, :, 0]], pf[bi, pr[:, :, 1]], off], 2)))
        x = x.view(B * Ns, Np, -1)
        v = b["valid"].view(B * Ns, Np)
        v = torch.logical_or(v, torch.eq(v.sum(-1), 0).unsqueeze(-1))
        if self.version != "no_transformer":
            x = self.topo_net.transformer_encoder(x, src_key_padding_mask=~v)
        lg = self.topo_net.output_proj(x).view(B, Ns, Np)
        return ml, TO.topo_loss(lg, b["connected"], b["valid"])


def _batch(B, N, Ns, Np, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randint(0, P + 1, (B, N, 2), generator=g)
    pairs = torch.randint(0, N, (B, Ns, Np, 2), generator=g)
    valid = torch.rand((B, Ns, Np), generator=g) < 0.7
    valid[0, 1] = False                                    # an all-invalid sample row
    return {"graph_points": pts, "pairs": pairs, "valid": valid,
            "connected": torch.rand((B, Ns, Np), generator=g) < 0.4,
            "keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
            "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}


@pytest.mark.parametrize("version,focal,Np", [("normal", False, 7), ("no_offset", True, 16),
                                              ("no_transformer", False, 5)])
def test_oracle_matches_torch_modules(version, focal, Np):
    torch.manual_seed(0)
    ref = _Heads(version).eval()       # eval + grad enabled: dropout off, torch's slow path
    params = {k: p.detach().clone().requires_grad_(True) for k, p in ref.named_parameters()}
    emb = torch.randn(2, 256, P // 16, P // 16)
    b = _batch(2, 9, 6, Np, seed=Np)
    ml, tl = ref.losses(emb, b, focal)
    (ml + tl).backward()
    oml, otl = TO.heads_losses(params, emb, b, P, focal, version)
    (oml + otl).backward()
    torch.testing.assert_close(oml, ml, rtol=1e-6, atol=0)
    torch.testing.assert_close(otl, tl, rtol=1e-6, atol=0)
    for k, p in ref.named_parameters():
        g, r = params[k].grad, p.grad
        assert g is not None, k
        assert (g - r).abs().max() <= 1e-5 * r.abs().max() + 1e-12, k
    if version == "no_offset":
        assert (params["topo_net.pair_proj.weight"].grad[:, 256:] == 0).all()


@pytest.mark.parametrize("version,counts", [("normal", (172770, 364929)), ("no_transformer", (172770, 66177))])
def test_configure_optimizers(version, counts, capsys):
    net = SAMRoad(_cfg(TOPONET_VERSION=version, BASE_LR=5e-4))
    out = net.configure_optimizers()
    opt, sch = out["optimizer"], out["lr_scheduler"]
    assert set(out) == {"optimizer", "lr_scheduler"}
    assert isinstance(opt, torch.optim.Adam) and isinstance(sch, torch.optim.lr_scheduler.MultiStepLR)
    assert [g["lr"] for g in opt.param_groups] == [5e-4, 5e-4]
    assert dict(sch.milestones) == {9: 1} and sch.gamma == 0.1
    named = dict(net.named_parameters())
    ids = [{id(p) for p in g["params"]} for g in opt.param_groups]
    assert ids[0] == {id(p) for k, p in named.items() if k.startswith("map_decoder.")}
    assert ids[1] == {id(p) for k, p in named.items() if k.startswith("topo_net.")}
    printed = capsys.readouterr().out
    for i, n in enumerate(counts):
        assert f"optim param dict {i} params num: {n}" in printed
    for k, p in named.items():   # heads are trained, the encoder stays frozen
        assert p.requires_grad == k.startswith(("map_decoder.", "topo_net.")), k


@pytest.mark.parametrize("cfg,key", [({"FREEZE_ENCODER": False}, "FREEZE_ENCODER"),
                                     ({"FREEZE_ENCODER": None}, "FREEZE_ENCODER"),
                                     ({"ENCODER_LORA": True, "LORA_RANK": 4}, "ENCODER_LORA"),
                                     ({"USE_SAM_DECODER": True}, "USE_SAM_DECODER")])
def test_unsupported_configs_raise_before_the_batch(cfg, key):
    net = SAMRoad(_cfg(**cfg))
    with pytest.raises(NotImplementedError, match=key):
        net.training_step(None, 0)
    with pytest.raises(NotImplementedError, match=key):
        net.configure_optimizers()
    assert not any(p.requires_grad for p in net.parameters())


def test_train_symbols_reject_bad_arguments_without_gpu():
    lib = _lib.load()
    a = _lib.SamRoadTrainArgs()
    a.B, a.N, a.Ns, a.Np = 1, 4, 4, 33
    n = C.c_size_t()
    assert lib.samroad_train_workspace_bytes(None, C.byref(a), C.byref(n)) != 0
    assert "null handle" in _lib.last_error()
    assert lib.samroad_train_workspace_bytes(None, C.byref(a), None) != 0
    assert lib.samroad_train_forward(None, C.byref(a), None, None, 0, None, 0, None, 0, None, 0, None, None, None,
                                     None, None, 0, None, None, None) != 0
    assert lib.samroad_train_backward(None, C.byref(a), None, None, None, 0, None, 0, None, None) != 0
    shape = (C.c_int64 * 1)(128)
    assert lib.samroad_update_tensor_device(None, b"map_decoder.1.weight", None, shape, 1, None) != 0
    assert "null samroad handle" in _lib.last_error()
    buf = (C.c_uint8 * 16)()
    for p, layer, site in ((1.0, 0, 0), (-0.1, 0, 0), (0.1, 3, 0), (0.1, 0, 4)):
        assert lib.samroad_debug_train_dropout_keep(p, 0, layer, site, 16, C.addressof(buf), None) != 0
        assert "layer=" in _lib.last_error()


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_heads_vitb_256.npz")


def _check_reference_training_step(focal, dtype):
    from oracle import samroad_oracle as O
    from tools.make_golden import train_heads_batch
    z = np.load(GOLDEN)
    tag = "focal" if focal else "bce"
    cfg = dict(_cfg(PATCH_SIZE=256), FOCAL_LOSS=focal, USE_SAM_DECODER=False, ENCODER_LORA=False, NO_SAM=False)
    sd = synth.make_state_dict(cfg, seed=12, logit_gain=4.0)
    b = train_heads_batch()
    with torch.no_grad():
        emb = O.infer_masks_and_img_features(sd, O.ModelSpec.from_config(cfg), b["rgb"])[1]
    d = emb.double()
    np.testing.assert_allclose([d.sum().item(), d.abs().sum().item(), (d * d).sum().item()], z[f"{tag}/emb_stats"],
                               rtol=1e-5)
    params = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items() if k.startswith(("map_decoder.", "topo_net."))}
    ml, tl = TO.heads_losses(params, emb.to(dtype), b, 256, focal, "normal", None, 0.0)
    assert ml.dtype == tl.dtype == dtype
    (ml + tl).backward()
    np.testing.assert_allclose([ml.item(), tl.item(), (ml + tl).item()], z[f"{tag}/losses"], rtol=1e-5)
    for k, p in params.items():
        g = p.grad.reshape(-1)
        norm, mx = z[f"{tag}/{k}/norm_maxabs"]
        assert abs(g.double().norm().item() - norm) <= 1e-4 * norm + 1e-30, k
        assert abs(g.abs().max().item() - mx) <= 1e-4 * mx + 1e-30, k
        idx = torch.from_numpy(z[f"{tag}/{k}/idx"].astype(np.int64))
        assert np.abs(g[idx].numpy() - z[f"{tag}/{k}/val"]).max() <= 1e-4 * mx + 1e-30, k
    assert list(z[f"{tag}/param_counts"]) == [172770, 364929]     # the reference's printed group sizes


@pytest.mark.parametrize("focal", [False, True])
def test_oracle_reproduces_reference_training_step(focal):
    """tests/golden/train_heads_vitb_256.npz holds the unmodified reference's training_step + loss.backward()
    (tools/make_golden.py --train-heads).  The embeddings are recomputed here by the fp32 encoder oracle, which
    agrees with the reference's within 2e-5 (tests/test_oracle_golden.py); that difference bounds the match."""
    _check_reference_training_step(focal, torch.float32)


@pytest.mark.parametrize("focal", [False, True])
def test_float64_oracle_reproduces_reference_training_step(focal):
    """The same step with the embeddings and the head parameters cast to float64: the float64 oracle, which the
    GPU tests measure the device gradients against, computes the reference's training step."""
    _check_reference_training_step(focal, torch.float64)


def test_enable_training_once():
    net = SAMRoad(_cfg())
    net.configure_optimizers()
    p = dict(net.named_parameters())["topo_net.output_proj.bias"]
    p.requires_grad_(False)               # a head the user freezes stays frozen
    net.configure_optimizers()
    assert not p.requires_grad


def test_synth_state_dict_keeps_training_off():
    net = SAMRoad(_cfg())
    net.load_state_dict(synth.make_state_dict(_cfg()))
    assert not any(p.requires_grad for p in net.parameters())
