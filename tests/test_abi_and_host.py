"""CPU: the C-ABI library loads and exports every symbol include/samroad_b200.h declares (no compute
calls without a GPU), and the host-side mirror of the reference interface behaves like the reference
(state_dict key set, config handling, error behaviour)."""
import ctypes
import os
import re

import pytest
import torch

from sam_road_b200 import SAMRoad, _lib, synth
from sam_road_b200.model import param_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "samroad_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(samroad_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/samroad_b200.h but not exported"
    assert set(_lib.SIGNATURES) == set(names), set(_lib.SIGNATURES) ^ set(names)
    bound = _lib.load()
    # the version is written in the header and in _lib.py; the library must report both
    src = open(os.path.join(ROOT, "include", "samroad_b200.h")).read()
    header_version = int(re.search(r"#define SAMROAD_ABI_VERSION (\d+)", src).group(1))
    assert bound.samroad_abi_version() == _lib.ABI_VERSION == header_version


@pytest.mark.parametrize("act", [3, 100])
def test_gemm_rejects_unknown_activation(act):
    # the activation is checked before any CUDA call, so this needs no GPU
    lib = _lib.load()
    rc = lib.samroad_op_gemm_f16(None, 64, None, 64, 128, 128, 64, None, act, None, 128, None)
    assert rc != 0 and f"act={act}" in _lib.last_error()
    rc = lib.samroad_op_gemm_ln(None, 64, None, 64, 128, 128, 64, None, None, None, None, 1e-6, 128, act,
                                None, None, None, 1, 128, None)
    assert rc != 0 and f"act={act}" in _lib.last_error()


def test_sam_decoder_hook_rejects_null_handle():
    # the handle is checked before any CUDA call, so this needs no GPU
    lib = _lib.load()
    out = ctypes.c_void_p(16)
    assert lib.samroad_op_sam_decoder(None, out, 1, None, None, None, None, out, out, None) != 0
    assert "null samroad handle" in _lib.last_error()
    assert lib.samroad_op_sam_decoder(None, None, 0, None, None, None, None, None, None, None) != 0
    assert "null samroad handle" in _lib.last_error()


def test_cfg_struct_matches_header():
    src = open(os.path.join(ROOT, "include", "samroad_b200.h")).read()
    body = re.search(r"typedef struct SamRoadCfg \{(.*?)\} SamRoadCfg;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"int32_t\s+([a-z_]+)(\[\d+\])?;", body)
    assert [f[0] for f in fields] == [f[0] for f in _lib.SamRoadCfg._fields_]
    assert ctypes.sizeof(_lib.SamRoadCfg) == 4 * (len(fields) + 3)


def test_error_reporting_without_gpu():
    lib = _lib.load()
    if torch.cuda.is_available():
        pytest.skip("needs a machine without CUDA devices")
    cfg = _lib.SamRoadCfg()
    cfg.patch_size, cfg.embed_dim, cfg.depth, cfg.num_heads, cfg.window_size = 256, 768, 12, 12, 14
    h = ctypes.c_void_p()
    rc = lib.samroad_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    assert rc != 0 and len(_lib.last_error()) > 0      # no CPU fallback: creating a handle fails loudly
    cfg.patch_size = 250
    assert lib.samroad_create(ctypes.byref(cfg), 0, ctypes.byref(h)) != 0
    assert "PATCH_SIZE" in _lib.last_error()


@pytest.mark.parametrize("version,patch,lora,topo", [("vit_b", 256, 0, "normal"), ("vit_b", 512, 4, "normal"),
                                                     ("vit_l", 256, 0, "no_transformer"),
                                                     ("vit_h", 256, 0, "normal")])
def test_state_dict_key_set(version, patch, lora, topo):
    cfg = dict(SAM_VERSION=version, PATCH_SIZE=patch, ENCODER_LORA=lora > 0, LORA_RANK=lora,
               TOPONET_VERSION=topo)
    shapes = param_shapes(cfg)
    D = {"vit_b": 768, "vit_l": 1024, "vit_h": 1280}[version]
    depth = {"vit_b": 12, "vit_l": 24, "vit_h": 32}[version]
    s = patch // 16
    assert shapes["image_encoder.pos_embed"] == (1, s, s, D)
    assert shapes[f"image_encoder.blocks.{depth - 1}.attn.qkv.weight"] == (3 * D, D)
    glob = {"vit_b": 2, "vit_l": 5, "vit_h": 7}[version]
    assert shapes[f"image_encoder.blocks.{glob}.attn.rel_pos_h"][0] == 2 * s - 1
    assert shapes["image_encoder.blocks.0.attn.rel_pos_h"][0] == 27
    assert ("topo_net.transformer_encoder.layers.0.linear1.weight" in shapes) == (topo != "no_transformer")
    assert ("image_encoder.blocks.0.attn.qkv.linear_a_q.weight" in shapes) == (lora > 0)
    n_params = sum(int(torch.tensor(v).prod()) for v in shapes.values())
    if version == "vit_b" and lora == 0 and patch == 256:
        assert abs(n_params - 87.2e6) < 0.2e6      # SURVEY.md §8b: ViT-B 87.2 M at 256


def test_samroad_module_mirrors_reference_interface(tmp_path):
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False)
    net = SAMRoad(cfg)
    sd = synth.make_state_dict(cfg, seed=0)
    assert set(net.state_dict().keys()) == set(sd.keys())
    res = net.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    with pytest.raises(RuntimeError):
        bad = dict(sd); bad.pop("topo_net.output_proj.bias")
        net.load_state_dict(bad, strict=True)
    for name in ("forward", "infer_masks_and_img_features", "infer_toponet"):
        assert callable(getattr(net, name))
    with pytest.raises(RuntimeError, match="CUDA"):     # no CPU path
        net.infer_masks_and_img_features(torch.zeros(1, 256, 256, 3))
    with pytest.raises(NotImplementedError):            # same as the reference, model.py:232-242
        SAMRoad(dict(cfg, NO_SAM=True))
    # SAM_CKPT_PATH: name+shape matches are loaded, pos_embed / global rel-pos resized (model.py:367-411)
    ck = {"image_encoder.pos_embed": torch.randn(1, 64, 64, 768),
          "image_encoder.blocks.2.attn.rel_pos_h": torch.randn(127, 64),
          "image_encoder.blocks.0.attn.rel_pos_h": torch.randn(27, 64),
          "image_encoder.blocks.0.norm1.weight": torch.full((768,), 2.0),
          "mask_decoder.iou_token.weight": torch.zeros(1, 256)}
    path = tmp_path / "sam.pth"
    torch.save(ck, path)
    net2 = SAMRoad(dict(cfg, SAM_CKPT_PATH=str(path)))
    got = net2.state_dict()
    assert torch.all(got["image_encoder.blocks.0.norm1.weight"] == 2.0)
    assert got["image_encoder.pos_embed"].abs().sum() > 0 and got["image_encoder.blocks.2.attn.rel_pos_h"].shape == (31, 64)
    assert "image_encoder.blocks.0.attn.rel_pos_h" in net2.matched_param_names


def test_sam_decoder_state_dict_keys():
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=True)
    net = SAMRoad(cfg)
    sd = synth.make_state_dict(cfg, seed=0)
    keys = set(net.state_dict().keys())
    assert keys == set(sd.keys()) and len(keys) == 350
    assert "prompt_encoder.pe_layer.positional_encoding_gaussian_matrix" in keys      # persistent buffer
    assert "map_decoder.0.weight" not in keys and "mask_decoder.iou_token.weight" in keys
    assert not net.load_state_dict(sd, strict=True).missing_keys


def test_addict_style_config_missing_keys():
    class Cfg(dict):
        def __getattr__(self, k):
            return self.get(k, Cfg())
    cfg = Cfg(SAM_VERSION="vit_b", PATCH_SIZE=256)     # toponet_vitb_256.yaml lacks NO_SAM, TOPONET_VERSION...
    net = SAMRoad(cfg)
    assert net.image_size == 256
