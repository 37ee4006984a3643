"""CPU: the oracle restatement against golden fixtures produced by the UNMODIFIED reference
(tests/golden/README.md).  This is what pins the oracle used by every GPU parity test."""
import os

import numpy as np
import pytest
import torch

from oracle import samroad_oracle as O
from sam_road_b200 import synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5


def _cfg(patch, topo="normal", lora=0, samdec=False, version="vit_b"):
    return dict(SAM_VERSION=version, PATCH_SIZE=patch, USE_SAM_DECODER=samdec, ENCODER_LORA=lora > 0,
                LORA_RANK=lora, TOPONET_VERSION=topo, NO_SAM=False)


def _stats(t):
    d = t.double()
    return np.array([d.sum().item(), d.abs().sum().item(), (d * d).sum().item()])


@pytest.mark.parametrize("name,patch,lora", [("vitb_256", 256, 0), ("vitb_512", 512, 0),
                                             ("vitb_256_lora4", 256, 4), ("vitb_256_samdec", 256, 0),
                                             ("vith_256", 256, 0), ("vitl_256", 256, 0),
                                             ("vitb_1024", 1024, 0),
                                             ("vitb_400", 400, 0),            # odd 25x25 grid
                                             ("vitb_192_samdec", 192, 0)])    # 12x12 grid < 14x14 window
def test_model_against_reference_golden(name, patch, lora):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    cfg = _cfg(patch, lora=lora, samdec=name.endswith("samdec"),
               version={"vith": "vit_h", "vitl": "vit_l"}.get(name[:4], "vit_b"))
    seed, n_points = int(g["seed"]), int(g["n_points"])
    sd = synth.make_state_dict(cfg, seed=seed)
    spec = O.ModelSpec.from_config(cfg)
    rgb = synth.make_tiles(1, patch, seed=seed + 21, dtype=torch.float32)
    pts, prs, val = synth.make_topo_inputs(1, patch, n_points, seed=seed + 22)
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    with torch.no_grad():
        logits, scores, t_logits, t_scores = O.forward(sd, spec, rgb, pts, prs, val)
        _, feat = O.infer_masks_and_img_features(sd, spec, rgb)
    assert np.abs(logits[0, ::8, ::8, :].numpy() - g["mask_logits_sub"]).max() < TOL
    assert np.abs(scores[0, ::8, ::8, :].numpy() - g["mask_scores_sub"]).max() < TOL
    assert np.abs(feat[0, ::8, ::2, ::2].numpy() - g["feat_sub"]).max() < 5 * TOL
    assert np.abs(t_logits.numpy() - g["topo_logits"]).max() < TOL
    assert np.abs(t_scores.numpy() - g["topo_scores"]).max() < TOL
    for got, key in ((logits, "mask_logits_stats"), (feat, "feat_stats"), (t_logits, "topo_logits_stats")):
        assert np.allclose(_stats(got), g[key], rtol=1e-5, atol=1e-3), key
    assert float(g["oracle_vs_reference_maxabs"].max()) < TOL


@pytest.mark.parametrize("topo", ["normal", "no_offset", "no_transformer", "no_tgt_features"])
def test_toponet_versions_against_reference_golden(topo):
    g = np.load(os.path.join(GOLD, "toponet_versions.npz"))
    cfg = _cfg(256, topo=topo)
    sd = synth.make_state_dict(cfg, seed=5)
    spec = O.ModelSpec.from_config(cfg)
    gen = torch.Generator().manual_seed(77)
    feat = torch.randn(2, 256, 16, 16, generator=gen)
    pts, prs, val = synth.make_topo_inputs(2, 256, 20, seed=9)
    val[1, 3] = False
    pts[0, 0] = torch.tensor([256, 256])
    with torch.no_grad():
        a = O.infer_toponet(sd, spec, feat, pts, prs, val)
        b = O.infer_toponet(sd, spec, feat, pts.float() + 0.25, prs, val)
    assert np.abs(a.numpy() - g[f"{topo}_int"]).max() < TOL
    assert np.abs(b.numpy() - g[f"{topo}_float"]).max() < TOL


@pytest.mark.parametrize("n_pairs", [1, 5, 15])
def test_toponet_npairs_against_reference_golden(n_pairs):
    """n_pairs != 16 (the layered CUDA TopoNet path) with pairs / valid covering fewer samples than
    there are points (Ns = 13, N = 20); inputs as tools/make_golden.py:toponet_npairs_inputs."""
    g = np.load(os.path.join(GOLD, "toponet_npairs.npz"))
    cfg = _cfg(256)
    sd = synth.make_state_dict(cfg, seed=5)
    spec = O.ModelSpec.from_config(cfg)
    gen = torch.Generator().manual_seed(78)
    feat = torch.randn(2, 256, 16, 16, generator=gen)
    pts, prs, val = synth.make_topo_inputs(2, 256, 20, seed=10 + n_pairs, max_nbr=n_pairs)
    prs, val = prs[:, :13].contiguous(), val[:, :13].contiguous()
    val[1, 3] = False
    with torch.no_grad():
        a = O.infer_toponet(sd, spec, feat, pts, prs, val)
        b = O.infer_toponet(sd, spec, feat, pts.float() + 0.25, prs, val)
    assert a.shape == g[f"np{n_pairs}_int"].shape == (2, 13, n_pairs, 1)
    assert np.abs(a.numpy() - g[f"np{n_pairs}_int"]).max() < TOL
    assert np.abs(b.numpy() - g[f"np{n_pairs}_float"]).max() < TOL


def test_tile_grid_and_keypoints_against_reference_golden():
    g = np.load(os.path.join(GOLD, "tileloop.npz"))
    for tag, args in {"c2_cityscale_16": (0, 2048, 64, 512, 16), "c4_cityscale_8": (0, 2048, 64, 512, 8),
                      "c3_spacenet_16": (0, 400, 0, 256, 16), "spacenet_4": (0, 400, 0, 256, 4)}.items():
        mine = np.array([[x0, y0, x1, y1] for _, (x0, y0), (x1, y1) in O.get_patch_info_one_img(*args)])
        assert np.array_equal(mine, g[f"tiles_{tag}"]), tag
    pts = O.extract_graph_points(g["kp_mask"], g["road_mask"], 0.3, 0.4, 8, 16)
    from numpy._core._multiarray_umath import __cpu_features__ as feat
    if feat.get("AVX512_SKX", False):     # the fixture's tie order is the AVX-512 argsort's (oracle.visiting_order)
        assert np.array_equal(pts, g["graph_points"])
    assert pts.shape[0] > 0 and abs(pts.shape[0] - g["graph_points"].shape[0]) <= 0.1 * g["graph_points"].shape[0]


def test_oracle_internal_consistency():
    """window attention with padding == attention on the unpadded grid when nothing is padded, and
    fuse_masks equals a float64 recomputation within one uint8 step."""
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(1, 28, 28, 64, generator=gen)
    w, pad = O.window_split(x, 14)
    assert w.shape == (4, 14, 14, 64) and pad == (28, 28)
    assert torch.equal(O.window_merge(w, 14, pad, (28, 28)), x)
    tiles = O.get_patch_info_one_img(0, 64, 0, 32, 3)
    sc = [np.random.RandomState(i).rand(32, 32, 2).astype(np.float32) for i in range(len(tiles))]
    kp, road = O.fuse_masks(sc, tiles, 64, 64)
    acc = np.zeros((64, 64, 2)); cnt = np.zeros((64, 64, 1))
    for s, (_, (x0, y0), (x1, y1)) in zip(sc, tiles):
        acc[y0:y1, x0:x1] += s; cnt[y0:y1, x0:x1] += 1
    ref = np.floor(acc / cnt * 255)
    assert np.abs(kp.astype(int) - ref[..., 0]).max() <= 1 and np.abs(road.astype(int) - ref[..., 1]).max() <= 1
