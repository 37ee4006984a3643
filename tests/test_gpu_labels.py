"""GPU: training / evaluation batches on the device (sam_road_b200.dataset, csrc/labels.cu) against the numpy
oracle (oracle/label_oracle.py, ties="index") with injected and exported draws, invariants, distributions,
determinism, and the batches feeding SAMRoad's training / validation / test steps."""
import json
import os

import cv2
import numpy as np
import pytest
import torch

from oracle import label_oracle as LO
from oracle import samroad_oracle as SO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200 import dataset as D

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CITY_TRAIN, CITY_TEST = (0, 1, 2, 3), (8, 9, 19, 28)     # the first four tiles of each split (dev_run)
EXTENT = 1200          # graphs lie in [16, 1200]^2 of the 2048-pixel cityscale scenes: later windows are empty


def _cfg(P=256, S=64, Np=16, r_nms=16, **kw):
    return dict(DATASET="cityscale", PATCH_SIZE=P, TOPO_SAMPLE_NUM=S, MAX_NEIGHBOR_QUERIES=Np, NEIGHBOR_RADIUS=64,
                ROAD_NMS_RADIUS=r_nms, **kw)


@pytest.fixture(scope="module")
def city_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("cityscale_scenes"))
    synth.write_label_scenes(root, "cityscale", CITY_TRAIN + CITY_TEST, 2048, seed=5, extent=EXTENT)
    return root


@pytest.fixture(scope="module")
def spacenet_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("spacenet_scenes"))
    names = {"train": ["AOI_2_Vegas_1", "AOI_2_Vegas_2"], "validation": ["AOI_3_Paris_3"],
             "test": ["AOI_4_Shanghai_4", "AOI_5_Khartoum_5", "AOI_2_Vegas_6"]}
    synth.write_label_scenes(root, "spacenet", sum(names.values(), []), 400, seed=9, extent=380,
                             empty=("AOI_5_Khartoum_5",))
    with open(os.path.join(root, "spacenet", "data_split.json"), "w") as f:
        json.dump(names, f)
    return root


def _dataset(root, monkeypatch, cfg, is_train=True):
    monkeypatch.chdir(root)
    return D.SatMapDataset(cfg, is_train=is_train, dev_run=True, device=DEV)


def _images(root, ds, scene):
    tile = [t for t in ds.tile_indices[:4]][scene]
    lay = D.LAYOUTS[ds.dataset]
    p = lambda k: os.path.join(root, lay[k].format(tile))  # noqa: E731
    rgb = cv2.cvtColor(cv2.imread(p("rgb")), cv2.COLOR_BGR2RGB)
    return rgb, cv2.imread(p("keypoint"), cv2.IMREAD_GRAYSCALE), cv2.imread(p("road"), cv2.IMREAD_GRAYSCALE)


def _oracle(ds, patch, score_u, source_u, noise):
    scene, x0, y0, rot = (int(v) for v in patch)
    sc = ds.scenes[scene]
    m = LO.candidates(sc.points, sc.excluded, x0, y0, ds.lc["P"], "index").shape[0]
    draws = dict(score=0.9 + (1.0 - 0.9) * np.asarray(score_u[:m]), source_u=source_u, noise=noise)
    return LO.sample_patch(sc, x0, y0, rot, ds.lc, draws, ties="index")


def _check_batch(ds, batch, draws, root=None):
    """Device batch == oracle on the same draws: points bit for bit, pairs / valid / connected, crops."""
    d = {k: v.cpu().numpy() for k, v in draws.items()}
    b = {k: v.cpu().numpy() for k, v in batch.items()}
    B, N = b["graph_points"].shape[:2]
    outs = []
    for i in range(B):
        o = _oracle(ds, d["patches"][i], d["score_u"][i], d["source_u"][i], d["noise"][i])
        n = o["points"].shape[0]
        assert n <= N
        assert np.array_equal(b["graph_points"][i, :n].view(np.uint32), o["points"].view(np.uint32)), i
        assert not b["graph_points"][i, n:].any()
        for k in ("pairs", "valid", "connected"):
            assert np.array_equal(b[k][i], o[k]), (i, k)
        if root is not None:
            rgb, kp, road = _images(root, ds, int(d["patches"][i, 0]))
            _, x0, y0, rot = (int(v) for v in d["patches"][i])
            P = ds.lc["P"]
            assert np.array_equal(b["rgb"][i], LO.crop(rgb, x0, y0, P, rot).astype(np.float32))
            assert np.array_equal(b["keypoint_mask"][i], LO.crop(kp, x0, y0, P, rot).astype(np.float32) / np.float32(255))
            assert np.array_equal(b["road_mask"][i], LO.crop(road, x0, y0, P, rot).astype(np.float32) / np.float32(255))
        outs.append(o)
    assert N == max(o["points"].shape[0] for o in outs)
    return outs


@pytest.mark.parametrize("Np,r_nms", [(1, 16), (16, 16), (32, 4)])
def test_injected_draws_match_oracle(city_root, monkeypatch, Np, r_nms):
    ds = _dataset(city_root, monkeypatch, _cfg(Np=Np, r_nms=r_nms))
    rng = np.random.RandomState(Np)
    # rot 0..3, a window past the graph (empty), windows on the overpass crossings, each scene
    patches = np.array([[0, 100, 80, 0], [1, 300, 200, 1], [2, 520, 610, 2], [3, 64, 64, 3], [0, 1700, 1500, 2],
                        [1, 560, 560, 0], [2, 900, 880, 1], [3, 1100, 100, 3]], dtype=np.int32)
    B = patches.shape[0]
    draws = dict(patches=patches, score_u=rng.rand(B, ds._scenes.cap), source_u=rng.rand(B, ds.lc["S"]),
                 noise=rng.randn(B, ds._scenes.cap, 2))
    batch = ds._scenes.batch(B, draws=draws)
    outs = _check_batch(ds, batch, {k: torch.as_tensor(v) for k, v in draws.items()}, city_root)
    assert outs[4]["survivors"].shape[0] == 0 and batch["graph_points"].shape[1] > 1
    P = ds.lc["P"]
    assert any((((ds.scenes[sc].crossovers >= [x0, y0]) & (ds.scenes[sc].crossovers <= [x0 + P, y0 + P])).all(1)).any()
               for sc, x0, y0, _ in patches)
    if Np == 32:   # more than 32 survivors strictly inside NEIGHBOR_RADIUS of some source
        o = outs[1]
        pts = ds.scenes[1].points[o["survivors"]]
        d2 = ((pts[:, None] - pts[None]) ** 2).sum(-1)
        assert ((d2 < 64.0 ** 2).sum(1) > 33).any()
        assert batch["valid"][1].sum(1).max().item() == 32


def _ids_of(ds, patch, points, noise, cand):
    """Subdivided ids (among the candidates) of the device points of one patch (noise removed, rotation undone)."""
    scene, x0, y0, rot = (int(v) for v in patch)
    sc, P = ds.scenes[scene], ds.lc["P"]
    q = points.astype(np.float64) - noise[:points.shape[0]] - 0.5 * P
    for _ in range(rot):              # inverse of (x, y) -> (y, -x)
        q = np.stack([-q[:, 1], q[:, 0]], 1)
    q = q + 0.5 * P + np.array([x0, y0])
    d2 = ((sc.points[cand][None] - q[:, None]) ** 2).sum(-1)
    ids = d2.argmin(1)
    assert d2[np.arange(len(ids)), ids].max() < 1e-6
    return cand[ids]


def test_seeded_invariants_and_oracle(city_root, monkeypatch):
    ds = _dataset(city_root, monkeypatch, _cfg(P=512, S=128, Np=16))
    torch.manual_seed(3)
    batch, draws = ds._scenes.batch(8, export_draws=True)
    _check_batch(ds, batch, draws, city_root)
    d = {k: v.cpu().numpy() for k, v in draws.items()}
    b = {k: v.cpu().numpy() for k, v in batch.items()}
    r2, R2 = 16.0 ** 2, 64.0 ** 2
    for i in range(8):
        scene, x0, y0, rot = (int(v) for v in d["patches"][i])
        sc = ds.scenes[scene]
        cand = LO.candidates(sc.points, sc.excluded, x0, y0, 512, "index")
        if cand.shape[0] == 0:
            continue
        surv_all = LO.sample_patch(sc, x0, y0, rot, ds.lc, dict(score=0.9 + (1.0 - 0.9) * d["score_u"][i][:len(cand)],
                                                                source_u=d["source_u"][i], noise=d["noise"][i]))
        nsurv = surv_all["survivors"].shape[0]
        ids = _ids_of(ds, d["patches"][i], b["graph_points"][i, :nsurv], d["noise"][i], cand)
        assert np.array_equal(ids, surv_all["survivors"])
        score = np.maximum(0.9 + (1.0 - 0.9) * d["score_u"][i][:len(cand)], sc.nms_override[cand])
        prio = {int(c): (-s, k) for k, (c, s) in enumerate(zip(cand, score))}
        pos = sc.points
        kept = set(ids.tolist())
        for c in cand.tolist():       # every suppressed point has an earlier-visited survivor within the radius
            if c in kept:
                continue
            near = [s for s in ids if ((pos[s] - pos[c]) ** 2).sum() <= r2 and prio[int(s)] < prio[c]]
            assert near, c
        free = [s for s in ids if sc.nms_override[s] < 1.0]
        fp = pos[free]
        dd = ((fp[:, None] - fp[None]) ** 2).sum(-1) + np.eye(len(free)) * 1e9
        assert len(free) < 2 or dd.min() > r2       # no two non-immune survivors within the radius
        pr, va, co = b["pairs"][i], b["valid"][i], b["connected"][i]
        for s in range(pr.shape[0]):
            k = int(va[s].sum())
            assert va[s, :k].all() and not va[s, k:].any()
            assert (pr[s, :, 0] == pr[s, 0, 0]).all()
            assert (pr[s, k:, 1] == pr[s, 0, 0]).all() and not co[s, k:].any()   # (src, src) padding
            for t in pr[s, :k, 1]:
                assert ((pos[ids[t]] - pos[ids[pr[s, 0, 0]]]) ** 2).sum() < R2


def test_distributions(city_root, monkeypatch):
    ds = _dataset(city_root, monkeypatch, _cfg(P=256, S=512, Np=16))
    torch.manual_seed(11)
    rots, xs, noise, chi, dof = [], [], [], 0.0, 0
    for _ in range(8):
        batch, draws = ds._scenes.batch(16, export_draws=True)
        d = {k: v.cpu().numpy() for k, v in draws.items()}
        rots += d["patches"][:, 3].tolist()
        xs += d["patches"][:, 1].tolist() + d["patches"][:, 2].tolist()
        noise.append(d["noise"].reshape(-1))
        pr, va = batch["pairs"].cpu().numpy(), batch["valid"].cpu().numpy()
        for i in range(16):
            scene, x0, y0, rot = (int(v) for v in d["patches"][i])
            sc = ds.scenes[scene]
            cand = LO.candidates(sc.points, sc.excluded, x0, y0, 256, "index")
            if cand.shape[0] == 0:
                continue
            o = _oracle(ds, d["patches"][i], d["score_u"][i], d["source_u"][i], d["noise"][i])
            w = sc.weights[o["survivors"]].astype(np.float64)
            heavy = w > 0.5
            if heavy.all() or not heavy.any():
                continue
            p = w[heavy].sum() / w.sum()
            obs = heavy[pr[i, :, 0, 0]].sum()
            chi += (obs - 512 * p) ** 2 / (512 * p * (1 - p))
            dof += 1
    from scipy import stats
    assert dof >= 20 and stats.chi2.sf(chi, dof) > 1e-3, (chi, dof)
    z = np.concatenate(noise)
    assert abs(z.mean()) < 4 / np.sqrt(z.size) and abs(z.var() - 1) < 0.02
    assert stats.chisquare(np.bincount(rots, minlength=4)).pvalue > 1e-3
    lo, hi = ds.sample_min, ds.sample_max
    assert min(xs) >= lo and max(xs) <= hi
    assert stats.chisquare(np.histogram(xs, bins=8, range=(lo, hi + 1))[0]).pvalue > 1e-3


def test_seed_determinism(city_root, monkeypatch):
    ds = _dataset(city_root, monkeypatch, _cfg(P=256))
    torch.manual_seed(7)
    a = ds.batch(6)
    torch.manual_seed(7)
    b = ds.batch(6)
    c = ds.batch(6)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a["rgb"], c["rgb"]) or not torch.equal(a["graph_points"], c["graph_points"])


def test_spacenet_layout_eval_order_and_loader(spacenet_root, monkeypatch):
    cfg = dict(_cfg(P=256, S=32, Np=8), DATASET="spacenet")
    ds = _dataset(spacenet_root, monkeypatch, cfg, is_train=False)
    assert len(ds.scenes) == 2                     # the empty tile is skipped
    want = []
    for i in range(3):                             # dataset.py:387-390 indexes the tiles, skipped or not
        want += SO.get_patch_info_one_img(i, 400, 0, 256, 2)
    assert ds.eval_patches == want
    good = [k for k, p in enumerate(ds.eval_patches) if p[0] < len(ds.scenes)]
    loader = ds.loader(3)
    assert len(loader) == (len(ds) + 2) // 3
    first = next(iter(loader))
    assert first["rgb"].shape == (3, 256, 256, 3) and first["pairs"].shape == (3, 32, 8, 2)
    assert first["pairs"].dtype == torch.int32 and first["valid"].dtype == torch.bool
    rgb, _, _ = _images(spacenet_root, ds, 0)
    for k in range(3):
        _, (x0, y0), _ = ds.eval_patches[k]
        assert np.array_equal(first["rgb"][k].cpu().numpy(), rgb[y0:y0 + 256, x0:x0 + 256].astype(np.float32))
    assert len(good) == 8
    with pytest.raises(RuntimeError, match="missing scene"):   # tiles past the skipped one, as the reference
        ds.batch(4, first=len(ds) - 4)


@pytest.mark.parametrize("P", [256, 512])
def test_batches_feed_training_validation_and_test_steps(city_root, monkeypatch, P):
    cfg = dict(_cfg(P=P, S=64, Np=16), SAM_VERSION="vit_b", FREEZE_ENCODER=True, BASE_LR=1e-3,
               TOPONET_VERSION="normal", FOCAL_LOSS=False)
    train_ds = _dataset(city_root, monkeypatch, cfg, is_train=True)
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=0))
    net = net.to(DEV)
    opt = net.configure_optimizers()["optimizer"]
    torch.manual_seed(0)
    for step, batch in zip(range(2), train_ds.loader(2)):
        loss = net.training_step(batch, step)
        opt.zero_grad()
        loss.backward()
        assert torch.isfinite(loss)
        assert all(torch.isfinite(p.grad).all() for _, p in net._head_params() if p.grad is not None)
        opt.step()
    val_ds = _dataset(city_root, monkeypatch, cfg, is_train=False)
    net.eval()
    loader = val_ds.loader(4)
    for step, batch in zip(range(2), loader):
        res = net.validation_step(batch, step)
        assert torch.isfinite(res["val_mask_loss"])
        net.test_step(batch, step)
    m = net.on_validation_epoch_end()
    assert m is not None
    net.on_test_end()
