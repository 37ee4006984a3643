"""Generate tests/golden/*.npz from the UNMODIFIED reference (only runs where /root/reference exists).

The reference has no golden vectors for the hot path (SURVEY.md §4), so the reference itself is the
source of truth: this script imports its modules as they lie under /root/reference (tools/ref_loader
stubs lightning/torchmetrics/matplotlib), runs them on seeded synthetic weights/inputs and stores
small slices + checksums of the outputs.  It also checks the oracle restatement against the same
runs and refuses to write fixtures if they disagree.  `tests/test_oracle_golden.py` re-checks the
oracle against these files on any machine (no reference needed).

    python tools/make_golden.py
"""
from __future__ import annotations

import ast
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import samroad_oracle as O  # noqa: E402
from sam_road_b200 import synth  # noqa: E402
from tools import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
ORACLE_TOL = 2e-5


def _cfg(patch, version="vit_b", topo="normal", lora=0, samdec=False):
    return dict(SAM_VERSION=version, PATCH_SIZE=patch, USE_SAM_DECODER=samdec, ENCODER_LORA=lora > 0,
                LORA_RANK=lora, TOPONET_VERSION=topo, NO_SAM=False, FOCAL_LOSS=False)


def _stats(t: torch.Tensor):
    d = t.double()
    return np.array([d.sum().item(), d.abs().sum().item(), (d * d).sum().item()])


def model_fixture(name, cfg, seed, n_points):
    torch.manual_seed(0)
    net = ref_loader.load_reference_model(cfg)
    sd = synth.make_state_dict(cfg, seed=seed)
    net.load_state_dict(sd, strict=True)
    P = cfg["PATCH_SIZE"]
    rgb = synth.make_tiles(1, P, seed=seed + 21, dtype=torch.float32)
    pts, prs, val = synth.make_topo_inputs(1, P, n_points, seed=seed + 22)
    with torch.no_grad():
        ref = net(rgb, pts, prs, val)                              # reference SAMRoad.forward
        ref_scores, ref_feat = net.infer_masks_and_img_features(rgb)
        ref_ts = net.infer_toponet(ref_feat, pts, prs, val)
        spec = O.ModelSpec.from_config(cfg)
        ora = O.forward(sd, spec, rgb, pts, prs, val)
        _, ora_feat = O.infer_masks_and_img_features(sd, spec, rgb)
    errs = [(a - b).abs().max().item() for a, b in zip(ref, ora)]
    errs.append((ref_feat - ora_feat).abs().max().item())
    assert max(errs) < ORACLE_TOL, f"{name}: oracle disagrees with the reference: {errs}"
    assert torch.equal(ref[1], ref_scores) and torch.equal(ref[3], ref_ts)
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        seed=seed, n_points=n_points, patch=P,
        mask_logits_sub=ref[0][0, ::8, ::8, :].numpy(), mask_scores_sub=ref[1][0, ::8, ::8, :].numpy(),
        feat_sub=ref_feat[0, ::8, ::2, ::2].numpy(),
        topo_logits=ref[2].numpy(), topo_scores=ref[3].numpy(),
        mask_logits_stats=_stats(ref[0]), feat_stats=_stats(ref_feat), topo_logits_stats=_stats(ref[2]),
        oracle_vs_reference_maxabs=np.array(errs))
    print(f"{name}: oracle-vs-reference max-abs {max(errs):.2e}  "
          f"(mask logits in [{ref[0].min():.3f}, {ref[0].max():.3f}])")


def toponet_fixture():
    out = {}
    for topo in ("normal", "no_offset", "no_transformer", "no_tgt_features"):
        cfg = _cfg(256, topo=topo)
        torch.manual_seed(0)
        net = ref_loader.load_reference_model(cfg)
        sd = synth.make_state_dict(cfg, seed=5)
        net.load_state_dict(sd, strict=True)
        g = torch.Generator().manual_seed(77)
        feat = torch.randn(2, 256, 16, 16, generator=g)
        pts, prs, val = synth.make_topo_inputs(2, 256, 20, seed=9)
        val[1, 3] = False          # an all-invalid row (flipped to valid, model.py:128-130)
        pts[0, 0] = torch.tensor([256, 256])   # border point (inclusive box query)
        with torch.no_grad():
            ref = net.infer_toponet(feat, pts, prs, val)
            ref_f = net.infer_toponet(feat, pts.float() + 0.25, prs, val)
            spec = O.ModelSpec.from_config(cfg)
            ora = O.infer_toponet(sd, spec, feat, pts, prs, val)
            ora_f = O.infer_toponet(sd, spec, feat, pts.float() + 0.25, prs, val)
        err = max((ref - ora).abs().max().item(), (ref_f - ora_f).abs().max().item())
        assert err < ORACLE_TOL, f"toponet {topo}: oracle disagrees with the reference: {err}"
        out[f"{topo}_int"] = ref.numpy()
        out[f"{topo}_float"] = ref_f.numpy()
        print(f"toponet[{topo}]: oracle-vs-reference max-abs {err:.2e}")
    np.savez_compressed(os.path.join(OUT, "toponet_versions.npz"), **out)


TOPO_NPAIRS = (1, 5, 15)
TOPO_NPAIRS_WIDE = (17, 24, 32)
TOPO_NPAIRS_NS = 13          # samples kept: fewer than the 20 points, not a multiple of 8


def toponet_npairs_inputs(n_pairs):
    """Inputs of toponet_npairs.npz: 2 images x 20 points, n_pairs neighbour slots, pairs / valid sliced
    to the first TOPO_NPAIRS_NS samples (Ns != N), sample 3 of image 1 all-invalid."""
    g = torch.Generator().manual_seed(78)
    feat = torch.randn(2, 256, 16, 16, generator=g)
    pts, prs, val = synth.make_topo_inputs(2, 256, 20, seed=10 + n_pairs, max_nbr=n_pairs)
    prs, val = prs[:, :TOPO_NPAIRS_NS].contiguous(), val[:, :TOPO_NPAIRS_NS].contiguous()
    val[1, 3] = False
    return feat, pts, prs, val


def toponet_npairs_fixture(npairs=TOPO_NPAIRS, name="toponet_npairs"):
    out = {}
    cfg = _cfg(256)
    torch.manual_seed(0)
    net = ref_loader.load_reference_model(cfg)
    sd = synth.make_state_dict(cfg, seed=5)
    net.load_state_dict(sd, strict=True)
    spec = O.ModelSpec.from_config(cfg)
    for n_pairs in npairs:
        feat, pts, prs, val = toponet_npairs_inputs(n_pairs)
        with torch.no_grad():
            ref = net.infer_toponet(feat, pts, prs, val)
            ref_f = net.infer_toponet(feat, pts.float() + 0.25, prs, val)
            ora = O.infer_toponet(sd, spec, feat, pts, prs, val)
            ora_f = O.infer_toponet(sd, spec, feat, pts.float() + 0.25, prs, val)
        assert ref.shape == (2, TOPO_NPAIRS_NS, n_pairs, 1), ref.shape
        err = max((ref - ora).abs().max().item(), (ref_f - ora_f).abs().max().item())
        assert err < ORACLE_TOL, f"toponet n_pairs={n_pairs}: oracle disagrees with the reference: {err}"
        out[f"np{n_pairs}_int"] = ref.numpy()
        out[f"np{n_pairs}_float"] = ref_f.numpy()
        print(f"toponet[n_pairs={n_pairs}, Ns={TOPO_NPAIRS_NS}, N=20]: oracle-vs-reference max-abs {err:.2e}")
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **out)


def _extract_functions(path, names):
    """exec selected top-level function definitions of a reference file (it cannot be imported as a
    whole here: rtree / igraph / shapely / tcod are absent) -- the source is read where it lies."""
    src = open(path).read()
    tree = ast.parse(src)
    ns = {"np": np, "numpy": np}
    import scipy
    import scipy.spatial
    ns["scipy"] = scipy
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), path, "exec"), ns)
    return ns


def tileloop_fixture():
    ref = ref_loader.REF_ROOT
    ds = _extract_functions(os.path.join(ref, "dataset.py"), {"get_patch_info_one_img"})
    gu = _extract_functions(os.path.join(ref, "graph_utils.py"), {"nms_points"})
    ge = _extract_functions(os.path.join(ref, "graph_extraction.py"),
                            {"get_points_and_scores_from_mask", "extract_graph_points"})
    ge["nms_points"] = gu["nms_points"]
    out = {}
    for tag, args in {"c2_cityscale_16": (0, 2048, 64, 512, 16), "c4_cityscale_8": (0, 2048, 64, 512, 8),
                      "c3_spacenet_16": (0, 400, 0, 256, 16), "spacenet_4": (0, 400, 0, 256, 4)}.items():
        info = ds["get_patch_info_one_img"](*args)
        mine = O.get_patch_info_one_img(*args)
        assert info == mine, tag
        out[f"tiles_{tag}"] = np.array([[x0, y0, x1, y1] for _, (x0, y0), (x1, y1) in info])
    # keypoint extraction on a seeded synthetic pair of masks
    rng = np.random.RandomState(5)
    kp = np.zeros((400, 400), np.uint8)
    road = np.zeros((400, 400), np.uint8)
    for _ in range(60):
        y, x = rng.randint(5, 395, 2)
        kp[y - 2:y + 3, x - 2:x + 3] = rng.randint(60, 255)
    for _ in range(25):
        y = rng.randint(5, 395)
        road[y - 1:y + 2, rng.randint(0, 200):rng.randint(200, 400)] = rng.randint(90, 255)

    class Cfg:
        ITSC_THRESHOLD, ROAD_THRESHOLD, ITSC_NMS_RADIUS, ROAD_NMS_RADIUS = 0.3, 0.4, 8, 16
    pts_ref = ge["extract_graph_points"](kp, road, Cfg)
    pts_mine = O.extract_graph_points(kp, road, 0.3, 0.4, 8, 16)
    assert np.array_equal(pts_ref, pts_mine)
    out.update(kp_mask=kp, road_mask=road, graph_points=pts_ref)
    np.savez_compressed(os.path.join(OUT, "tileloop.npz"), **out)
    print(f"tileloop: {len(pts_ref)} graph points, tile grids identical")


def shape_fixtures():
    # PATCH_SIZE 400: odd 25x25 token grid, windows padded to 28, 3x3 neck conv through im2col
    model_fixture("vitb_400", _cfg(400), seed=8, n_points=24)
    # PATCH_SIZE 192: 12x12 grid smaller than the 14x14 window (one padded window), SAM mask decoder
    model_fixture("vitb_192_samdec", _cfg(192, samdec=True), seed=9, n_points=16)
    toponet_npairs_fixture()
    toponet_npairs_fixture(TOPO_NPAIRS_WIDE, "toponet_npairs_wide")


TRAIN_SAMPLES = 64     # gradient entries kept per parameter (seeded positions)


def train_heads_batch(P=256, B=2, n_points=24, Ns=20, Np=16, seed=31):
    """The batch of train_heads_vitb_256.npz, regenerated from seeds (float tiles, k/255 keypoint targets,
    binary road targets, one all-invalid sample row)."""
    g = torch.Generator().manual_seed(seed)
    pts, prs, val = synth.make_topo_inputs(B, P, n_points, seed=seed, max_nbr=Np)
    prs, val = prs[:, :Ns].contiguous(), val[:, :Ns].contiguous()
    val[0, 0] = False
    return {"rgb": synth.make_tiles(B, P, seed=seed, dtype=torch.float32), "graph_points": pts, "pairs": prs,
            "valid": val, "connected": torch.rand(val.shape, generator=g) < 0.4,
            "keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
            "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}


def train_heads_fixture():
    """Reference training_step + loss.backward() (ViT-B @256, B=2, FREEZE_ENCODER: True, eval mode so no
    dropout, grad enabled so torch's slow path), BCE and focal; the oracle must agree on the same embeddings."""
    import contextlib
    import io

    from oracle import train_oracle as TO
    out = {}
    for focal in (False, True):
        cfg = dict(_cfg(256), FREEZE_ENCODER=True, FOCAL_LOSS=focal, BASE_LR=1e-3)
        torch.manual_seed(0)
        net = ref_loader.load_reference_model(cfg)
        net.load_state_dict(synth.make_state_dict(cfg, seed=12, logit_gain=4.0), strict=True)
        b = train_heads_batch()
        tag = "focal" if focal else "bce"
        heads = [(k, p) for k, p in net.named_parameters() if k.startswith(("map_decoder.", "topo_net."))]
        net.zero_grad(set_to_none=True)
        losses = {}
        net.log = lambda name, v, **k: losses.__setitem__(name, v.detach().clone())
        loss = net.training_step(b, 0)
        loss.backward()
        with torch.no_grad():
            emb = net.infer_masks_and_img_features(b["rgb"])[1]
        params = {k: p.detach().clone().requires_grad_(True) for k, p in heads}
        oml, otl = TO.heads_losses(params, emb, b, 256, focal, "normal", None, 0.0)
        (oml + otl).backward()
        for name, o in (("train_mask_loss", oml), ("train_topo_loss", otl)):
            r = losses[name]
            assert abs(o.item() - r.item()) <= 1e-6 * abs(r.item()), (tag, name, o.item(), r.item())
        gen = torch.Generator().manual_seed(99)
        worst = 0.0
        for k, p in heads:
            g, og = p.grad, params[k].grad
            rel = ((g - og).abs().max() / g.abs().max()).item()
            worst = max(worst, rel)
            assert rel <= 2e-6, (tag, k, rel)   # fp32 against fp32, summation orders differ
            idx = torch.randint(0, g.numel(), (TRAIN_SAMPLES,), generator=gen)
            out[f"{tag}/{k}/idx"] = idx.numpy().astype(np.int32)
            out[f"{tag}/{k}/val"] = g.reshape(-1)[idx].numpy()
            out[f"{tag}/{k}/norm_maxabs"] = np.array([g.double().norm().item(), g.abs().max().item()])
        out[f"{tag}/losses"] = np.array([losses["train_mask_loss"].item(), losses["train_topo_loss"].item(),
                                         losses["train_loss"].item()], np.float32)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            net.configure_optimizers()
        out[f"{tag}/param_counts"] = np.array([int(line.rsplit(":", 1)[1]) for line in buf.getvalue().splitlines()
                                               if line.startswith("optim param dict")])
        out[f"{tag}/emb_stats"] = _stats(emb)
        print(f"train_heads[{tag}]: losses {out[f'{tag}/losses']}, oracle-vs-reference max relative gradient "
              f"error {worst:.2e}, param counts {out[f'{tag}/param_counts']}")
    np.savez_compressed(os.path.join(OUT, "train_heads_vitb_256.npz"), **out)


EMB_GRAD_SAMPLES = 512   # gradient entries kept per loss kind (seeded positions)


def emb_grad_fixture():
    """d(loss)/d(image embeddings) of the reference's training_step + loss.backward() (the batch, weights and
    configurations of train_heads_fixture), taken by a forward hook that makes the image encoder's output a leaf
    which requires grad; the oracle must give the same gradient on the same embeddings."""
    from oracle import train_oracle as TO
    out = {}
    for focal in (False, True):
        cfg = dict(_cfg(256), FREEZE_ENCODER=True, FOCAL_LOSS=focal, BASE_LR=1e-3)
        torch.manual_seed(0)
        net = ref_loader.load_reference_model(cfg)
        net.load_state_dict(synth.make_state_dict(cfg, seed=12, logit_gain=4.0), strict=True)
        b = train_heads_batch()
        tag = "focal" if focal else "bce"
        taken = []

        def leaf(module, inputs, output):
            e = output.detach().requires_grad_(True)
            taken.append(e)
            return e

        hook = net.image_encoder.register_forward_hook(leaf)
        logged = {}
        net.log = lambda name, v, **k: logged.__setitem__(name, v)
        loss = net.training_step(b, 0)
        hook.remove()
        assert len(taken) == 1, len(taken)
        # the mask loss alone (it is small next to the topology loss), then the step's own backward
        gm, = torch.autograd.grad(logged["train_mask_loss"], taken[0], retain_graph=True)
        loss.backward()
        emb, g = taken[0].detach(), taken[0].grad
        params = {k: p.detach().clone() for k, p in net.named_parameters()
                  if k.startswith(("map_decoder.", "topo_net."))}
        oemb = emb.clone().requires_grad_(True)
        oml, otl = TO.heads_losses(params, oemb, b, 256, focal, "normal", None, 0.0)
        ogm, = torch.autograd.grad(oml, oemb, retain_graph=True)
        (oml + otl).backward()
        rel = ((oemb.grad - g).abs().max() / g.abs().max()).item()
        rel_m = ((ogm - gm).abs().max() / gm.abs().max()).item()
        assert rel <= 2e-6 and rel_m <= 2e-6, (tag, rel, rel_m)   # fp32 against fp32, summation orders differ
        dm = gm.double()
        out[f"{tag}/mask_norm_maxabs"] = np.array([dm.norm().item(), dm.abs().max().item()])
        out[f"{tag}/mask_texel_sum"] = dm.sum(1).numpy()
        idx = torch.randint(0, g.numel(), (EMB_GRAD_SAMPLES,), generator=torch.Generator().manual_seed(98))
        d = g.double()
        out[f"{tag}/idx"] = idx.numpy().astype(np.int32)
        out[f"{tag}/val"] = g.reshape(-1)[idx].numpy()
        out[f"{tag}/norm_maxabs"] = np.array([d.norm().item(), d.abs().max().item()])
        out[f"{tag}/channel_sum"] = d.sum((2, 3)).numpy()          # [B, 256]
        out[f"{tag}/texel_sum"] = d.sum(1).numpy()                 # [B, s, s]
        out[f"{tag}/emb_stats"] = _stats(emb)
        print(f"emb_grad[{tag}]: |g|_2 {d.norm().item():.4e} (mask loss alone {dm.norm().item():.4e}), "
              f"oracle-vs-reference max relative error {rel:.2e} ({rel_m:.2e})")
    np.savez_compressed(os.path.join(OUT, "emb_grad_vitb_256.npz"), **out)


LABEL_CFG = dict(PATCH_SIZE=256, TOPO_SAMPLE_NUM=24, MAX_NEIGHBOR_QUERIES=16, NEIGHBOR_RADIUS=64,
                 ROAD_NMS_RADIUS=16)
LABEL_EXTENT = 360                 # the synthetic graph lies in [16, 360]^2: windows past it are empty
# (x0, y0, rot): rot 0..3, the empty window, and windows holding the overpass crossings
LABEL_PATCHES = ((40, 20, 0), (96, 64, 1), (10, 100, 2), (60, 30, 3), (384, 384, 1), (0, 0, 0), (100, 100, 2))


def label_scene():
    """The synthetic ground-truth graph of labels_synth.npz and its coordinate transform (cityscale's)."""
    from sam_road_b200 import dataset as D
    return synth.make_road_graph(LABEL_EXTENT, seed=0), D.cityscale_transform


class _IndexLog(np.ndarray):
    """An ndarray that records the row indices it is fancy-indexed with (`pts[idx, :]`)."""

    def __getitem__(self, key):
        if isinstance(key, tuple) and len(key) == 2 and isinstance(key[0], np.ndarray):
            self.log.append(np.array(key[0]))
        return np.asarray(self).__getitem__(key)


def _reference_samples(cfg_dict, patches, seed):
    """sample_patch of the unmodified reference GraphLabelGenerator (dataset.py:71-231) on the synthetic graph of
    label_scene() with the configuration cfg_dict, at patches [(x0, y0, rot)], after np.random.seed(seed).  The draws
    are recorded by wrapping np.random.uniform / choice / normal and graph_utils.nms_points from outside; the
    candidate and source ids by indexing a logging view of subdivide_points.  Every sample is checked against the
    oracle (ties="scipy") before it is returned.  Returns (generator, precompute, {"p<k>/<key>": array})."""
    from oracle import label_oracle as LO
    from sam_road_b200 import dataset as D
    ref = ref_loader.load_reference_dataset()
    gu = sys.modules["graph_utils"]
    adj, transform = label_scene()
    cfg = ref_loader.AttrDict(cfg_dict)
    gen = ref.GraphLabelGenerator(cfg, adj, transform)
    mine = D.precompute_scene(adj, transform)
    ref_cross = np.array(gen.crossover_points, dtype=np.float64).reshape(-1, 2)
    assert np.array_equal(gen.subdivide_points, mine.points), "subdivision differs"
    assert np.array_equal(np.unique(ref_cross, axis=0), np.unique(mine.crossovers, axis=0)), "crossovers differ"
    assert set(np.nonzero(mine.excluded)[0].tolist()) == set(gen.exclude_indices), "excluded set differs"
    assert np.array_equal(gen.nms_score_override, mine.nms_override) and np.array_equal(gen.sample_weights,
                                                                                          mine.weights)
    points = gen.subdivide_points
    log = points.view(_IndexLog)
    log.log = []
    gen.subdivide_points = log
    out = {}
    drawn = {}
    real = {k: getattr(np.random, k) for k in ("uniform", "choice", "normal")}
    real_nms = gu.nms_points

    def wrap(name):
        def f(*a, **k):
            r = real[name](*a, **k)
            drawn[name] = np.array(r)
            return r
        return f

    def nms_rec(*a, **k):
        r = real_nms(*a, **k)
        drawn["kept"] = np.array(r[1])
        return r

    P = cfg_dict["PATCH_SIZE"]
    lc = dict(P=P, S=cfg_dict["TOPO_SAMPLE_NUM"], Np=cfg_dict["MAX_NEIGHBOR_QUERIES"],
              r_nms=cfg_dict["ROAD_NMS_RADIUS"], r_nbr=cfg_dict["NEIGHBOR_RADIUS"])
    np.random.seed(seed)
    try:
        for name in real:
            setattr(np.random, name, wrap(name))
        gu.nms_points = nms_rec
        for k, (x0, y0, rot) in enumerate(patches):
            drawn.clear()
            log.log.clear()
            pts, samples = gen.sample_patch(((x0, y0), (x0 + P, y0 + P)), rot)
            pairs, conn, valid = (np.array(v) for v in zip(*samples))
            rec = dict(points=np.asarray(pts, dtype=np.float64), pairs=pairs.astype(np.int32),
                       connected=conn.astype(bool), valid=valid.astype(bool))
            if log.log:
                cand, src_ids = log.log[0], log.log[1]
                rec.update(candidates=cand.astype(np.int64), score=drawn["uniform"],
                           survivors=cand[drawn["kept"]].astype(np.int64),
                           source_index=drawn["choice"].astype(np.int64), noise=drawn["normal"])
                assert np.array_equal(rec["survivors"][rec["source_index"]], src_ids)
                o = LO.sample_patch(mine, x0, y0, rot, lc, dict(score=rec["score"], source_index=rec["source_index"],
                                                               noise=rec["noise"]), ties="scipy")
                assert np.array_equal(o["candidates"], rec["candidates"]), f"patch {k}: candidate order"
                assert np.array_equal(o["survivors"], rec["survivors"]), f"patch {k}: NMS"
                assert np.array_equal(o["points"], rec["points"].astype(np.float32)), f"patch {k}: points"
            else:
                o = LO.sample_patch(mine, x0, y0, rot, lc, {}, ties="scipy")
            for key in ("pairs", "connected", "valid"):
                assert np.array_equal(o[key], rec[key]), f"patch {k}: {key}"
            for key, v in rec.items():
                out[f"p{k}/{key}"] = v
            print(f"labels patch {k} (x0={x0}, y0={y0}, rot={rot}, P={P}): {len(rec.get('candidates', []))} "
                  f"candidates, {len(rec.get('survivors', []))} survivors, {int(rec['valid'].sum())} valid pairs, "
                  f"{int(rec['connected'].sum())} connected; oracle (ties='scipy') identical")
    finally:
        for name, fn in real.items():
            setattr(np.random, name, fn)
        gu.nms_points = real_nms
        gen.subdivide_points = points
    return gen, mine, out


def labels_fixture():
    """labels_synth.npz: the reference's precompute and samples on the synthetic graph at LABEL_CFG."""
    gen, _, samples = _reference_samples(LABEL_CFG, LABEL_PATCHES, 1234)
    ref_cross = np.array(gen.crossover_points, dtype=np.float64).reshape(-1, 2)
    out = dict(cfg=np.array([LABEL_CFG[k] for k in sorted(LABEL_CFG)]), cfg_keys=np.array(sorted(LABEL_CFG)),
               extent=LABEL_EXTENT, subdivide_points=gen.subdivide_points, crossovers=ref_cross,
               excluded=np.array(sorted(gen.exclude_indices), dtype=np.int32),
               nms_override=gen.nms_score_override, sample_weights=gen.sample_weights,
               patches=np.array(LABEL_PATCHES, dtype=np.int32))
    out.update(samples)
    path = os.path.join(OUT, "labels_synth.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes, {len(ref_cross)} crossover points "
          f"({len(np.unique(ref_cross, axis=0))} distinct), {len(gen.exclude_indices)} excluded")


# labels_edges.npz: the same synthetic graph at settings the benched configurations never use.  Each group is
# (configuration, patches (x0, y0, rot), np.random seed).
LABEL_EDGE_GROUPS = {
    # ROAD_NMS_RADIUS 10 (cell = radius, inexact division), NEIGHBOR_RADIUS 30 (depth 7, not a multiple of 4),
    # Np 4 and S 5 (not a multiple of the pair kernel's 4 warps)
    "r10_30": (dict(PATCH_SIZE=256, TOPO_SAMPLE_NUM=5, MAX_NEIGHBOR_QUERIES=4, NEIGHBOR_RADIUS=30,
                    ROAD_NMS_RADIUS=10), ((40, 20, 0), (96, 64, 1), (100, 100, 2), (60, 30, 3)), 4321),
    # NEIGHBOR_RADIUS 3: depth 3 // 4 = 0, nothing is expanded; the kNN radius is below the NMS radius
    "r3": (dict(PATCH_SIZE=256, TOPO_SAMPLE_NUM=3, MAX_NEIGHBOR_QUERIES=4, NEIGHBOR_RADIUS=3,
                ROAD_NMS_RADIUS=2), ((40, 20, 0), (96, 64, 3)), 4322),
    # PATCH_SIZE 1024 at toponet_vitb_1024's radii and pair count; one window over the whole graph
    "p1024": (dict(PATCH_SIZE=1024, TOPO_SAMPLE_NUM=64, MAX_NEIGHBOR_QUERIES=16, NEIGHBOR_RADIUS=64,
                   ROAD_NMS_RADIUS=16), ((0, 0, 1),), 4323),
}


def labels_edges_fixture():
    out = dict(extent=LABEL_EXTENT, groups=np.array(sorted(LABEL_EDGE_GROUPS)))
    for name in sorted(LABEL_EDGE_GROUPS):
        cfg, patches, seed = LABEL_EDGE_GROUPS[name]
        _, _, samples = _reference_samples(cfg, patches, seed)
        out[f"{name}/cfg"] = np.array([cfg[k] for k in sorted(cfg)], dtype=np.float64)
        out[f"{name}/cfg_keys"] = np.array(sorted(cfg))
        out[f"{name}/patches"] = np.array(patches, dtype=np.int32)
        out.update({f"{name}/{k}": v for k, v in samples.items()})
    path = os.path.join(OUT, "labels_edges.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes")


# ---- TOPO metric (cityscale_metrics/topo/*.py) ----------------------------------------------------------------------


def topo_synth_tiles():
    """Three synthetic (GT, proposal) adjacency dicts in the graph pickle format, in tile order.  Tile 0 stays within
    1000 px of the top edge (r = 0.0015); tile 1 reaches x = 1250, so from it on the carried min_lat switches the
    cityscale driver to r = 0.003; tile 2 is small again and still scored at r = 0.003."""
    rng = np.random.default_rng(7)

    def add(adj, a, b, two_way=True):
        adj.setdefault(a, [])
        adj.setdefault(b, [])
        if b not in adj[a]:
            adj[a].append(b)
        if two_way and a not in adj[b]:
            adj[b].append(a)

    def street(adj, p, q, seg, two_way=True):
        n = max(1, int(round(math.hypot(q[0] - p[0], q[1] - p[1]) / seg)))
        pts = [(float(p[0] + (q[0] - p[0]) * k / n), float(p[1] + (q[1] - p[1]) * k / n)) for k in range(n + 1)]
        for a, b in zip(pts, pts[1:]):
            add(adj, a, b, two_way)

    def grid(adj, x0, y0, nx, ny, sp, seg):
        for i in range(nx):
            street(adj, (x0 + i * sp, y0), (x0 + i * sp, y0 + (ny - 1) * sp), seg)
        for j in range(ny):
            street(adj, (x0, y0 + j * sp), (x0 + (nx - 1) * sp, y0 + j * sp), seg)

    def proposal(gt, drop, shift, extra, oneway):
        prop = {}
        keys = list(gt)
        moved = {k: (k[0] + float(rng.integers(-shift, shift + 1)), k[1] + float(rng.integers(-shift, shift + 1)))
                 for k in keys}
        edges = [(a, b) for a in keys for b in gt[a]]
        for (a, b) in edges:
            if rng.random() < drop:
                continue
            add(prop, moved[a], moved[b], two_way=False)
        for (a, b) in extra:
            add(prop, a, b, two_way=rng.random() >= oneway)
        return prop

    tiles = []
    # tile 0: a 4 x 4 grid of 90 px blocks, nodes every 30 px, an overpass (a diagonal with no shared node), two dead
    # ends and a one-way street
    gt = {}
    grid(gt, 100.0, 100.0, 4, 4, 90.0, 30.0)
    street(gt, (80.0, 95.0), (395.0, 410.0), 25.0)               # overpass: crosses the grid without a node
    street(gt, (370.0, 190.0), (450.0, 190.0), 20.0)             # dead end
    street(gt, (190.0, 370.0), (190.0, 440.0), 35.0)             # dead end
    street(gt, (145.0, 100.0), (145.0, 370.0), 45.0, two_way=False)   # one-way
    prop = proposal(gt, 0.15, 7, [((300.0, 300.0), (330.0, 360.0)), ((120.0, 400.0), (160.0, 430.0)),
                              ((250.0, 120.0), (250.0, 260.0)), ((160.0, 200.0), (240.0, 215.0))], 0.5)
    tiles.append((gt, prop))
    # tile 1: a long arterial to x = 1250 and a small grid
    gt = {}
    street(gt, (100.0, 150.0), (1250.0, 150.0), 50.0)
    grid(gt, 200.0, 200.0, 3, 3, 100.0, 25.0)
    street(gt, (200.0, 150.0), (200.0, 200.0), 25.0)
    prop = proposal(gt, 0.1, 9, [((400.0, 400.0), (460.0, 400.0)), ((260.0, 230.0), (330.0, 260.0))], 0.0)
    tiles.append((gt, prop))
    # tile 2: a 3 x 3 grid, the proposal equal to the GT
    gt = {}
    grid(gt, 120.0, 120.0, 3, 3, 80.0, 40.0)
    prop = proposal(gt, 0.0, 0, [], 0.0)
    tiles.append((gt, prop))
    # tile 3: two parallel streets 12 px apart joined at both ends, with two spurs; the proposal draws one street between them with
    # spurious side branches, so nearby starting points compete for the same proposal edges with precisions below
    # 0.9 and TOPO121 drops some of them
    gt = {}
    street(gt, (200.0, 100.0), (200.0, 420.0), 20.0)
    street(gt, (212.0, 100.0), (212.0, 420.0), 20.0)
    street(gt, (200.0, 100.0), (212.0, 100.0), 12.0)
    street(gt, (200.0, 420.0), (212.0, 420.0), 12.0)
    street(gt, (212.0, 260.0), (270.0, 260.0), 29.0)             # dead-end spurs: degree-3 nodes start the chains
    street(gt, (200.0, 200.0), (160.0, 200.0), 20.0)
    prop = {}
    street(prop, (206.0, 100.0), (206.0, 420.0), 20.0)
    for y in (160.0, 260.0, 360.0):
        street(prop, (206.0, y), (150.0, y + 30.0), 20.0)
        street(prop, (206.0, y + 20.0), (280.0, y + 50.0), 20.0)
    tiles.append((gt, prop))
    # tile 4 (spacenet only): a GT with no starting point (one 3 px edge), where spacenet's topo.py writes its
    # zeros line; cityscale's divides by the start count first and raises
    tiles.append(({(300.0, 300.0): [(300.0, 303.0)]}, {(300.0, 300.0): [(300.0, 340.0)]}))
    return tiles


def adj_to_arrays(adj):
    keys = np.array([k for k in adj], dtype=np.float64).reshape(-1, 2)
    cnt = np.array([len(v) for v in adj.values()], dtype=np.int32)
    nb = np.array([n for v in adj.values() for n in v], dtype=np.float64).reshape(-1, 2)
    return keys, cnt, nb


def _load_reference_topo():
    import types
    ref_loader._install_graph_shims()
    if "svgwrite" not in sys.modules and not ref_loader._has("svgwrite"):
        # showTOPO's import: spacenet's topo.py renders coverage SVGs; here every drawing call does nothing
        svg = types.ModuleType("svgwrite")

        class Drawing:
            def __init__(self, *a, **k):
                pass

            def __getattr__(self, name):
                return lambda *a, **k: None

        svg.Drawing = Drawing
        sys.modules["svgwrite"] = svg
    if "hopcroftkarp" not in sys.modules and not ref_loader._has("hopcroftkarp"):
        import networkx as nx
        hk = types.ModuleType("hopcroftkarp")

        class HopcroftKarp:
            """hopcroftkarp.HopcroftKarp(graph).maximum_matching(): a maximum matching as a dict holding both
            directions (left -> right and right -> left), as the library documents."""

            def __init__(self, graph):
                self.graph = graph

            def maximum_matching(self):
                g = nx.Graph()
                left = [("L", k) for k in self.graph]
                g.add_nodes_from(left, bipartite=0)
                for k, vs in self.graph.items():
                    for v in vs:
                        g.add_edge(("L", k), ("R", v))
                m = nx.bipartite.hopcroft_karp_matching(g, top_nodes=left)
                out = {a[1]: b[1] for a, b in m.items()}
                HopcroftKarp.sizes.append(len(out) // 2)
                return out

        HopcroftKarp.sizes = []
        hk.HopcroftKarp = HopcroftKarp
        sys.modules["hopcroftkarp"] = hk
    tdir = os.path.join(ref_loader.REF_ROOT, "cityscale_metrics", "topo")
    if tdir not in sys.path:
        sys.path.insert(0, tdir)
    import graph as ref_graph  # noqa: the reference's cityscale_metrics/topo/graph.py
    import topo as ref_topo    # noqa: the reference's cityscale_metrics/topo/topo.py
    # spacenet_metrics/topo/topo.py under its own name; its graph.py and showTOPO.py are the same files as
    # cityscale's, so its `import graph` / `import showTOPO` resolve to the modules above
    if "spacenet_topo" not in sys.modules:
        import importlib.util
        spec = importlib.util.spec_from_file_location(
            "spacenet_topo", os.path.join(ref_loader.REF_ROOT, "spacenet_metrics", "topo", "topo.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules["spacenet_topo"] = mod
        spec.loader.exec_module(mod)
    topos = {"cityscale": ref_topo, "spacenet": sys.modules["spacenet_topo"]}
    return ref_graph, topos, sys.modules["hopcroftkarp"].HopcroftKarp


def _reference_topo_run(tiles, dataset, workdir):
    """main.py's loop (cityscale or spacenet) over `tiles`, restated around the reference's own graph.RoadGraph and
    topo.py functions; returns per-tile records."""
    import contextlib
    import io
    import pickle
    splfy, topos, HK = _load_reference_topo()
    topo = topos[dataset]
    lat_top_left, lon_top_left = 41.0, -71.0
    g = dict(min_lat=41.0, max_lon=-71.0)
    walk_lens = []
    orig_walk = splfy.RoadGraph.TOPOWalk

    def walk(self, *a, **k):
        out = orig_walk(self, *a, **k)
        walk_lens.append(len(out))
        return out

    seen_results = []
    orig_121 = topo.TOPO121

    def t121(res, rg):
        seen_results.append(list(res))
        return orig_121(res, rg)

    splfy.RoadGraph.TOPOWalk = walk
    topo.TOPO121 = t121
    records = []
    try:
        for t, (map1, map2) in enumerate(tiles):
            def xy2latlon(x, y):
                lat = lat_top_left - x * 1.0 / 111111.0
                lon = lon_top_left + (y * 1.0 / 111111.0) / math.cos(math.radians(lat_top_left))
                return lat, lon

            def create_graph(m):
                graph = splfy.RoadGraph()
                nid = 0
                idmap = {}
                for k, v in m.items():
                    n1 = k
                    lat1, lon1 = xy2latlon(n1[0], n1[1])
                    if lat1 < g["min_lat"]:
                        g["min_lat"] = lat1
                    if lon1 > g["max_lon"]:
                        g["max_lon"] = lon1
                    for n2 in v:
                        lat2, lon2 = xy2latlon(n2[0], n2[1])
                        if n1 in idmap:
                            id1 = idmap[n1]
                        else:
                            id1 = nid
                            idmap[n1] = nid
                            nid = nid + 1
                        if n2 in idmap:
                            id2 = idmap[n2]
                        else:
                            id2 = nid
                            idmap[n2] = nid
                            nid = nid + 1
                        graph.addEdge(id1, lat1, lon1, id2, lat2, lon2)
                graph.ReverseDirectionLink()
                for node in graph.nodes.keys():
                    graph.nodeScore[node] = 100
                for edge in graph.edges.keys():
                    graph.edgeScore[edge] = 100
                return graph

            output = os.path.join(workdir, "results", "topo", "%d.txt" % t)
            os.makedirs(os.path.dirname(output), exist_ok=True)
            with contextlib.redirect_stdout(io.StringIO()):
                graph_gt = create_graph(map1)
                graph_prop = create_graph(map2)
                region = [g["min_lat"] - 300 * 1.0 / 111111.0, lon_top_left - 500 * 1.0 / 111111.0,
                          lat_top_left + 300 * 1.0 / 111111.0, g["max_lon"] + 500 * 1.0 / 111111.0]
                graph_gt.region = region
                graph_prop.region = region
                losm = topo.TOPOGenerateStartingPoints(graph_gt, region=region, image="NULL", check=False,
                                                       direction=False, metaData=None)
                lmap = topo.TOPOGeneratePairs(graph_prop, graph_gt, losm, threshold=0.00010, region=region)
                if dataset == "cityscale":
                    r = 0.00300
                    if lat_top_left - g["min_lat"] < 0.01000:
                        r = 0.00150
                else:
                    r = 0.00150
                del walk_lens[:], seen_results[:], HK.sizes[:]
                kept = topo.TOPOWithPairs(graph_prop, graph_gt, lmap, losm, r=r, step=0.00005, threshold=0.00010,
                                          outputfile=output, one2oneMatching=True, metaData=None)
            pickle.dump([losm, kept, region], open(output.replace('txt', 'topo.p'), 'wb'))
            # per pair: 3 walks and the precision matching, then the recall matching unless the pair was skipped
            counts, sizes, w = [], list(HK.sizes), list(walk_lens)
            for _ in lmap:
                nm, nh, nhb = w[:3]
                del w[:3]
                mp = sizes.pop(0)
                mr = sizes.pop(0) if nm and nh else -1
                counts.append([nm, nh, nhb, mp, mr])
            with open(output) as f:
                text = f.read()
            records.append(dict(r=r, region=region, losm=losm, lmap=lmap, kept=kept, results=seen_results[0],
                                counts=counts, text=text))
    finally:
        splfy.RoadGraph.TOPOWalk = orig_walk
        topo.TOPO121 = orig_121
    return records


def _reference_aggregate(workdir, dataset, order):
    """The dataset's topo.py, run as it lies with os.listdir pinned to `order` (its own order is the file system's)."""
    import contextlib
    import io
    import runpy
    script = os.path.join(ref_loader.REF_ROOT, f"{dataset}_metrics", "topo.py")
    run_dir = os.path.join(workdir, "cwd")
    os.makedirs(run_dir, exist_ok=True)
    saved = (sys.argv, os.getcwd(), os.listdir)
    rel = os.path.relpath(workdir, os.path.dirname(run_dir))
    sys.argv = [script, "-savedir", rel]
    os.chdir(run_dir)
    os.listdir = lambda p: list(order)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            runpy.run_path(script, run_name="__main__")
    finally:
        sys.argv, _, os.listdir = saved
        os.chdir(saved[1])
    path = os.path.join(workdir, "score", "topo.json") if dataset == "cityscale" else os.path.join(workdir, "topo.json")
    with open(path) as f:
        return f.read()


def topo_fixture():
    import tempfile
    from oracle import topo_oracle
    from sam_road_b200 import topo_metric as TM
    tiles = topo_synth_tiles()
    out = {}
    for t, (gt, prop) in enumerate(tiles):
        for name, adj in (("gt", gt), ("prop", prop)):
            k, c, n = adj_to_arrays(adj)
            out[f"tile{t}/{name}_keys"], out[f"tile{t}/{name}_cnt"], out[f"tile{t}/{name}_nbrs"] = k, c, n
    for dataset in ("cityscale", "spacenet"):
        with tempfile.TemporaryDirectory() as wd:
            dtiles = tiles if dataset == "spacenet" else tiles[:4]
            recs = _reference_topo_run(dtiles, dataset, wd)
            order = ["%d.txt" % t for t in range(len(dtiles))] + ["%d.topo.p" % t for t in range(len(dtiles))]
            js = _reference_aggregate(wd, dataset, order)
        state = TM.TopoState()
        for t, rec in enumerate(recs):
            p, rr, d = TM.topo_tile(tiles[t][0], tiles[t][1], state, dataset, scorer=topo_oracle.scorer)
            mine = [tuple(x) for x in d.results]
            assert d.r == rec["r"] and d.region == rec["region"], (dataset, t)
            assert d.starts == rec["losm"] and d.pairs == rec["lmap"], (dataset, t)
            ref_counts = np.array(rec["counts"], dtype=np.int64).reshape(-1, 5)
            mc = np.asarray(d.counts, dtype=np.int64).reshape(-1, 6)[:, :5]
            defined = ref_counts[:, 4] >= 0
            assert np.array_equal(ref_counts[:, :4], mc[:, :4]) and np.array_equal(ref_counts[defined, 4],
                                                                                   mc[defined, 4]), (dataset, t)
            assert mine == [tuple(x) for x in rec["results"]], (dataset, t)
            assert [tuple(x) for x in d.kept] == [tuple(x) for x in rec["kept"]], (dataset, t)
            assert "".join(d.lines) == rec["text"], (dataset, t)
            if t == 3:   # the TOPO121 tile: the reference drops some scored starting points
                assert len(rec["kept"]) < len(rec["results"]), (dataset, len(rec["kept"]), len(rec["results"]))
            if t == 4:   # spacenet's no-starting-point tile: the zeros line
                assert rec["text"] == "0 0 0 0\n", rec["text"]
            pre = f"{dataset}/tile{t}/"
            out[pre + "r"] = np.float64(rec["r"])
            out[pre + "region"] = np.array(rec["region"], dtype=np.float64)
            out[pre + "starts"] = np.array(rec["losm"], dtype=np.float64).reshape(-1, 6)
            out[pre + "pair_keys"] = np.array(list(rec["lmap"]), dtype=np.int64)
            out[pre + "pairs"] = np.array(list(rec["lmap"].values()), dtype=np.float64).reshape(-1, 7)
            out[pre + "counts"] = ref_counts
            out[pre + "results"] = np.array(rec["results"], dtype=np.float64).reshape(-1, 8)
            out[pre + "kept"] = np.array(rec["kept"], dtype=np.float64).reshape(-1, 8)
            out[pre + "text"] = np.array(rec["text"])
            print(f"{dataset} tile {t}: r={rec['r']} starts={len(rec['losm'])} pairs={len(rec['lmap'])} "
                  f"scored={len(rec['results'])} kept={len(rec['kept'])} last={rec['text'].splitlines()[-1]!r}")
        out[f"{dataset}/topo_json"] = np.array(js)
    path = os.path.join(OUT, "topo_synth.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes")


def _label_mask_special(size, spacenet):
    """Adjacency entries that exercise the graph rules: a self-loop on a node with one other edge (degree 3), a
    lone self-loop (degree 2), repeated and one-way entries, float nodes that truncate to one node, end points
    outside the tile (negative, at the size and far beyond), and a key without neighbours."""
    s = float(size)
    adj = {
        (10.0, 10.0): [(10.0, 10.0), (30.5, 40.25), (30.5, 40.25)],
        (30.5, 40.25): [(10.0, 10.0)],
        (60.0, 60.0): [(60.0, 60.0)],
        (80.2, 20.7): [(95.0, 21.0)],                          # one-way
        (80.9, 20.1): [(70.0, 45.0)],                          # merges with (80.2, 20.7)
        (120.0, 5.0): [(-40.0, 2.0), (s - 1.0, s + 30.0)],
        (s - 2.0, 3.0): [(s + 5000.0, -7000.0)],
        (s * 0.5, s * 0.5): [],
        (s * 0.5 + 3.0, -2.0): [(s * 0.5 + 3.0, -2.0), (s * 0.5 + 20.0, 17.0)],
    }
    if spacenet:   # rows that map to y = 400 - int(row) = 400 and beyond
        adj[(0.0, 200.0)] = [(0.4, 230.0), (-3.0, 260.0)]
    return adj


def label_masks_fixture():
    """The reference scripts' own drawing functions on synthetic graphs: CityScale 2048^2 tiles from
    synth.city_tile (float nodes, diagonals), SpaceNet 400^2 tiles from synth.make_road_graph, the graph-rule
    cases of _label_mask_special and an empty dict.  Stored per tile: the adjacency entries, the key of every
    entry without neighbours and both masks as np.packbits."""
    import cv2
    import networkx as nx
    from oracle import label_mask_oracle as LM
    out = {"cv2_version": np.array(cv2.__version__), "networkx_version": np.array(nx.__version__)}
    tiles = [("city0", "cityscale", synth.city_tile(2048, seed=0)[0]),
             ("city1", "cityscale", synth.city_tile(2048, seed=1)[1]),
             ("city_special", "cityscale", _label_mask_special(2048, False)),
             ("city_empty", "cityscale", {}),
             ("space0", "spacenet", synth.make_road_graph(384, seed=0)),
             ("space1", "spacenet", synth.make_road_graph(400, seed=1, spacing=40, lo=0)),
             ("space_special", "spacenet", _label_mask_special(400, True))]
    for name, dataset, adj in tiles:
        script = os.path.join(ref_loader.REF_ROOT, dataset, "generate_labels.py")
        fns = _extract_functions(script, {"draw_points_on_image", "draw_line_segments_on_image"})
        fns["cv2"] = cv2
        size = 2048 if dataset == "cityscale" else 400
        graph = nx.Graph()
        for n, neis in adj.items():
            for nei in neis:
                if dataset == "cityscale":
                    graph.add_edge((int(n[1]), int(n[0])), (int(nei[1]), int(nei[0])))
                else:
                    graph.add_edge((int(n[1]), size - int(n[0])), (int(nei[1]), size - int(nei[0])))
        key_nodes = [node for node, degree in graph.degree() if degree != 2]
        kp = fns["draw_points_on_image"](size=size, points=key_nodes, radius=3)
        road = fns["draw_line_segments_on_image"](size=size, line_segments=graph.edges(), width=3)
        okp, oroad = LM.tile_masks(adj, dataset, size)
        assert np.array_equal(kp, okp) and np.array_equal(road, oroad), f"{name}: oracle disagrees with cv2"
        pairs = [(*n, *m) for n, neis in adj.items() for m in neis]
        out[f"{name}/dataset"] = np.array(dataset)
        out[f"{name}/pairs"] = np.array(pairs, np.float64).reshape(-1, 4)
        out[f"{name}/lonely"] = np.array([n for n, neis in adj.items() if not neis], np.float64).reshape(-1, 2)
        out[f"{name}/keypoint"] = np.packbits(kp > 0)
        out[f"{name}/road"] = np.packbits(road > 0)
        print(f"label masks {name}: {len(key_nodes)} keypoints, {graph.number_of_edges()} edges, "
              f"{int((kp > 0).sum())} / {int((road > 0).sum())} pixels set")
    path = os.path.join(OUT, "label_masks.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path)} bytes")


def main():
    assert ref_loader.available(), "needs /root/reference"
    if "--label-masks" in sys.argv:   # generate_labels.py's masks of CityScale and SpaceNet graphs
        os.makedirs(OUT, exist_ok=True)
        label_masks_fixture()
        return
    if "--topo" in sys.argv:          # the TOPO metric on three synthetic tiles, both drivers and aggregators
        os.makedirs(OUT, exist_ok=True)
        topo_fixture()
        return
    if "--labels-edges" in sys.argv:  # the same at non-default radii, odd pair counts and PATCH_SIZE 1024
        os.makedirs(OUT, exist_ok=True)
        labels_edges_fixture()
        return
    if "--labels" in sys.argv:        # GraphLabelGenerator / sample_patch on a synthetic graph
        os.makedirs(OUT, exist_ok=True)
        labels_fixture()
        return
    if "--emb-grad" in sys.argv:      # the same step's gradient of the image embeddings
        os.makedirs(OUT, exist_ok=True)
        emb_grad_fixture()
        return
    if "--train-heads" in sys.argv:   # training_step / backward of the heads with a frozen encoder
        os.makedirs(OUT, exist_ok=True)
        train_heads_fixture()
        return
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    if "--only-new" in sys.argv:      # fixtures added in round 2 (the round-1 files stay byte-identical)
        model_fixture("vitl_256", _cfg(256, version="vit_l"), seed=6, n_points=16)
        model_fixture("vitb_1024", _cfg(1024), seed=7, n_points=40)
        return
    if "--shapes" in sys.argv:        # tile sizes and pair counts outside the benched configs
        shape_fixtures()
        return
    if "--wide-pairs" in sys.argv:    # MAX_NEIGHBOR_QUERIES 17..32
        toponet_npairs_fixture(TOPO_NPAIRS_WIDE, "toponet_npairs_wide")
        return
    model_fixture("vitb_256", _cfg(256), seed=0, n_points=24)
    model_fixture("vitb_512", _cfg(512), seed=1, n_points=40)
    model_fixture("vitb_256_lora4", _cfg(256, lora=4), seed=2, n_points=16)
    model_fixture("vitb_256_samdec", _cfg(256, samdec=True), seed=3, n_points=16)
    model_fixture("vith_256", _cfg(256, version="vit_h"), seed=4, n_points=16)
    model_fixture("vitl_256", _cfg(256, version="vit_l"), seed=6, n_points=16)
    model_fixture("vitb_1024", _cfg(1024), seed=7, n_points=40)
    toponet_fixture()
    tileloop_fixture()
    shape_fixtures()


if __name__ == "__main__":
    main()
