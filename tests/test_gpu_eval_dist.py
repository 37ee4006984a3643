"""GPU, two processes: the evaluation commands (`inferencer`, `topo_metric`, `apls_metric`) with one process per rank,
against the same commands in one process.

Inputs are synthetic: weights from `synth.make_state_dict`, the 27 CityScale test scenes at 512² (PATCH_SIZE 256,
3 x 3 tiles) and a SpaceNet split of 5 test scenes at 400², plus a SpaceNet split of one scene (fewer scenes than
ranks).  The ground-truth graphs of the metrics are the single-process predictions with every fourth edge removed, so
that every tile has starting points and control points to score.  Checked:
- every file under mask/, viz/ and graph/ is byte-identical to the single-process run, and inference_time.txt is the
  same text up to its seconds; the CityScale run has no --output_dir, so both ranks must use rank 0's timestamped
  directory;
- every per-tile TOPO and APLS file is byte-identical; the summaries hold the same per-tile values (as multisets: TOPO
  lists them in os.listdir order) and the same means;
- no child process survives.
gloo runs both ranks on one GPU and joins its group before the commands start; with NCCL (one GPU per rank) every
command initialises and destroys its own group from the launcher's environment, as under torchrun."""
import filecmp
import json
import os
import pickle
import re
import socket
from collections import Counter

import numpy as np
import pytest
import torch

from sam_road_b200 import synth

pytestmark = pytest.mark.gpu
WORLD = 2
CITY_IDS = [x for x in range(180) if x % 10 == 9 or x % 20 == 8]
SN_IDS = ["AOI_2_Vegas_11", "AOI_3_Paris_12", "AOI_4_Shanghai_13", "AOI_5_Khartoum_14", "AOI_2_Vegas_15"]
CFG = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False, ENCODER_LORA=False, TOPONET_VERSION="normal",
           NO_SAM=False, INFER_BATCH_SIZE=16, SAMPLE_MARGIN=0, ITSC_NMS_RADIUS=32, ROAD_NMS_RADIUS=48,
           NEIGHBOR_RADIUS=64, MAX_NEIGHBOR_QUERIES=16)
# wide NMS radii: the masks of random weights are noise-like, and a keypoint every 16 px would make a web far denser
# than a road network (the TOPO walks would exceed the device's marble capacity)
# (directory, dataset, scene size, tiles per edge, test ids)
SPLITS = {"city": ("cityscale", 512, 3, CITY_IDS), "sn": ("spacenet", 400, 2, SN_IDS),
          "sn1": ("spacenet", 400, 2, SN_IDS[:1])}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gt_from(pred: dict) -> dict:
    """The prediction with every fourth undirected edge (in sorted order) removed."""
    edges = sorted({tuple(sorted((a, b))) for a, vs in pred.items() for b in vs})
    drop = set(edges[::4])
    return {a: [b for b in vs if tuple(sorted((a, b))) not in drop] for a, vs in pred.items()}


def _run_commands(dataset, out_name, tag):
    """The three commands in the split's directory (the current one); returns the run directory's name."""
    from sam_road_b200 import apls_metric, inferencer, topo_metric
    before = set(os.listdir("save")) if os.path.isdir("save") else set()
    args = ["--checkpoint", "ckpt.pt", "--config", f"{dataset}.yaml"]
    inferencer.main(args + (["--output_dir", out_name] if out_name else []))
    if out_name is None:
        (out_name,) = [d for d in os.listdir("save") if d not in before and d.startswith("infer_")]
    save = os.path.join("save", out_name)
    for cmd in (topo_metric, apls_metric):
        tag()
        cmd.main(["--savedir", save, "--dataset", dataset, "--gt-root", dataset])
    return out_name


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """The three split directories, the checkpoint and configs, and the single-process runs in them."""
    import cv2
    import yaml
    from sam_road_b200 import SAMRoad, apls_metric, inferencer, topo_metric
    from sam_road_b200.inferencer import infer_one_img
    base = tmp_path_factory.mktemp("eval_dist")
    sd = synth.make_state_dict(CFG, seed=7, logit_gain=6.0)
    dev = torch.device("cuda", 0)
    net = SAMRoad(CFG)
    net.load_state_dict(sd, strict=True)
    net.eval().to(dev)
    roots = {}
    for name, (dataset, size, per_edge, ids) in SPLITS.items():
        root = base / name
        synth.write_label_scenes(str(root), dataset, ids, size, seed=len(name))
        if dataset == "spacenet":
            (root / "spacenet" / "data_split.json").write_text(json.dumps({"test": ids}))
        torch.save({"state_dict": sd}, root / "ckpt.pt")
        roots[name] = root
    # thresholds from the first CityScale scene: about one edge per two keypoints, so that every scene has edges
    cfg = dict(CFG, INFER_PATCHES_PER_EDGE=3, ITSC_THRESHOLD=2.0, ROAD_THRESHOLD=2.0, TOPO_THRESHOLD=0.5)
    img = cv2.cvtColor(cv2.imread(str(roots["city"] / "cityscale/20cities/region_8_sat.png")), cv2.COLOR_BGR2RGB)
    _, _, kp, road = infer_one_img(net, img, cfg, device=dev)
    cfg.update(ITSC_THRESHOLD=float(np.quantile(kp, 0.99)) / 255, ROAD_THRESHOLD=float(np.quantile(road, 0.93)) / 255)
    for t in (0.5, 0.4, 0.3, 0.2, 0.1):
        cfg["TOPO_THRESHOLD"] = t
        nodes, edges, _, _ = infer_one_img(net, img, cfg, device=dev)
        if 2 * edges.shape[0] >= nodes.shape[0]:
            break
    del net
    cwd = os.getcwd()
    try:
        for name, (dataset, size, per_edge, ids) in SPLITS.items():
            os.chdir(roots[name])
            with open(f"{dataset}.yaml", "w") as f:
                yaml.safe_dump(dict(cfg, DATASET=dataset, INFER_PATCHES_PER_EDGE=per_edge), f)
            inferencer.main(["--checkpoint", "ckpt.pt", "--config", f"{dataset}.yaml", "--output_dir", "single"])
            for i in ids:
                with open(f"save/single/graph/{i}.p", "rb") as f:
                    pred = pickle.load(f)
                assert sum(len(v) for v in pred.values()) >= 6, (name, i)     # enough to score
                with open(topo_metric.gt_path(dataset, dataset, i), "wb") as f:
                    pickle.dump(_gt_from(pred), f)
            for cmd in (topo_metric, apls_metric):
                cmd.main(["--savedir", "save/single", "--dataset", dataset, "--gt-root", dataset])
    finally:
        os.chdir(cwd)
    torch.cuda.empty_cache()
    return roots


def _worker(rank, world, backend, ports, roots):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(ports[0]), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank % torch.cuda.device_count()))
    if backend == "gloo":
        dist.init_process_group("gloo")
    port = iter(ports[1:])

    def tag():      # a fresh rendezvous port for each command that makes its own group
        os.environ["MASTER_PORT"] = str(next(port))
    try:
        for name, (dataset, _, _, _) in SPLITS.items():
            os.chdir(roots[name])
            tag()
            _run_commands(dataset, None if name == "city" else "dist", tag)
    finally:
        if backend == "gloo":
            dist.destroy_process_group()


def _same_tree(a, b, skip=()):
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)), (a, b)
    for n in names:
        if n not in skip:
            assert filecmp.cmp(os.path.join(a, n), os.path.join(b, n), shallow=False), os.path.join(b, n)
    return names


def _same_topo_summary(a, b):
    ja, jb = json.loads(open(a).read()), json.loads(open(b).read())
    for k in ("prec", "recall"):
        assert Counter(ja[k]) == Counter(jb[k]) and len(ja[k]) > 0, k
    if isinstance(ja["f1"], list):
        assert Counter(ja["f1"]) == Counter(jb["f1"])
    if ja["prec"] == jb["prec"]:
        assert ja["mean topo"] == jb["mean topo"]
    else:       # np.mean over another listing order may round differently in the last bit
        np.testing.assert_allclose(ja["mean topo"], jb["mean topo"], rtol=1e-15, atol=0)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_eval_commands_on_two_ranks_equal_one_process(backend, tree):
    if backend == "nccl" and torch.cuda.device_count() < WORLD:
        pytest.skip(f"NCCL needs {WORLD} GPUs")
    import torch.multiprocessing as mp
    import shutil
    ctx = mp.get_context("spawn")
    for root in tree.values():     # the other backend's run, if any
        for d in os.listdir(root / "save"):
            if d != "single":
                shutil.rmtree(root / "save" / d)
    ports = [_free_port() for _ in range(1 + 3 * len(SPLITS))]
    procs = [ctx.Process(target=_worker, args=(r, WORLD, backend, ports, {k: str(v) for k, v in tree.items()}))
             for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=900)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    assert not mp.active_children()

    for name, (dataset, _, _, ids) in SPLITS.items():
        save = tree[name] / "save"
        runs = sorted(os.listdir(save))
        assert len(runs) == 2 and "single" in runs, runs
        if name == "city":
            assert runs[0].startswith("infer_")        # the one directory rank 0 named
        one, two = save / "single", save / [r for r in runs if r != "single"][0]
        _same_tree(one, two, skip=("mask", "viz", "graph", "inference_time.txt", "results", "score", "topo.json"))
        for sub in ("mask", "viz", "graph"):
            names = _same_tree(one / sub, two / sub)
            assert len(names) == len(ids) * (2 if sub == "mask" else 1)
        secs = re.compile(r" in [0-9.e+-]+ seconds\.$")
        t1, t2 = (d.joinpath("inference_time.txt").read_text() for d in (one, two))
        assert secs.sub("", t1) == secs.sub("", t2) and secs.search(t2)
        assert len(_same_tree(one / "results" / "topo", two / "results" / "topo")) == 2 * len(ids)
        assert len(_same_tree(one / "results" / "apls", two / "results" / "apls")) == len(ids)
        if dataset == "cityscale":
            _same_topo_summary(one / "score" / "topo.json", two / "score" / "topo.json")
            assert (one / "score" / "apls.json").read_bytes() == (two / "score" / "apls.json").read_bytes()
        else:
            _same_topo_summary(one / "topo.json", two / "topo.json")
            assert (one / "results" / "apls.json").read_bytes() == (two / "results" / "apls.json").read_bytes()
