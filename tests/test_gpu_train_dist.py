"""GPU, several processes: training and evaluation on every rank of torch.distributed.

Each rank first works alone (no process group yet) to record what a single process computes, then joins the
group and checks:
- under a common torch.manual_seed, rank 0's training batch is the single-process batch bit for bit and rank 1's
  differs; the dropout seeds (and so the keep masks) differ across ranks;
- SAMRoad wrapped in DistributedDataParallel the way Lightning's DDP strategy wraps it (a module whose forward
  calls training_step, after setup("fit")): the wrap-time broadcast from rank 0 reaches the packed head weights,
  one step's .grad is DDP's mean of the ranks' gradients, and GradScaler + Adam + zero_grad(set_to_none=True)
  keep the replicas bitwise identical;
- a sharded validation epoch gives on every rank the metrics of a single-process run over DistributedSampler's
  padded index list.
gloo runs both ranks on one GPU; NCCL needs one GPU per rank."""
import os
import socket

import numpy as np
import pytest
import torch

from sam_road_b200 import synth

pytestmark = pytest.mark.gpu
WORLD = 2
SEED = 3
CITY_TRAIN = (0, 1, 2, 3)
SPACENET = {"train": ["AOI_2_Vegas_1"], "validation": ["AOI_3_Paris_3"],
            "test": ["AOI_4_Shanghai_4", "AOI_5_Khartoum_5", "AOI_2_Vegas_6"]}
TRAIN_CFG = dict(DATASET="cityscale", SAM_VERSION="vit_b", PATCH_SIZE=256, TOPO_SAMPLE_NUM=64,
                 MAX_NEIGHBOR_QUERIES=16, NEIGHBOR_RADIUS=64, ROAD_NMS_RADIUS=16, FREEZE_ENCODER=True,
                 BASE_LR=1e-3, TOPONET_VERSION="normal", FOCAL_LOSS=False)
# 3 test tiles x 3 x 3 patches of 192: 27 patches, so the two shards are padded by one
VAL_CFG = dict(TRAIN_CFG, DATASET="spacenet", PATCH_SIZE=192, TOPO_SAMPLE_NUM=32, MAX_NEIGHBOR_QUERIES=8)
VAL_B = 4
METRICS = ("keypoint_iou", "road_iou", "topo_f1")


class _StepModule(torch.nn.Module):
    """What Lightning hands to DistributedDataParallel: a module whose forward is the LightningModule's
    training_step."""

    def __init__(self, net):
        super().__init__()
        self.module = net

    def forward(self, batch, batch_idx):
        return self.module.training_step(batch, batch_idx)


def _fixed_batch(seed, dev, B=2, P=256, N=40, Ns=20, Np=16):
    g = torch.Generator().manual_seed(seed)
    pts, pairs, valid = synth.make_topo_inputs(B, P, N, seed=seed, max_nbr=Np)
    pairs, valid = pairs[:, :Ns], valid[:, :Ns].clone()
    b = {"rgb": synth.make_tiles(B, P, seed=seed), "graph_points": pts, "pairs": pairs, "valid": valid,
         "connected": torch.rand(valid.shape, generator=g) < 0.4,
         "keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
         "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}
    return {k: v.to(dev) for k, v in b.items()}


def _infer(net, b):
    scores, emb = net.infer_masks_and_img_features(b["rgb"])
    topo = net.infer_toponet(emb, b["graph_points"], b["pairs"], b["valid"])
    return [t.clone() for t in (scores, emb, topo)]


def _equal(xs, ys):
    return all(torch.equal(x, y) for x, y in zip(xs, ys))


def _worker(rank, world, port, backend, city_root, spacenet_root, out_dir):
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel
    from sam_road_b200 import SAMRoad
    from sam_road_b200 import dataset as D
    from sam_road_b200 import train as T
    from sam_road_b200.ranks import rank_seed
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    res = {}
    seeds = []
    make_args = T.make_args

    def spy(b, focal, dropout_p, seed):            # the dropout seed training_step hands to the device
        seeds.append(seed)
        return make_args(b, focal, dropout_p, seed)
    T.make_args = spy

    # ---- alone: what a single process computes -------------------------------------------------------------
    os.chdir(city_root)
    train_ds = D.SatMapDataset(TRAIN_CFG, is_train=True, dev_run=True, device=dev)
    os.chdir(spacenet_root)
    val_ds = D.SatMapDataset(VAL_CFG, is_train=False, dev_run=True, device=dev)
    torch.manual_seed(SEED)
    single_batch = next(iter(train_ds.loader(4)))

    # heads differ per rank (DDP's broadcast must replace them), the frozen encoder is the same checkpoint
    sd = synth.make_state_dict(TRAIN_CFG, seed=0, logit_gain=4.0)
    own = synth.make_state_dict(TRAIN_CFG, seed=10 + rank, logit_gain=4.0)
    sd.update({k: v for k, v in own.items() if k.startswith(("map_decoder.", "topo_net."))})
    net = SAMRoad(TRAIN_CFG)
    net.load_state_dict(sd)
    net = net.to(dev)
    batches = [_fixed_batch(40 + r, dev) for r in range(world)]
    net.train()
    torch.manual_seed(SEED)
    net.training_step(batches[0], 0)
    single_seed = seeds[-1]
    net.eval()
    probe = _fixed_batch(99, dev)
    res["pre_wrap"] = _infer(net, probe)[2].cpu().numpy()     # packs this rank's own heads

    vnet = SAMRoad(VAL_CFG)
    vnet.load_state_dict(synth.make_state_dict(VAL_CFG, seed=1, logit_gain=6.0))
    vnet = vnet.to(dev).eval()
    n_val = len(val_ds)
    for r in range(world):       # every rank's batches, in one process, seeded as rank r seeds them
        idx = list(torch.utils.data.DistributedSampler(range(n_val), num_replicas=world, rank=r, shuffle=False))
        torch.manual_seed(SEED)
        for j, first in enumerate(range(0, len(idx), VAL_B)):
            chunk = idx[first:first + VAL_B]
            seed = rank_seed(int(torch.randint(0, 2 ** 62, (), dtype=torch.int64).item()), r)
            vnet.validation_step(val_ds._scenes.batch(len(chunk), patches=val_ds.patches_at(chunk), seed=seed), j)
    single_val = vnet.on_validation_epoch_end()
    res["single_val"] = np.array([single_val[k] for k in METRICS], np.float32)

    # ---- in the group ----------------------------------------------------------------------------------------
    kw = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        torch.manual_seed(SEED)
        loader = train_ds.loader(4)
        batch = next(iter(loader))
        res["train_len_ok"] = len(loader) == -(-(-(-len(train_ds) // world)) // 4)
        res["train_batch_is_single"] = all(torch.equal(batch[k], single_batch[k]) for k in batch) and \
            batch["graph_points"].shape == single_batch["graph_points"].shape

        net.train()
        torch.manual_seed(SEED)
        net.training_step(batches[0], 0)
        res["dropout_seed_is_single"] = seeds[-1] == single_seed
        res["keep"] = T.dropout_keep(0.1, seeds[-1], 1, 2, 1 << 16, dev).cpu().numpy()
        net.eval()                                   # no dropout from here on

        net.setup("fit")
        ddp = DistributedDataParallel(_StepModule(net), device_ids=[dev.index])
        heads = net._head_params()
        params = [p for _, p in heads]
        res["head_names"] = np.array([k for k, _ in heads])
        res["wrapped_heads"] = np.concatenate([p.detach().cpu().numpy().ravel() for p in params])
        res["post_wrap"] = _infer(net, probe)[2].cpu().numpy()

        # each batch alone (synced weights, identical on every rank); autograd.grad leaves .grad and DDP alone
        alone = [torch.autograd.grad(net.training_step(b, 0), params) for b in batches]
        mean = [sum(gs) / world for gs in zip(*alone)]

        opt = net.configure_optimizers()["optimizer"]
        scaler = torch.amp.GradScaler("cuda")
        for step in range(3):
            loss = ddp(batches[rank], step)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            if step == 0:
                res["grads"] = np.concatenate([p.grad.cpu().numpy().ravel() for p in params])
                worst = 0.0
                for p, m in zip(params, mean):
                    err, ref = (p.grad - m).abs().max().item(), m.abs().max().item()
                    worst = max(worst, err / ref if ref > 0 else (0.0 if err == 0 else float("inf")))
                res["grad_vs_mean"] = np.float64(worst)
            scaler.step(opt)
            scaler.update()
            opt.zero_grad(set_to_none=True)
            assert all(p.grad is None for p in params)
        res["scale"] = np.float64(scaler.get_scale())
        res["trained_heads"] = np.concatenate([p.detach().cpu().numpy().ravel() for p in params])
        after = _infer(net, probe)
        res["after"] = [t.cpu().numpy() for t in after]
        fresh = SAMRoad(TRAIN_CFG)                 # the host pack of the same parameters
        fresh.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()})
        res["repack_is_host_pack"] = _equal(after, _infer(fresh.to(dev).eval(), probe))
        enc = {k: v for k, v in sd.items() if k.startswith("image_encoder.")}
        res["encoder_unchanged"] = all(torch.equal(p.detach().cpu(), enc[k]) for k, p in net.named_parameters()
                                       if k in enc)

        torch.manual_seed(SEED)
        vloader = val_ds.loader(VAL_B)
        n_batches = 0
        for j, b in enumerate(vloader):
            vnet.validation_step(b, j)
            n_batches += 1
        res["val_len_ok"] = len(vloader) == n_batches == -(-(-(-n_val // world)) // VAL_B)
        out = vnet.on_validation_epoch_end()
        res["val"] = np.array([out[k] for k in METRICS], np.float32)
    finally:
        dist.destroy_process_group()
    after = res.pop("after")
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), scores=after[0], emb=after[1], topo=after[2], **res)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def city_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("cityscale_scenes"))
    synth.write_label_scenes(root, "cityscale", CITY_TRAIN, 2048, seed=5, extent=1200)
    return root


@pytest.fixture(scope="module")
def spacenet_root(tmp_path_factory):
    import json
    root = str(tmp_path_factory.mktemp("spacenet_scenes"))
    synth.write_label_scenes(root, "spacenet", sum(SPACENET.values(), []), 400, seed=9, extent=380)
    with open(os.path.join(root, "spacenet", "data_split.json"), "w") as f:
        json.dump(SPACENET, f)
    return root


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_ddp_training_and_sharded_validation(backend, city_root, spacenet_root, tmp_path):
    if backend == "nccl" and torch.cuda.device_count() < WORLD:
        pytest.skip(f"NCCL needs {WORLD} GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, WORLD, port, backend, city_root, spacenet_root, str(tmp_path)))
             for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=600)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    r0, r1 = (dict(np.load(os.path.join(str(tmp_path), f"rank{r}.npz"))) for r in range(WORLD))
    bits = lambda a: np.ascontiguousarray(a).view(np.uint32)  # noqa: E731

    # batches and dropout: rank 0 is the single process, rank 1 is not
    assert r0["train_len_ok"] and r1["train_len_ok"]
    assert r0["train_batch_is_single"] and not r1["train_batch_is_single"]
    assert r0["dropout_seed_is_single"] and not r1["dropout_seed_is_single"]
    assert not np.array_equal(r0["keep"], r1["keep"])

    # the wrap-time broadcast: rank 1's own heads are replaced by rank 0's, and so are their packed copies
    assert not np.array_equal(r0["pre_wrap"], r1["pre_wrap"])
    np.testing.assert_array_equal(bits(r1["wrapped_heads"]), bits(r0["wrapped_heads"]))
    np.testing.assert_array_equal(bits(r1["post_wrap"]), bits(r0["post_wrap"]))
    np.testing.assert_array_equal(bits(r0["post_wrap"]), bits(r0["pre_wrap"]))

    # one step: DDP's mean of the two ranks' gradients, the same bits on both ranks
    np.testing.assert_array_equal(bits(r0["grads"]), bits(r1["grads"]))
    assert r0["grad_vs_mean"] <= 1e-6 and r1["grad_vs_mean"] <= 1e-6, (r0["grad_vs_mean"], r1["grad_vs_mean"])

    # three GradScaler + Adam steps: moved, identical replicas, packed weights that follow them
    assert r0["scale"] == r1["scale"] == 65536.0        # no step was skipped
    assert not np.array_equal(r0["trained_heads"], r0["wrapped_heads"])
    np.testing.assert_array_equal(bits(r0["trained_heads"]), bits(r1["trained_heads"]))
    for k in ("scores", "emb", "topo"):
        np.testing.assert_array_equal(bits(r0[k]), bits(r1[k]), err_msg=k)
    assert r0["repack_is_host_pack"] and r1["repack_is_host_pack"]
    assert r0["encoder_unchanged"] and r1["encoder_unchanged"]

    # sharded validation: the whole padded split's metrics on every rank
    assert r0["val_len_ok"] and r1["val_len_ok"]
    for r in (r0, r1):
        np.testing.assert_array_equal(bits(r["val"]), bits(r0["single_val"]))
        np.testing.assert_array_equal(bits(r["single_val"]), bits(r0["single_val"]))
    assert np.isfinite(r0["val"]).all()
