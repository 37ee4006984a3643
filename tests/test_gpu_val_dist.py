"""GPU, several processes: under torch.distributed the validation metrics are those of every rank's steps
(the ranks sum their counts, as torchmetrics' sync on compute does) while each rank keeps its own epoch
losses (the reference logs them without sync_dist); a refused step on one rank raises on every rank, and a
rank that ran no step still joins.  gloo runs several ranks on one GPU; NCCL needs one GPU per rank."""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import val_oracle as VO

pytestmark = pytest.mark.gpu
WORLD = 2


def _data(rank, dev):
    g = torch.Generator(device=dev).manual_seed(200 + rank)
    B, P, Ns, Np = 2 + rank, 128, 20, 16                        # ragged shards
    ml = torch.randn((B, P, P, 2), generator=g, device=dev) * 4
    kp = (torch.rand((B, P, P), generator=g, device=dev) < 0.3).float()
    road = (torch.rand((B, P, P), generator=g, device=dev) < 0.5).float()
    tl = torch.randn((B, Ns, Np, 1), generator=g, device=dev) * 3
    connected = torch.rand((B, Ns, Np), generator=g, device=dev) < 0.4
    valid = torch.rand((B, Ns, Np), generator=g, device=dev) < 0.7
    return ml, torch.sigmoid(ml), kp, road, tl, torch.sigmoid(tl), connected, valid


def _worker(rank, world, port, backend, out_dir):
    import torch.distributed as dist
    from sam_road_b200 import SAMRoad, synth
    from sam_road_b200.metrics import ValidationMetrics
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    kw = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    res = {}
    try:
        args = _data(rank, dev)
        vm = ValidationMetrics(dev)
        res["step"] = vm.update(*args).cpu().numpy()
        out = vm.compute()
        res["metrics"] = np.array([out[k] for k in ("keypoint_iou", "road_iou", "topo_f1")], np.float32)
        res["losses"] = np.array([out[k] for k in ("val_mask_loss", "val_topo_loss", "val_loss")], np.float32)
        c = VO.step_counts(args[1].cpu().numpy(), args[2].cpu().numpy(), args[3].cpu().numpy(),
                           args[5].cpu().numpy(), args[6].cpu().numpy(), args[7].cpu().numpy())
        res["counts"] = np.array(list(c.values()), np.int64)
        res["count_names"] = np.array(list(c.keys()))

        bad = ValidationMetrics(dev)
        bad.update(*args)
        if rank == 1:
            worse = list(args)
            worse[3] = worse[3].clone()
            worse[3][0, 0, 1] = 0.5
            bad.update(*worse)
        try:
            bad.compute()
            res["refusal"] = "none"
        except RuntimeError as e:
            res["refusal"] = str(e)

        # SAMRoad: rank 0 runs a validation step, rank 1 none; both reach the epoch end
        cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False, ENCODER_LORA=False,
                   TOPONET_VERSION="normal", NO_SAM=False)
        net = SAMRoad(cfg)
        net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=8.0), strict=True)
        net.eval().to(dev)
        if rank == 0:
            gen = torch.Generator().manual_seed(300)
            pts, prs, val = synth.make_topo_inputs(2, 256, 30, seed=301)
            batch = {"rgb": synth.make_tiles(2, 256, seed=302, dtype=torch.float32),
                     "keypoint_mask": (torch.rand((2, 256, 256), generator=gen) < 0.3).float(),
                     "road_mask": (torch.rand((2, 256, 256), generator=gen) < 0.3).float(),
                     "graph_points": pts.float(), "pairs": prs.to(torch.int32),
                     "connected": torch.rand(val.shape, generator=gen) < 0.5, "valid": val}
            batch = {k: v.to(dev) for k, v in batch.items()}
            net.validation_step(batch, 0)
            ml, ms, tl, ts = net(batch["rgb"], batch["graph_points"], batch["pairs"], batch["valid"])
            c = VO.step_counts(ms.cpu().numpy(), batch["keypoint_mask"].cpu().numpy(),
                               batch["road_mask"].cpu().numpy(), ts.cpu().numpy(), batch["connected"].cpu().numpy(),
                               batch["valid"].cpu().numpy())
            res["net_expect"] = np.array([VO.epoch_metrics(c)[k] for k in ("keypoint_iou", "road_iou", "topo_f1")],
                                         np.float32)
        out = net.on_validation_epoch_end()
        res["net_metrics"] = np.array([out[k] for k in ("keypoint_iou", "road_iou", "topo_f1")], np.float32)
        res["net_loss"] = np.float32(out["val_loss"])
    finally:
        dist.destroy_process_group()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **res)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_metrics_sum_every_rank(backend, tmp_path):
    if backend == "nccl" and torch.cuda.device_count() < WORLD:
        pytest.skip(f"NCCL needs {WORLD} GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, WORLD, port, backend, str(tmp_path))) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=300)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    ranks = [dict(np.load(os.path.join(str(tmp_path), f"rank{r}.npz"))) for r in range(WORLD)]
    names = [str(n) for n in ranks[0]["count_names"]]
    union = dict(zip(names, (int(v) for v in ranks[0]["counts"] + ranks[1]["counts"])))
    expect = VO.epoch_metrics(union)
    for r in ranks:
        got = r["metrics"]
        want = np.array([expect[k] for k in ("keypoint_iou", "road_iou", "topo_f1")], np.float32)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
        np.testing.assert_array_equal(r["losses"].view(np.uint32), r["step"].view(np.uint32))   # its own
    assert not np.array_equal(ranks[0]["losses"], ranks[1]["losses"])
    refusal = [str(r["refusal"]) for r in ranks]
    assert "refused" in refusal[1] and "a mask target" in refusal[1], refusal
    assert "1 other rank(s) refused" in refusal[0], refusal
    for r in ranks:         # rank 1 ran no step: the metrics are rank 0's, on both ranks
        np.testing.assert_array_equal(r["net_metrics"].view(np.uint32), ranks[0]["net_expect"].view(np.uint32))
    assert np.isnan(ranks[1]["net_loss"]) and not np.isnan(ranks[0]["net_loss"])
