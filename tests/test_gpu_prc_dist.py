"""GPU, several processes: under torch.distributed the precision-recall curves and SAMRoad.on_test_end
report the whole split on every rank (the ranks gather their entries, as torchmetrics' sync on compute
does), bit for bit against the oracle on the concatenated data; a refused update on one rank raises on
every rank instead of leaving the others waiting.  gloo runs several ranks on one GPU; NCCL needs one GPU
per rank."""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import prc_oracle as PO

pytestmark = pytest.mark.gpu
WORLD = 2


def _data(n=40_000):
    gen = torch.Generator().manual_seed(11)
    k = torch.randint(0, 256, (n,), generator=gen)
    preds = torch.where(torch.rand(n, generator=gen) < 0.5, k.float() / 255.0, torch.rand(n, generator=gen))
    target = (torch.rand(n, generator=gen) < preds * 0.8).to(torch.uint8)
    return preds, target


def _shard(rank, n):
    cut = [0, n // 3, n]     # ragged shards
    return slice(cut[rank], cut[rank + 1])


def _worker(rank, world, port, backend, out_dir):
    import torch.distributed as dist
    from sam_road_b200 import SAMRoad, synth
    from sam_road_b200.metrics import PrecisionRecallCurve
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    kw = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    res = {}
    try:
        preds, target = _data()
        sl = _shard(rank, preds.numel())
        curve = PrecisionRecallCurve(dev)
        curve.update(preds[sl].to(dev), target[sl].to(dev))
        prec, rec, thr = (t.cpu().numpy() for t in curve.compute())
        res.update(prec=prec, rec=rec, thr=thr, best=np.array([x.item() for x in curve.best()], np.float32))

        bad = PrecisionRecallCurve(dev)
        bad.update(preds[sl].to(dev), target[sl].to(dev))
        if rank == 1:
            bad.update(torch.full((5,), 1.5, device=dev), torch.zeros(5, dtype=torch.uint8, device=dev))
        try:
            bad.compute()
            res["refusal"] = "none"
        except RuntimeError as e:
            res["refusal"] = str(e)

        cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False, ENCODER_LORA=False,
                   TOPONET_VERSION="normal", NO_SAM=False)
        net = SAMRoad(cfg)
        net.load_state_dict(synth.make_state_dict(cfg, seed=0, logit_gain=8.0), strict=True)
        net.eval().to(dev)
        gen = torch.Generator().manual_seed(100 + rank)        # each rank its own batches
        pts, prs, val = synth.make_topo_inputs(2, 256, 30, seed=30 + rank)
        masks = [(torch.rand((2, 256, 256), generator=gen) < 0.3).float() for _ in range(2)]
        batch = {"rgb": synth.make_tiles(2, 256, seed=40 + rank, dtype=torch.float32),
                 "keypoint_mask": masks[0], "road_mask": masks[1], "graph_points": pts.float(),
                 "pairs": prs.to(torch.int32), "connected": torch.rand(val.shape, generator=gen) < 0.5,
                 "valid": val}
        batch = {k: v.to(dev) for k, v in batch.items()}
        net.test_step(batch, 0)
        ms, emb = net.infer_masks_and_img_features(batch["rgb"])
        ts = net.infer_toponet(emb, batch["graph_points"], batch["pairs"], batch["valid"])
        kp, road, topo = PO.test_step_targets({k: v.cpu() for k, v in batch.items()})
        for name, s, t in (("keypoint", ms[..., 0], kp), ("road", ms[..., 1], road), ("topo", ts, topo)):
            res[f"s_{name}"] = s.cpu().numpy().ravel()
            res[f"t_{name}"] = t.numpy().ravel()
        best = net.on_test_end()
        for name, v in best.items():
            res[f"best_{name}"] = np.array(v, np.float32)
    finally:
        dist.destroy_process_group()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **res)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_array_equal(a[~np.isnan(a)].view(np.uint32), b[~np.isnan(b)].view(np.uint32))


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_curves_gather_every_rank(backend, tmp_path):
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
    preds, target = _data()
    oprec, orec, othr = PO.binary_pr_curve(preds.numpy(), target.numpy())
    obest = PO.find_best_threshold(oprec, orec, othr)[1:]
    for r in ranks:
        _same_bits(r["thr"], othr)
        _same_bits(r["prec"], oprec)
        _same_bits(r["rec"], orec)
        _same_bits(r["best"], obest)
    refusal = [str(r["refusal"]) for r in ranks]
    assert "refused" in refusal[1] and "element 0" in refusal[1], refusal
    assert "rank 1 could not contribute" in refusal[0], refusal
    for name in ("keypoint", "road", "topo"):
        s = np.concatenate([r[f"s_{name}"] for r in ranks])
        t = np.concatenate([r[f"t_{name}"] for r in ranks])
        expect = PO.find_best_threshold(*PO.binary_pr_curve(s, t))[1:]
        for r in ranks:
            _same_bits(r[f"best_{name}"], expect)
