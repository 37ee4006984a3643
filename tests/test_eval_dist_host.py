"""CPU: the evaluation commands under torch.distributed -- which rank takes which scene and tile, that the TOPO and
APLS files written rank by rank are those of one process (with the oracle scorers), the run directory rank 0 names
for every rank, and the status check that fails every rank when one rank's share fails (two gloo processes)."""
import filecmp
import json
import os
import pickle
import socket
from collections import Counter

import numpy as np
import pytest

from oracle import apls_oracle, topo_oracle
from sam_road_b200 import apls_metric as AM
from sam_road_b200 import ranks, synth
from sam_road_b200 import topo_metric as TM

WORLDS = (1, 2, 3, 8)
CITY_IDS = [x for x in range(180) if x % 10 == 9 or x % 20 == 8]      # the inferencer's CityScale test ids
TILES = [8, 9, 19, 28, 29]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("n", [0, 1, 2, 5, 27])
def test_shard_takes_every_item_once(n, world):
    got = [list(ranks.shard(n, r, world)) for r in range(world)]
    assert sorted(sum(got, [])) == list(range(n))
    for r, mine in enumerate(got):
        assert mine == list(range(n))[r::world]
    with pytest.raises(ValueError, match="rank"):
        ranks.shard(n, world, world)


@pytest.mark.parametrize("world", WORLDS)
def test_cityscale_scenes_over_ranks(world):
    per_rank = [[CITY_IDS[i] for i in ranks.shard(len(CITY_IDS), r, world)] for r in range(world)]
    assert [len(m) for m in per_rank] == [len(CITY_IDS[r::world]) for r in range(world)]
    assert sorted(sum(per_rank, [])) == CITY_IDS
    assert per_rank[0][0] == 8 and (world == 1 or per_rank[1][0] == 9)


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    """Five CityScale tiles.  Tile 8's ground truth has a key 1200 px down (no edges): the min_lat it carries makes
    every later tile score with r = 0.003 instead of 0.0015, so a rank that did not read it would write other files.
    In the APLS runs tile 19 has no proposal graph, so it is skipped."""
    root = tmp_path_factory.mktemp("eval_split")
    (root / "cityscale" / "20cities").mkdir(parents=True)
    (root / "graph").mkdir()
    for k, (t, ext) in enumerate(zip(TILES, (160, 200, 170, 180, 150))):
        gt = synth.make_road_graph(ext, seed=k)
        if k == 0:
            gt[(1200, 40)] = []
        with open(TM.gt_path("cityscale", str(root / "cityscale"), t), "wb") as f:
            pickle.dump(gt, f)
        with open(root / "graph" / f"{t}.p", "wb") as f:
            pickle.dump(synth.make_road_graph(ext, seed=k + 100), f)
    return root


def _save(root, name, apls=False):
    save = root / name
    (save / "graph").mkdir(parents=True)
    for t in TILES:
        if not (apls and t == 19):
            (save / "graph" / f"{t}.p").write_bytes((root / "graph" / f"{t}.p").read_bytes())
    return save


def _same_files(a, b):
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b))
    for n in names:
        assert filecmp.cmp(os.path.join(a, n), os.path.join(b, n), shallow=False), n
    return names


@pytest.fixture(scope="module")
def single(split):
    save = _save(split, "single")
    TM.run_tiles(str(save), "cityscale", str(split / "cityscale"), tiles=TILES, scorer=topo_oracle.scorer)
    topo = TM.aggregate(str(save), "cityscale")
    asave = _save(split, "single_apls", apls=True)
    AM.run_tiles(str(asave), "cityscale", str(split / "cityscale"), tiles=TILES, scorer=apls_oracle.scorer)
    AM.aggregate(str(asave), "cityscale")
    return save, topo, asave


@pytest.mark.parametrize("world", WORLDS)
def test_topo_tiles_over_ranks_write_the_single_process_files(split, single, world, tmp_path):
    save1, topo1, _ = single
    save = _save(split, f"topo_w{world}")
    for rank in reversed(range(world)):     # no rank depends on another's files
        TM.run_tiles(str(save), "cityscale", str(split / "cityscale"), tiles=TILES, scorer=topo_oracle.scorer,
                     rank=rank, world=world)
    names = _same_files(save1 / "results" / "topo", save / "results" / "topo")
    assert len(names) == 2 * len(TILES)
    got = TM.aggregate(str(save), "cityscale")
    for k in ("prec", "recall", "f1"):
        assert Counter(got[k]) == Counter(topo1[k])
    assert np.allclose(got["mean topo"], topo1["mean topo"], rtol=1e-15, atol=0)
    # the state carried from tile 8 reached every rank (each .topo.p holds the region it came from)
    for t in TILES:
        region = pickle.load(open(save / "results" / "topo" / f"{t}.topo.p", "rb"))[2]
        assert 41.0 - region[0] > 1200 / 111111.0


@pytest.mark.parametrize("world", WORLDS)
def test_apls_tiles_over_ranks_write_the_single_process_files(split, single, world):
    _, _, asave1 = single
    save = _save(split, f"apls_w{world}", apls=True)
    for rank in reversed(range(world)):
        AM.run_tiles(str(save), "cityscale", str(split / "cityscale"), tiles=TILES, scorer=apls_oracle.scorer,
                     rank=rank, world=world)
    names = _same_files(asave1 / "results" / "apls", save / "results" / "apls")
    assert names == sorted(f"{t}.txt" for t in TILES if t != 19)
    AM.aggregate(str(save), "cityscale")
    assert (save / "score" / "apls.json").read_bytes() == (asave1 / "score" / "apls.json").read_bytes()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, root, out):
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from sam_road_b200 import inferencer
    os.chdir(root)
    res = {}
    with ranks.process_group() as (r, w):
        res["rank_world"] = [r, w, dist.get_backend()]
        # rank 1's clock reads another second: the name is rank 0's all the same
        if rank == 1:
            inferencer.time.strftime = lambda fmt: "rank1_clock"
        res["out_dir"] = inferencer.output_dir(None)
        res["named_dir"] = inferencer.output_dir("named")
        res["max"] = ranks.max_over_ranks(1.5 + rank)
        res["ok"] = ranks.run_checked(lambda: rank * 10)

        def fails_on_rank_1():
            if rank == 1:
                raise FileNotFoundError("no proposal graph for tile 19")
            return "fine"
        try:
            ranks.run_checked(fails_on_rank_1)
            res["refusal"] = None
        except RuntimeError as e:
            res["refusal"] = [str(e), type(e.__cause__).__name__ if e.__cause__ else None]
        # the real loop: rank 1's second tile has no proposal graph; rank 0 stops after its own tile
        save = os.path.join(root, "topo_missing")
        try:
            ranks.run_checked(TM.run_tiles, save, "cityscale", os.path.join(root, "cityscale"), tiles=[8, 9],
                              scorer=topo_oracle.scorer, rank=r, world=w)
            res["topo_refusal"] = None
        except RuntimeError as e:
            res["topo_refusal"] = str(e)
    res["destroyed"] = not dist.is_initialized()
    with open(os.path.join(out, f"rank{rank}.json"), "w") as f:
        json.dump(res, f)


def test_two_gloo_ranks_share_the_run_directory_and_every_refusal(split, tmp_path):
    import torch.multiprocessing as mp
    root = tmp_path / "run"
    (root / "topo_missing" / "graph").mkdir(parents=True)
    (root / "cityscale").symlink_to(split / "cityscale")
    (root / "topo_missing" / "graph" / "8.p").write_bytes((split / "graph" / "8.p").read_bytes())
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(root), str(tmp_path))) for r in range(2)]
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
    assert not mp.active_children()
    r0, r1 = (json.loads((tmp_path / f"rank{r}.json").read_text()) for r in range(2))
    assert r0["rank_world"] == [0, 2, "gloo"] and r1["rank_world"] == [1, 2, "gloo"]
    assert r0["out_dir"] == r1["out_dir"] and r0["out_dir"].startswith("./save/infer_")
    assert "rank1_clock" not in r0["out_dir"]
    assert sorted(os.listdir(root / "save")) == sorted([os.path.basename(r0["out_dir"]), "named"])
    for d in (r0["out_dir"], "save/named"):
        assert sorted(os.listdir(root / d)) == ["graph", "mask", "viz"]
    assert r0["named_dir"] == r1["named_dir"] == "./save/named"
    assert r0["max"] == r1["max"] == 2.5
    assert (r0["ok"], r1["ok"]) == (0, 10)
    msg = "rank 1 of 2 failed: FileNotFoundError: no proposal graph for tile 19"
    assert r0["refusal"] == [msg, None] and r1["refusal"] == [msg, "FileNotFoundError"]
    for r in (r0, r1):
        assert r["topo_refusal"].startswith("rank 1 of 2 failed: FileNotFoundError") and "9.p" in r["topo_refusal"]
        assert r["destroyed"]
    assert sorted(os.listdir(root / "topo_missing" / "results" / "topo")) == ["8.topo.p", "8.txt"]
