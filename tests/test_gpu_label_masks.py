"""GPU: the label masks of csrc/label_masks.cu (sam_road_b200.label_masks) bit for bit against the OpenCV
restatement of oracle/label_mask_oracle.py and against tests/golden/label_masks.npz (the reference scripts' own
cv2 drawing); mixed tiles in one launch, 180 CityScale tiles in one call, and the command end to end on a
synthetic dataset layout that SatMapDataset then reads."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import label_mask_oracle as LM
from sam_road_b200 import dataset as D
from sam_road_b200 import label_masks as L
from sam_road_b200 import synth

from test_label_masks_host import GRID, golden_tiles

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NONE = np.zeros((0, 2), np.int32)


def _segments(segs, size, width):
    """One tile per segment: the device masks next to the oracle's."""
    edges = [np.array([p + q], np.int32) for p, q in segs]
    _, road = L.draw_masks([NONE] * len(segs), edges, size, DEV, road_width=width)
    got = road.cpu().numpy()
    for k, (p, q) in enumerate(segs):
        want = np.zeros((size, size), np.uint8)
        LM.thick_line(want, p, q, width)
        assert np.array_equal(got[k], want), (p, q, width, np.argwhere(got[k] != want)[:5].tolist())


@pytest.mark.parametrize("width", range(2, 9))
def test_every_grid_segment_equals_oracle(width):
    pts = [(x, y) for x in GRID for y in GRID]
    _segments([(p, q) for p in pts for q in pts], 24, width)


def test_long_segments_far_outside_equal_oracle():
    rng = np.random.default_rng(11)
    segs = []
    for k in range(24):
        p = tuple(int(v) for v in rng.integers(-100000, 100001, 2))
        q = tuple(int(v) for v in rng.integers(-300, 2400, 2))
        segs.append((q, p) if k % 2 else (p, q))
    _segments(segs, 2048, 3)


@pytest.mark.parametrize("radius", [0, 1, 2, 3, 5, 10, 40])
def test_discs_near_the_border_equal_oracle(radius):
    centres = [(cx, cy) for cx in range(-12, 36) for cy in (-12, -4, -1, 0, 1, 3, 11, 20, 22, 23, 24, 27, 35)]
    centres += [(y, x) for x, y in centres]
    kp, road = L.draw_masks([np.array([c], np.int32) for c in centres], [np.zeros((0, 4), np.int32)] * len(centres),
                            24, DEV, keypoint_radius=radius)
    got = kp.cpu().numpy()
    assert not road.any()
    for k, c in enumerate(centres):
        want = np.zeros((24, 24), np.uint8)
        LM.circle_fill(want, c[0], c[1], radius)
        assert np.array_equal(got[k], want), (c, radius)


@pytest.mark.parametrize("dataset", ["cityscale", "spacenet"])
def test_golden_tiles(dataset):
    tiles = [(name, adj, kp, road) for name, (ds, adj, kp, road) in golden_tiles().items() if ds == dataset]
    kp, road = L.masks_from_graphs([t[1] for t in tiles], dataset, DEV)
    kp, road = kp.cpu().numpy(), road.cpu().numpy()
    for k, (name, _, want_kp, want_road) in enumerate(tiles):
        assert np.array_equal(kp[k], want_kp) and np.array_equal(road[k], want_road), name


def test_mixed_tiles_in_one_launch():
    adjs = [synth.make_road_graph(400, seed=1, spacing=40, lo=0), {},
            {(10.0, 10.0): [(10.0, 10.0)], (200.0, 300.0): [(200.0, 300.0)], (399.0, 0.0): [(399.0, 0.0)]},
            synth.make_road_graph(384, seed=2), {(5.0, 5.0): []}]
    kp, road = L.masks_from_graphs(adjs, "spacenet", DEV)
    kp, road = kp.cpu().numpy(), road.cpu().numpy()
    for k, adj in enumerate(adjs):
        want_kp, want_road = LM.tile_masks(adj, "spacenet", 400)
        assert np.array_equal(kp[k], want_kp) and np.array_equal(road[k], want_road), k
    assert not kp[1].any() and not road[1].any() and not kp[4].any() and not road[4].any()
    assert not kp[2].any() and road[2].any()       # self-loops: degree 2, caps only


def test_180_cityscale_tiles_in_one_call():
    graphs = [synth.city_tile(2048, seed=s)[s % 2] for s in range(3)]
    wants = [LM.tile_masks(g, "cityscale", 2048) for g in graphs]
    kp, road = L.masks_from_graphs([graphs[t % 3] for t in range(180)], "cityscale", DEV)
    torch.cuda.synchronize()
    for t in range(180):
        want_kp, want_road = wants[t % 3]
        assert torch.equal(kp[t].cpu(), torch.from_numpy(want_kp)), t
        assert torch.equal(road[t].cpu(), torch.from_numpy(want_road)), t


def test_command_writes_what_the_dataset_reads(tmp_path, monkeypatch):
    import cv2
    names = {"train": ["AOI_2_Vegas_1"], "validation": ["AOI_3_Paris_3"], "test": ["AOI_4_Shanghai_4", "AOI_2_Vegas_6"]}
    root = str(tmp_path)
    synth.write_label_scenes(root, "spacenet", sum(names.values(), []), 400, seed=3, extent=380)
    with open(os.path.join(root, "spacenet", "data_split.json"), "w") as f:
        json.dump(names, f)
    keep = os.path.join(root, "spacenet", "processed", "notes.txt")
    open(keep, "w").write("kept")
    monkeypatch.chdir(root)
    L.main(["--dataset", "spacenet"])
    assert open(keep).read() == "kept"
    for tile in sum(names.values(), []):
        with open(os.path.join(root, "spacenet", "RGB_1.0_meter", f"{tile}__gt_graph.p"), "rb") as f:
            want_kp, want_road = LM.tile_masks(pickle.load(f), "spacenet", 400)
        for name, want in (("keypoint", want_kp), ("road", want_road)):
            got = cv2.imread(os.path.join(root, "spacenet", "processed", f"{name}_mask_{tile}.png"),
                             cv2.IMREAD_GRAYSCALE)
            assert np.array_equal(got, want), (tile, name)
    cfg = dict(DATASET="spacenet", PATCH_SIZE=256, TOPO_SAMPLE_NUM=32, MAX_NEIGHBOR_QUERIES=8, NEIGHBOR_RADIUS=64,
               ROAD_NMS_RADIUS=16)
    ds = D.SatMapDataset(cfg, is_train=False, dev_run=True, device=DEV)
    batch = ds.batch(2)
    with open(os.path.join(root, "spacenet", "RGB_1.0_meter", f"{names['test'][0]}__gt_graph.p"), "rb") as f:
        want_kp, want_road = LM.tile_masks(pickle.load(f), "spacenet", 400)
    for k in range(2):
        _, (x0, y0), _ = ds.eval_patches[k]
        for key, want in (("keypoint_mask", want_kp), ("road_mask", want_road)):
            got = batch[key][k].cpu().numpy()
            assert np.array_equal(got > 0, want[y0:y0 + 256, x0:x0 + 256] > 0), (k, key)
