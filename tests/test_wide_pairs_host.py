"""CPU: MAX_NEIGHBOR_QUERIES above 16.  The oracle TopoNet against the fixture the unmodified reference
produced at 17, 24 and 32 pairs per sample (tools/make_golden.py --wide-pairs), and the oracle's
index-ordered kNN (what the device kNN reproduces) against scipy's at K = 24 and 32."""
import os

import numpy as np
import pytest
import torch

from oracle import samroad_oracle as O
from sam_road_b200 import inferencer as I
from sam_road_b200 import synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5


@pytest.mark.parametrize("n_pairs", [17, 24, 32])
def test_toponet_wide_npairs_against_reference_golden(n_pairs):
    """Inputs as tools/make_golden.py:toponet_npairs_inputs: Ns = 13 samples of N = 20 points, an
    all-invalid row, int64 and float32 points."""
    g = np.load(os.path.join(GOLD, "toponet_npairs_wide.npz"))
    cfg = dict(SAM_VERSION="vit_b", PATCH_SIZE=256, USE_SAM_DECODER=False, ENCODER_LORA=False, LORA_RANK=0,
               TOPONET_VERSION="normal", NO_SAM=False)
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


@pytest.mark.parametrize("K", [24, 32])
def test_wide_pair_queries_index_ties_vs_scipy(K):
    """knn_by_index pins scipy's order of equidistant neighbours to ascending index; wherever the K + 2
    nearest distances of a query are all distinct the two must agree exactly, and some query must be
    truncated at K."""
    rng = np.random.RandomState(K)
    gp = np.unique(rng.randint(0, 400, size=(500, 2)), axis=0).astype(np.int64)
    tiles = I.get_patch_info_one_img(0, 400, 0, 256, 4)
    R = 64.0
    n_rows = n_tied = n_full = 0
    for t in tiles:
        a = O.build_pair_queries(gp, t, K, R, "scipy")
        b = O.build_pair_queries(gp, t, K, R, "index")
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[3], b[3])
        assert a[2].shape[1] == K
        pts = a[1]
        d2 = ((pts[:, None, :] - pts[None, :, :]) ** 2).sum(-1)
        for i in range(pts.shape[0]):
            near = np.sort(d2[i][d2[i] < R * R])[: K + 2]
            tied = np.any(np.diff(near) == 0)
            n_rows += 1
            n_tied += int(tied)
            n_full += int(b[3][i].all())
            if not tied:
                assert np.array_equal(a[2][i], b[2][i])
            else:   # same distances slot by slot, whatever the order inside a tie group
                da = d2[i][a[2][i, :, 1]][a[3][i]]
                db = d2[i][b[2][i, :, 1]][b[3][i]]
                assert np.array_equal(da, db)
    assert n_rows > 500 and n_tied > 0 and n_full > 0, (n_rows, n_tied, n_full)
