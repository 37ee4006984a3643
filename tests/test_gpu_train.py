"""GPU: SAMRoad.training_step / configure_optimizers for FREEZE_ENCODER training of the heads, against the fp32
torch oracle (oracle/train_oracle.py) on the engine's own image embeddings."""
import pytest
import torch

from oracle import train_oracle as TO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200 import train as T

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 5e-3       # ||g - g_ref||_inf <= BOUND * ||g_ref||_inf per tensor
LOSS_RTOL = 1e-5


def _cfg(P=256, version="normal", focal=False):
    return {"SAM_VERSION": "vit_b", "PATCH_SIZE": P, "FREEZE_ENCODER": True, "BASE_LR": 1e-3,
            "TOPONET_VERSION": version, "FOCAL_LOSS": focal}


def _net(cfg, seed=0):
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=seed, logit_gain=4.0))
    return net.to(DEV)


def _batch(B, P, N, Ns, Np, seed):
    g = torch.Generator().manual_seed(seed)
    pts, pairs, valid = synth.make_topo_inputs(B, P, N, seed=seed, max_nbr=Np)
    pairs, valid = pairs[:, :Ns], valid[:, :Ns].clone()
    valid[0, 0] = False                                   # an all-invalid sample row
    b = {"rgb": synth.make_tiles(B, P, seed=seed), "graph_points": pts, "pairs": pairs, "valid": valid,
         "connected": torch.rand(valid.shape, generator=g) < 0.4,
         "keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
         "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}
    return {k: v.to(DEV) for k, v in b.items()}


def _engine_step(net, b, dropout_p=0.0, seed=0):
    """(losses, grads by key, image embeddings) of one device step with incoming gradients 1."""
    net._enable_training()
    heads = net._head_params()
    bb = T.validate_batch(b, net.image_size, DEV)
    args = T.make_args(bb, net.focal_loss, dropout_p, seed)
    s = net.image_size // 16
    emb = torch.empty((bb["B"], 256, s, s), device=DEV)
    ml, tl = T.head_losses(net._handle(DEV), bb, args, [k for k, _ in heads], [p for _, p in heads], emb)
    grads = torch.autograd.grad(ml + tl, [p for _, p in heads])
    return (ml.detach(), tl.detach()), dict(zip([k for k, _ in heads], grads)), emb


def _oracle(net, emb, b, version, keep=None, dropout_p=0.1):
    params = {k: p.detach().clone().requires_grad_(True) for k, p in net._head_params()}
    ml, tl = TO.heads_losses(params, emb, b, net.image_size, net.focal_loss, version, keep, dropout_p)
    (ml + tl).backward()
    return (ml.detach(), tl.detach()), {k: p.grad for k, p in params.items()}


def _compare(got, want, bound=BOUND):
    (gl, gg), (wl, wg) = got, want
    for a, b in zip(gl, wl):
        assert abs(a.item() - b.item()) <= LOSS_RTOL * abs(b.item()), (a.item(), b.item())
    worst = 0.0
    for k, r in wg.items():
        g = gg[k]
        ref = r.abs().max().item()
        err = (g - r).abs().max().item()
        if ref == 0:
            assert err == 0, k
            continue
        assert err <= bound * ref, (k, err, ref)
        worst = max(worst, err / ref)
    return worst


@pytest.mark.parametrize("P,B,version,focal,Np,Ns", [
    (256, 2, "normal", False, 16, 20), (256, 2, "normal", True, 7, 12), (256, 2, "no_offset", False, 32, 9),
    (256, 2, "no_transformer", True, 16, 20), (512, 1, "normal", False, 16, 30), (512, 1, "no_offset", True, 7, 25)])
def test_gradient_parity_eval_mode(P, B, version, focal, Np, Ns):
    net = _net(_cfg(P, version, focal))
    b = _batch(B, P, 40, Ns, Np, seed=P + Np)
    got = _engine_step(net, b)
    want = _oracle(net, got[2], b, version, dropout_p=0.0)
    worst = _compare(got[:2], want)
    print(f"max relative gradient error {worst:.3e}")
    if version == "no_offset":
        assert (got[1]["topo_net.pair_proj.weight"][:, 256:] == 0).all()


def _keep_masks(net, b, seed, p=0.1):
    B, Ns, Np = b["valid"].shape
    rows, tok = B * Ns, B * Ns * Np
    keep = {}
    for l in range(3):
        keep[(l, 0)] = T.dropout_keep(p, seed, l, 0, rows * 4 * Np * Np, DEV).view(rows, 4, Np, Np)
        for site in (1, 2, 3):
            keep[(l, site)] = T.dropout_keep(p, seed, l, site, tok * 128, DEV).view(rows, Np, 128)
    return keep


def test_dropout_train_mode():
    net = _net(_cfg(256, "normal", False))
    b = _batch(2, 256, 40, 30, 16, seed=7)
    keep = _keep_masks(net, b, seed=1234)
    for (l, site), m in keep.items():
        n = m.numel()
        rate = m.float().mean().item()
        assert abs(rate - 0.9) <= 6 * (0.09 / n) ** 0.5, (l, site, rate)
    got = _engine_step(net, b, dropout_p=0.1, seed=1234)
    want = _oracle(net, got[2], b, "normal", keep=keep, dropout_p=0.1)
    _compare(got[:2], want)
    again = _engine_step(net, b, dropout_p=0.1, seed=1234)
    for k in got[1]:
        assert torch.equal(got[1][k], again[1][k]), k
    assert torch.equal(got[0][0], again[0][0]) and torch.equal(got[0][1], again[0][1])
    other = _keep_masks(net, b, seed=1235)
    assert any(not torch.equal(keep[k], other[k]) for k in keep)


def test_training_step_seed_reproducible():
    net = _net(_cfg(256, "normal", True)).train()
    b = _batch(2, 256, 40, 20, 16, seed=3)
    out = []
    for seed in (5, 5, 6):
        torch.manual_seed(seed)
        net.zero_grad(set_to_none=True)
        loss = net.training_step(b, 0)
        loss.backward()
        out.append((loss.detach().clone(), {k: p.grad.clone() for k, p in net._head_params()}))
    assert torch.equal(out[0][0], out[1][0])
    assert all(torch.equal(out[0][1][k], out[1][1][k]) for k in out[0][1])
    assert any(not torch.equal(out[0][1][k], out[2][1][k]) for k in out[0][1] if "transformer" in k)


@pytest.mark.parametrize("P,B,Ns,Np", [(256, 2, 20, 16), (512, 16, 512, 16)])
def test_determinism(P, B, Ns, Np):
    net = _net(_cfg(P))
    b = _batch(B, P, max(Ns, 40), Ns, Np, seed=11)
    first = _engine_step(net, b, dropout_p=0.1, seed=99)
    second = _engine_step(net, b, dropout_p=0.1, seed=99)
    for k in first[1]:
        assert torch.equal(first[1][k], second[1][k]), k


def test_scaling_and_routing():
    net = _net(_cfg(256))
    net._enable_training()
    b = _batch(2, 256, 40, 20, 16, seed=5)
    heads = net._head_params()
    params = [p for _, p in heads]
    bb = T.validate_batch(b, 256, DEV)
    args = T.make_args(bb, False, 0.0, 0)

    def grads(fm, ft):
        ml, tl = T.head_losses(net._handle(DEV), bb, args, [k for k, _ in heads], params)
        return torch.autograd.grad(fm * ml + ft * tl, params, allow_unused=True)

    g1, g1024 = grads(1.0, 1.0), grads(1024.0, 1024.0)
    for a, c in zip(g1, g1024):
        assert torch.equal(a * 1024, c)
    gm, gt = grads(1.0, 0.0), grads(0.0, 1.0)
    for (k, _), a, c in zip(heads, gm, gt):
        if k.startswith("map_decoder."):
            assert (c == 0).all() and (a != 0).any(), k
        else:
            assert (a == 0).all(), k


def test_optimizer_loop_and_refresh():
    cfg = _cfg(256)
    net = _net(cfg)
    b = _batch(2, 256, 40, 20, 16, seed=21)
    enc = {k: p.detach().clone() for k, p in net.named_parameters() if k.startswith("image_encoder.")}
    ref = {k: p.detach().clone().requires_grad_(True) for k, p in net._head_params()}
    start = {k: p.detach().clone() for k, p in ref.items()}
    opt = net.configure_optimizers()["optimizer"]
    ref_opt = torch.optim.Adam([ref[k] for k in ref], lr=cfg["BASE_LR"])
    net.eval()          # no dropout: the oracle follows the same trajectory
    losses = []
    for step in range(30):
        loss = net.training_step(b, step)
        loss.backward()
        if step == 0:
            _, _, emb = net._encode(b["rgb"], False)
        opt.step()
        opt.zero_grad()
        losses.append(loss.item())
        if step < 5:
            ml, tl = TO.heads_losses(ref, emb, b, 256, False, "normal", None, 0.0)
            (ml + tl).backward()
            ref_opt.step()
            ref_opt.zero_grad()
        if step == 4:
            # within BOUND of the parameters for all but 0.1 % of the elements; Adam moves an element by about
            # lr * sign(m), so where a gradient element is ~0 the engine and the oracle may round it to opposite
            # signs: such an element at most mirrors the oracle's own move (error <= twice its displacement)
            for k, p in net._head_params():
                disp = (ref[k].detach() - start[k]).abs()
                err = (ref[k].detach() - p.detach()).abs()
                tol = BOUND * ref[k].detach().abs().max().item()
                if k.endswith("in_proj_bias"):
                    # the key bias: its exact gradient is zero (softmax is invariant to a shift shared by all keys of
                    # a query), so both sides hold rounding noise, which Adam blows up to ~lr steps
                    keep = torch.ones_like(err, dtype=torch.bool)
                    keep[128:256] = False
                    disp, err = disp[keep], err[keep]
                assert (err > tol).float().mean().item() <= 1e-3, k
                assert (err <= 2 * disp + tol).all(), k
        if step in (0, 4, 29):
            # the device refresh equals the host pack of the same values, bit for bit
            fresh = SAMRoad(cfg)
            fresh.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()})
            fresh = fresh.to(DEV)
            with torch.no_grad():
                pts, pairs, valid = b["graph_points"], b["pairs"], b["valid"]
                a = net.forward(b["rgb"], pts, pairs, valid)
                c = fresh.forward(b["rgb"], pts, pairs, valid)
            for x, y in zip(a, c):
                assert torch.equal(x, y), step
    assert losses[-1] < losses[0]
    for k, p in net.named_parameters():
        if k in enc:
            assert torch.equal(p.detach(), enc[k]), k


def test_inference_does_not_refresh_frozen_parameters():
    net = _net(_cfg(256))
    b = _batch(1, 256, 20, 10, 8, seed=2)
    before = net.infer_masks_and_img_features(b["rgb"])[0].clone()
    with torch.no_grad():
        dict(net.named_parameters())["map_decoder.7.bias"].add_(5.0)
    assert torch.equal(net.infer_masks_and_img_features(b["rgb"])[0], before)   # requires_grad False: as before
    net.mark_weights_dirty()
    assert not torch.equal(net.infer_masks_and_img_features(b["rgb"])[0], before)


def test_bad_input_raises_before_launch():
    net = _net(_cfg(256))
    b = _batch(1, 256, 40, 10, 8, seed=1)
    bad = []
    x = dict(b); x["pairs"] = torch.zeros((1, 10, 33, 2), dtype=torch.int64, device=DEV); bad.append(x)
    x = dict(b); x["rgb"] = b["rgb"][:, :128]; bad.append(x)
    x = dict(b); x["valid"] = b["valid"].float(); bad.append(x)
    x = dict(b); x["road_mask"] = b["road_mask"].cpu(); bad.append(x)
    x = dict(b); x["connected"] = b["connected"][:, :5]; bad.append(x)
    x = dict(b); x["pairs"] = b["pairs"].float(); bad.append(x)
    torch.cuda.synchronize()
    from sam_road_b200 import _lib
    n0 = _lib.load().samroad_launch_count(0)
    for x in bad:
        with pytest.raises(ValueError):
            net.training_step(x, 0)
    torch.cuda.synchronize()
    assert _lib.load().samroad_launch_count(0) == n0
