"""GPU: SAMRoad.head_losses / train.head_losses on caller-supplied image embeddings, and the gradient of the
losses with respect to those embeddings (samroad_train_backward_embeddings), against the float64 oracle
(oracle/train_oracle.py) on the same embeddings and dropout keep masks.

The gradient is compared per tile and per block of 32 channels: both ||g - g64||_inf / ||g64||_inf and
||g - g64||_2 / ||g64||_2 must stay within BOUND, and a slice that is exactly 0 in float64 must be exactly 0.
The worst slice of every case is printed and, when EMB_GRAD_REPORT names a file, written there as JSON
(DESIGN.md §12)."""
import json
import os

import pytest
import torch

from oracle import samroad_oracle as O
from oracle import train_oracle as TO
from sam_road_b200 import SAMRoad, synth
from sam_road_b200 import train as T

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 5e-4
OUTLIER_BOUND = 5e-3   # test_gpu_train.py's per-tensor bound against the fp32 oracle
REPORT = {}


def _cfg(P=256, version="normal", focal=False, **kw):
    c = {"SAM_VERSION": "vit_b", "PATCH_SIZE": P, "FREEZE_ENCODER": False, "BASE_LR": 1e-3,
         "TOPONET_VERSION": version, "FOCAL_LOSS": focal}
    c.update(kw)
    return c


def _net(cfg, seed=0, heads_grad=True):
    net = SAMRoad(cfg)
    net.load_state_dict(synth.make_state_dict(cfg, seed=seed, logit_gain=4.0))
    net = net.to(DEV).eval()            # SAMRoad.head_losses without dropout; the tests pass dropout explicitly
    for _, p in net._head_params():
        p.requires_grad_(heads_grad)
    return net


def _batch(B, P, N, Ns, Np, seed, points=None):
    g = torch.Generator().manual_seed(seed)
    pts, pairs, valid = synth.make_topo_inputs(B, P, N, seed=seed, max_nbr=Np)
    pairs, valid = pairs[:, :Ns].contiguous(), valid[:, :Ns].clone()
    valid[0, 0] = False                                   # an all-invalid sample row
    b = {"rgb": synth.make_tiles(B, P, seed=seed), "graph_points": pts if points is None else points,
         "pairs": pairs, "valid": valid, "connected": torch.rand(valid.shape, generator=g) < 0.4,
         "keypoint_mask": torch.randint(0, 256, (B, P, P), generator=g).float() / 255.0,
         "road_mask": (torch.rand((B, P, P), generator=g) < 0.5).float()}
    return {k: v.to(DEV) for k, v in b.items()}


def _emb(B, P, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = P // 16
    return torch.randn((B, 256, s, s), generator=g, device=DEV) * 0.5


def _device(net, b, emb, w=(1.0, 1.0), dropout_p=0.0, seed=0):
    """(losses, d(w0 mask + w1 topo)/d(emb)) through train.head_losses with the embeddings as input."""
    heads = net._head_params()
    bb = T.validate_batch(b, net.image_size, DEV)
    args = T.make_args(bb, net.focal_loss, dropout_p, seed)
    e = emb.detach().clone().requires_grad_(True)
    ml, tl = T.head_losses(net._handle(DEV), bb, args, [k for k, _ in heads], [p for _, p in heads],
                           image_embeddings=e)
    g, = torch.autograd.grad(w[0] * ml + w[1] * tl, e)
    return (ml.detach(), tl.detach()), g


def _keep(b, seed, p=0.1):
    B, Ns, Np = b["valid"].shape
    rows, tok = B * Ns, B * Ns * Np
    keep = {}
    for l in range(3):
        keep[(l, 0)] = T.dropout_keep(p, seed, l, 0, rows * 4 * Np * Np, DEV).view(rows, 4, Np, Np)
        for site in (1, 2, 3):
            keep[(l, site)] = T.dropout_keep(p, seed, l, site, tok * 128, DEV).view(rows, Np, 128)
    return keep


def _oracle(net, b, emb, version, w=(1.0, 1.0), dropout_p=0.0, seed=0):
    params = {k: p.detach().double() for k, p in net._head_params()}
    e = emb.detach().double().requires_grad_(True)
    keep = _keep(b, seed, dropout_p) if dropout_p > 0 else None
    ml, tl = TO.heads_losses(params, e, b, net.image_size, net.focal_loss, version, keep, dropout_p)
    loss = (w[0] * ml if w[0] else 0) + (w[1] * tl if w[1] else 0)
    g, = torch.autograd.grad(loss, e)
    return (ml.detach(), tl.detach()), g


def _compare(name, g, g64, bound=BOUND, outliers=0):
    """Worst (inf, 2-norm) relative error over the (tile, 32-channel block) slices.  The slices of up to
    `outliers` tiles may exceed `bound`, each within OUTLIER_BOUND: at the benched shape a ReLU unit can sit so
    close to zero that fp32 and float64 take opposite sides, and the texels under the point whose features depend
    on it move in every channel (DESIGN.md §12)."""
    assert g.dtype == torch.float32 and g.shape == g64.shape
    worst = [0.0, 0.0, None]
    over = []
    B = g.shape[0]
    for bi in range(B):
        for c0 in range(0, 256, 32):
            a, r = g[bi, c0:c0 + 32].double(), g64[bi, c0:c0 + 32]
            if (r == 0).all():
                assert (a == 0).all(), (name, bi, c0)
                continue
            e_inf = ((a - r).abs().max() / r.abs().max()).item()
            e_2 = ((a - r).norm() / r.norm()).item()
            if e_inf > bound or e_2 > bound:
                assert e_inf <= OUTLIER_BOUND and e_2 <= OUTLIER_BOUND, (name, bi, c0, e_inf, e_2)
                over.append((bi, c0, e_inf, e_2))
                continue
            if max(e_inf, e_2) > max(worst[0], worst[1]):
                worst = [e_inf, e_2, (bi, c0)]
    REPORT[name] = {"inf": worst[0], "l2": worst[1], "slice": worst[2], "slices": B * 8, "outliers": over}
    out = os.environ.get("EMB_GRAD_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump(REPORT, f, indent=1)
    print(f"{name}: worst slice inf {worst[0]:.3e} l2 {worst[1]:.3e} at {worst[2]}; over {bound}: {over}")
    assert len({o[0] for o in over}) <= outliers, (name, over)
    return worst


def _losses_close(got, want):
    for a, c in zip(got, want):
        assert abs(a.item() - c.item()) <= 1e-5 * abs(c.item()), (a.item(), c.item())


# (name, P, B, version, focal, N, Ns, Np, dropout)
CASES = [
    ("vitb256_normal_bce", 256, 2, "normal", False, 40, 20, 16, 0.0),
    ("p400_no_transformer_focal", 400, 2, "no_transformer", True, 40, 25, 16, 0.0),
    ("p256_no_offset", 256, 2, "no_offset", False, 40, 20, 16, 0.0),
    ("bench_b16_p512_dropout", 512, 16, "normal", False, 512, 512, 16, 0.1),
    ("b16_p1024", 1024, 16, "normal", False, 64, 64, 16, 0.0),
    ("all_one", 256, 1, "normal", False, 1, 1, 1, 0.0),
]


@pytest.mark.parametrize("name,P,B,version,focal,N,Ns,Np,p", CASES, ids=[c[0] for c in CASES])
def test_parity_float64(name, P, B, version, focal, N, Ns, Np, p):
    net = _net(_cfg(P, version, focal))
    b = _batch(B, P, N, Ns, Np, seed=P + N)
    if N == 1:
        b["valid"][:] = True
    emb = _emb(B, P, seed=3)
    got = _device(net, b, emb, dropout_p=p, seed=77)
    want = _oracle(net, b, emb, version, dropout_p=p, seed=77)
    _losses_close(got[0], want[0])
    _compare(name, got[1], want[1], outliers=1 if B * N >= 4096 else 0)


def _fractional_points(B, P, N, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand((B, N, 2), generator=g) * P
    k = N // 4
    pts[:, :k] = torch.rand((B, k, 2), generator=g) * 8                      # within 8 px of the top-left border
    pts[:, k:2 * k] = P - torch.rand((B, k, 2), generator=g) * 8             # ... of the bottom-right border
    pts[:, 2 * k:2 * k + k // 2, 0] = torch.rand((B, k // 2), generator=g) * 8
    pts[:, 2 * k + k // 2:3 * k, 1] = P - torch.rand((B, k - k // 2), generator=g) * 8
    cent = torch.randint(0, P // 16, (B, N - 3 * k, 2), generator=g).float() * 16 + 8   # exact texel centres
    pts[:, 3 * k:] = cent
    return pts.float()


@pytest.mark.parametrize("kind", ["float32", "int32"])
def test_parity_point_dtypes(kind):
    P, B, N = 256, 2, 64
    pts = _fractional_points(B, P, N, seed=5)
    if kind == "int32":
        pts = pts.floor().to(torch.int32)
    net = _net(_cfg(P))
    b = _batch(B, P, N, 40, 16, seed=9, points=pts)
    emb = _emb(B, P, seed=4)
    got = _device(net, b, emb)
    want = _oracle(net, b, emb, "normal")
    _compare(f"points_{kind}", got[1], want[1])


def test_ragged_pile_on_texel_zero():
    """Padded points of a ragged batch all sit at (0,0), each read by a padded pair: thousands of sampler taps
    land on texel (0,0) of each tile."""
    P, B, N, Ns, Np = 256, 2, 3240, 200, 16
    b = _batch(B, P, 40, 40, Np, seed=13)
    pts = torch.zeros((B, N, 2), dtype=torch.int64, device=DEV)
    pts[:, :b["graph_points"].shape[1]] = b["graph_points"]
    pairs = torch.zeros((B, Ns, Np, 2), dtype=torch.int64, device=DEV)
    valid = torch.zeros((B, Ns, Np), dtype=torch.bool, device=DEV)
    pairs[:, :40], valid[:, :40] = b["pairs"], b["valid"]
    pad = 40 + torch.arange((Ns - 40) * Np, device=DEV).view(Ns - 40, Np)
    pairs[:, 40:, :, 0] = pad
    pairs[:, 40:, :, 1] = pad                  # padded samples read the padded points
    valid[:, 40:] = True                       # ... and count, so that their taps carry a gradient
    conn = torch.rand(valid.shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV) < 0.4
    b.update(graph_points=pts, pairs=pairs, valid=valid, connected=conn)
    net = _net(_cfg(P))
    emb = _emb(B, P, seed=6)
    got = _device(net, b, emb)
    want = _oracle(net, b, emb, "normal")
    _compare("ragged_pile", got[1], want[1])


def test_no_tgt_features_is_normal_bit_for_bit():
    b = _batch(2, 256, 40, 20, 16, seed=17)
    emb = _emb(2, 256, seed=7)
    a = _device(_net(_cfg(256, "normal")), b, emb, dropout_p=0.1, seed=5)
    c = _device(_net(_cfg(256, "no_tgt_features")), b, emb, dropout_p=0.1, seed=5)
    assert torch.equal(a[1], c[1]) and torch.equal(a[0][0], c[0][0]) and torch.equal(a[0][1], c[0][1])


def test_incoming_gradient_routing_and_scaling():
    net = _net(_cfg(256))
    b = _batch(2, 256, 40, 20, 16, seed=19)
    emb = _emb(2, 256, seed=8)
    for w in ((1.0, 0.0), (0.0, 1.0)):
        got = _device(net, b, emb, w=w)
        want = _oracle(net, b, emb, "normal", w=w)
        _compare(f"incoming_{int(w[0])}{int(w[1])}", got[1], want[1])
    one = _device(net, b, emb)[1]
    big = _device(net, b, emb, w=(1024.0, 1024.0))[1]
    assert torch.equal(one * 1024, big)


def test_bit_identity_with_training_step():
    cfg = _cfg(256, FREEZE_ENCODER=True)
    net = _net(cfg).train()
    b = _batch(2, 256, 40, 20, 16, seed=23)
    heads = net._head_params()
    torch.manual_seed(41)
    net.zero_grad(set_to_none=True)
    loss = net.training_step(b, 0)
    loss.backward()
    want = {k: p.grad.clone() for k, p in heads}
    # the device encoder's own embeddings, as the training step's forward makes them
    bb = T.validate_batch(b, 256, DEV)
    emb = torch.empty((2, 256, 16, 16), device=DEV)
    T.head_losses(net._handle(DEV), bb, T.make_args(bb, False, 0.0, 0), [k for k, _ in heads],
                  [p.detach() for _, p in heads], emb_out=emb)
    assert not emb.requires_grad
    torch.manual_seed(41)
    net.zero_grad(set_to_none=True)
    ml, tl = net.head_losses(b, emb)
    (ml + tl).backward()
    assert torch.equal(ml + tl, loss.detach())
    for k, p in heads:
        assert torch.equal(p.grad, want[k]), k


def test_determinism_and_repeated_backward():
    net = _net(_cfg(512))
    b = _batch(16, 512, 512, 512, 16, seed=29)
    emb = _emb(16, 512, seed=9)
    a = _device(net, b, emb, dropout_p=0.1, seed=3)
    c = _device(net, b, emb, dropout_p=0.1, seed=3)
    assert torch.equal(a[1], c[1])
    heads = net._head_params()
    bb = T.validate_batch(b, 512, DEV)
    e = emb.clone().requires_grad_(True)
    ml, tl = T.head_losses(net._handle(DEV), bb, T.make_args(bb, False, 0.1, 3), [k for k, _ in heads],
                           [p for _, p in heads], image_embeddings=e)
    params = [p for _, p in heads]
    g1 = torch.autograd.grad(ml + tl, [e] + params, retain_graph=True)
    g2 = torch.autograd.grad(ml + tl, [e] + params)
    assert torch.equal(g1[0], a[1])
    for x, y in zip(g1, g2):
        assert torch.equal(x, y)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_embeddings(dtype):
    net = _net(_cfg(256))
    b = _batch(2, 256, 40, 20, 16, seed=31)
    emb = _emb(2, 256, seed=10).to(dtype)
    e = emb.clone().requires_grad_(True)
    ml, tl = net.head_losses(b, e)
    (ml + tl).backward()
    assert e.grad.dtype == dtype
    ref = _device(net, b, emb.float())[1]
    assert torch.equal(e.grad, ref.to(dtype))
    # a channels-last input gets a channels-last gradient
    e2 = emb.float().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    ml, tl = net.head_losses(b, e2)
    (ml + tl).backward()
    assert e2.grad.stride() == e2.stride() and torch.equal(e2.grad, ref)


def test_heads_and_embeddings_only_where_asked():
    net = _net(_cfg(256), heads_grad=False)
    b = _batch(2, 256, 40, 20, 16, seed=37)
    emb = _emb(2, 256, seed=11)
    e = emb.clone().requires_grad_(True)
    ml, tl = net.head_losses(b, e)
    (ml + tl).backward()
    assert all(p.grad is None for _, p in net._head_params())
    assert torch.equal(e.grad, _device(net, b, emb)[1])
    frozen = dict(net._head_params())["topo_net.output_proj.bias"]
    for k, p in net._head_params():
        p.requires_grad_(k != "topo_net.output_proj.bias")
    ml, tl = net.head_losses(b, emb)                 # embeddings without requires_grad
    (ml + tl).backward()
    assert frozen.grad is None
    assert all(p.grad is not None for k, p in net._head_params() if k != "topo_net.output_proj.bias")


def test_no_valid_slot():
    net = _net(_cfg(256))
    b = _batch(2, 256, 40, 20, 16, seed=43)
    b["valid"][:] = False
    emb = _emb(2, 256, seed=12)
    got = _device(net, b, emb)[1]
    want = _oracle(net, b, emb, "normal")[1]
    assert torch.isnan(want).any() and (~torch.isnan(want)).any()
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    fin = ~torch.isnan(want)
    assert torch.isfinite(got[fin]).all()
    gm = _device(net, b, emb, w=(1.0, 0.0))[1]
    assert torch.isfinite(gm).all()


def test_lora_encoder_end_to_end():
    """The oracle encoder with rank-4 LoRA adapters on qkv, held in PyTorch on the GPU, feeds head_losses; the
    adapters' gradients match an all-oracle float64 step."""
    cfg = _cfg(256, ENCODER_LORA=True, LORA_RANK=4)
    sd = synth.make_state_dict(cfg, seed=2, logit_gain=4.0)
    lora = [k for k in sd if "linear_a_" in k or "linear_b_" in k]
    assert lora
    g = torch.Generator().manual_seed(3)
    for k in lora:
        if "linear_b_" in k:                                    # nonzero B, so every adapter has a gradient
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.02
    net = _net(cfg)
    net.load_state_dict(sd)
    for _, p in net._head_params():
        p.requires_grad_(False)
    spec = O.ModelSpec.from_config(cfg)
    b = _batch(2, 256, 40, 20, 16, seed=47)

    def run(dtype):
        w = {k: v.to(DEV, dtype) for k, v in sd.items()}
        for k in lora:
            w[k].requires_grad_(True)
        x = O.normalize_rgb(b["rgb"].to(dtype))
        emb = O.image_encoder(x, w, spec)
        if dtype == torch.float32:
            ml, tl = net.head_losses(b, emb)
        else:
            params = {k: v for k, v in w.items() if k.startswith(("map_decoder.", "topo_net."))}
            ml, tl = TO.heads_losses(params, emb, b, 256, False, "normal", None, 0.0)
        (ml + tl).backward()
        return {k: w[k].grad for k in lora}

    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False     # the encoder's convolutions in fp32, not TF32
    try:
        got, want = run(torch.float32), run(torch.float64)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    worst = 0.0
    for k in lora:
        a, r = got[k].double(), want[k]
        e_inf = ((a - r).abs().max() / r.abs().max()).item()
        e_2 = ((a - r).norm() / r.norm()).item()
        assert e_inf <= BOUND and e_2 <= BOUND, (k, e_inf, e_2)
        worst = max(worst, e_inf, e_2)
    REPORT["lora_adapters"] = {"worst": worst}
    print(f"LoRA adapter gradients: worst relative error {worst:.3e}")


def test_refusals():
    net = _net(_cfg(256))
    b = _batch(2, 256, 40, 20, 16, seed=53)
    emb = _emb(2, 256, seed=13)
    for bad in (emb[:1], emb[:, :128], emb.double(), emb.to(torch.int32), emb.cpu()):
        with pytest.raises(ValueError):
            net.head_losses(b, bad)
    cpu = dict(b)
    cpu["pairs"] = b["pairs"].cpu()
    with pytest.raises(ValueError):
        net.head_losses(cpu, emb)
    with pytest.raises(ValueError):
        net.head_losses({k: v.cpu() for k, v in b.items()}, emb)
    sam = _net(_cfg(256, USE_SAM_DECODER=True))
    with pytest.raises(NotImplementedError, match="USE_SAM_DECODER"):
        sam.head_losses(b, emb)
