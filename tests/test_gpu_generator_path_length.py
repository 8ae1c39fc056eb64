"""The generator differentiated twice (run on an H100: ``pytest -m gpu``): path-length regularisation.

* Every route of an attention layer's backward, run with create_graph=True, against an fp64 double backward through the oracle
  with the same Philox mask: the gradient of the squared norm of (d<out, gout>/dx, /dy, /dparams) with respect to x, y and every
  parameter.  Routes: the simplex kernel route without and with dropout, the duplex kernel route with dropout, the composite
  route (instance norm, two heads).
* A small generator (64^2, K = 8, exact fp32, B = 4): the gradients of the path-length penalty with respect to every parameter
  against the fp64 oracle (tests/generator_path_length_ref.py: mapping_forward, synthesis_forward), with dropout off and on.
* A third derivative through the kernels raises.
* ``Trainer`` with pl_weight = 2, g_reg_interval = 2, eager and graphed; with pl_weight = 0 the step is the default step bit for bit.
"""
import copy
import math
from importlib import import_module

import pytest
import torch

from oracle import bipartite as ob
from oracle import philox as ph
from tests import generator_path_length_ref as gref

pytestmark = pytest.mark.gpu

ATT = "gansformer-reproducibility-challenge_b200.attention"

# name, BipartiteAttention options, att_dp, (C, H, W, k), kernel route
ROUTES = [
    ("simplex", dict(integration="mul", norm="layer"), 0.0, (64, 8, 16, 8), True),
    ("simplex-dropout", dict(integration="both", norm="layer"), 0.25, (64, 10, 13, 20), True),
    ("simplex-dropout-add-none", dict(integration="add", norm=None), 0.5, (96, 8, 8, 4), True),
    ("simplex-dropout-mul", dict(integration="mul", norm="layer"), 0.12, (128, 8, 8, 8), True),
    ("duplex-dropout", dict(integration="mul", norm="layer", kmeans=True), 0.25, (64, 8, 16, 8), True),
    ("duplex-dropout-img2ltnt", dict(integration="mul", norm="layer", kmeans=True, img2ltnt=True), 0.12, (64, 10, 13, 20), True),
    ("composite-instance", dict(integration="mul", norm="instance"), 0.0, (64, 8, 8, 8), False),
    ("composite-heads", dict(integration="mul", norm="layer", num_heads=2), 0.0, (64, 8, 8, 8), False),
]
TOL_PL = 3e-5            # the same for the path-length penalty's gradient of each generator parameter (worst measured 1.5e-5)
TOL_ROUTE = 1e-5          # relative norm error of each second-order gradient, fp32 layer (exact_fp32) against fp64 (worst
                          # measured 1.6e-6 on an H100 80GB HBM3)


def _rel(a, b):
    return ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-300)).item()


def _grad_norm_grads(out_fn, leaves, gout):
    """d/d(leaves) of sum_i |d<out, gout>/d leaf_i|^2 (the unused leaves get None)."""
    out = out_fn()
    g1 = torch.autograd.grad((out * gout).sum(), leaves, create_graph=True, allow_unused=True)
    l2 = sum(g.square().sum() for g in g1 if g is not None)
    return torch.autograd.grad(l2, leaves, allow_unused=True)


@pytest.mark.parametrize("name,opts,att_dp,shape,kernel", ROUTES, ids=[r[0] for r in ROUTES])
def test_layer_double_backward_against_fp64(gf, cuda_dev, name, opts, att_dp, shape, kernel):
    am = import_module(ATT)
    C, H, W, k = shape
    B, D = 2, 16
    duplex, img2ltnt = opts.get("kmeans", False), opts.get("img2ltnt", False)
    integration, norm, heads = opts["integration"], opts["norm"], opts.get("num_heads", 1)
    g = torch.Generator().manual_seed(C + H + k)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    gout = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    attn = gf.BipartiteAttention(C, D, k, pos_dim=D, att_dp=att_dp, exact_fp32=True, **opts).to(cuda_dev).train()
    names = [n for n, _ in attn.named_parameters()]
    w0 = ob.init_params(C, D, k, D, integration, duplex, seed=4, bias_std=0.3, extras=img2ltnt)
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w0[n].float())
    mult = None
    if att_dp:
        seed, step = 55555 + C, 9
        am.set_dropout_seed(seed, cuda_dev, step)
        KP = 16 if k <= 16 else 32
        mult = torch.from_numpy(ph.dropout_mult(att_dp, seed, step, attn.dp_salt, B * H * W, KP).reshape(B, H * W, KP)[:, :, :k].copy())

    w = {n: w0[n].clone().requires_grad_(True) for n in names}
    xr, yr = x64.clone().requires_grad_(True), y64.clone().requires_grad_(True)
    leaves = [xr, yr] + [w[n] for n in names]
    ref = _grad_norm_grads(lambda: ob.transformer_layer(xr, yr, w, integration=integration, norm=norm, duplex=duplex, num_heads=heads,
                                                        img2ltnt=img2ltnt, att_mult=mult)[0], leaves, gout)

    xg = x64.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev).requires_grad_(True)
    yg = y64.float().to(cuda_dev).requires_grad_(True)
    prm = dict(attn.named_parameters())
    gl = [xg, yg] + [prm[n] for n in names]
    out = attn(xg, yg)[0]
    g1 = torch.autograd.grad((out * gout.permute(0, 2, 3, 1).float().to(cuda_dev)).sum(), gl, create_graph=True, allow_unused=True)
    l2 = sum(t.square().sum() for t in g1 if t is not None)
    torch.cuda.synchronize()
    launches = gf._lib.launch_count()
    got = torch.autograd.grad(l2, gl, allow_unused=True)
    torch.cuda.synchronize()
    assert (gf._lib.launch_count() > launches) == kernel                 # the double-backward kernels ran (kernel routes only)

    errs = {}
    scale = max(r.abs().max().item() for r in ref if r is not None)
    for nm, r, t in zip(["x", "y"] + names, ref, got):
        if r is None or r.abs().max().item() < 1e-9 * scale:             # unused, or constant over what a softmax normalises
            assert t is None or t.abs().max().item() < 1e-4 * scale, nm
            continue
        errs[nm] = _rel(t if nm != "x" else t.permute(0, 3, 1, 2), r)
    worst = max(errs, key=errs.get)
    print(f"[double backward {name}] worst {worst} {errs[worst]:.2e}  " + " ".join(f"{a}={b:.1e}" for a, b in errs.items()))
    assert {"x", "y", "wq", "wk" if not duplex else "wkc", "wv", "wo"} <= set(errs)
    assert errs[worst] <= TOL_ROUTE, worst


def test_third_derivative_raises(gf, cuda_dev):
    attn = gf.BipartiteAttention(64, 16, 8, pos_dim=16, exact_fp32=True).to(cuda_dev)
    x = torch.randn(2, 8, 8, 64, device=cuda_dev, requires_grad=True)
    y = torch.randn(2, 8, 16, device=cuda_dev)
    (g,) = torch.autograd.grad(attn(x, y)[0].square().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError, match="third derivative"):
        torch.autograd.grad(g.square().sum(), x, create_graph=True)
    (gg,) = torch.autograd.grad(g.square().sum(), x)                    # the second derivative itself is fine
    assert torch.isfinite(gg).all()


def _small_generator(gf, dev, att_dp, seed=0):
    torch.manual_seed(seed)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     exact_fp32=True, att_dp=att_dp).to(dev)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():                  # every term live: biases, noise strengths and attention biases away from zero
        for n, p in G.named_parameters():
            if n.endswith("noise_strength") or n.split(".")[-1].startswith("b"):
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
    return G


def _pl(img, ws, noise, mean):
    (pg,) = torch.autograd.grad((img * noise).sum(), ws, create_graph=True)
    lengths = pg.square().sum(dim=2).mean(dim=1).sqrt()
    return (lengths - mean).square().mean(), lengths


@pytest.mark.parametrize("att_dp", [0.0, 0.12])
def test_path_length_gradients_against_fp64(gf, cuda_dev, att_dp):
    am = import_module(ATT)
    G = _small_generator(gf, cuda_dev, att_dp).train()
    B = 4
    g = torch.Generator().manual_seed(3)
    z = torch.randn(B, 9, 32, generator=g, dtype=torch.float64)
    noise = torch.randn(B, 3, 64, 64, generator=g, dtype=torch.float64) / 64.0
    seed, step = 7, 3
    am.set_dropout_seed(seed, cuda_dev, step)
    params = dict(G.named_parameters())
    ws = G.mapping(z.float().to(cuda_dev))
    img, feats = G.synthesis(ws, noise_mode="const", return_features=True)
    # The leaky ReLUs make the penalty's gradients discontinuous at their kinks, and among the ~10^6 pre-activations of the
    # attention layers some lie within fp32 round-off of zero (min |x| / max |x| down to 1e-9).  fp32 and fp64 then take different
    # slopes there, and even the first-order gradient of the lengths moves from 2e-6 to 3e-4 off fp64 from one run to the next (the
    # fp32 round-off is not the same in every run).  The reference takes the slopes the GPU forward took (the sign of each layer's
    # output, which is also what the backward of the fused bias + activation reads); the 4x4 layer's pre-activations stay above
    # 3e-5 of their maximum.
    signs = [f.detach().cpu() > 0 for f in feats]
    _, lengths = _pl(img, ws, noise.float().to(cuda_dev), 0.0)
    mean = 0.8 * lengths.detach().mean().item()
    pen, _ = _pl(img, ws, noise.float().to(cuda_dev), mean)
    got = torch.autograd.grad(pen, list(params.values()), allow_unused=True)

    sd = {n: t.detach().cpu().double() for n, t in G.state_dict().items()}
    for n in params:
        if n.endswith("noise_strength"):  # one leaf per pixel and image: its gradient is the sum of the per-pixel terms, and the sum of
            hw = G.get_buffer(n.replace("noise_strength", "noise_const")).shape     # their absolute values is its magnitude companion
            sd[n] = sd[n].expand(B, 1, *hw).clone()
        sd[n].requires_grad_(True)
    mults = None
    if att_dp:
        mults = []
        for layer in G.synthesis.layers:
            if layer.attention is not None:
                n_ = layer.resolution ** 2
                mults.append(torch.from_numpy(ph.dropout_mult(att_dp, seed, step, layer.attention.dp_salt, B * n_, 16)
                                              .reshape(B, n_, 16)[:, :, :8].copy()))
    with torch.enable_grad():
        ws64 = gref.mapping_forward(sd, z, components_num=8, latent_dim=32, mapping_layers=4)
        img64 = gref.synthesis_forward(sd, ws64, resolution=64, components_num=8, noise_mode="const", att_mults=mults,
                                      lrelu_pos=signs)
        pen64, len64 = _pl(img64, ws64, noise, mean)
        ref = torch.autograd.grad(pen64, [sd[n] for n in params], allow_unused=True)
    print(f"[path length att_dp={att_dp}] lengths {_rel(lengths, len64):.2e}")
    assert _rel(lengths, len64) < 1e-4
    errs = {}
    scale = max(r.norm().item() for r in ref if r is not None)
    for n, r, t in zip(params, ref, got):
        if n.endswith("noise_strength"):  # a sum over the pixels that cancels: relative to the sum of its terms' magnitudes
            errs[n] = (abs(t.item() - r.sum().item()) / r.abs().sum().item())
            continue
        if r is None:                      # the tRGB biases: an image offset does not change the gradient with respect to ws
            assert t is None or torch.count_nonzero(t) == 0, n
            continue
        if r.norm().item() < 1e-9 * scale:     # the attention key biases: constant over what the softmax normalises
            assert t.norm().item() < 1e-5 * scale, n
            continue
        errs[n] = _rel(t, r)
    assert len(errs) >= len(params) - len(G.synthesis.torgbs) - G.synthesis.num_attention_layers
    worst = sorted(errs, key=errs.get, reverse=True)
    print(f"[path length att_dp={att_dp}] {len(errs)} parameters, median {errs[worst[len(errs) // 2]]:.2e}, worst "
          + " ".join(f"{n}={errs[n]:.1e}" for n in worst[:12]))
    worst = worst[0]
    assert errs[worst] < TOL_PL, worst


def _pair(gf, dev):
    tr = import_module("gansformer-reproducibility-challenge_b200.training")
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     att_dp=0.12).to(dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128).to(dev)
    return tr, G, D


def _data(dev):
    g = torch.Generator().manual_seed(5)
    return torch.randn(4, 9, 32, generator=g).to(dev), (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(dev)


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphed"])
def test_trainer_path_length(gf, cuda_dev, graphed):
    am = import_module(ATT)
    tr, G, D = _pair(gf, cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(pl_weight=2.0, g_reg_interval=2, d_reg_interval=2))
    z, reals = _data(cuda_dev)
    am.set_dropout_seed(7, cuda_dev)
    w0 = G.synthesis.layers[3].attention.wq.detach().clone()
    stats = [(trainer.step_graphed if graphed else trainer.step)(z, reals) for _ in range(6)]
    for i, s in enumerate(stats):
        assert math.isfinite(s.loss_g) and math.isfinite(s.loss_d) and math.isfinite(s.pl_penalty), (i, s)
        assert (s.pl_penalty > 0) == (i % 2 == 0), (i, s.pl_penalty)
    means = [s.pl_mean for s in stats]
    assert 0 < means[0] and means[0] == means[1] < means[2] == means[3] < means[4]   # moves towards the lengths on PL steps only
    assert (G.synthesis.layers[3].attention.wq - w0).abs().max() > 0
    if graphed:
        assert set(k for k in trainer._graphs if isinstance(k, tuple)) == {(True, True), (False, False)}


def test_pl_weight_zero_is_the_default_step(gf, cuda_dev):
    """pl_weight = 0 with the other path-length options changed: the same step as a default Trainer, bit for bit."""
    am = import_module(ATT)
    tr, G, D = _pair(gf, cuda_dev)
    G2, D2 = copy.deepcopy(G), copy.deepcopy(D)
    z, reals = _data(cuda_dev)
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        runs = []
        for g_, d_, cfg in ((G, D, tr.TrainConfig(d_reg_interval=2)),
                            (G2, D2, tr.TrainConfig(d_reg_interval=2, pl_weight=0.0, g_reg_interval=1, pl_batch_shrink=4, pl_decay=0.5))):
            t = tr.Trainer(g_, d_, cfg)
            am.set_dropout_seed(11, cuda_dev)
            torch.manual_seed(1)
            st = [t.step(z, reals) for _ in range(3)]
            runs.append((st, [p.detach().clone() for p in list(g_.parameters()) + list(d_.parameters())]))
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev
    (sa, pa), (sb, pb) = runs
    assert [(s.loss_g, s.loss_d, s.r1, s.pl_penalty, s.pl_mean) for s in sa] == [(s.loss_g, s.loss_d, s.r1, s.pl_penalty, s.pl_mean) for s in sb]
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
