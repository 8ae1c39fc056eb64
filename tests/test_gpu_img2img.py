"""Image self-attention (img2img, SURVEY A.4 item 18) on an H100 (``pytest -m gpu``).

* gf_self_attn_fwd / gf_self_attn_bwd, exact cases: queries and keys built so that one key wins every row by more than 160 in log2
  units (every other exp2 underflows to exactly 0) give O equal to that key's V row and, backward, dQ = dK = 0 and dV = P^T dO, bit for
  bit; all-zero queries give P = 1/n exactly, so O is the exact mean of integer V; another head's channels and other images do not
  change a head's bits.
* Against the fp64 oracle (oracle/self_attention.py) at n in {64, 192, 256, 576, 1024, 4096}, d in {32, 64}, B in {1, 3}: O and the three
  gradients under frozen bounds; the backward is deterministic.
* ``ImageSelfAttention`` on the kernels against its torch composite (exact_fp32=True), and the composite against fp64.
* Generator and discriminator with img2img against tests/img2img_ref.py in both precision modes; a small training run with R1, path
  length, style mixing and "bgc" augmentation, eager and CUDA-graphed; with cuDNN pinned, a graphed step and an eager one from one
  state give the same losses and gradients bit for bit.
"""
import copy
import math
from importlib import import_module

import pytest
import torch

from oracle import self_attention as osa
from tests import img2img_ref as iref
from tests import test_gpu_step_determinism as sdet

pytestmark = pytest.mark.gpu

SA = "gansformer-reproducibility-challenge_b200.self_attention"
TRAIN = "gansformer-reproducibility-challenge_b200.training"

# max |err| / max |ref| of O and of dQ, dK, dV against fp64 (inputs N(0, 1), TF32 operands, fp32 accumulation), and max |err| of
# lse (log2 units), over the sweep of test_against_fp64.  Measured worst cases on an NVIDIA H100 80GB HBM3 at a 700 W power limit:
# O 3.75e-3, gradients 4.39e-3, lse 3.19e-3; frozen at about 3x.
FWD_BOUND = 1.2e-2
GRAD_BOUND = 1.4e-2
LSE_BOUND = 1e-2


def _sa():
    return import_module(SA)


def _exact(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    bad = (a != b).sum().item()
    assert bad == 0, f"{what}: {bad} elements differ, max |diff| {(a.double() - b.double()).abs().max().item():.3e}"


def _one_hot_case(B, n, h, d, dev, seed=0):
    """Per head, query i carries 32 in channel c_i = i % d; the key w_c carries 32 in channel c and no other key does: the logit
    1024 / sqrt(d) beats 0 by more than 160 log2 units.  V, dO: integers in [-8, 8]."""
    g = torch.Generator().manual_seed(seed)
    C = h * d
    q = torch.zeros(B, n, C)
    k = torch.zeros(B, n, C)
    win = torch.zeros(B, h, n, dtype=torch.long)
    for b in range(B):
        for j in range(h):
            keys = torch.randperm(n, generator=g)[:d]
            c = torch.randint(0, d, (n,), generator=g)
            q[b, torch.arange(n), j * d + c] = 32.0
            k[b, keys, j * d + torch.arange(d)] = 32.0
            win[b, j] = keys[c]
    v = torch.randint(-8, 9, (B, n, C), generator=g).float()
    do = torch.randint(-8, 9, (B, n, C), generator=g).float()
    return [t.to(dev) for t in (q, k, v, do)] + [win]


@pytest.mark.parametrize("n,d", [(64, 32), (64, 64), (192, 32), (256, 64), (576, 64), (1024, 32)])
def test_one_hot_forward_and_backward_exact(gf, cuda_dev, n, d):
    sa = _sa()
    B, h = 2, 2
    q, k, v, do, win = _one_hot_case(B, n, h, d, cuda_dev)
    o, lse = sa.attention_fwd_native(q, k, v, h)
    want = torch.empty_like(o)
    dv_want = torch.zeros(B, n, h * d, dtype=torch.float64)
    for b in range(B):
        for j in range(h):
            cols = slice(j * d, (j + 1) * d)
            want[b, :, cols] = v[b, win[b, j].to(cuda_dev), cols]
            dv_want[b, :, cols].index_add_(0, win[b, j], do[b, :, cols].double().cpu())
    _exact(o, want, "O = V[winner]")
    dq, dk, dv = sa.attention_bwd_native(q, k, v, o, lse, do, h)
    _exact(dq, torch.zeros_like(dq), "dQ")
    _exact(dk, torch.zeros_like(dk), "dK")
    _exact(dv, dv_want.float().to(cuda_dev), "dV = P^T dO")


@pytest.mark.parametrize("n", [64, 256, 1024, 4096])
def test_uniform_attention_is_the_exact_mean(gf, cuda_dev, n):
    sa = _sa()
    B, h, d = 2, 2, 64
    g = torch.Generator().manual_seed(n)
    v = torch.randint(-8, 9, (B, n, h * d), generator=g).float().to(cuda_dev)
    q = torch.zeros_like(v)
    k = torch.randn(v.shape, generator=g).to(cuda_dev)
    o, lse = sa.attention_fwd_native(q, k, v, h)
    _exact(o, (v.double().sum(dim=1, keepdim=True) / n).float().expand_as(o).contiguous(), "O = mean V")
    _exact(lse, torch.full_like(lse, math.log2(n)), "lse = log2 n")


def test_heads_and_images_are_independent(gf, cuda_dev):
    sa = _sa()
    B, n, h, d = 3, 256, 4, 64
    g = torch.Generator().manual_seed(1)
    q, k, v, do = (torch.randn(B, n, h * d, generator=g).to(cuda_dev) for _ in range(4))
    o, lse = sa.attention_fwd_native(q, k, v, h)
    grads = sa.attention_bwd_native(q, k, v, o, lse, do, h)
    q2, k2, v2, do2 = (t.clone() for t in (q, k, v, do))
    for t in (q2, k2, v2, do2):
        t[:, :, 2 * d:3 * d] = torch.randn(B, n, d, generator=g).to(cuda_dev)       # head 2 only
    o2, lse2 = sa.attention_fwd_native(q2, k2, v2, h)
    grads2 = sa.attention_bwd_native(q2, k2, v2, o2, lse2, do2, h)
    keep = [c for c in range(h * d) if not 2 * d <= c < 3 * d]
    _exact(o2[..., keep], o[..., keep], "other heads' O")
    for a, b_, name in zip(grads2, grads, ("dQ", "dK", "dV")):
        _exact(a[..., keep], b_[..., keep], f"other heads' {name}")
    o1, lse1 = sa.attention_fwd_native(q[1:2].contiguous(), k[1:2].contiguous(), v[1:2].contiguous(), h)
    _exact(o1, o[1:2], "image 1 alone")
    g1 = sa.attention_bwd_native(q[1:2].contiguous(), k[1:2].contiguous(), v[1:2].contiguous(), o1, lse1, do[1:2].contiguous(), h)
    for a, b_, name in zip(g1, grads, ("dQ", "dK", "dV")):
        _exact(a, b_[1:2], f"image 1 alone, {name}")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("d", [32, 64])
@pytest.mark.parametrize("n", [64, 192, 256, 576, 1024, 4096])
def test_against_fp64(gf, cuda_dev, n, d, B):
    sa = _sa()
    h = 2
    g = torch.Generator().manual_seed(n + d + B)
    q, k, v, do = (torch.randn(B, n, h * d, generator=g, dtype=torch.float64).to(cuda_dev) for _ in range(4))
    o, lse = sa.attention_fwd_native(*(t.float() for t in (q, k, v)), h)
    q64, k64, v64 = (t.clone().requires_grad_(True) for t in (q, k, v))
    o64, lse64 = osa.attention(q64, k64, v64, h)
    ref = torch.autograd.grad(o64, [q64, k64, v64], do)
    grads = sa.attention_bwd_native(*(t.float() for t in (q, k, v)), o, lse, do.float(), h)
    rel = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    errs = {"O": rel(o, o64.detach()), "lse": (lse.double() - lse64).abs().max().item()}
    errs.update({name: rel(a, r) for name, a, r in zip(("dQ", "dK", "dV"), grads, ref)})
    print(f"[img2img fp64] n={n} d={d} B={B} " + " ".join(f"{k_}={v_:.2e}" for k_, v_ in errs.items()))
    assert errs["O"] <= FWD_BOUND and errs["lse"] <= LSE_BOUND, errs
    assert max(errs["dQ"], errs["dK"], errs["dV"]) <= GRAD_BOUND, errs


def test_backward_is_deterministic(gf, cuda_dev):
    sa = _sa()
    g = torch.Generator().manual_seed(2)
    q, k, v, do = (torch.randn(2, 1024, 256, generator=g).to(cuda_dev) for _ in range(4))
    o, lse = sa.attention_fwd_native(q, k, v, 4)
    a = sa.attention_bwd_native(q, k, v, o, lse, do, 4)
    b = sa.attention_bwd_native(q, k, v, o, lse, do, 4)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert torch.equal(o, sa.attention_fwd_native(q, k, v, 4)[0])


@pytest.mark.parametrize("C,integration,norm", [(64, "mul", "layer"), (128, "both", None), (32, "add", "layer")])
def test_layer_against_composite_and_fp64(gf, cuda_dev, C, integration, norm):
    torch.manual_seed(0)
    m = gf.ImageSelfAttention(C, 16, integration=integration, norm=norm).to(cuda_dev)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.copy_(torch.randn_like(p) * 0.2)
    me = copy.deepcopy(m)
    me.exact_fp32 = True
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 16, C, generator=g).to(cuda_dev)
    gy = torch.randn(2, 16, 16, C, generator=g).to(cuda_dev)
    outs = []
    for mod in (m, me):
        xs = x.clone().requires_grad_(True)
        y = mod(xs)
        grads = torch.autograd.grad(y, [xs, *mod.parameters()], gy)
        outs.append((y.detach(), grads))
    w64 = {n_: p.detach().double().cpu() for n_, p in m.named_parameters()}
    x64 = x.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
    p64 = {n_: t.requires_grad_(True) for n_, t in w64.items()}
    y64 = osa.self_attention_layer(x64, p64, integration=integration, norm=norm).permute(0, 2, 3, 1)
    g64 = torch.autograd.grad(y64, [x64, *p64.values()], gy.double().cpu())
    g64 = (g64[0].permute(0, 2, 3, 1),) + g64[1:]
    # bk's gradient is zero in exact arithmetic (a key bias shifts every logit of a row by the same amount): it is held against the
    # scale of bq's gradient instead of its own
    names = ["y", "x"] + [n_ for n_, _ in m.named_parameters()]
    scale = {n_: r.abs().max() for n_, r in zip(names, [y64.detach(), *g64])}
    scale["bk"] = scale["bq"]
    rel = lambda a, r, n_: ((a.double().cpu() - r).abs().max() / scale[n_]).item()
    kern = [rel(a, r, n_) for a, r, n_ in zip([outs[0][0], *outs[0][1]], [y64.detach(), *g64], names)]
    comp = [rel(a, r, n_) for a, r, n_ in zip([outs[1][0], *outs[1][1]], [y64.detach(), *g64], names)]
    vs = [rel(a, b_.double().cpu(), n_) for a, b_, n_ in zip([outs[0][0], *outs[0][1]], [outs[1][0], *outs[1][1]], names)]
    print(f"[img2img layer C={C}] kernels vs fp64 max {max(kern):.2e}, composite fp32 vs fp64 max {max(comp):.2e}, "
          f"kernels vs composite max {max(vs):.2e}")
    assert max(vs) <= 3e-2 and max(kern) <= 3e-2
    assert max(comp) <= 1e-4


def _small_g(gf, dev, **kw):
    torch.manual_seed(0)
    return gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2, **kw).to(dev)


@pytest.mark.parametrize("exact", [False, True], ids=["tf32", "fp32"])
def test_generator_and_discriminator_against_reference(gf, cuda_dev, exact):
    tr = import_module(TRAIN)
    G = _small_g(gf, cuda_dev, img2img=16, exact_fp32=exact)
    with torch.no_grad():
        G.synthesis.img2img.bo.normal_(0, 0.2)
    z = torch.randn(4, 5, 16, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        img = G(z.to(cuda_dev))
    ref = iref.generator_forward(iref.cast(G.state_dict()), z.double(), resolution=32, components_num=4, latent_dim=16, img2img=16,
                                 mapping_layers=2)
    rel_g = ((img.double().cpu() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    errs = {"G": rel_g}
    for transformer in (False, True):
        torch.manual_seed(0)
        D = tr.Discriminator(32, fmap_base=1024, fmap_max=128, transformer=transformer, components_num=4, latent_dim=16, img2img=16,
                             exact_fp32=exact).to(cuda_dev)
        x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(2))
        with torch.no_grad():
            lo = D(x.to(cuda_dev))
        lr = iref.discriminator_forward(iref.cast(D.state_dict()), x.double(), img2img=16)
        errs[f"D transformer={transformer}"] = ((lo.double().cpu() - lr).abs().max() / lr.abs().max()).item()
    print(f"[img2img networks exact_fp32={exact}] " + " ".join(f"{k_}={v_:.2e}" for k_, v_ in errs.items()))
    bound = 1e-4 if exact else 2e-2
    assert max(errs.values()) <= bound, errs


def _gan(gf, dev):
    tr = import_module(TRAIN)
    G = _small_g(gf, dev, img2img=16)
    torch.manual_seed(1)
    D = tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=16).to(dev)
    return G, D


def test_training_with_img2img(gf, cuda_dev):
    """R1, path length, style mixing and "bgc" augmentation with img2img in G and D, eagerly and CUDA-graphed: finite losses and
    finite gradients for every parameter.  Then a step without the random terms from one state, graphed and eager, with cuDNN pinned
    to its deterministic algorithms: the same D and G losses and the same gradient of every parameter of G and D, bit for bit.
    (Unpinned, cuDNN may pick a non-deterministic algorithm for D's weight gradients, and the G loss, read through D after its
    update, then differs by round-off between the two runs.)"""
    tr = import_module(TRAIN)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(4, 5, 16, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 32, 32, generator=g) * 2 - 1).to(cuda_dev)
    cfg = dict(d_reg_interval=2, g_reg_interval=2, pl_weight=2.0, style_mixing=0.9, augment="bgc", augment_p=0.5)
    for graphed in (False, True):
        G, D = _gan(gf, cuda_dev)
        trainer = tr.Trainer(G, D, tr.TrainConfig(**cfg))
        stats = [(trainer.step_graphed if graphed else trainer.step)(z, reals) for _ in range(4)]
        assert all(math.isfinite(v) for s in stats for v in (s.loss_d, s.loss_g, s.r1, s.pl_penalty)), stats
        assert stats[0].r1 > 0 and any(s.pl_penalty > 0 for s in stats), stats
        for name, p in list(G.named_parameters()) + list(D.named_parameters()):
            if "img2img" in name or name.startswith("synthesis.layers") or name.startswith("blocks"):
                assert p.grad is not None and torch.isfinite(p.grad).all(), (graphed, name)
    cfg = dict(noise_mode="const", d_reg_interval=2)
    with sdet._deterministic_cudnn():
        G, D = _gan(gf, cuda_dev)
        tg = tr.Trainer(G, D, tr.TrainConfig(**cfg))
        tg.step_graphed(z, reals)
        Ge, De = _gan(gf, cuda_dev)
        te = tr.Trainer(Ge, De, tr.TrainConfig(**cfg))
        Ge.load_state_dict(G.state_dict())
        De.load_state_dict(D.state_dict())
        te.opt_g.load_state_dict(copy.deepcopy(tg.opt_g.state_dict()))
        te.opt_d.load_state_dict(copy.deepcopy(tg.opt_d.state_dict()))
        te.it = tg.it
        sg, se = tg.step_graphed(z, reals), te.step(z, reals)
    print(f"[img2img graphed] loss_d eager {se.loss_d!r} graphed {sg.loss_d!r}; loss_g eager {se.loss_g!r} graphed {sg.loss_g!r}; "
          f"gradients differing: G {sdet.differing_grads(G, Ge)[:6]} D {sdet.differing_grads(D, De)[:6]}")
    assert sg.loss_d == se.loss_d and sg.loss_g == se.loss_g
    sdet.assert_same_grads(tg, te, "img2img graphed against eager")
