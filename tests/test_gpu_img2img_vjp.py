"""The image self-attention double backward on an H100 (``pytest -m gpu``; DESIGN 4.14).

* gf_self_attn_bwd_vjp through the C ABI against the fp64 restatement (oracle/self_attention_vjp.py) on N(0, 1) inputs and
  cotangents, every output (gQ, gK, gV, gdO and the row statistics) between NaN guards and written everywhere.
* One winning key per row with integer payloads (d = 64, so the scale 1/8 is exact and every sum is an exact fp32 value):
  gQ = gK = gV = 0 and gdO = Cv of the winner, bit for bit.
* Bits: two calls, image and head independence, CUDA-graph replay.
* The layer with ``kernel_double_backward`` against the composite route, the refused third derivative, Discriminator(r1_kernels)
  against its default route, and the training step graphed against eager with both options.
* The generator's path-length gradients against fp64 on the default route, on the default route with its recompute in TF32, and
  with pl_kernels.
* The peak memory of the discriminator layer's R1 gradient at 64^2, C = 512, batch 32 on the kernel route.
"""
import contextlib
import copy
import math
from importlib import import_module

import pytest
import torch

from oracle import self_attention_vjp as ov
from tests import generator_path_length_ref as gref
from tests import test_gpu_step_determinism as sdet
from tests.guards import Guarded, assert_exact
from tests.test_gpu_ops_exact import _call, _stream

pytestmark = pytest.mark.gpu

SA = "gansformer-reproducibility-challenge_b200.self_attention"
TRAIN = "gansformer-reproducibility-challenge_b200.training"

# max error over max |reference| per output, worst over test_against_fp64 (n = 4096), measured on an NVIDIA H100 80GB HBM3 at a
# 700 W power limit: gQ 5.41e-3, gK 5.52e-3, gV 3.54e-3, gdO 4.38e-3; frozen at about 3x (DESIGN 4.14).  They are TF32 operand
# truncation: the kernels' fp32 intermediates enter eight of the twelve products as TF32.
FP64_BOUNDS = {"gQ": 1.6e-2, "gK": 1.7e-2, "gV": 1.1e-2, "gdO": 1.3e-2}
# relative Frobenius error of every second-order gradient, kernel route (TF32 kernels) against the composite route (whose
# recompute of the n x n part runs in fp32 here: conftest turns TF32 matmuls off, and only the layer's forward forces them on):
# worst measured 3.6e-3 (same card), frozen at about 3x
ROUTE_BOUND = 1e-2
# the path-length gradients of the whole generator against fp64 (test_path_length_routes_against_fp64), worst relative error over
# pg, the penalty and every parameter, per route, same card: default 1.6e-2 (median 7.5e-3), default with its recompute in TF32
# 1.9e-2 (7.9e-3), pl_kernels 2.6e-2 (9.3e-3); frozen at about 3x.  Most of it is the rest of the generator's TF32 arithmetic,
# which every route shares; the kernel route is no farther from fp64 than TF32 in the n x n part accounts for (DESIGN 4.14).
PL_FP64_BOUNDS = {"default": 5e-2, "default_tf32": 6e-2, "kernels": 8e-2}
# a key bias (bk) shifts every logit of a query by the same amount, so softmax makes its true gradient exactly 0: both routes
# return round-off there


def _inputs(B, n, C, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, n, C, generator=g).to(dev) for _ in range(7)]


def run(gf, q, k, v, do, a, bk, cv, heads, dev, stream=None):
    """forward, first-order backward (for lse and Delta), then gf_self_attn_bwd_vjp into guarded outputs; -> dict of outputs."""
    sa = import_module(SA)
    q, k, v, do = (t.float().contiguous() for t in (q, k, v, do))
    o, lse = sa.attention_fwd_native(q, k, v, heads)
    *_, delta = sa._attention_bwd(q, k, v, o, lse, do, heads)
    return call_vjp(gf, q, k, v, do, lse, delta, a, bk, cv, heads, dev, stream)


def call_vjp(gf, q, k, v, do, lse, delta, a, bk, cv, heads, dev, stream=None):
    """gf_self_attn_bwd_vjp alone, given lse and Delta, into guarded outputs (checked, every element written); -> dict of outputs
    gQ, gK, gV, gdO, r, t."""
    B, n, C = q.shape
    d = C // heads
    q, k, v, do, a, bk, cv = (t.float().contiguous() for t in (q, k, v, do, a, bk, cv))
    qt, kt, vt, dot, at, bkt, cvt = (t.transpose(1, 2).contiguous() for t in (q, k, v, do, a, bk, cv))
    out = {"gQ": Guarded((B, n, C), dev), "gK": Guarded((B, n, C), dev), "gV": Guarded((B, n, C), dev), "gdO": Guarded((B, n, C), dev),
           "r": Guarded((B, heads, n), dev), "t": Guarded((B, heads, n), dev)}
    _call(gf, "gf_self_attn_bwd_vjp", q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), vt.data_ptr(),
          do.data_ptr(), dot.data_ptr(), lse.data_ptr(), delta.data_ptr(), a.data_ptr(), at.data_ptr(), bk.data_ptr(), bkt.data_ptr(),
          cv.data_ptr(), cvt.data_ptr(), out["r"].ptr(), out["t"].ptr(), out["gQ"].ptr(), out["gK"].ptr(), out["gV"].ptr(),
          out["gdO"].ptr(), B, n, C, d, 1.0 / math.sqrt(d), _stream(dev) if stream is None else stream)
    return {name: gd.check(name).clone() for name, gd in out.items()}


@pytest.mark.parametrize("B,n,C,d", [(1, 64, 64, 64), (3, 192, 128, 32), (2, 256, 512, 64), (1, 1024, 64, 64), (1, 4096, 128, 32)])
def test_against_fp64(gf, cuda_dev, B, n, C, d):
    h = C // d
    ins = _inputs(B, n, C, B + n + C + d, cuda_dev)
    got = run(gf, *ins, h, cuda_dev)
    want = ov.vjp(*(t.double() for t in ins), h)
    errs = {name: ((got[name].double() - w).abs().max() / w.abs().max()).item() for name, w in zip(("gQ", "gK", "gV", "gdO"), want)}
    print(f"[img2img vjp fp64] B={B} n={n} C={C} d={d} " + " ".join(f"{k_}={v_:.3e}" for k_, v_ in errs.items()))
    assert all(errs[x] <= FP64_BOUNDS[x] for x in errs), errs


def _one_winner_case(B, n, C, seed):
    """d = 64.  Per head, key selector channels [0, 32): 32 keys spread over the key tiles each carry 32 in one of them; every query
    carries 32 in the selector of one of those keys, so its logits are 1024 for that key and 0 for every other.  Query payloads in
    channels [32, 48), key payloads in [48, 64) (they never meet), V, dO, A, Bk, Cv integers in [-2, 2]."""
    d, h = 64, C // 64
    g = torch.Generator().manual_seed(seed)
    ri = lambda: torch.randint(-2, 3, (B, n, C), generator=g).float()
    q, k = torch.zeros(B, n, C), torch.zeros(B, n, C)
    win = torch.zeros(B, h, n, dtype=torch.long)
    for b in range(B):
        for j in range(h):
            off = j * d
            keys = torch.randperm(n, generator=g)[:32]
            k[b, keys, off + torch.arange(32)] = 32.0
            ch = torch.randint(0, 32, (n,), generator=g)
            q[b, torch.arange(n), off + ch] = 32.0
            win[b, j] = keys[ch]
            q[b, :, off + 32:off + 48] = torch.randint(-2, 3, (n, 16), generator=g).float()
            k[b, :, off + 48:off + 64] = torch.randint(-2, 3, (n, 16), generator=g).float()
    v, do, a, bk, cv = ri(), ri(), ri(), ri(), ri()
    gdo = torch.zeros(B, n, C)
    for b in range(B):
        for j in range(h):
            cols = slice(j * d, (j + 1) * d)
            gdo[b, :, cols] = cv[b, win[b, j], cols]
    return (q, k, v, do, a, bk, cv), gdo


@pytest.mark.parametrize("B,n,C", [(1, 64, 64), (3, 192, 128), (2, 256, 512), (1, 4096, 64)])
def test_one_winner_exact(gf, cuda_dev, B, n, C):
    ins, gdo = _one_winner_case(B, n, C, seed=n + C + B)
    got = run(gf, *(t.to(cuda_dev) for t in ins), C // 64, cuda_dev)
    zero = torch.zeros(B, n, C, device=cuda_dev)
    for name in ("gQ", "gK", "gV"):
        assert_exact(got[name], zero, f"{name} (B={B} n={n} C={C})")
    assert_exact(got["gdO"], gdo.to(cuda_dev), f"gdO (B={B} n={n} C={C})")


def test_bits(gf, cuda_dev):
    """Two calls agree bit for bit; image 1 alone and head 1 alone give the bits of the full call; a CUDA-graph replay equals the
    eager call."""
    B, n, C, h = 2, 256, 128, 2
    ins = _inputs(B, n, C, 11, cuda_dev)
    first, second = run(gf, *ins, h, cuda_dev), run(gf, *ins, h, cuda_dev)
    for name in first:
        assert torch.equal(first[name], second[name]), name
    alone = run(gf, *(t[1:2] for t in ins), h, cuda_dev)
    for name in ("gQ", "gK", "gV", "gdO"):
        assert torch.equal(alone[name], first[name][1:2]), name
    head = run(gf, *(t[:, :, 64:] for t in ins), 1, cuda_dev)
    for name in ("gQ", "gK", "gV", "gdO"):
        assert torch.equal(head[name], first[name][:, :, 64:]), name

    sa = import_module(SA)
    q, k, v, do, a, bk, cv = ins
    o, lse = sa.attention_fwd_native(q, k, v, h)
    *_, delta = sa._attention_bwd(q, k, v, o, lse, do, h)
    eager = sa.attention_bwd_vjp_native(q, k, v, do, lse, delta, a, bk, cv, h)
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(side):
        sa.attention_bwd_vjp_native(q, k, v, do, lse, delta, a, bk, cv, h)      # warm-up outside the capture
    torch.cuda.current_stream(cuda_dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = sa.attention_bwd_vjp_native(q, k, v, do, lse, delta, a, bk, cv, h)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(captured, eager):
        assert torch.equal(x, y)


def _r1_grads(m, x, keys):
    """R1-style: |d sum(m(x) w) / dx|^2, then its gradients with respect to x and every parameter."""
    xs = x.detach().requires_grad_(True)
    w = torch.randn(x.shape, generator=torch.Generator(device=x.device).manual_seed(3), device=x.device)
    (gx,) = torch.autograd.grad((m(xs) * w).sum(), xs, create_graph=True)
    pen = gx.square().sum()
    params = [p for _, p in m.named_parameters()]
    return dict(zip(keys, torch.autograd.grad(pen, [xs, *params]))), pen


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("C,res", [(64, 16), (128, 16), (512, 8), (32, 8)])
def test_layer_against_composite(gf, cuda_dev, C, res):
    torch.manual_seed(C)
    m = gf.ImageSelfAttention(C, 16, integration="both").to(cuda_dev)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.startswith("b"):
                p.normal_(0, 0.3)
    x = torch.randn(2, res, res, C, device=cuda_dev)
    keys = ["x"] + [n_ for n_, _ in m.named_parameters()]
    ref, _ = _r1_grads(m, x, keys)
    m.kernel_double_backward = True
    got, pen = _r1_grads(m, x, keys)
    errs = {k_: _rel(got[k_], ref[k_]) for k_ in keys if k_ != "bk"}
    print(f"[img2img vjp layer] C={C} {res}^2 " + " ".join(f"{k_}={v_:.2e}" for k_, v_ in errs.items()))
    assert max(errs.values()) <= ROUTE_BOUND, errs
    # a third derivative is refused: the second backward may not itself build a graph
    xs = x.detach().requires_grad_(True)
    (gx,) = torch.autograd.grad(m(xs).square().sum(), xs, create_graph=True)
    with pytest.raises(RuntimeError, match="third derivative"):
        torch.autograd.grad(gx.square().sum(), xs, create_graph=True)


def test_networks_against_default_routes(gf, cuda_dev):
    tr = import_module(TRAIN)
    x = torch.randn(4, 3, 32, 32, device=cuda_dev)
    grads = []
    for r1k in (False, True):
        torch.manual_seed(1)
        D = tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=16, r1_kernels=r1k).to(cuda_dev)
        xs = x.clone().requires_grad_(True)
        (gx,) = torch.autograd.grad(D(xs).sum(), xs, create_graph=True)
        pen = gx.square().sum()
        grads.append(dict(zip(["x"] + [n_ for n_, _ in D.named_parameters()],
                              torch.autograd.grad(pen, [xs, *D.parameters()], allow_unused=True))))
    errs = {k_: _rel(grads[1][k_], grads[0][k_]) for k_ in grads[0]
            if grads[0][k_] is not None and grads[0][k_].norm() > 0 and not k_.endswith("img2img.bk")}
    print(f"[img2img vjp D R1] worst {max(errs, key=errs.get)} {max(errs.values()):.2e}")
    assert max(errs.values()) <= ROUTE_BOUND, errs



class _Tf32Composite(torch.autograd.Function):
    """attention_composite with its forward and its first and second derivatives all in TF32 (the default route's recompute
    otherwise runs in whatever precision torch.backends.cuda.matmul.allow_tf32 holds: fp32 under this suite)."""

    @staticmethod
    def forward(ctx, q, k, v, heads, orig):
        ctx.heads, ctx.orig = heads, orig
        ctx.save_for_backward(q, k, v)
        with import_module(SA)._tf32_matmul():
            return orig(q, k, v, heads)

    @staticmethod
    def backward(ctx, g):
        q, k, v = ctx.saved_tensors
        return (*_Tf32CompositeGrad.apply(q, k, v, g, ctx.heads, ctx.orig), None, None)


class _Tf32CompositeGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, g, heads, orig):
        ctx.heads, ctx.orig = heads, orig
        ctx.save_for_backward(q, k, v, g)
        with torch.enable_grad(), import_module(SA)._tf32_matmul():
            leaves = [t.detach().requires_grad_(True) for t in (q, k, v)]
            return torch.autograd.grad(orig(*leaves, heads), leaves, g)

    @staticmethod
    def backward(ctx, *gg):
        saved = ctx.saved_tensors
        with torch.enable_grad(), import_module(SA)._tf32_matmul():
            q, k, v, g = [t.detach().requires_grad_(True) for t in saved]
            grads = torch.autograd.grad(ctx.orig(q, k, v, ctx.heads), [q, k, v], g, create_graph=True)
            outs = [(x, y) for x, y in zip(grads, gg) if y is not None]
            res = torch.autograd.grad([x for x, _ in outs], [q, k, v, g], [y for _, y in outs], allow_unused=True)
        return (*res, None, None)


@contextlib.contextmanager
def _recompute_in_tf32():
    """Test-local: the default route's recompute of the n x n part (``attention_composite``, differentiated twice) in TF32."""
    sa = import_module(SA)
    orig = sa.attention_composite
    sa.attention_composite = lambda q, k, v, heads: _Tf32Composite.apply(q, k, v, heads, orig)
    try:
        yield
    finally:
        sa.attention_composite = orig


def test_path_length_routes_against_fp64(gf, cuda_dev):
    """The generator's path-length gradients (resolution 32, img2img = 16, B = 4) on three routes against fp64
    (tests/generator_path_length_ref.py with the img2img layer, the leaky-ReLU branches pinned to those the GPU forward took):
    the default route (the layer's backward recomputed through the composite, fp32 under this suite), the same with that
    recompute in TF32, and pl_kernels (TF32 kernels).  pg, the penalty and every parameter's gradient, each under its route's
    bound."""
    z = torch.randn(4, 5, 16, generator=torch.Generator().manual_seed(2))
    res = {}
    for route in ("default", "default_tf32", "kernels"):
        torch.manual_seed(0)
        G = gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2, img2img=16,
                         pl_kernels=route == "kernels").to(cuda_dev)
        params = dict((n_, p) for n_, p in G.named_parameters() if p.requires_grad)
        ws = G.mapping(z.to(cuda_dev))
        img, feats = G.synthesis(ws, noise_mode="const", return_features=True)
        noise = torch.randn(img.shape, generator=torch.Generator(device=cuda_dev).manual_seed(5), device=cuda_dev) / 32.0
        with (_recompute_in_tf32() if route == "default_tf32" else contextlib.nullcontext()):
            (pg,) = torch.autograd.grad((img * noise).sum(), ws, create_graph=True)
            pen = pg.square().sum(dim=-1).mean(dim=1).sqrt().square().mean()
            grads = torch.autograd.grad(pen, list(params.values()), allow_unused=True)
        res[route] = (pg.detach().cpu().double(), pen.item(), dict(zip(params, grads)))
        if route == "default":
            signs = [f.detach().cpu() > 0 for f in feats]
            sd = {n_: t.detach().cpu().double() for n_, t in G.state_dict().items()}
            noise64 = noise.cpu().double()
            for n_ in params:
                if n_.endswith("noise_strength"):
                    hw = G.get_buffer(n_.replace("noise_strength", "noise_const")).shape
                    sd[n_] = sd[n_].expand(4, 1, *hw).clone()
                sd[n_].requires_grad_(True)
    with torch.enable_grad():
        ws64 = gref.mapping_forward(sd, z.double(), components_num=4, latent_dim=16, mapping_layers=2)
        img64 = gref.synthesis_forward(sd, ws64, resolution=32, components_num=4, noise_mode="const", lrelu_pos=signs, img2img=16)
        (pg64,) = torch.autograd.grad((img64 * noise64).sum(), ws64, create_graph=True)
        pen64 = pg64.square().sum(dim=-1).mean(dim=1).sqrt().square().mean()
        ref = dict(zip(params, torch.autograd.grad(pen64, [sd[n_] for n_ in params], allow_unused=True)))
    scale = max(r.norm().item() for r in ref.values() if r is not None)
    errs = {}
    for route, (pg, pen, grads) in res.items():
        e = {"pg": _rel(pg, pg64.detach()), "pen": abs(pen - pen64.item()) / abs(pen64.item())}
        for n_, r in ref.items():
            t = grads[n_]
            if n_.endswith("noise_strength"):       # a sum over pixels that cancels: relative to the sum of its terms' magnitudes
                e[n_] = abs(t.item() - r.sum().item()) / r.abs().sum().item()
            elif r is None:                         # the tRGB biases: an image offset does not change pg
                assert t is None or torch.count_nonzero(t) == 0, n_
            elif r.norm().item() < 1e-9 * scale:    # key biases (bk): constant over what the softmax normalises, true gradient
                continue                            # 0, every route returns round-off
            else:
                e[n_] = _rel(t.cpu(), r)
        errs[route] = e
        worst = sorted(e, key=e.get, reverse=True)
        print(f"[img2img vjp G PL fp64] {route}: pg {e['pg']:.2e} pen {e['pen']:.2e} median {e[worst[len(e) // 2]]:.2e} worst "
              + " ".join(f"{n_}={e[n_]:.1e}" for n_ in worst[:8]))
    assert any(n_.startswith("synthesis.img2img") for n_ in errs["kernels"])
    for route, e in errs.items():
        assert max(e.values()) <= PL_FP64_BOUNDS[route], (route, e)


def _gan(gf, dev):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2, img2img=16,
                     pl_kernels=True).to(dev)
    torch.manual_seed(1)
    D = tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=16, r1_kernels=True).to(dev)
    return G, D


def test_training_graphed_matches_eager(gf, cuda_dev):
    """As test_training_with_img2img, with r1_kernels and pl_kernels set and the R1 term on every step (so that it is in the
    compared step): from one state, graphed and eager, with cuDNN pinned to its deterministic algorithms, the same D and G losses,
    the same R1 value and the same gradient of every parameter, bit for bit.  (The path-length term draws its noise on the device,
    so a graphed and an eager step do not draw the same; test_networks_against_default_routes covers pl_kernels.)"""
    tr = import_module(TRAIN)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(4, 5, 16, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 32, 32, generator=g) * 2 - 1).to(cuda_dev)
    cfg = dict(noise_mode="const", d_reg_interval=1)
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
    print(f"[img2img vjp graphed] eager {se} graphed {sg}; gradients differing: "
          f"G {sdet.differing_grads(G, Ge)[:6]} D {sdet.differing_grads(D, De)[:6]}")
    assert sg.r1 > 0, sg
    assert (sg.loss_d, sg.loss_g, sg.r1) == (se.loss_d, se.loss_g, se.r1)
    sdet.assert_same_grads(tg, te, "img2img double-backward kernels, graphed against eager")


def test_r1_memory_at_64(gf, cuda_dev):
    """The discriminator layer's R1 gradient at 64^2, C = 512, batch 32: one n x n fp32 tensor of the composite would be
    32 * 8 * 4096^2 * 4 B = 17.2 GB.  On the kernels every tensor is [B, n, C] (268 MB) or [B, h, n]: the peak above the inputs stays
    under 40 of them."""
    B, R, C = 32, 64, 512
    torch.manual_seed(0)
    m = gf.ImageSelfAttention(C, 32).to(cuda_dev)
    m.kernel_double_backward = True
    x = torch.randn(B, R, R, C, device=cuda_dev)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(cuda_dev)
    base = torch.cuda.memory_allocated(cuda_dev)
    xs = x.requires_grad_(True)
    (gx,) = torch.autograd.grad(m(xs).sum(), xs, create_graph=True)
    grads = torch.autograd.grad(gx.square().sum(), [xs, *m.parameters()])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(cuda_dev) - base
    unit = B * R * R * C * 4
    print(f"[img2img vjp memory] peak above inputs {peak / 2**30:.2f} GiB = {peak / unit:.1f} x [B, n, C]")
    assert all(torch.isfinite(g_).all() for g_ in grads)
    assert peak <= 40 * unit
