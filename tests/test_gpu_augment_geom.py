"""ADA's fractional geometry on an H100 (``pytest -m gpu``; SURVEY A.4 item 16).

* gf_augment_resample_nchw and its adjoint through the C ABI, outputs between NaN guards: images with an identity fractional map equal
  gf_augment_nchw / gf_augment_adjoint_nchw bit for bit; sampled "bgc" parameters on Gaussian images against the fp64 definition,
  relative to a magnitude companion (the definition on |x| with |taps| and |M|); the shared-memory and the direct per-pixel paths;
  images outside the parameter domain (NaN for that image, its neighbours untouched); batches that wrap the grid.
* The adjoint identity in fp64 of the fp32 results; ops.augment(..., frac=...)'s first and second derivatives against fp64 autograd.
* Determinism and CUDA-graph replay, bit for bit; a captured sampler draws new maps on every replay and p = 0 replays the identity.
* R1 through "bgc" against fp64 autograd of the oracle discriminator; step_graphed with "bgc" and ADA against the eager step.
"""
import copy
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref
from tests.guards import Guarded, assert_exact
from tests.test_gpu_augment import _batch, _gan
from tests.test_gpu_ops_exact import F64, _call, _stream

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
BGC_NO_R90 = ("xflip", "xint", "scale", "rotate", "aniso", "xfrac", "brightness", "contrast", "lumaflip", "hue", "saturation")
# Sampled "bgc" at p = 1: max over elements of |y - y64| / companion (floored, see check_rel).  Measured on an H100 80GB HBM3 at a 700 W power limit: forward
# 2.0e-6 (16x16), 9.8e-6 (64x64), 2.6e-5 (256x256), 5.8e-6 (40x72); adjoint 4.9e-6, 3.3e-5, 2.5e-4 and 4.2e-5.  The error grows with
# the resolution: it is dominated by the fp32 sample positions nu = L q + e (an ulp of nu ~ 1000 is 6e-5 of a 2x-grid pixel).  Frozen
# with a margin.
FWD_REL_BOUND = 6e-5
ADJ_REL_BOUND = 6e-4


def run(gf, name, x, geom, frac, color, dev):
    B, C, H, W = x.shape
    out = Guarded((B, C, H, W), dev)
    xd, gd, fd = (t.contiguous().to(dev) for t in (x.float(), geom.to(torch.int32), frac.float()))
    cd = None if color is None else color.float().contiguous().to(dev)
    if name.startswith("gf_augment_resample"):
        _call(gf, name, xd.data_ptr(), out.ptr(), gd.data_ptr(), fd.data_ptr(), None if cd is None else cd.data_ptr(), B, C, H, W,
              _stream(dev))
    else:
        _call(gf, name, xd.data_ptr(), out.ptr(), gd.data_ptr(), None if cd is None else cd.data_ptr(), B, C, H, W, _stream(dev))
    return out.check(name).double().cpu()


def refs(ops, x, geom, frac, color, dev):
    """(forward, adjoint, forward companion, adjoint companion) of the definition in fp64 on `dev`: x is used as the cotangent too."""
    B, C, H, W = x.shape
    x, geom, frac = x.to(dev, F64), geom.to(dev), frac.to(dev)
    c64 = None if color is None else color.to(dev, F64)
    ab = lambda t: None if t is None else t.abs()
    fwd = ops.augment_ref(x, geom, c64, frac)
    adj = ops.augment_adjoint_ref(x, geom, c64, frac)
    taps = ops.sym6_filter(dev).abs()
    ident = ops.frac_flags(frac, H, W)[0].to(dev)[:, None, None, None]
    blit = ops.augment_ref(x.abs(), geom)
    res = ops.resample_ref(x.abs(), geom, frac, taps)
    comp = torch.where(ident, blit, res)
    with torch.enable_grad():
        x0 = torch.zeros_like(x).requires_grad_(True)
        (radj,) = torch.autograd.grad(ops.resample_ref(x0, geom, frac, taps), x0, x.abs() if c64 is None else
                                      torch.einsum("bij,bihw->bjhw", c64.reshape(B, 3, 4)[:, :, :3].abs(), x.abs()))
    ablit = ops.augment_adjoint_ref(x.abs(), geom, ab(c64))
    cadj = torch.where(ident, ablit, radj)
    if c64 is not None:
        M = c64.reshape(B, 3, 4).abs()
        comp = torch.einsum("bij,bjhw->bihw", M[:, :, :3], comp) + M[:, :, 3, None, None]
    return [t.cpu() for t in (fwd, adj, comp, cadj)]


def check_rel(gf, ops, x, geom, frac, color, dev, what, fb=FWD_REL_BOUND, ab=ADJ_REL_BOUND):
    fwd, adj, comp, cadj = refs(ops, x, geom, frac, color, dev)
    out = []
    for name, ref, c, bound in (("gf_augment_resample_nchw", fwd, comp, fb), ("gf_augment_resample_adjoint_nchw", adj, cadj, ab)):
        got = run(gf, name, x, geom, frac, color, dev)
        # the companion floored at 1e-6 of its image's maximum: a source pixel reached only by the edge of a bilinear footprint has a
        # companion of ~1e-9 while its tap weights carry the fp32 position error (DESIGN 4.12)
        floor = 1e-6 * c.amax(dim=(1, 2, 3), keepdim=True)
        rel = ((got - ref).abs() / torch.maximum(c, floor).clamp(min=1e-30)).max().item()
        print(f"[augment geom] {what} {name}: max |err| / companion = {rel:.3e}")
        assert rel <= bound, (what, name, rel)
        out.append(got)
    return out


# ------------------------------------------------------------------------------------------------ the kernels against fp64
@pytest.mark.parametrize("B,H,W", [(32, 16, 16), (16, 64, 64), (8, 256, 256), (16, 40, 72), (600, 16, 16)],
                         ids=lambda v: str(v))
def test_resample_bgc_against_fp64(gf, cuda_dev, B, H, W):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(H * 1000 + W + B)
    spec = tr.parse_augment("bgc") if H == W else BGC_NO_R90
    geom, color = tr.sample_augment(spec, 1.0, B, H, W, "cpu")
    frac = tr.sample_augment_frac(spec, 1.0, B, H, W, "cpu")
    assert not ops.frac_flags(frac, H, W)[0].any() and ops.frac_flags(frac, H, W)[1].all()
    x = torch.randn(B, 3, H, W, dtype=F64).float().double()
    check_rel(gf, ops, x, geom, frac, color, cuda_dev, f"bgc B{B} {H}x{W}")


def test_identity_images_are_the_blit_bit_for_bit(gf, cuda_dev):
    """A mixed batch: even images have the identity map (-0.0 entries included) and go through the blit, bit for bit."""
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(3)
    B, H, W = 12, 24, 20
    geom, color = tr.sample_augment(("xflip", "xint", "hue", "contrast"), 1.0, B, H, W, "cpu")
    frac = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, B, H, W, "cpu")
    frac[0::2] = torch.tensor([1.0, -0.0, 0.0, 0.0, 1.0, -0.0])
    x = torch.randn(B, 3, H, W)
    for col in (None, color):
        for name, blit in (("gf_augment_resample_nchw", "gf_augment_nchw"), ("gf_augment_resample_adjoint_nchw", "gf_augment_adjoint_nchw")):
            got = run(gf, name, x, geom, frac, col, cuda_dev)
            want = run(gf, blit, x, geom, frac, col, cuda_dev)
            assert_exact(got[0::2], want[0::2], name + " identity images")
            assert not torch.equal(got[1::2], want[1::2])
    check_rel(gf, ops, x.double(), geom, frac, color, cuda_dev, "mixed batch")


def test_shared_memory_and_direct_paths(gf, cuda_dev):
    """The forward's direct per-pixel path: a zoom-out by 8 (a 16 x 16 tile reads ~340 x 340 2x-grid points, beyond the 10240-float
    plan); the adjoint's chunked staging: a zoom-in by 8 (the preimage of a tile's 2x-grid box is ~340 points wide, 36 chunks of
    64 x 64); a zoom of 1.25 with a rotation stays in one shared-memory pass in both.  Each against fp64."""
    ops = import_module(OPS)
    torch.manual_seed(4)
    B, C, H, W = 4, 2, 20, 18
    x = torch.randn(B, C, H, W).double()
    geom = torch.tensor([[0, 0, 0, 0], [1, 3, -2, 0], [4, -1, 5, 0], [5, 0, 1, 0]], dtype=torch.int32)
    c, s = 0.8 * 0.8, 0.8 * 0.6
    for what, frac in (("zoom-out 8", torch.tensor([[8.0, 0.0, 0.5, 0.0, 8.0, -0.25]] * B)),
                       ("zoom-in 8", torch.tensor([[0.125, 0.0, 0.5, 0.0, 0.125, -0.25]] * B)),
                       ("rotation, zoom 1.25", torch.tensor([[c, -s, 0.3, s, c, -1.7]] * B))):
        check_rel(gf, ops, x, geom, frac, None, cuda_dev, what)


def test_out_of_domain_images_are_nan_and_alone(gf, cuda_dev):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(5)
    B, H, W = 8, 16, 24
    geom, color = tr.sample_augment(("xflip", "xint", "brightness"), 1.0, B, H, W, "cpu")
    frac = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, B, H, W, "cpu")
    x = torch.randn(B, 3, H, W)
    base = [run(gf, n, x, geom, frac, color, cuda_dev) for n in ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw")]
    bad = frac.clone()
    bad[1] = torch.tensor([float("nan"), 0, 0, 0, 1, 0])
    bad[3] = torch.tensor([20.0, 0, 0, 0, 1, 0])                                  # singular value 20 > 16
    bad[4] = torch.tensor([1.0, 0, 0, 0, 1 / 20, 0])                              # 1/20 < 1/16
    bad[6] = torch.tensor([1.0, 0, 64 * 24 + 1, 0, 1, 0])                         # translation beyond 64 max(H, W)
    ident, ok = ops.frac_flags(bad, H, W)
    assert ok.tolist() == [True, False, True, False, False, True, False, True]
    for name, b0 in zip(("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"), base):
        got = run(gf, name, x, geom, bad, color, cuda_dev)
        assert torch.isnan(got[~ok]).all(), name
        assert_exact(got[ok], b0[ok], name + " neighbours of out-of-domain images")


def test_sampler_on_the_device(cuda_dev):
    """A large draw on the device stays inside the domain, and TF32 matmuls (as bench.py enables them) do not touch the maps: the
    rotations stay orthogonal to fp32 round-off."""
    ops, tr = import_module(OPS), import_module(TRAIN)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        torch.manual_seed(11)
        big = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, 200000, 256, 256, cuda_dev).cpu()
        r = tr.sample_augment_frac(("rotate",), 1.0, 4096, 64, 64, cuda_dev).double().cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert ops.frac_flags(big, 256, 256)[1].all()
    R = r[:, [0, 1, 3, 4]].reshape(-1, 2, 2)
    assert (R @ R.transpose(1, 2) - torch.eye(2, dtype=F64)).abs().max() < 1e-6


# ------------------------------------------------------------------------------------------------ adjoint, autograd, replay
def test_adjoint_identity_of_the_fp32_results(gf, cuda_dev):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(6)
    B, H = 16, 32
    geom, _ = tr.sample_augment(("xflip", "rotate90", "xint"), 1.0, B, H, H, "cpu")
    frac = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, B, H, H, "cpu")
    x, g = torch.randn(B, 3, H, H), torch.randn(B, 3, H, H)
    ax = run(gf, "gf_augment_resample_nchw", x, geom, frac, None, cuda_dev)
    atg = run(gf, "gf_augment_resample_adjoint_nchw", g, geom, frac, None, cuda_dev)
    lhs, rhs = (ax * g.double()).sum(dim=(1, 2, 3)), (x.double() * atg).sum(dim=(1, 2, 3))
    scale = (ax.abs() * g.double().abs()).sum(dim=(1, 2, 3))
    rel = ((lhs - rhs).abs() / scale).max().item()
    print(f"[augment geom] adjoint identity: max |<Ax, g> - <x, A^T g>| / <|Ax|, |g|> = {rel:.3e}")
    assert rel < 1e-6


@pytest.mark.parametrize("colour", [False, True])
def test_autograd_against_fp64(gf, cuda_dev, colour):
    ops, tr = import_module(OPS), import_module(TRAIN)
    g = torch.Generator().manual_seed(7)
    torch.manual_seed(7)
    B, H = 6, 24
    geom, _ = tr.sample_augment(("xflip", "rotate90", "xint"), 1.0, B, H, H, "cpu")
    frac = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, B, H, H, "cpu")
    frac[2] = torch.tensor([1.0, 0, 0, 0, 1, 0])
    color = torch.randn(B, 12, generator=g, dtype=F64) if colour else None
    x64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    w64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    outs = []
    for dev, dt, fn in ((cuda_dev, torch.float32, ops.augment), ("cpu", F64, ops.augment_ref)):
        x = x64.to(dev, dt).requires_grad_(True)
        c = None if color is None else color.to(dev, dt)
        y = fn(x, geom.to(dev), c, frac.to(dev))
        (g1,) = torch.autograd.grad((y * w64.to(dev, dt)).square().sum(), x, create_graph=True)
        (g2,) = torch.autograd.grad((g1 * torch.sin(x)).sum(), x)
        outs.append([t.detach().double().cpu() for t in (y, g1, g2)])
    for what, got, want in zip(("value", "first derivative", "second derivative"), *outs):
        rel = ((got - want).norm() / want.norm()).item()
        print(f"[augment geom autograd] colour={colour} {what}: rel err {rel:.2e}")
        assert rel < 1e-5, what


def test_determinism_and_graph_replay(gf, cuda_dev):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(8)
    B, R = 16, 64
    spec = tr.parse_augment("bgc")
    geom, color = tr.sample_augment(spec, 1.0, B, R, R, cuda_dev)
    frac = tr.sample_augment_frac(spec, 1.0, B, R, R, cuda_dev)
    x, gy = torch.randn(B, 3, R, R, device=cuda_dev), torch.randn(B, 3, R, R, device=cuda_dev)
    names = ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw")
    first = [ops._augment_resample_native(n, t, geom, color, frac) for n, t in zip(names, (x, gy))]
    for _ in range(3):
        for n, t, f in zip(names, (x, gy), first):
            assert_exact(ops._augment_resample_native(n, t, geom, color, frac), f, n + " rerun")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops._augment_resample_native(names[0], x, geom, color, frac)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [ops._augment_resample_native(n, t, geom, color, frac) for n, t in zip(names, (x, gy))]
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for n, o, f in zip(names, outs, first):
            assert_exact(o, f, n + " replay")
    p = torch.ones((), device=cuda_dev)
    graph2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph2):
        g2, c2 = tr.sample_augment(spec, p, B, R, R, cuda_dev)
        f2 = tr.sample_augment_frac(spec, p, B, R, R, cuda_dev)
        y2 = ops.augment(x, g2, c2, f2)
    seen = []
    for _ in range(2):
        graph2.replay()
        torch.cuda.synchronize()
        seen.append(f2.clone())
        assert_exact(y2, ops._augment_resample_native(names[0], x, g2, c2, f2), "captured sampler")
    assert not torch.equal(seen[0], seen[1])
    p.zero_()
    graph2.replay()
    torch.cuda.synchronize()
    assert torch.equal(f2, torch.tensor([1.0, 0, 0, 0, 1, 0], device=cuda_dev).expand(B, 6)) and torch.equal(y2, x)


# ------------------------------------------------------------------------------------------------ training
def test_r1_through_bgc_against_fp64(gf, cuda_dev):
    ops = import_module(OPS)
    tr, _, D = _gan(gf, cuda_dev)
    B = 4
    torch.manual_seed(9)
    spec = tr.parse_augment("bgc")
    geom, color = tr.sample_augment(spec, 1.0, B, 64, 64, "cpu")
    frac = tr.sample_augment_frac(spec, 1.0, B, 64, 64, "cpu")
    reals = torch.rand(B, 3, 64, 64, generator=torch.Generator().manual_seed(4), dtype=F64) * 2 - 1
    x = reals.float().to(cuda_dev).requires_grad_(True)
    (g,) = torch.autograd.grad(D(ops.augment(x, geom.to(cuda_dev), color.to(cuda_dev), frac.to(cuda_dev))).sum(), x, create_graph=True)
    r1 = g.square().sum(dim=[1, 2, 3]).mean()
    (gw,) = torch.autograd.grad(r1, D.fromrgb.weight)
    sd = cref.cast(D.state_dict())
    sd["fromrgb.weight"].requires_grad_(True)
    x64 = reals.clone().requires_grad_(True)
    (g64,) = torch.autograd.grad(cref.discriminator_forward(sd, ops.augment_ref(x64, geom, color.double(), frac), None).sum(), x64,
                                 create_graph=True)
    r1_64 = g64.square().sum(dim=[1, 2, 3]).mean()
    (gw64,) = torch.autograd.grad(r1_64, sd["fromrgb.weight"])
    e_r1 = abs(r1.item() - r1_64.item()) / r1_64.item()
    e_g = ((g.detach().double().cpu() - g64.detach()).norm() / g64.norm()).item()
    e_w = ((gw.double().cpu() - gw64).norm() / gw64.norm()).item()
    print(f"[augment geom R1] r1 {r1.item():.6e} vs {r1_64.item():.6e}: rel {e_r1:.2e}; grad wrt reals {e_g:.2e}; d r1 / d fromrgb {e_w:.2e}")
    # measured 3.4e-5, 1.4e-3 and 2.4e-4 on an H100: the gradient with respect to the reals is 14x looser than with "bc" (DESIGN 4.12)
    assert e_r1 < 1e-4 and e_g < 5e-3 and e_w < 1e-3


def test_bgc_step_graphed_matches_eager(gf, cuda_dev):
    """As test_augmented_step_graphed_matches_eager, with "bgc": the p trajectory and the D loss bit for bit, R1 to 1e-3.  cuDNN is
    pinned to its deterministic algorithms, whose choice does not depend on timing: with autotuned algorithms the D loss of an R1 step
    has differed in its last bits between the two (DESIGN 4.12)."""
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        _graphed_against_eager(gf, cuda_dev)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


def _graphed_against_eager(gf, cuda_dev):
    cfg = dict(lr=0.0, noise_mode="const", d_reg_interval=2, augment="bgc", augment_p=0.5, ada_target=0.6, ada_interval=1, ada_kimg=0.2)
    z, reals, _, _ = _batch(cuda_dev)
    tr, G, D = _gan(gf, cuda_dev)
    tg = tr.Trainer(G, D, tr.TrainConfig(**cfg))
    tg.step_graphed(z, reals)
    _, Ge, De = _gan(gf, cuda_dev)
    te = tr.Trainer(Ge, De, tr.TrainConfig(**cfg))
    Ge.load_state_dict(G.state_dict())
    De.load_state_dict(D.state_dict())
    te.opt_g.load_state_dict(copy.deepcopy(tg.opt_g.state_dict()))
    te.opt_d.load_state_dict(copy.deepcopy(tg.opt_d.state_dict()))
    for a, b in ((te.augment_p, tg.augment_p), (te.ada_stats, tg.ada_stats), (te.ada_steps, tg.ada_steps)):
        a.copy_(b)
    te.it = tg.it
    for i in range(3):
        torch.cuda.manual_seed(2000 + i)
        sg = tg.step_graphed(z, reals)
        torch.cuda.manual_seed(2000 + i)
        se = te.step(z, reals)
        print(f"[augment geom graphed] step {i}: p {se.augment_p:.6f} / {sg.augment_p:.6f}; loss_d {se.loss_d:.6f} / {sg.loss_d:.6f}, "
              f"loss_g {se.loss_g:.6f} / {sg.loss_g:.6f}, r1 {se.r1:.6f} / {sg.r1:.6f}")
        assert sg.augment_p == se.augment_p, i
        assert (sg.r1 > 0) == (se.r1 > 0) == (i % 2 == 1)
        assert sg.loss_d == se.loss_d, i
        assert abs(se.r1 - sg.r1) <= 1e-3 * max(1.0, abs(se.r1)), i
