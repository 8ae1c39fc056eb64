"""ADA's image-space filtering and additive noise on an H100 (``pytest -m gpu``; SURVEY A.4 item 17).

* gf_augment_filter_nchw and its adjoint through the C ABI, outputs between NaN guards.  Exact cases: integer images in [-8, 8],
  identity gains, one-hot and power-of-two gains on the short bands 2 and 3, dyadic sigma on integer noise; a host proof (exact
  rational bounds) shows every partial sum of both kernels fits in 24 bits, so forward and adjoint equal the fp64 definition bit for
  bit.  22x22 to 256x256, non-square grids, C = 1 and 3, a batch that wraps the grid.  The impulse response of each one-hot gain is
  its bank row, exactly.  Realistic cases (sampled "bgcfn" at p = 1, Gaussian images) are held to a frozen bound relative to their
  magnitude companion (the definition on |x| with |bank|).
* ops.augment_filter's first and second derivatives against fp64 autograd; reruns and graph replays bit for bit.
* R1 through "bgcfn" against fp64 autograd of the oracle discriminator; step_graphed with "bgcfn" and ADA against the eager step.
"""
import copy
from fractions import Fraction
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref
from tests.guards import Guarded, assert_exact
from tests.test_gpu_augment import _batch, _gan
from tests.test_gpu_ops_exact import F64, _call, _stream, ints

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
# Sampled "bgcfn" at p = 1 on Gaussian images: max over elements of |y - y64| / companion.  Measured on an H100 80GB HBM3 at a 700 W
# power limit: forward 1.83e-7 (64x64), 2.39e-7 (256x256), 1.35e-7 (22x37); adjoint 1.79e-7, 2.29e-7, 2.02e-7.  Frozen with a margin.
FWD_REL_BOUND = 4e-7
ADJ_REL_BOUND = 4e-7


def run(gf, name, x, gains, sigma, noise, dev):
    B, C, H, W = x.shape
    out = Guarded((B, C, H, W), dev)
    d = lambda t: None if t is None else t.float().contiguous().to(dev)
    xd, gd, sd, nd = d(x), d(gains), d(sigma), d(noise)
    p = lambda t: None if t is None else t.data_ptr()
    if name == "gf_augment_filter_nchw":
        _call(gf, name, xd.data_ptr(), out.ptr(), p(gd), p(sd), p(nd), B, C, H, W, _stream(dev))
    else:
        _call(gf, name, xd.data_ptr(), out.ptr(), p(gd), B, C, H, W, _stream(dev))
    return out.check(name).double().cpu()


# ------------------------------------------------------------------------------------------------ exact cases
def _v2(fr):
    """The 2-adic valuation of a nonzero dyadic rational."""
    n, d = fr.numerator, fr.denominator
    assert d & (d - 1) == 0, fr
    v = -(d.bit_length() - 1)
    while n % 2 == 0:
        n //= 2
        v += 1
    return v


def _fits24(bound, q):
    """Every multiple of 2^q of magnitude at most `bound` is an fp32 value."""
    return bound <= Fraction(2) ** (q + 24)


def _axis_row_sums(h, N, adjoint):
    """max over outputs of sum |h[t]| over the terms of one axis (forward: the taps of a row; adjoint: the (j, t) pairs that reach
    source index m through the mirror R_N)."""
    if not adjoint:
        return sum(abs(v) for v in h)
    R = lambda i: -i if i < 0 else (2 * (N - 1) - i if i >= N else i)
    s = [Fraction(0)] * N
    for j in range(N):
        for t in range(43):
            if h[t]:
                s[R(j + t - 21)] += abs(h[t])
    return max(s)


def prove_exact(bank, gains, sigma, H, W, xmax=8, nmax=8):
    """Host proof for one image: the kernel's taps (the fmaf chain over the bands), every partial sum of the vertical and the
    horizontal pass (forward and adjoint, the reflected preimages included) and the noise add are fp32 values.  All of them are
    multiples of a common power of two and bounded by the sum of the absolute values of their terms."""
    g = [Fraction(v) for v in gains]
    if g == [1, 1, 1, 1]:
        return True                                                     # copied
    h = [Fraction(0)] * 43
    for i in range(4):                                                  # the taps, partial by partial
        for t in range(43):
            h[t] += g[i] * Fraction(int(bank[i][t]), 2 ** 15)
            if h[t] and not _fits24(abs(h[t]), _v2(h[t])):
                return False
    q = min(_v2(v) for v in h if v)
    for adjoint in (False, True):
        b1 = xmax * _axis_row_sums(h, H, adjoint)
        b2 = b1 * _axis_row_sums(h, W, adjoint)
        if not (_fits24(b1, q) and _fits24(b2, 2 * q)):
            return False
    if sigma:
        s = Fraction(sigma)
        b2 = xmax * _axis_row_sums(h, H, False) * _axis_row_sums(h, W, False)
        if not _fits24(b2 + abs(s) * nmax, min(2 * q, _v2(s))):
            return False
    return True


GAIN_PATTERNS = [(1.0, 1.0, 1.0, 1.0), (0.0, 0.0, 1.0, 0.0), (0.0, 0.0, 2.0, 0.0), (0.0, 0.0, 8.0, 0.0), (0.0, 0.0, 0.0, 1.0),
                 (0.0, 0.0, 0.0, 0.5), (0.0, 0.0, 0.0, 4.0), (0.0, 0.0, 1.0, 2.0 ** -5), (0.0, 0.0, 4.0, 0.125)]
SIGMAS = [0.0, 0.125, 0.5, 1.0, 0.0, 0.25, 2.0 ** -6]
EXACT_CASES = [(9, 3, 22, 22), (9, 1, 22, 37), (7, 3, 37, 22), (9, 3, 64, 64), (9, 1, 256, 256), (4, 3, 256, 256), (200, 3, 22, 22)]


def exact_params(B, C, H, W, seed):
    x = ints((B, C, H, W), -8, 8, seed)
    noise = ints((B, C, H, W), -8, 8, seed + 1)
    gains = torch.tensor([GAIN_PATTERNS[(i + seed) % len(GAIN_PATTERNS)] for i in range(B)], dtype=F64)
    sigma = torch.tensor([SIGMAS[(i * 3 + seed) % len(SIGMAS)] for i in range(B)], dtype=F64)
    return x, gains, sigma, noise


@pytest.mark.parametrize("case", EXACT_CASES, ids=lambda c: f"B{c[0]}-C{c[1]}-{c[2]}x{c[3]}")
def test_filter_exact(gf, cuda_dev, case):
    ops = import_module(OPS)
    B, C, H, W = case
    x, gains, sigma, noise = exact_params(B, C, H, W, seed=B + H * 3 + W)
    bank = ops.imgfilter_bank_numerators()
    for g, s in {(tuple(g.tolist()), s.item()) for g, s in zip(gains, sigma)}:
        assert prove_exact(bank, g, s, H, W), (g, s)
    fwd = ops.augment_filter_ref(x, gains, sigma, noise)
    assert_exact(run(gf, "gf_augment_filter_nchw", x, gains, sigma, noise, cuda_dev), fwd, "forward")
    assert_exact(run(gf, "gf_augment_filter_nchw", x, gains, None, None, cuda_dev), ops.augment_filter_ref(x, gains), "forward, no noise")
    assert_exact(run(gf, "gf_augment_filter_nchw", x, None, sigma, noise, cuda_dev), ops.augment_filter_ref(x, None, sigma, noise),
                 "noise alone")
    gy = ints((B, C, H, W), -8, 8, seed=B + H + W + 99)
    assert_exact(run(gf, "gf_augment_filter_adjoint_nchw", gy, gains, None, None, cuda_dev), ops.augment_filter_adjoint_ref(gy, gains),
                 "adjoint")


def test_impulse_response_is_the_bank_row(gf, cuda_dev):
    """A unit impulse at the centre of a 64 x 64 plane under the one-hot gains e_i gives bank_i (x) bank_i, exactly; the adjoint
    (symmetric taps) gives the same."""
    ops = import_module(OPS)
    bank = ops.imgfilter_bank()
    x = torch.zeros(4, 1, 64, 64, dtype=F64)
    x[:, :, 32, 32] = 1.0
    gains = torch.eye(4, dtype=F64)
    want = torch.zeros(4, 1, 64, 64, dtype=F64)
    for i in range(4):
        want[i, 0, 11:54, 11:54] = torch.outer(bank[i], bank[i])
    for name in ("gf_augment_filter_nchw", "gf_augment_filter_adjoint_nchw"):
        assert_exact(run(gf, name, x, gains, None, None, cuda_dev), want, name)


def test_identity_and_zero_sigma_images_are_copied_bit_for_bit(gf, cuda_dev):
    """Identity gains copy the plane (-0, inf and NaN neighbours included); sigma = 0 does not read the noise (NaN there)."""
    B, C, H, W = 6, 3, 40, 30
    x = torch.randn(B, C, H, W)
    x[:, :, 3, 4], x[:, :, 10, 10], x[:, :, 20, 7] = -0.0, float("inf"), float("nan")
    gains = torch.ones(B, 4)
    sigma = torch.zeros(B)
    noise = torch.full((B, C, H, W), float("nan"))
    for g in (gains, None):
        got = run(gf, "gf_augment_filter_nchw", x, g, sigma, noise, cuda_dev).float()
        assert torch.equal(got.view(torch.int32), x.view(torch.int32))
    got = run(gf, "gf_augment_filter_adjoint_nchw", x, gains, None, None, cuda_dev).float()
    assert torch.equal(got.view(torch.int32), x.view(torch.int32))


# ------------------------------------------------------------------------------------------------ realistic cases
def check_rel(gf, ops, x, gains, sigma, noise, dev, what):
    B, C, H, W = x.shape
    xd, gd, sd, nd = (t.to(dev, F64) for t in (x, gains, sigma, noise))
    absbank = ops.imgfilter_bank(dev).abs()
    fwd = ops.augment_filter_ref(xd, gd, sd, nd).cpu()
    comp = (ops.augment_filter_ref(xd.abs(), gd.abs(), bank=absbank) + sd.abs()[:, None, None, None] * nd.abs()).cpu()
    adj = ops.augment_filter_adjoint_ref(xd, gd).cpu()
    cadj = ops.augment_filter_adjoint_ref(xd.abs(), gd.abs(), bank=absbank).cpu()
    out = []
    for name, args, ref, c, bound in (("gf_augment_filter_nchw", (gains, sigma, noise), fwd, comp, FWD_REL_BOUND),
                                      ("gf_augment_filter_adjoint_nchw", (gains, None, None), adj, cadj, ADJ_REL_BOUND)):
        got = run(gf, name, x, *args, dev)
        rel = ((got - ref).abs() / c.clamp(min=1e-30)).max().item()
        print(f"[augment filter] {what} {name}: max |err| / companion = {rel:.3e}")
        assert rel <= bound, (what, name, rel)
        out.append(got)
    return out


@pytest.mark.parametrize("B,H,W", [(16, 64, 64), (8, 256, 256), (12, 22, 37)], ids=lambda v: str(v))
def test_bgcfn_against_fp64(gf, cuda_dev, B, H, W):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(H * 1000 + W + B)
    gains, sigma, noise = tr.sample_augment_filter(tr.FILTER_OPS, 1.0, B, 3, H, W, "cpu")
    assert not (gains == 1).all(dim=1).any() and (sigma > 0).all()
    x = torch.randn(B, 3, H, W)
    check_rel(gf, ops, x.double(), gains.double(), sigma.double(), noise.double(), cuda_dev, f"bgcfn B{B} {H}x{W}")


def test_adjoint_identity_of_the_fp32_results(gf, cuda_dev):
    tr = import_module(TRAIN)
    torch.manual_seed(6)
    B, H, W = 8, 48, 70
    gains, _, _ = tr.sample_augment_filter(("imgfilter",), 1.0, B, 3, H, W, "cpu")
    x, g = torch.randn(B, 3, H, W), torch.randn(B, 3, H, W)
    ax = run(gf, "gf_augment_filter_nchw", x, gains, None, None, cuda_dev)
    atg = run(gf, "gf_augment_filter_adjoint_nchw", g, gains, None, None, cuda_dev)
    lhs, rhs = (ax * g.double()).sum(dim=(1, 2, 3)), (x.double() * atg).sum(dim=(1, 2, 3))
    scale = (ax.abs() * g.double().abs()).sum(dim=(1, 2, 3))
    rel = ((lhs - rhs).abs() / scale).max().item()
    print(f"[augment filter] adjoint identity: max |<Fx, g> - <x, F^T g>| / <|Fx|, |g|> = {rel:.3e}")
    assert rel < 1e-6


# ------------------------------------------------------------------------------------------------ autograd, replay
@pytest.mark.parametrize("with_noise", [False, True])
def test_autograd_against_fp64(gf, cuda_dev, with_noise):
    ops, tr = import_module(OPS), import_module(TRAIN)
    g = torch.Generator().manual_seed(7)
    torch.manual_seed(7)
    B, H = 6, 32
    gains, sigma, noise = tr.sample_augment_filter(tr.FILTER_OPS, 1.0, B, 3, H, H, "cpu")
    gains[2] = 1.0
    if not with_noise:
        sigma = noise = None
    x64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    w64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    outs = []
    for dev, dt, fn in ((cuda_dev, torch.float32, ops.augment_filter), ("cpu", F64, ops.augment_filter_ref)):
        x = x64.to(dev, dt).requires_grad_(True)
        s, n = (None, None) if sigma is None else (sigma.to(dev, dt), noise.to(dev, dt))
        y = fn(x, gains.to(dev, dt), s, n)
        (g1,) = torch.autograd.grad((y * w64.to(dev, dt)).square().sum(), x, create_graph=True)
        (g2,) = torch.autograd.grad((g1 * torch.sin(x)).sum(), x)
        outs.append([t.detach().double().cpu() for t in (y, g1, g2)])
    for what, got, want in zip(("value", "first derivative", "second derivative"), *outs):
        rel = ((got - want).norm() / want.norm()).item()
        print(f"[augment filter autograd] noise={with_noise} {what}: rel err {rel:.2e}")
        assert rel < 1e-5, what


def test_determinism_and_graph_replay(gf, cuda_dev):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(8)
    B, C, R = 16, 3, 64
    gains, sigma, noise = tr.sample_augment_filter(tr.FILTER_OPS, 1.0, B, C, R, R, cuda_dev)
    x, gy = torch.randn(B, C, R, R, device=cuda_dev), torch.randn(B, C, R, R, device=cuda_dev)
    fwd = lambda: ops._augment_filter_native("gf_augment_filter_nchw", x, gains, sigma, noise)
    adj = lambda: ops._augment_filter_native("gf_augment_filter_adjoint_nchw", gy, gains)
    first = [fwd(), adj()]
    for _ in range(3):
        for f, w, n in zip((fwd, adj), first, ("forward", "adjoint")):
            assert_exact(f(), w, n + " rerun")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fwd()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [fwd(), adj()]
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for o, w, n in zip(outs, first, ("forward", "adjoint")):
            assert_exact(o, w, n + " replay")
    p = torch.ones((), device=cuda_dev)
    graph2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph2):
        g2, s2, n2 = tr.sample_augment_filter(tr.FILTER_OPS, p, B, C, R, R, cuda_dev)
        y2 = ops.augment_filter(x, g2, s2, n2)
    seen = []
    for _ in range(2):
        graph2.replay()
        torch.cuda.synchronize()
        seen.append(g2.clone())
        assert_exact(y2, ops._augment_filter_native("gf_augment_filter_nchw", x, g2, s2, n2), "captured sampler")
    assert not torch.equal(seen[0], seen[1])
    p.zero_()
    graph2.replay()
    torch.cuda.synchronize()
    assert torch.equal(g2, torch.ones(B, 4, device=cuda_dev)) and torch.equal(s2, torch.zeros(B, device=cuda_dev)) and torch.equal(y2, x)


# ------------------------------------------------------------------------------------------------ training
def test_r1_through_bgcfn_against_fp64(gf, cuda_dev):
    ops = import_module(OPS)
    tr, _, D = _gan(gf, cuda_dev)
    B = 4
    torch.manual_seed(9)
    spec = tr.parse_augment("bgcfn")
    geom, color = tr.sample_augment(spec, 1.0, B, 64, 64, "cpu")
    frac = tr.sample_augment_frac(spec, 1.0, B, 64, 64, "cpu")
    gains, sigma, noise = tr.sample_augment_filter(spec, 1.0, B, 3, 64, 64, "cpu")
    reals = torch.rand(B, 3, 64, 64, generator=torch.Generator().manual_seed(4), dtype=F64) * 2 - 1
    x = reals.float().to(cuda_dev).requires_grad_(True)
    d = lambda t: t.to(cuda_dev)
    y = ops.augment_filter(ops.augment(x, d(geom), d(color), d(frac)), d(gains), d(sigma), d(noise))
    (g,) = torch.autograd.grad(D(y).sum(), x, create_graph=True)
    r1 = g.square().sum(dim=[1, 2, 3]).mean()
    (gw,) = torch.autograd.grad(r1, D.fromrgb.weight)
    sd = cref.cast(D.state_dict())
    sd["fromrgb.weight"].requires_grad_(True)
    x64 = reals.clone().requires_grad_(True)
    y64 = ops.augment_filter_ref(ops.augment_ref(x64, geom, color.double(), frac), gains.double(), sigma.double(), noise.double())
    (g64,) = torch.autograd.grad(cref.discriminator_forward(sd, y64, None).sum(), x64, create_graph=True)
    r1_64 = g64.square().sum(dim=[1, 2, 3]).mean()
    (gw64,) = torch.autograd.grad(r1_64, sd["fromrgb.weight"])
    e_r1 = abs(r1.item() - r1_64.item()) / r1_64.item()
    e_g = ((g.detach().double().cpu() - g64.detach()).norm() / g64.norm()).item()
    e_w = ((gw.double().cpu() - gw64).norm() / gw64.norm()).item()
    print(f"[augment filter R1] r1 {r1.item():.6e} vs {r1_64.item():.6e}: rel {e_r1:.2e}; grad wrt reals {e_g:.2e}; d r1 / d fromrgb {e_w:.2e}")
    # the bounds of "bgc" (DESIGN 4.12): the filter adds a linear map with an exact adjoint after the resampler
    assert e_r1 < 1e-4 and e_g < 5e-3 and e_w < 1e-3


def test_bgcfn_step_graphed_matches_eager(gf, cuda_dev):
    """As test_bgc_step_graphed_matches_eager, with "bgcfn": the p trajectory, the D loss and the G loss bit for bit, R1 to 1e-3, with
    cuDNN pinned to its deterministic algorithms."""
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        cfg = dict(lr=0.0, noise_mode="const", d_reg_interval=2, augment="bgcfn", augment_p=0.5, ada_target=0.6, ada_interval=1,
                   ada_kimg=0.2)
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
            torch.cuda.manual_seed(3000 + i)
            sg = tg.step_graphed(z, reals)
            torch.cuda.manual_seed(3000 + i)
            se = te.step(z, reals)
            print(f"[augment filter graphed] step {i}: p {se.augment_p:.6f} / {sg.augment_p:.6f}; loss_d {se.loss_d:.6f} / {sg.loss_d:.6f}, "
                  f"loss_g {se.loss_g:.6f} / {sg.loss_g:.6f}, r1 {se.r1:.6f} / {sg.r1:.6f}")
            assert sg.augment_p == se.augment_p, i
            assert (sg.r1 > 0) == (se.r1 > 0) == (i % 2 == 1)
            assert sg.loss_d == se.loss_d, i
            assert sg.loss_g == se.loss_g, i
            assert abs(se.r1 - sg.r1) <= 1e-3 * max(1.0, abs(se.r1)), i
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev
