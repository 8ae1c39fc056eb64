"""Adaptive discriminator augmentation on an H100 (``pytest -m gpu``; SURVEY A.4 item 15).

* gf_augment_nchw and gf_augment_adjoint_nchw through the C ABI, outputs between NaN guards.  Exact cases: integer images, colour
  matrices with dyadic entries, so every output is an fp32 value in any order of summation; forward and adjoint equal the fp64
  definition (ops.augment_ref / augment_adjoint_ref) bit for bit.  They cover all 8 dihedral codes, codes above 7, maximal, negative
  and out-of-range translations, 2x2 to 256x256 and non-square grids, C = 1, 2 and 3, and batches that wrap the grid.  Realistic
  cases (sampled "bc" parameters, Gaussian images) are held to a frozen bound relative to their magnitude companion.
* ops.augment's first and second derivatives against fp64 autograd of the definition.
* Determinism and CUDA-graph replay, bit for bit; a captured sampler draws new parameters on every replay.
* Training with Discriminator(transformer=True), with and without labels: step_graphed against the eager step from the same state
  and the same RNG state, at lr = 0 (the p trajectory and the D loss bit for bit, R1 to 1e-3), and the R1 penalty and its
  gradient through the augmentation against fp64 autograd of the oracle discriminator.
"""
import copy
import math
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref
from tests.guards import Guarded, assert_exact
from tests.test_gpu_ops_exact import F64, _call, _stream, ints

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
# Realistic cases: max over elements of |y - y64| / companion (the same map on |x| with |M|).  Measured on an H100 80GB HBM3 at a
# 700 W power limit: forward 1.22e-7 (16x16) and 1.59e-7 (256x256), adjoint 1.39e-7 and 1.66e-7; frozen with a margin of 1.5x.
FWD_REL_BOUND = 2.5e-7
ADJ_REL_BOUND = 2.5e-7


# ------------------------------------------------------------------------------------------------ exact cases
EXACT_CASES = [  # (B, C, H, W, colour)
    (16, 3, 2, 2, True), (16, 1, 2, 2, False), (24, 3, 3, 3, True), (24, 1, 3, 3, False), (24, 3, 5, 7, True), (24, 2, 7, 5, False),
    (16, 3, 33, 33, True), (8, 3, 40, 72, True), (8, 3, 256, 256, True), (8, 1, 256, 256, False), (3000, 3, 2, 2, True),
    (600, 3, 16, 16, True)]


def case_id(c):
    return f"B{c[0]}-C{c[1]}-{c[2]}x{c[3]}-{'colour' if c[4] else 'blit'}"


def exact_params(B, C, H, W, colour, seed):
    """Integer images in [-8, 8]; geometry cycling through every code (and codes + 8), translations 0, +-(N-1), +-1, N/2 and beyond
    N - 1; colour entries multiples of 1/4 in [-1, 1], offsets multiples of 1/2."""
    x = ints((B, C, H, W), -8, 8, seed)
    tsx = [0, W - 1, -(W - 1), 1, -1, W // 2, W + 5, -(W + 5)]
    tsy = [0, -(H - 1), H - 1, -1, 1, -(H // 2), -(2 * H), 3 * H]
    geom = torch.tensor([[i % 8 + (8 if i % 11 == 5 else 0), tsx[(i // 8) % 8], tsy[(i // 8 + i) % 8], 0] for i in range(B)],
                        dtype=torch.int32)
    color = None
    if colour:
        color = ints((B, 3, 4), -4, 4, seed + 1) / 4
        color[:, :, 3] = ints((B, 3), -4, 4, seed + 2) / 2
        color = color.reshape(B, 12)
    return x, geom, color


def run_kernel(gf, name, x, geom, color, dev):
    B, C, H, W = x.shape
    out = Guarded((B, C, H, W), dev)
    xd, gd = x.float().contiguous().to(dev), geom.to(torch.int32).contiguous().to(dev)
    cd = None if color is None else color.float().contiguous().to(dev)
    _call(gf, name, xd.data_ptr(), out.ptr(), gd.data_ptr(), None if cd is None else cd.data_ptr(), B, C, H, W, _stream(dev))
    return out.check(name).double().cpu()


@pytest.mark.parametrize("case", EXACT_CASES, ids=case_id)
def test_augment_exact(gf, cuda_dev, case):
    ops = import_module(OPS)
    B, C, H, W, colour = case
    x, geom, color = exact_params(B, C, H, W, colour, seed=B * 7 + H * 3 + W)
    assert_exact(run_kernel(gf, "gf_augment_nchw", x, geom, color, cuda_dev), ops.augment_ref(x, geom, color), "forward " + case_id(case))
    gy = ints((B, C, H, W), -8, 8, seed=B + H + W + 99)
    assert_exact(run_kernel(gf, "gf_augment_adjoint_nchw", gy, geom, color, cuda_dev), ops.augment_adjoint_ref(gy, geom, color),
                 "adjoint " + case_id(case))


@pytest.mark.parametrize("res", [16, 256])
def test_augment_realistic(gf, cuda_dev, res):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(res)
    B = 32
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, res, res, "cpu")
    x, gy = torch.randn(B, 3, res, res, dtype=F64), torch.randn(B, 3, res, res, dtype=F64)
    x32, gy32 = x.float().double(), gy.float().double()             # the kernel's inputs, exactly
    c64 = color.double()
    cabs = c64.abs()
    for name, inp, ref, comp, bound in (
            ("gf_augment_nchw", x32, ops.augment_ref(x32, geom, c64), ops.augment_ref(x32.abs(), geom, cabs), FWD_REL_BOUND),
            ("gf_augment_adjoint_nchw", gy32, ops.augment_adjoint_ref(gy32, geom, c64), ops.augment_adjoint_ref(gy32.abs(), geom, cabs),
             ADJ_REL_BOUND)):
        got = run_kernel(gf, name, inp, geom, color, cuda_dev)
        rel = ((got - ref).abs() / comp.clamp(min=1e-30)).max().item()
        print(f"[augment realistic] {name} {res}x{res}: max |err| / companion = {rel:.3e}")
        assert rel <= bound, (name, rel)


# ------------------------------------------------------------------------------------------------ autograd, determinism, replay
@pytest.mark.parametrize("colour", [False, True])
def test_augment_autograd_against_fp64(gf, cuda_dev, colour):
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(5)
    B, H = 6, 24
    geom = torch.tensor([[c, t, -t, 0] for c, t in zip(range(2, 8), (0, 23, -23, 5, -7, 2))], dtype=torch.int32)
    color = torch.randn(B, 12, generator=g, dtype=F64) if colour else None
    x64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    w64 = torch.randn(B, 3, H, H, generator=g, dtype=F64)
    outs = []
    for dev, dt, fn in ((cuda_dev, torch.float32, ops.augment), ("cpu", F64, ops.augment_ref)):
        x = x64.to(dev, dt).requires_grad_(True)
        c = None if color is None else color.to(dev, dt)
        y = fn(x, geom.to(dev), c)
        (g1,) = torch.autograd.grad((y * w64.to(dev, dt)).square().sum(), x, create_graph=True)
        (g2,) = torch.autograd.grad((g1 * torch.sin(x)).sum(), x)
        outs.append([t.detach().double().cpu() for t in (y, g1, g2)])
    for what, got, want in zip(("value", "first derivative", "second derivative"), *outs):
        rel = ((got - want).norm() / want.norm()).item()
        print(f"[augment autograd] colour={colour} {what}: rel err {rel:.2e}")
        assert rel < 1e-6, what


def test_augment_determinism_and_graph_replay(gf, cuda_dev):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(2)
    B, R = 16, 64
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, R, R, cuda_dev)
    x = torch.randn(B, 3, R, R, device=cuda_dev)
    gy = torch.randn(B, 3, R, R, device=cuda_dev)
    names = ("gf_augment_nchw", "gf_augment_adjoint_nchw")
    first = [ops._augment_native(n, t, geom, color) for n, t in zip(names, (x, gy))]
    for _ in range(3):
        for n, t, f in zip(names, (x, gy), first):
            assert_exact(ops._augment_native(n, t, geom, color), f, n + " rerun")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops._augment_native(names[0], x, geom, color)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [ops._augment_native(n, t, geom, color) for n, t in zip(names, (x, gy))]
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for n, o, f in zip(names, outs, first):
            assert_exact(o, f, n + " replay")
    # a captured sampler + augmentation draws new parameters on each replay; p = 0 replays the identity
    p = torch.ones((), device=cuda_dev)
    graph2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph2):
        g2, c2 = tr.sample_augment(tr.AUGMENT_OPS, p, B, R, R, cuda_dev)
        y2 = ops.augment(x, g2, c2)
    seen = []
    for _ in range(2):
        graph2.replay()
        torch.cuda.synchronize()
        seen.append((g2.clone(), y2.clone()))
        assert_exact(y2, ops._augment_native(names[0], x, g2, c2), "captured sampler")
    assert not torch.equal(seen[0][0], seen[1][0])
    p.zero_()
    graph2.replay()
    torch.cuda.synchronize()
    assert not g2.any() and torch.equal(y2, x)


# ------------------------------------------------------------------------------------------------ training
def _gan(gf, dev, c_dim=0):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, exact_fp32=True,
                     c_dim=c_dim).to(dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, transformer=True, components_num=8, latent_dim=32, exact_fp32=True,
                         c_dim=c_dim).to(dev)
    return tr, G, D


def _batch(dev, B=4, c_dim=0, seed=5):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 9, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    if not c_dim:
        return z, reals, None, None
    oh = lambda: torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev)
    return z, reals, oh(), oh()


@pytest.mark.parametrize("c_dim", [0, 5], ids=["unconditional", "labels"])
def test_augmented_step_graphed_matches_eager(gf, cuda_dev, c_dim):
    """step_graphed with "bc" augmentation and ADA against the eager step.  After the graphed trainer's first call (warm-up, capture,
    replay) its weights, Adam states and ADA state go to an eager trainer; then both take three steps (the second with R1), each
    from the same CUDA RNG state, so both draw the same augmentation parameters.  lr = 0 keeps the weights of both trainers equal.
    p moves every step (interval 1); its trajectory and the D phase's loss (reals and fakes, both augmented) must be the same bits,
    and R1 must agree to 1e-3.  The G phase's loss is printed, not held: it has differed by up to 1.1 % between the two (DESIGN
    4.11, an open finding)."""
    cfg = dict(lr=0.0, noise_mode="const", d_reg_interval=2, augment="bc", augment_p=0.5, ada_target=0.6, ada_interval=1, ada_kimg=0.2)
    z, reals, gen_c, real_c = _batch(cuda_dev, c_dim=c_dim)
    tr, G, D = _gan(gf, cuda_dev, c_dim)
    tg = tr.Trainer(G, D, tr.TrainConfig(**cfg))
    s0 = tg.step_graphed(z, reals, gen_c, real_c)
    assert s0.r1 > 0 and abs(abs(s0.augment_p - 0.5) - 0.02) < 1e-6       # one update of 4 / (0.2 * 1000) from 0.5
    _, Ge, De = _gan(gf, cuda_dev, c_dim)
    te = tr.Trainer(Ge, De, tr.TrainConfig(**cfg))
    Ge.load_state_dict(G.state_dict())
    De.load_state_dict(D.state_dict())
    te.opt_g.load_state_dict(copy.deepcopy(tg.opt_g.state_dict()))
    te.opt_d.load_state_dict(copy.deepcopy(tg.opt_d.state_dict()))
    for a, b in ((te.augment_p, tg.augment_p), (te.ada_stats, tg.ada_stats), (te.ada_steps, tg.ada_steps)):
        a.copy_(b)
    te.it = tg.it
    ps = []
    for i in range(3):
        torch.cuda.manual_seed(1000 + i)
        sg = tg.step_graphed(z, reals, gen_c, real_c)
        torch.cuda.manual_seed(1000 + i)
        se = te.step(z, reals, gen_c, real_c)
        print(f"[augment graphed] step {i}: p eager {se.augment_p:.6f} graphed {sg.augment_p:.6f}; loss_d {se.loss_d:.6f} / {sg.loss_d:.6f}, "
              f"loss_g {se.loss_g:.6f} / {sg.loss_g:.6f}, r1 {se.r1:.6f} / {sg.r1:.6f}")
        assert sg.augment_p == se.augment_p, i
        assert (sg.r1 > 0) == (se.r1 > 0) == (i % 2 == 1)
        assert sg.loss_d == se.loss_d, i
        assert abs(se.r1 - sg.r1) <= 1e-3 * max(1.0, abs(se.r1)), i
        ps.append(se.augment_p)
    assert len(set(ps)) > 1 or ps[0] in (0.0, 1.0)


def test_r1_through_the_augmentation_against_fp64(gf, cuda_dev):
    """R1 = mean_b |d D(A_b x) / d x_b|^2 with fixed "bc" parameters, and its gradient with respect to D's fromrgb weight (the second
    derivative through the augmentation and the attention layers' composite route) against fp64 autograd of the oracle."""
    ops = import_module(OPS)
    tr, _, D = _gan(gf, cuda_dev)
    B = 4
    torch.manual_seed(9)
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, 64, 64, "cpu")
    reals = torch.rand(B, 3, 64, 64, generator=torch.Generator().manual_seed(4), dtype=F64) * 2 - 1
    x = reals.float().to(cuda_dev).requires_grad_(True)
    (g,) = torch.autograd.grad(D(ops.augment(x, geom.to(cuda_dev), color.to(cuda_dev))).sum(), x, create_graph=True)
    r1 = g.square().sum(dim=[1, 2, 3]).mean()
    (gw,) = torch.autograd.grad(r1, D.fromrgb.weight)
    sd = cref.cast(D.state_dict())
    sd["fromrgb.weight"].requires_grad_(True)
    x64 = reals.clone().requires_grad_(True)
    (g64,) = torch.autograd.grad(cref.discriminator_forward(sd, ops.augment_ref(x64, geom, color.double()), None).sum(), x64,
                                 create_graph=True)
    r1_64 = g64.square().sum(dim=[1, 2, 3]).mean()
    (gw64,) = torch.autograd.grad(r1_64, sd["fromrgb.weight"])
    e_r1 = abs(r1.item() - r1_64.item()) / r1_64.item()
    e_g = ((g.detach().double().cpu() - g64.detach()).norm() / g64.norm()).item()
    e_w = ((gw.double().cpu() - gw64).norm() / gw64.norm()).item()
    print(f"[augment R1] r1 {r1.item():.6e} vs {r1_64.item():.6e}: rel {e_r1:.2e}; grad wrt reals {e_g:.2e}; d r1 / d fromrgb {e_w:.2e}")
    assert e_r1 < 1e-4 and e_g < 1e-4 and e_w < 1e-3
