"""CPU checks of ADA's image-space filtering and additive noise (SURVEY A.4 item 17): the exact filter bank against a `fractions`
derivation and ADA's derivation from the sym2 taps, the fp64 definition against a restatement of ADA's own imgfilter and noise block,
the identity and adjoint identities, the custom autograd functions (kernels swapped for the definition), the sampler against a
restatement of ADA's loop, the presets, the refusals of the two new gf_ops.h entry points and a CPU training run with "bgcfn" and R1."""
import json
import math
import os
import subprocess
import sys
from fractions import Fraction
from importlib import import_module

import numpy as np
import pytest
import scipy.signal
import torch

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
# the sym2 wavelet's low-pass taps as ADA lists them
SYM2 = [-0.12940952255092145, 0.22414386804185735, 0.836516303737469, 0.48296291314469025]


def fraction_bank():
    """ADA's recipe in exact rational arithmetic from lo2 = conv(h, h[::-1]) / 2 and hi2 of the Deslauriers-Dubuc filters."""
    lo2 = [Fraction(v, 32) for v in (-1, 0, 9, 16, 9, 0, -1)]
    hi2 = [Fraction(v, 32) for v in (1, 0, -9, 16, -9, 0, 1)]

    def conv(a, b):
        out = [Fraction(0)] * (len(a) + len(b) - 1)
        for i, u in enumerate(a):
            for j, v in enumerate(b):
                out[i + j] += u * v
        return out
    bank = [[Fraction(1)], [Fraction(0)], [Fraction(0)], [Fraction(0)]]
    for i in range(1, 4):
        bank = [conv([v for a in r for v in (a, Fraction(0))][:-1], lo2) for r in bank]
        s = (len(bank[i]) - len(hi2)) // 2
        for k, v in enumerate(hi2):
            bank[i][s + k] += v
    return bank


def ada_bank():
    """ADA's own construction from the published sym2 taps, in fp64 (numpy / scipy)."""
    Hz_lo = np.asarray(SYM2)
    Hz_hi = Hz_lo * ((-1) ** np.arange(Hz_lo.size))
    Hz_lo2 = np.convolve(Hz_lo, Hz_lo[::-1]) / 2
    Hz_hi2 = np.convolve(Hz_hi, Hz_hi[::-1]) / 2
    Hz_fbank = np.eye(4, 1)
    for i in range(1, Hz_fbank.shape[0]):
        Hz_fbank = np.dstack([Hz_fbank, np.zeros_like(Hz_fbank)]).reshape(Hz_fbank.shape[0], -1)[:, :-1]
        Hz_fbank = scipy.signal.convolve(Hz_fbank, [Hz_lo2])
        Hz_fbank[i, (Hz_fbank.shape[1] - Hz_hi2.size) // 2: (Hz_fbank.shape[1] + Hz_hi2.size) // 2] += Hz_hi2
    return Hz_fbank


def test_bank_is_exact_and_matches_adas_derivation():
    ops = import_module(OPS)
    bank = ops.imgfilter_bank()
    exact = fraction_bank()
    assert bank.shape == (4, 43)
    for i in range(4):
        for t in range(43):
            assert Fraction(bank[i, t].item()) == exact[i][t], (i, t)
            assert exact[i][t] * 2 ** 15 == int(exact[i][t] * 2 ** 15) and abs(exact[i][t]) <= Fraction(1, 2)
        assert exact[i] == exact[i][::-1], i                              # symmetric: correlation = convolution
    assert [sum(r) for r in exact] == [1, 0, 0, 0]
    assert [sum(c) for c in zip(*exact)] == [1 if t == 21 else 0 for t in range(43)]
    assert torch.equal(ops.imgfilter_bank(dtype=torch.float32).double(), bank)
    d = np.abs(ada_bank() - bank.numpy()).max()
    assert d <= 1e-12, d
    print(f"[imgfilter bank] max |ADA's fp64 sym2 derivation - exact bank| = {d:.2e}")
    assert [sum(1 for v in r if v != 0) for r in exact][2:] == [15, 5]   # the short bands: 19 and 7 taps wide
    assert [max(t for t in range(43) if r[t] != 0) - min(t for t in range(43) if r[t] != 0) + 1 for r in exact[2:]] == [19, 7]


def ada_imgfilter(images, g, bank):
    """ADA's imgfilter block, restated: Hz_prime = g @ Hz_fbank, a reflect pad, a grouped conv2d along x then along y."""
    batch_size, num_channels, height, width = images.shape
    Hz_prime = g @ bank
    Hz_prime = Hz_prime.unsqueeze(1).repeat([1, num_channels, 1])
    Hz_prime = Hz_prime.reshape([batch_size * num_channels, 1, -1])
    p = bank.shape[1] // 2
    images = images.reshape([1, batch_size * num_channels, height, width])
    images = torch.nn.functional.pad(input=images, pad=[p, p, p, p], mode="reflect")
    images = torch.nn.functional.conv2d(input=images, weight=Hz_prime.unsqueeze(2), groups=batch_size * num_channels)
    images = torch.nn.functional.conv2d(input=images, weight=Hz_prime.unsqueeze(3), groups=batch_size * num_channels)
    return images.reshape([batch_size, num_channels, height, width])


def np_filter(x, h):
    """The spec pixel by pixel for one plane: (H x)[j] = sum_t h[t] x[R(j + t - 21)] along x, then along y."""
    H, W = x.shape
    R = lambda i, N: -i if i < 0 else (2 * (N - 1) - i if i >= N else i)
    a = np.array([[sum(h[t] * x[i, R(j + t - 21, W)] for t in range(43)) for j in range(W)] for i in range(H)])
    return np.array([[sum(h[t] * a[R(i + t - 21, H), j] for t in range(43)) for j in range(W)] for i in range(H)])


@pytest.mark.parametrize("H,W", [(22, 22), (22, 37), (40, 24)])
def test_definition_against_adas_block_and_the_pixel_by_pixel_spec(H, W):
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(H * 100 + W)
    B, C = 3, 2
    x = torch.randn(B, C, H, W, dtype=F64, generator=g)
    gains = torch.exp2(torch.randn(B, 4, dtype=F64, generator=g))
    sigma = torch.tensor([0.0, 0.05, 0.2], dtype=F64)
    noise = torch.randn(B, C, H, W, dtype=F64, generator=g)
    bank = ops.imgfilter_bank()
    got = ops.augment_filter_ref(x, gains, sigma, noise)
    want = ada_imgfilter(x, gains, bank) + noise * sigma[:, None, None, None]
    assert (got - want).abs().max() < 1e-12
    h = (gains @ bank).numpy()
    for b, c in ((0, 0), (2, 1)):
        ref = np_filter(x[b, c].numpy(), h[b]) + sigma[b].item() * noise[b, c].numpy()
        assert np.abs(got[b, c].numpy() - ref).max() < 1e-12, (b, c)


def test_identity_gains_and_zero_sigma_are_the_identity_bit_for_bit():
    ops = import_module(OPS)
    x = torch.randn(4, 3, 24, 30, dtype=F64)
    x[0, 0, 0, 0], x[1, 1, 5, 5], x[2, 2, 3, 4] = -0.0, float("inf"), float("nan")
    ones, zero = torch.ones(4, 4, dtype=F64), torch.zeros(4, dtype=F64)
    noise = torch.randn(4, 3, 24, 30, dtype=F64)
    noise[:, :, 0, 0] = float("nan")                                    # never read where sigma is 0
    for args in ((ones, None, None), (None, zero, noise), (ones, zero, noise)):
        y = ops.augment_filter_ref(x, *args)
        assert torch.equal(y.view(torch.int64), x.view(torch.int64)), [a is None for a in args]
        y = ops.augment_filter(x.float(), *args)
        assert torch.equal(y.view(torch.int32), x.float().view(torch.int32))
    assert ops.augment_filter(x) is x


@pytest.mark.parametrize("H,W", [(22, 22), (23, 40), (64, 50)])
def test_adjoint_identity(H, W):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(H + W)
    B = 6
    gains, _, _ = tr.sample_augment_filter(("imgfilter",), 1.0, B, 3, H, W, "cpu")
    gains = gains.double()
    gains[1] = 1.0
    x, gy = torch.randn(B, 3, H, W, dtype=F64), torch.randn(B, 3, H, W, dtype=F64)
    lhs = (ops.augment_filter_ref(x, gains) * gy).sum(dim=(1, 2, 3))
    rhs = (x * ops.augment_filter_adjoint_ref(gy, gains)).sum(dim=(1, 2, 3))
    assert (lhs - rhs).abs().max() < 1e-12 * max(1.0, lhs.abs().max().item())


@pytest.fixture
def host_kernels(monkeypatch):
    ops = import_module(OPS)
    calls = []

    def native(name, x, gains, sigma=None, noise=None):
        calls.append(name)
        if name == "gf_augment_filter_nchw":
            return ops.augment_filter_ref(x.detach(), gains, sigma, noise)
        return ops.augment_filter_adjoint_ref(x.detach(), gains)
    monkeypatch.setattr(ops, "_augment_filter_native", native)
    return ops, calls


@pytest.mark.parametrize("with_noise", [False, True])
def test_autograd_functions_gradcheck_and_gradgradcheck(host_kernels, with_noise):
    ops, calls = host_kernels
    g = torch.Generator().manual_seed(7)
    gains = torch.tensor([[1.3, 0.6, 1.9, 0.8], [1.0, 1.0, 1.0, 1.0]], dtype=F64)
    sigma = torch.tensor([0.1, 0.0], dtype=F64) if with_noise else None
    noise = torch.randn(2, 2, 22, 23, dtype=F64, generator=g) if with_noise else None
    x = torch.randn(2, 2, 22, 23, dtype=F64, generator=g, requires_grad=True)
    f = lambda t: ops._AugmentFilter.apply(t, gains, sigma, noise)
    assert torch.autograd.gradcheck(f, (x,))
    assert torch.autograd.gradgradcheck(f, (x,))
    assert "gf_augment_filter_adjoint_nchw" in calls
    if with_noise:                                   # noise only: the derivative is the identity
        fn = lambda t: ops._AugmentFilter.apply(t, None, sigma, noise)
        assert torch.autograd.gradcheck(fn, (x,)) and torch.autograd.gradgradcheck(fn, (x,))


def test_bad_arguments_raise():
    ops = import_module(OPS)
    x = torch.zeros(2, 3, 24, 24)
    for kw in (dict(gains=torch.ones(3, 4)), dict(gains=torch.ones(2, 3)), dict(sigma=torch.zeros(2)), dict(noise=torch.zeros(2, 3, 24, 24)),
               dict(sigma=torch.zeros(3), noise=torch.zeros(2, 3, 24, 24)), dict(sigma=torch.zeros(2), noise=torch.zeros(2, 3, 24, 23))):
        with pytest.raises(ValueError):
            ops.augment_filter(x, **kw)
    with pytest.raises(ValueError):
        ops.augment_filter(torch.zeros(2, 3, 21, 64), torch.ones(2, 4))
    with pytest.raises(ValueError):                                       # a 0-d sigma is refused like any misshaped one
        ops.augment_filter(torch.zeros(1, 3, 24, 24), None, torch.tensor(0.1), torch.zeros(1, 3, 24, 24))
    y = ops.augment_filter(torch.zeros(2, 3, 4, 4), None, torch.ones(2), torch.ones(2, 3, 4, 4))    # noise alone: any size
    assert torch.equal(y, torch.ones(2, 3, 4, 4))


# ------------------------------------------------------------------------------------------------ the sampler and the spec
def ada_sampler(p, B, C, H, W):
    """ADA's imgfilter and noise draws, restated (imgfilter = noise = 1, imgfilter_std = 1, noise_std = 0.1, every band strength 1)."""
    num_bands = 4
    expected_power = torch.tensor(np.array([10, 1, 1, 1]) / 13, dtype=torch.float32)
    g = torch.ones([B, num_bands])
    for i in range(num_bands):
        t_i = torch.exp2(torch.randn([B]) * 1.0)
        t_i = torch.where(torch.rand([B]) < p, t_i, torch.ones_like(t_i))
        t = torch.ones([B, num_bands])
        t[:, i] = t_i
        t = t / (expected_power * t.square()).sum(dim=-1, keepdims=True).sqrt()
        g = g * t
    sigma = torch.randn([B, 1, 1, 1]).abs() * 0.1
    sigma = torch.where(torch.rand([B, 1, 1, 1]) < p, sigma, torch.zeros_like(sigma))
    noise = torch.randn([B, C, H, W])
    return g, sigma.reshape(B), noise


@pytest.mark.parametrize("p", [0.0, 0.5, 1.0])
def test_sampler_against_adas_loop(p):
    tr = import_module(TRAIN)
    B, C, H, W = 4096, 3, 8, 8
    torch.manual_seed(5)
    gains, sigma, noise = tr.sample_augment_filter(tr.FILTER_OPS, p, B, C, H, W, "cpu")
    after = torch.get_rng_state()
    torch.manual_seed(5)
    ag, asg, an = ada_sampler(p, B, C, H, W)
    assert torch.equal(after, torch.get_rng_state())                     # the same draws, in the same order
    assert torch.equal(sigma, asg) and torch.equal(noise, an)
    assert (gains - ag).abs().max() < 1e-6                                # ADA's normaliser of a band that does not apply is 1 to rounding
    if p == 0.0:
        assert torch.equal(gains, torch.ones(B, 4)) and torch.equal(sigma, torch.zeros(B))
    if p == 0.5:
        torch.manual_seed(5)
        applied = []
        for _ in range(4):
            torch.randn(B)
            applied.append(torch.rand(B) < p)
        applied = torch.stack(applied, 1)
        for i in range(4):                                                # every band applies to about half the images
            assert abs(applied[:, i].double().mean().item() - 0.5) < 0.03, i
        none = ~applied.any(dim=1)                                        # no band applied: gains exactly (1, 1, 1, 1)
        assert none.any() and torch.equal(gains[none], torch.ones(int(none.sum()), 4))
        assert (gains[~none] != 1).any(dim=1).all()
        assert abs((sigma > 0).double().mean().item() - 0.5) < 0.03
    if p == 1.0:
        assert (sigma > 0).all() and abs(sigma.mean().item() - 0.1 * math.sqrt(2 / math.pi)) < 0.003


def test_no_extra_draws_without_the_new_names():
    tr = import_module(TRAIN)
    for spec in ("bc", "bgc", "xflip,hue", "scale,rotate"):
        torch.manual_seed(0)
        assert tr.sample_augment_filter(tr.parse_augment(spec), 0.7, 4, 3, 32, 32, "cpu") == (None, None, None)
        assert torch.equal(torch.get_rng_state(), torch.manual_seed(0).get_state())
    torch.manual_seed(0)
    gains, sigma, noise = tr.sample_augment_filter(("imgfilter",), 0.7, 4, 3, 32, 32, "cpu")
    assert gains is not None and sigma is None and noise is None


def test_presets():
    tr = import_module(TRAIN)
    bgc = tr.parse_augment("bgc")
    assert tr.FILTER_OPS == ("imgfilter", "noise")
    assert tr.parse_augment("bc") == tr.AUGMENT_OPS and bgc == tr.AUGMENT_OPS[:3] + tr.GEOM_OPS + tr.AUGMENT_OPS[3:]
    assert tr.parse_augment("bgcf") == bgc + ("imgfilter",)
    assert tr.parse_augment("bgcfn") == bgc + ("imgfilter", "noise")
    assert tr.parse_augment("noise, xflip,imgfilter") == ("xflip", "imgfilter", "noise")
    assert tr.parse_augment("hue,xfrac, xflip,rotate") == ("xflip", "rotate", "xfrac", "hue")
    for bad in ("bgcfnc", "noise,cutout", "cutout"):
        with pytest.raises(ValueError):
            tr.parse_augment(bad)


_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A, Y = 0x10000, 0x40000000
out = []
fn = lib.gf_augment_filter_nchw
for args in ([A, Y, A, A, A, 2, 3, 32, 32, None], [A, Y, None, None, None, 2, 3, 8, 8, None],
             [None, Y, A, A, A, 2, 3, 32, 32, None], [A, None, A, A, A, 2, 3, 32, 32, None], [A, Y, A, A, None, 2, 3, 32, 32, None],
             [A, Y, A, None, A, 2, 3, 32, 32, None], [A, Y, A, A, A, 0, 3, 32, 32, None], [A, Y, A, A, A, 2, 3, 21, 32, None],
             [A, Y, A, A, A, 2, 3, 32, 40000, None], [A, A + 64, A, A, A, 2, 3, 32, 32, None], [A, Y, None, None, None, 2, 3, 32, 21, None]):
    out.append(["gf_augment_filter_nchw", fn(*args), lib.gf_last_error().decode()])
fn = lib.gf_augment_filter_adjoint_nchw
for args in ([A, Y, A, 2, 3, 32, 32, None], [A, Y, None, 2, 3, 32, 32, None], [None, Y, A, 2, 3, 32, 32, None],
             [A, Y, A, 2, -1, 32, 32, None], [A, Y, A, 2, 3, 32, 21, None], [A, Y, A, 2, 3, 40000, 32, None], [A, A, A, 2, 3, 32, 32, None]):
    out.append(["gf_augment_filter_adjoint_nchw", fn(*args), lib.gf_last_error().decode()])
print(json.dumps(out))
"""


def test_entry_points_refuse_bad_arguments():
    """Refusals come before the device is touched; a valid call reaches the launch, which fails without a GPU (-3)."""
    gf = import_module("gansformer_b200")
    assert {"gf_augment_filter_nchw", "gf_augment_filter_adjoint_nchw"} <= set(gf._lib.OPS_EXPORTS)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    fwd = [(rc, msg) for n, rc, msg in out if n == "gf_augment_filter_nchw"]
    adj = [(rc, msg) for n, rc, msg in out if n == "gf_augment_filter_adjoint_nchw"]
    assert [rc for rc, _ in fwd] == [-3, -3, -1, -1, -1, -1, -1, -2, -2, -1, -3], fwd
    assert [rc for rc, _ in adj] == [-3, -1, -1, -1, -2, -2, -1], adj
    assert all(n in msg for n, rc, msg in out if rc != -3)
    assert "sigma and noise" in fwd[4][1] and "alias" in fwd[9][1] and "22" in fwd[7][1] and "alias" in adj[6][1]


# ------------------------------------------------------------------------------------------------ training
def test_trainer_bgcfn_with_r1(gf):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(32, fmap_base=256, fmap_max=32)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", d_reg_interval=2, augment="bgcfn", augment_p=0.8, ada_target=0.6,
                                              ada_interval=1))
    g = torch.Generator().manual_seed(3)
    z, reals = torch.randn(4, 5, 16, generator=g), torch.rand(4, 3, 32, 32, generator=g) * 2 - 1
    seen, filtered = [], []
    d_fwd = D.forward
    D.forward = lambda img, c=None: seen.append(img) or d_fwd(img)
    orig = tr.augment_filter
    tr.augment_filter = lambda *a: filtered.append(a) or orig(*a)
    try:
        stats = [trainer.step(z, reals) for _ in range(2)]
    finally:
        tr.augment_filter = orig
    assert stats[0].r1 > 0 and stats[1].r1 == 0
    assert all(math.isfinite(v) for s in stats for v in (s.loss_d, s.loss_g, s.r1, s.augment_p))
    assert len(seen) == 6 and seen[0].requires_grad and torch.isfinite(seen[0]).all()
    assert len(filtered) == 6 and all(a[1] is not None and a[2] is not None and a[3] is not None for a in filtered)


def test_trainer_filter_only_spec_skips_the_blit(gf):
    """A spec with only the new names draws and applies the filter alone; the bgc part draws nothing."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(32, fmap_base=256, fmap_max=32)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", augment="noise", augment_p=1.0))
    img = torch.rand(3, 3, 32, 32) * 2 - 1
    torch.manual_seed(1)
    got = trainer._augment(img)
    torch.manual_seed(1)
    _, sigma, noise = tr.sample_augment_filter(("noise",), 1.0, 3, 3, 32, 32, "cpu")
    assert torch.equal(got, img + sigma[:, None, None, None] * noise)


def test_trainer_refuses_imgfilter_below_22(gf):
    """The filter's size limit is checked when the trainer is built, not on the first (possibly captured) step; noise alone has none."""
    tr = import_module(TRAIN)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32)
    for spec in ("bgcf", "imgfilter", "xflip,imgfilter,noise"):
        with pytest.raises(ValueError, match="22x22"):
            tr.Trainer(G, D, tr.TrainConfig(augment=spec))
    tr.Trainer(G, D, tr.TrainConfig(augment="noise"))
