"""CPU checks of oracle/augment_resample.py, the fp32 restatement of ADA's fractional resampler (DESIGN 4.12) that
tests/test_gpu_augment_resample_exact.py holds both kernels to bit for bit.

* fma32 against exact rational arithmetic, on random triples and on constructed ties.
* On maps whose sample positions are exact, the restated forward and adjoint agree with the fp64 definition (ops.resample_ref with
  the same fp32 taps) within gamma_n times the magnitude companion, n the longest chain of roundings counted from the kernels.
* The restated forward and adjoint satisfy the adjoint identity to rounding.
* The plan really is chosen: a case with tiles on both forward paths, an adjoint case in several chunks.
"""
import math
import random
from fractions import Fraction
from importlib import import_module

import numpy as np
import pytest
import torch

from oracle import augment_resample as oar

OPS = "gansformer-reproducibility-challenge_b200.ops"
F64 = torch.float64
U32, U64 = 2.0 ** -24, 2.0 ** -53


def gamma(n, u):
    return n * u / (1 - n * u)


def round_fp32(v: Fraction) -> float:
    """v rounded to the nearest fp32 value, ties to even (normal range)."""
    if v == 0:
        return 0.0
    s, a = (-1 if v < 0 else 1), abs(v)
    e = math.floor(math.log2(a.numerator) - math.log2(a.denominator)) - 23
    while a / Fraction(2) ** e >= 2 ** 24:
        e += 1
    while a / Fraction(2) ** e < 2 ** 23:
        e -= 1
    q = a / Fraction(2) ** e
    n = math.floor(q)
    r = q - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return s * float(Fraction(n) * Fraction(2) ** e)


def exact_fma(a, b, c):
    return np.float32(round_fp32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))))


# ------------------------------------------------------------------------------------------------ fma32
def test_fma32_on_random_triples():
    rng = random.Random(1)
    a, b, c = [], [], []
    for _ in range(4000):
        ea, eb = rng.randint(-20, 20), rng.randint(-20, 20)
        a.append(np.float32(rng.uniform(-2, 2) * 2.0 ** ea))
        b.append(np.float32(rng.uniform(-2, 2) * 2.0 ** eb))
        # c near -a b half of the time: heavy cancellation
        c.append(np.float32(-float(a[-1]) * float(b[-1]) * (1 + rng.uniform(-1e-6, 1e-6))) if rng.random() < 0.5 else
                 np.float32(rng.uniform(-2, 2) * 2.0 ** (ea + eb + rng.randint(-30, 30))))
    got = oar.fma32(np.array(a), np.array(b), np.array(c))
    want = np.array([exact_fma(*t) for t in zip(a, b, c)], np.float32)
    assert np.array_equal(got, want)


def test_fma32_on_ties():
    """a b + c exactly on an fp32 midpoint (ties to even) and a hair beside one, below fp64's resolution of the sum: there the fp64
    sum rounds onto the midpoint and only the TwoSum error says which way the fp32 result must go."""
    one = np.float32(1)
    odd = np.float32(1 + 2.0 ** -23)                       # the midpoint above it, 1 + 3 2^-24, rounds to even: up
    lo, hi = np.float32(2.0 ** -12 * (1 + 2.0 ** -23)), np.float32(2.0 ** -12 * (1 - 2.0 ** -23))
    cases = [(np.float32(2.0 ** -12), np.float32(2.0 ** -12), one),       # 1 + 2^-24: tie, to even (1)
             (np.float32(2.0 ** -12), np.float32(2.0 ** -12), odd),       # tie, to even (1 + 2^-22)
             (lo, hi, odd),                                               # midpoint - 2^-70: down to odd
             (lo, hi, one)]                                               # 1 + 2^-24 - 2^-70: down to 1
    more = []
    for a, b, c in cases:
        for k in (-40, 0, 17):
            s = np.float32(2.0 ** k)
            more += [(a * s, b, c * s), (-a * s, b, -c * s), (a, -b * s, -c * s)]   # scaled, and negated (TwoSum error > 0)
    for a, b, c in cases + more:
        assert oar.fma32(a, b, c) == exact_fma(a, b, c), (a, b, c)
    assert oar.fma32(lo, hi, odd) == odd and np.float32(float(lo) * float(hi) + float(odd)) != odd


# ------------------------------------------------------------------------------------------------ against the definition
def definition(ops, x, geom, frac, color, gy):
    """(forward, adjoint, forward companion, adjoint companion) of the fp64 definition with the kernels' fp32 taps."""
    B = x.shape[0]
    taps = torch.from_numpy(oar.TAPS.astype(np.float64))
    fwd = ops.resample_ref(x, geom, frac, taps)
    comp = ops.resample_ref(x.abs(), geom, frac, taps.abs())
    g, ga = gy, gy.abs()
    if color is not None:
        M = color.reshape(B, 3, 4)
        fwd = torch.einsum("bij,bjhw->bihw", M[:, :, :3], fwd) + M[:, :, 3, None, None]
        comp = torch.einsum("bij,bjhw->bihw", M[:, :, :3].abs(), comp) + M[:, :, 3, None, None].abs()
        g, ga = (torch.einsum("bij,bihw->bjhw", m, t) for m, t in ((M[:, :, :3], gy), (M[:, :, :3].abs(), gy.abs())))
    x0 = torch.zeros_like(x).requires_grad_(True)
    (adj,) = torch.autograd.grad(ops.resample_ref(x0, geom, frac, taps), x0, g)
    (cadj,) = torch.autograd.grad(ops.resample_ref(x0, geom, frac, taps.abs()), x0, ga)
    return fwd, adj, comp, cadj


# The longest chain of fp32 roundings any term goes through (csrc/gf_augment.cu): forward, shared-memory plan 6 + 6 (up filter)
# + 4 (bilinear) + 12 + 12 (down filter) + 3 (colour) = 43; direct path 2 + 7 + 2 + 7 (weights and taps) + 24 + 3 = 45.  Adjoint
# 3 (colour) + 6 + 6 (transposed down filter) + 1 (round(wy wx)) + K (the in-order chain of one nu in one chunk) + A (chunk adds)
# + 12 + 12 (transposed up filter) + 9 (copies) = 49 + K + A, K and A counted by the oracle.
N_FWD = 45
CASES = {   # maps with exact sample positions: name -> (B, C, H, W, frac rows, geom rows, colour)
    "zoom-out 8 (direct path)": (2, 1, 24, 20, [[8, 0, 0.5, 0, 8, -0.25]] * 2, [[0, 0, 0, 0], [3, 2, -1, 0]], False),
    "zoom-in 8 (many chunks)": (1, 1, 64, 64, [[0.125, 0, 0.5, 0, 0.125, -0.25]], [[0, 0, 0, 0]], False),
    "zoom-out 3.75 (both paths)": (1, 3, 48, 48, [[3.75, 0, 0.25, 0, 3.75, -0.25]], [[0, 0, 0, 0]], True),
    "parallelograms": (3, 3, 20, 18, [[1, 1, 0.5, -1, 1, -0.25], [0.75, 0.5, -0.25, 0.5, 1, 0.5], [1, 1, 0, 1, -1, 0.125]],
                       [[1, 3, -2, 0], [4, -1, 5, 0], [5, 0, 1, 0]], True),
    "tiny": (2, 2, 3, 2, [[0.5, 0, 0.25, 0, 2, 0], [1, 0.5, 0, -0.5, 1, 0.5]], [[1, 1, 0, 0], [2, 0, -1, 0]], False),
}


def _case(name):
    B, C, H, W, rows, grows, colour = CASES[name]
    g = torch.Generator().manual_seed(len(name))
    x = torch.randn(B, C, H, W, generator=g).float().double()
    gy = torch.randn(B, C, H, W, generator=g).float().double()
    color = torch.randn(B, 12, generator=g).float().double() if colour else None
    return x, gy, torch.tensor(grows, dtype=torch.int32), torch.tensor(rows, dtype=F64), color


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_against_the_definition_on_exact_positions(name):
    ops = import_module(OPS)
    x, gy, geom, frac, color = _case(name)
    B, C, H, W = x.shape
    # the positions are exact: the fp32 nu of every 2x output point equals the fp64 one
    nx32, ny32 = oar.positions(geom, frac, H, W, check=True)
    L, e = ops.resample_map(geom, frac, H, W)
    qx, qy = torch.arange(1, 2 * W + 11, dtype=F64)[None, None, :], torch.arange(1, 2 * H + 11, dtype=F64)[None, :, None]
    assert np.array_equal(nx32, (L[:, 0, 0, None, None] * qx + L[:, 0, 1, None, None] * qy + e[:, 0, None, None]).numpy())
    assert np.array_equal(ny32, (L[:, 1, 0, None, None] * qx + L[:, 1, 1, None, None] * qy + e[:, 1, None, None]).numpy())
    fs, as_ = {}, {}
    y = torch.from_numpy(oar.forward(x, geom, frac, color, stats=fs)).double()
    a = torch.from_numpy(oar.adjoint(gy, geom, frac, color, stats=as_)).double()
    fwd, adj, comp, cadj = definition(ops, x, geom, frac, color, gy)
    n_adj = 49 + as_["chain"] + as_["chunk_adds"]
    for what, got, want, c, n in (("forward", y, fwd, comp, N_FWD), ("adjoint", a, adj, cadj, n_adj)):
        bound = (gamma(n, U32) + gamma(n, U64)) * c
        err = (got - want).abs()
        print(f"[resample oracle] {name} {what}: max |err| / bound = {(err / bound.clamp(min=1e-300)).max().item():.3f} (n = {n})")
        assert (err <= bound).all(), (name, what)
    assert as_["dropped"] == 0                       # every nonzero tap lies inside the kernel's preimage box
    if "direct" in name:
        assert fs["direct"] > 0
    if "both" in name:
        assert fs["plan"] > 0 and fs["direct"] > 0
    if "chunks" in name:
        assert as_["chunks"] > 1 and as_["chunk_adds"] > 1, as_


@pytest.mark.parametrize("name", ["zoom-out 3.75 (both paths)", "parallelograms", "bgc 16x16"])
def test_oracle_adjoint_identity(name):
    """<A x, g> = <x, A^T g> for the restated kernels, to gamma_n <|A| |x|, |g|>; the "bgc" case has inexact fp32 positions (both
    kernels compute the same fp32 nu(q), so they restate the same linear map), its |A| taken at those positions."""
    ops = import_module(OPS)
    if name.startswith("bgc"):
        tr = import_module("gansformer-reproducibility-challenge_b200.training")
        torch.manual_seed(12)
        B, H, W = 4, 16, 16
        geom, _ = tr.sample_augment(tr.parse_augment("bgc"), 1.0, B, H, W, "cpu")
        frac = tr.sample_augment_frac(tr.parse_augment("bgc"), 1.0, B, H, W, "cpu").double()
        frac[:, [0, 1, 3, 4]] = torch.round(frac[:, [0, 1, 3, 4]] * 256) / 256
        g = torch.Generator().manual_seed(13)
        x, gy = (torch.randn(B, 3, H, W, generator=g).float().double() for _ in range(2))
        color = None
    else:
        x, gy, geom, frac, color = _case(name)
    if color is not None:
        color = torch.cat([color.reshape(-1, 3, 4)[:, :, :3], torch.zeros(color.shape[0], 3, 1, dtype=F64)], 2).reshape(-1, 12)
    B, C, H, W = x.shape
    st = {}
    y = torch.from_numpy(oar.forward(x, geom, frac, color)).double()
    a = torch.from_numpy(oar.adjoint(gy, geom, frac, color, stats=st)).double()
    nx, ny = oar.positions(geom, frac, H, W, check=True)
    comp = oar.forward64_at(x.abs(), nx, ny, np.abs(oar.TAPS.astype(np.float64)))
    if color is not None:
        comp = torch.einsum("bij,bjhw->bihw", color.reshape(B, 3, 4)[:, :, :3].abs(), comp)
    lhs, rhs = (y * gy).sum(dim=(1, 2, 3)), (x * a).sum(dim=(1, 2, 3))
    scale = (comp * gy.abs()).sum(dim=(1, 2, 3))
    n = N_FWD + 49 + st["chain"] + st["chunk_adds"]
    rel = ((lhs - rhs).abs() / scale).max().item()
    print(f"[resample oracle] adjoint identity {name}: {rel:.3e} of <|A||x|, |g|>, bound {gamma(n, U32) + gamma(n, U64):.3e}")
    assert rel <= gamma(n, U32) + gamma(n, U64)


def test_res_map_refuses_inexact_products():
    """The host check that makes the result independent of nvcc's contractions: an entry with 20 significant bits squares to 40."""
    with pytest.raises(oar.InexactMap):
        oar.ResMap(np.array([1 + 2.0 ** -19, 0.3, 0, 0, 1, 0], np.float32), [0, 0, 0, 0], 16, 16, check=True)
    m = oar.ResMap(np.array([1 + 2.0 ** -19, 0.3, 0, 0, 1, 0], np.float32), [0, 0, 0, 0], 16, 16, check=False)
    assert not m.exact
