"""The image self-attention double backward on an H100, exactly (``pytest -m gpu``; DESIGN 4.14).

gf_self_attn_bwd_vjp through the C ABI, every output (gQ, gK, gV, gdO and the row statistics r, t) between NaN guards, checked
for writes outside it and for elements left unwritten; lse and Delta come from the kernels' own forward and backward.
* Tied cases (oracle/self_attention_exact.py: vjp_tied_case, proved exact by tests/test_host_cpu_img2img_vjp_exact.py): ties of 1,
  2 and 4 keys with integer cotangents that differ across the winners of a tie, so that r, u, GdP, GS, gQ, gK and gV are not zero
  (d = 64; at d = 32 the cotangent is Cv alone).  All six outputs equal the float64 algebra with the kernels' roundings bit for
  bit, after lse and Delta have been checked against the first order's exact reference.
* One cotangent at a time on N(0, 1) inputs: outputs whose reference is identically zero are 0 as values; the Cv-only gdO is the
  row pass's P Cv with exactly 0 added, as the bit-level sums against the A-and-Bk run show; every other output is held to the
  TF32-faithful restatement under its own bound.
* N(0, 1) and peaked inputs (Q and K times 3: P nearly one-hot, GdS - r cancelling) against the restatement, every output
  compared, under bounds frozen from a logged run.
"""
from importlib import import_module

import pytest
import torch

from oracle import self_attention_exact as sx
from tests.guards import assert_exact
from tests.test_gpu_img2img_exact import TIED
from tests.test_gpu_img2img_vjp import SA, call_vjp

pytestmark = pytest.mark.gpu

OUTS = ("gQ", "gK", "gV", "gdO", "r", "t")

# Worst cases over test_against_restatement (max error over max |reference|, per output), measured on an NVIDIA H100 80GB HBM3
# at a 700 W power limit (1980 MHz maximum SM clock), frozen at about 3x (DESIGN 4.14):
#   N(0, 1)  gQ 2.96e-4, gK 3.68e-4, gV 2.71e-4, gdO 2.55e-4, r 1.17e-6, t 1.65e-4
#   peaked   gQ 5.20e-4, gK 7.20e-4, gV 5.42e-4, gdO 6.87e-4, r 1.35e-5, t 5.91e-5
RESTATED_BOUNDS = {
    "normal": {"gQ": 9e-4, "gK": 1.1e-3, "gV": 8e-4, "gdO": 8e-4, "r": 4e-6, "t": 5e-4},
    "peaked": {"gQ": 1.6e-3, "gK": 2.2e-3, "gV": 1.6e-3, "gdO": 2.1e-3, "r": 4e-5, "t": 1.8e-4},
}
# Worst cases over test_one_cotangent_at_a_time, same card, same measure, frozen at about 3x.  (output, cotangent) pairs whose
# reference is identically zero are not here: they are compared as values.  Measured:
#   a   gQ 1.61e-4, gK 1.34e-4, gV 1.44e-4, gdO 1.16e-4, r 7.39e-7, t 1.24e-6
#   bk  gQ 3.06e-4, gK 4.57e-4, gV 2.41e-4, gdO 1.89e-4, r 1.11e-6, t 1.11e-6
#   cv  gQ 2.29e-4, gK 3.76e-4, gdO 7.84e-5, t 8.52e-5
ONE_BOUNDS = {
    "a": {"gQ": 5e-4, "gK": 4e-4, "gV": 4.5e-4, "gdO": 3.5e-4, "r": 2.2e-6, "t": 3.7e-6},
    "bk": {"gQ": 9e-4, "gK": 1.4e-3, "gV": 7e-4, "gdO": 6e-4, "r": 3.3e-6, "t": 3.3e-6},
    "cv": {"gQ": 7e-4, "gK": 1.1e-3, "gdO": 2.4e-4, "t": 2.6e-4},
}
ZERO = {"none": OUTS, "a": (), "bk": (), "cv": ("r", "gV")}


def _first_order(q, k, v, do, heads):
    sa = import_module(SA)
    o, lse = sa.attention_fwd_native(q, k, v, heads)
    *_, delta = sa._attention_bwd(q, k, v, o, lse, do, heads)
    return lse, delta


def _rel(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("B,n,C,d", TIED)
def test_tied_cases_exact(gf, cuda_dev, B, n, C, d):
    case = sx.vjp_tied_case(B, n, C, d, seed=B + n + C + d)
    h = case["heads"]
    ins = [case[x].to(cuda_dev) for x in ("q", "k", "v", "do", "a", "bk", "cv")]
    q, k, v, do, a, bk, cv = ins
    lse, delta = _first_order(q, k, v, do, h)
    _, lse_x, delta_x, *_ = sx.exact_reference(q, k, v, do, h)
    assert_exact(lse, lse_x, f"lse (B={B} n={n} C={C} d={d})")
    assert_exact(delta, delta_x, f"Delta (B={B} n={n} C={C} d={d})")
    got = call_vjp(gf, q, k, v, do, lse, delta, a, bk, cv, h, cuda_dev)
    want = sx.vjp_exact_reference(*ins, h)
    for name, w in zip(OUTS, want):
        assert_exact(got[name], w, f"{name} (B={B} n={n} C={C} d={d})")
    for name in ("gQ", "gK", "gdO", "t") + (("gV", "r") if d == 64 else ()):
        assert (got[name] != 0).any(), name


def _normal(B, n, C, seed, dev, peaked=False):
    g = torch.Generator().manual_seed(seed)
    ins = [torch.randn(B, n, C, generator=g) for _ in range(7)]
    if peaked:
        ins[0], ins[1] = ins[0] * 3, ins[1] * 3
    return [t.to(dev) for t in ins]


@pytest.mark.parametrize("B,n,C,d", [(2, 256, 128, 64), (3, 192, 32, 32), (1, 1024, 64, 64), (1, 1024, 128, 32)])
def test_one_cotangent_at_a_time(gf, cuda_dev, B, n, C, d):
    h = C // d
    q, k, v, do, a, bk, cv = _normal(B, n, C, 3 * n + C + d + B, cuda_dev)
    lse, delta = _first_order(q, k, v, do, h)
    zero = torch.zeros_like(a)
    cots = {"none": (zero, zero, zero), "a": (a, zero, zero), "bk": (zero, bk, zero), "cv": (zero, zero, cv),
            "a+bk": (a, bk, zero), "all": (a, bk, cv)}
    got = {c: call_vjp(gf, q, k, v, do, lse, delta, *x, h, cuda_dev) for c, x in cots.items()}
    for c, names in ZERO.items():
        for name in names:
            assert_exact(got[c][name], torch.zeros_like(got[c][name]), f"{name} with cotangent {c} (B={B} n={n} C={C} d={d})")
    # gdO = GdP V + PC, r and GdP do not depend on Cv, and t = (u - 2 Delta r) + dO . PC: the Cv-only run adds exactly 0 to P Cv
    full, ab, c_ = got["all"], got["a+bk"], got["cv"]
    assert_exact(full["gdO"], ab["gdO"] + c_["gdO"], "gdO = gdO(A, Bk) + gdO(Cv)")
    assert_exact(full["t"], ab["t"] + c_["t"], "t = t(A, Bk) + t(Cv)")
    assert_exact(full["r"], ab["r"], "r")
    assert_exact(full["gV"], ab["gV"], "gV")
    errs = {}
    for c, bounds in ONE_BOUNDS.items():
        want = dict(zip(OUTS, sx.vjp(q, k, v, do, *cots[c], lse, delta, h)))
        errs[c] = {name: _rel(got[c][name], want[name]) for name in bounds}
    print(f"[img2img vjp one cotangent] B={B} n={n} C={C} d={d} "
          + " ".join(f"{c}:" + ",".join(f"{x}={e:.2e}" for x, e in es.items()) for c, es in errs.items()))
    for c, es in errs.items():
        assert all(es[x] <= ONE_BOUNDS[c][x] for x in es), (c, es)


@pytest.mark.parametrize("kind", ["normal", "peaked"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("h", [1, 4])
@pytest.mark.parametrize("d", [32, 64])
@pytest.mark.parametrize("n", [64, 192, 256, 1024, 4096])
def test_against_restatement(gf, cuda_dev, n, d, h, B, kind):
    """The kernels against their own roundings restated in float64, r and t included."""
    ins = _normal(B, n, h * d, 11 * n + d + 5 * h + B + (kind == "peaked"), cuda_dev, peaked=kind == "peaked")
    q, k, v, do = ins[:4]
    lse, delta = _first_order(q, k, v, do, h)
    got = call_vjp(gf, q, k, v, do, lse, delta, *ins[4:], h, cuda_dev)
    want = sx.vjp(q, k, v, do, *ins[4:], lse, delta, h)
    errs = {name: _rel(got[name], w) for name, w in zip(OUTS, want)}
    print(f"[img2img vjp restated] {kind} n={n} d={d} h={h} B={B} " + " ".join(f"{k_}={v_:.3e}" for k_, v_ in errs.items()))
    assert all(errs[x] <= RESTATED_BOUNDS[kind][x] for x in errs), errs
