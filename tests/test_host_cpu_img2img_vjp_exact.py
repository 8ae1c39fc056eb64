"""The exact cases and the TF32-faithful restatement of the image self-attention double backward, without a GPU (DESIGN 4.14).

* Every tied case of tests/test_gpu_img2img_vjp_exact.py is proved exact for gf_self_attn_bwd_vjp, element by element
  (oracle.self_attention_exact.prove_vjp_exact), and covers what it is there for: at d = 64 non-zero GdP and GS, rows with r != 0
  and with Delta r != 0, and staged GS (and, with uniform rows at n = 256, staged GdP) whose RNE and truncation to TF32 differ.
* At d = 32 the scale fp32(1 / sqrt(32)) is not a power of two: with A and Bk the proof fails at gds, so those cases carry Cv alone.
* The exact reference and the restatement without their roundings are oracle.self_attention_vjp; with them, the restatement
  gives the exact reference's bits on the tied cases.
"""
import pytest
import torch

from oracle import self_attention as osa
from oracle import self_attention_exact as sx
from oracle import self_attention_vjp as ov
from tests.test_gpu_img2img_exact import TIED


@pytest.mark.parametrize("B,n,C,d", TIED)
def test_tied_case_is_exact(B, n, C, d):
    case = sx.vjp_tied_case(B, n, C, d, seed=B + n + C + d)
    st = sx.prove_vjp_exact(case)
    assert st["gs_nonzero"] > 0, st
    if d == 64:
        assert st["gdp_nonzero"] > 0 and st["r_rows"] > 0 and st["delta_r_rows"] > 0 and st["gs_rne_ne_trunc"] > 0, st
        assert (case["a"] != 0).any() and (case["bk"] != 0).any()
    else:
        assert not case["a"].any() and not case["bk"].any()
    if n == 256:
        assert st["gdp_rne_ne_trunc"] > 0, st


def test_d32_cotangents_a_and_bk_are_not_exact():
    """gds = fp32(GdS / s) * fp32(1 / sqrt(32)) is rounded, and the kernels' FMA contractions then decide its later bits."""
    case = sx.vjp_tied_case(1, 64, 32, 32, seed=3, ab=True)
    with pytest.raises(AssertionError, match="gds"):
        sx.prove_vjp_exact(case)


@pytest.mark.parametrize("B,n,C,d", [c for c in TIED if c[1] <= 1024])
def test_restatement_is_exact_on_tied_cases(B, n, C, d):
    case = sx.vjp_tied_case(B, n, C, d, seed=B + n + C + d)
    ins = [case[x] for x in ("q", "k", "v", "do", "a", "bk", "cv")]
    h = case["heads"]
    _, lse, delta, *_ = sx.exact_reference(*ins[:4], h)
    want = sx.vjp_exact_reference(*ins, h)
    for name, a, b in zip(("gQ", "gK", "gV", "gdO", "r", "t"), sx.vjp(*ins, lse, delta, h), want):
        assert torch.equal(a.float(), b), name


@pytest.mark.parametrize("n,C", [(64, 32), (192, 64), (128, 256)])
def test_without_roundings_is_the_oracle(n, C):
    g = torch.Generator().manual_seed(n + C)
    ins = [torch.randn(2, n, C, generator=g, dtype=torch.float64) * s for s in (2, 2, 1, 1, 1, 1, 1)]
    h = osa.heads_of(C)
    want = ov.vjp(*ins, h)
    ref = sx.vjp_exact_reference(*ins, h, rounded=False)
    o, lse = sx.forward(*ins[:3], h, rounded=False)
    delta = (sx._heads(o, h) * sx._heads(ins[3], h)).sum(dim=3)
    rest = sx.vjp(*ins, lse, delta, h, rounded=False)
    for name, w, a, b in zip(("gQ", "gK", "gV", "gdO"), want, ref, rest):
        assert torch.allclose(a, w, rtol=1e-12, atol=1e-12), (name, (a - w).abs().max().item())
        assert torch.allclose(b, w, rtol=1e-12, atol=1e-12), (name, (b - w).abs().max().item())
    for name, a, b in zip(("r", "t"), ref[4:], rest[4:]):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-12), (name, (a - b).abs().max().item())


def test_restatement_roundings():
    """The rounded restatement differs from the plain one by TF32-level amounts, and each of its outputs is an fp32 value."""
    g = torch.Generator().manual_seed(9)
    ins = [torch.randn(1, 128, 64, generator=g) for _ in range(7)]
    o, lse = sx.forward(*ins[:3], 1)
    delta =(sx._heads(o, 1) * sx._heads(ins[3].double(), 1)).sum(dim=3).float().double()
    got = sx.vjp(*ins, lse, delta, 1)
    plain = sx.vjp(*ins, lse, delta, 1, rounded=False)
    for name, a, b in zip(("gQ", "gK", "gV", "gdO", "r", "t"), got, plain):
        err = ((a - b).abs().max() / b.abs().max()).item()
        assert 1e-6 < err < 3e-2 and torch.equal(a, a.float().double()), (name, err)
