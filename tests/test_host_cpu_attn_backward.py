"""CPU checks behind tests/test_gpu_attn_backward.py: the dropout form of the folded oracle, and the exactness of every exact case.

The GPU tests demand bit-for-bit equality on their exact cases.  That is only a fair demand if every probability the kernels form
is 0, 1/2 or 1 and every intermediate is an fp32 value whatever the order of summation.  These tests build each exact case on the
host and check it: every partial sum of an intermediate is a multiple of its grain with a magnitude below 2^24 grains (the
companion bounds every partial sum), and the fp64 reference's outputs round-trip through float32 unchanged.
"""
import math

import pytest
import torch

from oracle import attn_bwd as ab
from oracle import bipartite as ob
from oracle import folded as of
from oracle import philox as ph
from tests.test_gpu_attn_backward import EXACT_A, EXACT_T, place_winners, split_ranges


def _check_exact(items):
    for name, value, comp, grain in items:
        fin = torch.isfinite(value)
        v, c = value[fin] / grain, comp.expand_as(value)[fin] / grain
        assert torch.equal(v.round(), v), f"{name}: not a multiple of {grain}"
        assert (c < 2.0 ** 24).all(), f"{name}: a partial sum may reach {c.max().item() * grain:.3g} ({c.max().item():.3g} grains)"


def _roundtrips(outs):
    for name, t in outs.items():
        fin = torch.isfinite(t)
        assert torch.equal(t[fin].float().double(), t[fin]), f"{name}: not an fp32 value"


def test_per_token_with_dropout_equals_the_direct_oracle():
    """folded.per_token(att_mult, cb) after fold_weights / prologue equals bipartite.transformer_layer(att_mult) in fp64, for the
    three integrations, with k padded to KP and with layer norm and none."""
    D, p, H, W, B = 16, 16, 4, 8, 2
    for C, k, integration, norm in ((32, 5, "mul", "layer"), (64, 16, "both", None), (32, 20, "add", "layer")):
        w = ob.init_params(C, D, k, p, integration, False, seed=k, bias_std=0.4)
        g = torch.Generator().manual_seed(C + k)
        x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
        y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
        KP = of.pad_k(k)
        mult = torch.from_numpy(ph.dropout_mult(0.3, 99, 4, 2, B * H * W, KP).reshape(B, H * W, KP).copy()).double()
        ref, _, _ = ob.transformer_layer(x, y, w, integration=integration, norm=norm, att_mult=mult[:, :, :k])
        f = of.fold_weights(w, C=C, k=k, integration=integration, duplex=False)
        Kp, Vt, Rt, Ct = of.prologue(y, f, C=C, H=H, W=W, p=p)
        cb = f["CV"] - w["bv"] @ of._e(w["wo"])
        X = x.permute(0, 2, 3, 1).reshape(B, H * W, C)
        out, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm, att_mult=mult, cb=cb)
        assert (out - ref.permute(0, 2, 3, 1).reshape(B, H * W, C)).abs().max() < 1e-10
        plain, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm)
        ones, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm, att_mult=torch.ones_like(mult), cb=cb)
        assert (ones - plain).abs().max() < 1e-10 and (out - plain).abs().max() > 1e-3


def test_centroid_softmax_is_the_pass_a_of_the_oracle():
    """centroid_softmax: columns of A sum to 1 over the tokens, Xbar = A^T X, lse = log sum exp of the logits; padded latents unused."""
    g = torch.Generator().manual_seed(3)
    B, H, W, C, k = 2, 5, 6, 32, 3
    X = torch.randn(B, H * W, C, generator=g, dtype=torch.float64)
    M = torch.randn(B, 16, C, generator=g, dtype=torch.float64)
    Rt2, Ct2 = torch.randn(B, H, 16, generator=g, dtype=torch.float64), torch.randn(B, W, 16, generator=g, dtype=torch.float64)
    Rt2[:, :, k:] = -math.inf
    A, xbar, lse = of.centroid_softmax(X, M, Rt2, Ct2, k=k)
    L = X @ M[:, :k].transpose(1, 2) + (Rt2[:, :, None, :k] + Ct2[:, None, :, :k]).reshape(B, H * W, k)
    assert torch.allclose(A.sum(dim=1), torch.ones(B, k, dtype=torch.float64))
    assert torch.allclose(xbar, A.transpose(1, 2) @ X) and torch.allclose(lse, torch.log(torch.exp(L).sum(dim=1)))


def test_pass_a_reference_with_r_equal_to_the_true_one_is_the_gradient():
    """centroid_backward with r = dXbar . Xbar is the plain gradient of <dXbar, Xbar>."""
    case = ab.random_centroid_case(2, 6, 7, 32, 5, mean=0.0, seed=1)
    args = (case["X"], case["M"], case["Rt2"], case["Ct2"])
    got = ab.centroid_backward(*args, case["dXbar"], case["r"], torch.zeros_like(case["X"]), k=5)
    X = case["X"].clone().requires_grad_(True)
    _, xbar, _ = of.centroid_softmax(X, case["M"], case["Rt2"], case["Ct2"], k=5)
    (case["dXbar"] * xbar).sum().backward()
    assert torch.allclose(got["dX"], X.grad, atol=1e-12)


@pytest.mark.parametrize("B,H,W,C,k,integration,dropout", EXACT_T, ids=str)
def test_stage_t_exact_case_is_exact(B, H, W, C, k, integration, dropout):
    case = ab.exact_stage_t_case(B, H, W, C, k, integration, dropout=dropout, seed=B * 1000 + C + k)
    args = (case["X"], case["dOut"], case["Kp"], case["Vt"], case["Rt"], case["Ct"])
    items, p = ab.stage_t_exactness(*args, k=k, integration=integration, mult=case["mult"], cb=case["cb"])
    assert set(p.unique().tolist()) <= {0.0, 0.5, 1.0}
    assert (p == 1.0).any() and ((p == 0.5).any() or k == 1)
    if dropout:
        assert set(case["mult"].unique().tolist()) == {0.0, 2.0}
    _check_exact(items)
    want = ab.stage_t_backward(*args, H=H, W=W, integration=integration, norm="none", mult=case["mult"], cb=case["cb"])
    _roundtrips(want)
    named = dict((n, v) for n, v, _, _ in items)                        # the explicit restatement agrees with autograd
    assert torch.equal(want["dX"], named["dX"]) and torch.equal(want["dCtl"], named["dCtl"])
    assert torch.equal(want["dS"][:, :, :k], named["dS"][:, :, :k]) and torch.equal(want["P"][:, :, :k], named["q"][:, :, :k])


@pytest.mark.parametrize("B,H,W,C,k", EXACT_A, ids=str)
def test_pass_a_exact_case_is_exact(B, H, W, C, k):
    n = H * W
    ranges = split_ranges(n, 16)
    case = ab.exact_centroid_case(B, H, W, C, k, winners=place_winners(B, n, k, ranges, seed=C + k), seed=B * 100 + C + k)
    args = (case["X"], case["M"], case["Rt2"], case["Ct2"], case["dXbar"], case["r"], case["dX0"])
    items, A = ab.centroid_exactness(*args, k=k)
    assert set(A.unique().tolist()) <= {0.0, 1.0} and torch.equal(A.sum(dim=1), torch.ones(B, k, dtype=torch.float64))
    _check_exact(items)
    want = {**ab.centroid_stats(*args[:4], k=k), **ab.centroid_backward(*args, k=k)}
    _roundtrips(want)
    named = dict((nm, v) for nm, v, _, _ in items)
    g = (case["X"] @ case["dXbar"].transpose(1, 2))
    assert torch.equal(want["dX"], named["dX"]) and torch.equal(want["dS"][:, :, :k], named["dS"])
    assert (named["dS"] != 0).any() and not torch.equal((A * g).sum(dim=1), case["r"])      # r != dXbar . Xbar


def test_split_ranges_cover_the_tokens():
    for n, ns in ((4186, 11), (4186, 16), (130, 1), (1, 1), (65536, 16)):
        r = split_ranges(n, ns)
        assert r[0][0] == 0 and r[-1][1] == n and all(a[1] == b[0] for a, b in zip(r, r[1:]))
