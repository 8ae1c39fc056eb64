"""Host checks of the double-backward references (tests/attn_double_backward_ref.py) that the GPU tests of
gf_attn_simplex_bwd_vjp and gf_attn_centroid_bwd_vjp rely on:

* each VJP reference against fp64 central differences of the first-order function it differentiates (the stage-T backward with
  its token reductions, the pass-A backward with its reductions), along random directions of every input;
* the identity that makes a third kernel unnecessary: the backward of gf_attn_centroid_stats with cotangents (dXbar, lseg) is
  gf_attn_centroid_bwd with r = dXbar . Xbar - lseg and dX starting from zero.
"""
import math

import pytest
import torch

from oracle import attn_bwd as ab
from tests import attn_double_backward_ref as vr

dt = torch.float64


def _tables(B, H, W, C, k, integration, seed, mean=0.0):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g, dtype=dt)
    KP = 16 if k <= 16 else 32
    Cout = 2 * C if integration == "both" else C
    n = H * W
    X, dOut = rn(B, n, C) + mean, rn(B, n, C)
    Kp, Vt, Rt, Ct = rn(B, KP, C) * 0.4, rn(B, Cout, KP), rn(B, H, KP), rn(B, W, KP)
    Kp = Kp - Kp.mean(dim=2, keepdim=True)
    Rt[:, :, k:] = -math.inf
    cots = [rn(B, n, C), rn(B, KP, C), rn(B, Cout, KP), rn(B, H, KP), rn(B, W, KP)]
    return [X, dOut, Kp, Vt, Rt, Ct], cots, g


def _fd(f, ins, dirs, eps=1e-6):
    plus = f([a + eps * d for a, d in zip(ins, dirs)])
    minus = f([a - eps * d for a, d in zip(ins, dirs)])
    return (plus - minus) / (2 * eps)


@pytest.mark.parametrize("integration", ["mul", "add", "both"])
@pytest.mark.parametrize("norm", ["layer", "none"])
@pytest.mark.parametrize("mean", [0.0, 30.0])
def test_stage_t_vjp_matches_finite_differences(integration, norm, mean):
    B, H, W, C, k = 2, 3, 4, 8, 5
    ins, cots, g = _tables(B, H, W, C, k, integration, seed=11, mean=mean)
    ref = vr.stage_t_vjp(*ins, *cots, H=H, W=W, integration=integration, norm=norm)

    def loss(args):
        X = args[0].clone().requires_grad_(True)
        with torch.enable_grad():
            outs = vr.stage_t_reductions(X, *args[1:], H=H, W=W, integration=integration, norm=norm)
        return sum((o.detach() * c).sum() for o, c in zip(outs, cots))

    names = ("Xg", "dOutg", "Kp", "Vt", "Rt", "Ct")
    for i, name in enumerate(names):
        d = torch.randn(ins[i].shape, generator=g, dtype=dt)
        if name == "Rt":
            d[:, :, k:] = 0.0
        dirs = [torch.zeros_like(t) if j != i else d for j, t in enumerate(ins)]
        dirs = [torch.where(torch.isfinite(t), dd, torch.zeros_like(dd)) for t, dd in zip(ins, dirs)]
        fd = _fd(loss, ins, dirs)
        an = (ref[name] * d).sum()
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (name, fd.item(), an.item())


def test_stage_t_vjp_padded_latents_are_inert():
    """Padded latents (Rt = -inf) have p = 0: their logit cotangent is 0 whatever their keys and cotangents."""
    B, H, W, C, k = 1, 2, 3, 8, 3
    ins, cots, _ = _tables(B, H, W, C, k, "mul", seed=3)
    ref = vr.stage_t_vjp(*ins, *cots, H=H, W=W, integration="mul", norm="layer")
    assert torch.count_nonzero(ref["Sg"][..., k:]) == 0 and torch.count_nonzero(ref["Rt"][..., k:]) == 0
    assert torch.count_nonzero(ref["Ct"][..., k:]) == 0


def _centroid(B, H, W, C, k, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g, dtype=dt)
    KP = 16 if k <= 16 else 32
    n = H * W
    X, M = rn(B, n, C), rn(B, KP, C) * 0.3
    Rt2, Ct2 = rn(B, H, KP), rn(B, W, KP)
    Rt2[:, :, k:] = -math.inf
    st = ab.centroid_stats(X, M, Rt2, Ct2, k=k)
    lse = st["lse"] + 0.25 * torch.nn.functional.pad(rn(B, k), (0, KP - k))      # any lse: an independent input at the boundary
    ins = [X, M, Rt2, Ct2, lse, rn(B, k, C), rn(B, k), rn(B, n, C)]
    cots = [rn(B, n, C), rn(B, KP, C), rn(B, H, KP), rn(B, W, KP)]
    return ins, cots, g, st


@pytest.mark.parametrize("k", [1, 5, 17])
def test_centroid_vjp_matches_finite_differences(k):
    B, H, W, C = 2, 3, 4, 8
    ins, cots, g, _ = _centroid(B, H, W, C, k, seed=5 + k)
    ref = vr.centroid_vjp(*ins, *cots, H=H, W=W, k=k)

    def loss(args):
        outs = vr.centroid_reductions(*args, H=H, W=W, k=k)
        return sum((o * c).sum() for o, c in zip(outs, cots))

    names = ("Xg", "M", "Rt2", "Ct2", "lse", "dXbar", "r", "dX0")
    for i, name in enumerate(names):
        d = torch.randn(ins[i].shape, generator=g, dtype=dt)
        if name in ("Rt2", "lse"):
            d[..., k:] = 0.0
        dirs = [torch.zeros_like(t) if j != i else d for j, t in enumerate(ins)]
        fd = _fd(loss, ins, dirs)
        an = (ref[name] * d).sum()
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (name, fd.item(), an.item())
    assert torch.equal(ref["dX0"], cots[0])                              # the cotangent of dX_in passes straight through


@pytest.mark.parametrize("k", [1, 7, 20])
def test_centroid_stats_backward_is_centroid_bwd_with_shifted_r(k):
    """d lse_j / d s[t,j] = A[t,j]: the lse cotangent only shifts r, so no third kernel is needed."""
    B, H, W, C = 2, 3, 5, 8
    ins, _, g, st = _centroid(B, H, W, C, k, seed=40 + k)
    X, M, Rt2, Ct2 = ins[:4]
    dXbar = torch.randn(B, k, C, generator=g, dtype=dt)
    lseg = torch.randn(B, k, generator=g, dtype=dt)
    want = vr.centroid_stats_backward(X, M, Rt2, Ct2, dXbar, lseg, k=k)
    r = (dXbar * st["Xbar"]).sum(dim=2) - lseg
    got = ab.centroid_backward(X, M, Rt2, Ct2, dXbar, r, torch.zeros_like(X), k=k)
    dS4 = got["dS"].reshape(B, H, W, -1)
    pairs = {"X": got["dX"], "M": got["dS"].transpose(1, 2) @ X, "Rt2": dS4.sum(dim=2), "Ct2": dS4.sum(dim=1)}
    for name, t in pairs.items():
        t = t.clone()
        if name == "Rt2":
            t[..., k:] = 0.0
        err = ((t - want[name]).norm() / want[name].norm()).item()
        assert err < 1e-12, (name, err)
