"""Host checks of the fp64 reference of the dropout-aware stage-T double backward (tests/attn_double_backward_dropout_ref.py)
that the GPU tests of gf_attn_simplex_bwd_vjp_ex rely on:

* the reference against fp64 central differences of the first-order function it differentiates (the stage-T backward with
  attention dropout and its token reductions, dcb among them), along random directions of every input, with Philox masks;
* with an all-ones mask it is the dropout-free reference (tests/attn_double_backward_ref.stage_t_vjp), to fp64 round-off: the
  two differ only in computing ctl as sum_j p_j (Vt_j - cb) + cb instead of sum_j p_j Vt_j.
"""
import math

import pytest
import torch

from tests import attn_double_backward_dropout_ref as dr
from tests import attn_double_backward_ref as vr

dt = torch.float64


def _case(B, H, W, C, k, integration, seed, mean=0.0, p=0.5):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g, dtype=dt)
    KP = 16 if k <= 16 else 32
    Cout = 2 * C if integration == "both" else C
    n = H * W
    X, dOut = rn(B, n, C) + mean, rn(B, n, C)
    Kp, Vt, Rt, Ct = rn(B, KP, C) * 0.4, rn(B, Cout, KP), rn(B, H, KP), rn(B, W, KP)
    Kp = Kp - Kp.mean(dim=2, keepdim=True)
    Rt[:, :, k:] = -math.inf
    cb = rn(Cout)
    mult = dr.philox_mult(p, 1234 + seed, 7, 0x9E3779B1 * seed & 0xFFFFFFFF, B, n, KP)
    cots = [rn(B, n, C), rn(B, KP, C), rn(B, Cout, KP), rn(B, H, KP), rn(B, W, KP), rn(Cout)]
    return [X, dOut, Kp, Vt, Rt, Ct, cb], mult, cots, g


def _fd(f, ins, dirs, eps=1e-6):
    plus = f([a + eps * d for a, d in zip(ins, dirs)])
    minus = f([a - eps * d for a, d in zip(ins, dirs)])
    return (plus - minus) / (2 * eps)


@pytest.mark.parametrize("integration", ["mul", "add", "both"])
@pytest.mark.parametrize("norm", ["layer", "none"])
@pytest.mark.parametrize("mean", [0.0, 30.0])
@pytest.mark.parametrize("p", [0.12, 0.5])
def test_stage_t_vjp_dropout_matches_finite_differences(integration, norm, mean, p):
    B, H, W, C, k = 2, 3, 4, 8, 5
    ins, mult, cots, g = _case(B, H, W, C, k, integration, seed=11, mean=mean, p=p)
    assert 0 < torch.count_nonzero(mult[..., :k]) < mult[..., :k].numel()           # some latents dropped, some kept
    ref = dr.stage_t_vjp_dropout(*ins, mult, *cots, H=H, W=W, integration=integration, norm=norm)

    def loss(args):
        X = args[0].clone().requires_grad_(True)
        with torch.enable_grad():
            outs = dr.stage_t_reductions_dropout(X, *args[1:], mult, H=H, W=W, integration=integration, norm=norm)
        return sum((o.detach() * c).sum() for o, c in zip(outs, cots))

    names = ("Xg", "dOutg", "Kp", "Vt", "Rt", "Ct", "cb")
    for i, name in enumerate(names):
        d = torch.randn(ins[i].shape, generator=g, dtype=dt)
        if name == "Rt":
            d[:, :, k:] = 0.0
        dirs = [torch.zeros_like(t) if j != i else d for j, t in enumerate(ins)]
        dirs = [torch.where(torch.isfinite(t), dd, torch.zeros_like(dd)) for t, dd in zip(ins, dirs)]
        fd = _fd(loss, ins, dirs)
        an = (ref[name] * d).sum()
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (name, fd.item(), an.item())


@pytest.mark.parametrize("integration", ["mul", "add", "both"])
@pytest.mark.parametrize("norm", ["layer", "none"])
def test_all_ones_mask_is_the_dropout_free_reference(integration, norm):
    B, H, W, C, k = 2, 3, 4, 8, 5
    ins, mult, cots, _ = _case(B, H, W, C, k, integration, seed=3, mean=30.0)
    ones = torch.ones_like(mult)
    got = dr.stage_t_vjp_dropout(*ins, ones, *cots, H=H, W=W, integration=integration, norm=norm)
    want = vr.stage_t_vjp(*ins[:6], *cots[:5], H=H, W=W, integration=integration, norm=norm)
    for name in ("Xg", "dOutg", "Kp", "Vt", "Rt", "Ct", "Sg", "Ctlg"):
        err = ((got[name] - want[name]).abs().max() / want[name].abs().max().clamp_min(1e-300)).item()
        assert err < 1e-12, (name, err)
    # without dropout dcb is 0 for every input: its cotangent cbg changes nothing, and cb has no gradient
    assert got["cb"].abs().max() < 1e-12 * got["Vt"].abs().max()


def test_dropped_latents_only_reach_the_softmax():
    """A dropped latent keeps its logit cotangent (through the softmax normalisation) but its values get no gradient: the Vt
    reduction dCtl^T q has q = 0 there, and dp_j enters the softmax backward only through mk_j = 0."""
    B, H, W, C, k = 1, 2, 3, 8, 5
    ins, mult, cots, _ = _case(B, H, W, C, k, "mul", seed=9, p=0.5)
    ref = dr.stage_t_vjp_dropout(*ins, mult, *cots, H=H, W=W, integration="mul", norm="layer")
    dropped = mult[0] == 0                                                # [n, KP]
    assert torch.all(ref["P"][0][dropped] == 0)
    assert torch.count_nonzero(ref["Sg"][..., k:]) == 0 and torch.count_nonzero(ref["Rt"][..., k:]) == 0
