"""fp64 references of the attention backward kernels at their C boundary, their magnitude companions, and the exact-integer
test cases (csrc/gf_bwd.cu: gf_attn_simplex_bwd_ex, gf_attn_centroid_stats, gf_attn_centroid_bwd).

TEST INFRASTRUCTURE ONLY (see oracle/bipartite.py).  The references are torch autograd in float64 through the folded oracle
(``folded.per_token`` and ``folded.centroid_softmax``) with the logits and the control signal retained, so they give the same
per-token quantities the kernels write:

  stage T   dX [B,n,C], dS [B,n,KP] (gradient of the logits), P [B,n,KP] (= q, the probabilities after dropout) and
            dCtl [B,n,Cout] (gradient of the control signal, both halves with integration "both");
  pass A    Xbar [B,k,C], lse [B,KP] (-inf in the padded latents), dX = dX_in + the pass-A part, dS [B,n,KP].

The companions are the same expressions evaluated on absolute values (the role conv(|x|, |w|) plays for a convolution): an
fp32 evaluation in any order is within a few ulps of the companion.  Every quantity that depends on the probabilities is
scaled by 1 + the largest |logit| companion of its token, because a logit rounded relative to its own magnitude moves the
probabilities by that much.

The exact cases make every probability 0, 1/2 or 1 and every intermediate a small multiple of a power of two; ``*_exactness``
lists the intermediates so that a test can check that claim instead of assuming it.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import folded as of
from . import philox as ph
from .bipartite import LN_EPS

Tensor = torch.Tensor
OFFSET = 2.0 ** 21        # planted logit offset: every latent outside the chosen set lies more than 745 below (exp == 0 in fp64)
GAP = 1024.0              # logits inside the chosen pair differ by a multiple of this: a tie or exp(-1024) == 0


# ---- stage T ------------------------------------------------------------------------------------------------------------------
def stage_t_backward(X, dOut, Kp, Vt, Rt, Ct, *, H, W, integration, norm, mult=None, cb=None) -> Dict[str, Tensor]:
    """What gf_attn_simplex_bwd_ex writes, in fp64: dX, dS, P (= q) and dCtl."""
    Xg = X.detach().double().requires_grad_(True)
    keep: dict = {}
    with torch.enable_grad():
        out, _ = of.per_token(Xg, Kp.double(), Vt.double(), Rt.double(), Ct.double(), H=H, W=W, integration=integration, norm=norm,
                              att_mult=mult, cb=None if cb is None else cb.double(), retain=keep)
        keep["S"].retain_grad()
        keep["ctl"].retain_grad()
        (out * dOut.double()).sum().backward()
    return dict(dX=Xg.grad, dS=keep["S"].grad, P=keep["Q"].detach(), dCtl=keep["ctl"].grad)


def stage_t_companions(X, dOut, Kp, Vt, Rt, Ct, *, H, W, k, integration, norm, mult=None, cb=None) -> Dict[str, Tensor]:
    """Magnitude companions of dX, dS, P and dCtl (see the module docstring)."""
    X, dOut, Kp, Vt, Rt, Ct = (t.double() for t in (X, dOut, Kp, Vt, Rt, Ct))
    B, n, C = X.shape
    KP = Kp.shape[1]
    S = X @ Kp.transpose(1, 2) + (Rt[:, :, None, :] + Ct[:, None, :, :]).reshape(B, n, KP)
    p = torch.softmax(S, dim=2)
    s_abs = X.abs() @ Kp.abs().transpose(1, 2) + (Rt[:, :, None, :].abs() + Ct[:, None, :, :].abs()).reshape(B, n, KP)
    F = 1.0 + s_abs[:, :, :k].amax(dim=2, keepdim=True)                 # [B,n,1]
    mk = torch.ones_like(p) if mult is None else torch.nn.functional.pad(mult.double(), (0, KP - mult.shape[2]), value=1.0)
    q = p * mk
    if norm == "layer":                      # the kernel's mean is mean(x - x0) + x0, x0 = the token's first channel (the shift)
        mu = X.mean(dim=2, keepdim=True)
        rstd = 1.0 / torch.sqrt(((X - mu) ** 2).mean(dim=2, keepdim=True) + LN_EPS)
        x0 = X[:, :, :1]
        xn_abs = (X.abs() + (X - x0).abs().mean(dim=2, keepdim=True) + x0.abs()) * rstd
    else:
        rstd, xn_abs = None, X.abs()
    go = dOut.abs()
    Vg = Vt[:, :C].abs()                                                  # gain half (or the only half)
    cbg = cb[:C].double().abs() if mult is not None else torch.zeros(C, dtype=torch.float64)
    qs = q.sum(dim=2, keepdim=True)
    g_abs = F * (q @ Vg.transpose(1, 2) + (1.0 + qs) * cbg)              # [B,n,C]
    if integration == "add":
        dc, dxn = go, go
        dctl = go
    else:
        dc, dxn = go * xn_abs, go * g_abs
        dctl = dc if integration == "mul" else torch.cat([dc, go], dim=2)
    dp = dc @ Vg                                                          # [B,n,KP]
    if integration == "both":
        dp = dp + go @ Vt[:, C:].abs()
    if mult is not None:
        dp = dp + (dctl * cb.double().abs()).sum(dim=2, keepdim=True)
    dp = dp * mk
    pd = (p * dp).sum(dim=2, keepdim=True)
    dS = F * p * (dp + pd)
    dX = dS @ Kp.abs()
    if norm == "layer":
        m1 = dxn.mean(dim=2, keepdim=True)
        m2 = (dxn * xn_abs).mean(dim=2, keepdim=True)
        dX = dX + rstd * (dxn + m1 + xn_abs * m2)
    else:
        dX = dX + dxn
    return dict(dX=dX, dS=dS, P=F * q, dCtl=dctl)


def stage_t_exactness(X, dOut, Kp, Vt, Rt, Ct, *, k, integration, mult=None, cb=None):
    """The intermediates of the kernel's arithmetic on an exact case (norm none), as (name, value, companion, grain): every
    partial sum of a value is a multiple of grain whose magnitude is at most the companion, so when companion / grain < 2^24
    fp32 holds every partial sum exactly in any order.  Also returns the probabilities p (before dropout)."""
    X, dOut, Kp, Vt, Rt, Ct = (t.double() for t in (X, dOut, Kp, Vt, Rt, Ct))
    B, n, C = X.shape
    KP = Kp.shape[1]
    RC = (Rt[:, :, None, :] + Ct[:, None, :, :]).reshape(B, n, KP)
    fin = torch.isfinite(RC)
    RCf = torch.where(fin, RC, torch.zeros_like(RC))
    RCa = (Rt[:, :, None, :].abs() + Ct[:, None, :, :].abs()).reshape(B, n, KP)
    S = X @ Kp.transpose(1, 2) + RCf
    s_abs = X.abs() @ Kp.abs().transpose(1, 2) + torch.where(fin, RCa, torch.zeros_like(RCa))
    p = torch.softmax(torch.where(fin, S, torch.full_like(S, -math.inf)), dim=2)
    mk = torch.ones_like(p) if mult is None else torch.nn.functional.pad(mult.double(), (0, KP - mult.shape[2]), value=1.0)
    q = p * mk
    cbd = cb.double() if mult is not None else torch.zeros(Vt.shape[1], dtype=torch.float64)
    qdef = 1.0 - q.sum(dim=2, keepdim=True)
    Vg = Vt[:, :C]
    g = q @ Vg.transpose(1, 2) + qdef * cbd[:C]
    g_abs = q @ Vg.abs().transpose(1, 2) + qdef.abs() * cbd[:C].abs()
    if integration == "add":
        dc = dxn = dOut
        dctl = dOut
    else:
        dc, dxn = dOut * X, dOut * g
        dctl = dc if integration == "mul" else torch.cat([dc, dOut], dim=2)
    dp = dc @ Vg
    dp_abs = dc.abs() @ Vg.abs()
    if integration == "both":
        dp = dp + dOut @ Vt[:, C:]
        dp_abs = dp_abs + dOut.abs() @ Vt[:, C:].abs()
    dcb = (dctl * cbd).sum(dim=2, keepdim=True)
    dcb_abs = (dctl.abs() * cbd.abs()).sum(dim=2, keepdim=True)
    dpm = (dp - dcb) * mk
    dpm_abs = (dp_abs + dcb_abs) * mk
    pd = (p * dpm).sum(dim=2, keepdim=True)
    pd_abs = (p * dpm_abs).sum(dim=2, keepdim=True)
    ds = p * (dpm - pd)
    ds_abs = p * (dpm_abs + pd_abs)
    dX = dxn + ds @ Kp
    dX_abs = dxn.abs() + ds_abs @ Kp.abs()
    items = [("logits", S, s_abs, 1.0), ("p", p, p, 0.5), ("q", q, q, 0.5), ("qdef", qdef, 1.0 + q.sum(2, keepdim=True), 0.5),
             ("g", g, g_abs, 0.5), ("dxn", dxn, dxn.abs() if integration == "add" else dOut.abs() * g_abs, 0.5),
             ("dCtl", dctl, dctl.abs(), 1.0), ("dp", dp, dp_abs, 1.0), ("dcb", dcb, dcb_abs, 1.0), ("dp_masked", dpm, dpm_abs, 1.0),
             ("pd", pd, pd_abs, 0.5), ("dS", ds, ds_abs, 0.25), ("dX", dX, dX_abs, 0.25)]
    return items, p[:, :, :k]


def exact_stage_t_case(B, H, W, C, k, integration, *, dropout: bool, seed: int, salt: int = 7, dp_seed: int = 20260901, step: int = 5):
    """Synthetic tables for gf_attn_simplex_bwd_ex whose arithmetic is exact (norm none).  Latents come in pairs (2i, 2i+1).  Rt
    adds OFFSET to the pair alpha(b, h) of each row, so every other latent's probability is exactly 0.  The two keys of a pair
    share small-integer channels and differ by GAP in two channels; Rt and Ct add multiples of GAP; so inside the pair the
    logits differ by a multiple of GAP, a one-hot pair or an exact tie at 1/2.  x, dOut, Vt and cb are small integers, and with
    dropout p = 0.5 the multipliers are 0 or 2.  The padded latents have Rt = -inf and nonzero keys, values and Ct."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(k)
    Cout = 2 * C if integration == "both" else C
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    sparse = lambda lo, hi, keep, *shape: ri(lo, hi, *shape) * (torch.rand(shape, generator=g) < keep).double()
    X = ri(-2, 2, B, n, C)
    dOut = sparse(-1, 1, 0.25, B, n, C)
    Kp = ri(-1, 1, B, KP, C)
    for j in range(1, k, 2):                                               # the partner shares the keys up to two channels
        Kp[:, j] = Kp[:, j - 1]
        ch = torch.randint(0, C, (B, 2), generator=g)
        Kp[torch.arange(B)[:, None], j, ch] += GAP * torch.tensor([1.0, -1.0]).expand(B, 2)
    npairs = (k + 1) // 2
    alpha = torch.randint(0, npairs, (B, H), generator=g)
    pair = torch.arange(KP) // 2
    Rt = GAP * sparse(-1, 1, 0.25, B, H, KP) + OFFSET * (pair[None, None, :] == alpha[:, :, None]).double()
    Ct = GAP * sparse(-1, 1, 0.25, B, W, KP)
    Rt[:, :, k:] = -math.inf
    Ct[:, :, k:] = ri(-3, 3, B, W, KP - k)
    Vt = ri(-1, 1, B, Cout, KP)
    cb = ri(-2, 2, Cout)
    mult = None
    if dropout:
        mult = torch.from_numpy(ph.dropout_mult(0.5, dp_seed, step, salt, B * n, KP).reshape(B, n, KP).copy()).double()
    return dict(X=X, dOut=dOut, Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct, cb=cb, mult=mult, att_dp=0.5 if dropout else 0.0,
                salt=salt, dp_seed=dp_seed, step=step)


def random_stage_t_case(B, H, W, C, k, integration, *, att_dp: float, mean: float, seed: int, salt: int = 3,
                        dp_seed: int = 77001, step: int = 9):
    """Realistic tables: logits of order one, a gain near 1 (mul / both), x with the given mean and unit spread."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(k)
    Cout = 2 * C if integration == "both" else C
    rn = lambda *shape: torch.randn(shape, generator=g, dtype=torch.float64)
    X = rn(B, n, C) + mean
    dOut = rn(B, n, C)
    Kp = rn(B, KP, C) / math.sqrt(C)
    if mean:
        Kp = Kp - Kp.mean(dim=2, keepdim=True)                          # keys orthogonal to the mean: logits of order one
    Kp[:, k:] = 0.0
    Rt, Ct = rn(B, H, KP), rn(B, W, KP)
    Rt[:, :, k:] = -math.inf
    Ct[:, :, k:] = 0.0
    Vt = 0.3 * rn(B, Cout, KP)
    cb = 0.3 * rn(Cout)
    if integration != "add":
        Vt[:, :C] += 1.0
        cb[:C] += 1.0
    Vt[:, :, k:] = 0.0
    mult = None
    if att_dp:
        mult = torch.from_numpy(ph.dropout_mult(att_dp, dp_seed, step, salt, B * n, KP).reshape(B, n, KP).copy()).double()
    return dict(X=X, dOut=dOut, Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct, cb=cb, mult=mult, att_dp=att_dp, salt=salt, dp_seed=dp_seed, step=step)


# ---- duplex pass A ------------------------------------------------------------------------------------------------------------
def centroid_stats(X, M, Rt2, Ct2, *, k) -> Dict[str, Tensor]:
    """What gf_attn_centroid_stats writes, in fp64: Xbar [B,k,C] and lse [B,KP] (-inf in the padded latents)."""
    B, KP = X.shape[0], M.shape[1]
    _, xbar, lse = of.centroid_softmax(X.double(), M.double(), Rt2.double(), Ct2.double(), k=k)
    return dict(Xbar=xbar, lse=torch.nn.functional.pad(lse, (0, KP - k), value=-math.inf))


def centroid_backward(X, M, Rt2, Ct2, dXbar, r, dX0, *, k) -> Dict[str, Tensor]:
    """What gf_attn_centroid_bwd writes, in fp64, for any r: dX = dX0 + A dXbar + dS M and dS = A (X dXbar^T - r).  With
    r = dXbar . Xbar this is the gradient of <dXbar, Xbar>; a different r adds -(r - dXbar . Xbar) lse to that loss."""
    Xg = X.detach().double().requires_grad_(True)
    dXbar, r = dXbar.double(), r.double()
    keep: dict = {}
    with torch.enable_grad():
        _, xbar, lse = of.centroid_softmax(Xg, M.double(), Rt2.double(), Ct2.double(), k=k, retain=keep)
        keep["L"].retain_grad()
        r_true = (dXbar * xbar).sum(dim=2).detach()
        ((dXbar * xbar).sum() - ((r - r_true) * lse).sum()).backward()
    KP = M.shape[1]
    return dict(dX=dX0.double() + Xg.grad, dS=torch.nn.functional.pad(keep["L"].grad, (0, KP - k)))


def _centroid_parts(X, M, Rt2, Ct2, k):
    X, M, Rt2, Ct2 = (t.double() for t in (X, M, Rt2, Ct2))
    B, n, C = X.shape
    RC = (Rt2[:, :, None, :k] + Ct2[:, None, :, :k]).reshape(B, n, k)
    RCa = (Rt2[:, :, None, :k].abs() + Ct2[:, None, :, :k].abs()).reshape(B, n, k)
    L = X @ M[:, :k].transpose(1, 2) + RC
    L_abs = X.abs() @ M[:, :k].abs().transpose(1, 2) + RCa
    return X, M, L, L_abs


def centroid_companions(X, M, Rt2, Ct2, dXbar, r, dX0, *, k) -> Dict[str, Tensor]:
    """Magnitude companions of Xbar, lse, dX and dS of pass A (see the module docstring)."""
    X, M, L, L_abs = _centroid_parts(X, M, Rt2, Ct2, k)
    dXbar, r, dX0 = dXbar.double(), r.double(), dX0.double()
    KP = M.shape[1]
    A = torch.softmax(L, dim=1)
    lse = torch.logsumexp(L, dim=1)                                      # [B,k]
    F = 1.0 + L_abs.amax(dim=1) + lse.abs()                              # [B,k]: the logits' scale per latent
    g_abs = X.abs() @ dXbar.abs().transpose(1, 2)                        # [B,n,k]
    dS = A * F[:, None, :] * (g_abs + r.abs()[:, None, :])
    dX = dX0.abs() + (A * F[:, None, :]) @ dXbar.abs() + dS @ M[:, :k].abs()
    pad = lambda t: torch.nn.functional.pad(t, (0, KP - k))
    return dict(Xbar=F[:, :, None] * (A.transpose(1, 2) @ X.abs()), lse=pad(F), dX=dX, dS=pad(dS))


def centroid_exactness(X, M, Rt2, Ct2, dXbar, r, dX0, *, k):
    """Intermediates of the pass-A kernels on an exact case, as (name, value, companion, grain) (see stage_t_exactness), and A."""
    X, M, L, L_abs = _centroid_parts(X, M, Rt2, Ct2, k)
    dXbar, r, dX0 = dXbar.double(), r.double(), dX0.double()
    A = torch.softmax(L, dim=1)
    lse = torch.logsumexp(L, dim=1)
    xbar = A.transpose(1, 2) @ X
    g = X @ dXbar.transpose(1, 2)
    g_abs = X.abs() @ dXbar.abs().transpose(1, 2)
    ds = A * (g - r[:, None, :])
    ds_abs = A * (g_abs + r.abs()[:, None, :])
    dX = dX0 + A @ dXbar + ds @ M[:, :k]
    dX_abs = dX0.abs() + A @ dXbar.abs() + ds_abs @ M[:, :k].abs()
    items = [("logits", L, L_abs, 1.0), ("A", A, A, 1.0), ("lse", lse, lse.abs(), 1.0), ("Xbar", xbar, A.transpose(1, 2) @ X.abs(), 1.0),
             ("g", g, g_abs, 1.0), ("dS", ds, ds_abs, 1.0), ("dX", dX, dX_abs, 1.0)]
    return items, A


def exact_centroid_case(B, H, W, C, k, *, winners: Tensor, seed: int):
    """Synthetic pass-A tables whose arithmetic is exact: winners [B,k] token indices.  Rt2 and Ct2 add OFFSET on the winner's
    row and column, so the winner's logit is 2 OFFSET plus a small integer, its row and column lie OFFSET below and every
    other token further: A is one-hot, Xbar_j = x_{t_j} and lse_j = s_{t_j}.  x, M, dXbar, r and the preloaded dX are small
    integers, with r != dXbar . Xbar.  The padded latents have Rt2 = -inf and nonzero M and Ct2."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(k)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    X = ri(-2, 2, B, n, C)
    M = ri(-1, 1, B, KP, C)
    Rt2 = ri(-3, 3, B, H, KP)
    Ct2 = ri(-3, 3, B, W, KP)
    bi = torch.arange(B)[:, None].expand(B, k)
    ji = torch.arange(k)[None, :].expand(B, k)
    Rt2[bi, winners // W, ji] += OFFSET
    Ct2[bi, winners % W, ji] += OFFSET
    Rt2[:, :, k:] = -math.inf
    dXbar = ri(-2, 2, B, k, C)
    r = ri(-5, 5, B, k)
    xw = X[bi, winners]                                                  # [B,k,C]
    r = torch.where(r == (dXbar * xw).sum(dim=2), r + 1.0, r)          # r != dXbar . Xbar: ds != 0 on the winners
    dX0 = ri(-4, 4, B, n, C)
    return dict(X=X, M=M, Rt2=Rt2, Ct2=Ct2, dXbar=dXbar, r=r, dX0=dX0)


def random_centroid_case(B, H, W, C, k, *, mean: float, seed: int):
    """Realistic pass-A tables: logits of order one over the tokens; r = dXbar . Xbar as the layer's backward passes it."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(k)
    rn = lambda *shape: torch.randn(shape, generator=g, dtype=torch.float64)
    X = rn(B, n, C) + mean
    M = rn(B, KP, C) / math.sqrt(C)
    if mean:
        M = M - M.mean(dim=2, keepdim=True)
    M[:, k:] = 0.0
    Rt2, Ct2 = rn(B, H, KP), rn(B, W, KP)
    Rt2[:, :, k:] = -math.inf
    Ct2[:, :, k:] = 0.0
    dXbar = rn(B, k, C)
    xbar = centroid_stats(X, M, Rt2, Ct2, k=k)["Xbar"]
    r = (dXbar * xbar).sum(dim=2)
    dX0 = rn(B, n, C)
    return dict(X=X, M=M, Rt2=Rt2, Ct2=Ct2, dXbar=dXbar, r=r, dX0=dX0)
