"""fp64 references of the attention double-backward kernels at their C boundary (csrc/gf_bwd.cu: gf_attn_simplex_bwd_vjp,
gf_attn_centroid_bwd_vjp), shared by tests/test_host_cpu_attn_double_backward.py, tests/test_gpu_attn_double_backward.py and the
exact tests (tests/test_host_cpu_attn_double_backward_exact.py, tests/test_gpu_attn_double_backward_exact.py).

Test infrastructure only, beside the first-order references of oracle/attn_bwd.py: each first-order backward is taken together
with its token reductions as one function, built as a graph with fp64 autograd (create_graph=True through folded.per_token and the
pass-A softmax), and differentiated again for the cotangents the double-backward kernels take.

The exact cases (``exact_stage_t_vjp_case``, ``exact_centroid_vjp_case``) make every intermediate of the kernels a small multiple
of a power of two; ``stage_t_vjp_exactness`` and ``centroid_vjp_exactness`` restate the kernels' arithmetic in fp64 and list those
intermediates, so that a test can check the claim instead of assuming it.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle import attn_bwd as ab
from oracle import folded as of
from oracle.folded import pad_k

Tensor = torch.Tensor


def stage_t_reductions(X, dOut, Kp, Vt, Rt, Ct, *, H, W, integration, norm, retain: Optional[dict] = None):
    """(dX, dKp = dS^T X, dVt = dCtl^T P, dRt, dCt) of stage T without dropout, as a graph that can be differentiated again (X
    must require grad).  retain receives the forward's logits "S" and control signal "ctl"."""
    keep = {} if retain is None else retain
    out, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm, retain=keep)
    dX, dS, dCtl = torch.autograd.grad((out * dOut).sum(), [X, keep["S"], keep["ctl"]], create_graph=True)
    B, n, KP = dS.shape
    dS4 = dS.reshape(B, H, W, KP)
    return dX, dS.transpose(1, 2) @ X, dCtl.transpose(1, 2) @ keep["Q"], dS4.sum(dim=2), dS4.sum(dim=1)


def stage_t_vjp(X, dOut, Kp, Vt, Rt, Ct, U, Kpg, Vtg, Rtg, Ctg, *, H, W, integration, norm) -> Dict[str, Tensor]:
    """What gf_attn_simplex_bwd_vjp gives, in fp64: the cotangents Xg, dOutg of X and dOut, Sg of the logits and Ctlg of the
    control signal per token, and the reduced cotangents Kp, Vt, Rt, Ct of the tables (0 in the padded latents of Rt)."""
    ins = [t.detach().double().requires_grad_(True) for t in (X, dOut, Kp, Vt, Rt, Ct)]
    keep: dict = {}
    with torch.enable_grad():
        outs = stage_t_reductions(*ins, H=H, W=W, integration=integration, norm=norm, retain=keep)
        loss = sum((o * c.double()).sum() for o, c in zip(outs, (U, Kpg, Vtg, Rtg, Ctg)))
        g = torch.autograd.grad(loss, ins + [keep["S"], keep["ctl"]], allow_unused=True)
    z = lambda t, like: torch.zeros_like(like) if t is None else t
    names = ("Xg", "dOutg", "Kp", "Vt", "Rt", "Ct", "Sg", "Ctlg")
    res = {nm: z(t, ref).detach() for nm, t, ref in zip(names, g, ins + [keep["S"], keep["ctl"]])}
    res["Rt"] = torch.where(torch.isfinite(Rt.double()), res["Rt"], torch.zeros_like(res["Rt"])).nan_to_num(0.0)
    return res


def centroid_reductions(X, M, Rt2, Ct2, lse, dXbar, r, dX0, *, H, W, k, retain: Optional[dict] = None):
    """(dX, dM = dS^T X, dRt2, dCt2) of gf_attn_centroid_bwd as a graph, with lse and r independent inputs as at the C
    boundary: a = exp(s - lse), g = x.dXbar, dS = a (g - r), dX = dX0 + A dXbar + dS M.  retain receives "L", "g" and "A"."""
    B, n, C = X.shape
    KP = M.shape[1]
    L = X @ M[:, :k].transpose(1, 2) + (Rt2[:, :, None, :k] + Ct2[:, None, :, :k]).reshape(B, n, k)
    A = torch.exp(L - lse[:, None, :k])
    g = X @ dXbar.transpose(1, 2)
    dS = A * (g - r[:, None, :])
    if retain is not None:
        retain.update(L=L, g=g, A=A)
    dSp = torch.nn.functional.pad(dS, (0, KP - k))
    dS4 = dSp.reshape(B, H, W, KP)
    return dX0 + A @ dXbar + dS @ M[:, :k], dSp.transpose(1, 2) @ X, dS4.sum(dim=2), dS4.sum(dim=1)


def centroid_vjp(X, M, Rt2, Ct2, lse, dXbar, r, dX0, U, Mg, Rt2g, Ct2g, *, H, W, k) -> Dict[str, Tensor]:
    """What gf_attn_centroid_bwd_vjp gives, in fp64: Xg, Sg (of the logits), Gg (of g = x.dXbar), A and dS per token (padded to
    KP), and the reduced cotangents M, Rt2, Ct2, lse, dXbar, r, dX0."""
    ins = [t.detach().double().requires_grad_(True) for t in (X, M, Rt2, Ct2, lse, dXbar, r, dX0)]
    keep: dict = {}
    KP = M.shape[1]
    with torch.enable_grad():
        outs = centroid_reductions(*ins, H=H, W=W, k=k, retain=keep)
        loss = sum((o * c.double()).sum() for o, c in zip(outs, (U, Mg, Rt2g, Ct2g)))
        g = torch.autograd.grad(loss, ins + [keep["L"], keep["g"]], allow_unused=True)
    pad = lambda t: torch.nn.functional.pad(t.detach(), (0, KP - k))
    names = ("Xg", "M", "Rt2", "Ct2", "lse", "dXbar", "r", "dX0")
    res = {nm: (torch.zeros_like(ref) if t is None else t).detach().nan_to_num(0.0) for nm, t, ref in zip(names, g[:8], ins)}
    for nm in ("Rt2", "lse"):
        res[nm][..., k:] = 0.0
    A = keep["A"]
    res.update(Sg=pad(g[8]), Gg=pad(g[9]), A=pad(A), dS=pad(A * (keep["g"] - ins[6][:, None, :])))
    return res


# ---- exact cases ----------------------------------------------------------------------------------------------------------------
# Every intermediate of the double-backward kernels on these cases is a small multiple of a power of two, so fp32 holds each of its
# partial sums exactly in any order and the kernels must equal the fp64 references bit for bit.  The *_exactness functions restate
# the kernels' arithmetic in fp64 and list each intermediate as (name, value, companion, grain), as oracle/attn_bwd.py does for the
# first-order kernels: every partial sum of value is a multiple of grain whose magnitude is at most companion.

class _Abs:
    """A value together with its magnitude companion (the same expression on absolute values)."""

    def __init__(self, v, a=None):
        self.v, self.a = v, (v.abs() if a is None else a)

    def __add__(self, o):
        return _Abs(self.v + o.v, self.a + o.a)

    def __sub__(self, o):
        return _Abs(self.v - o.v, self.a + o.a)

    def __mul__(self, o):
        return _Abs(self.v * o.v, self.a * o.a)

    def __matmul__(self, o):
        return _Abs(self.v @ o.v, self.a @ o.a)

    def sum(self, dim):
        return _Abs(self.v.sum(dim=dim, keepdim=True), self.a.sum(dim=dim, keepdim=True))

    def m(self):
        """The value once it is held in a register: exact, so its companion restarts at |value|."""
        return _Abs(self.v)

    @property
    def T(self):
        return _Abs(self.v.transpose(1, 2), self.a.transpose(1, 2))


def _rc(R, Cc):
    """Per-token row + column table [B,n,KP] from [B,H,KP] and [B,W,KP]."""
    B, H, KP = R.shape
    return (R[:, :, None, :] + Cc[:, None, :, :]).reshape(B, H * Cc.shape[1], KP)


def exact_stage_t_vjp_case(B, H, W, C, k, integration, *, dropout: bool, seed: int):
    """Tables of oracle/attn_bwd.exact_stage_t_case (norm none; one selected pair of latents per row, every probability 0, 1/2 or
    1; with dropout p = 1/2, multipliers 0 or 2) and small-integer cotangents U, Kg (a quarter of the channels nonzero), Vg, Rg,
    Cg and cbg.  Only the selected pair's probabilities are nonzero, and the partner's key differs by 1024 in two channels: U is
    zero in those two channels of each token, so the cotangent of dS (which has a term U . Kp) stays a small integer, and its
    products with dp stay far inside 2^24 grains up to C = 1024.  The padded latents get nonzero rows of Kg, Vg and Cg."""
    case = ab.exact_stage_t_case(B, H, W, C, k, integration, dropout=dropout, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    n, KP = H * W, pad_k(k)
    Cout = case["Vt"].shape[1]
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    sparse = lambda lo, hi, keep, *shape: ri(lo, hi, *shape) * (torch.rand(shape, generator=g) < keep).double()
    Kp = case["Kp"]
    U = sparse(-1, 1, 0.25, B, n, C)
    sel = (case["Rt"][:, :, :k] >= ab.OFFSET / 2).double()                # [B,H,k]: the row's selected pair
    gap = torch.zeros(B, H, C, dtype=torch.float64)
    for j in range(1, k, 2):                                               # the partner's two channels at +-1024
        gap += sel[:, :, j:j + 1] * ((Kp[:, j] - Kp[:, j - 1]).abs() >= ab.GAP / 2).double()[:, None, :]
    U = U * (gap == 0).double().repeat_interleave(W, dim=1)
    cots = dict(U=U, Kg=sparse(-1, 1, 0.25, B, KP, C), Vg=ri(-1, 1, B, Cout, KP), Rg=ri(-2, 2, B, H, KP), Cg=ri(-2, 2, B, W, KP),
                cbg=ri(-2, 2, Cout))
    return case, cots


def stage_t_vjp_exactness(X, dOut, Kp, Vt, Rt, Ct, U, Kg, Vg, Rg, Cg, *, k, integration, mult=None, cb=None, cbg=None):
    """The arithmetic of token_bwd_vjp_kernel (norm none; with mult, the dropout variant) restated in fp64.  Returns the
    intermediates as (name, value, companion, grain) and the eight per-token outputs.  A latent with p = 0 is inert: every term it
    contributes to another latent or channel is multiplied by p = 0 exactly (s * x, fma(s, x, acc)), so its own intermediates need
    not be exact, only finite; the items hold 0 there and the returned bound covers them unmasked."""
    X, dOut, Kp, Vt, Rt, Ct, U, Kg, Vg, Rg, Cg = (t.double() for t in (X, dOut, Kp, Vt, Rt, Ct, U, Kg, Vg, Rg, Cg))
    B, n, C = X.shape
    KP = Kp.shape[1]
    both, add, drop = integration == "both", integration == "add", mult is not None
    RC = _rc(Rt, Ct)
    fin = torch.isfinite(RC)
    z = torch.zeros_like(RC)
    S = _Abs(X) @ _Abs(Kp).T + _Abs(torch.where(fin, RC, z), torch.where(fin, _rc(Rt.abs(), Ct.abs()), z))
    p = torch.softmax(torch.where(fin, S.v, torch.full_like(S.v, -math.inf)), dim=2)
    P = _Abs(p)
    live = (p > 0).double()
    mk = _Abs(mult.double() if drop else torch.ones_like(p))
    q = (P * mk).m()
    one = _Abs(torch.ones(B, n, 1, dtype=torch.float64))
    qdef = (one - q.sum(2)).m()
    zc = torch.zeros(Vt.shape[1], dtype=torch.float64)
    cbv, cbgv = (cb.double(), cbg.double()) if drop else (zc, zc)
    cba, cbb, cga, cgb = (_Abs(t[None, None, :]) for t in (cbv[:C], cbv[C:], cbgv[:C], cbgv[C:]))
    Va, Wa = _Abs(Vt[:, :C]), _Abs(Vg[:, :C])                              # [B,C,KP]
    Vb, Wb = _Abs(Vt[:, C:]), _Abs(Vg[:, C:])
    x, go, u = _Abs(X), _Abs(dOut), _Abs(U)

    e = (_Abs(_rc(Rg, Cg), _rc(Rg.abs(), Cg.abs())) + x @ _Abs(Kg).T + u @ _Abs(Kp).T).m()
    # sweep 2: the gain, dCtl, dp and the cotangent of P accumulated against Vg
    if add:
        gain, dc = None, go
    else:
        gain = q @ Va.T
        if drop:
            gain = gain + qdef * cba
        gain = gain.m()
        dc = (go * x).m()
    dp, pb = dc @ Va, dc @ Wa
    if both:
        dp, pb = dp + go @ Vb, pb + go @ Wb
    dp = dp.m()
    dcbt = ((dc * cba).sum(2) + ((go * cbb).sum(2) if both else _Abs(torch.zeros(B, n, 1, dtype=torch.float64)))).m()
    dcg = ((dc * cga).sum(2) + ((go * cgb).sum(2) if both else _Abs(torch.zeros(B, n, 1, dtype=torch.float64)))).m()
    # the softmax backward and its reverse
    dpp = ((dp - dcbt) * mk).m() if drop else dp
    pd = (P * dpp).sum(2).m()
    pe = (P * e).sum(2).m()
    d = (dpp - pd).m()
    dr = e * d - pe * dpp
    dS = (P * d).m()
    f = (mk * (P * (e - pe).m()).m()).m()
    fsum = f.sum(2).m()
    if drop:
        dr = dr.m()                                                        # staged in Sg
    else:
        pb = pb + dr
    # sweep 3: the cotangents of dCtl (both halves), dOut, ctl and xn, and the cotangent of P against Vt
    cg = q @ Wa.T + f @ Va.T
    if drop:
        cg = cg + qdef * cga - fsum * cba
    cbias = None
    if both:
        cbias = q @ Wb.T + f @ Vb.T
        if drop:
            cbias = cbias + qdef * cgb - fsum * cbb
        cbias = cbias.m()
    cg = cg.m()
    if add:
        dog, xnb, gbar = u + cg, _Abs(torch.zeros_like(X)), _Abs(torch.zeros_like(X))
        gcb = _Abs(torch.zeros(B, n, 1, dtype=torch.float64))
    else:
        gbar = (u * go).m()
        pb = pb + gbar @ Va
        gcb = (gbar * cba).sum(2).m()
        dog = u * gain + (cg * x).m()
        if both:
            dog = dog.m() + cbias
        xnb = (cg * go).m()
    dog = dog.m()
    if drop:
        pb = mk * (pb.m() - (dcg + gcb).m()).m() + dr
    pb = pb.m()
    pp = (P * pb).sum(2).m()
    Sg = (P * (pb - pp).m()).m()
    Xg = xnb + Sg @ _Abs(Kp) + dS @ _Abs(Kg)

    lat = lambda t: (t.v * live, t.a * live)                               # per-latent: inert latents masked
    items = [("logits", S.v, S.a, 1.0), ("p", p, p, 0.5), ("q", q.v, q.a, 0.5), ("qdef", qdef.v, qdef.a, 0.5),
             ("e", *lat(e), 1.0), ("pe", pe.v, pe.a, 0.5), ("dCtl.cb", dcbt.v, dcbt.a, 1.0), ("dCtl.cbg", dcg.v, dcg.a, 1.0),
             ("dp", *lat(dpp), 1.0), ("pd", pd.v, pd.a, 0.5), ("dp - pd", *lat(d), 0.5), ("direct pbar", *lat(dr), 0.5),
             ("dS", dS.v, dS.a, 0.25), ("f", f.v, f.a, 0.25), ("F", fsum.v, fsum.a, 0.25), ("dCtl bar", cg.v, cg.a, 0.25),
             ("gbar", gbar.v, gbar.a, 1.0), ("gbar.cb", gcb.v, gcb.a, 1.0), ("dOut bar", dog.v, dog.a, 0.25),
             ("xn bar", xnb.v, xnb.a, 0.25), ("pbar", *lat(pb), 0.5), ("<p,pbar>", pp.v, pp.a, 0.25), ("Sg", Sg.v, Sg.a, 0.125),
             ("Xg", Xg.v, Xg.a, 0.125)]
    if gain is not None:
        items.append(("g", gain.v, gain.a, 0.5))
    if cbias is not None:
        items.append(("dCtl bar bias", cbias.v, cbias.a, 0.25))
    bound = max(t.a.max().item() for t in (e, dpp, d, dr, pb))
    Ctlg = torch.cat([gbar.v, torch.zeros_like(gbar.v)], dim=2) if both else gbar.v
    dCtl = torch.cat([dc.v, dOut], dim=2) if both else dc.v
    outs = dict(Xg=Xg.v, dOutg=dog.v, Sg=Sg.v, dPg=f.v, Ctlg=Ctlg, dS=dS.v, P=q.v, dCtl=dCtl)
    return items, outs, bound


def exact_centroid_vjp_case(B, H, W, C, k, *, rows: Tensor, seed: int):
    """Pass-A tables and cotangents for gf_attn_centroid_bwd_vjp whose arithmetic is exact.  rows [B,k]: latent j is active on the
    whole row rows[b, j].  Rt2 adds 2^21 on that row, and Ct2[w, j] = c_j - x[rows, w] . M_j, so every token of the row has the
    logit Rt2[row, j] + c_j, which is also lse_j: a = exp(0) = 1 there, and every other token lies about 2^21 below, a = 0.  x, M,
    dXbar, r and the cotangents are small integers (U and Mg thinned to a few channels per token, which keeps the cotangent of dS
    small); r != x . dXbar on most active tokens, so dS != 0.  The padded latents have lse = -inf and nonzero M, Mg and Ct2."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, pad_k(k)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    sparse = lambda lo, hi, keep, *shape: ri(lo, hi, *shape) * (torch.rand(shape, generator=g) < keep).double()
    X = ri(-2, 2, B, n, C)
    M = ri(-1, 1, B, KP, C)
    Rt2 = ri(-3, 3, B, H, KP)
    bi = torch.arange(B)[:, None].expand(B, k)
    ji = torch.arange(k)[None, :].expand(B, k)
    Rt2[bi, rows, ji] += ab.OFFSET
    Rt2[:, :, k:] = -math.inf
    c = ri(-3, 3, B, k)
    xrow = X.reshape(B, H, W, C)[bi, rows]                                  # [B,k,W,C]: the active row of every latent
    Ct2 = ri(-3, 3, B, W, KP)
    Ct2[:, :, :k] = c[:, None, :] - torch.einsum("bjwc,bjc->bwj", xrow, M[:, :k])
    lse = torch.full((B, KP), -math.inf, dtype=torch.float64)
    lse[:, :k] = Rt2[bi, rows, ji] + c
    dXbar = ri(-2, 2, B, k, C)
    r = ri(-6, 6, B, k)
    dX0 = ri(-4, 4, B, n, C)
    cots = dict(U=sparse(-1, 1, 0.25, B, n, C), Mg=sparse(-1, 1, 0.25, B, KP, C), Rt2g=ri(-2, 2, B, H, KP),
                Ct2g=ri(-2, 2, B, W, KP))
    return dict(X=X, M=M, Rt2=Rt2, Ct2=Ct2, lse=lse, dXbar=dXbar, r=r, dX0=dX0), cots


def centroid_vjp_exactness(X, M, Rt2, Ct2, lse, dXbar, r, U, Mg, Rt2g, Ct2g, *, k):
    """The arithmetic of centroid_bwd_vjp_kernel restated in fp64: the intermediates as (name, value, companion, grain) and the
    per-token outputs Xg, Sg, Gg, A, dS [B,n,KP].  Tokens with a = 0 are inert in the same way as the latents of
    stage_t_vjp_exactness; here every intermediate is an integer and the unmasked bound is returned as well."""
    X, M, Rt2, Ct2, lse, dXbar, r, U, Mg, Rt2g, Ct2g = (t.double() for t in (X, M, Rt2, Ct2, lse, dXbar, r, U, Mg, Rt2g, Ct2g))
    B, n, C = X.shape
    KP = M.shape[1]
    Gp = torch.nn.functional.pad(dXbar, (0, 0, 0, KP - k))                 # [B,KP,C]: zero rows in the padded latents
    rp = torch.nn.functional.pad(r, (0, KP - k))
    x, u = _Abs(X), _Abs(U)
    RC = _rc(Rt2, Ct2)
    fin = torch.isfinite(RC)
    zr = torch.zeros_like(RC)
    s = x @ _Abs(M).T + _Abs(torch.where(fin, RC, zr), torch.where(fin, _rc(Rt2.abs(), Ct2.abs()), zr))
    lfin = torch.isfinite(lse)[:, None, :]
    a = torch.where(lfin, torch.exp(torch.where(fin, s.v, zr) - torch.where(lfin, lse[:, None, :], 0.0)), zr)
    A = _Abs(a)
    live = (a > 0).double()
    gg = x @ _Abs(Gp).T
    e = _Abs(_rc(Rt2g, Ct2g), _rc(Rt2g.abs(), Ct2g.abs())) + x @ _Abs(Mg).T + u @ _Abs(M).T
    ug = u @ _Abs(Gp).T
    gr = gg - _Abs(rp[:, None, :])
    dS = A * gr
    Sg = A * (e * gr + ug)
    Gg = A * e
    Xg = Sg @ _Abs(M) + Gg @ _Abs(Gp) + dS @ _Abs(Mg)
    lat = lambda t: (t.v * live, t.a * live)
    items = [("logits", s.v, s.a, 1.0), ("a", a, a, 1.0), ("g", gg.v, gg.a, 1.0), ("e", *lat(e), 1.0),
             ("U.dXbar", ug.v, ug.a, 1.0), ("g - r", gr.v, gr.a, 1.0), ("dS", dS.v, dS.a, 1.0), ("Gg", Gg.v, Gg.a, 1.0),
             ("Sg", Sg.v, Sg.a, 1.0), ("Xg", Xg.v, Xg.a, 1.0)]
    bound = max(t.a.max().item() for t in (s, e))
    return items, dict(Xg=Xg.v, Sg=Sg.v, Gg=Gg.v, A=a, dS=dS.v), bound


def centroid_stats_backward(X, M, Rt2, Ct2, dXbar, lseg, *, k) -> Dict[str, Tensor]:
    """fp64 autograd of <dXbar, Xbar> + <lseg, lse> through folded.centroid_softmax: the gradients of X, M, Rt2, Ct2 that
    gf_attn_centroid_bwd gives with r = dXbar . Xbar - lseg and dX0 = 0 (the backward of gf_attn_centroid_stats)."""
    ins = [t.detach().double().requires_grad_(True) for t in (X, M, Rt2, Ct2)]
    with torch.enable_grad():
        _, xbar, lse = of.centroid_softmax(*ins, k=k)
        g = torch.autograd.grad((xbar * dXbar.double()).sum() + (lse * lseg.double()).sum(), ins)
    res = dict(zip(("X", "M", "Rt2", "Ct2"), (t.nan_to_num(0.0) for t in g)))
    res["Rt2"][..., k:] = 0.0
    return res
