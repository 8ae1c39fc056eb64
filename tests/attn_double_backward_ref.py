"""fp64 references of the attention double-backward kernels at their C boundary (csrc/gf_bwd.cu: gf_attn_simplex_bwd_vjp,
gf_attn_centroid_bwd_vjp), shared by tests/test_host_cpu_attn_double_backward.py and tests/test_gpu_attn_double_backward.py.

Test infrastructure only, beside the first-order references of oracle/attn_bwd.py: each first-order backward is taken together
with its token reductions as one function, built as a graph with fp64 autograd (create_graph=True through folded.per_token and the
pass-A softmax), and differentiated again for the cotangents the double-backward kernels take.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import folded as of

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
