"""fp64 reference of the dropout-aware stage-T double backward (csrc/gf_bwd.cu: gf_attn_simplex_bwd_vjp_ex), shared by
tests/test_host_cpu_attn_double_backward_dropout.py and tests/test_gpu_attn_double_backward_dropout.py.

Test infrastructure only, beside tests/attn_double_backward_ref.py: the first-order backward of stage T with attention dropout
(oracle/folded.py per_token with att_mult / cb, the form the kernels use: ctl = sum_j q_j (Vt_j - cb) + cb, q = p * mult) is taken
together with its token reductions, dcb = sum_tokens (1 - sum_j q_j) dCtl among them, built as a graph with fp64 autograd and
differentiated again.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import folded as of
from oracle import philox as ph

Tensor = torch.Tensor


def philox_mult(p: float, seed: int, step: int, salt: int, B: int, n: int, KP: int) -> Tensor:
    """The kernels' dropout multipliers [B, n, KP] (oracle/philox.py), fp64."""
    return torch.from_numpy(ph.dropout_mult(p, seed, step, salt, B * n, KP).reshape(B, n, KP).copy()).double()


def stage_t_reductions_dropout(X, dOut, Kp, Vt, Rt, Ct, cb, mult, *, H, W, integration, norm, retain: Optional[dict] = None):
    """(dX, dKp = dS^T X, dVt = dCtl^T Q, dRt, dCt, dcb) of stage T with the dropout multipliers mult [B,n,KP], as a graph that
    can be differentiated again (X must require grad).  retain receives the forward's "S", "ctl" and "Q"."""
    keep = {} if retain is None else retain
    out, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm, att_mult=mult, cb=cb, retain=keep)
    dX, dS, dCtl = torch.autograd.grad((out * dOut).sum(), [X, keep["S"], keep["ctl"]], create_graph=True)
    B, n, KP = dS.shape
    dS4 = dS.reshape(B, H, W, KP)
    Q = keep["Q"]
    dcb = ((1.0 - Q.sum(dim=2, keepdim=True)) * dCtl).sum(dim=(0, 1))
    return dX, dS.transpose(1, 2) @ X, dCtl.transpose(1, 2) @ Q, dS4.sum(dim=2), dS4.sum(dim=1), dcb


def stage_t_vjp_dropout(X, dOut, Kp, Vt, Rt, Ct, cb, mult, U, Kpg, Vtg, Rtg, Ctg, cbg, *, H, W, integration,
                        norm) -> Dict[str, Tensor]:
    """What gf_attn_simplex_bwd_vjp_ex gives, in fp64: Xg, dOutg, Sg (of the logits), Ctlg (of the control signal) per token, the
    reduced cotangents Kp, Vt, Rt, Ct, cb of the tables, and the first-order dS, P (= q), dCtl."""
    ins = [t.detach().double().requires_grad_(True) for t in (X, dOut, Kp, Vt, Rt, Ct, cb)]
    m = mult.double()
    keep: dict = {}
    with torch.enable_grad():
        outs = stage_t_reductions_dropout(*ins, m, H=H, W=W, integration=integration, norm=norm, retain=keep)
        loss = sum((o * c.double()).sum() for o, c in zip(outs, (U, Kpg, Vtg, Rtg, Ctg, cbg)))
        g = torch.autograd.grad(loss, ins + [keep["S"], keep["ctl"]], allow_unused=True)
        k1: dict = {}
        out1, _ = of.per_token(ins[0], *ins[2:6], H=H, W=W, integration=integration, norm=norm, att_mult=m, cb=ins[6], retain=k1)
        first = torch.autograd.grad((out1 * ins[1]).sum(), [k1["S"], k1["ctl"]])
    z = lambda t, like: torch.zeros_like(like) if t is None else t
    names = ("Xg", "dOutg", "Kp", "Vt", "Rt", "Ct", "cb", "Sg", "Ctlg")
    res = {nm: z(t, ref).detach() for nm, t, ref in zip(names, g, ins + [keep["S"], keep["ctl"]])}
    res["Rt"] = torch.where(torch.isfinite(Rt.double()), res["Rt"], torch.zeros_like(res["Rt"])).nan_to_num(0.0)
    res.update(dS=first[0].detach(), P=keep["Q"].detach(), dCtl=first[1].detach())
    return res
