"""fp64 restatement of the image self-attention double backward (gf_self_attn_bwd_vjp; DESIGN 4.14).

TEST INFRASTRUCTURE ONLY.  The vector-Jacobian product of the first-order backward (Q, K, V, dO) -> (dQ, dK, dV) of
``oracle.self_attention.attention``, with cotangents A of dQ, Bk of dK and Cv of dV, per image and head, in the kernels' algebra
(s = 1/sqrt(d), P materialised here):

    dP = dO V^T,  Delta = rowsum(P o dP),  dS = P o (dP - Delta),  GdS = s (A K^T + Q Bk^T)
    r = rowsum(P o GdS),  u = rowsum(P o GdS o dP),  PC = P Cv
    GdP = P o (GdS - r),  GP = GdS o (dP - Delta) - r o dP + dO Cv^T,  t = u - 2 Delta r + dO . PC,  GS = P o (GP - t)
    gQ = s (dS Bk + GS K),  gK = s (dS^T A + GS^T Q),  gV = GdP^T dO,  gdO = GdP V + PC
Runs in the dtype of its inputs (float64 = truth).
"""
from __future__ import annotations

import math

import torch

from .bipartite import _split_heads


def _merge(t):
    B, h, n, d = t.shape
    return t.transpose(1, 2).reshape(B, n, h * d)


def vjp(q, k, v, do, a, bk, cv, heads: int):
    """[B,n,C] tensors -> (gQ, gK, gV, gdO) [B,n,C]."""
    C = q.shape[2]
    s = 1.0 / math.sqrt(C / heads)
    Q, K, V, dO, A, Bk, Cv = (_split_heads(t, heads) for t in (q, k, v, do, a, bk, cv))
    P = torch.softmax((Q @ K.transpose(2, 3)) * s, dim=3)
    dP = dO @ V.transpose(2, 3)
    delta = (P * dP).sum(dim=3, keepdim=True)
    dS = P * (dP - delta)
    GdS = s * (A @ K.transpose(2, 3) + Q @ Bk.transpose(2, 3))
    r = (P * GdS).sum(dim=3, keepdim=True)
    u = (P * GdS * dP).sum(dim=3, keepdim=True)
    PC = P @ Cv
    GdP = P * (GdS - r)
    GP = GdS * (dP - delta) - r * dP + dO @ Cv.transpose(2, 3)
    t = u - 2.0 * delta * r + (dO * PC).sum(dim=3, keepdim=True)
    GS = P * (GP - t)
    gQ = s * (dS @ Bk + GS @ K)
    gK = s * (dS.transpose(2, 3) @ A + GS.transpose(2, 3) @ Q)
    gV = GdP.transpose(2, 3) @ dO
    gdO = GdP @ V + PC
    return tuple(_merge(x) for x in (gQ, gK, gV, gdO))


def vjp_autograd(q, k, v, do, a, bk, cv, heads: int):
    """The same product by torch's double autograd through ``oracle.self_attention.attention``."""
    from .self_attention import attention
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, k, v, do)]
    Qa, Ka, Va, dOa = leaves
    with torch.enable_grad():
        o, _ = attention(Qa, Ka, Va, heads)
        dq, dk, dv = torch.autograd.grad(o, [Qa, Ka, Va], dOa, create_graph=True)
        return torch.autograd.grad((dq * a).sum() + (dk * bk).sum() + (dv * cv).sum(), leaves)
