"""Image self-attention (upstream GANsformer's ``img2img``; SURVEY A.4 item 18): ``transformer_layer(from = X, to = X)``, the bipartite
layer with the image itself as the key / value source.

    X [B,n,C] channels-last, n = H W;  h = max(1, C // 64) heads of d = C / h channels (d in {32, 64})
    Q = X Wq + bq + Pg Wpq,   K = X Wk + bk + Pg Wpk,   V = X Wv + bv           (equalised LR; Pg only with use_pos)
    per head: P = softmax over the n keys of Q_h K_h^T / sqrt(d);   ctrl = concat_h(P V_h) Wo + bo
    out = integrate(X, ctrl, integration, norm)

The n x n part runs on the fused kernels of csrc/gf_self_attn.cu (``gf_self_attn_fwd`` / ``gf_self_attn_bwd``: online softmax, no n x n
tensor in memory, deterministic backward) through one autograd Function.  The four projections and ``integrate`` are ordinary GEMM and
elementwise work: TF32 matmuls here, true fp32 with ``exact_fp32=True``, which also runs the n x n part as the torch composite.
A backward run with grad mode on (the generator's path-length phase, the discriminator's R1 pass) recomputes the n x n part through
the composite with create_graph=True, which materialises P and the n x n tensors of its own backward graph.  A layer whose
``kernel_double_backward`` is set runs that backward on the kernels instead (``_SelfAttentionBackward``: gf_self_attn_bwd, and the
double-backward kernel gf_self_attn_bwd_vjp as its derivative), so that every tensor it keeps is [B,n,C] or [B,h,n].  No attention
dropout, no attention map, no CPU path.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
from typing import Optional

import torch
from torch import nn

from . import _lib
from .autograd import _alias, _differentiable_twice, _e, _fp32_matmul, _zeros_if_none, grid_pos_table, integrate


def heads_of(C: int):
    """(h, d) of a layer of width C: head size 64, or 32 when C = 32.  ValueError for a width the kernels cannot split so."""
    h = max(1, C // 64)
    d = C // h
    if C % h or d not in (32, 64):
        raise ValueError(f"image self-attention needs C = 32 or a multiple of 64 channels (head size 32 or 64), got C={C}")
    return h, d


@contextlib.contextmanager
def _tf32_matmul():
    """The projections of the layer run as TF32 GEMMs whatever torch.backends.cuda.matmul.allow_tf32 says (the mirror image of
    autograd._fp32_matmul)."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def attention_composite(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """The n x n part in torch ops, materialising P: q, k, v [B,n,C] -> concat_h(softmax(Q_h K_h^T / sqrt(d)) V_h) [B,n,C]."""
    B, n, C = q.shape
    d = C // heads
    sp = lambda t: t.reshape(B, n, heads, d).transpose(1, 2)
    P = torch.softmax((sp(q) @ sp(k).transpose(2, 3)) * (1.0 / math.sqrt(d)), dim=3)
    return (P @ sp(v)).transpose(1, 2).reshape(B, n, C)


def _stream(t: torch.Tensor):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def attention_fwd_native(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int):
    """gf_self_attn_fwd: q, k, v [B,n,C] contiguous fp32 CUDA -> (o [B,n,C], lse [B,h,n] in log2 units)."""
    B, n, C = q.shape
    d = C // heads
    vt = v.transpose(1, 2).contiguous()                       # per-head V^T [B, h, d, n]: the B operand of O = P V
    o = torch.empty_like(q)
    lse = torch.empty((B, heads, n), device=q.device, dtype=torch.float32)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().gf_self_attn_fwd(q.data_ptr(), k.data_ptr(), vt.data_ptr(), o.data_ptr(), lse.data_ptr(), B, n, C, d,
                                                1.0 / math.sqrt(d), _stream(q)), "gf_self_attn_fwd")
    return o, lse


def attention_bwd_native(q, k, v, o, lse, do, heads: int):
    """gf_self_attn_bwd: -> (dq, dk, dv) [B,n,C]."""
    return _attention_bwd(q, k, v, o, lse, do, heads)[:3]


def _attention_bwd(q, k, v, o, lse, do, heads: int):
    """gf_self_attn_bwd: -> (dq, dk, dv, delta), delta [B,h,n] = rowsum(dO o O), which the double backward takes."""
    B, n, C = q.shape
    d = C // heads
    qt, kt, dot = (t.transpose(1, 2).contiguous() for t in (q, k, do))
    delta = torch.empty_like(lse)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().gf_self_attn_bwd(q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                lse.data_ptr(), do.data_ptr(), dot.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                                                dk.data_ptr(), dv.data_ptr(), B, n, C, d, 1.0 / math.sqrt(d), _stream(q)),
                   "gf_self_attn_bwd")
    return dq, dk, dv, delta


def attention_bwd_vjp_native(q, k, v, do, lse, delta, a, bk, cv, heads: int):
    """gf_self_attn_bwd_vjp: the cotangents a, bk, cv of (dq, dk, dv) -> (gq, gk, gv, gdo) [B,n,C], the gradients of
    <a, dq> + <bk, dk> + <cv, dv> with respect to q, k, v and dO."""
    B, n, C = q.shape
    d = C // heads
    qt, kt, vt, dot, at, bkt, cvt = (t.transpose(1, 2).contiguous() for t in (q, k, v, do, a, bk, cv))
    row_r, row_t = torch.empty_like(lse), torch.empty_like(lse)
    gq, gk, gv, gdo = (torch.empty_like(q) for _ in range(4))
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().gf_self_attn_bwd_vjp(q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), vt.data_ptr(),
                                                    do.data_ptr(), dot.data_ptr(), lse.data_ptr(), delta.data_ptr(), a.data_ptr(),
                                                    at.data_ptr(), bk.data_ptr(), bkt.data_ptr(), cv.data_ptr(), cvt.data_ptr(),
                                                    row_r.data_ptr(), row_t.data_ptr(), gq.data_ptr(), gk.data_ptr(), gv.data_ptr(),
                                                    gdo.data_ptr(), B, n, C, d, 1.0 / math.sqrt(d), _stream(q)), "gf_self_attn_bwd_vjp")
    return gq, gk, gv, gdo


class _SelfAttention(torch.autograd.Function):
    """The n x n part on the kernels: forward gf_self_attn_fwd, first-order backward gf_self_attn_bwd.  A backward under grad mode
    runs ``_SelfAttentionBackward`` when ``double_kernels`` is set, and otherwise recomputes through ``attention_composite`` with
    create_graph=True."""

    @staticmethod
    def forward(ctx, q, k, v, heads, double_kernels=False):
        o, lse = attention_fwd_native(q, k, v, heads)
        ctx.heads, ctx.double_kernels = heads, double_kernels
        ctx.save_for_backward(q, k, v, o, lse)
        return o

    @staticmethod
    def backward(ctx, g):
        q, k, v, o, lse = ctx.saved_tensors
        if torch.is_grad_enabled():
            if ctx.double_kernels:
                return (*_SelfAttentionBackward.apply(q, k, v, o.detach(), lse, g.contiguous(), ctx.heads), None, None)
            qs, ks, vs = _alias(q), _alias(k), _alias(v)
            out = attention_composite(qs, ks, vs, ctx.heads)
            return (*torch.autograd.grad(out, [qs, ks, vs], g, create_graph=True), None, None)
        return (*attention_bwd_native(q, k, v, o, lse, g.contiguous(), ctx.heads), None, None)


class _SelfAttentionBackward(torch.autograd.Function):
    """The first-order backward as a differentiable function of (q, k, v, dO): forward gf_self_attn_bwd, backward the
    double-backward kernel gf_self_attn_bwd_vjp.  o and lse are recomputation aids, not inputs of the function: Delta =
    rowsum(dO o O) carries the whole dependence on O.  Saved for the second pass: q, k, v, dO, lse and Delta.  A third derivative
    raises."""

    @staticmethod
    def forward(ctx, q, k, v, o, lse, do, heads):
        dq, dk, dv, delta = _attention_bwd(q, k, v, o, lse, do, heads)
        ctx.heads = heads
        ctx.save_for_backward(q, k, v, do, lse, delta)
        return dq, dk, dv

    @staticmethod
    @_differentiable_twice
    def backward(ctx, ga, gb, gc):
        q, k, v, do, lse, delta = ctx.saved_tensors
        a, bk, cv = (_zeros_if_none(g_, t) for g_, t in ((ga, q), (gb, k), (gc, v)))
        gq, gk, gv, gdo = attention_bwd_vjp_native(q, k, v, do, lse, delta, a, bk, cv, ctx.heads)
        return gq, gk, gv, None, None, gdo, None


class ImageSelfAttention(nn.Module):
    """One img2img layer: x [B,H,W,C] channels-last fp32 CUDA -> [B,H,W,C].  Parameters follow ``BipartiteAttention``'s names
    (wq bq wk bk wv bv wo bo, wpq wpk with use_pos), [fan_in, fan_out], weights N(0, 1), biases zero.

    ``kernel_double_backward`` (the meaning of ``BipartiteAttention.kernel_double_backward``): a backward run with create_graph=True
    (R1, path length) stays on the kernels, differentiated by gf_self_attn_bwd_vjp, instead of recomputing through the composite.
    Its second-order gradients then differ from the composite route by TF32 round-off.  Off by default; ignored with exact_fp32."""

    kernel_double_backward = False

    def __init__(self, C: int, pos_dim: int, integration: str = "mul", norm: Optional[str] = "layer", use_pos: bool = True,
                 exact_fp32: bool = False):
        super().__init__()
        self.heads, self.head_dim = heads_of(C)
        if integration not in ("mul", "add", "both"):
            raise ValueError(f"unknown integration {integration!r}")
        if norm not in (None, "none", "layer", "instance", "batch"):
            raise ValueError(f"unknown norm {norm!r}")
        if use_pos and (pos_dim <= 0 or pos_dim % 4):
            raise ValueError(f"pos_dim must be a positive multiple of 4, got {pos_dim}")
        self.dim, self.pos_dim, self.integration, self.norm = C, pos_dim, integration, norm
        self.use_pos, self.exact_fp32 = use_pos, exact_fp32
        cout = 2 * C if integration == "both" else C
        shapes = {"wq": (C, C), "bq": (C,), "wk": (C, C), "bk": (C,), "wv": (C, C), "bv": (C,), "wo": (C, cout), "bo": (cout,)}
        if use_pos:
            shapes.update({"wpq": (pos_dim, C), "wpk": (pos_dim, C)})
        for name, shape in shapes.items():
            self.register_parameter(name, nn.Parameter(torch.zeros(shape) if name.startswith("b") else torch.randn(shape)))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError(f"image self-attention has no CPU path (tensor is on {x.device})")
        if x.dim() != 4 or x.shape[3] != self.dim or x.dtype != torch.float32:
            raise ValueError(f"x must be a float32 [B, H, W, {self.dim}] tensor, got {x.dtype} {tuple(x.shape)}")
        B, H, W, C = x.shape
        X = x.reshape(B, H * W, C)
        with (_fp32_matmul() if self.exact_fp32 else _tf32_matmul()):
            Q = X @ _e(self.wq) + self.bq
            K = X @ _e(self.wk) + self.bk
            V = X @ _e(self.wv) + self.bv
            if self.use_pos:
                Pg = grid_pos_table(H, W, self.pos_dim, x.device, x.dtype)
                Q = Q + Pg @ _e(self.wpq)
                K = K + Pg @ _e(self.wpk)
            if self.exact_fp32:
                A = attention_composite(Q, K, V, self.heads)
            else:
                A = _SelfAttention.apply(Q.contiguous(), K.contiguous(), V.contiguous(), self.heads, bool(self.kernel_double_backward))
            ctl = A @ _e(self.wo) + self.bo
        return integrate(X, ctl, self.integration, self.norm).reshape(B, H, W, C)
