"""Differentiable wrapper of the fused attention op (needed by the G/D training step, SURVEY row f2).

Forward = the C-ABI CUDA kernels.  ``_FusedAttention.backward`` takes one of three routes:
* simplex kernels (``_simplex_kernel_backward``), for a simplex layer with layer norm (or none): the hand-written stage-T backward
  kernel ``gf_attn_simplex_bwd_ex`` (activation gradient + the per-token gradients of logits / control signal), two batched GEMMs
  for the reductions over tokens, and torch autograd through the tiny per-image tables of stages W and I (``folded_tables``);
* duplex kernels (``_duplex_kernel_backward``), for a duplex layer (one k-means iteration, layer norm / none) whose forward ran with
  attention dropout, or whose module sets ``kernel_backward`` (the discriminator's layers, whose centroids output is then
  differentiable): the same stage-T kernel with keys from the centroids, plus the pass-A kernels ``gf_attn_centroid_stats`` /
  ``gf_attn_centroid_bwd`` and autograd through the pass-A tables (``centroid_tables``);
* composite (``_composite_backward``), everything else (duplex without dropout, instance / batch norm, multi-head, CPU tensors):
  PyTorch autograd through a recomputation of the direct-form algebra with torch ops (``composite_forward``).
Each route serves both orders.  Run with create_graph=True (the generator's path-length penalty; the discriminator's R1 penalty
when its modules set ``kernel_double_backward``), a kernel route builds a graph: the per-token work runs in three Functions,
``_StageTBackward``, ``_CentroidStats`` and ``_CentroidBackward``, whose own backward are the double-backward kernels
``gf_attn_simplex_bwd_vjp`` (``_ex`` with the forward's dropout mask) / ``gf_attn_centroid_bwd_vjp``.  A first-order backward calls
their forward bodies directly and leaves no graph behind.
"""
from __future__ import annotations

import contextlib
import ctypes
import math

import torch
from torch.autograd.function import once_differentiable

from . import _lib


def _e(w):
    return w * (1.0 / math.sqrt(w.shape[0]))


def _axis(length, dim, device):
    pos = (torch.arange(length, dtype=torch.float64, device=device) + 0.5) / length * 2.0 - 1.0
    freq = (math.pi / 2.0) * torch.pow(2.0, torch.arange(dim // 2, dtype=torch.float64, device=device))
    ang = pos[:, None] * freq[None, :]
    return torch.cat([torch.sin(ang), torch.cos(ang)], dim=1)            # float64: callers cast to their dtype


def composite_forward(x, y, p, *, integration, norm, duplex, use_pos, centroids=None, kmeans_iters=1, img2ltnt=False, num_heads=1):
    """Same math as the kernels, in torch ops (direct op order), on whatever device x lives on.  x [B,H,W,C]."""
    B, H, W, C = x.shape
    n = H * W
    X = x.reshape(B, n, C)
    s = 1.0 / math.sqrt(C)
    if use_pos:
        Pg = grid_pos_table(H, W, p["pos_latent"].shape[1], x.device, x.dtype)
        Pl = p["pos_latent"]
    cen = None
    if duplex:
        if centroids is not None:
            cen = centroids
        else:
            Qy = y @ _e(p["wq2"]) + p["bq2"]
            Kx = X @ _e(p["wk2"]) + p["bk2"]
            if use_pos:
                Qy = Qy + (Pl @ _e(p["wpq2"]))[None]
                Kx = Kx + (Pg @ _e(p["wpk2"]))[None]
            Vx = X @ _e(p["wv2"]) + p["bv2"]
            for it in range(max(1, kmeans_iters)):
                if it > 0:
                    Qy = cen @ _e(p["wcq"]) + p["bq2"]
                    if use_pos:
                        Qy = Qy + (Pl @ _e(p["wpq2"]))[None]
                A = torch.softmax((Qy @ Kx.transpose(1, 2)) * s, dim=2)
                cen = A @ Vx
        K = cen @ _e(p["wkc"]) + p["bk"]
    else:
        K = y @ _e(p["wk"]) + p["bk"]
    Q = X @ _e(p["wq"]) + p["bq"]
    if use_pos:
        K = K + (Pl @ _e(p["wpk"]))[None]
        Q = Q + (Pg @ _e(p["wpq"]))[None]
    yv = y
    if duplex and img2ltnt:
        ym = y.mean(dim=2, keepdim=True)
        yv = (y - ym) * torch.rsqrt(((y - ym) ** 2).mean(dim=2, keepdim=True) + 1e-8) * (1.0 + cen @ _e(p["wi2l"]) + p["bi2l"])
    V = yv @ _e(p["wv"]) + p["bv"]
    if num_heads == 1:
        P = torch.softmax((Q @ K.transpose(1, 2)) * s, dim=2)
        ctl = (P @ V) @ _e(p["wo"]) + p["bo"]
    else:                                   # heads split the channels; softmax over the latents per head; scale 1/sqrt(C/heads)
        h, kk = num_heads, K.shape[1]
        sp = lambda t, L: t.reshape(B, L, h, C // h).permute(0, 2, 1, 3)
        Ph = torch.softmax((sp(Q, n) @ sp(K, kk).transpose(2, 3)) * (1.0 / math.sqrt(C / h)), dim=3)
        ctl = (Ph @ sp(V, kk)).permute(0, 2, 1, 3).reshape(B, n, C) @ _e(p["wo"]) + p["bo"]
    return integrate(X, ctl, integration, norm).reshape(B, H, W, C), cen


def grid_pos_table(H, W, pd, device, dtype):
    """The grid's sinusoidal table Pg [H*W, pd]: the row embedding of h, then the column embedding of w (pd / 2 each)."""
    half = pd // 2
    row, col = _axis(H, half, device).to(dtype), _axis(W, half, device).to(dtype)
    return torch.cat([row[:, None, :].expand(H, W, half), col[None, :, :].expand(H, W, half)], dim=2).reshape(H * W, pd)


def integrate(X, ctl, integration, norm):
    """X [B,n,C] normalised (att_norm, eps 1e-8) and modulated by the control signal ctl [B,n,C or 2C] (after its dense)."""
    C = X.shape[-1]
    if norm == "layer":
        mu = X.mean(dim=2, keepdim=True)
        Xn = (X - mu) * torch.rsqrt(((X - mu) ** 2).mean(dim=2, keepdim=True) + 1e-8)
    elif norm in (None, "none"):
        Xn = X
    else:
        dims = (1,) if norm == "instance" else (0, 1)
        mu = X.mean(dim=dims, keepdim=True)
        Xn = (X - mu) * torch.rsqrt(((X - mu) ** 2).mean(dim=dims, keepdim=True) + 1e-8)
    if integration == "mul":
        return Xn * (1.0 + ctl)
    if integration == "add":
        return Xn + ctl
    return Xn * (1.0 + ctl[..., :C]) + ctl[..., C:]


def centroid_tables(y, p, H, W, C, use_pos):
    """Duplex pass A in differentiable torch ops: (latents y [B,k,D], raw parameters) -> the tables of the centroid softmax,
    M [B,KP,C] (zero rows in the padded latents), Rt2 [B,H,KP] (-inf in the padded latents), Ct2 [B,W,KP], such that the logit
    of token (h, w) for latent j is x.M_j + Rt2[h,j] + Ct2[w,j].  Same algebra as duplex_tables in csrc/gf_fold.cu, in natural-log
    units and without TF32 rounding: M_j = Qy_j Wk2_e^T / sqrt(C), the positional terms Qy_j (Pg Wpk2_e)^T / sqrt(C) split into
    their row and column halves; bk2 is constant over the tokens and cancels in the softmax."""
    B, k, _ = y.shape
    KP = 16 if k <= 16 else 32
    s = 1.0 / math.sqrt(C)
    qy = y @ _e(p["wq2"]) + p["bq2"]
    if use_pos:
        qy = qy + (p["pos_latent"] @ _e(p["wpq2"]))[None]
    M = torch.nn.functional.pad((qy @ _e(p["wk2"]).t()) * s, (0, 0, 0, KP - k))
    if use_pos:
        half = p["pos_latent"].shape[1] // 2
        row, col = _axis(H, half, y.device).to(y.dtype), _axis(W, half, y.device).to(y.dtype)
        qp = (qy @ _e(p["wpk2"]).t()) * s                                # [B, k, pd]
        rt = torch.einsum("hp,bjp->bhj", row, qp[:, :, :half])
        ct = torch.einsum("wp,bjp->bwj", col, qp[:, :, half:])
    else:
        rt = torch.zeros(B, H, k, device=y.device, dtype=y.dtype)
        ct = torch.zeros(B, W, k, device=y.device, dtype=y.dtype)
    Rt2 = torch.cat([rt, torch.full((B, H, KP - k), -math.inf, device=y.device, dtype=y.dtype)], dim=2) if KP > k else rt
    Ct2 = torch.nn.functional.pad(ct, (0, KP - k))
    return M.contiguous(), Rt2.contiguous(), Ct2.contiguous()


def folded_tables(y, p, *, H, W, C, integration, use_pos, centroids=None, img2ltnt=False):
    """Stages W + I in differentiable torch ops: (latents y [B,k,D], raw parameters) -> the per-image tables stage T and its
    backward consume, in the workspace layout: Kp [B,KP,C], Vt [B,Cout,KP], Rt [B,H,KP] (-inf in the padded latents),
    Ct [B,W,KP].  Same algebra as csrc/gf_fold.cu.  Simplex: keys from the latents through wk.  Duplex (centroids [B,k,C] given):
    keys from the centroids through wkc; with img2ltnt the values come from the latents modulated by the centroids,
    LN(y) (1 + centroids Wi2l_e + bi2l)."""
    B, k, _ = y.shape
    KP = 16 if k <= 16 else 32
    s = 1.0 / math.sqrt(C)
    cols = [_e(p["wq"]).t() * s]
    pd = p["pos_latent"].shape[1] if use_pos else 0
    if use_pos:
        cols.append(_e(p["wpq"]).t() * s)
    cols.append((p["bq"] * s)[:, None])
    qfold = torch.cat(cols, dim=1)                                       # [C, C + pd + 1]
    kconst = p["bk"][None, :].expand(k, C)
    if use_pos:
        kconst = kconst + p["pos_latent"] @ _e(p["wpk"])
    ksrc, wk = (y, p["wk"]) if centroids is None else (centroids, p["wkc"])
    kp_all = ksrc @ (_e(wk) @ qfold) + (kconst @ qfold)[None]            # [B, k, C + pd + 1]
    Kp = torch.nn.functional.pad(kp_all[:, :, :C], (0, 0, 0, KP - k))
    kap0 = kp_all[:, :, C + pd]
    if use_pos:
        half = pd // 2
        row, col = _axis(H, half, y.device).to(y.dtype), _axis(W, half, y.device).to(y.dtype)
        rt = torch.einsum("hp,bjp->bhj", row, kp_all[:, :, C:C + half]) + kap0[:, None, :]
        ct = torch.einsum("wp,bjp->bwj", col, kp_all[:, :, C + half:C + pd])
    else:
        rt = kap0[:, None, :].expand(B, H, k)
        ct = torch.zeros(B, W, k, device=y.device, dtype=y.dtype)
    Rt = torch.cat([rt, torch.full((B, H, KP - k), -math.inf, device=y.device, dtype=y.dtype)], dim=2) if KP > k else rt
    Ct = torch.nn.functional.pad(ct, (0, KP - k))
    wo = _e(p["wo"])
    cv = p["bv"] @ wo + p["bo"]
    if integration in ("mul", "both"):
        cv = cv + torch.cat([torch.ones(C, device=y.device, dtype=y.dtype), torch.zeros(cv.numel() - C, device=y.device, dtype=y.dtype)])
    yv = y
    if centroids is not None and img2ltnt:
        ym = y.mean(dim=2, keepdim=True)
        yv = (y - ym) * torch.rsqrt(((y - ym) ** 2).mean(dim=2, keepdim=True) + 1e-8) * (1.0 + centroids @ _e(p["wi2l"]) + p["bi2l"])
    v = yv @ (_e(p["wv"]) @ wo) + cv                                     # [B, k, Cout]
    Vt = torch.nn.functional.pad(v.transpose(1, 2), (0, KP - k))
    cb = cv - p["bv"] @ wo                       # bo (+1 on the gain half): the constants attention dropout leaves unscaled
    return Kp.contiguous(), Vt.contiguous(), Rt.contiguous(), Ct.contiguous(), cb.contiguous()


class _FusedAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, centroids, return_att, names, x, y, *params):
        from .attention import bipartite_attention_forward
        pd = dict(zip(names, params))
        out, att, cen = bipartite_attention_forward(
            x.detach(), y.detach(), {k: v.detach() for k, v in pd.items()}, module._plan,
            integration=module.integration, norm=module.norm, duplex=module.kmeans_iters if module.duplex else 0, num_heads=module.num_heads,
            use_pos=module.use_pos, return_att=return_att, centroids=centroids, exact_fp32=module.exact_fp32,
            weights_version=tuple((v.data_ptr(), v._version) for v in params), img2ltnt=module.img2ltnt,
            postop=({"act": "linear", "gain": 1.0, **module.dropout_postop(x.device)} if module.dropout_postop(x.device) else None))
        ctx.module, ctx.names, ctx.centroids = module, names, centroids
        ctx.dropout = module.dropout_postop(x.device)                  # the backward regenerates the same mask (same device state)
        ctx.save_for_backward(x, y, *params)
        ctx.cen_grad = module.kernel_backward and module.duplex and centroids is None     # computed centroids, differentiable
        ctx.mark_non_differentiable(*[t for t in (att, cen) if t is not None and not (t is cen and ctx.cen_grad)])
        return out, att, cen

    @staticmethod
    def backward(ctx, g_out, g_att, g_cen):
        m = ctx.module
        x, y, *params = ctx.saved_tensors
        # grad mode on: the backward runs with create_graph=True (the generator's path-length penalty, the discriminator's R1
        # penalty) and must itself be differentiable; each route below serves both orders
        create_graph = torch.is_grad_enabled()
        kernels = m.backward_kernels_serve() and x.is_cuda and x.dtype == torch.float32
        if m.kernel_backward and m.duplex:
            if create_graph and not m.kernel_double_backward:
                raise RuntimeError("the duplex kernel backward has no derivative of its own (create_graph=True): run the layer "
                                   "through composite_forward for higher-order gradients, as Discriminator does in the R1 pass")
            if create_graph and (ctx.dropout or ctx.centroids is not None or not kernels):
                raise NotImplementedError("kernel_double_backward serves single-head duplex layers with kmeans_iters == 1, "
                                          "norm layer / none, computed centroids, no attention dropout, float32 CUDA tensors")
            if not kernels:
                raise NotImplementedError("kernel_backward serves single-head duplex layers with kmeans_iters == 1, norm layer / none, "
                                          "float32 CUDA tensors")
            route = _duplex_kernel_backward
        elif kernels and not m.duplex:
            route = _simplex_kernel_backward
        elif kernels and ctx.dropout:
            if create_graph and ctx.centroids is not None:
                raise NotImplementedError("a duplex layer with attention dropout and given centroids has no second derivative "
                                          "on the kernels")
            route = _duplex_kernel_backward
        elif ctx.dropout:
            raise NotImplementedError("attention dropout needs the backward kernels: single-head layers with norm layer / none, "
                                      "simplex or duplex with kmeans_iters == 1")
        else:
            route = _composite_backward
        return (None, None, None, None, *route(m, ctx.names, x, y, params, g_out, ctx.dropout, ctx.centroids,
                                               g_cen if ctx.cen_grad else None))


@contextlib.contextmanager
def _fp32_matmul():
    """The tables, the token reductions (K = n, up to 65,536) and the autograd through the tables of the kernel backward run as
    true fp32 GEMMs whatever torch.backends.cuda.matmul.allow_tf32 says: with TF32 the layer gradients are about 4e-4 to 9e-4
    relative off the fp64 reference instead of 1e-6 (DESIGN.md section 5)."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _alias(t):
    """A differentiable alias of t: autograd.grad with respect to it does not follow the other paths that reach t."""
    return t.view_as(t) if t.requires_grad else t.detach().requires_grad_(True)


def _leaf(t, create_graph):
    """What a backward route differentiates its recomputation with respect to: under create_graph an alias of the saved tensor, so
    the gradients it returns stay connected to the graph; otherwise a detached leaf, so that no graph outlives the call."""
    return _alias(t) if create_graph else t.detach().requires_grad_(True)


def _sum_grads(a, b):
    return [u if v is None else (v if u is None else u + v) for u, v in zip(a, b)]


# The three routes share one signature, (module, parameter names, x, y, parameters, dOut, dropout post-op, given centroids,
# cotangent of the centroids output); a route ignores what its layers cannot have.

@_fp32_matmul()
def _simplex_kernel_backward(m, names, x, y, params, g_out, dropout=None, centroids=None, g_cen=None):
    """d(loss)/d(x, y, params) of a simplex layer through gf_attn_simplex_bwd_ex (see the module docstring): the tables (with cb
    under dropout) from leaves of y and the parameters, the per-token work of ``_stage_t_backward`` (``_StageTBackward`` under
    create_graph), and autograd back through stages W and I."""
    create_graph = torch.is_grad_enabled()
    B, H, W, C = x.shape
    with torch.enable_grad():
        ys, ps = _leaf(y, create_graph), [_leaf(p, create_graph) for p in params]
        Kp, Vt, Rt, Ct, cb = folded_tables(ys, dict(zip(names, ps)), H=H, W=W, C=C, integration=m.integration, use_pos=m.use_pos)
    stage_t = _StageTBackward.apply if create_graph else _stage_t_backward
    dX, *grads = stage_t(m, y.shape[1], y.shape[2], dropout, x.contiguous(), g_out, Kp, Vt, Rt, Ct, cb if dropout else None)
    outs = [Kp, Vt, Rt, Ct] + ([cb] if dropout else [])
    return (dX, *torch.autograd.grad(outs, [ys, *ps], grads, allow_unused=True, create_graph=create_graph))


@_fp32_matmul()
def _duplex_kernel_backward(m, names, x, y, params, g_out, dropout=None, centroids=None, g_cen=None):
    """d(loss)/d(x, y, params) of a duplex layer (one k-means iteration, norm layer / none):
      1. gf_attn_centroid_stats recomputes pass A in fp32 from the tables of ``centroid_tables``: Xbar [B,k,C], lse [B,KP];
      2. Cen = Xbar Wv2_e + bv2 in torch (Xbar a leaf) and the stage-T tables from it (``folded_tables`` with centroids);
      3. stage T's backward (gf_attn_simplex_bwd_ex with a simplex descriptor of the same shape, same dropout), its token
         reductions and autograd over the tables: dX, and the gradients of y, the parameters and Xbar; with ``g_cen`` (the
         cotangent of the centroids output) Cen is one more (output, cotangent) pair of that autograd call;
      4. r = dXbar . Xbar, then gf_attn_centroid_bwd adds the pass-A part into dX and gives dS of the pass-A logits;
      5. dM = dS^T X, dRt2 / dCt2 = sums of dS, and autograd over the pass-A tables.
    y and the parameters enter the stage-T tables and the pass-A tables through separate leaves, so that the gradient of the
    stage-T tables stops at Xbar, while under create_graph Xbar stays connected to X and the pass-A tables.  There the per-token
    work of steps 1, 3 and 4 runs in ``_CentroidStats``, ``_StageTBackward`` and ``_CentroidBackward``, whose backward are the
    double-backward kernels; saved for the second pass: X, dOut and the per-image tables.  In first order it runs in their forward
    bodies, and gf_attn_centroid_bwd adds into stage T's dX in place.
    With ``centroids`` given, pass A did not run in the forward: steps 1, 4 and 5 are skipped and the centroids get no gradient."""
    create_graph = torch.is_grad_enabled()
    if create_graph:
        stats, stage_t, pass_a_backward = _CentroidStats.apply, _StageTBackward.apply, _CentroidBackward.apply
    else:
        stats, stage_t, pass_a_backward = _centroid_stats, _stage_t_backward, _centroid_backward
    B, H, W, C = x.shape
    k, D = y.shape[1], y.shape[2]
    xc = x.contiguous()
    y1, y2 = _leaf(y, create_graph), _leaf(y, create_graph)
    p1, p2 = [_leaf(p, create_graph) for p in params], [_leaf(p, create_graph) for p in params]
    d1, d2 = dict(zip(names, p1)), dict(zip(names, p2))
    if centroids is None:
        with torch.enable_grad():
            cen_tabs = centroid_tables(y2, d2, H, W, C, m.use_pos)
        xbar, lse = stats(m, k, D, xc, *cen_tabs)
        xbar.requires_grad_(True)                  # first order: a leaf of its own; under create_graph already connected
    with torch.enable_grad():
        cen = centroids.detach() if centroids is not None else xbar @ _e(d1["wv2"]) + d1["bv2"]
        Kp, Vt, Rt, Ct, cb = folded_tables(y1, d1, H=H, W=W, C=C, integration=m.integration, use_pos=m.use_pos, centroids=cen,
                                           img2ltnt=m.img2ltnt)
    dX, *grads = stage_t(m, k, D, dropout, xc, g_out, Kp, Vt, Rt, Ct, cb if dropout else None)
    outs = [Kp, Vt, Rt, Ct] + ([cb] if dropout else [])
    if g_cen is not None:
        outs, grads = outs + [cen], grads + [g_cen.contiguous()]
    leaves = [y1, *p1] + ([xbar] if centroids is None else [])
    g = list(torch.autograd.grad(outs, leaves, grads, allow_unused=True, create_graph=create_graph))
    if centroids is None:
        dxbar = g.pop()
        r = (dxbar * xbar).sum(dim=2)              # [B, k]
        dX, *g_tabs = pass_a_backward(m, k, D, xc, *cen_tabs, lse, dxbar, r, dX)
        g = _sum_grads(g, torch.autograd.grad(list(cen_tabs), [y2, *p2], g_tabs, allow_unused=True, create_graph=create_graph))
        i = 1 + names.index("bk2")     # constant over the tokens, bk2 cancels in pass A's softmax: its gradient is exactly 0
        g[i] = torch.zeros_like(params[i - 1])
    return (dX, *g)


def _composite_backward(m, names, x, y, params, g_out, dropout=None, centroids=None, g_cen=None):
    """Autograd through ``composite_forward`` recomputed from leaves of the saved tensors (the layers of this route have no
    attention dropout and no centroid cotangent)."""
    create_graph = torch.is_grad_enabled()
    with torch.enable_grad():
        xs, ys, ps = _leaf(x, create_graph), _leaf(y, create_graph), [_leaf(p, create_graph) for p in params]
        out, _ = composite_forward(xs, ys, dict(zip(names, ps)), integration=m.integration, norm=m.norm, duplex=m.duplex,
                                   use_pos=m.use_pos, centroids=centroids, kmeans_iters=m.kmeans_iters, img2ltnt=m.img2ltnt,
                                   num_heads=m.num_heads)
    return torch.autograd.grad(out, [xs, ys, *ps], g_out, allow_unused=True, create_graph=create_graph)


def _differentiable_twice(backward):
    """once_differentiable, and refusing a third derivative at once: the error node once_differentiable leaves behind is not
    visited by autograd.grad(..., inputs=...) when the inputs are reached by other paths, which would drop terms silently."""
    inner = once_differentiable(backward)

    def wrapper(ctx, *grads):
        if torch.is_grad_enabled() and any(isinstance(g, torch.Tensor) and g.requires_grad for g in grads):
            raise RuntimeError("the attention double-backward kernels have no derivative of their own: a third derivative "
                               "(create_graph=True through the R1 penalty's backward) is not supported")
        return inner(ctx, *grads)
    return wrapper


def _zeros_if_none(g, like):
    return torch.zeros_like(like) if g is None else g.contiguous()


class _StageTBackward(torch.autograd.Function):
    """The stage-T backward with its token reductions, (X, dOut, Kp, Vt, Rt, Ct) -> (dX, dKp, dVt, dRt, dCt); with attention
    dropout (the forward's mask, regenerated) cb is one more table and dcb = sum_tokens (1 - sum q) dCtl one more output.
    Forward: ``_stage_t_backward``.  Backward: gf_attn_simplex_bwd_vjp_ex (without dropout its att_dp = 0 form,
    gf_attn_simplex_bwd_vjp) and the reductions of its per-token cotangents, Kp: Sg^T X + dS^T U, Vt: Ctlg^T P + dCtl^T dPg,
    Rt / Ct: sums of Sg, cb: (1 - sum P) Ctlg - (sum dPg) dCtl."""

    @staticmethod
    def forward(ctx, m, k, D, dropout, x, g_out, Kp, Vt, Rt, Ct, cb):
        gc = g_out.contiguous()
        ctx.m, ctx.k, ctx.D, ctx.dropout = m, k, D, dropout or {}
        ctx.save_for_backward(x, gc, Kp, Vt, Rt, Ct, cb)
        return _stage_t_backward(m, k, D, dropout, x, gc, Kp, Vt, Rt, Ct, cb)

    @staticmethod
    @_differentiable_twice
    @_fp32_matmul()
    def backward(ctx, gdX, gKp, gVt, gRt, gCt, *gcb):
        x, go, Kp, Vt, Rt, Ct, cb = ctx.saved_tensors
        dpo = ctx.dropout
        B, H, W, C = x.shape
        n, KP, Cout = H * W, Kp.shape[1], Vt.shape[1]
        U = _zeros_if_none(gdX, x)
        cots = [_zeros_if_none(g, t) for g, t in ((gKp, Kp), (gVt, Vt), (gRt, Rt), (gCt, Ct))]
        Xg, dOg = torch.empty_like(x), torch.empty_like(x)
        Sg, dPg, dS, P = (torch.empty((B, n, KP), dtype=torch.float32, device=x.device) for _ in range(4))
        Ctlg, dCtl = (torch.empty((B, n, Cout), dtype=torch.float32, device=x.device) for _ in range(2))
        if dpo:                                  # the mask of the forward, regenerated from the same device state
            name, dp_args = "gf_attn_simplex_bwd_vjp_ex", (*_dropout_args(dpo), cb, _zeros_if_none(gcb[0], cb))
        else:                                    # the same kernel: the dropout-free entry is _ex at att_dp = 0
            name, dp_args = "gf_attn_simplex_bwd_vjp", ()
        _launch(name, _desc(ctx.m, x, ctx.k, ctx.D, duplex=0), x, go, Kp, Vt, Rt, Ct, U, *cots, Xg, dOg, Sg, dPg, Ctlg, dS, P, dCtl,
                *dp_args)
        X2, U2 = x.reshape(B, n, C), U.reshape(B, n, C)
        gKp_ = torch.bmm(Sg.transpose(1, 2), X2) + torch.bmm(dS.transpose(1, 2), U2)
        gVt_ = torch.bmm(Ctlg.transpose(1, 2), P) + torch.bmm(dCtl.transpose(1, 2), dPg)
        Sg4 = Sg.reshape(B, H, W, KP)
        gcb_ = None
        if dpo:                                  # cb: sum_tokens qdef gbar - F dCtl, qdef = 1 - sum q, F = sum_j fq_j
            gcb_ = ((1.0 - P.sum(dim=2, keepdim=True)) * Ctlg - dPg.sum(dim=2, keepdim=True) * dCtl).sum(dim=(0, 1))
        return None, None, None, None, Xg, dOg, gKp_, gVt_, Sg4.sum(dim=2), Sg4.sum(dim=1), gcb_


class _CentroidStats(torch.autograd.Function):
    """Pass A's statistics, (X, M, Rt2, Ct2) -> (Xbar, lse) (``_centroid_stats``).  Backward: with cotangents dXbar and lseg,
    d lse_j / d s[t,j] = A[t,j], so it is ``_centroid_backward`` with r = dXbar . Xbar - lseg and dX starting from zero."""

    @staticmethod
    def forward(ctx, m, k, D, x, Mt, Rt2, Ct2):
        xbar, lse = _centroid_stats(m, k, D, x, Mt, Rt2, Ct2)
        ctx.m, ctx.k, ctx.D = m, k, D
        ctx.save_for_backward(x, Mt, Rt2, Ct2, xbar, lse)
        return xbar, lse

    @staticmethod
    @_differentiable_twice
    @_fp32_matmul()
    def backward(ctx, gxbar, glse):
        x, Mt, Rt2, Ct2, xbar, lse = ctx.saved_tensors
        gxbar = _zeros_if_none(gxbar, xbar)
        r = (gxbar * xbar).sum(dim=2)
        if glse is not None:
            r = r - glse[:, :ctx.k]
        return None, None, None, *_centroid_backward(ctx.m, ctx.k, ctx.D, x, Mt, Rt2, Ct2, lse, gxbar, r, torch.zeros_like(x))


class _CentroidBackward(torch.autograd.Function):
    """The pass-A backward with its token reductions, (X, M, Rt2, Ct2, lse, dXbar, r, dX_in) -> (dX_out, dM, dRt2, dCt2).
    Forward: ``_centroid_backward`` into a copy of dX_in (never into a tensor autograd tracks).  Backward:
    gf_attn_centroid_bwd_vjp and the reductions dXbar: A^T U + Gg^T X, M: Sg^T X + dS^T U, r: -sum_t Gg, lse: -sum_t Sg."""

    @staticmethod
    def forward(ctx, m, k, D, x, Mt, Rt2, Ct2, lse, dxbar, r, dX_in):
        dxbar, r = dxbar.contiguous(), r.contiguous()
        ctx.m, ctx.k, ctx.D = m, k, D
        ctx.save_for_backward(x, Mt, Rt2, Ct2, lse, dxbar, r)
        return _centroid_backward(m, k, D, x, Mt, Rt2, Ct2, lse, dxbar, r, dX_in.contiguous().clone())

    @staticmethod
    @_differentiable_twice
    @_fp32_matmul()
    def backward(ctx, gdX, gM, gRt2, gCt2):
        x, Mt, Rt2, Ct2, lse, dxbar, r = ctx.saved_tensors
        B, H, W, C = x.shape
        n, KP, k = H * W, Mt.shape[1], ctx.k
        U = _zeros_if_none(gdX, x)
        cots = [_zeros_if_none(g, t) for g, t in ((gM, Mt), (gRt2, Rt2), (gCt2, Ct2))]
        Xg = torch.empty_like(x)
        Sg, Gg, A, dS = (torch.empty((B, n, KP), dtype=torch.float32, device=x.device) for _ in range(4))
        _launch("gf_attn_centroid_bwd_vjp", _desc(ctx.m, x, k, ctx.D, duplex=1), x, Mt, Rt2, Ct2, lse, dxbar, r, U, *cots, Xg, Sg, Gg,
                A, dS)
        X2, U2 = x.reshape(B, n, C), U.reshape(B, n, C)
        gM_ = torch.bmm(Sg.transpose(1, 2), X2) + torch.bmm(dS.transpose(1, 2), U2)
        gxbar = (torch.bmm(A.transpose(1, 2), U2) + torch.bmm(Gg.transpose(1, 2), X2))[:, :k]
        Sg4 = Sg.reshape(B, H, W, KP)
        return (None, None, None, Xg, gM_, Sg4.sum(dim=2), Sg4.sum(dim=1), -Sg.sum(dim=1), gxbar, -Gg.sum(dim=1)[:, :k], U)


def _desc(m, x, k, D, duplex):
    """The descriptor of a backward entry for layer m on x [B,H,W,C]: one head, no flags; duplex = 0 for stage T (a duplex
    layer's too, its keys are folded from the centroids), 1 for pass A."""
    B, H, W, C = x.shape
    return _lib.make_desc(B, H, W, C, k, D, heads=1, norm=m.norm, integration=m.integration, pos_dim=m.pos_dim if m.use_pos else 0,
                          duplex=duplex, flags=0)


def _launch(name, desc, *args):
    """The library entry ``name`` on (desc, *args, the current stream) of the device of args[0], the X every backward entry
    takes first.  Tensors go by data pointer, None as NULL."""
    dev = args[0].device
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.load(), name)(ctypes.byref(desc), *ptrs, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   name)


def _dropout_args(dropout):
    """(att_dp, dp_salt, dp_state) of the forward's dropout post-op, with which a backward entry regenerates its mask: att_dp = 0
    and a NULL state without dropout."""
    dpo = dropout or {}
    return ctypes.c_float(dpo.get("att_dp", 0.0)), int(dpo.get("dp_salt", 0)), dpo.get("dp_state")


def _centroid_stats(m, k, D, x, Mt, Rt2, Ct2):
    """gf_attn_centroid_stats: pass A recomputed in fp32 -> (Xbar [B,k,C], lse [B,KP])."""
    B, _, _, C = x.shape
    desc = _desc(m, x, k, D, duplex=1)
    xbar = torch.empty((B, k, C), dtype=torch.float32, device=x.device)
    lse = torch.empty((B, Mt.shape[1]), dtype=torch.float32, device=x.device)
    part = torch.empty(_lib.workspace_bytes(desc), dtype=torch.uint8, device=x.device)       # split-n partials
    _launch("gf_attn_centroid_stats", desc, x, Mt, Rt2, Ct2, xbar, lse, part)
    return xbar, lse


def _centroid_backward(m, k, D, x, Mt, Rt2, Ct2, lse, dxbar, r, dX):
    """gf_attn_centroid_bwd, which adds the pass-A part of the activation gradient into dX in place and gives dS [B,n,KP] of the
    pass-A logits, and the reductions of dS over the tokens: (dX, dM = dS^T X, dRt2, dCt2)."""
    B, H, W, C = x.shape
    KP = Mt.shape[1]
    dS = torch.empty((B, H * W, KP), dtype=torch.float32, device=x.device)
    _launch("gf_attn_centroid_bwd", _desc(m, x, k, D, duplex=1), x, Mt, Rt2, Ct2, lse, dxbar.contiguous(), r.contiguous(), dX, dS)
    dS4 = dS.reshape(B, H, W, KP)
    return dX, torch.bmm(dS.transpose(1, 2), x.reshape(B, H * W, C)), dS4.sum(dim=2), dS4.sum(dim=1)


def _stage_t_backward(m, k, D, dropout, x, g_out, Kp, Vt, Rt, Ct, cb):
    """gf_attn_simplex_bwd_ex and the reductions over the tokens: (dX, dKp, dVt, dRt, dCt), and dcb under dropout, the gradients
    autograd takes back through stages W and I.  cb: the unscaled control-signal constants, None without dropout."""
    B, H, W, C = x.shape
    n = H * W
    KP, Cout = Kp.shape[1], Vt.shape[1]
    xc, gc = x.detach().contiguous(), g_out.detach().contiguous()
    dX = torch.empty_like(xc)
    dS = torch.empty((B, n, KP), dtype=torch.float32, device=x.device)
    P = torch.empty_like(dS)
    dCtl = torch.empty((B, n, Cout), dtype=torch.float32, device=x.device)
    _launch("gf_attn_simplex_bwd_ex", _desc(m, x, k, D, duplex=0), xc, gc, Kp, Vt, Rt, Ct, dX, dS, P, dCtl, *_dropout_args(dropout), cb)
    # reductions over the tokens: plain batched GEMMs / sums
    dKp = torch.bmm(dS.transpose(1, 2), xc.reshape(B, n, C))             # [B, KP, C]
    dVt = torch.bmm(dCtl.transpose(1, 2), P)                             # [B, Cout, KP]
    dS4 = dS.reshape(B, H, W, KP)
    grads = [dKp, dVt, dS4.sum(dim=2), dS4.sum(dim=1)]
    if dropout:                                  # ctl = sum_j q_j (Vt_j - cb) + cb: the constants' own gradient
        grads.append((dCtl * (1.0 - P.sum(dim=2, keepdim=True))).sum(dim=(0, 1)))
    return (dX, *grads)


def bipartite_attention_autograd(module, x, y, centroids, return_att):
    names = tuple(n for n, _ in module.named_parameters(recurse=False))
    params = tuple(p for _, p in module.named_parameters(recurse=False))
    return _FusedAttention.apply(module, centroids, return_att, names, x, y, *params)
