"""fp64 references of the attention forward kernels at their C boundary, and the exact-integer test cases (csrc/gf_tc.cu
token_tc_kernel and csrc/gf_simt.cu token_simt_kernel through gf_attn_simplex_fwd_ex; csrc/gf_tc_cen.cu centroid_tc_kernel through
gf_attn_duplex_fwd_ex).

TEST INFRASTRUCTURE ONLY (see oracle/bipartite.py).  The stage-T reference is ``folded.per_token`` in fp64 followed by the fused
epilogue of ``gf_attn_postop``:

  y   = per_token(x * d)                                  (d = in_scale: K' already carries it, as stage I folds it)
  y'' = act(y + noise * strength + bias) * gain            (leaky-ReLU(0.2) or linear)
  rgb = sum_c y'' rgb_w + rgb_bias                         (fused tRGB: reads the output BEFORE post_scale)
  out = y'' * post_scale

Multi-head layers run one softmax per segment of ``seg`` table columns, and the attention map is the mean over the heads.

The exact cases are those of ``attn_bwd.exact_stage_t_case`` per head: every probability is 0, 1/2 or 1, every logit an integer
below 2^24, so the same tables give the same outputs in natural and in log2 units (both kernel families run them).
``stage_t_exactness`` lists the intermediates so that a test can check that claim instead of assuming it.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import folded as of
from . import philox as ph
from .attn_bwd import GAP, OFFSET

Tensor = torch.Tensor
TF32_TRUNC_COMP = 1.000352220        # K' and pass A's flush carry this factor (gf_fold.cu GF_TF32_TRUNC_COMP), as float32
LOG2E = 1.4426950408889634


def _combine(Xn, GB, integration, C):
    if integration == "mul":
        return Xn * GB
    if integration == "add":
        return Xn + GB
    return Xn * GB[..., :C] + GB[..., C:]


def stage_t_forward(X, Kp, Vt, Rt, Ct, *, H, W, k, integration, norm, heads=1, mult=None, cb=None,
                    post: Optional[dict] = None) -> Dict[str, Optional[Tensor]]:
    """What gf_attn_simplex_fwd_ex writes for tables in natural-log units, in fp64: Xout [B,n,C], att [B,n,k] and rgb [B,3,n]
    (None without a tRGB).  Kp is the table as stage I writes it (in_scale folded in).  post: in_scale [B,C], bias [C],
    noise [n] or [B,n], strength, act (0 / 1), gain, post_scale [B,C], rgb_w [B,3,C], rgb_bias [3]; any may be missing."""
    post = post or {}
    X, Kp, Vt, Rt, Ct = (t.double() for t in (X, Kp, Vt, Rt, Ct))
    B, n, C = X.shape
    KP = Kp.shape[1]
    d = post.get("in_scale")
    d = torch.ones(B, 1, C, dtype=torch.float64) if d is None else d.double()[:, None, :]
    Xin = X * d
    cbd = None if cb is None else cb.double()
    if heads == 1:
        out, att = of.per_token(Xin, Kp / d, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm, return_att=True, k=k,
                                att_mult=mult, cb=cbd)
    else:
        assert mult is None and norm in (None, "none")
        seg = KP // heads
        S = X @ Kp.transpose(1, 2) + (Rt[:, :, None, :] + Ct[:, None, :, :]).reshape(B, n, KP)
        P = torch.softmax(S.reshape(B, n, heads, seg), dim=3).reshape(B, n, KP)
        att = P.reshape(B, n, heads, seg)[..., :k].mean(dim=2)
        out = _combine(Xin, P @ Vt.transpose(1, 2), integration, C)
    rgb = None
    if post:
        y = out
        if post.get("noise") is not None:
            y = y + post["noise"].double().reshape(-1, n)[:, :, None] * post.get("strength", 1.0)
        if post.get("bias") is not None:
            y = y + post["bias"].double()
        gain = post.get("gain", 1.0)
        y = torch.where(y >= 0, y * gain, y * (0.2 * gain)) if post.get("act", 0) == 1 else y * gain   # 0.2 * 5 == 1 in fp64
        if post.get("rgb_w") is not None:
            rgb = torch.einsum("btc,boc->bot", y, post["rgb_w"].double())
            if post.get("rgb_bias") is not None:
                rgb = rgb + post["rgb_bias"].double()[None, :, None]
        if post.get("post_scale") is not None:
            y = y * post["post_scale"].double()[:, None, :]
        out = y
    return dict(Xout=out, att=att, rgb=rgb)


def exact_stage_t_case(B, H, W, C, k, integration, *, heads=1, dropout=False, seed: int, salt: int = 11, dp_seed: int = 20261015,
                       step: int = 3):
    """Synthetic stage-T tables whose arithmetic is exact (norm none), in the construction of attn_bwd.exact_stage_t_case, once per
    head: in each head's segment the latents come in pairs, Rt adds OFFSET to one pair of each row (a different pair per head),
    and the two keys of a pair differ by +-GAP in two channels, so inside the pair the logits differ by a multiple of GAP: a
    one-hot pair or an exact tie at 1/2.  The padded columns have Rt = -inf and nonzero keys, values and Ct.  x, V^T and cb are
    small integers; with dropout (p = 1/2) the multipliers are 0 or 2."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(heads * (8 if k <= 8 else 16)) if heads > 1 else of.pad_k(k)
    seg = KP // heads
    Cout = 2 * C if integration == "both" else C
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    sparse = lambda lo, hi, keep, *shape: ri(lo, hi, *shape) * (torch.rand(shape, generator=g) < keep).double()
    X = ri(-2, 2, B, n, C)
    Kp = ri(-1, 1, B, KP, C)
    Rt = GAP * sparse(-1, 1, 0.25, B, H, KP)
    Ct = GAP * sparse(-1, 1, 0.25, B, W, KP)
    npairs = (k + 1) // 2
    for h in range(heads):
        c0 = h * seg
        for j in range(1, k, 2):                                           # the partner shares the keys up to two channels
            Kp[:, c0 + j] = Kp[:, c0 + j - 1]
            ch = torch.randint(0, C, (B, 2), generator=g)
            Kp[torch.arange(B)[:, None], c0 + j, ch] += GAP * torch.tensor([1.0, -1.0]).expand(B, 2)
        alpha = torch.randint(0, npairs, (B, H), generator=g)              # the winning pair of each row, drawn per head
        pair = torch.arange(seg) // 2
        Rt[:, :, c0:c0 + seg] += OFFSET * (pair[None, None, :] == alpha[:, :, None]).double()
        Rt[:, :, c0 + k:c0 + seg] = -math.inf
        Ct[:, :, c0 + k:c0 + seg] = ri(-3, 3, B, W, seg - k)
    Vt = ri(-1, 1, B, Cout, KP)
    cb = ri(-2, 2, Cout)
    mult = None
    if dropout:
        mult = torch.from_numpy(ph.dropout_mult(0.5, dp_seed, step, salt, B * n, KP).reshape(B, n, KP).copy()).double()
    return dict(X=X, Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct, cb=cb, mult=mult, att_dp=0.5 if dropout else 0.0, salt=salt, dp_seed=dp_seed,
                step=step, heads=heads, KP=KP)


def exact_postop(B, n, C, *, seed: int, act: int, rgb: bool, per_image_noise: bool, scales: bool):
    """A fused epilogue whose every step is exact on an exact case: integer bias, noise and tRGB weights, strength 1/2, leaky-ReLU
    with gain 5 (0.6f * 5 == 3 and 0.4f * 5 == 2 in fp32) or linear with gain 1, in_scale 1 or 2 and post_scale a power of two (not
    all 1, so tRGB before or after it differ)."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    post = dict(bias=ri(-3, 3, C), noise=ri(-2, 2, B if per_image_noise else 1, n), strength=0.5, act=act,
                gain=5.0 if act == 1 else 1.0)
    if scales:
        post["in_scale"] = 2.0 ** ri(0, 1, B, C)                        # 1 or 2: the logits of a pair still differ by GAP multiples
        post["post_scale"] = 2.0 ** ri(-2, 2, B, C)
        post["post_scale"][:, 0] = 4.0
    if rgb:
        post["rgb_w"] = ri(-3, 3, B, 3, C)
        post["rgb_bias"] = ri(-2, 2, 3)
    return post


def _grain(*terms):
    """The largest power of two (at most 1) that divides every finite entry of the terms."""
    m = 0
    for t in terms:
        v = t[torch.isfinite(t)].abs()
        v = v[v > 0]
        while m < 60 and not torch.equal((v * 2.0 ** m).round(), v * 2.0 ** m):
            m += 1
    return 2.0 ** -m


def stage_t_exactness(case, *, k, integration, post: Optional[dict] = None):
    """The intermediates of both kernels' arithmetic on an exact case (norm none), as (name, value, companion, grain): every
    partial sum of a value is a multiple of grain whose magnitude is at most the companion, so when companion / grain < 2^24
    fp32 holds every partial sum exactly in any order.  Also returns the probabilities p (before dropout), [B,n,KP]."""
    post = post or {}
    X, Kp, Vt, Rt, Ct = (case[n].double() for n in ("X", "Kp", "Vt", "Rt", "Ct"))
    heads, KP = case["heads"], case["KP"]
    B, n, C = X.shape
    seg = KP // heads
    d = post.get("in_scale")
    d = torch.ones(B, 1, C, dtype=torch.float64) if d is None else d.double()[:, None, :]
    Kt = Kp * d                                                          # the table as stage I writes it
    RC = (Rt[:, :, None, :] + Ct[:, None, :, :]).reshape(B, n, KP)
    fin = torch.isfinite(RC)
    RCf = torch.where(fin, RC, torch.zeros_like(RC))
    RCa = torch.where(fin, (Rt[:, :, None, :].abs() + Ct[:, None, :, :].abs()).reshape(B, n, KP), torch.zeros_like(RC))
    S = X @ Kt.transpose(1, 2) + RCf
    s_abs = X.abs() @ Kt.abs().transpose(1, 2) + RCa
    p = torch.softmax(torch.where(fin, S, torch.full_like(S, -math.inf)).reshape(B, n, heads, seg), dim=3).reshape(B, n, KP)
    mult = case["mult"]
    mk = torch.ones_like(p) if mult is None else mult.double()
    q = p * mk
    cbd = case["cb"].double() if mult is not None else torch.zeros(Vt.shape[1], dtype=torch.float64)
    qdef = 1.0 - q.sum(dim=2, keepdim=True)
    G = q @ Vt.transpose(1, 2) + qdef * cbd
    G_abs = q @ Vt.abs().transpose(1, 2) + qdef.abs() * cbd.abs()
    att = p.reshape(B, n, heads, seg)[..., :k].mean(dim=2)
    xin = X * d
    if integration == "add":
        y, y_abs = xin + G, xin.abs() + G_abs
    elif integration == "mul":
        y, y_abs = xin * G, xin.abs() * G_abs
    else:
        y, y_abs = xin * G[..., :C] + G[..., C:], xin.abs() * G_abs[..., :C] + G_abs[..., C:]
    items = [("logits", S, s_abs, _grain(X[..., None, :] * Kt[:, None, :, :], RCf)), ("p", p, p, 0.5), ("q", q, q, 0.5),
             ("qdef", qdef, 1.0 + q.sum(2, keepdim=True), 0.5), ("att", att, att, 0.5 / heads),
             ("ctl", G, G_abs, _grain(q[..., None] * Vt[:, None].transpose(2, 3), qdef * cbd)),
             ("xin", xin, xin.abs(), _grain(xin)), ("modulated", y, y_abs, _grain(xin, G) ** 2)]
    if post:
        nz = post["noise"].double().reshape(-1, n)[:, :, None] * post.get("strength", 1.0)
        y = y + nz + post["bias"].double()
        y_abs = y_abs + nz.abs() + post["bias"].double().abs()
        items.append(("noise_bias", y, y_abs, _grain(y, nz, post["bias"].double()) * _grain(xin, G) ** 2))
        gain = post.get("gain", 1.0)
        a, b = (0.6 * gain, 0.4 * gain) if post.get("act", 0) == 1 else (gain, 0.0)
        assert float(torch.tensor(a, dtype=torch.float32)) == a and float(torch.tensor(b, dtype=torch.float32)) == b
        y, y_abs = a * y + b * y.abs(), (a + b) * y_abs
        items.append(("act", y, y_abs, _grain(y)))
        if post.get("rgb_w") is not None:
            w = post["rgb_w"].double()
            rgb = torch.einsum("btc,boc->bot", y, w) + post["rgb_bias"].double()[None, :, None]
            rgb_abs = torch.einsum("btc,boc->bot", y_abs, w.abs()) + post["rgb_bias"].double().abs()[None, :, None]
            items.append(("rgb", rgb, rgb_abs, _grain(y) * _grain(w)))
        if post.get("post_scale") is not None:
            ps = post["post_scale"].double()[:, None, :]
            items.append(("post_scale", y * ps, y_abs * ps, _grain(y * ps)))
    return items, p


# ---- duplex pass A on wgmma --------------------------------------------------------------------------------------------------
def pass_a_split_ranges(n, nsplit):
    """Token range of every split of centroid_tc_kernel, empty ones included: contiguous runs of ceil(tiles / nsplit) 64-token
    tiles (the split count is chosen in 128-token tiles, so the last splits can be empty)."""
    tiles = (n + 63) // 64
    per = (tiles + nsplit - 1) // nsplit
    return [(min(n, s * per * 64), min(n, (s + 1) * per * 64)) for s in range(nsplit)]


def exact_pass_a_case(B, H, W, C, k, *, winners: Tensor, seed: int, runners_up: Optional[Tensor] = None,
                      ties: Optional[Tensor] = None):
    """Pass-A tables in log2 units whose arithmetic is exact on the tensor path; winners [B,k] token indices.  The winner's row and
    column carry OFFSET in Rt2 / Ct2, so its logit is 2 OFFSET plus a small integer and every other token lies at least OFFSET
    below it (E = 2^(s - m) is 1 or 0).  x is an integer in [-8, 8] and M is 0 or +-1 (TF32 values).  The padded latents have
    Rt2 = -inf and nonzero M and Ct2.

    runners_up [B,k,2] / ties [B,k] (entries < 0: none) plant tokens in the winner's column whose row carries OFFSET plus exactly
    what puts their logit one below the winner's (a runner-up) or equal to it (a tie); no other token of that row or column
    comes near.  Returns the tables, the logits L [B,n,KP] and the planted tokens' relative weights wts [B,k,n] (2^(L - max))."""
    g = torch.Generator().manual_seed(seed)
    n, KP = H * W, of.pad_k(k)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    X = ri(-8, 8, B, n, C)
    M = ri(-1, 1, B, KP, C)
    Rt2 = ri(-3, 3, B, H, KP)
    Ct2 = ri(-3, 3, B, W, KP)
    bi = torch.arange(B)[:, None].expand(B, k)
    ji = torch.arange(k)[None, :].expand(B, k)
    Rt2[bi, winners // W, ji] += OFFSET
    Ct2[bi, winners % W, ji] += OFFSET
    Rt2[:, :, k:] = -math.inf
    planted = []
    if runners_up is not None:
        planted += [(runners_up[..., i], -1.0) for i in range(runners_up.shape[-1])]
    if ties is not None:
        planted.append((ties, 0.0))
    for toks, delta in planted:
        for b in range(B):
            for j in range(k):
                t, w_ = int(toks[b, j]), int(winners[b, j])
                if t < 0:
                    continue
                assert t % W == w_ % W and t // W != w_ // W, "a planted token shares the winner's column, not its row"
                lw = X[b, w_] @ M[b, j] + Rt2[b, w_ // W, j] + Ct2[b, w_ % W, j]
                Rt2[b, t // W, j] = lw + delta - X[b, t] @ M[b, j] - Ct2[b, t % W, j]
    L = X @ M.transpose(1, 2) + (Rt2[:, :, None, :] + Ct2[:, None, :, :]).reshape(B, n, KP)
    Lk = L[:, :, :k].transpose(1, 2)                                     # [B,k,n]
    wts = torch.exp2(Lk - Lk.amax(dim=2, keepdim=True))
    wts = torch.where(wts >= 2.0 ** -60, wts, torch.zeros_like(wts))    # what fp32 makes of 2^(-OFFSET)
    return dict(X=X, M=M, Rt2=Rt2, Ct2=Ct2), L, wts


def exact_pass_a_xbar(X, wts, ranges, scale=None):
    """Xbar of an exact pass-A case as the tensor path forms it: per split, acc = sum_t w_t x_t and l = sum_t w_t (exact), the
    flush multiplies acc by the truncation compensation in fp32; the merge (every split at the maximum has weight exactly 1) adds
    the partials in split order in fp32, divides by the summed l and scales by the load-side scale d."""
    B, k, n = wts.shape
    c = torch.tensor(TF32_TRUNC_COMP, dtype=torch.float32)
    num = torch.zeros(B, k, X.shape[2], dtype=torch.float32)
    den = torch.zeros(B, k, 1, dtype=torch.float32)
    for lo, hi in ranges:
        if hi <= lo:
            continue
        w = wts[:, :, lo:hi]
        acc = (w @ X[:, lo:hi].double()).float()                         # exact: few nonzero weights of 1 or 1/2, small integers
        l = w.sum(dim=2, keepdim=True).float()
        live = (l > 0).float()                                          # a split without a planted token has weight 0 here
        num = num + live * (acc * c)
        den = den + l
    out = num / den
    if scale is not None:
        out = out * scale.float()[:, None, :]
    return out.double()
