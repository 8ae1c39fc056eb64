"""Exact cases of stage W (gf_attn_fold_weights) and stage I (the per-image tables), and the bits the kernels must write for them.

TEST INFRASTRUCTURE ONLY (see oracle/bipartite.py).  csrc/gf_fold.cu folds the weights with a chain of fp32 GEMMs and scaled copies
and builds the tables with fp32 FMA chains; ``stage_w`` and ``tables`` restate that chain step by step in fp64.  Every step checks
that its fp32 counterpart is exact (``exact_mm``): all operands fp32 values, every product and every partial sum, in any order,
a multiple of the step's grid and below 2^24 of it.  Then the fp64 value IS the fp32 result, whatever order the kernel sums in.

The cases (``exact_weights``): raw weights in {-2..2}, integer latents, every fan-in a power of four, so every equalised-LR scale is a
power of two.  The positional weights are one-hot: wpq and wpk (wpk2 and wpq2) map positional channel q to key channel c_q alone,
the key weights see nothing of the c_q channels and the latents' positional rows hold one power of two per half.  Then each
latent's kappa row has at most one nonzero entry per half, a power of two, and every Rt / Ct entry is one fp32 sin / cos value times
that power of two (exact), plus kappa_0 (one fp32 rounding).

The only inexact steps are the ones the kernels round on purpose, emulated here bit for bit:
  * the positional axis tables: fp32(sin / cos) of the fp64 angle (``pos_axis``; ``pos_midpoint_margin`` shows that no value
    lies near an fp32 rounding midpoint, so a few-ulp difference between the device's and the host's fp64 sin cannot flip it);
  * Rt / Ct: fp32(product + kappa_0), then (tensor path) fp32(. * log2 e);
  * K' (tensor path): tf32_rne(fp32(K' d kf)), kf = fp32(1.000352220f * log2 e); V^T: tf32_rne(V^T);
  * the TF32 key GEMM: one fma.rn.f32 of alpha = fp32(1.000352220f^2) with the exact sum S and the constant row, fp32(alpha S + CK).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .bipartite import LN_EPS, sinusoidal_axis
from .tf32 import tf32_rne, tf32_trunc

Tensor = torch.Tensor
F32 = torch.float32
COMP = float(torch.tensor(1.000352220, dtype=F32))
LOG2E_F = float(torch.tensor(1.4426950408889634, dtype=F32))
KF = float(torch.tensor(COMP, dtype=F32) * torch.tensor(LOG2E_F, dtype=F32))        # constexpr kf of finalize / stage_i_kernel
COMP2 = float(torch.tensor(COMP, dtype=F32) * torch.tensor(COMP, dtype=F32))        # gemm_tc's alpha * comp with alpha = 1


def _lsb_log2(x: Tensor) -> Tensor:
    """log2 of the lowest set bit of each (fp64, finite) value; zeros get a huge value (no constraint)."""
    m, e = torch.frexp(x)
    mi = (m.abs() * 2.0 ** 53).to(torch.int64)
    low = mi & (-mi)
    tz = torch.log2(low.clamp_min(1).double()).round().to(torch.int64)
    return torch.where(x == 0, torch.full_like(e, 1 << 20, dtype=torch.int64), e.to(torch.int64) - 53 + tz)


def significant_bits(x: Tensor) -> Tensor:
    """Significant bits of each fp64 value (0 for zero)."""
    m, _ = torch.frexp(x)
    mi = (m.abs() * 2.0 ** 53).to(torch.int64)
    low = mi & (-mi)
    tz = torch.log2(low.clamp_min(1).double()).round()
    return torch.where(x == 0, torch.zeros_like(tz), 53 - tz)


def assert_f32(x: Tensor, name: str):
    assert torch.equal(x.float().double(), x), f"{name}: not an fp32 value"


def exact_mm(A: Tensor, B: Tensor, *, alpha: float = 1.0, E: Optional[Tensor] = None, name: str = "") -> Tensor:
    """alpha * A @ B (+ E) in fp64, after proving that fp32 arithmetic forms it exactly in any summation order: the operands are fp32
    values, alpha a power of two, and for each output element the sum of |products| (+ |E|) stays below 2^24 times the coarsest
    grid all of its terms lie on (the lowest set bit of A's row times that of B's column, and of E's element)."""
    assert alpha != 0 and math.frexp(abs(alpha))[0] == 0.5, f"{name}: alpha {alpha} is not a power of two"
    assert_f32(A, name + " A")
    assert_f32(B, name + " B")
    ga = _lsb_log2(A).amin(dim=-1, keepdim=True)                       # [.., M, 1]
    gb = _lsb_log2(B).amin(dim=-2, keepdim=True)                       # [.., 1, N]
    g = ga + gb
    tot = A.abs() @ B.abs()
    out = A @ B
    if E is not None:
        E = E.expand_as(out)
        assert_f32(E, name + " E")
        g = torch.minimum(g, _lsb_log2(E) - int(round(math.log2(abs(alpha)))))
        tot = tot + E.abs() / abs(alpha)
    g = g.clamp(max=1000)
    ok = torch.ldexp(tot, -g) < 2.0 ** 24
    assert ok.all(), f"{name}: {int((~ok).sum())} elements not exact in fp32"
    r = alpha * out + (E if E is not None else 0.0)
    assert_f32(r, name)
    return r


# ---- the cases ---------------------------------------------------------------------------------------------------------------
def pos_channels(C: int, p: int):
    """Key channel c_q of positional channel q (spread over the channels, so over the heads)."""
    return [q * (C // p) for q in range(p)] if p else []


def exact_weights(C: int, D: int, k: int, p: int, integration: str, *, duplex: bool = False, wcq: bool = False,
                  seed: int) -> Dict[str, Tensor]:
    """Raw weights of an exact case (see the module docstring); fp64."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda *shape: torch.randint(-2, 3, shape, generator=g).double()
    cout = 2 * C if integration == "both" else C
    w = dict(wq=ri(C, C), bq=ri(C), wk=ri(D, C), bk=ri(C), wv=ri(D, C), bv=ri(C), wo=ri(C, cout), bo=ri(cout))
    cq = pos_channels(C, p)
    onehot = torch.zeros(p, C, dtype=torch.float64)
    for q, c in enumerate(cq):
        onehot[q, c] = 1.0
    w["wpq"], w["wpk"] = onehot.clone(), onehot.clone()
    pl = torch.zeros(k, p, dtype=torch.float64)
    half = p // 2
    for j in range(k):
        for h0 in (0, half):
            if p:
                q = h0 + int(torch.randint(0, half, (1,), generator=g))
                pl[j, q] = float(2 ** int(torch.randint(-1, 2, (1,), generator=g))) * (1 - 2 * int(torch.randint(0, 2, (1,), generator=g)))
    w["pos_latent"] = pl
    if duplex:
        # wv2 a signed permutation (entries +-1, +-2): AK2 = WV2 AK keeps AK's significant bits, so it stays a TF32 value
        wv2 = torch.zeros(C, C, dtype=torch.float64)
        wv2[torch.arange(C), torch.randperm(C, generator=g)] = ri(C).masked_fill(ri(C) == 0, 1.0).sign() * (1 + (ri(C) > 0).double())
        w.update(wq2=ri(D, C), bq2=ri(C), wk2=ri(C, C), bk2=ri(C), wv2=wv2, bv2=ri(C), wkc=ri(C, C))
        w["wpq2"], w["wpk2"] = onehot.clone(), onehot.clone()
        if wcq:
            w["wcq"] = ri(C, C)
    for name in ("wk", "wkc", "wq2", "wcq"):               # the key / query folds see nothing of the positional channels
        if name in w:
            w[name][:, cq] = 0.0
    for name in ("bk", "bq2"):
        if name in w:
            w[name][cq] = 0.0
    return w


def exact_latents(B: int, k: int, D: int, seed: int) -> Tensor:
    """Integer latents in [-8, 8]: the V^T values reach 12 and 13 significant bits, so the TF32 rounding of V^T meets ties."""
    return torch.randint(-8, 9, (B, k, D), generator=torch.Generator().manual_seed(seed)).double()


# ---- stage W, in the kernel's order ------------------------------------------------------------------------------------------
def _pow2_rsqrt(n: int) -> float:
    r = 1.0 / math.sqrt(n)
    assert float(torch.tensor(r, dtype=F32)) == r and math.frexp(r)[0] == 0.5, f"1/sqrt({n}) is not a power of two"
    return r


def _build_fold(wq, wp, bias, C, p, a, ap, s):
    LDK = (C + p + 4 + 3) & ~3
    out = torch.zeros(C, LDK, dtype=torch.float64)
    out[:, :C] = wq.t() * a
    if p:
        out[:, C:C + p] = wp.t() * ap
    if bias is not None:
        out[:, C + p] = bias * s
    assert_f32(out, "fold")
    return out


def stage_w(w: Dict[str, Tensor], *, C: int, D: int, k: int, integration: str, heads: int = 1, duplex: bool = False):
    """gf_fold.cu fold_weights() step by step, every step proven exact: the folded buffers the kernel writes, in fp64."""
    p = w["pos_latent"].shape[1]
    ch = C // heads
    s, rC, rD = _pow2_rsqrt(ch), _pow2_rsqrt(C), _pow2_rsqrt(D)
    rp = _pow2_rsqrt(p) if p else 0.0
    f = {}
    qfold = _build_fold(w["wq"], w.get("wpq"), w["bq"], C, p, s * rC, s * rp, s)
    kconst = (exact_mm(w["pos_latent"], w["wpk"], alpha=rp, E=w["bk"][None], name="KCONST") if p else w["bk"][None].expand(k, C).clone())
    if duplex:
        f["AK"] = exact_mm(w["wkc"], qfold, alpha=rC, name="AK")[None]
        f["CK"] = exact_mm(kconst, qfold, name="CK")[None]
        f["WV2"] = w["wv2"] * rC
        f["BV2"] = w["bv2"].clone()
        f["AK2"] = exact_mm(f["WV2"], f["AK"][0], name="AK2")
        row0 = exact_mm(f["BV2"][None], f["AK"][0], name="CK2 row 0")
        f["CK2"] = exact_mm(torch.ones(k, 1, dtype=torch.float64), row0, E=f["CK"][0], name="CK2")
        mfold = _build_fold(w["wk2"], w.get("wpk2"), None, C, p, s * rC, s * rp, 0.0)
        qconst = (exact_mm(w["pos_latent"], w["wpq2"], alpha=rp, E=w["bq2"][None], name="QCONST") if p
                  else w["bq2"][None].expand(k, C).clone())
        f["AM"] = exact_mm(w["wq2"], mfold, alpha=rD, name="AM")
        f["CM"] = exact_mm(qconst, mfold, name="CM")
        if "wcq" in w:
            f["ACQ"] = exact_mm(w["wcq"], mfold, alpha=rC, name="ACQ")
    else:
        hs = [slice(h * ch, (h + 1) * ch) for h in range(heads)]
        f["AK"] = torch.stack([exact_mm(w["wk"][:, sl], qfold[sl], alpha=rD, name=f"AK{h}") for h, sl in enumerate(hs)])
        f["CK"] = torch.stack([exact_mm(kconst[:, sl], qfold[sl], name=f"CK{h}") for h, sl in enumerate(hs)])
    nh = 1 if duplex else heads
    hs = [slice(h * ch, (h + 1) * ch) for h in range(nh)] if not duplex else [slice(0, C)]
    one = torch.zeros_like(w["bo"])
    if integration != "add":
        one[:C] = 1.0
    f["AV"] = torch.stack([exact_mm(w["wv"][:, sl], w["wo"][sl], alpha=rD * rC, name=f"AV{h}") for h, sl in enumerate(hs)])
    cv = []
    for h, sl in enumerate(hs):
        v = exact_mm(w["bv"][sl][None], w["wo"][sl], alpha=rC, name=f"CV{h}")[0]
        if h == 0:
            v = exact_mm(torch.ones(1, 1, dtype=torch.float64), v[None], E=(w["bo"] + one)[None], name="CV0 + bo")[0]
        cv.append(v)
    f["CV"] = torch.stack(cv)
    f["CB"] = w["bo"] + one
    return f


# ---- the positional axis tables ----------------------------------------------------------------------------------------------
def pos_axis(length: int, half: int) -> Tensor:
    """pos_axis_kernel: fp32 of the fp64 sin / cos (the same angle arithmetic as oracle/bipartite.sinusoidal_axis)."""
    return sinusoidal_axis(length, half).float()


def pos_midpoint_margin(length: int, half: int) -> float:
    """Smallest distance, relative to the value, of an fp64 sin / cos of the axis table from an fp32 rounding midpoint (the value
    halfway between two neighbouring fp32 numbers).  Exact zeros and fp32 values count as infinitely far."""
    v = sinusoidal_axis(length, half)
    r = v.float().double()
    nxt = torch.nextafter(r.float(), torch.where(v > r, torch.full_like(r, math.inf), torch.full_like(r, -math.inf)).float()).double()
    mid = (r + nxt) / 2.0
    d = (v - mid).abs() / v.abs().clamp_min(1e-300)
    d = torch.where(v == r, torch.full_like(d, math.inf), d)
    return d.min().item()


# ---- stage I -----------------------------------------------------------------------------------------------------------------
def _pos_entry(axis: Tensor, kap: Tensor, kap0: Optional[Tensor]):
    """Rt / Ct entries of one latent: axis [L, half] fp32, kap [half] with at most one nonzero power of two -> fp32 [L]."""
    nz = (kap != 0).nonzero().flatten()
    assert nz.numel() <= 1, "kappa row is not one-hot"
    prod = torch.zeros(axis.shape[0], dtype=torch.float64)
    if nz.numel():
        q = int(nz[0])
        assert math.frexp(abs(kap[q].item()))[0] == 0.5, "kappa entry is not a power of two"
        prod = axis[:, q].double() * kap[q]
    prod = prod.float()
    return prod if kap0 is None else (prod + torch.tensor(kap0.item(), dtype=F32))


def tables(kp_all: Tensor, v: Optional[Tensor], *, C: int, p: int, H: int, W: int, k: int, heads: int, seg: int, KP: int,
           tf32_k: bool, tf32_v: bool, d: Optional[Tensor] = None):
    """The tables of one layer from its exact per-head key rows kp_all [h, B, k, LDK] and values v [h, B, k, Cout] (fp64, fp32
    values): K' [B,KP,C], V^T [B,Cout,KP], Rt [B,H,KP], Ct [B,W,KP] as float32, rounded as the kernels round them."""
    _, B, _, _ = kp_all.shape
    half = p // 2
    row, col = (pos_axis(H, half), pos_axis(W, half)) if p else (None, None)
    Kp = torch.zeros(B, KP, C, dtype=F32)
    Rt = torch.full((B, H, KP), -math.inf, dtype=F32)
    Ct = torch.zeros(B, W, KP, dtype=F32)
    Vt = None
    if v is not None:
        Vt = torch.zeros(B, v.shape[3], KP, dtype=F32)
    for h in range(heads):
        for b in range(B):
            for j in range(k):
                J = h * seg + j
                r = kp_all[h, b, j, :C]
                if d is not None:
                    r = r * d[b]
                    assert_f32(r, "K' d")
                Kp[b, J] = tf32_rne((r * KF).float()) if tf32_k else r.float()
                kap = kp_all[h, b, j, C:C + p + 1]
                rt = _pos_entry(row, kap[:half], kap[p]) if p else torch.full((H,), kap[p].item(), dtype=F32)
                ct = _pos_entry(col, kap[half:p], None) if p else torch.zeros(W, dtype=F32)
                if tf32_k:
                    rt, ct = rt * LOG2E_F, ct * LOG2E_F
                Rt[b, :, J], Ct[b, :, J] = rt, ct
                if v is not None:
                    Vt[b, :, J] = tf32_rne(v[h, b, j].float()) if tf32_v else v[h, b, j].float()
    return Kp, Vt, Rt, Ct


def simplex_rows(f, y: Tensor, *, heads: int):
    """Exact key rows [h, B, k, LDK] and values [h, B, k, Cout] of the stage-I kernel."""
    kp = torch.stack([exact_mm(y, f["AK"][h], E=f["CK"][h][None], name=f"kp{h}") for h in range(heads)])
    v = torch.stack([exact_mm(y, f["AV"][h], E=f["CV"][h][None, None], name=f"v{h}") for h in range(heads)])
    return kp, v


def key_rows(src: Tensor, A: Tensor, Cst: Tensor, *, tc: bool) -> Tensor:
    """The duplex key GEMM KPALL = src A + Cst[row % k] ([B, k, LDK]).  tc: gemm_tc_kernel, whose operands must be TF32 values (the
    tensor core's truncation is then the identity) and whose epilogue is one fma.rn.f32 of fp32(1.000352220f^2) with the exact
    sum; the fp64 sum alpha S + CK is checked exact, so its fp32 rounding is that of the fma.  Otherwise the CUDA-core GEMM, exact."""
    S = exact_mm(src, A, name="key S")
    if not tc:
        return exact_mm(src, A, E=Cst[None], name="key rows")
    assert torch.equal(tf32_trunc(src.float()).double(), src), "key GEMM: source not on the TF32 grid"
    assert torch.equal(tf32_trunc(A.float()).double(), A), "key GEMM: AK not on the TF32 grid"
    prod = S * COMP2                                                  # 24 x 24 bits: exact in fp64
    r = prod + Cst[None]
    assert torch.equal(r - Cst[None], prod) and torch.equal(r - prod, Cst[None].expand_as(r)), "alpha S + CK not exact in fp64"
    return r.float().double()


# ---- instance / batch statistics ---------------------------------------------------------------------------------------------
def norm_stats(X: Tensor, batch: bool):
    """NSCALE, NSHIFT [B,C] float32 of norm_finish_kernel from integer-valued X [B,n,C]: the fp64 sums are exact (checked), then
    mean = s / cnt, var = max(q / cnt - mean * mean, 0), rstd = 1 / sqrt(var + 1e-8), scale = fp32(rstd), shift = fp32(-mean rstd),
    each IEEE-rounded as on the device."""
    B, n, C = X.shape
    assert torch.equal(X.round(), X)
    s, q = X.sum(dim=1), (X * X).sum(dim=1)
    assert (X.abs() * X.abs()).sum(dim=(0, 1)).max() < 2.0 ** 53, "sums not exact in fp64"
    cnt = float(n)
    if batch:
        s, q, cnt = s.sum(dim=0, keepdim=True).expand(B, C), q.sum(dim=0, keepdim=True).expand(B, C), float(B * n)
    mean = s / cnt
    var = (q / cnt - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + LN_EPS)
    return rstd.float(), (-(mean * rstd)).float()
