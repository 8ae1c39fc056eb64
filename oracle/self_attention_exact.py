"""Image self-attention as csrc/gf_self_attn.cu computes it, and exact cases for its kernels (DESIGN 4.14).

TEST INFRASTRUCTURE ONLY.  Four parts:

* ``forward`` / ``backward``: a tile-by-tile restatement of the kernels in float64 that applies their roundings (``rounded=True``):
  operands read from memory truncated to TF32, S and dP rounded to fp32, x = fp32(fp32(S) * sl2) with sl2 = fp32(scale * log2 e),
  p = fp32(exp2(fp32(x - m))) per 64-key tile, l = l * alpha + sum of the unrounded p, o = o * alpha + rne(p) V, O = o * fp32(1 / L),
  lse = m + log2 L; backward P recomputed from lse, dS = fp32(p * fp32(dP - Delta)) staged with RNE, as is P^T, dK and dQ times
  scale.  With ``rounded=False`` it is the same streaming in plain float64, which equals ``oracle.self_attention.attention``.
* ``tied_case`` builds inputs whose every logit is 1024 or 0 with ties of 2^k winning keys, and ``exact_reference`` is the float64
  definition with the one rounding the kernels add there (dS to fp32, then to TF32 with RNE); P is taken as fp32, as the kernels
  hold it, so that a float64 exp2 that is not exact at integers cannot leave 1e-17 where O is exactly 0.
* ``prove_exact`` checks, element by element, that such a case really is exact for the kernels: every exp2f that must vanish has
  an argument <= -151, m + k is exact, every dS is an fp32 value before it is rounded, and every sum the tensor core or the delta
  kernel forms is order-free exact (all terms multiples of one 2^-e, sum of |terms| < 2^(24 - e)).
* The double backward (gf_self_attn_bwd_vjp): ``vjp`` restates its three kernels tile by tile with their roundings;
  ``vjp_tied_case`` adds integer cotangents to a tied case, ``vjp_exact_reference`` is the float64 algebra with the roundings the
  kernels add there, and ``prove_vjp_exact`` checks such a case element by element.
Tensors may live on any device; the GPU tests run the restatement there in float64.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .tf32 import tf32_rne, tf32_trunc

T = 64                                   # tokens per tile
LOG2E = np.float32(1.4426950408889634)   # the kernels' LOG2E constant
SEL = 32.0                               # the selector value of the exact cases: a logit is 32 * 32 = 1024 or 0


def kernel_scales(d: int):
    """(scale, sl2) as the entry points form them: scale = fp32(1 / sqrt(d)) (the Python wrapper's value passed as a C float),
    sl2 = fp32(scale * LOG2E)."""
    scale = np.float32(1.0 / math.sqrt(d))
    return float(scale), float(np.float32(scale * LOG2E))


def _heads(t, h):
    B, n, C = t.shape
    return t.reshape(B, n, h, C // h).transpose(1, 2)                     # [B,h,n,d]


def _merge(t):
    B, h, n, d = t.shape
    return t.transpose(1, 2).reshape(B, n, h * d)


def _ops(rounded: bool):
    if not rounded:
        ident = lambda t: t
        return ident, ident, ident
    f32 = lambda t: t.float().double()
    tr = lambda t: tf32_trunc(t.float()).double()
    rne = lambda t: tf32_rne(t.float()).double()
    return f32, tr, rne


def _scales(d, rounded):
    return kernel_scales(d) if rounded else (1.0 / math.sqrt(d), 1.0 / math.sqrt(d) / math.log(2.0))


def forward(q, k, v, heads: int, rounded: bool = True):
    """gf_self_attn_fwd restated: q, k, v [B,n,C] -> (O [B,n,C], lse [B,h,n]), float64 (fp32 values when rounded)."""
    B, n, C = q.shape
    d = C // heads
    f32, tr, rne = _ops(rounded)
    _, sl2 = _scales(d, rounded)
    qh, kh, vh = (tr(_heads(t.double(), heads)) for t in (q, k, v))
    m = torch.full((B, heads, n, 1), -math.inf, dtype=torch.float64, device=q.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, heads, n, d, dtype=torch.float64, device=q.device)
    for k0 in range(0, n, T):
        x = f32(f32(qh @ kh[:, :, k0:k0 + T].transpose(2, 3)) * sl2)
        mn = torch.maximum(m, x.amax(dim=3, keepdim=True))
        alpha = f32(torch.exp2(f32(m - mn)))
        p = f32(torch.exp2(f32(x - mn)))
        l = l * alpha + p.sum(dim=3, keepdim=True)
        o = o * alpha + rne(p) @ vh[:, :, k0:k0 + T]
        m = mn
    L = f32(l)
    O = f32(f32(o) * f32(1.0 / L))
    lse = f32(m + f32(torch.log2(L)))
    return _merge(O), lse[..., 0]


def backward(q, k, v, o, lse, do, heads: int, rounded: bool = True):
    """gf_self_attn_bwd restated, given the forward's O and lse: -> (dQ, dK, dV) [B,n,C], float64."""
    B, n, C = q.shape
    d = C // heads
    f32, tr, rne = _ops(rounded)
    scale, sl2 = _scales(d, rounded)
    qh, kh, vh, doh = (tr(_heads(t.double(), heads)) for t in (q, k, v, do))
    delta = f32((_heads(o.double(), heads) * _heads(do.double(), heads)).sum(dim=3, keepdim=True))   # CUDA cores: no truncation
    L = lse.double()[..., None]
    dq = torch.zeros_like(qh)
    dk, dv = torch.zeros_like(kh), torch.zeros_like(vh)
    for k0 in range(0, n, T):
        ks = slice(k0, k0 + T)
        p = f32(torch.exp2(f32(f32(f32(qh @ kh[:, :, ks].transpose(2, 3)) * sl2) - L)))
        ds = f32(p * f32(f32(doh @ vh[:, :, ks].transpose(2, 3)) - delta))
        dv[:, :, ks] = rne(p).transpose(2, 3) @ doh
        dk[:, :, ks] = rne(ds).transpose(2, 3) @ qh
        dq = dq + rne(ds) @ kh[:, :, ks]
    return _merge(f32(f32(dq) * scale)), _merge(f32(f32(dk) * scale)), _merge(f32(dv))


# ------------------------------------------------------------------------------------------------------------------------------
# exact cases
# ------------------------------------------------------------------------------------------------------------------------------
def uniform_rows_allowed(n: int) -> str:
    """Where a query may carry no selector (a uniform row, P = 1/n): 'full' at n = 2^j <= 256 (1/n, the mean and log2 n are exact
    and the backward sums still fit 24 bits); 'forward' at n >= 1024 (those rows get dO = 0); 'none' otherwise (log2 192 and
    1/192 are not fp32 values)."""
    if n <= 256 and n & (n - 1) == 0:
        return "full"
    return "forward" if n >= 1024 else "none"


def tied_case(B: int, n: int, C: int, d: int, seed: int = 0, uniform: bool = True, max_tie: int = 5):
    """Inputs [B,n,C] (fp32, CPU) for which the kernels are exact, and per (image, head) the selector channel of each query and
    key (-1 for none).  ``uniform=False``: no uniform rows at all; ``max_tie``: tie sets of at most 2^max_tie keys.

    Per head, channels [0, d/2) are selectors, [d/2, 3d/4) the query payload, [3d/4, d) the key payload.  A key carries 32 in at
    most one selector channel c; the keys of channel c are a tie set of 2^k keys (k drawn from 0..5, placed at random across the
    key tiles).  A query carries 32 in the selector of a channel that has keys, or, where ``uniform_rows_allowed``, none (about one
    in eight).  Payloads are integers in [-2, 2], so every logit is exactly 1024 or 0.  V and dO are integers in [-2, 2]."""
    h = C // d
    g = torch.Generator().manual_seed(seed)
    uni_mode = uniform_rows_allowed(n) if uniform else "none"
    q, k = torch.zeros(B, n, C), torch.zeros(B, n, C)
    v = torch.randint(-2, 3, (B, n, C), generator=g).float()
    do = torch.randint(-2, 3, (B, n, C), generator=g).float()
    qsel = torch.full((B, h, n), -1, dtype=torch.long)
    ksel = torch.full((B, h, n), -1, dtype=torch.long)
    for b in range(B):
        for j in range(h):
            off = j * d
            keys = torch.randperm(n, generator=g)
            ks = torch.randperm(max_tie + 1, generator=g)
            used, pos = [], 0
            for i, c in enumerate(torch.randperm(d // 2, generator=g).tolist()):
                size = 2 ** int(ks[i % (max_tie + 1)])
                if pos + size > n:
                    continue
                w = keys[pos:pos + size]
                pos += size
                k[b, w, off + c] = SEL
                ksel[b, j, w] = c
                used.append(c)
            k[b, :, off + 3 * d // 4:off + d] = torch.randint(-2, 3, (n, d // 4), generator=g).float()
            q[b, :, off + d // 2:off + 3 * d // 4] = torch.randint(-2, 3, (n, d // 4), generator=g).float()
            sel = torch.tensor(used)[torch.randint(0, len(used), (n,), generator=g)]
            uni = torch.rand(n, generator=g) < 0.125 if uni_mode != "none" else torch.zeros(n, dtype=torch.bool)
            rows = torch.arange(n)[~uni]
            q[b, rows, off + sel[~uni]] = SEL
            qsel[b, j, rows] = sel[~uni]
            if uni_mode == "forward":
                do[b, uni, off:off + d] = 0.0
    return dict(q=q, k=k, v=v, do=do, heads=h, d=d, qsel=qsel, ksel=ksel)


def exact_reference(q, k, v, do, heads: int):
    """The float64 definition (logits in log2 units with the kernels' sl2), with the one rounding the kernels add in a tied case:
    dS to fp32 and then to TF32 (RNE) before dK = scale dS^T Q and dQ = scale dS K, each scale applied as one fp32 multiply.
    -> fp32 (O, lse, Delta, dQ, dK, dV)."""
    d = q.shape[2] // heads
    scale, sl2 = kernel_scales(d)
    qh, kh, vh, doh = (_heads(t.double(), heads) for t in (q, k, v, do))
    x = (qh @ kh.transpose(2, 3)) * sl2
    m = x.amax(dim=3, keepdim=True)
    lse = m + torch.log2(torch.exp2(x - m).sum(dim=3, keepdim=True))
    P = torch.exp2(x - lse).float().double()          # the kernels' p is fp32: 2^-k, 1/n or 0 without a float64 exp2's last bit
    O = P @ vh
    delta = (O * doh).sum(dim=3, keepdim=True)
    ds = P * (doh @ vh.transpose(2, 3) - delta)
    dsr = tf32_rne(ds.float()).double()
    dq = (dsr @ kh).float().double() * scale
    dk = (dsr.transpose(2, 3) @ qh).float().double() * scale
    dv = P.transpose(2, 3) @ doh
    return tuple(t.float() for t in (_merge(O), lse[..., 0], delta[..., 0], _merge(dq), _merge(dk), _merge(dv)))


def _grain(x: torch.Tensor) -> torch.Tensor:
    """e such that x * 2^e is an odd integer (float64 x; -10^6 for zeros, so they never set a maximum)."""
    mant, ex = torch.frexp(x)
    M = (mant * 2.0 ** 53).to(torch.int64)
    tz = torch.log2((M & -M).abs().double()).round().long()
    return torch.where(x == 0, torch.full_like(tz, -10 ** 6), 53 - ex.long() - tz)


def _product_bound(a: torch.Tensor, b: torch.Tensor):
    """For a [r, l] @ b [l, c]: (e, tot), every term of element (i, j) a multiple of 2^-e[i, j] and tot[i, j] = sum |terms|."""
    ga = _grain(a)
    gb = _grain(b).amax(dim=0)
    nzb = b != 0
    e = torch.stack([torch.where(nzb[:, j][None, :], ga, torch.full_like(ga, -10 ** 6)).amax(dim=1) for j in range(b.shape[1])], 1)
    return e + gb[None, :], a.abs() @ b.abs()


def _fits(e: torch.Tensor, tot: torch.Tensor) -> torch.Tensor:
    return (tot == 0) | (torch.ldexp(tot, e.clamp(-1000, 1000).double()) < 2.0 ** 24)


def order_free_exact(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """For the product a [r, l] @ b [l, c] (float64, every entry an fp32 value, b integer-valued): True where every order of
    fp32 additions gives the exact sum.  Terms of element (i, j) are multiples of 2^-e with e = max over the terms of
    grain(a[i, l]) + max_l grain(b[l, j]); the condition is sum |terms| < 2^(24 - e)."""
    return _fits(*_product_bound(a, b))


def _fp32_value(x: torch.Tensor) -> torch.Tensor:
    return x.float().double() == x


def prove_exact(case) -> dict:
    """Checks that a ``tied_case`` is exact for the kernels; raises AssertionError naming the first failing claim.  Returns counts
    that show what the case exercises."""
    q, k, v, do, h, d = (case[n] for n in ("q", "k", "v", "do", "heads", "d"))
    B, n, _ = q.shape
    _, sl2 = kernel_scales(d)
    xw = np.float32(np.float32(1024.0) * np.float32(sl2))
    assert float(xw) == 1024.0 * sl2, "x = 1024 sl2 is not exact"
    assert -float(xw) <= -151.0, f"the winner's margin {float(xw)} does not underflow exp2f"
    stats = dict(alpha_reset=0, alpha_one=0, ties=set(), uniform=0, ds_rne_ne_trunc=0, ds_nonzero=0)
    for b in range(B):
        for j in range(h):
            cols = slice(j * d, (j + 1) * d)
            Q, K, V, dO = (t[b, :, cols].double() for t in (q, k, v, do))
            S = Q @ K.T
            assert order_free_exact(Q, K.T).all(), "S"
            assert ((S == 0) | (S == 1024.0)).all(), "a logit is neither 0 nor 1024"
            win = S == 1024.0
            cnt = win.sum(dim=1)
            tie = cnt > 0
            stats["uniform"] += int((~tie).sum())
            if (~tie).any():
                assert uniform_rows_allowed(n) != "none", "a uniform row where 1/n or log2 n is not exact"
            kk = torch.log2(cnt[tie].double())
            assert (kk == kk.round()).all() and kk.max() <= 5, "a tie set is not 2^k keys, k <= 5"
            stats["ties"] |= set(int(x) for x in kk.unique())
            # forward: every row's p is 0 or 1 (args 0 or -x_win), alpha is 0 or 1, l = 2^k (or n), lse = m + log2 l exact
            lse = torch.where(tie, float(xw) + torch.log2(cnt.double().clamp(min=1)), math.log2(n))
            assert _fp32_value(lse).all(), "m + k (or log2 n) is not an fp32 value"
            tiles = win.reshape(n, n // T, T).any(dim=2)
            first = tiles.float().argmax(dim=1)
            stats["alpha_reset"] += int((tie & (first > 0)).sum())
            stats["alpha_one"] += int((tiles.sum(dim=1) > 1).sum())
            # every forward partial sum of p V (p in {0, 1}, whatever the tile order) is bounded by sum |V|
            assert (V.abs().sum(dim=0) < 2.0 ** 24).all(), "P V"
            # backward exp2f arguments x - lse: -k for a winner, -(x_win + k) for any other key of a tied row, -log2 n in a uniform row
            arg = torch.where(win, float(xw), 0.0) - lse[:, None]
            assert (arg[win] == arg[win].round()).all() and (arg[~tie] == -math.log2(n)).all(), "backward exp2f argument"
            assert (arg[~win & tie[:, None]] <= -151).all(), "a non-winner's exp2f argument is above -151"
            P = torch.where(tie[:, None], win / cnt.double().clamp(min=1)[:, None], 1.0 / n)
            O = P @ V
            assert order_free_exact(P, V).all() and _fp32_value(O).all(), "O"
            prod = O * dO
            g = _grain(prod).amax(dim=1)
            assert (torch.ldexp(prod.abs().sum(dim=1), g.clamp(-1000, 1000).double()) < 2.0 ** 24).all(), "Delta"
            delta = prod.sum(dim=1, keepdim=True)
            assert order_free_exact(dO, V.T).all(), "dP"
            diff = dO @ V.T - delta
            assert _fp32_value(diff).all(), "dP - Delta is not an fp32 value"
            ds = P * diff
            assert _fp32_value(ds).all(), "dS is not an fp32 value before it is rounded"
            dsr = tf32_rne(ds.float()).double()
            nz = ds != 0
            stats["ds_nonzero"] += int(nz.sum())
            stats["ds_rne_ne_trunc"] += int((dsr != tf32_trunc(ds.float()).double()).sum())
            assert order_free_exact(P.T, dO).all(), "dV = P^T dO"
            assert order_free_exact(dsr.T, Q).all(), "dK = dS^T Q"
            assert order_free_exact(dsr, K).all(), "dQ = dS K"
    stats["ties"] = sorted(stats["ties"])
    return stats


# ------------------------------------------------------------------------------------------------------------------------------
# double backward (gf_self_attn_bwd_vjp)
# ------------------------------------------------------------------------------------------------------------------------------
def vjp(q, k, v, do, a, bk, cv, lse, delta, heads: int, rounded: bool = True):
    """gf_self_attn_bwd_vjp restated, given the first order's lse and Delta [B,h,n]: -> (gQ, gK, gV, gdO [B,n,C], r, t [B,h,n]),
    float64 (fp32 values when rounded).

    A row pass over every 64-key tile sums r and u over the fp32 terms pg = fp32(p gds) and pg dP, and PC = rne(P) Cv; then
    t = fp32(fp32(u - 2 Delta r) + dO . PC), dO read as fp32 (CUDA cores).  A second pass per key tile forms, as both output
    kernels do, dS = fp32(p fp32(dP - Delta)), GdP = fp32(p fp32(gds - r)), GP = fp32(fp32(gds (dP - Delta)) - fp32(r dP)) plus
    dO Cv^T on the accumulator, GS = fp32(p fp32(GP - t)), stages dS, GdP and GS with RNE, and accumulates gQ / s, gdO and the
    key tile's gK / s and gV.  Out: gQ and gK times scale in one fp32 multiply, gdO = fp32(GdP V) + PC.  S, dP and GdS / s come
    out of the accumulators as fp32, p = fp32(exp2(fp32(fp32(S) sl2) - lse)) and gds = fp32((GdS / s) scale); operands read from
    memory are truncated to TF32.  With ``rounded=False`` it is the same algebra in plain float64 (oracle.self_attention_vjp)."""
    B, n, C = q.shape
    d = C // heads
    f32, tr, rne = _ops(rounded)
    scale, sl2 = _scales(d, rounded)
    qh, kh, vh, doh, ah, bkh, cvh = (tr(_heads(t.double(), heads)) for t in (q, k, v, do, a, bk, cv))
    do_full = _heads(do.double(), heads)
    L, Dl = lse.double()[..., None], delta.double()[..., None]

    def tile(ks):
        S = f32(qh @ kh[:, :, ks].transpose(2, 3))
        dP = f32(doh @ vh[:, :, ks].transpose(2, 3))
        G = f32(ah @ kh[:, :, ks].transpose(2, 3) + qh @ bkh[:, :, ks].transpose(2, 3))
        p = f32(torch.exp2(f32(f32(S * sl2) - L)))
        return p, dP, f32(G * scale)

    r = torch.zeros_like(L)
    u = torch.zeros_like(L)
    pc = torch.zeros_like(qh)
    for k0 in range(0, n, T):
        ks = slice(k0, k0 + T)
        p, dP, gds = tile(ks)
        pg = f32(p * gds)
        r = r + pg.sum(dim=3, keepdim=True)
        u = u + f32(pg * dP).sum(dim=3, keepdim=True)
        pc = pc + rne(p) @ cvh[:, :, ks]
    r, u, pc = f32(r), f32(u), f32(pc)
    t = f32(f32(u - f32(2.0 * Dl * r)) + (do_full * pc).sum(dim=3, keepdim=True))

    gq, gdo = torch.zeros_like(qh), torch.zeros_like(qh)
    gk, gv = torch.zeros_like(kh), torch.zeros_like(vh)
    for k0 in range(0, n, T):
        ks = slice(k0, k0 + T)
        p, dP, gds = tile(ks)
        dpm = f32(dP - Dl)
        gdp = rne(f32(p * f32(gds - r)))
        ds = rne(f32(p * dpm))
        gp = f32(f32(f32(gds * dpm) - f32(r * dP)) + doh @ cvh[:, :, ks].transpose(2, 3))
        gs = rne(f32(p * f32(gp - t)))
        gq = gq + ds @ bkh[:, :, ks] + gs @ kh[:, :, ks]
        gdo = gdo + gdp @ vh[:, :, ks]
        gk[:, :, ks] = ds.transpose(2, 3) @ ah + gs.transpose(2, 3) @ qh
        gv[:, :, ks] = gdp.transpose(2, 3) @ doh
    return (_merge(f32(f32(gq) * scale)), _merge(f32(f32(gk) * scale)), _merge(f32(gv)), _merge(f32(f32(gdo) + pc)),
            r[..., 0], t[..., 0])


def vjp_tied_case(B: int, n: int, C: int, d: int, seed: int = 0, ab=None):
    """A ``tied_case`` with tie sets of 1, 2 or 4 keys, uniform rows only where ``uniform_rows_allowed`` is 'full' (and dO = 0 in
    them), and integer cotangents a (of dQ), bk (of dK) and cv (of dV).  cv is in [-2, 2] everywhere.  With ``ab`` (default:
    d = 64, where scale = 1/8 is exact) a holds [-1, 1] in the key-payload channels and bk in the selector and query-payload
    channels, so that GdS = s (A K^T + Q Bk^T) differs between the winners of one tie set and GdP, r, GS, gQ, gK and gV are not
    zero; otherwise a = bk = 0 (GdS = 0).

    Why so: GS = P o (GP - t) carries the grain of t's 2 Delta r, 2^-(3k+3) in a tie of 2^k keys, and gK sums it over every query
    of the tie set; ties beyond 4 keys overflow 24 bits there.  A uniform row with dO = 0 has dS = GP = t = GS = 0, but its
    GdP = (gds - r) / n needs more than TF32's 11 bits, so RNE and truncation of the staged GdP differ (at n = 256)."""
    case = tied_case(B, n, C, d, seed, uniform=uniform_rows_allowed(n) == "full", max_tie=2)
    h = C // d
    ab = d == 64 if ab is None else ab
    g = torch.Generator().manual_seed(10 ** 6 + seed)
    a, bk = torch.zeros(B, n, C), torch.zeros(B, n, C)
    cv = torch.randint(-2, 3, (B, n, C), generator=g).float()
    if ab:
        ri = lambda w: torch.randint(-1, 2, (B, n, w), generator=g).float()
        for j in range(h):
            off = j * d
            a[:, :, off + 3 * d // 4:off + d] = ri(d // 4)
            bk[:, :, off:off + 3 * d // 4] = ri(3 * d // 4)
    for j in range(h):
        case["do"][:, :, j * d:(j + 1) * d][case["qsel"][:, j] < 0] = 0.0
    return dict(case, a=a, bk=bk, cv=cv)


def vjp_exact_reference(q, k, v, do, a, bk, cv, heads: int, rounded: bool = True):
    """The float64 algebra of oracle.self_attention_vjp with P held in fp32 (from the kernels' sl2), plus the roundings the
    kernels add in a ``vjp_tied_case``: dS, GdP and GS to fp32 and then TF32 (RNE) before their products; gQ and gK take scale as
    one fp32 multiply; gdO = fp32(GdP V) + PC in fp32.  -> fp32 (gQ, gK, gV, gdO, r, t).  ``rounded=False``: none of that (scale
    1/sqrt(d), P the float64 softmax), float64 out."""
    d = q.shape[2] // heads
    scale, sl2 = _scales(d, rounded)
    f32, _, _ = _ops(rounded)
    rne = (lambda t: tf32_rne(t.float()).double()) if rounded else (lambda t: t)
    Q, K, V, dO, A, Bk, Cv = (_heads(t.double(), heads) for t in (q, k, v, do, a, bk, cv))
    x = (Q @ K.transpose(2, 3)) * sl2
    m = x.amax(dim=3, keepdim=True)
    lse = m + torch.log2(torch.exp2(x - m).sum(dim=3, keepdim=True))
    P = f32(torch.exp2(x - lse))
    dP = dO @ V.transpose(2, 3)
    delta = (P * dP).sum(dim=3, keepdim=True)
    dS = P * (dP - delta)
    GdS = f32(A @ K.transpose(2, 3) + Q @ Bk.transpose(2, 3)) * scale
    r = (P * GdS).sum(dim=3, keepdim=True)
    u = (P * GdS * dP).sum(dim=3, keepdim=True)
    PC = P @ Cv
    GdP = P * (GdS - r)
    GP = GdS * (dP - delta) - r * dP + dO @ Cv.transpose(2, 3)
    t = u - 2.0 * delta * r + (dO * PC).sum(dim=3, keepdim=True)
    GS = P * (GP - t)
    dS, GdP, GS = rne(dS), rne(GdP), rne(GS)
    gQ = f32(f32(dS @ Bk + GS @ K) * scale)
    gK = f32(f32(dS.transpose(2, 3) @ A + GS.transpose(2, 3) @ Q) * scale)
    gV = f32(GdP.transpose(2, 3) @ dO)
    gdO = f32(f32(GdP @ V) + f32(PC))
    out = (_merge(gQ), _merge(gK), _merge(gV), _merge(gdO), r[..., 0], t[..., 0])
    return tuple(o.float() for o in out) if rounded else out


def _int_product_fits(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """order_free_exact for a product of integer-valued a [r, l] and b [l, c], without the per-column loop: every term is an
    integer, so the condition is sum |terms| < 2^24 (the grains are at most 0)."""
    assert (a == a.round()).all() and (b == b.round()).all()
    return a.abs() @ b.abs() < 2.0 ** 24


def _product_fits(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """order_free_exact, trying first the coarser bound e = max_l grain(a[i, l]) + max_l grain(b[l, j]) (one GEMM, no column loop)."""
    fast = _fits(_grain(a).amax(dim=1)[:, None] + _grain(b).amax(dim=0)[None, :], a.abs() @ b.abs())
    return fast if fast.all() else order_free_exact(a, b)


def _sum_exact(terms: torch.Tensor, init=None) -> torch.Tensor:
    """True per row where every fp32 order of adding the row's terms (and ``init``, an accumulator's starting value) is exact."""
    e, tot = _grain(terms).amax(dim=1), terms.abs().sum(dim=1)
    if init is not None:
        e, tot = torch.maximum(e, _grain(init)), tot + init.abs()
    return _fits(e, tot)


def prove_vjp_exact(case) -> dict:
    """Checks that a ``vjp_tied_case`` is exact for gf_self_attn_bwd_vjp (after ``prove_exact`` for the first order it rests on);
    raises AssertionError naming the first failing claim.  Per element: gds = fp32(GdS / s) scale is exact; every value the
    kernels form on CUDA cores before it is staged or summed is an fp32 value whatever FMA contraction nvcc picks (r, u, 2 Delta r,
    u - 2 Delta r, t, gds - r, GdP, the two products of GP and their difference, GP - t, GS); r, u and dO . PC are order-free exact
    sums; and every tensor-core product is order-free exact: GdS / s = [A | Q][K | Bk]^T, PC = P Cv, GP = (its CUDA-core part) +
    dO Cv^T, gQ / s = [dS | GS][Bk ; K], gK / s = [dS^T | GS^T][A ; Q], gV = GdP^T dO, GdP V.  The staged dS, GdP and GS are the
    RNE TF32 values.  Returns counts that show what the case exercises."""
    prove_exact(case)
    q, k, v, do, a, bk, cv, h, d = (case[x] for x in ("q", "k", "v", "do", "a", "bk", "cv", "heads", "d"))
    B, n, _ = q.shape
    scale, _ = kernel_scales(d)
    st = dict(gdp_nonzero=0, gs_nonzero=0, r_rows=0, delta_r_rows=0, ds_rne_ne_trunc=0, gdp_rne_ne_trunc=0, gs_rne_ne_trunc=0)
    for b in range(B):
        for j in range(h):
            cols = slice(j * d, (j + 1) * d)
            Q, K, V, dO, A, Bk, Cv = (t[b, :, cols].double() for t in (q, k, v, do, a, bk, cv))
            win = (Q @ K.T) == 1024.0
            cnt = win.sum(dim=1)
            P = torch.where((cnt > 0)[:, None], win / cnt.double().clamp(min=1)[:, None], 1.0 / n)
            dP = dO @ V.T
            delta = ((P @ V) * dO).sum(dim=1, keepdim=True)
            dpm = dP - delta
            AQ, KB = torch.cat([A, Q], 1), torch.cat([K, Bk], 1)
            assert _int_product_fits(AQ, KB.T).all(), "GdS / s = [A | Q][K | Bk]^T"
            gds = (AQ @ KB.T) * scale
            assert _fp32_value(gds).all(), "gds = (GdS / s) scale is not exact"
            pg = P * gds
            assert _fp32_value(pg).all() and _fp32_value(pg * dP).all(), "p gds or p gds dP"
            assert _sum_exact(pg).all() and _sum_exact(pg * dP).all(), "r or u"
            r, u = pg.sum(dim=1, keepdim=True), (pg * dP).sum(dim=1, keepdim=True)
            assert _product_fits(P, Cv).all(), "PC = P Cv"
            PC = P @ Cv
            assert _fp32_value(dO * PC).all() and _sum_exact(dO * PC).all(), "dO . PC"
            dr2 = 2.0 * delta * r
            t = u - dr2 + (dO * PC).sum(dim=1, keepdim=True)
            for name, x in (("r", r), ("u", u), ("2 Delta r", dr2), ("u - 2 Delta r", u - dr2), ("t", t), ("gds - r", gds - r),
                            ("GdP", P * (gds - r)), ("gds (dP - Delta)", gds * dpm), ("r dP", r * dP),
                            ("GP before dO Cv^T", gds * dpm - r * dP)):
                assert _fp32_value(x).all(), f"{name} is not an fp32 value"
            gp0 = gds * dpm - r * dP
            assert (dO == dO.round()).all() and (Cv == Cv.round()).all()
            assert _fits(torch.clamp(_grain(gp0), min=0), dO.abs() @ Cv.abs().T + gp0.abs()).all(), "GP = ... + dO Cv^T (integer)"
            GP = gp0 + dO @ Cv.T
            assert _fp32_value(GP - t).all() and _fp32_value(P * (GP - t)).all(), "GP - t or GS"
            ds, gdp, gs = P * dpm, P * (gds - r), P * (GP - t)
            staged = []
            for name, x in (("ds", ds), ("gdp", gdp), ("gs", gs)):
                xr = tf32_rne(x.float()).double()
                st[name + "_rne_ne_trunc"] += int((xr != tf32_trunc(x.float()).double()).sum())
                staged.append(xr)
            dsr, gdpr, gsr = staged
            assert _product_fits(torch.cat([dsr, gsr], 1), torch.cat([Bk, K], 0)).all(), "gQ / s = [dS | GS][Bk ; K]"
            assert _product_fits(torch.cat([dsr.T, gsr.T], 1), torch.cat([A, Q], 0)).all(), "gK / s = [dS^T | GS^T][A ; Q]"
            assert _product_fits(gdpr.T, dO).all(), "gV = GdP^T dO"
            assert _product_fits(gdpr, V).all(), "GdP V"
            st["gdp_nonzero"] += int((gdp != 0).sum())
            st["gs_nonzero"] += int((gs != 0).sum())
            st["r_rows"] += int((r != 0).sum())
            st["delta_r_rows"] += int((dr2 != 0).sum())
    return st
