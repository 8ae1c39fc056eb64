"""The bits gf_augment_resample_nchw and gf_augment_resample_adjoint_nchw must write: their fp32 arithmetic restated, rounding included.

TEST INFRASTRUCTURE ONLY.  csrc/gf_augment.cu resamples with the sym6 taps rs_f, which are non-dyadic fp32 constants, so no choice of
inputs makes its sums exact; this module instead restates every fp32 operation of both kernels in the kernels' order, on the CPU
(numpy), with ``fma32`` a correctly rounded fmaf.  Restated from DESIGN 4.12 and the kernels' documented order:

  * ``res_map`` in its source order.  The build leaves -fmad on, so nvcc may contract any mul/add pair there and in the adjoint's
    det; ``res_map`` therefore checks, per image, that every product that takes part in L, e and det is exact in fp32 (6 (l00 + l01)
    among them): then the result is the same whichever pairs were contracted.  The domain test (``ok``) is taken from fp64 with a
    margin check instead: its products are not exact, but only a comparison far from its threshold depends on them.
  * forward, shared-memory plan: U over its whole extent (x pass, then y, m ascending, doubled), V by the kernel's bilinear, the down
    filter x then y with k ascending.  The tile's boxes only decide which of these values are read, so this part has no tile plan.
  * forward, direct path: res_axis_weights and res_sample_direct, then the same down filter.
  * the tile plan, the first place the result depends on it: res_nu_box, ``empty`` and ``fits`` per 16 x 16 tile pick its path.
  * adjoint: gV (colour-transposed gy, transposed down filter x then y, o ascending) has no plan.  gU of a (tile, copy) box does, the
    second place: it is the sum over the box's 64 x 64 chunks, in chunk order, of each chunk's in-order sum of
    fma(round(wy wx), gV(q), acc) over q row-major, restricted to the kernel's per-nu preimage box.  The chunk origins come from the
    (tile, copy) box through i = L^-1 as the kernel computes it.  Then the transposed up filter (x, then y) and the sum over the nine
    copies in order.  The in-order sums are vectorised as segmented reductions across U points.

``fma32`` adds the exact fp64 product to c (the product of two fp32 values has at most 48 bits), takes the TwoSum error e of that
addition and rounds the fp64 sum to fp32; when that sum lies exactly on an fp32 midpoint and e != 0, the true value lies on e's side
of it, so the result moves one ulp towards e.  Away from a midpoint the double rounding cannot change the result.
"""
from __future__ import annotations

import math

import numpy as np
import torch

F32 = np.float32
SYM6 = (0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
        0.787641141030194, 0.3379294217276218, -0.07263752278646252, -0.021060292512300564, 0.04472490177066578,
        0.0017677118642428036, -0.007800708325034148)
_SUM = 0.0
for _v in SYM6:                                   # RS_SUM: left to right in double, as the constexpr sum
    _SUM += _v
TAPS = np.array([v / _SUM for v in SYM6], dtype=np.float64).astype(F32)     # rs_f: (float)(RS_SYM6[i] / RS_SUM)
T, QC = 16, 64                                    # RS_T, RS_QC
CAP = 10240                                       # RS_CAP
SV_MAX, T_MAX = 16.0, 64                          # the domain of a map (ops.frac_flags)


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def fma32(a, b, c):
    """Correctly rounded fmaf(a, b, c), elementwise on fp32 arrays."""
    a, b, c = np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32)
    p = a.astype(np.float64) * b.astype(np.float64)                 # exact
    cd = c.astype(np.float64)
    s = p + cd
    bb = s - p
    e = (p - (s - bb)) + (cd - bb)                                  # TwoSum: p + c = s + e exactly
    r = s.astype(F32)
    with np.errstate(invalid="ignore"):
        towards = np.nextafter(r, np.where(e > 0, F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (e != 0) & (r.astype(np.float64) + towards.astype(np.float64) == 2 * s)
    return np.where(mid, towards, r).astype(F32)


def _cdiv2(a):
    return -((-np.asarray(a)) >> 1)


def _fdiv2(a):
    return np.asarray(a) >> 1


class InexactMap(AssertionError):
    pass


class ResMap:
    """res_map of one image: l00, l01, l10, l11, e0, e1 (fp32), ident, ok; det and the inverse i00..i11, hx, hy as the adjoint
    computes them.  ``check``: assert that every product that takes part is exact in fp32 (see the module docstring)."""

    def __init__(self, frac6, geom4, H, W, check=True):
        a = np.asarray(frac6, dtype=F32).reshape(6)
        self.ident = bool(np.all(a == np.array([1, 0, 0, 0, 1, 0], F32)))
        fin = bool(np.all(np.isfinite(a)))
        ok = fin
        if fin:
            A = a.astype(np.float64)
            s2 = A[0] ** 2 + A[1] ** 2 + A[3] ** 2 + A[4] ** 2
            det = abs(A[0] * A[4] - A[1] * A[3])
            smax2 = 0.5 * (s2 + math.sqrt(max(s2 * s2 - 4 * det * det, 0.0)))
            smin2 = det * det / smax2 if smax2 > 0 else 0.0
            ok = smax2 <= SV_MAX ** 2 and smin2 >= SV_MAX ** -2 and abs(a[2]) <= F32(T_MAX * max(H, W)) and \
                abs(a[5]) <= F32(T_MAX * max(H, W))
            if check:                                                # the fp32 test cannot land on the other side
                for v, lim in ((smax2, SV_MAX ** 2), (smin2, SV_MAX ** -2)):
                    if abs(v - lim) <= 1e-4 * lim:
                        raise InexactMap(f"singular value {v} too close to the domain's edge {lim}")
        self.ok = bool(ok)
        if not self.ok:
            a = np.array([1, 0, 0, 0, 1, 0], F32)
        self.exact = True

        def mul(x, y):
            p = F32(F32(x) * F32(y))
            if float(p) != float(F32(x)) * float(F32(y)):
                self.exact = False
                if check:
                    raise InexactMap(f"product {x!r} * {y!r} is not exact in fp32")
            return p
        code = int(geom4[0]) & 7
        if H != W:
            code &= ~2
        gtx = min(max(int(geom4[1]), -(W - 1)), W - 1)
        gty = min(max(int(geom4[2]), -(H - 1)), H - 1)
        fl = F32(-1) if code & 1 else F32(1)
        k = code >> 1
        cs = F32(1 if k == 0 else (-1 if k == 2 else 0))
        sn = F32(1 if k == 1 else (-1 if k == 3 else 0))
        d00, d01, d10, d11 = F32(cs * fl), sn, F32(-sn * fl), cs
        self.l00 = F32(mul(d00, a[0]) + mul(d01, a[3]))
        self.l01 = F32(mul(d00, a[1]) + mul(d01, a[4]))
        self.l10 = F32(mul(d10, a[0]) + mul(d11, a[3]))
        self.l11 = F32(mul(d10, a[1]) + mul(d11, a[4]))
        cx, cy = F32(F32(0.5) * F32(W - 1)), F32(F32(0.5) * F32(H - 1))
        w0 = F32(a[2] - F32(mul(a[0], cx) + mul(a[1], cy)))
        w1 = F32(a[5] - F32(mul(a[3], cx) + mul(a[4], cy)))
        o0 = F32(F32(F32(mul(d00, w0) + mul(d01, w1)) - F32(gtx)) + cx)
        o1 = F32(F32(F32(mul(d10, w0) + mul(d11, w1)) - F32(gty)) + cy)
        self.e0 = F32(mul(2, o0) - mul(6, F32(self.l00 + self.l01)))
        self.e1 = F32(mul(2, o1) - mul(6, F32(self.l10 + self.l11)))
        self.code, self.tx, self.ty = code, gtx, gty
        # the adjoint's inverse of L
        self.det = F32(mul(self.l00, self.l11) - mul(self.l01, self.l10))
        with np.errstate(divide="ignore", invalid="ignore"):
            self.i00, self.i01 = F32(self.l11 / self.det), F32(-self.l01 / self.det)
            self.i10, self.i11 = F32(-self.l10 / self.det), F32(self.l00 / self.det)
        self.hx = F32(abs(self.i00) + abs(self.i01))
        self.hy = F32(abs(self.i10) + abs(self.i11))

    def nu(self, qx, qy):
        qx, qy = np.asarray(qx, F32), np.asarray(qy, F32)
        return fma32(self.l00, qx, fma32(self.l01, qy, self.e0)), fma32(self.l10, qx, fma32(self.l11, qy, self.e1))

    def nu_box(self, qx0, qx1, qy0, qy1, H, W):
        """res_nu_box, elementwise over arrays of boxes."""
        cs = [self.nu(qx, qy) for qx, qy in ((qx0, qy0), (qx1, qy0), (qx0, qy1), (qx1, qy1))]
        xmin = np.minimum(np.minimum(cs[0][0], cs[1][0]), np.minimum(cs[2][0], cs[3][0]))
        xmax = np.maximum(np.maximum(cs[0][0], cs[1][0]), np.maximum(cs[2][0], cs[3][0]))
        ymin = np.minimum(np.minimum(cs[0][1], cs[1][1]), np.minimum(cs[2][1], cs[3][1]))
        ymax = np.maximum(np.maximum(cs[0][1], cs[1][1]), np.maximum(cs[2][1], cs[3][1]))
        fi = lambda v: np.floor(v).astype(np.int64)
        return (np.maximum(fi(xmin) - 1, -2 * (W - 1)), np.minimum(fi(xmax) + 2, 4 * W - 3),
                np.maximum(fi(ymin) - 1, -2 * (H - 1)), np.minimum(fi(ymax) + 2, 4 * H - 3))


def _mirror(i, N):
    i = np.asarray(i)
    return np.where(i < 0, -i, np.where(i >= N, 2 * (N - 1) - i, i))


# ------------------------------------------------------------------------------------------------ shared pieces
def _up_axis(E, N):
    """One up-filter pass along the last axis of E [..., 3N - 2] (extended index m = i - (N - 1)) to U's extent
    [-2(N-1), 4N-3]: 2 * sum over m ascending of fmaf(f[nu + 5 - 2m], E[m], acc), m inside E's extent."""
    nu = np.arange(-2 * (N - 1), 4 * N - 2)
    mlo = _cdiv2(nu - 6)
    acc = np.zeros(E.shape[:-1] + nu.shape, F32)
    for t in range(6):
        m = mlo + t
        ok = (m >= -(N - 1)) & (m <= 2 * (N - 1))
        w = np.where(ok, TAPS[np.clip(nu + 5 - 2 * m, 0, 11)], F32(0))
        acc = fma32(w, E[..., np.clip(m + N - 1, 0, 3 * N - 3)], acc)
    return F32(2) * acc


def _down(V, H, W):
    """The down filter of V [C, 2H + 10, 2W + 10] (index q - 1): x then y, k ascending."""
    acc = np.zeros(V.shape[:-1] + (W,), F32)
    ox = np.arange(W)
    for k in range(12):
        acc = fma32(TAPS[k], V[..., 2 * ox + k], acc)
    out = np.zeros(V.shape[:-2] + (H, W), F32)
    oy = np.arange(H)
    for k in range(12):
        out = fma32(TAPS[k], acc[..., 2 * oy + k, :], out)
    return out


def _axis_weights(nu, N):
    """res_axis_weights over an array of nu: (m0 [...], wt [..., 7])."""
    f0 = np.floor(nu)
    n0 = f0.astype(np.int64)
    a = F32(nu - f0)
    m0 = _cdiv2(n0 - 6)
    v0 = (n0 >= -2 * (N - 1)) & (n0 <= 4 * N - 3)
    v1 = (n0 + 1 >= -2 * (N - 1)) & (n0 + 1 <= 4 * N - 3)
    one_a = F32(F32(1) - a)
    wt = np.zeros(nu.shape + (7,), F32)
    for j in range(7):
        mm = m0 + j
        k0 = n0 + 5 - 2 * mm
        k1 = k0 + 1
        w = np.where(v0 & (k0 >= 0) & (k0 < 12), F32(one_a * TAPS[np.clip(k0, 0, 11)]), F32(0)).astype(F32)
        w = np.where(v1 & (k1 >= 0) & (k1 < 12), fma32(a, TAPS[np.clip(k1, 0, 11)], w), w).astype(F32)
        wt[..., j] = np.where((mm >= -(N - 1)) & (mm <= 2 * (N - 1)), F32(2) * w, F32(0))
    return m0, wt


def _blit_index(m, H, W):
    """(sy, sx) [H, W] of the blit's source pixels (augment_kernel)."""
    py, px = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    x = W - 1 - px if m.code & 1 else px
    k = m.code >> 1
    u = [x, py, W - 1 - x, H - 1 - py][k]
    v = [py, W - 1 - x, H - 1 - py, x][k]
    return _mirror(v - m.ty, H), _mirror(u - m.tx, W)


def _colour(v, M):
    """fmaf(M2, v2, fmaf(M1, v1, fmaf(M0, v0, M3))) per output channel."""
    M = np.asarray(M, F32).reshape(3, 4)
    return np.stack([fma32(M[c, 2], v[2], fma32(M[c, 1], v[1], fma32(M[c, 0], v[0], M[c, 3]))) for c in range(3)])


def _np(t, dt=F32):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        t = t.detach().cpu().numpy()
    return np.asarray(t).astype(dt)


def tile_plan(m, H, W, footprint=False):
    """The forward's plan per 16 x 16 output tile: 'empty', 'plan' (shared memory) or 'direct' [tiles_y, tiles_x]; with
    ``footprint`` also the largest of the three shared-memory regions the tile asks for, in floats."""
    ty_, tx_ = np.meshgrid(np.arange((H + T - 1) // T), np.arange((W + T - 1) // T), indexing="ij")
    ox0, oy0 = tx_ * T, ty_ * T
    nox, noy = np.minimum(T, W - ox0), np.minimum(T, H - oy0)
    qx0, qy0 = 2 * ox0 + 1, 2 * oy0 + 1
    nqx, nqy = 2 * nox + 10, 2 * noy + 10
    ux0, ux1, uy0, uy1 = m.nu_box(qx0, qx0 + nqx - 1, qy0, qy0 + nqy - 1, H, W)
    ex0, ex1 = np.maximum(_cdiv2(ux0 - 6), -(W - 1)), np.minimum(_fdiv2(ux1 + 5), 2 * (W - 1))
    ey0, ey1 = np.maximum(_cdiv2(uy0 - 6), -(H - 1)), np.minimum(_fdiv2(uy1 + 5), 2 * (H - 1))
    nux, nuy, nex, ney = ux1 - ux0 + 1, uy1 - uy0 + 1, ex1 - ex0 + 1, ey1 - ey0 + 1
    empty = (nux <= 0) | (nuy <= 0) | (nex <= 0) | (ney <= 0)
    fits = empty | ((nex * ney <= CAP) & (ney * nux <= CAP) & (nuy * nux <= CAP))
    plan = np.where(empty, "empty", np.where(fits, "plan", "direct"))
    if footprint:
        return plan, np.where(empty, 0, np.maximum(np.maximum(nex * ney, ney * nux), nuy * nux))
    return plan


# ------------------------------------------------------------------------------------------------ forward
def forward(x, geom, frac, color=None, check=True, stats=None):
    """gf_augment_resample_nchw's output [B, C, H, W] (fp32).  ``stats`` (a dict) collects the tiles per path."""
    x, frac, geom = _np(x), _np(frac), _np(geom, np.int64)
    color = _np(color)
    B, C, H, W = x.shape
    y = np.empty_like(x)
    for b in range(B):
        m = ResMap(frac[b], geom[b], H, W, check)
        if m.ident:
            sy, sx = _blit_index(m, H, W)
            v = x[b][:, sy, sx]
            y[b] = v if color is None else _colour(v, color[b])
            continue
        if not m.ok:
            y[b] = np.nan
            continue
        plan = tile_plan(m, H, W)
        if stats is not None:
            for kind in ("empty", "plan", "direct"):
                stats[kind] = stats.get(kind, 0) + int((plan == kind).sum())
        qx = np.arange(1, 2 * W + 11, dtype=F32)[None, :]
        qy = np.arange(1, 2 * H + 11, dtype=F32)[:, None]
        nx, ny = m.nu(np.broadcast_to(qx, (2 * H + 10, 2 * W + 10)), np.broadcast_to(qy, (2 * H + 10, 2 * W + 10)))
        E = x[b][:, _mirror(np.arange(-(H - 1), 2 * H - 1), H)][:, :, _mirror(np.arange(-(W - 1), 2 * W - 1), W)]
        out = np.zeros((C, H, W), F32)
        if (plan != "direct").any():
            U = np.swapaxes(_up_axis(np.swapaxes(_up_axis(E, W), -1, -2), H), -1, -2)      # [C, 6H - 4, 6W - 4]
            fx, fy = np.floor(nx), np.floor(ny)
            ax, ay = F32(nx - fx), F32(ny - fy)
            jx, jy = fx.astype(np.int64) + 2 * (W - 1), fy.astype(np.int64) + 2 * (H - 1)

            def at(yy, xx):
                inside = (xx >= 0) & (xx < 6 * W - 4) & (yy >= 0) & (yy < 6 * H - 4)
                return np.where(inside, U[:, np.clip(yy, 0, 6 * H - 5), np.clip(xx, 0, 6 * W - 5)], F32(0))
            top = fma32(ax, at(jy, jx + 1), F32(F32(1) - ax) * at(jy, jx))
            bot = fma32(ax, at(jy + 1, jx + 1), F32(F32(1) - ax) * at(jy + 1, jx))
            out = _down(fma32(ay, bot, F32(F32(1) - ay) * top), H, W)
        if (plan == "direct").any():
            mx0, wx = _axis_weights(nx, W)
            my0, wy = _axis_weights(ny, H)
            acc = np.zeros((C,) + nx.shape, F32)
            for j in range(7):
                rows = np.clip(my0 + j, -(H - 1), 2 * (H - 1))
                r = np.zeros_like(acc)
                for i in range(7):
                    cols = np.clip(mx0 + i, -(W - 1), 2 * (W - 1))
                    r = fma32(wx[..., i], x[b][:, _mirror(rows, H), _mirror(cols, W)], r)
                acc = fma32(wy[..., j], r, acc)
            od = _down(acc, H, W)
            sel = np.repeat(np.repeat(plan == "direct", T, 0), T, 1)[:H, :W]
            out = np.where(sel, od, out)
        out = np.where(np.repeat(np.repeat(plan == "empty", T, 0), T, 1)[:H, :W], F32(0), out)
        y[b] = out if color is None else _colour(out, color[b])
    return y


# ------------------------------------------------------------------------------------------------ adjoint
def _copy_box(k, i0, i1, N):
    if k == 0:
        return i0, i1
    if k == 1:
        return -i1, -max(i0, 1)
    return 2 * (N - 1) - min(i1, N - 2), 2 * (N - 1) - i0


def _copy_index(k, i, N):
    return i if k == 0 else (-i if k == 1 else 2 * (N - 1) - i)


def _segmented_fma(seg, w, g, nseg):
    """acc[:, s] = in-order fma chain over the entries of segment s (entries already sorted within each segment)."""
    n = seg.shape[0]
    acc = np.zeros((g.shape[0], nseg), F32)
    if n == 0:
        return acc, 0
    start = np.r_[True, seg[1:] != seg[:-1]]
    first = np.flatnonzero(start)
    rank = np.arange(n) - first[np.cumsum(start) - 1]
    order = np.argsort(rank, kind="stable")
    counts = np.bincount(rank)
    pos = 0
    for cnt in counts:
        sl = order[pos:pos + cnt]
        pos += cnt
        acc[:, seg[sl]] = fma32(w[sl], g[:, sl], acc[:, seg[sl]])
    return acc, len(counts)


def _segmented_add(seg, v, nseg):
    """out[:, s] = 0 + v_1 + v_2 + ... in fp32, in entry order within each segment."""
    out = np.zeros((v.shape[0], nseg), F32)
    n = seg.shape[0]
    if n == 0:
        return out, 0
    start = np.r_[True, seg[1:] != seg[:-1]]
    first = np.flatnonzero(start)
    rank = np.arange(n) - first[np.cumsum(start) - 1]
    counts = np.bincount(rank)
    for r in range(len(counts)):
        sl = np.flatnonzero(rank == r)
        out[:, seg[sl]] = F32(1) * (out[:, seg[sl]] + v[:, sl])
    return out, len(counts)


def adjoint(gy, geom, frac, color=None, check=True, stats=None):
    """gf_augment_resample_adjoint_nchw's output [B, C, H, W] (fp32).  ``stats`` collects the largest number of chunks a (tile,
    copy) box has, the longest in-order chain of one nu in one chunk, and whether any nu's box left out a nonzero tap."""
    gy, frac, geom = _np(gy), _np(frac), _np(geom, np.int64)
    color = _np(color)
    B, C, H, W = gy.shape
    gx = np.empty_like(gy)
    st = stats if stats is not None else {}
    st.setdefault("chunks", 0)
    st.setdefault("chain", 0)
    st.setdefault("chunk_adds", 0)
    st.setdefault("dropped", 0)
    for b in range(B):
        m = ResMap(frac[b], geom[b], H, W, check)
        g = gy[b]
        if m.ident:
            gx[b] = _blit_adjoint(g, m, None if color is None else color[b], H, W)
            continue
        if not m.ok:
            gx[b] = np.nan
            continue
        if color is not None:
            M = color[b].reshape(3, 4)
            g = np.stack([fma32(M[2, c], g[2], fma32(M[1, c], g[1], F32(M[0, c] * g[0]))) for c in range(3)])
        # transposed down filter: gVx [C, H, 2W + 10], gV [C, 2H + 10, 2W + 10] (index q - 1)
        def tdown(a, N):                                                # along the last axis
            q = np.arange(1, 2 * N + 11)
            olo = _cdiv2(q - 12)
            acc = np.zeros(a.shape[:-1] + q.shape, F32)
            for t in range(6):
                o = olo + t
                ok = (o >= 0) & (o <= N - 1) & (o <= _fdiv2(q - 1))
                acc = fma32(np.where(ok, TAPS[np.clip(q - 1 - 2 * o, 0, 11)], F32(0)), a[..., np.clip(o, 0, N - 1)], acc)
            return acc
        gV = np.swapaxes(tdown(np.swapaxes(tdown(g, W), -1, -2), H), -1, -2)
        QX, QY = 2 * W + 10, 2 * H + 10
        qxg = np.broadcast_to(np.arange(1, QX + 1, dtype=F32)[None, :], (QY, QX))
        qyg = np.broadcast_to(np.arange(1, QY + 1, dtype=F32)[:, None], (QY, QX))
        nx, ny = m.nu(qxg, qyg)
        fxg, fyg = np.floor(nx), np.floor(ny)
        axg, ayg = F32(nx - fxg), F32(ny - fyg)
        jxg, jyg = fxg.astype(np.int64), fyg.astype(np.int64)
        rx0, rx1, ry0, ry1 = (int(v) for v in m.nu_box(1, QX, 1, QY, H, W))
        rmx0, rmx1 = max(int(_cdiv2(rx0 - 6)), -(W - 1)), min(int(_fdiv2(rx1 + 5)), 2 * (W - 1))
        rmy0, rmy1 = max(int(_cdiv2(ry0 - 6)), -(H - 1)), min(int(_fdiv2(ry1 + 5)), 2 * (H - 1))
        total = np.zeros((C, H, W), F32)
        for sy0 in range(0, H, T):
            for sx0 in range(0, W, T):
                nsx, nsy = min(T, W - sx0), min(T, H - sy0)
                for k in range(9):
                    kx, ky = k % 3, k // 3
                    mx0, mx1 = _copy_box(kx, sx0, sx0 + nsx - 1, W)
                    my0, my1 = _copy_box(ky, sy0, sy0 + nsy - 1, H)
                    if mx0 > mx1 or my0 > my1:
                        continue
                    mx0, mx1, my0, my1 = max(mx0, rmx0), min(mx1, rmx1), max(my0, rmy0), min(my1, rmy1)
                    if mx0 > mx1 or my0 > my1 or rx0 > rx1 or ry0 > ry1:
                        continue
                    ux0, ux1 = max(2 * mx0 - 5, -2 * (W - 1)), min(2 * mx1 + 6, 4 * W - 3)
                    uy0, uy1 = max(2 * my0 - 5, -2 * (H - 1)), min(2 * my1 + 6, 4 * H - 3)
                    nux, nuy = ux1 - ux0 + 1, uy1 - uy0 + 1
                    if nux <= 0 or nuy <= 0:
                        continue
                    cq = []
                    for j in range(4):
                        dx = F32(F32((ux0 - 1, ux1 + 1)[j & 1]) - m.e0)
                        dy = F32(F32((uy0 - 1, uy1 + 1)[j >> 1]) - m.e1)
                        cq.append((fma32(m.i00, dx, F32(m.i01 * dy)), fma32(m.i10, dx, F32(m.i11 * dy))))
                    cxmin, cxmax = min(c[0] for c in cq), max(c[0] for c in cq)
                    cymin, cymax = min(c[1] for c in cq), max(c[1] for c in cq)
                    qx0 = max(int(np.floor(max(cxmin, F32(-1e8)))) - 1, 1)
                    qx1 = min(int(np.ceil(min(cxmax, F32(1e8)))) + 1, QX)
                    qy0 = max(int(np.floor(max(cymin, F32(-1e8)))) - 1, 1)
                    qy1 = min(int(np.ceil(min(cymax, F32(1e8)))) + 1, QY)
                    if qx0 > qx1 or qy0 > qy1:
                        continue
                    st["chunks"] = max(st["chunks"], ((qx1 - qx0) // QC + 1) * ((qy1 - qy0) // QC + 1))
                    gU = _gather(m, gV, jxg, jyg, axg, ayg, qx0, qx1, qy0, qy1, ux0, ux1, uy0, uy1, st)    # [C, nuy, nux]
                    # transposed up filter along x: Ax [C, nuy, nmx]
                    mm = np.arange(mx0, mx1 + 1)
                    acc = np.zeros((C, nuy, mm.size), F32)
                    for t in range(12):
                        nu = 2 * mm - 5 + t
                        ok = (nu >= ux0) & (nu <= ux1)
                        acc = fma32(np.where(ok, TAPS[t], F32(0)), gU[:, :, np.clip(nu - ux0, 0, nux - 1)], acc)
                    Ax = F32(2) * acc
                    # ... along y at this tile's pixels in this copy
                    py, px = np.meshgrid(np.arange(sy0, sy0 + nsy), np.arange(sx0, sx0 + nsx), indexing="ij")
                    mxp, myp = _copy_index(kx, px, W), _copy_index(ky, py, H)
                    here = ((kx != 1) | (px >= 1)) & ((kx != 2) | (px <= W - 2)) & ((ky != 1) | (py >= 1)) & \
                           ((ky != 2) | (py <= H - 2)) & (mxp >= mx0) & (mxp <= mx1) & (myp >= my0) & (myp <= my1)
                    acc = np.zeros((C, nsy, nsx), F32)
                    col = np.clip(mxp - mx0, 0, mm.size - 1)
                    for t in range(12):
                        nu = 2 * myp - 5 + t
                        ok = (nu >= uy0) & (nu <= uy1)
                        acc = fma32(np.where(ok, TAPS[t], F32(0)), Ax[:, np.clip(nu - uy0, 0, nuy - 1), col], acc)
                    blk = total[:, sy0:sy0 + nsy, sx0:sx0 + nsx]
                    total[:, sy0:sy0 + nsy, sx0:sx0 + nsx] = np.where(here, F32(1) * (blk + F32(2) * acc), blk)
        gx[b] = total
    return gx


def _gather(m, gV, jxg, jyg, axg, ayg, qx0, qx1, qy0, qy1, ux0, ux1, uy0, uy1, st):
    """gU over one (tile, copy) box: per nu, the sum over 64 x 64 chunks of the q box in chunk order (cy0 outer), of the chunk's
    in-order sum over q row-major of fmaf(round(wy wx), gV(q), acc), q inside the kernel's preimage box of nu."""
    C = gV.shape[0]
    nux, nuy = ux1 - ux0 + 1, uy1 - uy0 + 1
    sl = (slice(qy0 - 1, qy1), slice(qx0 - 1, qx1))
    jx, jy, ax, ay = jxg[sl], jyg[sl], axg[sl], ayg[sl]
    qy, qx = np.meshgrid(np.arange(qy0, qy1 + 1), np.arange(qx0, qx1 + 1), indexing="ij")
    ncx = (qx1 - qx0) // QC + 1
    parts = []
    for dy in (0, 1):
        for dx in (0, 1):
            tx_, ty_ = jx + dx, jy + dy
            wx = F32(F32(1) - ax) if dx == 0 else ax
            wy = F32(F32(1) - ay) if dy == 0 else ay
            keep = (tx_ >= ux0) & (tx_ <= ux1) & (ty_ >= uy0) & (ty_ <= uy1) & (wx != 0) & (wy != 0)
            idx = np.flatnonzero(keep)
            parts.append((idx, (ty_.ravel()[idx] - uy0) * nux + tx_.ravel()[idx] - ux0, F32(wy.ravel()[idx] * wx.ravel()[idx])))
    qidx = np.concatenate([p[0] for p in parts])
    tgt = np.concatenate([p[1] for p in parts])
    w = np.concatenate([p[2] for p in parts]).astype(F32)
    qxs, qys = qx.ravel()[qidx], qy.ravel()[qidx]
    # the kernel's per-nu preimage box [floor(c - h), ceil(c + h)]
    tnx, tny = tgt % nux + ux0, tgt // nux + uy0
    ddx, ddy = F32(tnx.astype(F32) - m.e0), F32(tny.astype(F32) - m.e1)
    cx, cy = fma32(m.i00, ddx, F32(m.i01 * ddy)), fma32(m.i10, ddx, F32(m.i11 * ddy))
    inbox = (qxs >= np.floor(F32(cx - m.hx))) & (qxs <= np.ceil(F32(cx + m.hx))) & \
            (qys >= np.floor(F32(cy - m.hy))) & (qys <= np.ceil(F32(cy + m.hy)))
    st["dropped"] += int((~inbox).sum())
    qidx, tgt, w, qxs, qys = qidx[inbox], tgt[inbox], w[inbox], qxs[inbox], qys[inbox]
    chunk = ((qys - qy0) // QC) * ncx + (qxs - qx0) // QC
    order = np.lexsort((qxs, qys, chunk, tgt))
    qidx, tgt, w, chunk = qidx[order], tgt[order], w[order], chunk[order]
    seg_key = tgt * (ncx * ((qy1 - qy0) // QC + 1)) + chunk
    start = np.r_[True, seg_key[1:] != seg_key[:-1]] if seg_key.size else np.zeros(0, bool)
    seg = np.cumsum(start) - 1
    nseg = int(seg[-1]) + 1 if seg.size else 0
    gflat = gV[:, qy0 - 1:qy1, qx0 - 1:qx1].reshape(C, -1)[:, qidx]
    partial, chain = _segmented_fma(seg, w, gflat, nseg)
    st["chain"] = max(st["chain"], chain)
    seg_tgt = tgt[start] if seg_key.size else tgt
    sums, nadd = _segmented_add(seg_tgt, partial, nux * nuy)
    st["chunk_adds"] = max(st["chunk_adds"], nadd)
    return sums.reshape(C, nuy, nux)


def _blit_adjoint(g, m, M, H, W):
    """augment_adjoint_kernel for one image: each source pixel gathers its preimages (q, then its one reachable mirror) in order."""
    C = g.shape[0]

    def pre(q, t, N):
        out = []
        if -t <= q <= N - 1 - t:
            out.append(q)
        if 0 < q <= t:
            out.append(-q)
        if N - 1 + t <= q < N - 1:
            out.append(2 * (N - 1) - q)
        return out

    def dinv(u, v):
        k = m.code >> 1
        x, y = [(u, v), (W - 1 - v, u), (W - 1 - u, H - 1 - v), (v, H - 1 - u)][k]
        return (W - 1 - x if m.code & 1 else x), y
    out = np.zeros((C, H, W), F32)
    if M is not None:
        M = np.asarray(M, F32).reshape(3, 4)
    for qy in range(H):
        for qx in range(W):
            acc = np.zeros(C, F32)
            for sy in pre(qy, m.ty, H):
                for sx in pre(qx, m.tx, W):
                    px, py = dinv(sx + m.tx, sy + m.ty)
                    v = g[:, py, px]
                    if M is None:
                        acc = F32(1) * (acc + v)
                    else:
                        acc = F32(1) * (acc + np.array([fma32(M[2, c], v[2], fma32(M[1, c], v[1], F32(M[0, c] * v[0])))
                                                        for c in range(3)], F32))
            out[:, qy, qx] = acc
    return out


# ------------------------------------------------------------------------------------------------ fp64 at given positions
def forward64_at(x, nx, ny, taps=None):
    """The resampler in fp64 (ops.resample_ref's steps) with the sample positions nu given [B, 2H + 10, 2W + 10] (index q - 1):
    ``forward64_at(x, *positions64(...))`` is the definition; with the kernel's fp32 positions it isolates their share of the error."""
    x = torch.as_tensor(x, dtype=torch.float64)
    B, C, H, W = x.shape
    f = torch.as_tensor(TAPS.astype(np.float64) if taps is None else taps, dtype=torch.float64)
    fl = f.flip(0)
    mi = lambda N: torch.as_tensor(_mirror(np.arange(-(N - 1), 2 * N - 1), N))
    E = x[:, :, mi(H)][:, :, :, mi(W)].reshape(B * C, 1, 3 * H - 2, 3 * W - 2)
    Z = E.new_zeros(B * C, 1, 6 * H - 4, 6 * W - 4)
    Z[:, :, ::2, ::2] = E
    Z = torch.nn.functional.pad(Z, [6, 5, 6, 5])
    U = torch.nn.functional.conv2d(torch.nn.functional.conv2d(Z, 2 * fl.reshape(1, 1, 1, 12)), 2 * fl.reshape(1, 1, 12, 1))
    UH, UW = 6 * H - 4, 6 * W - 4
    nx = torch.as_tensor(nx, dtype=torch.float64).reshape(B, 1, -1) + 2 * (W - 1)
    ny = torch.as_tensor(ny, dtype=torch.float64).reshape(B, 1, -1) + 2 * (H - 1)
    x0, y0 = nx.floor(), ny.floor()
    ax, ay = nx - x0, ny - y0
    Uf = U.reshape(B, C, UH * UW)
    V = 0
    for dy, wy in ((0, 1 - ay), (1, ay)):
        for dx, wx in ((0, 1 - ax), (1, ax)):
            ix, iy = x0 + dx, y0 + dy
            inside = (ix >= 0) & (ix < UW) & (iy >= 0) & (iy < UH)
            idx = (iy.clamp(0, UH - 1) * UW + ix.clamp(0, UW - 1)).long().expand(B, C, -1)
            V = V + torch.where(inside, wx * wy, torch.zeros_like(wx)) * Uf.gather(2, idx)
    V = V.reshape(B * C, 1, 2 * H + 10, 2 * W + 10)
    y = torch.nn.functional.conv2d(torch.nn.functional.conv2d(V, f.reshape(1, 1, 1, 12), stride=(1, 2)), f.reshape(1, 1, 12, 1),
                                   stride=(2, 1))
    return y.reshape(B, C, H, W)


def positions(geom, frac, H, W, check=False):
    """The kernels' fp32 sample positions (nu_x, nu_y) [B, 2H + 10, 2W + 10] as float64 arrays."""
    geom, frac = _np(geom, np.int64), _np(frac)
    qx = np.broadcast_to(np.arange(1, 2 * W + 11, dtype=F32)[None, :], (2 * H + 10, 2 * W + 10))
    qy = np.broadcast_to(np.arange(1, 2 * H + 11, dtype=F32)[:, None], (2 * H + 10, 2 * W + 10))
    out = [ResMap(frac[b], geom[b], H, W, check).nu(qx, qy) for b in range(frac.shape[0])]
    return np.stack([o[0] for o in out]).astype(np.float64), np.stack([o[1] for o in out]).astype(np.float64)
