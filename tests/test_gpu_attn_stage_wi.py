"""GPU tests of stage W (gf_attn_fold_weights), stage I (the per-image tables) and the instance / batch statistics (run on an H100:
``pytest -m gpu``).  The kernels are a black box behind the exported entry points; the tables are read from a workspace filled
with a NaN pattern before the call, at the offsets gf_attn_debug_layout reports, and the test checks that every table element was
written and (where the call writes nothing else) that nothing outside the tables was.

* Exact cases (``oracle/stage_wi.py``): small-integer weights and latents, every fan-in a power of four, one-hot positional weights.
  The tables equal the host's fp64 restatement of the kernel chain bit for bit, in fp32 mode and in the default (TF32) mode, where
  K' is tf32_rne(fp32(K' d kf)), V^T tf32_rne(V^T) (ties among them: round-to-nearest-even is pinned) and Rt / Ct carry
  fp32(. * log2 e).  Simplex with 1 and 4 heads (two heads cannot make both C and C/2 powers of four: section 4 covers them), three
  integrations, in_scale, k on both sides of 16, the batched prologue, duplex pass-A tables, duplex keys from given centroids and
  from Xbar, and the k-means query fold ACQ.  The key GEMM reaches gemm_tc_kernel (default mode: ragged row and column tiles, k = 13
  against the 64-row tiles, 2 and 8 k-tiles) and gemm64_kernel / gemm_kernel (fp32 mode).
* Realistic shapes: the benchmarked generator's layer shapes on random weights against fp64, per element relative to the same
  expression on absolute values.
* gf_attn_norm_stats: exact integer cases bit for bit (both modes, B = 1 in batch mode, C = 96 and 1024, a constant channel, a
  channel at mean 1000, split counts derived from the SM count, an empty last split), float cases within one fp32 ulp, and the
  affine path of token_simt_kernel on statistics that are powers of two.
``tests/test_host_cpu_attn_stage_wi.py`` proves on the host that every exact case here is exact.
"""
import ctypes
import math

import pytest
import torch

from oracle import bipartite as ob
from oracle import folded as of
from oracle import stage_wi as sw
from oracle import attn_fwd as af
from tests.guards import GUARD_BITS, Guarded, assert_exact
from tests.test_gpu_attn_forward import Postop, _f32, _lib, _region, _stream, _weights_struct, make_ws, sm_count

pytestmark = pytest.mark.gpu


def _id(v):
    return str(v)


# Per-element bounds of |kernel - fp64| (less half a TF32 ulp where the table is TF32-rounded) relative to the same expression on
# absolute values, over REALISTIC.  Measured worst cases on an H100 80GB HBM3 at a 700 W power limit: 4.69e-8 for the fp32 sums
# of stages W and I (both modes), 6.40e-6 for the duplex keys of the default mode, whose GEMM truncates the centroids and AK to
# TF32 (the compensation 1.000352220^2 removes the bias, not the spread); frozen at 1.5x.
BOUND = {"fp32": 7.1e-8, "tc_gemm": 9.6e-6}


# ---- exact cases: host side (also run by the CPU test) ------------------------------------------------------------------------
# (heads, C, D, p, k, integration, in_scale)
SIMPLEX = [
    (1, 64, 16, 4, 13, "mul", False),
    (1, 64, 64, 0, 20, "add", True),
    (1, 256, 16, 16, 27, "mul", True),
    (1, 256, 64, 16, 5, "mul", False),
    (4, 64, 16, 16, 5, "mul", True),
    (4, 64, 64, 4, 8, "both", False),
    (4, 256, 16, 0, 7, "add", False),
    (4, 256, 64, 16, 3, "mul", True),
]
HW = (8, 12)


def simplex_case(heads, C, D, p, k, integration, in_scale, *, B=3):
    seed = heads * 1000 + C + D + p + k
    w = sw.exact_weights(C, D, k, p, integration, seed=seed)
    y = sw.exact_latents(B, k, D, seed + 1)
    d = None
    if in_scale:
        d = 2.0 ** torch.randint(-1, 2, (B, C), generator=torch.Generator().manual_seed(seed + 2)).double()
    return w, y, d


def simplex_expected(w, y, d, *, heads, C, D, k, integration, tf32):
    p = w["pos_latent"].shape[1]
    H, W = HW
    f = sw.stage_w(w, C=C, D=D, k=k, integration=integration, heads=heads)
    seg = of.head_segment(k, heads)
    KP = of.pad_k(heads * seg) if heads > 1 else of.pad_k(k)
    kp, v = sw.simplex_rows(f, y, heads=heads)
    Kp, Vt, Rt, Ct = sw.tables(kp, v, C=C, p=p, H=H, W=W, k=k, heads=heads, seg=seg, KP=KP, tf32_k=tf32, tf32_v=tf32, d=d)
    return dict(Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct, CB=f["CB"].float()), f


# duplex key cases (B, C, D, p, k): B*k = 143 rows (3 row tiles, the last one ragged), 260 (gemm64_kernel in fp32 mode)
DUPLEX = [(11, 64, 16, 0, 13), (20, 256, 64, 16, 13), (5, 64, 16, 4, 20), (3, 256, 16, 16, 32)]


def duplex_case(B, C, D, p, k, *, wcq=False):
    seed = 7 * B + C + D + p + k
    w = sw.exact_weights(C, D, k, p, "mul", duplex=True, wcq=wcq, seed=seed)
    y = sw.exact_latents(B, k, D, seed + 1)
    cen = torch.randint(-8, 9, (B, k, C), generator=torch.Generator().manual_seed(seed + 2)).double()
    return w, y, cen


def duplex_key_expected(f, src, y, *, C, p, k, tc, key="AK"):
    H, W = HW
    A, Cst = (f["AK"][0], f["CK"][0]) if key == "AK" else (f["AK2"], f["CK2"])
    kp = sw.key_rows(src, A, Cst, tc=tc)
    v = sw.exact_mm(y, f["AV"][0], E=f["CV"][0][None, None], name="v")
    Kp, Vt, Rt, Ct = sw.tables(kp[None], v[None], C=C, p=p, H=H, W=W, k=k, heads=1, seg=of.pad_k(k), KP=of.pad_k(k),
                               tf32_k=tc, tf32_v=tc)
    return dict(Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct)


def duplex_passa_expected(f, y, *, C, p, k, tc, cen=None):
    """Pass-A tables M, Rt2, Ct2 from the latents (AM, CM) or, with cen, from the centroids (ACQ, CM: fp32 GEMM); V^T."""
    H, W = HW
    m = sw.key_rows(cen, f["ACQ"], f["CM"], tc=False) if cen is not None else sw.exact_mm(y, f["AM"], E=f["CM"][None], name="m")
    v = sw.exact_mm(y, f["AV"][0], E=f["CV"][0][None, None], name="v")
    M, Vt, Rt2, Ct2 = sw.tables(m[None], v[None], C=C, p=p, H=H, W=W, k=k, heads=1, seg=of.pad_k(k), KP=of.pad_k(k),
                                tf32_k=tc, tf32_v=tc)
    return dict(M=M, Vt=Vt, Rt2=Rt2, Ct2=Ct2)


# ---- device helpers ------------------------------------------------------------------------------------------------------------
def fold(gf, dev, desc, w):
    folded = torch.empty(gf._lib.folded_floats(desc), device=dev)
    wst, keep = _weights_struct(gf, w, dev)
    gf._lib.check(_lib(gf).gf_attn_fold_weights(ctypes.byref(desc), ctypes.byref(wst), folded.data_ptr(), _stream(dev)), "fold")
    torch.cuda.synchronize()
    return folded


def shapes(B, C, k, KP, Cout, duplex=False, H=HW[0], W=HW[1]):
    s = {"Kp": (B, KP, C), "Vt": (B, Cout, KP), "Rt": (B, H, KP), "Ct": (B, W, KP), "CB": (Cout,)}
    if duplex:
        s.update(M=(B, KP, C), Rt2=(B, H, KP), Ct2=(B, W, KP))
    return s


def read(ws, lay, shp, names, *, only=False):
    """The named tables (fp32, CPU) of a NaN-filled workspace; every element must be written.  only: nothing else was."""
    bits = ws.view(torch.int32).cpu()
    inside = torch.zeros_like(bits, dtype=torch.bool)
    out = {}
    for name in names:
        off, n = lay[name], math.prod(shp[name])
        assert not (bits[off:off + n] == GUARD_BITS).any(), f"{name}: elements left unwritten"
        inside[off:off + n] = True
        out[name] = ws[off:off + n].view(shp[name]).cpu()
    if only:
        assert (bits[~inside] == GUARD_BITS).all(), f"written outside {names}"
    return out


def check_tables(got, want):
    for name in want:
        assert_exact(got[name], want[name], name)


def prologue_ex(gf, dev, desc, folded, y, d, C):
    B = y.shape[0]
    ws, lay = make_ws(gf, desc, dev)
    Y = _f32(y, dev)
    po = Postop(gf, {"in_scale": d} if d is not None else None, dev, B, 1, C)
    gf._lib.check(_lib(gf).gf_attn_prologue_ex(ctypes.byref(desc), Y.data_ptr(), folded.data_ptr(), ws.data_ptr(), ctypes.byref(po.s),
                                               _stream(dev)), "gf_attn_prologue_ex")
    torch.cuda.synchronize()
    return ws, lay


def prologue_batch(gf, dev, descs, foldeds, ys, ds, Cs):
    lib = _lib(gf)
    n = len(descs)
    wss, keep = [], []
    for desc, y, d, C in zip(descs, ys, ds, Cs):
        ws, lay = make_ws(gf, desc, dev)
        wss.append((ws, lay))
        keep += [_f32(y, dev), Postop(gf, {"in_scale": d} if d is not None else None, dev, y.shape[0], 1, C)]
    P = ctypes.c_void_p * n
    dp = (ctypes.POINTER(gf._lib.GfAttnDesc) * n)(*[ctypes.pointer(x) for x in descs])
    pp = (ctypes.POINTER(gf._lib.GfAttnPostop) * n)(*[ctypes.pointer(keep[2 * i + 1].s) for i in range(n)])
    gf._lib.check(lib.gf_attn_prologue_batch(n, dp, P(*[keep[2 * i].data_ptr() for i in range(n)]), P(*[x.data_ptr() for x in foldeds]),
                                             P(*[w.data_ptr() for w, _ in wss]), pp, _stream(dev)), "gf_attn_prologue_batch")
    torch.cuda.synchronize()
    return wss


# ---- exact stage W + I: simplex ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ("fp32", "tf32"))
@pytest.mark.parametrize("heads,C,D,p,k,integration,in_scale", SIMPLEX, ids=_id)
def test_simplex_tables_exact(gf, cuda_dev, mode, heads, C, D, p, k, integration, in_scale):
    """gf_attn_fold_weights + gf_attn_prologue_ex on an exact case: K', V^T, Rt, Ct and CB equal the host's bits, every padded
    column (j % seg >= k) is 0 / -inf, and nothing else in the workspace is written."""
    B, (H, W) = 3, HW
    w, y, d = simplex_case(heads, C, D, p, k, integration, in_scale)
    flags = gf._lib.FLAG_FP32_EXACT if mode == "fp32" else 0
    desc = gf._lib.make_desc(B, H, W, C, k, D, heads=heads, norm="layer", integration=integration, pos_dim=p, flags=flags)
    assert _lib(gf).gf_attn_tc_eligible(ctypes.byref(desc)) == (mode == "tf32")
    want, _ = simplex_expected(w, y, d, heads=heads, C=C, D=D, k=k, integration=integration, tf32=mode == "tf32")
    folded = fold(gf, cuda_dev, desc, w)
    ws, lay = prologue_ex(gf, cuda_dev, desc, folded, y, d, C)
    KP, Cout = want["Kp"].shape[1], want["Vt"].shape[1]
    got = read(ws, lay, shapes(B, C, k, KP, Cout), ("Kp", "Vt", "Rt", "Ct", "CB"), only=True)
    check_tables(got, want)


def test_prologue_batch_exact(gf, cuda_dev):
    """gf_attn_prologue_batch with five layers of different shapes (one head and four, both modes, a duplex layer's pass-A tables)
    in one launch: every layer's tables equal the host's bits, and those of a call per layer."""
    B, (H, W) = 3, HW
    descs, foldeds, ys, ds, Cs, wants = [], [], [], [], [], []
    for i, (heads, C, D, p, k, integration, in_scale) in enumerate(SIMPLEX[::2]):
        w, y, d = simplex_case(heads, C, D, p, k, integration, in_scale)
        flags = gf._lib.FLAG_FP32_EXACT if i % 2 else 0
        desc = gf._lib.make_desc(B, H, W, C, k, D, heads=heads, norm="layer", integration=integration, pos_dim=p, flags=flags)
        descs.append(desc), foldeds.append(fold(gf, cuda_dev, desc, w)), ys.append(y), ds.append(d), Cs.append(C)
        wants.append(simplex_expected(w, y, d, heads=heads, C=C, D=D, k=k, integration=integration, tf32=not flags)[0])
    Bd, C, D, p, k = 3, 64, 16, 4, 13
    w, y, _ = duplex_case(Bd, C, D, p, k)
    desc = gf._lib.make_desc(Bd, H, W, C, k, D, norm="layer", integration="mul", pos_dim=p, duplex=1)
    descs.append(desc), foldeds.append(fold(gf, cuda_dev, desc, w)), ys.append(y), ds.append(None), Cs.append(C)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    wants.append(duplex_passa_expected(f, y, C=C, p=p, k=k, tc=True))
    wss = prologue_batch(gf, cuda_dev, descs, foldeds, ys, ds, Cs)
    for i, ((ws, lay), want) in enumerate(zip(wss, wants)):
        if "M" in want:
            shp = shapes(Bd, C, k, 16, C, duplex=True)
            got = read(ws, lay, shp, ("M", "Vt", "Rt2", "Ct2"), only=True)
        else:
            KP, Cout = want["Kp"].shape[1], want["Vt"].shape[1]
            shp = shapes(B, Cs[i], 0, KP, Cout)
            got = read(ws, lay, shp, ("Kp", "Vt", "Rt", "Ct", "CB"), only=True)
            ws1, _ = prologue_ex(gf, cuda_dev, descs[i], foldeds[i], ys[i], ds[i], Cs[i])
            assert torch.equal(ws.view(torch.int32), ws1.view(torch.int32)), f"layer {i}: batched and single calls differ"
        check_tables(got, want)


# ---- exact duplex: pass-A tables, keys from centroids and from Xbar, ACQ --------------------------------------------------------
def duplex_call(gf, dev, desc, folded, X, y, cen, *, post=None):
    B, n, C = X.shape
    ws, lay = make_ws(gf, desc, dev)
    Xd, Y = _f32(X, dev), _f32(y, dev)
    Xout = torch.empty_like(Xd)
    cd = _f32(cen, dev) if cen is not None else None
    gf._lib.check(_lib(gf).gf_attn_duplex_fwd_ex(ctypes.byref(desc), Xd.data_ptr(), Y.data_ptr(), folded.data_ptr(), Xout.data_ptr(),
                                                 None, cd.data_ptr() if cd is not None else None, ws.data_ptr(), None, _stream(dev)),
                  "gf_attn_duplex_fwd_ex")
    torch.cuda.synchronize()
    return ws, lay


@pytest.mark.parametrize("mode", ("fp32", "tf32"))
@pytest.mark.parametrize("B,C,D,p,k", DUPLEX, ids=_id)
def test_duplex_keys_from_centroids_exact(gf, cuda_dev, mode, B, C, D, p, k):
    """GF_FLAG_CENTROIDS_IN: KPALL = Cen AK + CK on gemm_tc_kernel (default mode; fp32(fp32(1.000352220f^2) S + CK[row % k])) or the
    CUDA-core GEMMs (fp32 mode), then finalize_kernel: K', V^T, Rt and Ct equal the host's bits."""
    H, W = HW
    w, y, cen = duplex_case(B, C, D, p, k)
    flags = gf._lib.FLAG_CENTROIDS_IN | (gf._lib.FLAG_FP32_EXACT if mode == "fp32" else 0)
    desc = gf._lib.make_desc(B, H, W, C, k, D, norm="layer", integration="mul", pos_dim=p, duplex=1, flags=flags)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    want = duplex_key_expected(f, cen, y, C=C, p=p, k=k, tc=mode == "tf32")
    X = torch.randint(-4, 5, (B, H * W, C), generator=torch.Generator().manual_seed(B)).double()
    ws, lay = duplex_call(gf, cuda_dev, desc, fold(gf, cuda_dev, desc, w), X, y, cen)
    got = read(ws, lay, shapes(B, C, k, of.pad_k(k), C), ("Kp", "Vt", "Rt", "Ct"))
    check_tables(got, want)


@pytest.mark.parametrize("B,C,D,p,k", [(3, 64, 16, 4, 13), (2, 256, 64, 16, 20)], ids=_id)
def test_duplex_keys_from_xbar_exact(gf, cuda_dev, B, C, D, p, k):
    """Centroids pointer NULL: the keys come straight from Xbar through AK2 = WV2 AK and CK2.  Pass A runs on planted one-hot tables
    (GF_FLAG_TABLES_READY, the construction of test_pass_a_exact), so Xbar = fp32(x_w 1.000352220f) for each latent's winner x_w,
    which the key GEMM's TF32 truncation takes back to x_w exactly."""
    H, W = HW
    n = H * W
    w, y, _ = duplex_case(B, C, D, p, k)
    desc = gf._lib.make_desc(B, H, W, C, k, D, norm="layer", integration="mul", pos_dim=p, duplex=1, flags=gf._lib.FLAG_TABLES_READY)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    win = torch.randint(0, n, (B, k), generator=torch.Generator().manual_seed(C + k))
    tabs, _, _ = af.exact_pass_a_case(B, H, W, C, k, winners=win, seed=C + k)
    xw = tabs["X"][torch.arange(B)[:, None], win]                                  # [B,k,C]
    want = duplex_key_expected(f, xw, y, C=C, p=p, k=k, tc=True, key="AK2")
    folded = fold(gf, cuda_dev, desc, w)
    ws, lay = make_ws(gf, desc, cuda_dev)
    for name in ("M", "Rt2", "Ct2"):
        _region(ws, lay[name], tabs[name].shape).copy_(_f32(tabs[name], cuda_dev))
    Xd, Y = _f32(tabs["X"], cuda_dev), _f32(y, cuda_dev)
    Xout = torch.empty_like(Xd)
    gf._lib.check(_lib(gf).gf_attn_duplex_fwd_ex(ctypes.byref(desc), Xd.data_ptr(), Y.data_ptr(), folded.data_ptr(), Xout.data_ptr(),
                                                 None, None, ws.data_ptr(), None, _stream(cuda_dev)), "gf_attn_duplex_fwd_ex")
    torch.cuda.synchronize()
    xbar = _region(ws, lay["XBAR"], (B, k, C)).double().cpu()
    assert torch.equal(xbar, (xw.float() * torch.tensor(sw.COMP, dtype=torch.float32)).double()), "Xbar"
    got = read(ws, lay, shapes(B, C, k, of.pad_k(k), C), ("Kp", "Rt", "Ct"))
    check_tables(got, {a: want[a] for a in ("Kp", "Rt", "Ct")})


@pytest.mark.parametrize("mode", ("fp32", "tf32"))
@pytest.mark.parametrize("B,C,D,p,k", [(3, 64, 16, 4, 13), (2, 256, 64, 16, 27)], ids=_id)
def test_duplex_pass_a_tables_exact(gf, cuda_dev, mode, B, C, D, p, k):
    """Pass-A tables of the latents (gf_attn_prologue_batch on a duplex layer) and of carried-in centroids (GF_FLAG_CENTROIDS_INIT:
    M = Cen ACQ + CM on the fp32 GEMM, then finalize_kernel): M, Rt2 and Ct2 (and V^T) equal the host's bits."""
    H, W = HW
    tc = mode == "tf32"
    fl = gf._lib.FLAG_FP32_EXACT if not tc else 0
    w, y, cen = duplex_case(B, C, D, p, k, wcq=True)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    desc = gf._lib.make_desc(B, H, W, C, k, D, norm="layer", integration="mul", pos_dim=p, duplex=1, flags=fl)
    (ws, lay), = prologue_batch(gf, cuda_dev, [desc], [fold(gf, cuda_dev, desc, w)], [y], [None], [C])
    shp = shapes(B, C, k, of.pad_k(k), C, duplex=True)
    check_tables(read(ws, lay, shp, ("M", "Vt", "Rt2", "Ct2"), only=True), duplex_passa_expected(f, y, C=C, p=p, k=k, tc=tc))
    desc = gf._lib.make_desc(B, H, W, C, k, D, norm="layer", integration="mul", pos_dim=p, duplex=1, flags=fl | gf._lib.FLAG_CENTROIDS_INIT)
    X = torch.randint(-4, 5, (B, H * W, C), generator=torch.Generator().manual_seed(B)).double()
    ws, lay = duplex_call(gf, cuda_dev, desc, fold(gf, cuda_dev, desc, w), X, y, cen)
    want = duplex_passa_expected(f, y, C=C, p=p, k=k, tc=tc, cen=cen)
    check_tables(read(ws, lay, shp, ("M", "Rt2", "Ct2")), {a: want[a] for a in ("M", "Rt2", "Ct2")})


# ---- realistic shapes ----------------------------------------------------------------------------------------------------------
# (B, H, W, C, heads, k, p, duplex): the benchmarked generator's attention layers (D = 32, k = 16) and a duplex layer, and two heads
REALISTIC = [(2, 16, 16, 512, 1, 16, 32, 0), (2, 32, 32, 256, 1, 16, 16, 0), (2, 64, 64, 128, 1, 16, 32, 0),
             (2, 16, 16, 128, 2, 16, 16, 0), (2, 16, 16, 256, 1, 16, 16, 1), (2, 32, 32, 512, 1, 16, 32, 1)]


def _companion_tables(w, y, cen, *, C, H, W, p, k, heads, duplex):
    """fp64 tables and the same expression on absolute values (weights, latents, centroids and positional tables)."""
    fw = of.fold_weights(w, C=C, k=k, integration="mul", duplex=bool(duplex), num_heads=heads)
    wa = {a: v.abs() for a, v in w.items()}
    fa = of.fold_weights(wa, C=C, k=k, integration="mul", duplex=bool(duplex), num_heads=heads)
    kw = dict(C=C, H=H, W=W, p=p, num_heads=heads)
    if duplex:
        kw.update(key_source=cen)
    Kp, Vt, Rt, Ct = of.prologue(y, fw, **kw)
    if duplex:
        kw.update(key_source=cen.abs())
    Ka, Va, _, _ = of.prologue(y.abs(), fa, **kw)
    # positional tables: |axis| against |kappa| (the kappa rows are the positional columns of the absolute key rows)
    half = p // 2
    row, col = ob.sinusoidal_axis(H, half).abs(), ob.sinusoidal_axis(W, half).abs()
    if heads == 1:
        kap = ((cen.abs() if duplex else y.abs()) @ fa["AK"] + fa["CK"][None])[:, :, C:][None]
    else:
        kap = torch.stack([y.abs() @ fa["AK"][h] + fa["CK"][h][None] for h in range(heads)])[:, :, :, C:]
    seg = of.head_segment(k, heads)
    Ra, Ca = torch.zeros_like(Rt), torch.zeros_like(Ct)
    for h in range(kap.shape[0]):
        cols = slice(h * seg, h * seg + k)
        Ra[:, :, cols] = torch.einsum("hq,bjq->bhj", row, kap[h][:, :, :half]) + kap[h][:, None, :, p]
        Ca[:, :, cols] = torch.einsum("wq,bjq->bwj", col, kap[h][:, :, half:p])
    return dict(Kp=Kp, Vt=Vt, Rt=Rt, Ct=Ct), dict(Kp=Ka, Vt=Va, Rt=Ra, Ct=Ca)


@pytest.mark.parametrize("mode", ("fp32", "tf32"))
@pytest.mark.parametrize("B,H,W,C,heads,k,p,duplex", REALISTIC, ids=_id)
def test_realistic_tables(gf, cuda_dev, mode, B, H, W, C, heads, k, p, duplex):
    """Random weights (N(0, 1), biases N(0, 0.2)), latents and centroids: every table element within BOUND times its companion (plus
    half a TF32 ulp where the default mode rounds it) of the fp64 table, scaled by kf / log2 e in the default mode."""
    D = 32
    tc = mode == "tf32"
    w = ob.init_params(C, D, k, p, "mul", bool(duplex), seed=C + p, bias_std=0.2)
    g = torch.Generator().manual_seed(C + k)
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64).float().double()
    cen = torch.randn(B, k, C, generator=g, dtype=torch.float64).float().double() if duplex else None
    want, comp = _companion_tables(w, y, cen, C=C, H=H, W=W, p=p, k=k, heads=heads, duplex=duplex)
    flags = 0 if tc else gf._lib.FLAG_FP32_EXACT
    if duplex:
        flags |= gf._lib.FLAG_CENTROIDS_IN
    desc = gf._lib.make_desc(B, H, W, C, k, D, heads=heads, norm="layer", integration="mul", pos_dim=p, duplex=duplex, flags=flags)
    folded = fold(gf, cuda_dev, desc, w)
    if duplex:
        X = torch.randn(B, H * W, C, generator=g)
        ws, lay = duplex_call(gf, cuda_dev, desc, folded, X.double(), y, cen)
    else:
        ws, lay = prologue_ex(gf, cuda_dev, desc, folded, y, None, C)
    KP = want["Kp"].shape[1]
    got = read(ws, lay, shapes(B, C, k, KP, C, H=H, W=W), ("Kp", "Vt", "Rt", "Ct"))
    for name in ("Kp", "Vt", "Rt", "Ct"):
        gv, wv, cv = got[name].double(), want[name], comp[name]
        live = torch.isfinite(wv) & (cv > 0)
        assert torch.equal(gv[~live], wv[~live]), f"{name}: padding"
        scale = {"Kp": sw.KF, "Rt": sw.LOG2E_F, "Ct": sw.LOG2E_F, "Vt": 1.0}[name] if tc else 1.0
        err = (gv - wv * scale).abs()
        if tc and name in ("Kp", "Vt"):
            err = (err - 2.0 ** (torch.floor(torch.log2(gv.abs().clamp_min(2.0 ** -126))) - 11)).clamp_min(0.0)
        r = (err[live] / (cv[live] * scale)).max().item()
        bound = BOUND["tc_gemm"] if duplex and tc and name != "Vt" else BOUND["fp32"]
        print(f"[stage-wi] {mode} B={B} {H}x{W} C={C} heads={heads} k={k} p={p} duplex={duplex} {name}: worst {r:.3e}")
        assert r <= bound, f"{name}: {r:.3e} > {bound:.1e}"


# ---- instance / batch statistics -----------------------------------------------------------------------------------------------
def norm_n(sms, B, *, empty_last):
    """A token count n for which norm_partial_kernel runs nsplit = min(ceil(2 SMs / B), ceil(n / 64)) >= 3 splits of
    ceil(n / nsplit) tokens, n divisible by neither nsplit nor 8, and the last split empty (or not)."""
    for n in range(200, 200000):
        ns = max(1, min((2 * sms + B - 1) // B, (n + 63) // 64))
        per = -(-n // ns)
        if ns >= 3 and n % ns and n % 8 and ((ns - 1) * per >= n) == empty_last:
            return n, ns
    raise AssertionError("no token count found")


def norm_x(B, n, C, seed, *, mean1000=True):
    g = torch.Generator().manual_seed(seed)
    X = torch.randint(-8, 9, (B, n, C), generator=g).double()
    X[:, :, 0] = 5.0                                                       # constant channel: var = 0
    if mean1000:
        X[:, :, 1] = 1000.0 + (torch.arange(n) % 2 * 2 - 1).double()        # mean ~1000, variance ~1
    return X


def run_norm(gf, dev, X, mode):
    B, n, C = X.shape
    desc = gf._lib.make_desc(B, 1, n, C, 8, 16, norm=mode, integration="mul", pos_dim=0)
    ws, lay = make_ws(gf, desc, dev)
    Xd = _f32(X, dev)
    gf._lib.check(_lib(gf).gf_attn_norm_stats(ctypes.byref(desc), Xd.data_ptr(), ws.data_ptr(), _stream(dev)), "gf_attn_norm_stats")
    torch.cuda.synchronize()
    got = read(ws, lay, {"NSCALE": (B, C), "NSHIFT": (B, C)}, ("NSCALE", "NSHIFT"))
    return got["NSCALE"], got["NSHIFT"]


@pytest.mark.parametrize("mode,B,C,empty_last", [("instance", 3, 96, False), ("instance", 2, 1024, True), ("batch", 1, 1024, False),
                                                 ("batch", 2, 96, True), ("batch", 5, 96, False)], ids=_id)
def test_norm_stats_exact(gf, cuda_dev, mode, B, C, empty_last):
    """Integer X: the fp64 sums are exact, so NSCALE / NSHIFT equal the host's IEEE-rounded mean, variance and 1/sqrt bit for bit."""
    n, ns = norm_n(sm_count(cuda_dev), B, empty_last=empty_last)
    X = norm_x(B, n, C, seed=B * C + n)
    sc, sh = run_norm(gf, cuda_dev, X, mode)
    want_sc, want_sh = sw.norm_stats(X, mode == "batch")
    assert_exact(sc, want_sc, "NSCALE")
    assert_exact(sh, want_sh, "NSHIFT")


@pytest.mark.parametrize("mode", ("instance", "batch"))
def test_norm_stats_float(gf, cuda_dev, mode):
    """Float X (mean 3, a channel at mean 1000): within one fp32 ulp of the fp64 statistics."""
    B, C = 3, 256
    n, _ = norm_n(sm_count(cuda_dev), B, empty_last=False)
    g = torch.Generator().manual_seed(5)
    X = (torch.randn(B, n, C, generator=g) * 2 + 3).float()
    X[:, :, 1] += 997.0
    sc, sh = run_norm(gf, cuda_dev, X.double(), mode)
    dims = (1,) if mode == "instance" else (0, 1)
    Xd = X.double()
    mu = Xd.mean(dim=dims, keepdim=True)
    rstd = 1.0 / torch.sqrt(((Xd - mu) ** 2).mean(dim=dims, keepdim=True) + 1e-8)
    want_sc, want_sh = rstd.expand(B, 1, C)[:, 0], (-mu * rstd).expand(B, 1, C)[:, 0]
    for name, gv, wv in (("NSCALE", sc, want_sc), ("NSHIFT", sh, want_sh)):
        ulp = torch.nextafter(wv.float().abs(), torch.tensor(math.inf)).double() - wv.float().abs().double()
        assert ((gv.double() - wv).abs() <= ulp).all(), name


@pytest.mark.parametrize("mode", ("instance", "batch"))
@pytest.mark.parametrize("integration", ("mul", "add", "both"))
def test_norm_affine_token_simt_exact(gf, cuda_dev, mode, integration):
    """The affine path of token_simt_kernel, x_n = fma(x, NSCALE, NSHIFT): X is m_c +- a_c with a_c = 2^14 or 2^15, balanced per image,
    so the statistics are powers of two (rstd = 1/a_c, the 1e-8 vanishes in fp64) and x_n = +-1; with K' = 0 and one-hot Rt every
    probability is 0 or 1, and Xout equals oracle/attn_fwd.stage_t_forward on the kernel's own NSCALE / NSHIFT bit for bit."""
    B, H, W, C, k = 2, 8, 16, 64, 13
    n, KP = H * W, 16
    g = torch.Generator().manual_seed(C + len(integration))
    m = torch.randint(-50, 51, (C,), generator=g).double()
    a = 2.0 ** torch.randint(14, 16, (C,), generator=g).double()
    sig = torch.cat([torch.ones(n // 2), -torch.ones(n // 2)]).double()
    sgn = torch.stack([torch.stack([sig[torch.randperm(n, generator=g)] for _ in range(C)], dim=1) for _ in range(B)])
    X = m + a * sgn
    Cout = 2 * C if integration == "both" else C
    Kp = torch.zeros(B, KP, C, dtype=torch.float64)
    Vt = torch.randint(-4, 5, (B, Cout, KP), generator=g).double()
    Vt[:, :, k:] = 0.0
    win = torch.randint(0, k, (B, H), generator=g)
    Rt = torch.full((B, H, KP), -2000.0, dtype=torch.float64)
    Rt[torch.arange(B)[:, None], torch.arange(H)[None], win] = 0.0
    Rt[:, :, k:] = -math.inf
    Ct = torch.zeros(B, W, KP, dtype=torch.float64)
    desc = gf._lib.make_desc(B, H, W, C, k, 16, norm=mode, integration=integration, pos_dim=0, flags=gf._lib.FLAG_FP32_EXACT)
    ws, lay = make_ws(gf, desc, cuda_dev)
    for name, t in (("Kp", Kp), ("Vt", Vt), ("Rt", Rt), ("Ct", Ct)):
        _region(ws, lay[name], t.shape).copy_(_f32(t, cuda_dev))
    outs = {"Xout": Guarded((B, n, C), cuda_dev), "att": Guarded((B, n, k), cuda_dev)}
    Xd = _f32(X, cuda_dev)
    gf._lib.check(_lib(gf).gf_attn_simplex_fwd_ex(ctypes.byref(desc), Xd.data_ptr(), outs["Xout"].ptr(), outs["att"].ptr(), ws.data_ptr(),
                                                  None, _stream(cuda_dev)), "gf_attn_simplex_fwd_ex")
    torch.cuda.synchronize()
    assert gf._lib.last_path() == "simt_fp32"
    nsc = _region(ws, lay["NSCALE"], (B, C)).double().cpu()
    nsh = _region(ws, lay["NSHIFT"], (B, C)).double().cpu()
    assert_exact(nsc, (1.0 / a).expand(B, C), "NSCALE")
    assert_exact(nsh, (-m / a).expand(B, C), "NSHIFT")
    want = af.stage_t_forward(X, Kp, Vt, Rt, Ct, H=H, W=W, k=k, integration=integration, norm=mode, nscale=nsc, nshift=nsh)
    assert_exact(outs["Xout"].check("Xout").double().cpu(), want["Xout"], "Xout")
    assert_exact(outs["att"].check("att").double().cpu(), want["att"], "att")
