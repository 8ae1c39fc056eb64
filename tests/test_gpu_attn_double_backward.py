"""GPU tests of the double-backward kernels at their C boundary (csrc/gf_bwd.cu; run on an H100: ``pytest -m gpu``).

* ``gf_attn_simplex_bwd_vjp`` (``token_bwd_vjp_kernel``): the VJP of the stage-T backward with its token reductions;
* ``gf_attn_centroid_bwd_vjp`` (``centroid_bwd_vjp_kernel``): the VJP of the pass-A backward with its reductions.

Both are called through ``_lib`` with synthetic fp32 tables and cotangents.  Every output sits between NaN guards; the tests
check the guards and that every element was written.  The reference is fp64 autograd differentiated twice through the folded
oracle (``tests/attn_double_backward_ref.py``: ``stage_t_vjp``, ``centroid_vjp``).  The per-token outputs are compared per
tensor, max |kernel - reference| / max |reference|; the reductions the caller forms from them (in fp64 here) relative to their
magnitude companion, the same reduction over absolute values, because a sum over the tokens can cancel far below its terms (the
lse cotangent at mean 30).  Cases: every integration, norm layer and none, x with mean 0 and 30 (the LayerNorm shift), 1 to 32 channel chunks, padded latents, ragged tiles, B = 300, and
the attention layers of the 256^2 discriminator (K = 16).  Then determinism, batch independence and CUDA-graph replay, bit for bit.
"""
import ctypes
import math

import pytest
import torch

from oracle import attn_bwd as ab
from tests import attn_double_backward_ref as vr
from oracle.folded import pad_k
from tests.guards import Guarded

pytestmark = pytest.mark.gpu

# Bound on max |kernel - fp64| / max |fp64| per output tensor, frozen at >= 1.5x the measured worst on an H100 80GB HBM3 (DESIGN.md
# section 5).
BOUND_T = 2e-5
BOUND_A = 2e-5
D_LATENT = 16

# B, H, W, C, k, integration, norm, mean
CASES_T = [
    (1, 1, 1, 32, 1, "mul", "none", 0.0),              # one token, one latent, one chunk
    (3, 8, 8, 32, 4, "add", "layer", 30.0),
    (1, 1, 128, 96, 16, "both", "layer", 0.0),         # one full tile, three chunks
    (3, 128, 1, 96, 17, "mul", "layer", 30.0),         # KP = 32 with 15 padded latents
    (3, 10, 13, 512, 31, "both", "none", 30.0),        # ragged n = 130, Cout = 1024
    (1, 10, 13, 1024, 32, "mul", "layer", 30.0),       # 32 chunks
    (1, 8, 8, 1024, 20, "both", "layer", 0.0),         # Cout = 2048
    (300, 5, 7, 32, 16, "mul", "layer", 30.0),         # B in the hundreds, n < 128
    (2, 10, 13, 96, 4, "add", "none", 0.0),
    # the attention layers of Discriminator(256, transformer=True) (K = 16): mul, layer norm
    (2, 256, 256, 64, 16, "mul", "layer", 0.0),
    (2, 128, 128, 128, 16, "mul", "layer", 0.0),
    (2, 64, 64, 256, 16, "mul", "layer", 0.0),
    (2, 32, 32, 512, 16, "mul", "layer", 0.0),
    (2, 16, 16, 512, 16, "mul", "layer", 0.0),
]
# B, H, W, C, k, mean
CASES_A = [
    (3, 46, 91, 96, 20, 0.0),
    (1, 46, 91, 512, 32, 30.0),
    (3, 10, 13, 32, 1, 30.0),
    (2, 64, 64, 512, 16, 0.0),
    (300, 5, 7, 32, 4, 0.0),
    (2, 256, 256, 64, 16, 0.0),
]


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t, dev):
    return t.float().contiguous().to(dev)


def stage_t_case(B, H, W, C, k, integration, mean, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g, dtype=torch.float64)
    KP, n = pad_k(k), H * W
    Cout = 2 * C if integration == "both" else C
    X, dOut = rn(B, n, C) + mean, rn(B, n, C)
    Kp = rn(B, KP, C) / math.sqrt(C)
    Kp = Kp - Kp.mean(dim=2, keepdim=True)                      # keys orthogonal to the mean: logits of order one
    Rt, Ct = rn(B, H, KP), rn(B, W, KP)
    Rt[:, :, k:] = -math.inf                                    # padded latents: nonzero keys, values, Ct and cotangents
    Vt = 0.3 * rn(B, Cout, KP)
    if integration != "add":
        Vt[:, :C] += 1.0
    cots = [rn(B, n, C), rn(B, KP, C) / math.sqrt(C), rn(B, Cout, KP), rn(B, H, KP), rn(B, W, KP)]
    return [X, dOut, Kp, Vt, Rt, Ct], cots


def run_stage_t(gf, dev, ins, cots, *, H, W, k, integration, norm, guards=True):
    X = _f32(ins[0], dev)
    B, n, C = X.shape
    KP, Cout = pad_k(k), ins[3].shape[1]
    tabs = [_f32(t, dev) for t in ins[1:]]
    cg = [_f32(t, dev) for t in cots]
    shapes = {"Xg": (B, n, C), "dOutg": (B, n, C), "Sg": (B, n, KP), "dPg": (B, n, KP), "Ctlg": (B, n, Cout), "dS": (B, n, KP),
              "P": (B, n, KP), "dCtl": (B, n, Cout)}
    outs = {nm: Guarded(s, dev) for nm, s in shapes.items()}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm=norm, integration=integration, pos_dim=0, duplex=False)
    gf._lib.check(gf._lib.load().gf_attn_simplex_bwd_vjp(ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs + cg),
                                                         *(o.ptr() for o in outs.values()), _stream(dev)), "gf_attn_simplex_bwd_vjp")
    torch.cuda.synchronize(dev)
    return {nm: (o.check(nm) if guards else o.t).clone() for nm, o in outs.items()}


def reduce_stage_t(o, ins, cots, H, W):
    """The caller's reductions, in fp64: Kp: Sg^T X + dS^T U, Vt: Ctlg^T P + dCtl^T dPg, Rt / Ct: sums of Sg."""
    d = {nm: t.double().cpu() for nm, t in o.items()}
    X, U = ins[0], cots[0]
    B, n, KP = d["Sg"].shape
    Sg4 = d["Sg"].reshape(B, H, W, KP)
    return {"Kp": d["Sg"].transpose(1, 2) @ X + d["dS"].transpose(1, 2) @ U,
            "Vt": d["Ctlg"].transpose(1, 2) @ d["P"] + d["dCtl"].transpose(1, 2) @ d["dPg"],
            "Rt": Sg4.sum(dim=2), "Ct": Sg4.sum(dim=1)}


def _err(got, want, scale=None):
    """max |got - want| / max scale, scale = |want| by default (per-token outputs) or the magnitude companion of a reduction."""
    scale = want.abs() if scale is None else scale
    return ((got.double().cpu() - want).abs().max() / scale.max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("case", CASES_T, ids=lambda c: "x".join(map(str, c[:5])) + f"-{c[5]}-{c[6]}-m{int(c[7])}")
def test_stage_t_vjp_against_fp64(gf, cuda_dev, case):
    B, H, W, C, k, integration, norm, mean = case
    ins, cots = stage_t_case(B, H, W, C, k, integration, mean, seed=B * 7 + C + k)
    got = run_stage_t(gf, cuda_dev, ins, cots, H=H, W=W, k=k, integration=integration, norm=norm)
    ref = vr.stage_t_vjp(*ins, *cots, H=H, W=W, integration=integration, norm=norm)
    first = ab.stage_t_backward(ins[0], *ins[1:], H=H, W=W, integration=integration, norm=norm)
    red = reduce_stage_t(got, ins, cots, H, W)
    comp = reduce_stage_t({nm: t.abs() for nm, t in got.items()}, [t.abs() for t in ins], [t.abs() for t in cots], H, W)
    errs = {nm: _err(got[nm], ref[nm]) for nm in ("Xg", "dOutg", "Sg")}
    errs.update({nm: _err(red[nm], ref[nm], comp[nm]) for nm in ("Kp", "Vt", "Rt", "Ct")})
    errs.update({nm: _err(got[nm], first[nm]) for nm in ("dS", "P", "dCtl")})
    want_ctlg = ref["Ctlg"]
    if integration == "add":                                      # ctl does not enter the first-order backward
        assert torch.count_nonzero(got["Ctlg"]) == 0
    else:
        errs["Ctlg"] = _err(got["Ctlg"], want_ctlg)
        if integration == "both":
            assert torch.count_nonzero(got["Ctlg"][..., C:]) == 0
    assert torch.count_nonzero(got["Sg"][..., k:]) == 0 and torch.count_nonzero(got["dPg"][..., k:]) == 0
    worst = max(errs, key=errs.get)
    print(f"[vjp stage T] {case}: worst {worst} {errs[worst]:.2e}  " + " ".join(f"{a}={b:.1e}" for a, b in errs.items()))
    assert errs[worst] <= BOUND_T, worst


def centroid_case(B, H, W, C, k, mean, seed):
    c = ab.random_centroid_case(B, H, W, C, k, mean=mean, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    rn = lambda *s: torch.randn(s, generator=g, dtype=torch.float64)
    KP, n = pad_k(k), H * W
    lse = ab.centroid_stats(c["X"], c["M"], c["Rt2"], c["Ct2"], k=k)["lse"]
    ins = [c["X"], c["M"], c["Rt2"], c["Ct2"], lse, c["dXbar"], c["r"] + 0.1 * rn(B, k), c["dX0"]]
    cots = [rn(B, n, C), rn(B, KP, C) / math.sqrt(C), rn(B, H, KP), rn(B, W, KP)]
    return ins, cots


def run_centroid(gf, dev, ins, cots, *, H, W, k):
    X = _f32(ins[0], dev)
    B, n, C = X.shape
    KP = pad_k(k)
    tabs = [_f32(t, dev) for t in ins[1:7]]
    cg = [_f32(t, dev) for t in cots]
    outs = {"Xg": Guarded((B, n, C), dev), **{nm: Guarded((B, n, KP), dev) for nm in ("Sg", "Gg", "A", "dS")}}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    gf._lib.check(gf._lib.load().gf_attn_centroid_bwd_vjp(ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs + cg),
                                                          *(o.ptr() for o in outs.values()), _stream(dev)), "gf_attn_centroid_bwd_vjp")
    torch.cuda.synchronize(dev)
    return {nm: o.check(nm).clone() for nm, o in outs.items()}


def reduce_centroid(o, X, U, H, W, k):
    """The caller's reductions, in fp64: M: Sg^T X + dS^T U, Rt2 / Ct2: sums of Sg, lse: -sum_t Sg, dXbar: A^T U + Gg^T X,
    r: -sum_t Gg (0 in the padded latents of Rt2 and lse)."""
    d = {nm: t.double().cpu() for nm, t in o.items()}
    B, n, KP = d["Sg"].shape
    Sg4 = d["Sg"].reshape(B, H, W, KP)
    red = {"M": d["Sg"].transpose(1, 2) @ X + d["dS"].transpose(1, 2) @ U, "Rt2": Sg4.sum(dim=2), "Ct2": Sg4.sum(dim=1),
           "lse": -d["Sg"].sum(dim=1), "dXbar": (d["A"].transpose(1, 2) @ U + d["Gg"].transpose(1, 2) @ X)[:, :k],
           "r": -d["Gg"].sum(dim=1)[:, :k]}
    red["Rt2"][..., k:] = 0.0
    red["lse"][..., k:] = 0.0
    return red


@pytest.mark.parametrize("case", CASES_A, ids=lambda c: "x".join(map(str, c[:5])) + f"-m{int(c[5])}")
def test_centroid_vjp_against_fp64(gf, cuda_dev, case):
    B, H, W, C, k, mean = case
    ins, cots = centroid_case(B, H, W, C, k, mean, seed=B + C + k)
    got = run_centroid(gf, cuda_dev, ins, cots, H=H, W=W, k=k)
    ref = vr.centroid_vjp(*ins, *cots, H=H, W=W, k=k)
    red = reduce_centroid(got, ins[0], cots[0], H, W, k)
    comp = reduce_centroid({nm: t.abs() for nm, t in got.items()}, ins[0].abs(), cots[0].abs(), H, W, k)
    errs = {nm: _err(got[nm], ref[nm]) for nm in ("Xg", "Sg", "Gg", "A", "dS")}
    errs.update({nm: _err(red[nm], ref[nm], comp[nm].abs()) for nm in red})
    for nm in ("Sg", "Gg", "A", "dS"):
        assert torch.count_nonzero(got[nm][..., k:]) == 0, nm
    worst = max(errs, key=errs.get)
    print(f"[vjp pass A] {case}: worst {worst} {errs[worst]:.2e}  " + " ".join(f"{a}={b:.1e}" for a, b in errs.items()))
    assert errs[worst] <= BOUND_A, worst


def test_vjp_deterministic_batch_independent_and_graph_replay(gf, cuda_dev):
    """Both kernels: two calls give the same bits, image 0 of a batch of 3 equals a batch of 1, and a CUDA-graph replay equals
    the eager call."""
    H, W, C, k = 10, 13, 96, 20
    ins, cots = stage_t_case(3, H, W, C, k, "both", 30.0, seed=1)
    a = run_stage_t(gf, cuda_dev, ins, cots, H=H, W=W, k=k, integration="both", norm="layer")
    b = run_stage_t(gf, cuda_dev, ins, cots, H=H, W=W, k=k, integration="both", norm="layer")
    one = run_stage_t(gf, cuda_dev, [t[:1] for t in ins], [t[:1] for t in cots], H=H, W=W, k=k, integration="both", norm="layer")
    for nm in a:
        assert torch.equal(a[nm], b[nm]), nm
        assert torch.equal(a[nm][:1], one[nm]), nm
    cins, ccots = centroid_case(3, 46, 91, 96, 20, 0.0, seed=2)
    ca = run_centroid(gf, cuda_dev, cins, ccots, H=46, W=91, k=20)
    cb = run_centroid(gf, cuda_dev, cins, ccots, H=46, W=91, k=20)
    cone = run_centroid(gf, cuda_dev, [t[:1] for t in cins], [t[:1] for t in ccots], H=46, W=91, k=20)
    for nm in ca:
        assert torch.equal(ca[nm], cb[nm]), nm
        assert torch.equal(ca[nm][:1], cone[nm]), nm

    # graph replay of both entries, on device buffers owned by the test
    dev = cuda_dev
    X = _f32(ins[0], dev)
    B, n, _ = X.shape
    KP, Cout = pad_k(k), ins[3].shape[1]
    tabs = [_f32(t, dev) for t in ins[1:] + cots]
    o = {nm: torch.empty(s, device=dev) for nm, s in (("Xg", (B, n, C)), ("dOutg", (B, n, C)), ("Sg", (B, n, KP)), ("dPg", (B, n, KP)),
                                                      ("Ctlg", (B, n, Cout)), ("dS", (B, n, KP)), ("P", (B, n, KP)), ("dCtl", (B, n, Cout)))}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="both", pos_dim=0, duplex=False)
    cX = _f32(cins[0], dev)
    ctabs = [_f32(t, dev) for t in cins[1:7] + ccots]
    co = {nm: torch.empty(ca[nm].shape, device=dev) for nm in ca}
    cdesc = gf._lib.make_desc(3, 46, 91, 96, 20, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    lib = gf._lib.load()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            st = _stream(dev)
            gf._lib.check(lib.gf_attn_simplex_bwd_vjp(ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs),
                                                      *(t.data_ptr() for t in o.values()), st), "capture")
            gf._lib.check(lib.gf_attn_centroid_bwd_vjp(ctypes.byref(cdesc), cX.data_ptr(), *(t.data_ptr() for t in ctabs),
                                                       *(t.data_ptr() for t in co.values()), st), "capture")
    torch.cuda.current_stream(dev).wait_stream(side)
    for t in list(o.values()) + list(co.values()):
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize(dev)
    for nm in o:
        assert torch.equal(o[nm], a[nm]), nm
    for nm in co:
        assert torch.equal(co[nm], ca[nm]), nm


def test_entries_refuse_unsupported_descriptors(gf, cuda_dev):
    lib = gf._lib.load()
    desc = gf._lib.make_desc(1, 4, 4, 32, 4, D_LATENT, heads=1, norm="instance", integration="mul", pos_dim=0, duplex=False)
    t = torch.zeros(4096, device=cuda_dev)
    rc = lib.gf_attn_simplex_bwd_vjp(ctypes.byref(desc), *([t.data_ptr()] * 19), _stream(cuda_dev))
    assert rc != 0 and b"norm must be layer or none" in lib.gf_last_error()
    desc = gf._lib.make_desc(1, 4, 4, 32, 4, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=2)
    rc = lib.gf_attn_centroid_bwd_vjp(ctypes.byref(desc), *([t.data_ptr()] * 16), _stream(cuda_dev))
    assert rc != 0 and b"one k-means iteration" in lib.gf_last_error()
