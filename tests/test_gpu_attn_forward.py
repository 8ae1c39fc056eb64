"""GPU tests of the attention forward kernels at their C boundary (run on an H100: ``pytest -m gpu``).

* Stage T, ``gf_attn_simplex_fwd_ex`` without a prologue: the test fills the whole workspace with a NaN pattern and writes K',
  V^T, Rt, Ct (and CB with dropout) at the offsets ``gf_attn_debug_layout`` reports, so any read outside those tables shows up
  as NaN.  Xout, att and rgb_out sit between NaN guards (``tests/guards.py``).
  - Exact cases (the one-hot construction of ``oracle/attn_bwd.py``: every probability 0, 1/2 or 1, every logit an integer below
    2^24) run on both kernel families, ``token_tc_kernel`` (default flags) and ``token_simt_kernel`` (``GF_FLAG_FP32_EXACT``),
    and must equal ``oracle/attn_fwd.stage_t_forward`` in fp64 bit for bit: every <KP, NS, MODE> instantiation, short tiles
    (one warpgroup, a partial second box), whole tiles, the persistent schedule, the ring at its minimum depth, dropout at
    p = 1/2, multi-head segments and the exact fused epilogue with tRGB.  ``tests/test_host_cpu_attn_forward.py`` checks on the
    host that each of these cases really is exact.
  - TF32 emulation cases run realistic weights through stages W and I and check the two GEMMs separately: (a) the attention map
    against softmax_2(tf32_trunc(x) K'^T + Rt + Ct), (b) Xout (and rgb_out) against the store side rebuilt from the kernel's own
    map, P = tf32_rna(f32(att * mask)).
  - Stage I: the tables ``gf_attn_prologue_ex`` writes are on the TF32 grid, within one TF32 ulp of rne(kf K'64 d), with the
    truncation compensation as their slope; the batched prologue writes the same bits.
* Duplex pass A, ``centroid_tc_kernel`` through ``gf_attn_duplex_fwd_ex`` with ``GF_FLAG_TABLES_READY``: M, Rt2 and Ct2 written
  in log2 units, Xbar read back from the workspace.  Exact cases (one winner per latent, runners-up that force the online
  rescale, ties, the C = 512 channel split, padded latents, an empty last split) and an emulation case.
* Determinism, batch independence and CUDA-graph replay, bit for bit.
"""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import attn_fwd as af
from oracle import bipartite as ob
from oracle import folded as of
from oracle.bipartite import LN_EPS
from oracle.tf32 import tf32_low_bits, tf32_rna, tf32_rne, tf32_trunc
from tests.guards import GUARD_BITS, Guarded, assert_exact

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D_LATENT = 16
POS = 8                                          # pos_dim of the folded buffers (stage-T tables are written directly)
GF_ERR_UNSUPPORTED = -2
GAIN = float(torch.tensor(math.sqrt(2.0), dtype=torch.float32))    # the post-op gain is a float argument
# Per-element bounds of |kernel - emulation| / companion.  Measured worst cases over the emulation cases below on an H100 80GB
# HBM3 at a 400 W power limit (att 4.1e-7, Xout 1.2e-6, rgb 5.7e-8, Xbar 3.2e-6), frozen at 1.5x or more (DESIGN.md section 5).
BOUND = {"att": 1e-6, "Xout": 2e-6, "rgb": 1e-7, "Xbar": 5e-6}

FAMILIES = ("tc", "simt")
# <KP, NS, MODE>: k = 13 (KP 16) and 27 (KP 32), C = 64 .. 512 (NS = 2 .. 16; 16 is the two-pass kernel), three integrations
INSTANCES = [(kk, C, integ) for kk in (13, 27) for C in (64, 128, 256, 512) for integ in ("mul", "add", "both")]
# on an H100 (227 KB of shared memory per block) K' and V^T of these leave too few ring stages: gf_attn_tc_eligible says 0 and the
# CUDA-core kernel serves them under the default flags
TC_FALLBACK = {(27, 256, "both"), (27, 512, "both")}
# short tiles (n < 128: one warpgroup up to 64 tokens, a partial second box above), a whole tile, several tiles per image
TILES = [(1, 8), (4, 8), (8, 8), (8, 9), (8, 12), (8, 15), (8, 16), (16, 32)]
# (integration, C, k, act, rgb, per-image noise, scales)
EPILOGUES = [("mul", 64, 13, 1, True, False, True), ("both", 256, 13, 1, True, True, True), ("add", 128, 5, 0, False, True, True),
             ("mul", 512, 16, 1, True, True, False), ("both", 512, 16, 0, False, False, True), ("add", 256, 27, 1, True, True, True)]


def _lib(gf):
    return gf._lib.load()


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t, dev):
    return t.float().contiguous().to(dev)


def layout(gf, desc):
    out = (ctypes.c_longlong * 15)()
    gf._lib.check(_lib(gf).gf_attn_debug_layout(ctypes.byref(desc), out, 15), "gf_attn_debug_layout")
    names = ("PART", "XBAR", "nsplit", "KP", "M", "Rt2", "Ct2", "total", "Kp", "Vt", "Rt", "Ct", "CB", "NSCALE", "NSHIFT")
    return dict(zip(names, (int(v) for v in out)))


def _region(ws, off, shape):
    return ws[off:off + math.prod(shape)].view(shape)


class Postop:
    """A gf_attn_postop with its device tensors kept alive; `post` is the host dict of oracle/attn_fwd.stage_t_forward."""

    def __init__(self, gf, post, dev, B, n, C, dp=None, rgb_out=None):
        self.s = gf._lib.GfAttnPostop()
        self.keep = []
        s = self.s

        def put(t):
            t = _f32(t, dev)
            self.keep.append(t)
            return t.data_ptr()
        post = post or {}
        if post.get("bias") is not None:
            s.bias = put(post["bias"])
        if post.get("noise") is not None:
            s.noise = put(post["noise"].reshape(-1))
            s.noise_bstride = n if post["noise"].shape[0] > 1 else 0
        if "strength" in post:
            s.strength = put(torch.tensor([post["strength"]]))
        s.act = post.get("act", 0)
        s.gain = post.get("gain", 1.0)
        if post.get("in_scale") is not None:               # rows with a padded leading dimension
            t = torch.zeros(B, C + 4, dtype=torch.float64)
            t[:, :C] = post["in_scale"]
            s.in_scale, s.in_scale_ld = put(t), C + 4
        if post.get("post_scale") is not None:
            t = torch.zeros(B, C + 8, dtype=torch.float64)
            t[:, :C] = post["post_scale"]
            s.post_scale, s.post_scale_ld = put(t), C + 8
        if post.get("rgb_w") is not None:
            s.rgb_w = put(post["rgb_w"])
            s.rgb_bias = put(post["rgb_bias"])
            s.rgb_out = rgb_out
        if dp is not None:
            att_dp, salt, seed, step = dp
            state = torch.tensor([seed, step], dtype=torch.int64, device=dev)
            self.keep.append(state)
            s.att_dp, s.dp_salt, s.dp_state = att_dp, salt, state.data_ptr()


def make_ws(gf, desc, dev, fill="nan"):
    lay = layout(gf, desc)
    if fill == "nan":
        ws = torch.full((lay["total"],), GUARD_BITS, dtype=torch.int32, device=dev).view(torch.float32)
    else:
        ws = torch.zeros(lay["total"], dtype=torch.float32, device=dev)
    return ws, lay


def stage_t(gf, dev, case, *, H, W, k, integration, family, norm="none", post=None, expect_rc=0, tc_expected=True):
    """gf_attn_simplex_fwd_ex on the case's tables, written into a NaN-filled workspace; returns the checked outputs as fp64 on
    the CPU (or the status, when expect_rc is an error).  family "tc" runs the default flags, which must reach the tensor kernel
    unless tc_expected is False (then gf_attn_tc_eligible must say 0 and the CUDA-core kernel must serve the call)."""
    X = _f32(case["X"], dev)
    B, n, C = X.shape
    heads = case.get("heads", 1)
    flags = gf._lib.FLAG_FP32_EXACT if family == "simt" else 0
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=heads, norm=norm, integration=integration, pos_dim=0, duplex=False,
                             flags=flags)
    lib = _lib(gf)
    tc = family == "tc" and tc_expected
    if family == "tc":
        assert lib.gf_attn_tc_eligible(ctypes.byref(desc)) == int(tc_expected)
    ws, lay = make_ws(gf, desc, dev)
    KP = lay["KP"]
    assert KP == case["Kp"].shape[1]
    Kt = case["Kp"].double()
    if post and post.get("in_scale") is not None:
        Kt = Kt * post["in_scale"].double()[:, None, :]               # what stage I folds into K'
    for name, t in (("Kp", Kt), ("Vt", case["Vt"]), ("Rt", case["Rt"]), ("Ct", case["Ct"])):
        _region(ws, lay[name], t.shape).copy_(_f32(t, dev))
    dp = None
    if case.get("att_dp"):
        _region(ws, lay["CB"], case["cb"].shape).copy_(_f32(case["cb"], dev))
        dp = (case["att_dp"], case["salt"], case["dp_seed"], case["step"])
    outs = {"Xout": Guarded((B, n, C), dev), "att": Guarded((B, n, k), dev)}
    if post and post.get("rgb_w") is not None:
        outs["rgb"] = Guarded((B, 3, n), dev)
    po = Postop(gf, post, dev, B, n, C, dp=dp, rgb_out=outs["rgb"].ptr() if "rgb" in outs else None) if (post or dp) else None
    rc = lib.gf_attn_simplex_fwd_ex(ctypes.byref(desc), X.data_ptr(), outs["Xout"].ptr(), outs["att"].ptr(), ws.data_ptr(),
                                    ctypes.byref(po.s) if po else None, _stream(dev))
    if expect_rc:
        assert rc == expect_rc, (rc, lib.gf_last_error())
        return rc
    gf._lib.check(rc, "gf_attn_simplex_fwd_ex")
    torch.cuda.synchronize()
    assert gf._lib.last_path() == ("wgmma_tf32" if tc else "simt_fp32")
    return {name: g.check(name).double().cpu() for name, g in outs.items()}


def reference(case, *, H, W, k, integration, norm="none", post=None):
    Kt = case["Kp"].double()
    if post and post.get("in_scale") is not None:
        Kt = Kt * post["in_scale"].double()[:, None, :]
    return af.stage_t_forward(case["X"], Kt, case["Vt"], case["Rt"], case["Ct"], H=H, W=W, k=k, integration=integration, norm=norm,
                              heads=case.get("heads", 1), mult=case["mult"], cb=case["cb"] if case["mult"] is not None else None,
                              post=post)


def check_exact(got, want):
    for name in got:
        assert_exact(got[name], want[name], name)


def _id(v):
    return str(v)


def sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


# ---- stage T, exact --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES + ("tc_min_ring",))
@pytest.mark.parametrize("k,C,integration", INSTANCES, ids=_id)
def test_stage_t_exact_every_instantiation(gf, cuda_dev, monkeypatch, family, k, C, integration):
    """Every tensor instantiation <KP, NS, MODE> (and the CUDA-core kernel on the same tables) on 3 images of two tiles each:
    Xout and att equal the fp64 reference bit for bit.  tc_min_ring runs the tensor kernel with the ring at its minimum depth
    (NS slabs single-pass, 4 two-pass), so every tile wraps the ring.  The shapes of TC_FALLBACK are not tensor-eligible: the
    test asserts that, and that the default flags then run the CUDA-core kernel."""
    if family == "tc_min_ring":
        monkeypatch.setenv("GF_TC_MAX_STAGES", str(4 if C == 512 else C // 32))
    H, W = 8, 32
    case = af.exact_stage_t_case(3, H, W, C, k, integration, seed=C + k)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, family="tc" if family.startswith("tc") else "simt",
                  tc_expected=(k, C, integration) not in TC_FALLBACK)
    want = reference(case, H=H, W=W, k=k, integration=integration)
    assert (want["att"] == 1.0).any() and (want["att"] == 0.5).any()
    check_exact(got, want)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("H,W", TILES, ids=_id)
def test_stage_t_exact_tiles(gf, cuda_dev, family, H, W):
    """n = 8 .. 120 (one tile per image: one warpgroup up to 64 rows, then a partial second box of n - 64 rows), a whole tile and
    four tiles per image, with KP 16 and 32."""
    for k, C, integration in ((16, 128, "mul"), (27, 64, "both")):
        case = af.exact_stage_t_case(5, H, W, C, k, integration, seed=H * W + k)
        got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, family=family)
        check_exact(got, reference(case, H=H, W=W, k=k, integration=integration))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("H,W", [(8, 9), (8, 16), (16, 16)], ids=_id)
def test_stage_t_exact_persistent_schedule(gf, cuda_dev, family, H, W):
    """More tiles than SMs, and not a multiple of the SM count: the batch is derived from the device, so each persistent CTA walks
    a contiguous range of tiles that crosses images."""
    sms = sm_count(cuda_dev)
    n = H * W
    tpi = max(1, n // 128)
    B = (2 * sms + 7) // tpi + 1
    tiles = B * tpi
    assert tiles > sms and tiles % sms != 0
    case = af.exact_stage_t_case(B, H, W, 64, 13, "mul", seed=B)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=13, integration="mul", family=family)
    check_exact(got, reference(case, H=H, W=W, k=13, integration="mul"))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("H,W,C,k,integration", [(8, 16, 128, 16, "mul"), (8, 9, 64, 7, "add"), (4, 32, 512, 27, "add"),
                                                 (8, 32, 256, 31, "mul")], ids=_id)
def test_stage_t_exact_dropout(gf, cuda_dev, family, H, W, C, k, integration):
    """Attention dropout at p = 1/2: multipliers 0 or 2, so q * cb is exact.  The mask gf_attn_dropout_mask writes equals the
    host Philox draw the reference uses; the attention map stays the probabilities before dropout."""
    B = 3
    case = af.exact_stage_t_case(B, H, W, C, k, integration, dropout=True, seed=C + k + 1)
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, norm="none", integration=integration)
    mask = torch.empty(B, H * W, case["KP"], device=cuda_dev)
    state = torch.tensor([case["dp_seed"], case["step"]], dtype=torch.int64, device=cuda_dev)
    gf._lib.check(_lib(gf).gf_attn_dropout_mask(ctypes.byref(desc), ctypes.c_float(0.5), case["salt"], state.data_ptr(),
                                                mask.data_ptr(), _stream(cuda_dev)), "gf_attn_dropout_mask")
    torch.cuda.synchronize()
    assert torch.equal(mask.double().cpu(), case["mult"])
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, family=family)
    want = reference(case, H=H, W=W, k=k, integration=integration)
    nodrop = reference({**case, "mult": None}, H=H, W=W, k=k, integration=integration)
    assert not torch.equal(want["Xout"], nodrop["Xout"])
    check_exact(got, want)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("heads,k,C", [(2, 5, 128), (2, 12, 256), (4, 7, 64), (4, 8, 512)], ids=_id)
def test_stage_t_exact_multi_head(gf, cuda_dev, family, heads, k, C):
    """Multi-head layers: one softmax per segment of 8 or 16 table columns, with a different winner per head; the map is the mean
    over the heads (exact for 2 and 4)."""
    H, W = 8, 16
    case = af.exact_stage_t_case(3, H, W, C, k, "mul", heads=heads, seed=heads * 100 + k)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration="mul", family=family)
    want = reference(case, H=H, W=W, k=k, integration="mul")
    assert ((want["att"] > 0) & (want["att"] < 0.5)).any()         # heads disagree somewhere
    check_exact(got, want)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("integration,C,k,act,rgb,per_image,scales", EPILOGUES, ids=_id)
def test_stage_t_exact_epilogue(gf, cuda_dev, family, integration, C, k, act, rgb, per_image, scales):
    """The fused epilogue on an exact case: noise (shared or per image) times a device strength, bias, leaky-ReLU with gain 5 or
    linear, in_scale (folded into K' here as stage I does) and post_scale, and the fused tRGB, which reads the output before
    post_scale (integer rgb_w, post_scale != 1).  The CUDA-core kernel runs the same epilogue without tRGB, and linear (its
    leaky-ReLU multiplies by 0.2f, which is not exact)."""
    B, H, W = 3, 8, 16
    case = af.exact_stage_t_case(B, H, W, C, k, integration, dropout=(C == 256), seed=C + k + act)
    # the CUDA-core kernel forms leaky-ReLU as max(y, 0.2f y): 0.2f is not exact, so it runs the linear activation here
    post = af.exact_postop(B, H * W, C, seed=C + k, act=act if family == "tc" else 0, rgb=rgb and family == "tc",
                           per_image_noise=per_image, scales=scales)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, family=family, post=post)
    want = reference(case, H=H, W=W, k=k, integration=integration, post=post)
    check_exact(got, want)


def test_trgb_unsupported_shapes(gf, cuda_dev):
    """The fused tRGB is refused (GF_ERR_UNSUPPORTED) for C = 512 with KP = 32 and on the CUDA-core path."""
    B, H, W = 2, 8, 16
    for C, k, family in ((512, 27, "tc"), (64, 13, "simt"), (512, 13, "simt")):
        case = af.exact_stage_t_case(B, H, W, C, k, "mul", seed=1)
        post = af.exact_postop(B, H * W, C, seed=2, act=1, rgb=True, per_image_noise=False, scales=False)
        assert stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration="mul", family=family, post=post,
                       expect_rc=GF_ERR_UNSUPPORTED) == GF_ERR_UNSUPPORTED


# ---- stage T, TF32 emulation -----------------------------------------------------------------------------------------------------
def _weights_struct(gf, w, dev):
    ws, keep = gf._lib.GfAttnWeights(), []
    for name in gf._lib.WEIGHT_FIELDS:
        if name in w:
            t = _f32(w[name], dev)
            keep.append(t)
            setattr(ws, name, t.data_ptr())
    return ws, keep


def real_tables(gf, dev, *, B, H, W, C, k, integration, norm, seed, in_scale=None, batch=False):
    """Stages W and I on random weights (gf_attn_fold_weights, then gf_attn_prologue_ex or gf_attn_prologue_batch); returns the
    workspace, its layout, the desc, the fp64 weights and latents."""
    w = ob.init_params(C, D_LATENT, k, POS, integration, False, seed=seed, bias_std=0.2)
    y = torch.randn(B, k, D_LATENT, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, norm=norm, integration=integration, pos_dim=POS)
    lib = _lib(gf)
    folded = torch.empty(gf._lib.folded_floats(desc), device=dev)
    wst, keep = _weights_struct(gf, w, dev)
    gf._lib.check(lib.gf_attn_fold_weights(ctypes.byref(desc), ctypes.byref(wst), folded.data_ptr(), _stream(dev)), "fold")
    ws, lay = make_ws(gf, desc, dev)
    Y = _f32(y, dev)
    post = Postop(gf, {"in_scale": in_scale} if in_scale is not None else None, dev, B, H * W, C)
    if batch:
        descs = (ctypes.POINTER(gf._lib.GfAttnDesc) * 1)(ctypes.pointer(desc))
        ptr = lambda v: (ctypes.c_void_p * 1)(v)
        posts = (ctypes.POINTER(gf._lib.GfAttnPostop) * 1)(ctypes.pointer(post.s))
        gf._lib.check(lib.gf_attn_prologue_batch(1, descs, ptr(Y.data_ptr()), ptr(folded.data_ptr()), ptr(ws.data_ptr()), posts,
                                                 _stream(dev)), "gf_attn_prologue_batch")
    else:
        gf._lib.check(lib.gf_attn_prologue_ex(ctypes.byref(desc), Y.data_ptr(), folded.data_ptr(), ws.data_ptr(), ctypes.byref(post.s),
                                              _stream(dev)), "gf_attn_prologue_ex")
    torch.cuda.synchronize()
    return ws, lay, desc, w, y


def read_tables(ws, lay, B, H, W, C, KP, Cout):
    return {name: _region(ws, lay[name], shape).double().cpu() for name, shape in
            (("Kp", (B, KP, C)), ("Vt", (B, Cout, KP)), ("Rt", (B, H, KP)), ("Ct", (B, W, KP)), ("CB", (Cout,)))}


# B, H, W, C, k, integration, norm, att_dp, mean, post-op (in_scale, noise, bias, lrelu, post_scale, tRGB where served)
EMUL = [
    (2, 16, 16, 256, 16, "mul", "layer", 0.0, 0.0, False),
    (2, 16, 16, 256, 16, "mul", "layer", 0.12, 30.0, True),
    (2, 8, 16, 128, 20, "both", "none", 0.5, 0.0, True),
    (3, 8, 8, 64, 8, "add", "layer", 0.12, 30.0, False),
    (1, 16, 32, 512, 32, "add", "layer", 0.0, 30.0, True),
    (2, 8, 9, 128, 16, "mul", "none", 0.5, 30.0, True),
    # the six attention layers of the 256^2 K = 16 training generator: mul, layer norm, att_dp = 0.12
    (2, 8, 8, 512, 16, "mul", "layer", 0.12, 0.0, False),
    (2, 16, 16, 512, 16, "mul", "layer", 0.12, 0.0, False),
    (2, 32, 32, 512, 16, "mul", "layer", 0.12, 0.0, False),
    (2, 64, 64, 512, 16, "mul", "layer", 0.12, 0.0, False),
    (2, 128, 128, 256, 16, "mul", "layer", 0.12, 0.0, False),
    (1, 256, 256, 128, 16, "mul", "layer", 0.12, 0.0, False),
    # the five C / resolution pairs of the benchmarked synthesis (inference: no dropout, the fused post-op)
    (2, 16, 16, 512, 16, "mul", "layer", 0.0, 0.0, True),
    (2, 32, 32, 512, 16, "mul", "layer", 0.0, 0.0, True),
    (2, 64, 64, 512, 16, "mul", "layer", 0.0, 0.0, True),
    (2, 128, 128, 256, 16, "mul", "layer", 0.0, 0.0, True),
    (1, 256, 256, 128, 16, "mul", "layer", 0.0, 0.0, True),
]


def _ln64(x):
    mu = x.mean(dim=2, keepdim=True)
    return (x - mu) / torch.sqrt(((x - mu) ** 2).mean(dim=2, keepdim=True) + LN_EPS)


def _worst(got, want, comp, name):
    err = (got - want).abs()
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    assert (err[comp == 0] == 0).all(), f"{name}: nonzero error where the companion is 0"
    c = comp > 0
    return (err[c] / comp[c]).max().item() if c.any() else 0.0


@pytest.mark.parametrize("B,H,W,C,k,integration,norm,att_dp,mean,with_post", EMUL, ids=_id)
def test_stage_t_tf32_emulation(gf, cuda_dev, B, H, W, C, k, integration, norm, att_dp, mean, with_post):
    """token_tc_kernel on the tables of stages W and I (realistic weights), GEMM by GEMM:
    (a) att against softmax_2(tf32_trunc(x) K'^T + f32(Rt + Ct)) in fp64, per element relative to (1 + the row's largest |logit|
        companion) p;
    (b) Xout against LN64(x d) (P V^T + qdef cb) plus the post-op, with P = tf32_rna(f32(att * mask)) rebuilt from the kernel's
        own map, per element relative to the same expression on absolute values (LayerNorm companion with the shift term); rgb_out
        the same way."""
    dev = cuda_dev
    g = torch.Generator().manual_seed(B * 7 + H + C + k)
    n, KP = H * W, of.pad_k(k)
    Cout = 2 * C if integration == "both" else C
    post = None
    if with_post:
        post = dict(in_scale=(0.5 + torch.rand(B, C, generator=g, dtype=torch.float64)).float().double(),
                    bias=0.3 * torch.randn(C, generator=g, dtype=torch.float64), noise=torch.randn(B, n, generator=g, dtype=torch.float64),
                    strength=0.25, act=1, gain=GAIN, post_scale=(0.5 + torch.rand(B, C, generator=g, dtype=torch.float64)))
        if C <= 256 or KP == 16:
            post.update(rgb_w=torch.randn(B, 3, C, generator=g, dtype=torch.float64) / math.sqrt(C),
                        rgb_bias=torch.randn(3, generator=g, dtype=torch.float64))
        post = {a: (v.float().double() if torch.is_tensor(v) else v) for a, v in post.items()}
    ws, lay, desc, _, _ = real_tables(gf, dev, B=B, H=H, W=W, C=C, k=k, integration=integration, norm=norm, seed=C + k,
                                      in_scale=None if post is None else post["in_scale"])
    tabs = read_tables(ws, lay, B, H, W, C, KP, Cout)
    X = (torch.randn(B, n, C, generator=g) + mean).float()
    Xd = X.to(dev)
    outs = {"Xout": Guarded((B, n, C), dev), "att": Guarded((B, n, k), dev)}
    if post and "rgb_w" in post:
        outs["rgb"] = Guarded((B, 3, n), dev)
    dp = (att_dp, 5, 1234, 2) if att_dp else None
    po = Postop(gf, post, dev, B, n, C, dp=dp, rgb_out=outs["rgb"].ptr() if "rgb" in outs else None) if (post or dp) else None
    lib = _lib(gf)
    assert lib.gf_attn_tc_eligible(ctypes.byref(desc)) == 1
    gf._lib.check(lib.gf_attn_simplex_fwd_ex(ctypes.byref(desc), Xd.data_ptr(), outs["Xout"].ptr(), outs["att"].ptr(), ws.data_ptr(),
                                             ctypes.byref(po.s) if po else None, _stream(dev)), "gf_attn_simplex_fwd_ex")
    mask = torch.ones(B, n, KP)
    if dp:
        md = torch.empty(B, n, KP, device=dev)
        state = torch.tensor([dp[2], dp[3]], dtype=torch.int64, device=dev)
        gf._lib.check(lib.gf_attn_dropout_mask(ctypes.byref(desc), ctypes.c_float(att_dp), dp[1], state.data_ptr(), md.data_ptr(),
                                               _stream(dev)), "gf_attn_dropout_mask")
        torch.cuda.synchronize()
        mask = md.cpu()
    torch.cuda.synchronize()
    assert gf._lib.last_path() == "wgmma_tf32"
    got = {name: gv.check(name).cpu() for name, gv in outs.items()}

    # (a) GEMM1 + softmax (log2 units)
    Xt = tf32_trunc(X).double()
    RC = (tabs["Rt"][:, :, None, :].float() + tabs["Ct"][:, None, :, :].float()).double().reshape(B, n, KP)
    fin = torch.isfinite(RC)
    S = Xt @ tabs["Kp"].transpose(1, 2) + RC
    s_abs = Xt.abs() @ tabs["Kp"].abs().transpose(1, 2) + torch.where(fin, RC.abs(), torch.zeros_like(RC))
    p = torch.softmax(S * math.log(2.0), dim=2)[:, :, :k]
    F = 1.0 + s_abs[:, :, :k].amax(dim=2, keepdim=True)
    tiny = p < 2.0 ** -126                     # ex2.approx.ftz flushes probabilities below the smallest normal float to zero
    assert (got["att"].double()[tiny] < 2.0 ** -126).all()
    worst = {"att": _worst(got["att"].double()[~tiny], p[~tiny], (F * p)[~tiny], "att")}

    # (b) GEMM2 + the store side, from the kernel's own map
    q = torch.nn.functional.pad(got["att"], (0, KP - k)) * mask                       # f32 product, as the kernel forms it
    Pt = tf32_rna(q).double()
    Vt = tabs["Vt"]
    G = Pt @ Vt.transpose(1, 2)
    G_abs = Pt @ Vt.abs().transpose(1, 2)
    if dp:
        qdef = 1.0 - q.double().sum(dim=2, keepdim=True)
        G, G_abs = G + qdef * tabs["CB"], G_abs + qdef.abs() * tabs["CB"].abs()
    xin = (X * post["in_scale"].float()[:, None, :]).double() if post else X.double()
    if norm == "layer":
        xn = _ln64(xin)
        x0 = xin[:, :, :1]
        rstd = 1.0 / torch.sqrt(((xin - xin.mean(2, keepdim=True)) ** 2).mean(2, keepdim=True) + LN_EPS)
        xn_abs = (xin.abs() + (xin - x0).abs().mean(dim=2, keepdim=True) + x0.abs()) * rstd
    else:
        xn, xn_abs = xin, xin.abs()
    y = af._combine(xn, G, integration, C)
    y_abs = xn_abs * G_abs if integration == "mul" else (xn_abs + G_abs if integration == "add"
                                                         else xn_abs * G_abs[..., :C] + G_abs[..., C:])
    rgb = rgb_abs = None
    if post:
        nz = post["noise"][:, :, None] * post["strength"]
        y, y_abs = y + nz + post["bias"], y_abs + nz.abs() + post["bias"].abs()
        y = torch.where(y >= 0, y, 0.2 * y) * post["gain"]
        y_abs = y_abs * post["gain"]
        if "rgb_w" in post:
            rgb = torch.einsum("btc,boc->bot", y, post["rgb_w"]) + post["rgb_bias"][None, :, None]
            rgb_abs = torch.einsum("btc,boc->bot", y_abs, post["rgb_w"].abs()) + post["rgb_bias"].abs()[None, :, None]
        y, y_abs = y * post["post_scale"][:, None, :], y_abs * post["post_scale"][:, None, :]
    worst["Xout"] = _worst(got["Xout"].double(), y, y_abs, "Xout")
    if rgb is not None:
        worst["rgb"] = _worst(got["rgb"].double(), rgb, rgb_abs, "rgb")
    print(f"[attn-fwd] stage T {B}x{H}x{W} C={C} k={k} {integration} {norm} p={att_dp} mean={mean} post={with_post}: "
          + " ".join(f"{a}={v:.3e}" for a, v in worst.items()))
    for name, v in worst.items():
        assert v <= BOUND[name], f"{name}: {v:.3e} > {BOUND[name]:.1e}"


# ---- stage I ---------------------------------------------------------------------------------------------------------------------
def _ulp(v):
    a = v.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


@pytest.mark.parametrize("B,H,W,C,k,integration", [(4, 8, 16, 128, 16, "mul"), (3, 8, 16, 512, 20, "mul"), (8, 16, 16, 64, 5, "both")],
                         ids=_id)
def test_stage_i_tables(gf, cuda_dev, B, H, W, C, k, integration):
    """gf_attn_prologue_ex with in_scale on random weights: every K' and V^T element is a TF32 value, within one TF32 ulp (plus
    2^-20 of its row's largest element, for the cancellation in the fp32 sums) of rne(kf K'64 d) (kf = 1.000352220f log2 e) and rne(V^T64); the least-squares slope of K' against log2e K'64 d is the truncation
    compensation 1.000352220 within 2.2e-5 (measured on an H100 80GB HBM3 at 400 W: 6.3e-6, 2.8e-6 and 1.45e-5 off for the three
    cases, frozen at 1.5x the worst; dropping the compensation moves it by 3.5e-4); Rt / Ct are the fp64 tables in log2 units, -inf / 0 in the padded columns; the batched
    gf_attn_prologue_batch writes the same bits."""
    g = torch.Generator().manual_seed(C + k)
    KP, Cout = of.pad_k(k), 2 * C if integration == "both" else C
    d = (0.5 + torch.rand(B, C, generator=g, dtype=torch.float64)).float().double()
    ws, lay, desc, w, y = real_tables(gf, cuda_dev, B=B, H=H, W=W, C=C, k=k, integration=integration, norm="layer", seed=C,
                                      in_scale=d)
    got = read_tables(ws, lay, B, H, W, C, KP, Cout)
    f = of.fold_weights(w, C=C, k=k, integration=integration, duplex=False)
    Kp64, Vt64, Rt64, Ct64 = of.prologue(y, f, C=C, H=H, W=W, p=POS)
    kf = float(torch.tensor(af.TF32_TRUNC_COMP, dtype=torch.float32) * torch.tensor(af.LOG2E, dtype=torch.float32))
    for name in ("Kp", "Vt"):
        assert (tf32_low_bits(got[name].float()) == 0).all(), f"{name}: not on the TF32 grid"
    want_k = tf32_rne((Kp64 * d[:, None, :]).float() * kf).double()
    want_v = tf32_rne(Vt64.float()).double()
    for name, gv, wv, ax in (("Kp", got["Kp"], want_k, 2), ("Vt", got["Vt"], want_v, 1)):
        # one TF32 ulp, plus what the fp32 sums of stages W and I may lose to cancellation: 2^-20 of the row's largest element
        tol = torch.maximum(_ulp(gv), _ulp(wv)) + 2.0 ** -20 * wv.abs().amax(dim=ax, keepdim=True)
        assert ((gv - wv).abs() <= tol).all(), f"{name}: more than one TF32 ulp off"
    assert (got["Kp"][:, k:] == 0).all() and (got["Vt"][:, :, k:] == 0).all()
    a, b = got["Kp"][:, :k].reshape(-1), (Kp64 * d[:, None, :] * af.LOG2E)[:, :k].reshape(-1)
    slope = (a * b).sum() / (b * b).sum()
    print(f"[attn-fwd] stage I C={C} k={k}: K' slope {slope.item():.7f}")
    assert abs(slope.item() - af.TF32_TRUNC_COMP) < 2.2e-5
    assert (got["Rt"][:, :, k:] == -math.inf).all() and (got["Ct"][:, :, k:] == 0).all()
    for name, gv, wv in (("Rt", got["Rt"][:, :, :k], Rt64[:, :, :k] * af.LOG2E), ("Ct", got["Ct"][:, :, :k], Ct64[:, :, :k] * af.LOG2E)):
        assert ((gv - wv).abs() <= 1e-5 * (1.0 + wv.abs())).all(), name
    ws2, _, _, _, _ = real_tables(gf, cuda_dev, B=B, H=H, W=W, C=C, k=k, integration=integration, norm="layer", seed=C, in_scale=d,
                                  batch=True)
    for name in ("Kp", "Vt", "Rt", "Ct", "CB"):
        size = {"Kp": B * KP * C, "Vt": B * Cout * KP, "Rt": B * H * KP, "Ct": B * W * KP, "CB": Cout}[name]
        assert torch.equal(ws[lay[name]:lay[name] + size].view(torch.int32), ws2[lay[name]:lay[name] + size].view(torch.int32)), name


# ---- duplex pass A on wgmma ------------------------------------------------------------------------------------------------------
def pass_a_setup(gf, dev, tabs, *, B, H, W, C, k, scale=None):
    """A zeroed workspace holding M, Rt2 and Ct2, a folded buffer and the inputs of gf_attn_duplex_fwd_ex with GF_FLAG_TABLES_READY;
    returns launch() (enqueues the call on the current stream), the workspace and its layout."""
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, norm="layer", integration="mul", pos_dim=POS, duplex=1,
                             flags=gf._lib.FLAG_TABLES_READY)
    lib = _lib(gf)
    w = ob.init_params(C, D_LATENT, k, POS, "mul", True, seed=3, bias_std=0.2)
    folded = torch.empty(gf._lib.folded_floats(desc), device=dev)
    wst, keep = _weights_struct(gf, w, dev)
    gf._lib.check(lib.gf_attn_fold_weights(ctypes.byref(desc), ctypes.byref(wst), folded.data_ptr(), _stream(dev)), "fold")
    ws, lay = make_ws(gf, desc, dev, fill="zero")
    for name, key in (("M", "M"), ("Rt2", "Rt2"), ("Ct2", "Ct2")):
        _region(ws, lay[name], tabs[key].shape).copy_(_f32(tabs[key], dev))
    Xd = _f32(tabs["X"], dev)
    Y = torch.randn(B, k, D_LATENT, device=dev)
    Xout = torch.empty_like(Xd)
    po = Postop(gf, {"in_scale": scale} if scale is not None else None, dev, B, H * W, C)
    keep += [folded, Xd, Y, Xout, po]

    def launch():
        gf._lib.check(lib.gf_attn_duplex_fwd_ex(ctypes.byref(desc), Xd.data_ptr(), Y.data_ptr(), folded.data_ptr(), Xout.data_ptr(),
                                                None, None, ws.data_ptr(), ctypes.byref(po.s), _stream(dev)), "gf_attn_duplex_fwd_ex")
        assert gf._lib.last_centroid_path() == "wgmma_tf32"
    launch.keep = keep
    return launch, ws, lay


def pass_a(gf, dev, tabs, *, B, H, W, C, k, scale=None):
    """One eager gf_attn_duplex_fwd_ex call of pass_a_setup; returns Xbar (fp64, CPU, read from w_XBAR) and the layout."""
    launch, ws, lay = pass_a_setup(gf, dev, tabs, B=B, H=H, W=W, C=C, k=k, scale=scale)
    launch()
    torch.cuda.synchronize()
    return _region(ws, lay["XBAR"], (B, k, C)).double().cpu(), lay


def plant(B, H, W, k, ranges, seed):
    """Winners cycling through the first, a middle and the last non-empty split; latents j % 3 == 1 get two runners-up one log2
    unit below in earlier tiles of the winner's split (rows a and a + 1 above it, a W >= 64), latents j % 3 == 2 a tie in
    the winner's column in row 0 (or the last row when the winner is in row 0).  That row lies in the first (last) split, so the
    tie is in another split than the winner's when the winner is not there, and in the same split otherwise."""
    g = torch.Generator().manual_seed(seed)
    live = [r for r in ranges if r[1] > r[0]]
    picks = [live[0], live[len(live) // 2], live[-1]]
    a = -(-64 // W)
    win = torch.empty(B, k, dtype=torch.long)
    run = torch.full((B, k, 2), -1, dtype=torch.long)
    tie = torch.full((B, k), -1, dtype=torch.long)
    for b in range(B):
        for j in range(k):
            lo, hi = picks[(b + j) % 3]
            if j % 3 == 1 and lo + (a + 1) * W < hi:
                w = int(torch.randint(lo + (a + 1) * W, hi, (1,), generator=g))
                run[b, j] = torch.tensor([w - a * W, w - (a + 1) * W])
            else:
                w = int(torch.randint(lo, hi, (1,), generator=g))
            if j % 3 == 2:
                row = 0 if w // W != 0 else H - 1
                tie[b, j] = row * W + w % W
            win[b, j] = w
    return win, run, tie


# B, H, W, C, k, scaled: n = 4186 is 66 tiles of 64; the split count comes from the cost model (gf_attn_debug_layout): 11 on an
# H100 SXM (132 SMs), 6 tiles per split
EXACT_A = [
    (1, 46, 91, 64, 16, False),
    (2, 46, 91, 128, 27, True),
    (1, 46, 91, 256, 32, False),
    (1, 46, 91, 512, 13, True),                 # two CTAs per split share the channels
    (2, 46, 91, 512, 32, False),
    (3, 10, 13, 64, 5, True),                   # n = 130: three tiles of 64, the third holding 2 tokens (2 splits on 132 SMs)
]


def _pass_a_exact(gf, dev, B, H, W, C, k, scaled, seed):
    n = H * W
    lay = layout(gf, gf._lib.make_desc(B, H, W, C, k, D_LATENT, norm="layer", integration="mul", pos_dim=POS, duplex=1))
    ranges = af.pass_a_split_ranges(n, lay["nsplit"])
    win, run, tie = plant(B, H, W, k, ranges, seed)
    tabs, _, wts = af.exact_pass_a_case(B, H, W, C, k, winners=win, runners_up=run, ties=tie, seed=seed)
    d = 2.0 ** torch.randint(-1, 2, (B, C), generator=torch.Generator().manual_seed(seed)).double() if scaled else None
    got, _ = pass_a(gf, dev, tabs, B=B, H=H, W=W, C=C, k=k, scale=d)
    assert ((wts == 0.5).sum(dim=2) == 2).any() or n < 4 * 64, "no latent has its runners-up rescaled"
    assert_exact(got, af.exact_pass_a_xbar(tabs["X"], wts, ranges, scale=d), "Xbar")
    return ranges


@pytest.mark.parametrize("B,H,W,C,k,scaled", EXACT_A, ids=_id)
def test_pass_a_exact(gf, cuda_dev, B, H, W, C, k, scaled):
    """centroid_tc_kernel + centroid_merge_kernel on exact tables: with an integer winner x_w alone, Xbar = f32(f32(x_w)
    1.000352220f) d bit for bit; two runners-up one log2 unit below in an earlier tile make the online rescale multiply by exactly
    1/2 (l = 2); a tie is summed inside its split, or merged in split order when it lies in another split (see plant).  Padded
    latents, KP 16 and 32, C = 64 .. 512."""
    _pass_a_exact(gf, cuda_dev, B, H, W, C, k, scaled, seed=B * 1000 + C + k)


def test_pass_a_exact_empty_last_split(gf, cuda_dev):
    """The split count is chosen in 128-token tiles and the kernel walks 64-token tiles, so the last split can be empty (it writes
    a neutral partial).  The cost model never picks such a count on an H100 for these shapes, so a child process forces it with
    GF_NSPLIT_CEN (read once per process) and runs the exact case there."""
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import torch, gansformer_b200 as gf\n"
            "from tests import test_gpu_attn_forward as t\n"
            "r = t._pass_a_exact(gf, torch.device('cuda:0'), 2, 9, 64, 256, 20, True, seed=77)\n"
            "assert len(r) == 4 and r[-1][0] == r[-1][1] and all(b > a for a, b in r[:-1]), r\n"
            "r = t._pass_a_exact(gf, torch.device('cuda:0'), 1, 9, 64, 512, 13, False, seed=78)\n"
            "assert r[-1][0] == r[-1][1], r\n"
            "print('empty-split cases exact')\n") % ROOT
    env = dict(os.environ, GF_NSPLIT_CEN="4")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "empty-split cases exact" in res.stdout


@pytest.mark.parametrize("B,H,W,C,k,mean", [(2, 46, 91, 128, 20, 0.0), (1, 32, 32, 512, 32, 0.0), (2, 16, 16, 64, 16, 30.0)], ids=_id)
def test_pass_a_tf32_emulation(gf, cuda_dev, B, H, W, C, k, mean):
    """centroid_tc_kernel on realistic log2-unit tables (M rounded to TF32): Xbar against A^T tf32_trunc(x) 1.000352220 d with
    A = softmax_2(tf32_trunc(x) M^T + Rt2 + Ct2) in fp64, per element relative to (1 + the latent's largest |logit| companion)
    A^T |x| d.  The kernel rounds each weight E = 2^(s - m) to TF32 (cvt.rna) against the running maximum of its split; that
    rounding is not emulated here, so its error (up to 2^-11 of each weight) is part of what the bound holds.  The bound does not
    see the 1.000352220 of the flush (3.5e-4 relative, inside the companion's logit factor): the exact cases pin it."""
    g = torch.Generator().manual_seed(B + H + C + k)
    n, KP = H * W, of.pad_k(k)
    X = (torch.randn(B, n, C, generator=g) + mean).float()
    M = torch.randn(B, KP, C, generator=g) / math.sqrt(C) * af.LOG2E
    if mean:
        M = M - M.mean(dim=2, keepdim=True)
    M[:, k:] = 0.0
    M = tf32_rne(M.float())
    Rt2, Ct2 = (torch.randn(B, H, KP, generator=g) * af.LOG2E).float(), (torch.randn(B, W, KP, generator=g) * af.LOG2E).float()
    Rt2[:, :, k:] = -math.inf
    Ct2[:, :, k:] = 0.0
    d = (0.5 + torch.rand(B, C, generator=g)).float()
    got, _ = pass_a(gf, cuda_dev, dict(X=X, M=M, Rt2=Rt2, Ct2=Ct2), B=B, H=H, W=W, C=C, k=k, scale=d)
    Xt = tf32_trunc(X).double()
    RC = (Rt2[:, :, None, :k].double() + Ct2[:, None, :, :k].double()).reshape(B, n, k)
    L = Xt @ M[:, :k].double().transpose(1, 2) + RC
    L_abs = Xt.abs() @ M[:, :k].double().abs().transpose(1, 2) + RC.abs()
    A = torch.softmax(L * math.log(2.0), dim=1)
    want = (A.transpose(1, 2) @ Xt) * float(torch.tensor(af.TF32_TRUNC_COMP, dtype=torch.float32)) * d.double()[:, None, :]
    comp = (1.0 + L_abs.amax(dim=1))[:, :, None] * (A.transpose(1, 2) @ X.double().abs()) * d.double()[:, None, :]
    worst = _worst(got, want, comp, "Xbar")
    print(f"[attn-fwd] pass A {B}x{H}x{W} C={C} k={k} mean={mean}: Xbar={worst:.3e}")
    assert worst <= BOUND["Xbar"], f"Xbar: {worst:.3e} > {BOUND['Xbar']:.1e}"


# ---- properties ------------------------------------------------------------------------------------------------------------------
def test_properties_determinism_batch_independence_graph_replay(gf, cuda_dev):
    """Stage T on the tensor path with dropout, the post-op and tRGB, and pass A (gf_attn_duplex_fwd_ex with tables ready): two
    calls give identical bits; each image of a batch equals that image run alone (stage T without dropout: its mask is keyed by
    the global token index); a CUDA-graph replay equals the eager call bit for bit."""
    dev = cuda_dev
    B, H, W, C, k = 3, 16, 16, 128, 16
    g = torch.Generator().manual_seed(11)
    post = dict(in_scale=(0.5 + torch.rand(B, C, generator=g, dtype=torch.float64)).float().double(),
                bias=0.3 * torch.randn(C, generator=g, dtype=torch.float64), noise=torch.randn(B, H * W, generator=g, dtype=torch.float64),
                strength=0.25, act=1, gain=GAIN, post_scale=(0.5 + torch.rand(B, C, generator=g, dtype=torch.float64)),
                rgb_w=torch.randn(B, 3, C, generator=g, dtype=torch.float64) / math.sqrt(C), rgb_bias=torch.randn(3, generator=g, dtype=torch.float64))
    ws, lay, desc, _, _ = real_tables(gf, dev, B=B, H=H, W=W, C=C, k=k, integration="both", norm="layer", seed=4, in_scale=post["in_scale"])
    X = torch.randn(B, H * W, C, generator=g, device="cpu").to(dev) + 1.0
    lib = _lib(gf)

    def run(x, wsp, dsc, p, with_dp, nb=B):
        outs = (torch.empty(nb, H * W, C, device=dev), torch.empty(nb, H * W, k, device=dev), torch.empty(nb, 3, H * W, device=dev))
        po = Postop(gf, p, dev, nb, H * W, C, dp=(0.12, 9, 555, 1) if with_dp else None, rgb_out=outs[2].data_ptr())
        gf._lib.check(lib.gf_attn_simplex_fwd_ex(ctypes.byref(dsc), x.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), wsp.data_ptr(),
                                                 ctypes.byref(po.s), _stream(dev)), "gf_attn_simplex_fwd_ex")
        torch.cuda.synchronize()
        return outs, po

    a, _ = run(X, ws, desc, post, True)
    b, _ = run(X, ws, desc, post, True)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    full, _ = run(X, ws, desc, post, False)
    one = {n_: (v[1:2] if torch.is_tensor(v) and v.dim() >= 2 and v.shape[0] == B else v) for n_, v in post.items()}
    ws1, lay1, desc1, _, _ = real_tables(gf, dev, B=1, H=H, W=W, C=C, k=k, integration="both", norm="layer", seed=4, in_scale=one["in_scale"])
    # the one-image tables are image 0 of a batch drawn with the same latents seed: copy image 1's tables instead
    KP, Cout = of.pad_k(k), 2 * C
    for name, per in (("Kp", KP * C), ("Vt", Cout * KP), ("Rt", H * KP), ("Ct", W * KP)):
        ws1[lay1[name]:lay1[name] + per].copy_(ws[lay[name] + per:lay[name] + 2 * per])
    alone, _ = run(X[1:2].contiguous(), ws1, desc1, one, False, nb=1)
    for u, v in zip(full, alone):
        assert torch.equal(u[1:2], v)

    # pass A: determinism and batch independence
    n = H * W
    tabs = dict(X=torch.randn(B, n, C, generator=g), M=tf32_rne((torch.randn(B, 16, C, generator=g) / math.sqrt(C)).float()),
                Rt2=torch.randn(B, H, 16, generator=g), Ct2=torch.randn(B, W, 16, generator=g))
    x1, _ = pass_a(gf, dev, tabs, B=B, H=H, W=W, C=C, k=16)
    x2, _ = pass_a(gf, dev, tabs, B=B, H=H, W=W, C=C, k=16)
    x3, _ = pass_a(gf, dev, {a_: v[1:2] for a_, v in tabs.items()}, B=1, H=H, W=W, C=C, k=16)
    assert torch.equal(x1, x2) and torch.equal(x1[1:2], x3)

    # graph replay: stage T with dropout (the state is read at run time), post-op and tRGB, and the pass-A call, captured together
    outs = (torch.empty(B, n, C, device=dev), torch.empty(B, n, k, device=dev), torch.empty(B, 3, n, device=dev))
    po = Postop(gf, post, dev, B, n, C, dp=(0.12, 9, 555, 1), rgb_out=outs[2].data_ptr())
    launch_a, ws_a, lay_a = pass_a_setup(gf, dev, tabs, B=B, H=H, W=W, C=C, k=16)
    xbar = _region(ws_a, lay_a["XBAR"], (B, 16, C))

    def call():
        gf._lib.check(lib.gf_attn_simplex_fwd_ex(ctypes.byref(desc), X.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), ws.data_ptr(),
                                                 ctypes.byref(po.s), _stream(dev)), "gf_attn_simplex_fwd_ex")
        launch_a()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (*outs, xbar)]
    assert torch.equal(eager[0], a[0]) and torch.equal(eager[3].double().cpu(), x1)
    for t in (*outs, xbar):
        t.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    graph.replay()
    torch.cuda.synchronize()
    for i, (e, t) in enumerate(zip(eager, (*outs, xbar))):
        assert torch.equal(e, t), ("Xout", "att", "rgb", "Xbar")[i]
