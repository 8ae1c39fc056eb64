"""Exact and one-cotangent-at-a-time GPU tests of the double-backward kernels (csrc/gf_bwd.cu; run on an H100: ``pytest -m gpu``).

* ``gf_attn_simplex_bwd_vjp`` / ``gf_attn_simplex_bwd_vjp_ex`` (``token_bwd_vjp_kernel<KP, false>`` / ``<KP, true>``);
* ``gf_attn_centroid_bwd_vjp`` (``centroid_bwd_vjp_kernel<KP>``).

Each output of these kernels is a sum of several terms, and the tolerance tests of tests/test_gpu_attn_double_backward.py and
tests/test_gpu_attn_double_backward_dropout.py judge a whole tensor with every cotangent on at once, so a wrong term that is small
next to the tensor's largest element can pass them.  Here:

* Exact cases (``tests/attn_double_backward_ref.py``: ``exact_stage_t_vjp_case``, ``exact_centroid_vjp_case``).  Stage T uses the
  one-hot pairs of the first-order exact cases (norm none, every probability 0, 1/2 or 1, dropout at p = 1/2) with small-integer
  cotangents; pass A makes every token of one row per latent active with a = exp(0) = 1 (lse is an input) and every other token
  a = 0.  Every intermediate is then an fp32 value whatever the order of summation (tests/test_host_cpu_attn_double_backward_exact.py
  proves it on the host for exactly these cases), so every per-token output, and every reduction the caller forms from them in
  fp64, equals the fp64 reference bit for bit; dS, P and dCtl (stage T) and dS (pass A) also equal the first-order entry's.  The
  stage-T cases are the matrix of the first-order exact tests: C = 32 to 1024, k = 1 to 32, n = 1 to 4096 with ragged tiles,
  B = 300, every integration with and without dropout.  Layer norm is not exact (rsqrtf): it is covered by the runs below.
* One cotangent at a time.  The VJP is linear in its cotangents: each realistic case runs once per cotangent with the others zero,
  against the fp64 reference of that run, so only the terms that cotangent reaches are left.  An output whose reference is
  identically zero must be exactly 0; every other output is held, as in the tolerance tests (per-token outputs max |kernel - fp64|
  / max |fp64|, reductions relative to their magnitude companion), to a bound per (kernel, cotangent).
* All cotangents zero: the cotangent outputs are exactly 0 and dS, P, dCtl are the first-order kernel's bits.

Every output sits between NaN guards; the runners check the guards and that every element was written.
"""
import ctypes

import pytest
import torch

from oracle import attn_bwd as ab
from oracle.folded import pad_k
from tests import attn_double_backward_dropout_ref as dr
from tests import attn_double_backward_ref as vr
from tests.guards import Guarded, assert_exact
from tests.test_gpu_attn_backward import EXACT_T, stage_t as first_order_stage_t
from tests.test_gpu_attn_double_backward import (D_LATENT, _err, _f32, _stream, centroid_case, reduce_centroid, reduce_stage_t,
                                                 run_centroid, run_stage_t, stage_t_case)
from tests.test_gpu_attn_double_backward_dropout import SALT, _state, dropout_case, reduce_ex

pytestmark = pytest.mark.gpu

T_INS = ("X", "dOut", "Kp", "Vt", "Rt", "Ct")
T_COTS = ("U", "Kg", "Vg", "Rg", "Cg")
A_INS = ("X", "M", "Rt2", "Ct2", "lse", "dXbar", "r", "dX0")
A_COTS = ("U", "Mg", "Rt2g", "Ct2g")

# Stage T: the matrix of the first-order exact tests (B, H, W, C, k, integration, dropout at p = 1/2; norm none).
EXACT_T_VJP = EXACT_T
# Pass A: B, H, W, C, k.  n = 4186 is 33 tiles with a ragged last one of 90 tokens.
EXACT_A_VJP = [
    (1, 46, 91, 32, 1),
    (3, 46, 91, 96, 16),
    (1, 46, 91, 512, 17),                   # KP = 32 with 15 padded latents
    (3, 46, 91, 96, 32),
    (1, 46, 91, 32, 32),
    (3, 10, 13, 512, 16),
    (2, 1, 1, 32, 4),                       # one token
    (300, 5, 7, 32, 4),                     # B in the hundreds
]

# One cotangent at a time.  B, H, W, C, k, integration, norm, mean (stage T; with att_dp for the dropout variant).
ISO_T = [
    (3, 10, 13, 96, 20, "mul", "layer", 30.0),
    (2, 8, 8, 64, 16, "both", "layer", 0.0),
    (3, 128, 1, 96, 17, "mul", "none", 0.0),        # KP = 32 with 15 padded latents
    (1, 10, 13, 1024, 32, "both", "layer", 30.0),   # 32 chunks
    (2, 10, 13, 96, 4, "add", "none", 0.0),
]
ISO_D = [
    (2, 10, 13, 96, 20, "mul", "layer", 30.0, 0.12),
    (1, 8, 8, 1024, 32, "both", "layer", 0.0, 0.5),
    (2, 9, 11, 64, 17, "add", "none", 0.0, 0.5),
    (3, 10, 13, 96, 4, "both", "none", 30.0, 0.12),
]
# B, H, W, C, k, mean (pass A)
ISO_A = [
    (3, 10, 13, 96, 20, 30.0),
    (1, 46, 91, 64, 32, 0.0),
    (2, 10, 13, 512, 16, 0.0),
]
# Bound on the error of a one-cotangent run, per (kernel, cotangent): max |kernel - fp64| / max |fp64| for the per-token outputs,
# relative to the magnitude companion for the reductions.  Frozen at >= 1.5x the worst measured over the cases above on an H100
# 80GB HBM3 (the worst values are in DESIGN.md section 5).  T: gf_attn_simplex_bwd_vjp, D: gf_attn_simplex_bwd_vjp_ex with dropout,
# A: gf_attn_centroid_bwd_vjp.
BOUND_ISO = {
    ("T", "U"): 1.6e-5, ("T", "Kg"): 1.6e-5, ("T", "Vg"): 1.5e-5, ("T", "Rg"): 1.2e-5, ("T", "Cg"): 2e-5,
    ("D", "U"): 1.6e-5, ("D", "Kg"): 7e-6, ("D", "Vg"): 5e-6, ("D", "Rg"): 9e-6, ("D", "Cg"): 8e-6, ("D", "cbg"): 8e-6,
    ("A", "U"): 1.4e-5, ("A", "Mg"): 1.4e-5, ("A", "Rt2g"): 1.4e-5, ("A", "Ct2g"): 8e-6,
}


def _id(v):
    return str(v)


def run_ex(gf, dev, ins, cb, cots, cbg, *, H, W, k, integration, norm, att_dp, salt, state):
    """gf_attn_simplex_bwd_vjp_ex with the given salt; the eight outputs, guards checked."""
    X = _f32(ins[0], dev)
    B, n, C = X.shape
    KP, Cout = pad_k(k), ins[3].shape[1]
    tabs = [_f32(t, dev) for t in list(ins[1:]) + list(cots)]
    cbd, cbgd = _f32(cb, dev), _f32(cbg, dev)
    shapes = {"Xg": (B, n, C), "dOutg": (B, n, C), "Sg": (B, n, KP), "dPg": (B, n, KP), "Ctlg": (B, n, Cout), "dS": (B, n, KP),
              "P": (B, n, KP), "dCtl": (B, n, Cout)}
    outs = {nm: Guarded(s, dev) for nm, s in shapes.items()}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm=norm, integration=integration, pos_dim=0, duplex=False)
    gf._lib.check(gf._lib.load().gf_attn_simplex_bwd_vjp_ex(
        ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs), *(o.ptr() for o in outs.values()), ctypes.c_float(att_dp),
        salt, state.data_ptr(), cbd.data_ptr(), cbgd.data_ptr(), _stream(dev)), "gf_attn_simplex_bwd_vjp_ex")
    torch.cuda.synchronize(dev)
    return {nm: o.check(nm).clone() for nm, o in outs.items()}


def first_order_centroid(gf, dev, ins, *, H, W, k):
    """gf_attn_centroid_bwd on the same X, M, Rt2, Ct2, lse, dXbar, r, with dX preloaded with dX0: (dX, dS) as fp64."""
    X = _f32(ins[0], dev)
    B, n, C = X.shape
    M, Rt2, Ct2, lse, dXbar, r = (_f32(t, dev) for t in ins[1:7])
    dX, dS = Guarded((B, n, C), dev, init=_f32(ins[7], dev)), Guarded((B, n, pad_k(k)), dev)
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    gf._lib.check(gf._lib.load().gf_attn_centroid_bwd(ctypes.byref(desc), X.data_ptr(), M.data_ptr(), Rt2.data_ptr(), Ct2.data_ptr(),
                                                      lse.data_ptr(), dXbar.data_ptr(), r.data_ptr(), dX.ptr(), dS.ptr(), _stream(dev)),
                  "gf_attn_centroid_bwd")
    torch.cuda.synchronize(dev)
    return dX.check("dX", written=False).double().cpu(), dS.check("dS").double().cpu()


def active_rows(B, H, k, seed):
    """rows [B,k] of the pass-A exact cases: the first, a middle and the last row (the ragged last tile) in turn, and random rows."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.randint(0, H, (B, k), generator=g)
    for b in range(B):
        for j in range(k):
            pick = (b + j) % 4
            if pick < 3:
                rows[b, j] = (0, H // 2, H - 1)[pick]
    return rows


def stage_t_exact_inputs(B, H, W, C, k, integration, dropout):
    case, cots = vr.exact_stage_t_vjp_case(B, H, W, C, k, integration, dropout=dropout, seed=B * 1000 + C + k + 1)
    return case, [case[nm] for nm in T_INS], [cots[nm] for nm in T_COTS], cots["cbg"]


def centroid_exact_inputs(B, H, W, C, k):
    rows = active_rows(B, H, k, seed=C + k)
    case, cots = vr.exact_centroid_vjp_case(B, H, W, C, k, rows=rows, seed=B * 100 + C + k)
    return [case[nm] for nm in A_INS], [cots[nm] for nm in A_COTS]


def _cpu(o):
    return {nm: t.double().cpu() for nm, t in o.items()}


@pytest.mark.parametrize("B,H,W,C,k,integration,dropout", EXACT_T_VJP, ids=_id)
def test_stage_t_vjp_exact(gf, cuda_dev, B, H, W, C, k, integration, dropout):
    """token_bwd_vjp_kernel on exact tables and cotangents: the eight per-token outputs and the caller's reductions equal the fp64
    reference bit for bit, and dS, P, dCtl equal gf_attn_simplex_bwd_ex's."""
    case, ins, cots, cbg = stage_t_exact_inputs(B, H, W, C, k, integration, dropout)
    kw = dict(H=H, W=W, integration=integration, norm="none")
    if dropout:
        got = run_ex(gf, cuda_dev, ins, case["cb"], cots, cbg, k=k, att_dp=case["att_dp"], salt=case["salt"],
                     state=_state(cuda_dev, case["dp_seed"], case["step"]), **kw)
        ref = dr.stage_t_vjp_dropout(*ins, case["cb"], case["mult"], *cots, cbg, **kw)
        red = reduce_ex(got, ins, cots)
    else:
        got = run_stage_t(gf, cuda_dev, ins, cots, k=k, **kw)
        ref = vr.stage_t_vjp(*ins, *cots, **kw)
        red = reduce_stage_t(got, ins, cots, H, W)
    first = ab.stage_t_backward(*ins, **kw, mult=case["mult"], cb=case["cb"])
    _, restated, _ = vr.stage_t_vjp_exactness(*ins, *cots, k=k, integration=integration, mult=case["mult"], cb=case["cb"], cbg=cbg)
    got = _cpu(got)
    p = restated["P"][:, :, :k] if not dropout else None
    if p is not None:                                   # one-hot rows and ties both happen
        assert (p == 1.0).any() and ((p == 0.5).any() or k == 1)
    for nm in ("Xg", "dOutg", "Sg", "Ctlg"):
        assert_exact(got[nm], ref[nm], nm)
    for nm in ("dS", "P", "dCtl"):
        assert_exact(got[nm], first[nm], nm)
    assert_exact(got["dPg"], restated["dPg"], "dPg")
    for nm, t in red.items():
        assert_exact(t, ref[nm], "reduction " + nm)
    kernel_first = first_order_stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, norm="none")
    for nm in ("dS", "P", "dCtl"):
        assert_exact(got[nm], kernel_first[nm], "first-order " + nm)
    assert torch.count_nonzero(got["Xg"]) and torch.count_nonzero(got["dOutg"])


@pytest.mark.parametrize("B,H,W,C,k", EXACT_A_VJP, ids=_id)
def test_centroid_vjp_exact(gf, cuda_dev, B, H, W, C, k):
    """centroid_bwd_vjp_kernel with every token of one row per latent active (a = 1) and the rest a = 0: Xg, Sg, Gg, A, dS and the
    caller's reductions equal the fp64 reference bit for bit; dS equals gf_attn_centroid_bwd's, and its dX the fp64 dX."""
    ins, cots = centroid_exact_inputs(B, H, W, C, k)
    got = run_centroid(gf, cuda_dev, ins, cots, H=H, W=W, k=k)
    ref = vr.centroid_vjp(*ins, *cots, H=H, W=W, k=k)
    red = reduce_centroid(got, ins[0], cots[0], H, W, k)
    got = _cpu(got)
    for nm in ("Xg", "Sg", "Gg", "A", "dS"):
        assert_exact(got[nm], ref[nm], nm)
    for nm, t in red.items():
        assert_exact(t, ref[nm], "reduction " + nm)
    assert (got["dS"] != 0).any() and (got["Sg"] != 0).any() and (got["Gg"] != 0).any()
    dX, dS = first_order_centroid(gf, cuda_dev, ins, H=H, W=W, k=k)
    assert_exact(dS, got["dS"], "first-order dS")
    assert_exact(dX, vr.centroid_reductions(*(t.double() for t in ins), H=H, W=W, k=k)[0], "first-order dX")


def _iso_check(kernel, cot, case, got, ref, red, comp, per_token):
    """Zero references need exact zeros; every other output within BOUND_ISO[(kernel, cot)]."""
    errs = {}
    for nm in per_token:
        if torch.count_nonzero(ref[nm]) == 0:
            assert torch.count_nonzero(got[nm]) == 0, f"{nm}: nonzero where the reference is identically 0"
        else:
            errs[nm] = _err(got[nm], ref[nm])
    for nm, t in red.items():
        if torch.count_nonzero(ref[nm]) == 0:
            assert torch.count_nonzero(t) == 0, f"reduction {nm}: nonzero where the reference is identically 0"
        else:
            errs[nm] = _err(t, ref[nm], comp[nm])
    worst = max(errs, key=errs.get)
    print(f"[iso {kernel} {cot}] {case}: worst {worst} {errs[worst]:.2e}  " + " ".join(f"{a}={b:.1e}" for a, b in errs.items()))
    assert errs[worst] <= BOUND_ISO[(kernel, cot)], worst


def _only(names, tensors, keep):
    return [t if nm == keep else torch.zeros_like(t) for nm, t in zip(names, tensors)]


@pytest.mark.parametrize("cot", T_COTS)
@pytest.mark.parametrize("case", ISO_T, ids=_id)
def test_stage_t_vjp_one_cotangent(gf, cuda_dev, case, cot):
    B, H, W, C, k, integration, norm, mean = case
    ins, cots = stage_t_case(B, H, W, C, k, integration, mean, seed=B * 7 + C + k)
    cots = _only(T_COTS, cots, cot)
    kw = dict(H=H, W=W, integration=integration, norm=norm)
    got = run_stage_t(gf, cuda_dev, ins, cots, k=k, **kw)
    ref = vr.stage_t_vjp(*ins, *cots, **kw)
    red = reduce_stage_t(got, ins, cots, H, W)
    comp = reduce_stage_t({nm: t.abs() for nm, t in got.items()}, [t.abs() for t in ins], [t.abs() for t in cots], H, W)
    _iso_check("T", cot, case, got, ref, red, comp, ("Xg", "dOutg", "Sg", "Ctlg"))


@pytest.mark.parametrize("cot", T_COTS + ("cbg",))
@pytest.mark.parametrize("case", ISO_D, ids=_id)
def test_stage_t_vjp_dropout_one_cotangent(gf, cuda_dev, case, cot):
    B, H, W, C, k, integration, norm, mean, att_dp = case
    seed = B * 7 + C + k
    ins, cb, cots, cbg = dropout_case(B, H, W, C, k, integration, mean, seed)
    cots_all = _only(T_COTS + ("cbg",), list(cots) + [cbg], cot)
    cots, cbg = cots_all[:5], cots_all[5]
    dseed, step = 0x1234567 + seed, 5
    kw = dict(H=H, W=W, integration=integration, norm=norm)
    got = run_ex(gf, cuda_dev, ins, cb, cots, cbg, k=k, att_dp=att_dp, salt=SALT, state=_state(cuda_dev, dseed, step), **kw)
    mult = dr.philox_mult(att_dp, dseed, step, SALT, B, H * W, pad_k(k))
    ref = dr.stage_t_vjp_dropout(*ins, cb, mult, *cots, cbg, **kw)
    red = reduce_ex(got, ins, cots)
    comp = reduce_ex({nm: t.abs() for nm, t in got.items()}, [t.abs() for t in ins], [t.abs() for t in cots], companion=True)
    _iso_check("D", cot, case, got, ref, red, comp, ("Xg", "dOutg", "Sg", "Ctlg"))


@pytest.mark.parametrize("cot", A_COTS)
@pytest.mark.parametrize("case", ISO_A, ids=_id)
def test_centroid_vjp_one_cotangent(gf, cuda_dev, case, cot):
    B, H, W, C, k, mean = case
    ins, cots = centroid_case(B, H, W, C, k, mean, seed=B + C + k)
    cots = _only(A_COTS, cots, cot)
    got = run_centroid(gf, cuda_dev, ins, cots, H=H, W=W, k=k)
    ref = vr.centroid_vjp(*ins, *cots, H=H, W=W, k=k)
    red = reduce_centroid(got, ins[0], cots[0], H, W, k)
    comp = reduce_centroid({nm: t.abs() for nm, t in got.items()}, ins[0].abs(), cots[0].abs(), H, W, k)
    comp = {nm: t.abs() for nm, t in comp.items()}
    _iso_check("A", cot, case, got, ref, red, comp, ("Xg", "Sg", "Gg"))


@pytest.mark.parametrize("integration,norm,att_dp", [("both", "layer", 0.0), ("mul", "none", 0.0), ("mul", "layer", 0.12),
                                                     ("both", "none", 0.5)], ids=_id)
def test_zero_cotangents(gf, cuda_dev, integration, norm, att_dp):
    """All cotangents zero: Xg, dOutg, Sg, dPg and Ctlg are exactly 0, and dS, P, dCtl are gf_attn_simplex_bwd_ex's bits."""
    B, H, W, C, k = 3, 10, 13, 96, 20
    ins, cb, cots, cbg = dropout_case(B, H, W, C, k, integration, 30.0, seed=8)
    cots, cbg = [torch.zeros_like(t) for t in cots], torch.zeros_like(cbg)
    kw = dict(H=H, W=W, k=k, integration=integration, norm=norm)
    if att_dp:
        dseed, step = 4242, 3
        got = run_ex(gf, cuda_dev, ins, cb, cots, cbg, att_dp=att_dp, salt=SALT, state=_state(cuda_dev, dseed, step), **kw)
        case = dict(zip(T_INS, ins), att_dp=att_dp, dp_seed=dseed, step=step, salt=SALT, cb=cb)
    else:
        got = run_stage_t(gf, cuda_dev, ins, cots, **kw)
        case = dict(zip(T_INS, ins), att_dp=0.0, salt=0)
    first = first_order_stage_t(gf, cuda_dev, case, **kw)
    for nm in ("Xg", "dOutg", "Sg", "dPg", "Ctlg"):
        assert torch.count_nonzero(got[nm]) == 0, nm
    for nm in ("dS", "P", "dCtl"):
        assert torch.equal(got[nm].double().cpu(), first[nm]), nm
