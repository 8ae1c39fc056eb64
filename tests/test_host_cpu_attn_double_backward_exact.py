"""CPU checks behind tests/test_gpu_attn_double_backward_exact.py, and the host-side validation of the double-backward entries.

* The exact cases.  The GPU tests demand that token_bwd_vjp_kernel and centroid_bwd_vjp_kernel equal the fp64 references bit for
  bit on them.  That is only a fair demand if every intermediate of the kernels' arithmetic is an fp32 value whatever the order of
  summation.  ``stage_t_vjp_exactness`` / ``centroid_vjp_exactness`` (tests/attn_double_backward_ref.py) restate that arithmetic in
  fp64; for every case of the GPU file these tests check that every partial sum of every intermediate is a multiple of its grain
  below 2^24 grains, that the restatement's outputs equal the autograd references (tests/attn_double_backward_ref.py,
  tests/attn_double_backward_dropout_ref.py, oracle/attn_bwd.py) exactly, and so do the reductions the caller forms from them.
* The entries gf_attn_simplex_bwd_vjp, gf_attn_simplex_bwd_vjp_ex and gf_attn_centroid_bwd_vjp refuse every unsupported call
  before they touch the device, so these run without a GPU.
"""
import ctypes
import math

import pytest
import torch

from oracle import attn_bwd as ab
from tests import attn_double_backward_dropout_ref as dr
from tests import attn_double_backward_ref as vr
from tests.test_gpu_attn_double_backward import reduce_centroid, reduce_stage_t
from tests.test_gpu_attn_double_backward_dropout import reduce_ex
from tests.test_gpu_attn_double_backward_exact import (EXACT_A_VJP, EXACT_T_VJP, centroid_exact_inputs, stage_t_exact_inputs)
from tests.test_host_cpu_attn_backward import _check_exact, _roundtrips


@pytest.mark.parametrize("B,H,W,C,k,integration,dropout", EXACT_T_VJP, ids=str)
def test_stage_t_vjp_exact_case_is_exact(B, H, W, C, k, integration, dropout):
    case, ins, cots, cbg = stage_t_exact_inputs(B, H, W, C, k, integration, dropout)
    items, outs, bound = vr.stage_t_vjp_exactness(*ins, *cots, k=k, integration=integration, mult=case["mult"], cb=case["cb"], cbg=cbg)
    p = dict((nm, v) for nm, v, _, _ in items)["p"][:, :, :k]
    assert set(p.unique().tolist()) <= {0.0, 0.5, 1.0}
    assert (p == 1.0).any() and ((p == 0.5).any() or k == 1)
    if dropout:
        assert set(case["mult"].unique().tolist()) == {0.0, 2.0}
    _check_exact(items)
    assert bound < 2.0 ** 100                             # the masked (inert) latents stay finite
    assert all(torch.count_nonzero(t) for t in cots + ([cbg] if dropout else []))
    if cots[1].shape[1] > k:                              # padded latents: nonzero rows of Kg, Vg and Cg
        assert torch.count_nonzero(cots[1][:, k:]) and torch.count_nonzero(cots[2][..., k:]) and torch.count_nonzero(cots[4][..., k:])

    kw =dict(H=H, W=W, integration=integration, norm="none")
    if dropout:
        ref = dr.stage_t_vjp_dropout(*ins, case["cb"], case["mult"], *cots, cbg, **kw)
        red = reduce_ex(outs, ins, cots)
    else:
        ref = vr.stage_t_vjp(*ins, *cots, **kw)
        red = reduce_stage_t(outs, ins, cots, H, W)
    first = ab.stage_t_backward(*ins, **kw, mult=case["mult"], cb=case["cb"])
    for nm in ("Xg", "dOutg", "Sg", "Ctlg"):
        assert torch.equal(outs[nm], ref[nm]), nm
    for nm in ("dS", "P", "dCtl"):
        assert torch.equal(outs[nm], first[nm]), nm
    for nm, t in red.items():
        assert torch.equal(t, ref[nm]), "reduction " + nm
    _roundtrips(outs)
    _roundtrips(red)
    assert (outs["Sg"] != 0).any() or k == 1              # the cotangent of the logits is exercised (k = 1: p = 1, Sg = 0)


@pytest.mark.parametrize("B,H,W,C,k", EXACT_A_VJP, ids=str)
def test_centroid_vjp_exact_case_is_exact(B, H, W, C, k):
    ins, cots = centroid_exact_inputs(B, H, W, C, k)
    items, outs, bound = vr.centroid_vjp_exactness(*ins[:7], *cots, k=k)
    A = outs["A"][:, :, :k]
    assert set(A.unique().tolist()) <= {0.0, 1.0} and torch.count_nonzero(outs["A"][:, :, k:]) == 0
    n = H * W
    active = A.sum(dim=2) > 0                                           # [B,n]
    assert (A.sum(dim=1) == W).all()                                    # every latent: one whole row
    tiles = {int(t) // 128 for t in active.nonzero()[:, 1]}
    if n > 128 and B * k >= 3:                                          # several tiles, the ragged last one among them
        assert len(tiles) >= min(3, (n + 127) // 128) and (n - 1) // 128 in tiles
    _check_exact(items)
    assert bound < 2.0 ** 24
    ref = vr.centroid_vjp(*ins, *cots, H=H, W=W, k=k)
    for nm in outs:
        assert torch.equal(outs[nm], ref[nm]), nm
    red = reduce_centroid(outs, ins[0], cots[0], H, W, k)
    for nm, t in red.items():
        assert torch.equal(t, ref[nm]), "reduction " + nm
    _roundtrips(outs)
    _roundtrips(red)
    assert (outs["dS"] != 0).any() and (outs["Sg"] != 0).any() and (outs["Gg"] != 0).any()
    if ins[1].shape[1] > k:                                             # padded latents: lse = -inf, nonzero M, Mg and Ct2g
        assert torch.count_nonzero(cots[1][:, k:]) and torch.count_nonzero(ins[1][:, k:]) and torch.count_nonzero(cots[3][..., k:])
        assert (ins[4][:, k:] == -math.inf).all()


# ---- host-side validation ------------------------------------------------------------------------------------------------------
def _desc(gf, B=2, C=64, k=8, heads=1, norm="layer", duplex=0):
    return gf._lib.make_desc(B, 8, 8, C, k, 16, heads=heads, norm=norm, integration="mul", pos_dim=0, duplex=duplex)


def _simplex(lib, desc, ptrs=None, att_dp=0.0, state=None, cb=None, cbg=None):
    ptrs = [1] * 19 if ptrs is None else ptrs
    return lib.gf_attn_simplex_bwd_vjp_ex(ctypes.byref(desc), *ptrs, ctypes.c_float(att_dp), 0, state, cb, cbg, None)


def test_simplex_vjp_entries_validate_before_touching_the_device(gf):
    lib = gf._lib.load()
    err = lambda: lib.gf_last_error().decode()
    for i in range(19):                                                 # every pointer, through both entries
        ptrs = [1] * 19
        ptrs[i] = None
        assert lib.gf_attn_simplex_bwd_vjp(ctypes.byref(_desc(gf)), *ptrs, None) == -1 and "null pointer" in err(), i
        assert _simplex(lib, _desc(gf), ptrs) == -1 and "null pointer" in err(), i
    assert _simplex(lib, _desc(gf, duplex=1)) == -2 and "simplex descriptor" in err()
    assert lib.gf_attn_simplex_bwd_vjp(ctypes.byref(_desc(gf, duplex=1)), *([1] * 19), None) == -2 and "simplex descriptor" in err()
    assert _simplex(lib, _desc(gf, heads=2)) == -2 and "one head" in err()
    for norm in ("instance", "batch"):
        assert _simplex(lib, _desc(gf, norm=norm)) == -2 and "norm must be layer or none" in err()
    assert _simplex(lib, _desc(gf, B=65536)) == -2 and "B > 65535" in err()
    bad = _desc(gf)
    bad.C = 48
    assert _simplex(lib, bad) == -2 and "C=48" in err()
    # att_dp outside [0, 1) with a state pointer (never dereferenced on the host); without a state the entry ignores att_dp
    for p in (-0.25, 1.0, 1.5, float("nan")):
        assert _simplex(lib, _desc(gf), att_dp=p, state=1, cb=1, cbg=1) == -1 and "must be in [0, 1)" in err(), p
    assert _simplex(lib, _desc(gf), att_dp=0.12, state=1, cb=None, cbg=1) == -1 and "needs cb" in err()
    assert _simplex(lib, _desc(gf), att_dp=0.12, state=1, cb=1, cbg=None) == -1 and "cbg" in err()


def test_centroid_vjp_entry_validates_before_touching_the_device(gf):
    lib = gf._lib.load()
    err = lambda: lib.gf_last_error().decode()
    call = lambda desc, ptrs=None: lib.gf_attn_centroid_bwd_vjp(ctypes.byref(desc), *([1] * 16 if ptrs is None else ptrs), None)
    for i in range(16):
        ptrs = [1] * 16
        ptrs[i] = None
        assert call(_desc(gf, duplex=1), ptrs) == -1 and "null pointer" in err() and "gf_attn_centroid_bwd_vjp" in err(), i
    assert call(_desc(gf, duplex=0)) == -1 and "desc.duplex is 0" in err()
    assert call(_desc(gf, duplex=2)) == -2 and "one k-means iteration" in err()
    for norm in ("instance", "batch"):
        assert call(_desc(gf, norm=norm, duplex=1)) == -2 and "norm must be layer or none" in err()
    assert call(_desc(gf, B=65536, duplex=1)) == -2 and "B > 65535" in err()
    bad = _desc(gf, duplex=1)
    bad.C = 48
    assert call(bad) == -2 and "C=48" in err()
