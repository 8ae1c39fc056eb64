"""Host-side proofs behind tests/test_gpu_attn_stage_wi.py (no GPU needed).

* The oracle's multi-head fold and the duplex folds (keys from Xbar, the centroid query fold ACQ) equal the direct form of
  oracle/bipartite.py in fp64.
* The kernel-order restatement of stage W and I (oracle/stage_wi.py) agrees with oracle/folded.py, and every exact GPU case is exact:
  each fp32 step of the chain is proven exact (the restatement asserts it), the positional axis tables are far from fp32 rounding
  midpoints, the default-mode V^T tables hold ties that round-to-nearest-even and ties-away round differently, the key GEMM's
  operands are TF32 values and the Xbar route gives back the integer winners.
* The statistics cases: the split structure the GPU test asks for, exact fp64 sums, and the power-of-two statistics of the affine case.
"""
import math

import pytest
import torch

from oracle import attn_fwd as af
from oracle import bipartite as ob
from oracle import folded as of
from oracle import stage_wi as sw
from oracle.tf32 import tf32_rna, tf32_rne, tf32_trunc
from tests import test_gpu_attn_stage_wi as g

H, W = g.HW


def _id(v):
    return str(v)


# ---- the oracle against the direct form ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,integration", [(2, "mul"), (4, "both"), (2, "add"), (4, "mul")], ids=_id)
def test_multi_head_fold_matches_direct(heads, integration):
    """fold_weights / prologue with num_heads (per-head 1/sqrt(C/h), AK / CK / AV / CV copies, bo and +1 on head 0) followed by the
    per-segment softmax of stage T equals transformer_layer with num_heads in fp64."""
    B, C, D, k, p = 2, 64, 8, 7, 8
    w = ob.init_params(C, D, k, p, integration, False, seed=heads, bias_std=0.3)
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    y = torch.randn(B, k, D, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    ref, att, _ = ob.transformer_layer(x, y, w, integration=integration, norm=None, num_heads=heads, return_att=True)
    f = of.fold_weights(w, C=C, k=k, integration=integration, duplex=False, num_heads=heads)
    Kp, Vt, Rt, Ct = of.prologue(y, f, C=C, H=H, W=W, p=p, num_heads=heads)
    assert Kp.shape[1] == heads * of.head_segment(k, heads)
    X = x.reshape(B, C, H * W).transpose(1, 2)
    out = af.stage_t_forward(X, Kp, Vt, Rt, Ct, H=H, W=W, k=k, integration=integration, norm="none", heads=heads)
    assert torch.allclose(out["Xout"], ref.reshape(B, C, H * W).transpose(1, 2), rtol=1e-12, atol=1e-12)
    assert torch.allclose(out["att"], att.reshape(B, k, H * W).transpose(1, 2), rtol=1e-12, atol=1e-12)


def test_duplex_folds_match_direct():
    """Keys straight from Xbar (AK2, CK2) equal the keys of the centroids Xbar WV2 + bv2; the centroid query fold ACQ reproduces
    transformer_layer with carried-in centroids (centroids_init) in fp64."""
    B, C, D, k, p = 2, 32, 8, 5, 8
    w = ob.init_params(C, D, k, p, "mul", True, seed=3, bias_std=0.3, extras=True)
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    y = torch.randn(B, k, D, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    c0 = torch.randn(B, k, C, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    f = of.fold_weights(w, C=C, k=k, integration="mul", duplex=True)
    X = x.reshape(B, C, H * W).transpose(1, 2)
    xbar = torch.randn(B, k, C, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    assert torch.allclose(xbar @ f["AK2"] + f["CK2"], (xbar @ f["WV2"] + f["BV2"]) @ f["AK"] + f["CK"], rtol=1e-12, atol=1e-12)
    ref, _, cen_ref = ob.transformer_layer(x, y, w, integration="mul", norm="layer", duplex=True, centroids_init=c0)
    m_all = c0 @ f["ACQ"] + f["CM"][None]
    Rt2, Ct2 = of._pos_tables(m_all, C, p, H, W, of.pad_k(k), True)
    _, xb, _ = of.centroid_softmax(X, m_all[:, :, :C], Rt2, Ct2, k=k)
    cen = xb @ f["WV2"] + f["BV2"]
    assert torch.allclose(cen, cen_ref, rtol=1e-12, atol=1e-12)
    Kp, Vt, Rt, Ct = of.prologue(y, {**f, "AK": f["AK2"], "CK": f["CK2"]}, C=C, H=H, W=W, p=p, key_source=xb)
    out, _ = of.per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration="mul", norm="layer")
    assert torch.allclose(out, ref.reshape(B, C, H * W).transpose(1, 2), rtol=1e-12, atol=1e-12)


def test_single_head_folds_unchanged():
    """num_heads = 1 keeps the single-head layout and values (AK [D, C+p+4], CV [Cout])."""
    w = ob.init_params(64, 16, 5, 8, "both", False, seed=1, bias_std=0.2)
    f = of.fold_weights(w, C=64, k=5, integration="both", duplex=False)
    assert f["AK"].shape == (16, 76) and f["CV"].shape == (128,)
    assert torch.equal(f["CB"][:64], w["bo"][:64] + 1) and torch.equal(f["CB"][64:], w["bo"][64:])


# ---- the exact cases are exact -------------------------------------------------------------------------------------------------
def _agree(f_kernel, f_oracle, heads):
    """The kernel-order fold equals oracle/folded.py's (different order; both exact here)."""
    for name in ("AK", "CK", "AV", "CV"):
        got = f_kernel[name] if heads > 1 else f_kernel[name][0]
        assert torch.equal(got, f_oracle[name]), name


@pytest.mark.parametrize("heads,C,D,p,k,integration,in_scale", g.SIMPLEX, ids=_id)
def test_simplex_cases_exact(heads, C, D, p, k, integration, in_scale):
    w, y, d = g.simplex_case(heads, C, D, p, k, integration, in_scale)
    for tf32 in (False, True):
        want, f = g.simplex_expected(w, y, d, heads=heads, C=C, D=D, k=k, integration=integration, tf32=tf32)
    fo = of.fold_weights(w, C=C, k=k, integration=integration, duplex=False, num_heads=heads, use_pos=p > 0)
    _agree(f, fo, heads)
    Kp64, Vt64, Rt64, Ct64 = of.prologue(y, fo, C=C, H=H, W=W, p=p, num_heads=heads, use_pos=p > 0)
    fp32, _ = g.simplex_expected(w, y, d, heads=heads, C=C, D=D, k=k, integration=integration, tf32=False)
    dd = torch.ones(1, 1, C, dtype=torch.float64) if d is None else d[:, None, :]
    assert torch.equal(fp32["Kp"].double(), Kp64 * dd) and torch.equal(fp32["Vt"].double(), Vt64)
    assert torch.allclose(fp32["Rt"].double(), Rt64, rtol=2 ** -23, atol=0) and torch.allclose(fp32["Ct"].double(), Ct64, rtol=2 ** -23, atol=0)
    seg = of.head_segment(k, heads)
    pad = torch.tensor([J % seg >= k for J in range(fp32["Kp"].shape[1])])
    assert (fp32["Rt"][:, :, pad] == -math.inf).all() and (fp32["Rt"][:, :, ~pad] > -math.inf).all()
    if p:
        assert (fp32["Rt"][:, :, ~pad] != fp32["Rt"][:, :1, ~pad]).any(), "Rt does not depend on the row"


def test_vt_ties_pin_round_to_nearest_even():
    """In the default mode the exact V^T values include TF32 ties, and round-to-nearest-even differs from ties-away on some."""
    ties = 0
    for case in g.SIMPLEX:
        heads, C, D, p, k, integration, in_scale = case
        w, y, d = g.simplex_case(*case)
        f = sw.stage_w(w, C=C, D=D, k=k, integration=integration, heads=heads)
        _, v = sw.simplex_rows(f, y, heads=heads)
        v32 = v.float()
        ties += int((tf32_rne(v32) != tf32_rna(v32)).sum())
    assert ties > 0


@pytest.mark.parametrize("B,C,D,p,k", g.DUPLEX, ids=_id)
def test_duplex_key_cases_exact(B, C, D, p, k):
    """Both GEMM routes of the key path are exact; the tiles: B k rows (ragged), k = 13 not dividing 64, LDK columns."""
    w, y, cen = g.duplex_case(B, C, D, p, k)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    fo = of.fold_weights(w, C=C, k=k, integration="mul", duplex=True, use_pos=p > 0)
    for name in ("AK", "CK"):
        assert torch.equal(f[name][0], fo[name]), name
    for name in ("AK2", "CK2", "AM", "CM"):
        assert torch.equal(f[name], fo[name]), name
    for tc in (False, True):
        g.duplex_key_expected(f, cen, y, C=C, p=p, k=k, tc=tc)
    kp = sw.key_rows(cen, f["AK"][0], f["CK"][0], tc=True)
    assert (sw.significant_bits(f["AK"][0]) <= 11).all() and (sw.significant_bits(cen) <= 11).all()
    assert not torch.equal(kp, (cen @ f["AK"][0] + f["CK"][0]).float().double()), "the compensation is invisible"
    assert (B * k) % 64 and B * k > 64
    assert (C + p + 4 + 3) // 4 * 4 % 64


@pytest.mark.parametrize("B,C,D,p,k", [(3, 64, 16, 4, 13), (2, 256, 64, 16, 20)], ids=_id)
def test_duplex_xbar_cases_exact(B, C, D, p, k):
    """The Xbar route: fp32(x_w 1.000352220f) truncates to x_w, and AK2 / CK2 keys are exact."""
    w, y, _ = g.duplex_case(B, C, D, p, k)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    win = torch.randint(0, H * W, (B, k), generator=torch.Generator().manual_seed(C + k))
    tabs, _, _ = af.exact_pass_a_case(B, H, W, C, k, winners=win, seed=C + k)
    xw = tabs["X"][torch.arange(B)[:, None], win]
    xbar = xw.float() * torch.tensor(sw.COMP, dtype=torch.float32)
    assert torch.equal(tf32_trunc(xbar).double(), xw)
    g.duplex_key_expected(f, xw, y, C=C, p=p, k=k, tc=True, key="AK2")


@pytest.mark.parametrize("B,C,D,p,k", [(3, 64, 16, 4, 13), (2, 256, 64, 16, 27)], ids=_id)
def test_duplex_pass_a_cases_exact(B, C, D, p, k):
    w, y, cen = g.duplex_case(B, C, D, p, k, wcq=True)
    f = sw.stage_w(w, C=C, D=D, k=k, integration="mul", duplex=True)
    assert torch.equal(f["ACQ"], of.fold_weights(w, C=C, k=k, integration="mul", duplex=True)["ACQ"])
    for tc in (False, True):
        g.duplex_passa_expected(f, y, C=C, p=p, k=k, tc=tc)
        g.duplex_passa_expected(f, y, C=C, p=p, k=k, tc=tc, cen=cen)


def test_pos_tables_far_from_fp32_midpoints():
    """No fp64 sin / cos of the axis tables the exact cases use lies within 2^-40 (relative) of an fp32 rounding midpoint."""
    for length in (H, W):
        for half in (2, 8):
            assert sw.pos_midpoint_margin(length, half) > 2.0 ** -40, (length, half)


# ---- statistics ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", (132, 114, 78))
def test_norm_split_structure(sms):
    """The token counts the GPU test derives from the SM count: >= 3 splits, n divisible by neither the split count nor 8, and an
    empty last split where asked."""
    for B, empty in ((1, False), (3, False), (5, False), (1, True), (2, True)):
            n, ns = g.norm_n(sms, B, empty_last=empty)
            per = -(-n // ns)
            assert ns >= 3 and n % ns and n % 8 and ((ns - 1) * per >= n) == empty


@pytest.mark.parametrize("mode,B,C,empty_last", [("instance", 3, 96, False), ("batch", 1, 1024, False), ("batch", 2, 96, True)], ids=_id)
def test_norm_cases_exact(mode, B, C, empty_last):
    """Integer X: the fp64 sums are exact (checked by sw.norm_stats); the constant channel gives var = 0 and the 1000 channel a
    variance near 1 under a mean square of 10^6."""
    n, _ = g.norm_n(132, B, empty_last=empty_last)
    X = g.norm_x(B, n, C, seed=1)
    sc, sh = sw.norm_stats(X, mode == "batch")
    assert sc[0, 0] == torch.tensor(1.0 / math.sqrt(1e-8), dtype=torch.float32)
    assert abs(sc[0, 1].item() - 1.0) < 1e-3


def test_affine_case_statistics_are_powers_of_two():
    """m +- 2^14 (or 2^15), balanced: mean m and variance a^2 are exact, a^2 + 1e-8 rounds to a^2, rstd = 1/a, shift = -m/a."""
    for a in (2.0 ** 14, 2.0 ** 15):
        for m in (-50.0, 0.0, 37.0):
            X = torch.tensor([m + a, m - a] * 64, dtype=torch.float64).reshape(1, 128, 1)
            sc, sh = sw.norm_stats(X, False)
            assert sc.item() == 1.0 / a and sh.item() == -m / a
