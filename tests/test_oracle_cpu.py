"""CPU tests of the oracle itself: golden vectors, folded-vs-direct algebra, algebraic properties (SURVEY section 4).

PARITY UNPINNED: the reference ships no tests/fixtures (and no source) for this path; these pins are ours.
"""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import bipartite as ob
from oracle import folded as of
from tests.golden import make_golden as mg

GOLD = os.path.join(os.path.dirname(__file__), "golden", "attn_cases.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _run_case(c, seed, dtype=torch.float64):
    x, y, w = mg.make_inputs(c, seed)
    norm = None if c["norm"] == "none" else c["norm"]
    x, y = x.to(dtype), y.to(dtype)
    w = {k: v.to(dtype) for k, v in w.items()}
    return ob.transformer_layer(x, y, w, integration=c["integration"], norm=norm, duplex=c["duplex"],
                                use_pos=c["use_pos"], return_att=True, kmeans_iters=c.get("kmeans_iters", 1), img2ltnt=bool(c.get("img2ltnt")),
                                num_heads=c.get("num_heads", 1))


@pytest.mark.parametrize("idx", range(len(mg.cases())))
def test_oracle_matches_golden(gold, idx):
    c = mg.cases()[idx]
    out, att, cen = _run_case(c, 100 + idx)
    name = mg.case_name(c)
    flat = out.permute(0, 2, 3, 1).contiguous().numpy().reshape(-1)
    np.testing.assert_allclose(flat[mg.out_sample_index(flat.size)], gold[name + "/out"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(att.numpy(), gold[name + "/att"], rtol=2e-6, atol=1e-7)
    if cen is not None:
        np.testing.assert_allclose(cen.numpy(), gold[name + "/cen"], rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("idx", [0, 5, 12, 15, 19])
def test_oracle_fp32_close_to_fp64(gold, idx):
    """e_ref of SURVEY 8c: the fp32 oracle (reference-Python-path stand-in) against fp64 truth."""
    c = mg.cases()[idx]
    out32, _, _ = _run_case(c, 100 + idx, torch.float32)
    ref = torch.from_numpy(gold[mg.case_name(c) + "/out"]).double()
    flat = out32.permute(0, 2, 3, 1).contiguous().double().reshape(-1)
    err = (flat[torch.from_numpy(mg.out_sample_index(flat.numel()))] - ref).abs()
    assert (err <= 2e-5 + 2e-4 * ref.abs()).all(), err.max()


@pytest.mark.parametrize("integration,norm,duplex,k,use_pos",
                         list(itertools.product(["mul", "add", "both"], ["layer", "instance", "batch", None],
                                                [False, True], [3, 16], [True, False])))
def test_folded_equals_direct(integration, norm, duplex, k, use_pos):
    """The three-stage folded form (what the CUDA kernels implement) is exact algebra of the direct form."""
    torch.manual_seed(1)
    B, C, H, W, D, p = 2, 32, 4, 8, 8, 8
    w = ob.init_params(C, D, k, p, integration, duplex, seed=1, bias_std=0.5)
    x = torch.randn(B, C, H, W, dtype=torch.float64)
    y = torch.randn(B, k, D, dtype=torch.float64)
    o, att, cen = ob.transformer_layer(x, y, w, integration=integration, norm=norm, duplex=duplex, use_pos=use_pos, return_att=True)
    o2, att2, cen2 = of.transformer_layer_folded(x.permute(0, 2, 3, 1).contiguous(), y, w, integration=integration, norm=norm,
                                                 duplex=duplex, use_pos=use_pos, return_att=True)
    assert (o.permute(0, 2, 3, 1) - o2).abs().max() < 1e-9
    assert (att - att2).abs().max() < 1e-10
    if duplex:
        assert (cen - cen2).abs().max() < 1e-10


def _simple(k=4, duplex=False, integration="mul", seed=3, B=3):
    C, H, W, D, p = 32, 4, 4, 8, 8
    g = torch.Generator().manual_seed(seed)
    w = ob.init_params(C, D, k, p, integration, duplex, seed=seed, bias_std=0.3)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    return x, y, w


def test_attention_rows_sum_to_one():
    x, y, w = _simple()
    _, att, _ = ob.transformer_layer(x, y, w, return_att=True)
    assert torch.allclose(att.sum(dim=1), torch.ones_like(att.sum(dim=1)), atol=1e-12)
    assert (att >= 0).all()


def test_single_latent_gives_uniform_modulation():
    """k = 1: softmax over one latent is 1, so the gain is the same vector for every grid cell."""
    x, y, w = _simple(k=1)
    out, att, _ = ob.transformer_layer(x, y, w, return_att=True)
    assert torch.allclose(att, torch.ones_like(att))
    B, C, H, W = x.shape
    X = x.reshape(B, C, -1).permute(0, 2, 1)
    gain = out.reshape(B, C, -1).permute(0, 2, 1) / ob.att_norm(X, "layer")
    assert (gain - gain[:, :1]).abs().max() < 1e-8


def test_latent_permutation_equivariance():
    """Permuting the latents together with their positional embeddings leaves x' unchanged and permutes att."""
    x, y, w = _simple(k=5)
    perm = torch.tensor([3, 0, 4, 1, 2])
    out, att, _ = ob.transformer_layer(x, y, w, return_att=True)
    w2 = dict(w)
    w2["pos_latent"] = w["pos_latent"][perm]
    out2, att2, _ = ob.transformer_layer(x, y[:, perm], w2, return_att=True)
    assert (out - out2).abs().max() < 1e-10
    assert (att[:, perm] - att2).abs().max() < 1e-12


@pytest.mark.parametrize("duplex", [False, True])
def test_batch_independence(duplex):
    """Every image is independent through the block (the basis of the data-parallel sharding, SURVEY 8e)."""
    x, y, w = _simple(k=4, duplex=duplex)
    out, _, _ = ob.transformer_layer(x, y, w, duplex=duplex)
    out1, _, _ = ob.transformer_layer(x[1:2], y[1:2], w, duplex=duplex)
    assert (out[1:2] - out1).abs().max() < 1e-10


def test_positional_table_is_separable():
    t = ob.grid_pos_table(4, 8, 8)
    assert t.shape == (32, 8)
    row, col = ob.sinusoidal_axis(4, 4), ob.sinusoidal_axis(8, 4)
    assert torch.equal(t.reshape(4, 8, 8)[2, 5], torch.cat([row[2], col[5]]))


def test_philox_oracle_matches_random123_known_answers():
    """oracle/philox.py against the published Philox4x32-10 known-answer vectors (Random123 kat_vectors) -- the one part of the
    oracle a third party pins; the GPU suite then checks the kernels' mask against this oracle bit for bit."""
    from oracle import philox as ph
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(int(x) for x in ph.philox4x32_10(*ctr, *key)) == want
    m = ph.dropout_mult(0.25, seed=1234567890123, step=7, salt=5, tokens=4096, KP=16)
    assert m.shape == (4096, 16) and set(np.unique(m).tolist()) == {0.0, float(np.float32(1.0) / np.float32(0.75))}
    keep = (m > 0).mean()
    assert abs(keep - 0.75) < 4 * (0.25 * 0.75 / m.size) ** 0.5 + 1e-3
    assert not np.array_equal(m, ph.dropout_mult(0.25, seed=1234567890123, step=8, salt=5, tokens=4096, KP=16))     # next step: new mask
    assert not np.array_equal(m, ph.dropout_mult(0.25, seed=1234567890123, step=7, salt=6, tokens=4096, KP=16))     # another layer


def test_attention_dropout_algebra_of_the_oracle():
    """att_mult: an all-ones mask is the plain layer; an all-zero mask leaves only the un-droppable constants -- the output then does
    not depend on the latents' values (what the kernels re-add as (1 - sum q) * cb)."""
    C, D, k, p = 32, 16, 4, 16
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, C, 8, 8, generator=g, dtype=torch.float64)
    y = torch.randn(2, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, "mul", False, seed=2, bias_std=0.3)
    ref, _, _ = ob.transformer_layer(x, y, w, integration="mul")
    ones = torch.ones(2, 64, k, dtype=torch.float64)
    out1, _, _ = ob.transformer_layer(x, y, w, integration="mul", att_mult=ones)
    assert torch.allclose(out1, ref, atol=1e-12)
    zeros = torch.zeros(2, 64, k, dtype=torch.float64)
    out0a, _, _ = ob.transformer_layer(x, y, w, integration="mul", att_mult=zeros)
    out0b, _, _ = ob.transformer_layer(x, y + 3.0, w, integration="mul", att_mult=zeros)
    assert torch.allclose(out0a, out0b, atol=1e-12) and not torch.allclose(out0a, ref, atol=1e-3)


def _f32(bits):
    return torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in bits], dtype=torch.int32).view(torch.float32)


def _u32(x):
    return [b & 0xFFFFFFFF for b in x.view(torch.int32).tolist()]


def test_tf32_helpers_on_hand_picked_bit_patterns():
    """oracle/tf32.py: truncation (what the tensor core does to a streamed float32 operand) and round-to-nearest-even (what the
    library does before an operand reaches the tensor core), on ties, signs, carries into the exponent and signed zeros."""
    from oracle.tf32 import tf32_rne, tf32_trunc
    cases = [  # bits in, truncated, rounded to nearest even
        (0x3F800000, 0x3F800000, 0x3F800000),   # 1.0 is a TF32 value
        (0x3F801800, 0x3F800000, 0x3F802000),   # 1 + 3 * 2^-12: below halfway drops, above halfway rounds up
        (0x3F801000, 0x3F800000, 0x3F800000),   # exact tie, even kept bit: stays
        (0x3F803000, 0x3F802000, 0x3F804000),   # exact tie, odd kept bit: rounds up to even
        (0x3F800FFF, 0x3F800000, 0x3F800000),   # just below a tie
        (0x3F801001, 0x3F800000, 0x3F802000),   # just above a tie
        (0xBF803000, 0xBF802000, 0xBF804000),   # negative: both act on the magnitude, the sign stays
        (0xBF801000, 0xBF800000, 0xBF800000),   # negative exact tie, even kept bit
        (0xBF801800, 0xBF800000, 0xBF802000),   # -(1 + 3 * 2^-12)
        (0x3FFFF000, 0x3FFFE000, 0x40000000),   # tie on an all-ones kept mantissa: carries into the exponent, 2.0
        (0x3FFFFFFF, 0x3FFFE000, 0x40000000),
        (0xC07FFFFF, 0xC07FE000, 0xC0800000),   # the same carry, negative: -4.0
        (0x00000000, 0x00000000, 0x00000000),   # +0
        (0x80000000, 0x80000000, 0x80000000),   # -0 keeps its sign
        (0x00001000, 0x00000000, 0x00000000),   # subnormal tie, even kept bit
        (0x00003000, 0x00002000, 0x00004000),   # subnormal tie, odd kept bit
        (0x807FFFFF, 0x807FE000, 0x80800000),   # largest negative subnormal carries into the smallest normal
        (0x7F7FFFFF, 0x7F7FE000, 0x7F800000),   # largest finite float rounds to +inf, as the bit trick on the GPU does
    ]
    x = _f32([c[0] for c in cases])
    assert _u32(tf32_trunc(x)) == [c[1] for c in cases]
    assert _u32(tf32_rne(x)) == [c[2] for c in cases]
    assert x.view(torch.int32).tolist() == _f32([c[0] for c in cases]).view(torch.int32).tolist()    # inputs untouched


def test_tf32_helpers_match_an_arithmetic_definition():
    """On random normal values of many magnitudes: rounding x / ulp to an integer, where ulp = 2^(exponent - 10), with numpy's
    half-to-even rounding or toward zero, gives the same values as the bit tricks.  Shapes are kept; results are TF32 values."""
    from oracle.tf32 import tf32_low_bits, tf32_rne, tf32_trunc
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, 1000, generator=g) * torch.pow(2.0, torch.randint(-60, 60, (4, 1000), generator=g).float())
    ties = (x.view(torch.int32) & -0x2000) | 0x1000                                        # every kept-bit parity, exact ties
    for v in (x, ties.view(torch.float32)):
        x64 = v.double().numpy()
        ulp = np.exp2(np.floor(np.log2(np.abs(x64))) - 10)
        assert np.array_equal(tf32_rne(v).double().numpy(), np.round(x64 / ulp) * ulp)
        assert np.array_equal(tf32_trunc(v).double().numpy(), np.trunc(x64 / ulp) * ulp)
        assert tf32_rne(v).shape == v.shape
        assert (tf32_low_bits(tf32_rne(v)) == 0).all() and (tf32_low_bits(tf32_trunc(v)) == 0).all()
    with pytest.raises(TypeError):
        tf32_rne(torch.ones(3, dtype=torch.float64))


def test_tf32_rna_rounds_ties_away_from_zero():
    """tf32_rna (what cvt.rna.tf32.f32 does to the attention probabilities): nearest, ties away from zero whatever the kept bit,
    on hand-picked patterns and against the arithmetic definition; it differs from tf32_rne only on ties with an even kept bit."""
    from oracle.tf32 import tf32_low_bits, tf32_rna, tf32_rne
    cases = [  # bits in, rounded to nearest with ties away from zero
        (0x3F800000, 0x3F800000),
        (0x3F801000, 0x3F802000),   # exact tie, even kept bit: away from zero (rne stays)
        (0x3F803000, 0x3F804000),   # exact tie, odd kept bit: away from zero (as rne)
        (0x3F800FFF, 0x3F800000),
        (0x3F801001, 0x3F802000),
        (0xBF801000, 0xBF802000),   # negative tie: away from zero, i.e. more negative
        (0x3FFFF000, 0x40000000),   # carry into the exponent
        (0x00001000, 0x00002000),   # subnormal tie
        (0x80000000, 0x80000000),
    ]
    x = _f32([c[0] for c in cases])
    assert _u32(tf32_rna(x)) == [c[1] for c in cases]
    g = torch.Generator().manual_seed(6)
    v = torch.randn(4, 1000, generator=g) * torch.pow(2.0, torch.randint(-60, 60, (4, 1000), generator=g).float())
    ties = ((v.view(torch.int32) & -0x2000) | 0x1000).view(torch.float32)
    for t in (v, ties):
        x64 = t.double().numpy()
        ulp = np.exp2(np.floor(np.log2(np.abs(x64))) - 10)
        want = np.sign(x64) * np.floor(np.abs(x64) / ulp + 0.5) * ulp
        assert np.array_equal(tf32_rna(t).double().numpy(), want)
        assert (tf32_low_bits(tf32_rna(t)) == 0).all()
    differ = tf32_rna(ties) != tf32_rne(ties)
    assert torch.equal(differ, ((ties.view(torch.int32) >> 13) & 1) == 0)
