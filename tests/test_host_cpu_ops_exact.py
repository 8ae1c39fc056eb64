"""CPU checks behind tests/test_gpu_ops_exact.py, and the alignment checks of the gf_ops.h entry points.

The GPU tests demand bit-for-bit equality on their exact cases (demodulation: 2 ulp).  That is only fair if every intermediate the
kernels form is an fp32 value in any order of summation.  These tests build each exact case on the host and check it, as
tests/test_host_cpu_attn_forward.py does for the attention kernels: every partial sum of an intermediate is a multiple of its grain
with a magnitude below 2^24 grains (the companion, the same sum of absolute values, bounds every partial sum), and a float32
restatement of the kernel's arithmetic equals the fp64 reference the GPU test compares with.

The alignment checks run the entry points in a child process that sees no GPU, with fake device pointers: an entry that lacked
the check would attempt a launch there and fail with a CUDA error instead of touching memory.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from tests import test_gpu_ops_exact as ex
from tests.test_host_cpu_attn_backward import _check_exact, _roundtrips

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = torch.float32, torch.float64
H100_SMEM_OPTIN = 232448                 # bytes of shared memory per block an H100 grants on opt-in (227 KB)


def _fir_items(x, pad, gain, scale):
    """Horizontal sums (grain 1/8), vertical sums (1/64) and the scaled output (min scale / 64) of the blur of integer x."""
    a = x.abs()
    y, c = ex._scaled(ex.blur(x, pad, gain), scale), ex._scaled(ex.blur(a, pad, gain), scale)
    smin = 1.0 if scale is None else scale.min().item()
    return [("h", ex.blur(x, pad, 1.0, hpass_only=True), ex.blur(a, pad, 1.0, hpass_only=True), 1 / 8),
            ("v", ex.blur(x, pad, 1.0), ex.blur(a, pad, 1.0), 1 / 64), ("y", y, c, smin / 64)]


def _check_fir(x, pad, gain, scale, want):
    assert (x.abs() <= 8).all() and torch.equal(x.round(), x)
    _check_exact(_fir_items(x, pad, gain, scale))
    s32 = None if scale is None else scale.float()
    assert torch.equal(ex._scaled(ex.blur(x.float(), pad, gain, dtype=F32), s32).double(), want)
    _roundtrips({"y": want})


@pytest.mark.parametrize("case", ex.FIR4_CASES, ids=ex.fir_id)
def test_fir4_cases_are_exact(case):
    pad, B, Hin, Win, C, gain = case
    x = ex.fir4_case(*case)
    _check_fir(x, pad, gain, None, ex.blur_def(x, pad, gain))


@pytest.mark.parametrize("case", ex.BLUR_UP_CASES, ids=ex.fir_id)
def test_blur_up_cases_are_exact(case):
    gain = case[-1]
    for scaled in (False, True):
        x, scale = ex.blur_up_case(*case, scaled)
        _check_fir(x, 1, gain, scale, ex._scaled(ex.blur_def(x, 1, gain), scale))


@pytest.mark.parametrize("case", ex.PHASE_CASES, ids=ex.fir_id)
def test_blur_up_phase_cases_are_exact(case):
    """The interleaved T has the shape the kernel assumes, [B, Hout+1, Wout+1, C], and its blur is exact."""
    B, Hout, Wout, C, gain = case
    for scaled in (False, True):
        ps, scale = ex.phase_case(*case, scaled)
        T = ex.interleave(ps)
        assert T.shape == (B, Hout + 1, Wout + 1, C)
        assert torch.equal(T[:, 1::2, 1::2], ps[3]) and torch.equal(T[:, 0::2, 1::2], ps[1])
        _check_fir(T, 1, gain, scale, ex._scaled(ex.blur_def(T, 1, gain), scale))


@pytest.mark.parametrize("pad", [0, 1, 2, 3])
def test_fir4_autograd_cases_are_exact(pad):
    """The forward, the pad-(3-p) first derivative and the pad-p second derivative are exact blurs, and fp64 autograd through the
    definition equals those blurs (the adjoint the native backward relies on)."""
    gain = float(pad + 1)
    ops = ex._ops()
    for B, C, H, W in ex.fir4_grad_shapes(pad):
        x, gy, v = ex.fir4_grad_case(pad, B, C, H, W)
        nhwc = lambda t: t.permute(0, 2, 3, 1)
        _check_exact(_fir_items(nhwc(x), pad, gain, None))
        _check_exact(_fir_items(nhwc(gy), 3 - pad, gain, None))
        _check_exact(_fir_items(nhwc(v), pad, gain, None))
        x64, gy64 = x.clone().requires_grad_(True), gy.clone().requires_grad_(True)
        y64 = ops.upfirdn2d_ref(x64, ops.fir_filter(dtype=F64), pad=(pad,) * 4, gain=gain)
        (gx64,) = torch.autograd.grad(y64, x64, gy64, create_graph=True)
        (ggy64,) = torch.autograd.grad(gx64, gy64, v)
        assert torch.equal(nhwc(gx64.detach()), ex.blur(nhwc(gy), 3 - pad, gain, dtype=F32).double())
        assert torch.equal(nhwc(ggy64), ex.blur(nhwc(v), pad, gain, dtype=F32).double())


def _upsample_restated(x, add, dtype):
    """gf_upsample2x_nchw's arithmetic: vertical taps 1/4, 3/4 on the zero-padded input, then horizontal, then + add."""
    q, t = torch.tensor(0.25, dtype=dtype), torch.tensor(0.75, dtype=dtype)
    xp = torch.nn.functional.pad(x.to(dtype), (1, 1, 1, 1))
    lo = q * xp[:, :, :-2] + t * xp[:, :, 1:-1]
    hi = t * xp[:, :, 1:-1] + q * xp[:, :, 2:]
    B, C, H, W2 = lo.shape
    y = torch.empty(B, C, 2 * H, 2 * (W2 - 2), dtype=dtype)
    for r, rows in ((lo, slice(0, None, 2)), (hi, slice(1, None, 2))):
        y[:, :, rows, 0::2] = q * r[..., :-2] + t * r[..., 1:-1]
        y[:, :, rows, 1::2] = t * r[..., 1:-1] + q * r[..., 2:]
    return y if add is None else y + add.to(dtype)


@pytest.mark.parametrize("case", ex.UPSAMPLE_CASES, ids=ex.fir_id)
def test_upsample_cases_are_exact(case):
    x, add = ex.upsample_case(*case)
    a = x.abs()
    ap = torch.nn.functional.pad(a, (1, 1, 1, 1))
    items = [("lo", _upsample_restated(x, None, F64), _upsample_restated(a, None, F64), 1 / 16),
             ("vertical", 0.25 * ap[:, :, :-2] + 0.75 * ap[:, :, 1:-1], 0.25 * ap[:, :, :-2] + 0.75 * ap[:, :, 1:-1], 1 / 4),
             ("y+add", ex.upsample_def(x, add), ex.upsample_def(a, add.abs()), 1 / 16)]
    _check_exact(items)
    for ad in (None, add):
        want = ex.upsample_def(x, ad)
        assert torch.equal(_upsample_restated(x, ad, F32).double(), want)
        _roundtrips({"y": want})


def test_bias_act_cases_are_exact():
    """Every pre-activation is a multiple of 5 (so 0.2f * v is exactly v / 5 in fp32), one is exactly 0, and the float32
    restatement x + (noise * st + bias), max(v, 0.2f * v), times gain equals the fp64 reference."""
    f02 = torch.tensor(0.2, dtype=F32)
    for B, HW, C in ex.BIAS_ACT_SHAPES:
        for mode in ex.NOISE_MODES:
            for with_bias in (False, True):
                for with_strength in (False, True):
                    x, bias, noise, st = ex.bias_act_case(B, HW, C, mode, with_bias, with_strength)
                    pre = ex.bias_act_pre(x, bias, noise, st)
                    comp = ex.bias_act_pre(x.abs(), None if bias is None else bias.abs(), None if noise is None else noise.abs(), st)
                    _check_exact([("pre", pre, comp, 5.0), ("act", ex.lrelu5(pre), comp, 1.0)])
                    assert pre[0, 0, 0] == 0 and (pre < 0).any() and (pre > 0).any()
                    v32 = ex.bias_act_pre(x.float(), None if bias is None else bias.float(), None if noise is None else noise.float(),
                                          torch.tensor(st, dtype=F32))
                    assert torch.equal(v32.double(), pre)
                    assert torch.equal(torch.maximum(v32, f02 * v32).double(), ex.lrelu5(pre))
                    _roundtrips({"lin": pre * 2, "lrelu": ex.lrelu5(pre) * 2})


def test_chan_scale_cases_are_exact():
    for case in ex.CHAN_SCALE_CASES:
        B, HW, C, s_ld, off = case
        assert off % 4 == 0 and off + C <= s_ld and s_ld % 4 == 0
        x, s_full = ex.chan_scale_case(*case)
        s = s_full[:, None, off:off + C]
        _check_exact([("y", x * s, (x * s).abs(), s.min().item())])
        assert torch.equal((x.float() * s.float()).double(), x * s)


@pytest.mark.parametrize("case", ex.TORGB_CASES, ids=ex.torgb_id)
def test_torgb_cases_are_exact(case):
    """The folded weights w * s * wscale, every product with x and every partial sum of the channel reduction (any order: the
    companion bounds them all) are multiples of min(s) * wscale, and the float32 restatement equals the fp64 reference."""
    C, HW, B = ex.resolve_torgb(case, ex.H100_SMS)
    for strided in (True, False):
        t = ex.torgb_case(C, HW, B, strided)
        x, w, s = t["x"], t["w"], t["st"][:, :C]
        grain = s.min().item() * ex.TORGB_WSCALE
        wr = w[None] * s[:, None] * ex.TORGB_WSCALE                                   # [B, 3, C]
        want = ex.torgb_def(x, w, s, ex.TORGB_WSCALE, t["bias"])
        comp = ex.torgb_def(x.abs(), w.abs(), s, ex.TORGB_WSCALE, None if t["bias"] is None else t["bias"].abs())
        _check_exact([("wr", wr, wr.abs(), grain), ("y", want, comp, grain)])
        got32 = ex.torgb_def(x.float(), w.float(), s.float(), torch.tensor(ex.TORGB_WSCALE, dtype=F32),
                             None if t["bias"] is None else t["bias"].float())
        assert torch.equal(got32.double(), want)
        _roundtrips({"y": want, "xs": x * t["s2"][:, None, :C]})


def _bits_apart(a, b):
    return (a.float().view(torch.int32).long() - b.float().view(torch.int32).long()).abs()


def test_demod_cases_are_exact_and_a_wrong_term_shows():
    """Every term s^2 wsq is a positive integer and the sum is below 2^24, so it is exact in any order; f32(sum + 1e-8) = sum.
    Dropping or doubling the smallest term moves float32(1/sqrt(sum)) by more than 4 ulp, twice the tolerance."""
    cases = [(B, O, I, ex._seed(B, O, I)) for B, O, I in ex.DEMOD_SHAPES] + ex.demod_batch_jobs()
    assert len(ex.demod_batch_jobs()) == 32
    for B, O, I, seed in cases:
        st, wsq = ex.demod_case(B, O, I, seed)
        terms = st[:, None, :I].square() * wsq[None]                                  # [B, O, I]
        total = ex.demod_sum(st, wsq)
        assert (terms >= 1).all() and torch.equal(terms.round(), terms)
        _check_exact([("sum", total, total, 1.0)])
        t32 = total.float()
        assert torch.equal(t32 + torch.tensor(ex.DEMOD_EPS, dtype=F32), t32)
        d = ex.demod_want(st, wsq)
        tmin = terms.min(dim=2).values
        for moved in (total - tmin, total + tmin):
            alt = torch.where(moved > 0, 1.0 / moved.clamp_min(1e-300).sqrt(), torch.full_like(moved, math.inf))
            assert (_bits_apart(alt, d) > 4).all(), (B, O, I)


@pytest.mark.parametrize("case", ex.MAPPING_CASES, ids=ex.mapping_id)
def test_mapping_cases_are_exact(case):
    """Every pre-activation a multiple of 5 below 2^24 * 5, every activation an integer, the lerp at psi = 1/2 a multiple of 1/2;
    the float32 restatement (pixel norm 1, max(v, 0.2f * v)) equals the fp64 reference."""
    D, L, k = case
    B = ex.mapping_batch(k, ex.H100_SMS)
    z, W, b, w_avg = ex.mapping_case(D, L, k, B)
    assert set(z.unique().tolist()) == {-1.0, 1.0}
    assert ((W != 0).sum(dim=2) == (2 if L <= 2 else 1)).all() and set(W.abs().unique().tolist()) == {0.0, 5.0}
    items = []
    for path, sl in ((0, slice(0, k)), (1, slice(k, k + 1))):
        h, c = z[:, sl], z[:, sl].abs()
        for l in range(L):
            pre, c = h @ W[path, l] + b[path, l], c @ W[path, l].abs() + b[path, l].abs()
            h = ex.lrelu5(pre)
            items += [(f"pre p{path} l{l}", pre, c, 5.0), (f"act p{path} l{l}", h, c, 1.0)]
        a = w_avg[path]
        items += [(f"lerp diff p{path}", h - a, c + a.abs(), 1.0),
                  (f"lerp p{path}", a + ex.MAPPING_PSI * (h - a), a.abs() + ex.MAPPING_PSI * (c + a.abs()), 0.5)]
    _check_exact(items)
    f02 = torch.tensor(0.2, dtype=F32)
    for avg in (w_avg, None):
        want = ex.mapping_want(z, W, b, avg, k)
        got32 = ex.mapping_def(z.float(), W.float(), b.float(), None if avg is None else avg.float(), ex.MAPPING_PSI, k,
                               exact_norm=True, lrelu=lambda v: torch.maximum(v, f02 * v))
        assert torch.equal(got32.double(), want)
        _roundtrips({"out": want})
    # the pixel norm of a +-1 latent in fp32: mean 1, 1 + 1e-8 rounds to 1
    assert (torch.tensor(float(D), dtype=F32) / D + torch.tensor(1e-8, dtype=F32)).item() == 1.0


def test_exact_cases_reach_the_edges_they_claim():
    """The case lists cover what the GPU file's docstrings say, at the H100's 132 SMs."""
    fir_shapes = [(pad, B, Hin + 2 * pad - 3, Win + 2 * pad - 3, C) for pad, B, Hin, Win, C, _ in ex.FIR4_CASES]
    assert {p for p, *_ in fir_shapes} == {0, 1, 2, 3} and {c[-1] for c in ex.FIR4_CASES} >= {1, 2, 3, 4}
    assert any(Ho % 8 and Ho > 8 for _, _, Ho, _, _ in fir_shapes)
    assert any(Wo * C // 4 > 256 and (Wo * C // 4) % 256 for _, _, _, Wo, C in fir_shapes)
    assert {C for *_, C in fir_shapes} >= {4, 12, 36, 512}
    assert (0, 2, 4, 4, 4, 1) in ex.FIR4_CASES and any(c[0] == 3 and c[2] == 1 for c in ex.FIR4_CASES)
    assert any(c[1] == 65535 for c in ex.FIR4_CASES) and any(c[0] == 65535 for c in ex.BLUR_UP_CASES + ex.PHASE_CASES)
    assert any((Wo // 2) * C // 4 > 256 and ((Wo // 2) * C // 4) % 256 for _, _, Wo, C, _ in ex.PHASE_CASES)
    toks = {ex.tok_per_cta(HW, ex.resolve_torgb((C, HW, B), ex.H100_SMS)[2], ex.H100_SMS) for C, HW, B in ex.TORGB_CASES}
    assert toks == {256, 512, 1024}
    assert sorted({-(-(C // 4) // 32) for C in ex.TORGB_C}) == [1, 2, 3, 4]
    assert {I for *_, I in ex.DEMOD_SHAPES} == {1, 31, 512, 513, 1100} and all(O % 8 for _, O, _ in ex.DEMOD_SHAPES)
    for D, L, k in ex.MAPPING_CASES:
        assert ex.mapping_batch(k, ex.H100_SMS) * (k + 1) > 2 * 8 * ex.H100_SMS
        assert (2 * L * D * D + 2 * L * D + 8 * D) * 4 <= H100_SMEM_OPTIN, (D, L)
    assert (2 * 8 * 64 * 64 + 2 * 8 * 64 + 8 * 64) * 4 > H100_SMEM_OPTIN                 # the rejected case
    assert {k for *_, k in ex.MAPPING_CASES} == {0, 1, 31}


# ------------------------------------------------------------------------------------------------ alignment checks
_ALIGN_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A = 0x10000
calls = {   # valid shapes; A is 16-byte aligned; the float4 operand positions come from the parent
    "gf_chan_scale_nhwc": [A, A, 4, A, 1, 4, 4, None],
    "gf_blur_up_nhwc": [A, A, A, 1, 4, 4, 4, 4.0, None],
    "gf_blur_up_phases_nhwc": [A, A, A, A, A, A, 1, 4, 4, 4, 4.0, None],
    "gf_fir4_nhwc": [A, A, 1, 5, 5, 4, 1, 1.0, None],
    "gf_bias_act_nhwc": [A, A, A, A, A, 0, 1, 4, 4, 1, 2.0, None],
    "gf_torgb_scale_nhwc": [A, A, A, 4, A, 1.0, A, A, 4, A, 1, 4, 4, None],
}
slots = json.loads(sys.argv[2])
out = {}
for name, args in calls.items():
    fn = getattr(lib, name)
    res = [[None, fn(*args), lib.gf_last_error().decode()]]
    for s in slots[name]:
        for off in (4, 8, 12):
            a = list(args)
            a[s] = A + off
            res.append([s, fn(*a), lib.gf_last_error().decode()])
    out[name] = res
print(json.dumps(out))
"""


def test_float4_operands_are_checked_for_alignment():
    """Each entry point of include/gf_ops.h that moves float4s returns GF_ERR_INVALID with a "16-byte aligned" message for every
    float4 operand 4, 8 or 12 bytes off, before it touches the device.  The child sees no GPU: with every pointer aligned the same
    call gets as far as the launch and fails there with GF_ERR_CUDA."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _ALIGN_CHILD, ROOT, json.dumps(ex.FLOAT4_OPERANDS)], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    assert sorted(out) == sorted(ex.FLOAT4_OPERANDS)
    for name, results in out.items():
        (_, rc, msg), rest = results[0], results[1:]
        assert rc == -3, f"{name}: the aligned call should fail at the launch (no device), got {rc}: {msg}"
        assert len(rest) == 3 * len(ex.FLOAT4_OPERANDS[name])
        for slot, rc, msg in rest:
            assert rc == -1 and "16-byte aligned" in msg, f"{name}: operand {slot} misaligned gave {rc}: {msg}"
