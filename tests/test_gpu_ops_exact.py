"""GPU tests of the streaming kernels of csrc/gf_ops.cu, called through the C ABI (run on an H100: ``pytest -m gpu``).

These kernels (FIR blurs, skip upsampling, bias + noise + activation, channel scaling, tRGB, demodulation coefficients and the
mapping network) run in every generator forward.  Each can compute every output exactly when its inputs are chosen for it: the
FIR taps are 1/8 and 3/8, the upsampling taps 1/4 and 3/4, gains and weight scales are ABI arguments, and 0.2f * 5k == k in fp32.
So the exact cases below use small integers, multiples of 5 and powers of two, and demand bit-for-bit equality with an fp64
restatement (demodulation: within 2 ulp of float32(1/sqrt(sum)), the accuracy the CUDA guide states for rsqrtf).
tests/test_host_cpu_ops_exact.py proves on the host that each case is exact: every partial sum is a multiple of its grain below
2^24 grains, and a float32 restatement equals the fp64 reference.

Every output sits between the NaN guards of tests/guards.py; the tests check that the guards are intact and that every element
was written.  One realistic-data case per kernel is held per element to a frozen multiple of fp32 round-off of its magnitude
companion (the same expression on absolute values).  The wrappers in ops.py are checked to hand every float4 operand over
16-byte aligned, with the library replaced by a recorder that launches nothing.
"""
import ctypes
import math
from importlib import import_module

import pytest
import torch

from tests.guards import Guarded, assert_exact

pytestmark = pytest.mark.gpu

F64 = torch.float64
H100_SMS = 132                   # SM count of the H100 SXM; the host proofs size the SM-dependent batches with it
# Realistic-data bounds: max over elements of |y - y64| / companion, the companion being the same expression on absolute values.
# Measured worst case on an H100 80GB HBM3 at a 700 W power limit: fir4 1.56e-7, blur_up 1.58e-7, blur_up_phases 1.60e-7,
# upsample2x 1.71e-7, bias_act 1.56e-7, chan_scale 5.96e-8 (one rounding), torgb 4.15e-8, demod 1.42e-7, mapping 2.33e-7 (fir4,
# blur_up, chan_scale, demod and mapping measured the same at 400 W); frozen with a margin of at least 1.5x.
REL_BOUND = {
    "fir4": 2.5e-7, "blur_up": 2.5e-7, "blur_up_phases": 2.5e-7, "upsample2x": 3e-7, "bias_act": 2.5e-7, "chan_scale": 9e-8,
    "torgb": 7e-8, "demod": 2.5e-7, "mapping": 4e-7,
}


def _ops():
    return import_module("gansformer-reproducibility-challenge_b200.ops")


def _seed(*vals):
    s = 17
    for v in vals:
        s = (s * 1000003 + int(v)) % (2 ** 31 - 1)
    return s


def ints(shape, lo, hi, seed):
    """Integers in [lo, hi] as float64 (CPU, reproducible on the host)."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=torch.Generator().manual_seed(seed)).to(F64)


def pow2(shape, lo, hi, seed):
    return 2.0 ** ints(shape, lo, hi, seed)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _call(gf, name, *args):
    gf._lib.check(getattr(gf._lib.load(), name)(*args), name)
    torch.cuda.synchronize()


def _dev(t, dev):
    return None if t is None else t.float().contiguous().to(dev)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ references (any dtype)
def fir1d(dtype):
    return torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=dtype) / 8


def blur(x, pad, gain, dtype=F64, hpass_only=False):
    """The separable [1,3,3,1]/8 blur of x [B,H,W,C] with zero padding `pad`, times gain: [B,H+2p-3,W+2p-3,C] (with hpass_only,
    the horizontal pass on the padded rows, unscaled).  In float32 a restatement of the kernel's arithmetic; in fp64 the definition."""
    f = fir1d(dtype)
    x = torch.nn.functional.pad(x.to(dtype), (0, 0, pad, pad, pad, pad))
    Wo = x.shape[2] - 3
    h = f[0] * x[:, :, 0:Wo] + f[1] * x[:, :, 1:Wo + 1] + f[2] * x[:, :, 2:Wo + 2] + f[3] * x[:, :, 3:Wo + 3]
    if hpass_only:
        return h
    Ho = h.shape[1] - 3
    v = f[0] * (h[:, 0:Ho] + h[:, 3:Ho + 3]) + f[1] * (h[:, 1:Ho + 1] + h[:, 2:Ho + 2])
    return v * torch.tensor(gain, dtype=dtype)


def blur_def(x, pad, gain):
    """The definition: ops.upfirdn2d_ref with the 2-D [1,3,3,1]^2/64 filter, fp64, x [B,H,W,C]."""
    ops = _ops()
    y = ops.upfirdn2d_ref(x.to(F64).permute(0, 3, 1, 2), ops.fir_filter(dtype=F64), pad=(pad,) * 4, gain=gain)
    return y.permute(0, 2, 3, 1)


def interleave(ps):
    """The four polyphase components -> T [B, 2H+1, 2W+1, C], T[2i+a, 2j+b] = p_ab[i, j]."""
    p00, p01, p10, p11 = ps
    B, H1, W1, C = p00.shape
    T = torch.zeros(B, 2 * H1 - 1, 2 * W1 - 1, C, dtype=p00.dtype)
    T[:, 0::2, 0::2], T[:, 0::2, 1::2], T[:, 1::2, 0::2], T[:, 1::2, 1::2] = p00, p01, p10, p11
    return T


def upsample_def(x, add=None):
    ops = _ops()
    y = ops.upfirdn2d_ref(x.to(F64), ops.fir_filter(dtype=F64), up=2, pad=(2, 1, 2, 1), gain=4.0)
    return y if add is None else y + add


def lrelu5(v):
    """Leaky-ReLU(0.2) of values whose negative entries are multiples of 5 (exact: v / 5)."""
    return torch.where(v < 0, v / 5, v)


def bias_act_pre(x, bias, noise, st):
    """x [B,HW,C] + (noise [B or 1, HW] * st + bias [C]), in the kernel's order."""
    add = torch.zeros_like(x)
    if noise is not None:
        add = add + (noise * st)[:, :, None]
    if bias is not None:
        add = add + bias
    return x + add


def torgb_def(x, w, styles, wscale, bias):
    """y [B,3,HW] = sum_c x[b,t,c] w[o,c] styles[b,c] wscale + bias[o]."""
    y = torch.einsum("btc,oc,bc->bot", x, w, styles) * wscale
    return y if bias is None else y + bias[None, :, None]


def mapping_def(z, W, b, w_avg, psi, k, *, exact_norm, lrelu=None):
    """G_mapping on z [B, k+1, D] with effective weights W [2, L, D, D] ([in][out]) and biases b [2, L, D]; path 1 for the last
    latent of every sample.  exact_norm: the pixel norm is taken as 1 (z entries +-1: rsqrtf(f32(1 + 1e-8)) = 1)."""
    D = z.shape[-1]
    x = z if exact_norm else z / torch.sqrt(z.square().mean(dim=-1, keepdim=True) + 1e-8)
    act = lrelu or (lambda v: torch.nn.functional.leaky_relu(v, 0.2))
    outs = []
    for path, sl in ((0, slice(0, k)), (1, slice(k, k + 1))):
        h = x[:, sl]
        for l in range(W.shape[1]):
            h = act(h @ W[path, l] + b[path, l])
        if w_avg is not None:
            h = w_avg[path] + psi * (h - w_avg[path])
        outs.append(h)
    return torch.cat(outs, dim=1).reshape(z.shape[0], k + 1, D)


# ------------------------------------------------------------------------------------------------ case builders (CPU)
# gf_fir4_nhwc: (pad, B, Hin, Win, C, gain).  Rows are 8-row blocks, columns blocks of 256 threads of 4 channels.
FIR4_CASES = [
    (0, 2, 4, 4, 4, 1),          # the smallest input pad 0 accepts: one output pixel
    (0, 3, 12, 67, 36, 2),       # Hout 9 (one block + 1 row); Wout * C/4 = 576: three column blocks, the last partial
    (0, 2, 19, 70, 12, 3),       # Hout 16, Wout 67
    (1, 2, 12, 101, 12, 3),      # Hout 11; Wout * C/4 = 300
    (1, 1, 10, 4, 512, 4),       # C = 512: Wout * C/4 = 384
    (1, 2, 2, 2, 4, 1),          # the smallest input pad 1 accepts
    (2, 3, 1, 1, 4, 4),          # 1x1 input
    (2, 2, 1, 37, 36, 1),        # 1xN input; Wout * C/4 = 342
    (3, 2, 1, 1, 12, 2),         # the smallest input pad 3 accepts
    (3, 1, 1, 70, 4, 3),         # 1xN input
    (3, 2, 17, 9, 36, 4),        # Hout 20, Wout 12
    (0, 65535, 4, 5, 4, 1),      # B at the grid-z limit, tiny images
    (2, 65535, 1, 1, 4, 2),
]
# gf_blur_up_nhwc: (B, Hout, Wout, C, gain); x is [B, Hout+1, Wout+1, C]
BLUR_UP_CASES = [(2, 11, 100, 12, 4), (3, 1, 1, 4, 1), (1, 9, 3, 512, 2), (2, 16, 64, 36, 3), (2, 1, 70, 4, 4), (65535, 1, 2, 4, 4)]
# gf_blur_up_phases_nhwc: (B, Hout, Wout, C, gain); the column blocks are over Wout/2 * C/4 output pairs
PHASE_CASES = [(2, 10, 64, 36, 4), (3, 2, 2, 4, 1), (1, 18, 6, 512, 2), (2, 2, 70, 12, 3), (3, 6, 4, 4, 4), (65535, 2, 2, 4, 4)]


def fir_id(c):
    return "x".join(str(v) for v in c)


def fir4_case(pad, B, Hin, Win, C, gain):
    return ints((B, Hin, Win, C), -8, 8, _seed(pad, B, Hin, Win, C, gain))


def blur_up_case(B, Hout, Wout, C, gain, scaled):
    s = _seed(B, Hout, Wout, C, gain)
    x = ints((B, Hout + 1, Wout + 1, C), -8, 8, s)
    return x, (pow2((B, C), -3, 3, s + 1) if scaled else None)


def phase_case(B, Hout, Wout, C, gain, scaled):
    H, W = Hout // 2, Wout // 2
    s = _seed(B, Hout, Wout, C, gain, 7)
    shapes = [(B, H + 1, W + 1, C), (B, H + 1, W, C), (B, H, W + 1, C), (B, H, W, C)]
    ps = [ints(sh, -8, 8, s + i) for i, sh in enumerate(shapes)]
    return ps, (pow2((B, C), -3, 3, s + 9) if scaled else None)


def _scaled(y, scale):
    return y if scale is None else y * scale[:, None, None, :]


@pytest.mark.parametrize("case", FIR4_CASES, ids=fir_id)
def test_fir4_exact(gf, cuda_dev, case):
    """gf_fir4_nhwc on integer x in [-8, 8] at pads 0..3 and gains 1..4 equals the fp64 blur bit for bit."""
    pad, B, Hin, Win, C, gain = case
    x = fir4_case(*case)
    Ho, Wo = Hin + 2 * pad - 3, Win + 2 * pad - 3
    xd = _dev(x, cuda_dev)
    y = Guarded((B, Ho, Wo, C), cuda_dev)
    _call(gf, "gf_fir4_nhwc", xd.data_ptr(), y.ptr(), B, Hin, Win, C, pad, float(gain), _stream(cuda_dev))
    assert_exact(y.check("fir4 y").double().cpu(), blur_def(x, pad, gain), f"fir4 {case}")


@pytest.mark.parametrize("scaled", [False, True], ids=["noscale", "scale"])
@pytest.mark.parametrize("case", BLUR_UP_CASES, ids=fir_id)
def test_blur_up_exact(gf, cuda_dev, case, scaled):
    """gf_blur_up_nhwc (pad 1) on integer x, with and without a power-of-two per-(b, c) scale."""
    B, Hout, Wout, C, gain = case
    x, scale = blur_up_case(*case, scaled)
    xd, sd = _dev(x, cuda_dev), _dev(scale, cuda_dev)
    y = Guarded((B, Hout, Wout, C), cuda_dev)
    _call(gf, "gf_blur_up_nhwc", xd.data_ptr(), y.ptr(), _ptr(sd), B, Hout, Wout, C, float(gain), _stream(cuda_dev))
    assert_exact(y.check("blur_up y").double().cpu(), _scaled(blur_def(x, 1, gain), scale), f"blur_up {case}")


@pytest.mark.parametrize("scaled", [False, True], ids=["noscale", "scale"])
@pytest.mark.parametrize("case", PHASE_CASES, ids=fir_id)
def test_blur_up_phases_exact(gf, cuda_dev, case, scaled):
    """gf_blur_up_phases_nhwc on four independent integer phase tensors equals the fp64 blur of their interleaving T."""
    B, Hout, Wout, C, gain = case
    ps, scale = phase_case(*case, scaled)
    pd = [_dev(p, cuda_dev) for p in ps]
    sd = _dev(scale, cuda_dev)
    y = Guarded((B, Hout, Wout, C), cuda_dev)
    _call(gf, "gf_blur_up_phases_nhwc", *[p.data_ptr() for p in pd], y.ptr(), _ptr(sd), B, Hout, Wout, C, float(gain),
          _stream(cuda_dev))
    assert_exact(y.check("phases y").double().cpu(), _scaled(blur_def(interleave(ps), 1, gain), scale), f"phases {case}")


MIN_HIN = {0: 4, 1: 2, 2: 1, 3: 1}


def fir4_grad_case(pad, B, C, H, W):
    s = _seed(pad, B, C, H, W, 3)
    Ho, Wo = H + 2 * pad - 3, W + 2 * pad - 3
    return ints((B, C, H, W), -8, 8, s), ints((B, C, Ho, Wo), -4, 4, s + 1), ints((B, C, H, W), -4, 4, s + 2)


def fir4_grad_shapes(pad):
    return [(2, 12, 7, 9), (1, 4, MIN_HIN[pad], MIN_HIN[pad] + 1)]


@pytest.mark.parametrize("pad", [0, 1, 2, 3])
def test_fir4_autograd_exact(gf, cuda_dev, pad):
    """ops.fir4 under autograd: the output, the first derivative (a pad-(3-p) blur of the integer cotangent) and the second
    derivative (the pad-p blur of a second integer cotangent) equal fp64 autograd through the definition bit for bit, and all
    three run on the native kernel."""
    ops = _ops()
    f32, f64 = ops.fir_filter(cuda_dev), ops.fir_filter(dtype=F64)
    gain = float(pad + 1)
    for B, C, H, W in fir4_grad_shapes(pad):
        x, gy, v = fir4_grad_case(pad, B, C, H, W)
        xg = x.float().to(cuda_dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        gyg = gy.float().to(cuda_dev).requires_grad_(True)
        n0 = gf._lib.launch_count()
        y = ops.fir4(xg, f32, pad, gain)
        (gx,) = torch.autograd.grad(y, xg, gyg, create_graph=True)
        (ggy,) = torch.autograd.grad(gx, gyg, v.float().to(cuda_dev))
        torch.cuda.synchronize()
        assert gf._lib.launch_count() - n0 == 3                       # forward, backward, double backward: all gf_fir4_nhwc
        x64, gy64 = x.clone().requires_grad_(True), gy.clone().requires_grad_(True)
        y64 = ops.upfirdn2d_ref(x64, f64, pad=(pad,) * 4, gain=gain)
        (gx64,) = torch.autograd.grad(y64, x64, gy64, create_graph=True)
        (ggy64,) = torch.autograd.grad(gx64, gy64, v)
        tag = f"pad {pad} {(B, C, H, W)}"
        assert_exact(y.detach().double().cpu(), y64.detach(), f"fir4 y {tag}")
        assert_exact(gx.detach().double().cpu(), gx64.detach(), f"fir4 dx {tag}")
        assert_exact(ggy.double().cpu(), ggy64, f"fir4 d2 {tag}")


# ------------------------------------------------------------------------------------------------ skip upsampling
UPSAMPLE_CASES = [(2, 3, 1, 1), (1, 3, 1, 17), (3, 3, 13, 1), (2, 3, 9, 14), (1, 5, 6, 31), (8, 3, 256, 256)]   # (B, C, H, W)


def upsample_case(B, C, H, W):
    s = _seed(B, C, H, W, 5)
    return ints((B, C, H, W), -8, 8, s), ints((B, C, 2 * H, 2 * W), -8, 8, s + 1)


@pytest.mark.parametrize("with_add", [False, True], ids=["noadd", "add"])
@pytest.mark.parametrize("case", UPSAMPLE_CASES, ids=fir_id)
def test_upsample2x_exact(gf, cuda_dev, case, with_add):
    """gf_upsample2x_nchw on integer x (+ integer add): H or W = 1, non-square, and 8 x 3 planes of 256^2 (more input pixels than
    threads in the capped grid, so the grid-stride loop runs several rounds)."""
    B, C, H, W = case
    x, add = upsample_case(*case)
    add = add if with_add else None
    if H == 256:
        assert B * C * H * W > _sms() * 16 * 256
    xd, ad = _dev(x, cuda_dev), _dev(add, cuda_dev)
    y = Guarded((B, C, 2 * H, 2 * W), cuda_dev)
    _call(gf, "gf_upsample2x_nchw", xd.data_ptr(), _ptr(ad), y.ptr(), B, C, H, W, _stream(cuda_dev))
    assert_exact(y.check("upsample y").double().cpu(), upsample_def(x, add), f"upsample {case}")


# ------------------------------------------------------------------------------------------------ bias + noise + activation
BIAS_ACT_SHAPES = [(3, 37, 12), (2, 1024, 512)]      # (B, HW, C)
NOISE_MODES = ["none", "shared", "per_image"]
STRENGTH = 0.25


def bias_act_case(B, HW, C, noise_mode, with_bias, with_strength):
    """Multiples of 5 everywhere, so every pre-activation is one (0.2f * 5k == k); one pre-activation planted at exactly 0."""
    s = _seed(B, HW, C, NOISE_MODES.index(noise_mode), with_bias, with_strength)
    x = 5 * ints((B, HW, C), -6, 6, s)
    bias = 5 * ints((C,), -3, 3, s + 1) if with_bias else None
    noise = None
    if noise_mode != "none":
        noise = 20 * ints((B if noise_mode == "per_image" else 1, HW), -3, 3, s + 2)     # * 0.25 or * 1: a multiple of 5
    st = STRENGTH if (with_strength and noise is not None) else 1.0
    pre = bias_act_pre(torch.zeros_like(x), bias, noise, st)
    x[0, 0, 0] = -pre[0, 0, 0]                                                          # pre-activation exactly 0
    return x, bias, noise, st


@pytest.mark.parametrize("noise_mode", NOISE_MODES)
@pytest.mark.parametrize("act", [0, 1], ids=["linear", "lrelu"])
def test_bias_act_exact(gf, cuda_dev, act, noise_mode):
    """gf_bias_act_nhwc with gain 2: bias, noise and strength each present or NULL, noise shared (noise_bstride 0) or per image,
    y separate from x and aliasing it."""
    for B, HW, C in BIAS_ACT_SHAPES:
        for with_bias in (False, True):
            for with_strength in (False, True):
                x, bias, noise, st = bias_act_case(B, HW, C, noise_mode, with_bias, with_strength)
                pre = bias_act_pre(x, bias, noise, st)
                assert pre[0, 0, 0] == 0
                want = (lrelu5(pre) if act else pre) * 2
                xd, bd, nd = _dev(x, cuda_dev), _dev(bias, cuda_dev), _dev(noise, cuda_dev)
                sd = torch.tensor([STRENGTH], device=cuda_dev) if with_strength else None
                bstride = HW if noise_mode == "per_image" else 0
                tag = f"act={act} noise={noise_mode} bias={with_bias} strength={with_strength} {(B, HW, C)}"
                for alias in (False, True):
                    y = Guarded((B, HW, C), cuda_dev, init=xd if alias else None)
                    src = y.ptr() if alias else xd.data_ptr()
                    _call(gf, "gf_bias_act_nhwc", src, y.ptr(), _ptr(bd), _ptr(nd), _ptr(sd), bstride, B, HW, C, act, 2.0,
                          _stream(cuda_dev))
                    assert_exact(y.check("bias_act y").double().cpu(), want, f"bias_act {tag} alias={alias}")


@pytest.mark.parametrize("per_image", [False, True], ids=["shared_noise", "per_image_noise"])
def test_ops_bias_act_sqrt2_exact(gf, cuda_dev, per_image):
    """ops.bias_act (gain sqrt(2) for lrelu, 1 for linear) equals float32(act(v)) * float32(sqrt(2)): one rounding."""
    ops = _ops()
    B, C, H, W = 3, 12, 5, 7
    x, bias, noise, st = bias_act_case(B, H * W, C, "per_image" if per_image else "shared", True, True)
    pre = bias_act_pre(x, bias, noise, st)
    xd = x.float().reshape(B, H, W, C).permute(0, 3, 1, 2).to(cuda_dev)             # channels-last storage
    nd = (noise.float().reshape(B, 1, H, W) if per_image else noise.float().reshape(H, W)).to(cuda_dev)
    with torch.no_grad():
        for act in ("lrelu", "linear"):
            n0 = gf._lib.launch_count()
            got = ops.bias_act(xd, bias.float().to(cuda_dev), act, noise=nd, strength=torch.tensor(st, device=cuda_dev))
            torch.cuda.synchronize()
            assert gf._lib.launch_count() - n0 == 1
            got = got.permute(0, 2, 3, 1).reshape(B, H * W, C).cpu()
            if act == "lrelu":
                want = lrelu5(pre).float() * torch.tensor(math.sqrt(2.0), dtype=torch.float32)
            else:
                want = pre.float()
            assert_exact(got, want, f"ops.bias_act {act}")


# ------------------------------------------------------------------------------------------------ channel scaling
CHAN_SCALE_CASES = [(3, 37, 4, 4, 0), (2, 29, 12, 20, 8), (3, 50, 4, 12, 4), (2, 4096, 12, 16, 4)]   # (B, HW, C, s_ld, column offset)


def chan_scale_case(B, HW, C, s_ld, off):
    s = _seed(B, HW, C, s_ld, off)
    return ints((B, HW, C), -100, 100, s), pow2((B, s_ld), -3, 3, s + 1)


@pytest.mark.parametrize("case", CHAN_SCALE_CASES, ids=fir_id)
def test_chan_scale_exact(gf, cuda_dev, case):
    """gf_chan_scale_nhwc: integer x times power-of-two styles taken as a column slice of a wider matrix (s_ld > C), y separate
    and aliasing x."""
    B, HW, C, s_ld, off = case
    x, s_full = chan_scale_case(*case)
    want = x * s_full[:, None, off:off + C]
    xd, sd = _dev(x, cuda_dev), _dev(s_full, cuda_dev)
    for alias in (False, True):
        y = Guarded((B, HW, C), cuda_dev, init=xd if alias else None)
        _call(gf, "gf_chan_scale_nhwc", y.ptr() if alias else xd.data_ptr(), sd.data_ptr() + 4 * off, s_ld, y.ptr(), B, HW, C,
              _stream(cuda_dev))
        assert_exact(y.check("chan_scale y").double().cpu(), want, f"chan_scale {case} alias={alias}")


# ------------------------------------------------------------------------------------------------ tRGB
TORGB_C = [4, 128, 132, 384, 512]            # NQ = 1, 1, 2, 3, 4 float4 chunks per lane
TORGB_HW = [(2, 1), (3, 31), (2, 33), (3, 1500)]
TORGB_WSCALE = 2.0 ** -4
TOK_HW = 4100


def tok_per_cta(HW, B, sms):
    """gf_torgb_scale_nhwc's tokens per CTA."""
    t = 1024
    while t > 256 and -(-HW // t) * B < 4 * sms:
        t >>= 1
    return t


def batch_for_tok(tok, sms, HW=TOK_HW):
    """The smallest batch for which the host picks `tok` tokens per CTA at this HW."""
    B = 1
    while tok_per_cta(HW, B, sms) != tok:
        B += 1
    return B


TORGB_CASES = [(C, HW, B) for C in TORGB_C for B, HW in TORGB_HW] + [(4, TOK_HW, -tok) for tok in (1024, 512, 256)]


def torgb_id(c):
    C, HW, B = c
    return f"C{C}_HW{HW}_" + (f"tok{-B}" if B < 0 else f"B{B}")


def resolve_torgb(case, sms):
    C, HW, B = case
    if B < 0:
        B = batch_for_tok(-B, sms)
        assert tok_per_cta(HW, B, sms) == -case[2]
    return C, HW, B


def torgb_case(C, HW, B, strided):
    """Integer x, w in [-4, 4], power-of-two styles (and s2), bias a multiple of 1/4; s_ld, s2_ld > C when strided."""
    s = _seed(C, HW, B, strided)
    s_ld, s2_ld = (C + 8, C + 4) if strided else (C, C)
    return dict(x=ints((B, HW, C), -4, 4, s), w=ints((3, C), -4, 4, s + 1), st=pow2((B, s_ld), -2, 2, s + 2),
                s2=pow2((B, s2_ld), -2, 2, s + 3), bias=ints((3,), -40, 40, s + 4) / 4 if strided else None, s_ld=s_ld, s2_ld=s2_ld)


@pytest.mark.parametrize("case", TORGB_CASES, ids=torgb_id)
def test_torgb_exact(gf, cuda_dev, case):
    """gf_torgb_scale_nhwc: integer x and w, power-of-two styles and wscale.  Strided s_ld / s2_ld with bias and the xs_out second
    output, and s_ld = C without bias or second output."""
    C, HW, B = resolve_torgb(case, _sms())
    for strided in (True, False):
        t = torgb_case(C, HW, B, strided)
        want = torgb_def(t["x"], t["w"], t["st"][:, :C], TORGB_WSCALE, t["bias"])
        xd, wd, sd, s2d, bd = (_dev(t[n], cuda_dev) for n in ("x", "w", "st", "s2", "bias"))
        y = Guarded((B, 3, HW), cuda_dev)
        xs = Guarded((B, HW, C), cuda_dev) if strided else None
        _call(gf, "gf_torgb_scale_nhwc", xd.data_ptr(), wd.data_ptr(), sd.data_ptr(), t["s_ld"], _ptr(bd), TORGB_WSCALE, y.ptr(),
              s2d.data_ptr() if strided else None, t["s2_ld"] if strided else 0, xs.ptr() if strided else None, B, HW, C,
              _stream(cuda_dev))
        assert_exact(y.check("torgb y").double().cpu(), want, f"torgb y C={C} HW={HW} B={B} strided={strided}")
        if strided:
            assert_exact(xs.check("torgb xs_out").double().cpu(), t["x"] * t["s2"][:, None, :C], f"torgb xs_out C={C} HW={HW}")


# ------------------------------------------------------------------------------------------------ demodulation
DEMOD_SHAPES = [(3, 13, 1), (5, 7, 31), (1, 20, 512), (3, 9, 513), (7, 11, 1100)]     # (B, O, I): both sides of the 512 cache
DEMOD_EPS = 1e-8
DEMOD_BATCH_B = 5                                                                      # odd: the last sample runs alone


def demod_case(B, O, I, seed):
    """Nonzero integer styles in [-3, 3] (row stride I + 5) and wsq in [1, 4]: every term is a positive integer, the sum exact."""
    st = ints((B, I + 5), 1, 3, seed) * (2 * ints((B, I + 5), 0, 1, seed + 1) - 1)
    return st, ints((O, I), 1, 4, seed + 2)


def demod_sum(st, wsq):
    I = wsq.shape[1]
    return st[:, :I].square() @ wsq.t()


def demod_want(st, wsq):
    return (1.0 / demod_sum(st, wsq).sqrt()).float()


def demod_batch_jobs():
    """32 jobs cycling through the shapes (O, I) of DEMOD_SHAPES at batch DEMOD_BATCH_B."""
    return [(DEMOD_BATCH_B, O, I, _seed(j, O, I)) for j in range(32) for _, O, I in [DEMOD_SHAPES[j % len(DEMOD_SHAPES)]]]


def _assert_ulps(got, want, name, ulps=2):
    diff = (got.view(torch.int32).long() - want.view(torch.int32).long()).abs()        # positive floats: bit distance = ulps
    assert (got > 0).all() and diff.max().item() <= ulps, f"{name}: {diff.max().item()} ulp from float32(1/sqrt(sum))"


def _demod_one(gf, dev, st, wsq, B, O, I):
    sd, wd = _dev(st, dev), _dev(wsq, dev)
    d = Guarded((B, O), dev)
    _call(gf, "gf_demod_coef", sd.data_ptr(), I + 5, wd.data_ptr(), d.ptr(), B, O, I, DEMOD_EPS, _stream(dev))
    return d.check("demod d").cpu()


@pytest.mark.parametrize("case", DEMOD_SHAPES, ids=fir_id)
def test_demod_coef_within_2_ulp(gf, cuda_dev, case):
    """gf_demod_coef: d within 2 ulp of float32(1/sqrt(sum)) (sum >= 1, so adding eps = 1e-8 changes nothing)."""
    B, O, I = case
    st, wsq = demod_case(B, O, I, _seed(*case))
    _assert_ulps(_demod_one(gf, cuda_dev, st, wsq, B, O, I), demod_want(st, wsq), f"demod {case}")


def test_demod_coef_batch_equals_per_layer(gf, cuda_dev):
    """gf_demod_coef_batch with 32 jobs (O not a multiple of 8, I across the 512-column register cache, odd B): every job equals
    gf_demod_coef bit for bit and is within 2 ulp of float32(1/sqrt(sum))."""
    jobs_spec = demod_batch_jobs()
    jobs = (gf._lib.GfDemodJob * len(jobs_spec))()
    keep, outs = [], []
    for j, (B, O, I, seed) in enumerate(jobs_spec):
        st, wsq = demod_case(B, O, I, seed)
        sd, wd = _dev(st, cuda_dev), _dev(wsq, cuda_dev)
        d = Guarded((B, O), cuda_dev)
        jobs[j].styles, jobs[j].wsq, jobs[j].d = sd.data_ptr(), wd.data_ptr(), d.ptr()
        jobs[j].s_ld, jobs[j].O, jobs[j].I = I + 5, O, I
        keep += [sd, wd]
        outs.append((d, st, wsq, B, O, I))
    _call(gf, "gf_demod_coef_batch", ctypes.cast(jobs, ctypes.c_void_p), len(jobs_spec), DEMOD_BATCH_B, DEMOD_EPS, _stream(cuda_dev))
    for j, (d, st, wsq, B, O, I) in enumerate(outs):
        got = d.check(f"demod batch job {j}").cpu()
        _assert_ulps(got, demod_want(st, wsq), f"demod batch job {j} (O={O}, I={I})")
        assert torch.equal(got.view(torch.int32), _demod_one(gf, cuda_dev, st, wsq, B, O, I).view(torch.int32)), j


# ------------------------------------------------------------------------------------------------ mapping network
MAPPING_CASES = [(16, 8, 0), (16, 8, 31), (48, 8, 1), (96, 3, 31), (128, 1, 1), (128, 1, 0)]     # (D, L, k)
MAPPING_PSI = 0.5


def mapping_batch(k, sms):
    """Rows B (k + 1) above twice the 8 rows per CTA times the grid of sms CTAs: every warp takes more than one row."""
    return 2 * sms * 8 // (k + 1) + 1


def mapping_case(D, L, k, B):
    """z entries +-1; per output column one weight +-5 (two when L <= 2); biases in {-5, 0, 5}; w_avg integers."""
    s = _seed(D, L, k, B)
    g = torch.Generator().manual_seed(s)
    z = 2 * ints((B, k + 1, D), 0, 1, s) - 1
    nnz = 2 if L <= 2 else 1
    W = torch.zeros(2, L, D, D, dtype=F64)
    for p in range(2):
        for l in range(L):
            rows = torch.stack([torch.randperm(D, generator=g)[:nnz] for _ in range(D)], dim=1)     # [nnz, D]: input rows per column
            vals = 5 * (2 * torch.randint(0, 2, (nnz, D), generator=g) - 1).to(F64)
            W[p, l].scatter_(0, rows, vals)
    b = 5 * ints((2, L, D), -1, 1, s + 1)
    return z, W, b, ints((2, D), -20, 20, s + 2)


def mapping_want(z, W, b, w_avg, k):
    return mapping_def(z, W, b, w_avg, MAPPING_PSI, k, exact_norm=True, lrelu=lrelu5)


def _mapping_run(gf, dev, z, W, b, w_avg, psi, k):
    B, _, D = z.shape
    zd, Wd, bd, ad = (_dev(t, dev) for t in (z, W, b, w_avg))
    out = Guarded((B, k + 1, D), dev)
    _call(gf, "gf_mapping_fwd", zd.data_ptr(), Wd.data_ptr(), bd.data_ptr(), _ptr(ad), psi, out.ptr(), B, k, D, W.shape[1],
          _stream(dev))
    return out.check("mapping out").double().cpu()


def mapping_id(c):
    return "D{}_L{}_k{}".format(*c)


@pytest.mark.parametrize("case", MAPPING_CASES, ids=mapping_id)
def test_mapping_exact(gf, cuda_dev, case):
    """gf_mapping_fwd with the exact construction: every pre-activation a multiple of 5, every activation an integer, the
    truncation lerp at psi = 1/2 exact; with and without w_avg."""
    D, L, k = case
    B = mapping_batch(k, _sms())
    z, W, b, w_avg = mapping_case(D, L, k, B)
    for avg in (w_avg, None):
        got = _mapping_run(gf, cuda_dev, z, W, b, avg, MAPPING_PSI, k)
        assert_exact(got, mapping_want(z, W, b, avg, k), f"mapping {case} w_avg={avg is not None}")


def test_mapping_pixel_norm_of_unit_latents_is_one(gf, cuda_dev):
    """rsqrtf(f32(1 + 1e-8)) = rsqrtf(1.0f) = 1 on this GPU: with z = +-1 and W = 5 I, the output is exactly 5 z (z > 0) or z."""
    D = 16
    z = 2 * ints((4, 1, D), 0, 1, 1) - 1
    W = (5 * torch.eye(D, dtype=F64))[None, None].repeat(2, 1, 1, 1)
    got = _mapping_run(gf, cuda_dev, z, W, torch.zeros(2, 1, D, dtype=F64), None, 1.0, 0)
    assert torch.equal(got, torch.where(z > 0, 5 * z, z)), "rsqrtf(1.0f) is not 1"


def test_mapping_rejects_oversized_weights(gf, cuda_dev):
    """2 L D^2 floats beyond the opt-in shared memory (D = 64 at L = 8) come back as GF_ERR_UNSUPPORTED."""
    lib = gf._lib.load()
    buf = torch.zeros(2 * 8 * 64 * 64, device=cuda_dev)
    rc = lib.gf_mapping_fwd(buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), None, 1.0, buf.data_ptr(), 1, 0, 64, 8, _stream(cuda_dev))
    assert rc == -2 and "shared memory" in lib.gf_last_error().decode()


# ------------------------------------------------------------------------------------------------ realistic data
def _rel_check(name, got, want, comp):
    got = got.double().cpu()
    assert got.shape == want.shape
    err = (got - want).abs()
    zero = comp == 0
    assert not err[zero].any(), f"{name}: an output with a zero companion is not exact"
    rel = (err[~zero] / comp[~zero]).max().item()
    print(f"[ops-exact] {name}: max |y - y64| / companion = {rel:.3e} (bound {REL_BOUND[name]:.1e})")
    assert rel <= REL_BOUND[name], f"{name}: {rel:.3e} > {REL_BOUND[name]}"


def _randn(shape, seed, mean=0.0):
    return torch.randn(tuple(shape), generator=torch.Generator().manual_seed(seed), dtype=F64) + mean


REALISTIC = ["fir4", "blur_up", "blur_up_phases", "upsample2x", "bias_act", "chan_scale", "torgb", "demod", "mapping"]


@pytest.mark.parametrize("name", REALISTIC)
def test_realistic_data(gf, cuda_dev, name):
    """Random fp32 data at generator-like shapes against fp64, per element relative to the magnitude companion."""
    dev, st = cuda_dev, _stream(cuda_dev)
    keep = []                                                               # device inputs stay alive until the call returns

    def dv(t):
        keep.append(_dev(t, dev))
        return keep[-1]

    f32 = lambda t: t.float().double()                                      # the fp32 inputs the kernel sees, in fp64
    if name == "fir4":
        B, H, W, C, pad = 4, 33, 40, 256, 2
        x = f32(_randn((B, H, W, C), 1))
        y = Guarded((B, H + 1, W + 1, C), dev)
        _call(gf, "gf_fir4_nhwc", dv(x).data_ptr(), y.ptr(), B, H, W, C, pad, 1.0, st)
        _rel_check(name, y.check(name), blur_def(x, pad, 1.0), blur_def(x.abs(), pad, 1.0))
    elif name == "blur_up":
        B, Ho, Wo, C = 4, 32, 32, 256
        x, s = f32(_randn((B, Ho + 1, Wo + 1, C), 2)), f32(torch.rand(B, C, generator=torch.Generator().manual_seed(3)) + 0.5)
        y = Guarded((B, Ho, Wo, C), dev)
        _call(gf, "gf_blur_up_nhwc", dv(x).data_ptr(), y.ptr(), dv(s).data_ptr(), B, Ho, Wo, C, 4.0, st)
        _rel_check(name, y.check(name), _scaled(blur_def(x, 1, 4.0), s), _scaled(blur_def(x.abs(), 1, 4.0), s))
    elif name == "blur_up_phases":
        B, Ho, Wo, C = 4, 32, 32, 256
        ps = [f32(_randn(sh, 10 + i)) for i, sh in enumerate([(B, 17, 17, C), (B, 17, 16, C), (B, 16, 17, C), (B, 16, 16, C)])]
        s = f32(torch.rand(B, C, generator=torch.Generator().manual_seed(4)) + 0.5)
        y = Guarded((B, Ho, Wo, C), dev)
        _call(gf, "gf_blur_up_phases_nhwc", *[dv(p).data_ptr() for p in ps], y.ptr(), dv(s).data_ptr(), B, Ho, Wo, C,
              4.0, st)
        T = interleave(ps)
        _rel_check(name, y.check(name), _scaled(blur_def(T, 1, 4.0), s), _scaled(blur_def(T.abs(), 1, 4.0), s))
    elif name == "upsample2x":
        B, C, H, W = 8, 3, 128, 128
        x, add = f32(_randn((B, C, H, W), 5)), f32(_randn((B, C, 2 * H, 2 * W), 6))
        y = Guarded((B, C, 2 * H, 2 * W), dev)
        _call(gf, "gf_upsample2x_nchw", dv(x).data_ptr(), dv(add).data_ptr(), y.ptr(), B, C, H, W, st)
        _rel_check(name, y.check(name), upsample_def(x, add), upsample_def(x.abs(), add.abs()))
    elif name == "bias_act":
        B, HW, C = 4, 1024, 256
        x, bias, noise = f32(_randn((B, HW, C), 7)), f32(_randn((C,), 8)), f32(_randn((B, HW), 9))
        strength, gain = 0.37, math.sqrt(2.0)
        s32, g32 = float(torch.tensor(strength, dtype=torch.float32)), float(torch.tensor(gain, dtype=torch.float32))
        y = Guarded((B, HW, C), dev)
        _call(gf, "gf_bias_act_nhwc", dv(x).data_ptr(), y.ptr(), dv(bias).data_ptr(), dv(noise).data_ptr(),
              dv(torch.tensor([strength])).data_ptr(), HW, B, HW, C, 1, gain, st)
        want = torch.nn.functional.leaky_relu(bias_act_pre(x, bias, noise, s32), 0.2) * g32
        comp = bias_act_pre(x.abs(), bias.abs(), noise.abs(), s32) * g32
        _rel_check(name, y.check(name), want, comp)
    elif name == "chan_scale":
        B, HW, C = 4, 1024, 512
        x, s = f32(_randn((B, HW, C), 11)), f32(_randn((B, C), 12))
        y = Guarded((B, HW, C), dev)
        _call(gf, "gf_chan_scale_nhwc", dv(x).data_ptr(), dv(s).data_ptr(), C, y.ptr(), B, HW, C, st)
        _rel_check(name, y.check(name), x * s[:, None, :], (x * s[:, None, :]).abs())
    elif name == "torgb":
        B, HW, C = 4, 4096, 512
        x, w, sty, bias = f32(_randn((B, HW, C), 13)), f32(_randn((3, C), 14)), f32(_randn((B, C), 15, mean=1.0)), f32(_randn((3,), 16))
        wscale = 1.0 / math.sqrt(C)
        ws32 = float(torch.tensor(wscale, dtype=torch.float32))
        y = Guarded((B, 3, HW), dev)
        _call(gf, "gf_torgb_scale_nhwc", dv(x).data_ptr(), dv(w).data_ptr(), dv(sty).data_ptr(), C,
              dv(bias).data_ptr(), wscale, y.ptr(), None, 0, None, B, HW, C, st)
        _rel_check(name, y.check(name), torgb_def(x, w, sty, ws32, bias), torgb_def(x.abs(), w.abs(), sty.abs(), ws32, bias.abs()))
    elif name == "demod":
        B, O, I = 8, 512, 1100
        sty = f32(_randn((B, I), 17, mean=1.0))
        wsq = f32(torch.rand(O, I, generator=torch.Generator().manual_seed(18), dtype=F64) / I)
        d = Guarded((B, O), dev)
        _call(gf, "gf_demod_coef", dv(sty).data_ptr(), I, dv(wsq).data_ptr(), d.ptr(), B, O, I, DEMOD_EPS, st)
        want = 1.0 / torch.sqrt(sty.square() @ wsq.t() + DEMOD_EPS)
        _rel_check(name, d.check(name), want, want)
    elif name == "mapping":
        D, L, k, B = 128, 1, 16, 64
        z = f32(_randn((B, k + 1, D), 19))
        W = f32(_randn((2, L, D, D), 20) * math.sqrt(2.0 / D))
        b = f32(_randn((2, L, D), 21) * 0.1)
        w_avg, psi = f32(_randn((2, D), 22)), 0.7
        got = _mapping_run(gf, dev, z, W, b, w_avg, psi, k)
        psi32 = float(torch.tensor(psi, dtype=torch.float32))
        want = mapping_def(z, W, b, w_avg, psi32, k, exact_norm=False)
        comp = mapping_def(z.abs(), W.abs(), b.abs(), None, psi32, k, exact_norm=False, lrelu=lambda v: v)
        a = w_avg.abs()[[0] * k + [1]]                                       # the w_avg row of each latent's path
        _rel_check(name, got, want, a + psi32 * (comp + a))


# ------------------------------------------------------------------------------------------------ the wrappers' alignment
FLOAT4_OPERANDS = {                    # argument positions of the float4 operands of each entry (include/gf_ops.h)
    "gf_chan_scale_nhwc": (0, 1, 3), "gf_blur_up_nhwc": (0, 1, 2), "gf_blur_up_phases_nhwc": (0, 1, 2, 3, 4, 5),
    "gf_fir4_nhwc": (0, 1), "gf_bias_act_nhwc": (0, 1, 2), "gf_torgb_scale_nhwc": (0, 1, 2, 7, 9),
}


class _Recorder:
    """Stands in for the loaded library: records every call and returns GF_OK without launching anything."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


def _offset_view(shape, dev, seed):
    """A contiguous tensor of `shape` that starts 4 bytes into its storage."""
    n = math.prod(shape)
    buf = torch.randn(n + 4, generator=torch.Generator().manual_seed(seed)).to(dev)
    t = buf[1:1 + n].view(shape)
    assert t.is_contiguous() and t.data_ptr() % 16 == 4
    return t


def test_wrappers_pass_aligned_float4_operands(gf, cuda_dev, monkeypatch):
    """ops.chan_scale, fir4, blur_up, bias_act and torgb given contiguous views that start 4 bytes into their storage (x, styles,
    bias, weight, scale) hand the library 16-byte aligned copies.  The library is replaced by a recorder: nothing is launched."""
    ops = _ops()
    rec = _Recorder()
    monkeypatch.setattr(gf._lib, "load", lambda: rec)
    B, C, H, W = 2, 12, 5, 6
    x = _offset_view((B, H, W, C), cuda_dev, 1).permute(0, 3, 1, 2)              # channels-last storage, misaligned
    s = _offset_view((B, C), cuda_dev, 2)
    f = ops.fir_filter(cuda_dev)
    with torch.no_grad():
        ops.chan_scale(x, s)
        ops.fir4(x, f, 2)
        ops.blur_up(x, f, scale=s)
        ops.bias_act(x, _offset_view((C,), cuda_dev, 3), "lrelu", noise=torch.randn(H, W, device=cuda_dev),
                     strength=torch.tensor(0.5, device=cuda_dev))
        ops.bias_act(x, _offset_view((C,), cuda_dev, 4), "linear")
        ops.torgb(x, _offset_view((3, C, 1, 1), cuda_dev, 5), s, torch.randn(3, device=cuda_dev), next_styles=_offset_view((B, C), cuda_dev, 6))
    seen = [name for name, _ in rec.calls]
    assert seen == ["gf_chan_scale_nhwc", "gf_fir4_nhwc", "gf_blur_up_nhwc", "gf_bias_act_nhwc", "gf_bias_act_nhwc",
                    "gf_torgb_scale_nhwc"], seen
    for name, args in rec.calls:
        for i in FLOAT4_OPERANDS[name]:
            assert args[i] is None or args[i] % 16 == 0, f"{name}: operand {i} at {args[i]:#x} is not 16-byte aligned"
