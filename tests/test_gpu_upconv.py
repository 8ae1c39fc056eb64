"""GPU tests of the fused upsampling kernel (``upconv_blur_tc_kernel``, csrc/gf_conv.cu; run on an H100: ``pytest -m gpu``):
stride-2 transposed 3x3 convolution + [1,3,3,1] FIR blur + demodulation in one launch, TF32.

The arithmetic (DESIGN.md section 5): packed weights rounded to the nearest TF32 value, activations truncated by the tensor core,
fp32 sums; the blur sums the raw phase values in a fixed order with integer weights (horizontal, then vertical), multiplies by
1/64 and then once by the fp32 factor ``alpha * gain * d[b, c]``.

* Exact integers (indexing, halo, strip walk and scheduling): with x, w in {-2..2} and powers of two for d and gain, y must equal
  ``float32(S / 64) * float32(alpha * gain * d)`` bit for bit, S the exact integer blur sum; NaN guards around y.
* Realistic data against the truncation emulation and, by least-squares slope, against the exact result of the unrounded operands.
* Against today's path (four cuDNN polyphase convolutions + the polyphase blur) at the generator's shapes.
* Determinism, batch independence, CUDA-graph replay, and the 256^2 generator end to end against the fp64 oracle.
"""
import ctypes
import json
import math
import os
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from oracle import generator as og
from oracle.tf32 import tf32_trunc

pytestmark = pytest.mark.gpu

ALPHA32 = float(torch.tensor(1.000352220, dtype=torch.float32))
# max over elements of |y - alpha gain d blur(convT_fp64(tf32_trunc(x), wt))| / (gain d blur(convT_fp64(|tf32_trunc(x)|, |wt|))):
# measured worst 2.9e-7 (2 x 16 x 16, 512 -> 512) on an H100 80GB HBM3 at a 400 W power limit; held at the stride-1 kernel's 3e-6
EMULATED_REL_BOUND = 3e-6
SLOPE_BOUND = 5e-5               # measured within 4.1e-6
PHASES_REL_RMS = 2e-3            # against cuDNN's TF32 polyphase convolutions, which round x differently: measured 3.7e-4
GUARD = 64
GUARD_BITS = 0x7FC0DEAD
STRIP, STEP = 14, 8              # output column pairs per strip, phase rows per step (csrc/gf_conv.cu U_OC, U_PR)
F4 = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64)
F44 = torch.outer(F4, F4)        # the blur's integer weights, sum 64


def _ops():
    return import_module("gansformer-reproducibility-challenge_b200.ops")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _units(B, H, W, cout):
    return B * ((W + STRIP - 1) // STRIP) * (cout // 64)


def _ref64(x_nhwc, w, sum_only=False):
    """fp64 blur(conv_transpose2d(x, w^T, stride 2)) * 64 (the integer blur sum S): x [B,H,W,I], w [O,I,3,3] -> [B,2H,2W,O]."""
    t = F.conv_transpose2d(x_nhwc.permute(0, 3, 1, 2).double(), w.double().transpose(0, 1), stride=2)     # [B, O, 2H+1, 2W+1]
    C = t.shape[1]
    s = F.conv2d(F.pad(t, [1, 1, 1, 1]), F44.to(t.device)[None, None].expand(C, 1, 4, 4).contiguous(), groups=C)
    return s.permute(0, 2, 3, 1)


def _run_guarded(gf, x, wt, d, gain):
    B, H, W, cin = x.shape
    cout = wt.shape[1]
    n = B * 4 * H * W * cout
    buf = torch.full((n + 2 * GUARD,), GUARD_BITS, dtype=torch.int32, device=x.device)
    y = buf[GUARD:GUARD + n].view(torch.float32)
    stream = ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
    gf._lib.check(gf._lib.load().gf_upconv3x3_blur_nhwc_tf32(x.data_ptr(), wt.data_ptr(), d.data_ptr(), y.data_ptr(), B, H, W, cin, cout,
                                                             ctypes.c_float(gain), stream), "gf_upconv3x3_blur_nhwc_tf32")
    torch.cuda.synchronize()
    assert (buf[:GUARD] == GUARD_BITS).all(), "the kernel wrote before its output"
    assert (buf[GUARD + n:] == GUARD_BITS).all(), "the kernel wrote past its output"
    y = y.view(B, 2 * H, 2 * W, cout)
    assert not torch.isnan(y).any(), f"{int(torch.isnan(y).sum())} output elements never written"
    return y


def _integer_case(gf, dev, B, H, W, cin, cout, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-2, 3, (B, H, W, cin), generator=g).float().to(dev)
    w = torch.randint(-2, 3, (cout, cin, 3, 3), generator=g).float().to(dev)
    d = (2.0 ** torch.randint(-3, 3, (B, cout), generator=g)).float().to(dev)
    gain = 4.0
    wt = _ops().conv3x3_pack(w)
    y = _run_guarded(gf, x, wt, d, gain)
    S = _ref64(x, w)
    f = (torch.tensor(ALPHA32 * gain, dtype=torch.float32) * d.cpu()).to(dev)          # float32(alpha * gain * d): exact
    want = (S / 64).float() * f[:, None, None, :]
    bad = (y != want)
    assert not bad.any(), f"{int(bad.sum())} of {y.numel()} elements differ; first at {bad.nonzero()[0].tolist()}"


# (B, H, W, Cin, Cout): every N-tile count for Cout 64 .. 512, 1 to 16 chunks, sizes off the strip and the step, 4x4 and 8x8 inputs
COVERAGE = [
    (1, 4, 4, 32, 64), (2, 8, 8, 64, 128), (1, 5, 7, 96, 192), (1, 13, 29, 512, 256), (2, 16, 30, 256, 320),
    (1, 9, 15, 160, 512), (1, 7, 14, 32, 448), (1, 17, 43, 128, 384), (3, 1, 1, 32, 64), (1, 24, 28, 480, 64),
]
GENERATOR = [(2, 4, 4, 512, 512), (2, 8, 8, 512, 512), (2, 16, 16, 512, 512), (2, 32, 32, 512, 512), (2, 64, 64, 512, 256),
             (1, 128, 128, 256, 128), (1, 256, 256, 128, 64)]     # the 256^2 generator's six layers + the 512^2 one's 128 -> 64


@pytest.mark.parametrize("shape", COVERAGE + GENERATOR, ids=lambda s: "x".join(map(str, s)))
def test_integer_exact(gf, cuda_dev, shape):
    _integer_case(gf, cuda_dev, *shape)


@pytest.mark.parametrize("hwc", [(16, 30, 64, 192), (9, 43, 96, 64)], ids=lambda s: "x".join(map(str, s)))
def test_integer_exact_persistent(gf, cuda_dev, hwc):
    """More than twice as many work units as SMs and not a multiple of the SM count: every CTA walks several units."""
    H, W, cin, cout = hwc
    sms = _sms()
    per = _units(1, H, W, cout)
    B = 2 * sms // per + 1
    while (B * per) % sms == 0:
        B += 1
    assert B * per > 2 * sms
    _integer_case(gf, cuda_dev, B, H, W, cin, cout)


@pytest.mark.parametrize("shape", [(2, 16, 16, 512, 512), (2, 32, 32, 256, 128), (1, 13, 29, 96, 192)], ids=lambda s: "x".join(map(str, s)))
def test_emulated_and_slope(gf, cuda_dev, shape):
    B, H, W, cin, cout = shape
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, H, W, cin, generator=g).to(cuda_dev)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / math.sqrt(9 * cin)).to(cuda_dev)
    d = (torch.rand(B, cout, generator=g) + 0.5).to(cuda_dev)
    gain = 4.0
    wt = _ops().conv3x3_pack(w)
    y = _run_guarded(gf, x, wt, d, gain).double()
    wr = wt.reshape(3, 3, cout, cin).permute(2, 3, 0, 1)                           # the packed (TF32-rounded) weights as [O, I, 3, 3]
    scale = (gain * d.double() / 64)[:, None, None, :]
    emu = ALPHA32 * _ref64(tf32_trunc(x), wr) * scale
    mag = _ref64(tf32_trunc(x).abs(), wr.abs()) * scale
    rel = ((y - emu).abs() / mag.clamp_min(1e-30)).max().item()
    exact = _ref64(x, w) * scale
    slope = ((y * exact).sum() / (exact * exact).sum()).item() - 1.0
    print(f"[upconv] {shape}: emulated rel {rel:.3e}  slope-1 {slope:.2e}")
    assert rel <= EMULATED_REL_BOUND
    assert abs(slope) <= SLOPE_BOUND


@pytest.mark.parametrize("shape", GENERATOR[:6], ids=lambda s: "x".join(map(str, s)))
def test_against_phases_path(gf, cuda_dev, shape):
    B, H, W, cin, cout = shape
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, cin, H, W, generator=g).to(cuda_dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / math.sqrt(9 * cin)).to(cuda_dev)
    d = (torch.rand(B, cout, generator=g) + 0.5).to(cuda_dev)
    old = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = True
        with torch.no_grad():
            ref = ops.upconv_blur_phases(x, ops.upconv_phase_weights(w), scale=d, gain=4.0)
            got = ops.upconv_blur_native(x, ops.conv3x3_pack(w), scale=d, gain=4.0)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    rms = ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    print(f"[upconv] vs phases {shape}: rel-rms {rms:.3e}")
    assert got.shape == ref.shape and rms <= PHASES_REL_RMS


def test_determinism_batch_independence_graph(gf, cuda_dev):
    ops = _ops()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(3, 256, 32, 32, generator=g).to(cuda_dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(256, 256, 3, 3, generator=g) / 48).to(cuda_dev)
    d = (torch.rand(3, 256, generator=g) + 0.5).to(cuda_dev)
    wt = ops.conv3x3_pack(w)
    with torch.no_grad():
        a = ops.upconv_blur_native(x, wt, d).clone()
        b = ops.upconv_blur_native(x, wt, d).clone()
        one = ops.upconv_blur_native(x[1:2].contiguous(memory_format=torch.channels_last), wt, d[1:2].contiguous()).clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.upconv_blur_native(x, wt, d)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = ops.upconv_blur_native(x, wt, d)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(a[1:2], one)
    assert torch.equal(a, yg)


def test_generator_e2e_tf32(gf, cuda_dev):
    """The 256^2 generator (K = 16) with TF32 convolutions, upsampling layers on the fused kernel, against the fp64 oracle within
    tolerances.json e2e (wgmma_tf32)."""
    tol = json.load(open(os.path.join(os.path.dirname(__file__), "tolerances.json")))["e2e"]["wgmma_tf32"]
    torch.manual_seed(0)
    G = gf.Generator(resolution=256, components_num=16, latent_dim=32).to(cuda_dev).eval()
    z = torch.randn(2, 17, 32, generator=torch.Generator().manual_seed(1))
    old = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = True
        with torch.no_grad():
            img = G(z.to(cuda_dev)).double().cpu()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    ref = og.generator_forward(G.state_dict(), z, resolution=256, components_num=16, latent_dim=32)
    err = (img - ref).abs()
    peak = ref.abs().max().item()
    rmse = err.pow(2).mean().sqrt().item()
    rel = rmse / ref.pow(2).mean().sqrt().item()
    psnr = 20 * math.log10(peak / rmse)
    print(f"[upconv e2e] max_abs/peak={err.max().item() / peak:.3e} rel_rms={rel:.3e} psnr={psnr:.1f} dB")
    assert err.max().item() <= tol["max_abs_rel_peak"] * peak and rel <= tol["rel_rms"] and psnr >= tol["psnr_db"]
