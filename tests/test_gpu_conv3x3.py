"""GPU tests of the 3x3 implicit-GEMM convolution (``conv3x3_tc_kernel<BN>``, csrc/gf_conv.cu; run on an H100: ``pytest -m gpu``).

The kernel's arithmetic, as DESIGN.md section 5 states it: the packed weights are rounded to the nearest TF32 value by
``gf_conv3x3_pack_weights``, the tensor core truncates the streamed activations to TF32, products are summed in fp32, and the
result is multiplied by ``alpha = 1.000352220`` in fp32 to cancel the mean truncation bias.  The tests pin each part:

* Exact integers (the check of indexing and scheduling): with x and w small integers every product and partial sum is exact, so
  the output must equal ``float32(acc) * alpha`` bit for bit whatever the summation order.  The shapes cover every N tile width
  (BN = 64 / 128 / 256) with 1, 2, 3 and 5 N tiles, 1 to 16 input-channel chunks, single-patch images whose halo is outside the
  image on all four sides, the persistent schedule with several tiles per CTA, and the five layers of the 256^2 generator.
* The conversion rule: one input value 1 + 3 * 2^-12 through a one-hot filter comes out as alpha * 1 (truncated), not
  alpha * (1 + 2^-10) (rounded) nor alpha * v (not converted).
* Realistic data, against the truncation emulation ``alpha * conv_fp64(tf32_trunc(x), wt)`` within a frozen per-element bound
  relative to ``conv_fp64(|x|, |wt|)`` (what is left is fp32 accumulation order), and against the exact convolution of the
  unrounded operands by least-squares slope (a missing alpha or a changed rounding moves it by about 3.5e-4).
* Packing bit for bit, determinism, batch independence and CUDA-graph replay.
"""
import ctypes
import math
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from oracle.tf32 import tf32_rne, tf32_trunc

pytestmark = pytest.mark.gpu

ALPHA = 1.000352220              # P.alpha of csrc/gf_conv.cu
ALPHA32 = float(torch.tensor(ALPHA, dtype=torch.float32))          # the float32 value the kernel multiplies by
# Emulated-reference bound: max over elements of |y - alpha * conv_fp64(tf32_trunc(x), wt)| / conv_fp64(|tf32_trunc(x)|, |wt|).
# Measured worst case 1.42e-6 (2 x 64 x 64, 512 -> 512) on an H100 80GB HBM3 at a 700 W power limit; frozen with a 2.1x margin.
EMULATED_REL_BOUND = 3e-6
SLOPE_BOUND = 5e-5               # |<y, want> / <want, want> - 1| against the exact convolution of the unrounded operands
GUARD = 64                       # floats of NaN guard before and after every output buffer (256 bytes: keeps y 16-byte aligned)
GUARD_BITS = 0x7FC0DEAD          # a quiet NaN no arithmetic produces


def _ops():
    return import_module("gansformer-reproducibility-challenge_b200.ops")


def _bn(cout):
    return 256 if cout % 256 == 0 else 128 if cout % 128 == 0 else 64       # the host's choice: the widest N tile dividing Cout


def _tiles(B, H, W, cout):
    return B * (H // 8) * (W // 16) * (cout // _bn(cout))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _persistent_batch(H, W, cout, sms):
    """The smallest batch whose tile count exceeds twice the SM count and is not a multiple of it: every CTA walks at least two
    tiles and the last round is partial."""
    per_image = _tiles(1, H, W, cout)
    B = 2 * sms // per_image + 1
    while (B * per_image) % sms == 0:
        B += 1
    return B


def _conv_guarded(gf, x, wt):
    """gf_conv3x3_nhwc_tf32 through the C ABI on x [B,H,W,Cin] (contiguous), writing y into the middle of a NaN-filled buffer.
    Checks that the guard regions on both sides are untouched and that every element of y was written."""
    B, H, W, cin = x.shape
    cout = wt.shape[1]
    n = B * H * W * cout
    buf = torch.full((n + 2 * GUARD,), GUARD_BITS, dtype=torch.int32, device=x.device)
    y = buf[GUARD:GUARD + n].view(torch.float32)
    assert y.data_ptr() % 16 == 0 and x.is_contiguous() and wt.is_contiguous()
    stream = ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
    gf._lib.check(gf._lib.load().gf_conv3x3_nhwc_tf32(x.data_ptr(), wt.data_ptr(), y.data_ptr(), B, H, W, cin, cout, stream),
                  "gf_conv3x3_nhwc_tf32")
    torch.cuda.synchronize()
    assert (buf[:GUARD] == GUARD_BITS).all(), "the convolution wrote before its output"
    assert (buf[GUARD + n:] == GUARD_BITS).all(), "the convolution wrote past its output"
    y = y.view(B, H, W, cout)
    assert not torch.isnan(y).any(), f"{int(torch.isnan(y).sum())} output elements never written"
    return y


def _conv64(x_nhwc, w):
    """fp64 zero-padded 3x3 convolution: x [B,H,W,Cin] (any float dtype), w [Cout,Cin,3,3] -> [B,H,W,Cout] float64."""
    return F.conv2d(x_nhwc.permute(0, 3, 1, 2).double(), w.double(), padding=1).permute(0, 2, 3, 1)


def _unpack(wt):
    """[9][Cout][Cin] (tap = dy * 3 + dx) -> [Cout][Cin][3][3]."""
    return wt.reshape(3, 3, *wt.shape[1:]).permute(2, 3, 0, 1)


def _unpack_inverse(w):
    """[Cout][Cin][3][3] -> the packed [9][Cout][Cin] layout, no rounding."""
    return w.permute(2, 3, 0, 1).reshape(9, w.shape[0], w.shape[1]).contiguous()


# (B, H, W, Cin, Cout); B = None: the persistent regime, batch derived from the device's SM count
COVERAGE = [
    (1, 8, 16, 32, 64),        # one patch: the halo is outside the image on all four sides; BN 64, 1 N tile, 1 chunk
    (2, 8, 16, 96, 192),       # one patch per image; BN 64, 3 N tiles, 3 chunks
    (1, 8, 16, 512, 768),      # one patch; BN 256, 3 N tiles, 16 chunks
    (1, 8, 256, 256, 320),     # one patch row; BN 64, 5 N tiles, 8 chunks
    (3, 128, 16, 512, 128),    # one patch column; BN 128, 1 N tile, 16 chunks
    (1, 24, 48, 96, 384),      # BN 128, 3 N tiles
    (2, 8, 256, 32, 256),      # BN 256, 1 N tile
    (1, 24, 48, 256, 512),     # BN 256, 2 N tiles
    # the shapes of the convolution's first parity test
    (2, 16, 16, 64, 64), (3, 32, 16, 128, 128), (1, 8, 32, 256, 256), (2, 24, 48, 96, 192), (1, 64, 64, 32, 512),
]
PERSISTENT = [  # (H, W, Cin, Cout): for each BN an odd and an even chunk count (an odd count flips the ring parity per tile)
    (24, 48, 96, 320), (64, 64, 256, 192),                          # BN 64
    (64, 64, 32, 384), (128, 16, 96, 128), (8, 256, 512, 384),      # BN 128
    (64, 64, 96, 768), (24, 48, 256, 512),                          # BN 256
]
GENERATOR = [(2, r, r, c, c) for r, c in ((16, 512), (32, 512), (64, 512), (128, 256), (256, 128))]   # the 256^2 generator's layers


def _case_id(c):
    return "B{}_{}x{}_{}to{}".format("P" if c[0] is None else c[0], *c[1:])


INTEGER_CASES = COVERAGE + [(None,) + p for p in PERSISTENT] + GENERATOR


def _resolve(case):
    B, H, W, cin, cout = case
    if B is None:
        sms = _sms()
        B = _persistent_batch(H, W, cout, sms)
        t = _tiles(B, H, W, cout)
        assert t > 2 * sms and t % sms != 0, (t, sms)                                    # several tiles per CTA, partial last round
    return B, H, W, cin, cout


@pytest.mark.parametrize("case", INTEGER_CASES, ids=_case_id)
def test_integer_inputs_bit_exact(gf, cuda_dev, case):
    """x, w in {-2, ..., 2}, packed with scale 1 and 1/8: every product and partial sum is an integer or a multiple of 1/8 far
    below 2^22, exact in TF32 and fp32, so y == float32(acc) * float32(alpha) bit for bit, acc the exact convolution."""
    B, H, W, cin, cout = _resolve(case)
    g = torch.Generator(device=cuda_dev).manual_seed(B * 1000003 + H * 1009 + W * 101 + cin * 7 + cout)
    x = torch.randint(-2, 3, (B, H, W, cin), generator=g, device=cuda_dev).float()
    w = torch.randint(-2, 3, (cout, cin, 3, 3), generator=g, device=cuda_dev).float()
    acc = _conv64(x, w).round()                                     # exact already; rounding guards against any fp64 algorithm
    assert acc.abs().max().item() < 2 ** 15
    for scale in (1.0, 0.125):
        wt = _ops().conv3x3_pack(w, scale=scale)
        assert torch.equal(wt, _unpack_inverse(w * scale))                                 # integers and eighths are TF32 values
        got = _conv_guarded(gf, x, wt)
        want = (acc * scale).float() * torch.tensor(ALPHA32, device=cuda_dev)          # one fp32 rounding, as the kernel's store
        bad = got != want                                                                # (+0 and -0 compare equal)
        if bad.any():
            idx = bad.nonzero()[0].tolist()
            pytest.fail(f"scale={scale}: {int(bad.sum())} of {bad.numel()} outputs differ; first at [b,h,w,o]={idx}: "
                        f"got {got[tuple(idx)].item()!r}, want {want[tuple(idx)].item()!r}")


def test_activation_operand_is_truncated_to_tf32(gf, cuda_dev):
    """The conversion rule alpha compensates: one nonzero input v = +-(1 + 3 * 2^-12) and a one-hot centre tap equal to 1.  The
    tensor core truncates v to 1 (output +-alpha); rounding to nearest would give +-alpha * (1 + 2^-10), no conversion alpha * v."""
    B, H, W, cin, cout = 2, 8, 16, 32, 64
    v = 1.0 + 3.0 * 2.0 ** -12
    spots = [(0, 3, 5, 7, 10, v), (1, 0, 15, 31, 63, -v), (1, 7, 0, 0, 0, v)]   # (b, h, w, i, o, value); the last two at corners
    x = torch.zeros(B, H, W, cin, device=cuda_dev)
    w = torch.zeros(cout, cin, 3, 3, device=cuda_dev)
    for b, h, ww, i, o, val in spots:
        x[b, h, ww, i] = val
        w[o, i, 1, 1] = 1.0
    got = _conv_guarded(gf, x, _ops().conv3x3_pack(w)).cpu()
    want = torch.zeros_like(got)
    for b, h, ww, i, o, val in spots:
        want[b, h, ww, o] = math.copysign(ALPHA32, val)
        seen = got[b, h, ww, o].item()
        assert seen == want[b, h, ww, o].item(), (
            f"input {val!r} came out as {seen!r}: truncation gives {math.copysign(ALPHA32, val)!r}, nearest rounding "
            f"{float(torch.tensor(math.copysign(ALPHA32, val)) * (1 + 2 ** -10))!r}, no conversion {ALPHA32 * val!r}")
    assert torch.equal(got, want)                                                        # nothing else lit up


REALISTIC = [(2, 16, 16, 64, 64), (3, 32, 16, 128, 128), (1, 8, 32, 256, 256), (2, 24, 48, 96, 192), (1, 64, 64, 32, 512),
             (1, 8, 16, 512, 768), (2, 64, 64, 512, 512), (None, 64, 64, 96, 768), (None, 24, 48, 96, 320)]


@pytest.mark.parametrize("case", REALISTIC, ids=_case_id)
def test_realistic_data_tight(gf, cuda_dev, case):
    """N(0,1) x and w, scale 1/sqrt(9 Cin): (1) against the truncation emulation alpha * conv_fp64(tf32_trunc(x), wt), per element
    relative to conv_fp64(|tf32_trunc(x)|, |wt|); (2) least-squares slope against the exact fp64 convolution of the unrounded
    operands; (3) the TF32 contract bounds of the convolution (rel-RMS <= 5e-4, max <= 3e-3 of the peak)."""
    B, H, W, cin, cout = _resolve(case)
    g = torch.Generator(device=cuda_dev).manual_seed(B + H + cin + cout)
    x = torch.randn(B, H, W, cin, generator=g, device=cuda_dev)
    w = torch.randn(cout, cin, 3, 3, generator=g, device=cuda_dev)
    scale = 1.0 / math.sqrt(9 * cin)
    wt = _ops().conv3x3_pack(w, scale=scale)
    got = _conv_guarded(gf, x, wt).double()
    xt, wu = tf32_trunc(x), _unpack(wt)
    emu = ALPHA32 * _conv64(xt, wu)
    mag = _conv64(xt.abs(), wu.abs())
    rel = ((got - emu).abs() / mag).max().item()
    exact = _conv64(x, w.double() * scale)
    slope = ((got * exact).sum() / (exact * exact).sum()).item()
    err = (got - exact).abs()
    rel_rms = (err.pow(2).mean().sqrt() / exact.pow(2).mean().sqrt()).item()
    peak_ratio = (err.max() / exact.abs().max()).item()
    print(f"[conv3x3] B={B} {H}x{W} {cin}->{cout} emulated_rel={rel:.3e} slope-1={slope - 1:+.3e} rel_rms={rel_rms:.3e} "
          f"max/peak={peak_ratio:.3e}")
    problems = []                                                                        # report every check that fails
    if not rel <= EMULATED_REL_BOUND:
        problems.append(f"emulated: max |y - emu| / conv(|x|, |wt|) = {rel:.3e} > {EMULATED_REL_BOUND}")
    if not abs(slope - 1) <= SLOPE_BOUND:
        problems.append(f"slope: least-squares slope - 1 = {slope - 1:+.3e}, bound {SLOPE_BOUND}")
    if not (rel_rms <= 5e-4 and peak_ratio <= 3e-3):
        problems.append(f"contract: rel_rms {rel_rms:.3e} (bound 5e-4), max/peak {peak_ratio:.3e} (bound 3e-3)")
    assert not problems, "; ".join(problems)


@pytest.mark.parametrize("cout,cin,scale", [(64, 32, 1.0), (320, 96, 0.125), (512, 512, 1.0 / math.sqrt(9 * 512))])
def test_pack_weights_bit_exact(gf, cuda_dev, cout, cin, scale):
    """gf_conv3x3_pack_weights == tf32_rne(float32(w * scale)) in the [9][Cout][Cin] layout, bit for bit, with exact ties of both
    kept-bit parities planted in a quarter of the weights (512 x 512 x 9 also runs the grid-stride loop more than once)."""
    g = torch.Generator().manual_seed(cout + cin)
    w = torch.randn(cout, cin, 3, 3, generator=g)
    bits = w.view(torch.int32)
    ties = torch.rand(w.shape, generator=g) < 0.25
    w = torch.where(ties, ((bits & -0x2000) | 0x1000).view(torch.float32), w)
    assert 0.2 < ((w.view(torch.int32) >> 13) & 1)[ties].float().mean().item() < 0.8         # odd and even kept bits both present
    got = _ops().conv3x3_pack(w.to(cuda_dev), scale=scale).cpu()
    want = _unpack_inverse(tf32_rne(w * torch.tensor(scale, dtype=torch.float32)))
    assert got.shape == (9, cout, cin)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_repeat_calls_and_batch_independence_bit_exact(gf, cuda_dev):
    """Two calls give bit-identical output, and each image of a batched call (persistent regime) equals that image convolved
    alone: a tile's summation order does not depend on which CTA runs it or on the batch."""
    H, W, cin, cout = 24, 48, 96, 320
    B = _persistent_batch(H, W, cout, _sms())
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    x = torch.randn(B, H, W, cin, generator=g, device=cuda_dev)
    wt = _ops().conv3x3_pack(torch.randn(cout, cin, 3, 3, generator=g, device=cuda_dev), scale=1.0 / math.sqrt(9 * cin))
    y1 = _conv_guarded(gf, x, wt)
    y2 = _conv_guarded(gf, x, wt)
    assert torch.equal(y1.view(torch.int32), y2.view(torch.int32))
    for b in (0, B // 2, B - 1):
        alone = _conv_guarded(gf, x[b:b + 1].contiguous(), wt)
        assert torch.equal(alone[0].view(torch.int32), y1[b].view(torch.int32)), b


def test_graph_replay_matches_eager(gf, cuda_dev):
    """ops.conv3x3_native captured in a CUDA graph (as bench.py replays it): new input copied into the static buffer, replayed,
    equals an eager call on the same input bit for bit."""
    ops = _ops()
    B, cin, cout, H, W = 4, 128, 128, 32, 32
    g = torch.Generator(device=cuda_dev).manual_seed(11)
    new = lambda: torch.randn(B, cin, H, W, generator=g, device=cuda_dev).contiguous(memory_format=torch.channels_last)
    wt = ops.conv3x3_pack(torch.randn(cout, cin, 3, 3, generator=g, device=cuda_dev), scale=1.0 / math.sqrt(9 * cin))
    x_static = new()
    with torch.no_grad():
        first = ops.conv3x3_native(x_static, wt).clone()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y_static = ops.conv3x3_native(x_static, wt)
        x_new = new()
        x_static.copy_(x_new)
        graph.replay()
        torch.cuda.synchronize()
        eager = ops.conv3x3_native(x_new, wt)
    torch.cuda.synchronize()
    assert not torch.equal(eager, first)
    assert torch.equal(y_static.contiguous().view(torch.int32), eager.contiguous().view(torch.int32))
