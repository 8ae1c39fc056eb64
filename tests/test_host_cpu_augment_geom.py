"""CPU checks of ADA's fractional geometry (SURVEY A.4 item 16): the fp64 definition of the resampler against a pixel-by-pixel numpy
restatement and against a restatement of ADA's own batch pipeline, the identity and adjoint identities, the custom autograd functions (kernels swapped for the definition), the sym6 taps,
the sampler, parse_augment("bgc"), the refusals of the two new gf_ops.h entry points and a CPU training run with "bgc" and R1."""
import json
import math
import os
import subprocess
import sys
from importlib import import_module

import numpy as np
import pytest
import torch

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
I6 = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]


def np_resample(x, code, tx, ty, A):
    """The four steps of include/gf_ops.h for one image [C, H, W], pixel by pixel: output pixel o reads V at the 12 x 12 2x-grid
    points q = 2o + k + 1, V[q] is U sampled bilinearly at nu = 2 (source index) of the point's preimage, U[nu] = 4 sum_m E[m] f f."""
    C, H, W = x.shape
    h = np.array(import_module(OPS).SYM6)
    f = h / h.sum()
    code &= 7
    if H != W:
        code &= 5
    tx, ty = max(-(W - 1), min(W - 1, tx)), max(-(H - 1), min(H - 1, ty))
    R = lambda i, N: -i if i < 0 else (2 * (N - 1) - i if i >= N else i)

    def E(c, my, mx):
        if not (-(H - 1) <= my <= 2 * (H - 1) and -(W - 1) <= mx <= 2 * (W - 1)):
            return 0.0
        return x[c, R(my, H), R(mx, W)]

    def U(c, ny, nx):
        if not (-2 * (H - 1) <= ny <= 4 * H - 3 and -2 * (W - 1) <= nx <= 4 * W - 3):
            return 0.0
        s = 0.0
        for my in range(-H, 2 * H):
            for mx in range(-W, 2 * W):
                ky, kx = ny + 5 - 2 * my, nx + 5 - 2 * mx
                if 0 <= ky < 12 and 0 <= kx < 12:
                    s += 4 * f[ky] * f[kx] * E(c, my, mx)
        return s

    def D(u, v):                                                         # the dihedral map in centred coordinates
        if code & 1:
            u = -u
        return [(u, v), (v, -u), (-u, -v), (-v, u)][code >> 1]
    y = np.zeros_like(x)
    for c in range(C):
        Uc = {}
        for oy in range(H):
            for ox in range(W):
                acc = 0.0
                for ky in range(12):
                    for kx in range(12):
                        px, py = ox - (W - 1) / 2 + (kx - 5) / 2, oy - (H - 1) / 2 + (ky - 5) / 2   # ADA's -0.5 shift
                        wx, wy = A[0] * px + A[1] * py + A[2], A[3] * px + A[4] * py + A[5]
                        sx, sy = D(wx, wy)
                        nx, ny = 2 * (sx - tx + (W - 1) / 2), 2 * (sy - ty + (H - 1) / 2)
                        x0, y0 = math.floor(nx), math.floor(ny)
                        v = 0.0
                        for dy in (0, 1):
                            for dx in (0, 1):
                                w = (nx - x0 if dx else 1 - (nx - x0)) * (ny - y0 if dy else 1 - (ny - y0))
                                key = (y0 + dy, x0 + dx)
                                if key not in Uc:
                                    Uc[key] = U(c, *key)
                                v += w * Uc[key]
                        acc += f[ky] * f[kx] * v
                y[c, oy, ox] = acc
    return y


@pytest.mark.parametrize("H,W", [(3, 3), (4, 6), (9, 7)])
def test_definition_against_the_pixel_by_pixel_restatement(H, W):
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(H * 10 + W)
    rows = [([1, 1, 0, 0], [0.6, 0.2, 0.3, -0.1, 0.7, -0.4]),            # zoom in, flip, shift into the mirror
            ([4, -W + 1, 2, 0], [1.7, -0.3, 1.1, 0.4, 1.4, 0.2]),        # zoom out
            ([0, 0, 0, 0], [1.0, 0.0, 2.5 * W, 0.0, 1.0, -1.5 * H]),      # translation into the zero region
            ([6, 1, -1, 0], [0.9, 0.5, -0.25, -0.5, 0.9, 0.75])]
    geom = torch.tensor([r[0] for r in rows], dtype=torch.int32)
    frac = torch.tensor([r[1] for r in rows])
    x = torch.randn(len(rows), 2, H, W, dtype=F64, generator=g)
    got = ops.augment_ref(x, geom, None, frac)
    for b, (gm, _) in enumerate(rows):
        want = np_resample(x[b].numpy(), gm[0], gm[1], gm[2], frac[b].double().tolist())
        assert np.abs(got[b].numpy() - want).max() < 1e-12, b


def _upfirdn(x, f, up=1, down=1, pad=(0, 0, 0, 0), flip_filter=False, gain=1.0):
    """StyleGAN2-ADA's reference upfirdn2d for a separable 1-D filter, restated: zero insertion, pad (negative = crop), the filter
    flipped unless flip_filter (a convolution), gain**0.5 per axis, then every down-th sample."""
    B, C, H, W = x.shape
    if up > 1:
        x = torch.nn.functional.pad(x.reshape(B, C, H, 1, W, 1), [0, up - 1, 0, 0, 0, up - 1]).reshape(B, C, H * up, W * up)
    px0, px1, py0, py1 = pad
    x = torch.nn.functional.pad(x, [max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)])
    x = x[:, :, max(-py0, 0): x.shape[2] - max(-py1, 0), max(-px0, 0): x.shape[3] - max(-px1, 0)]
    f = f * gain ** 0.5
    if not flip_filter:
        f = f.flip(0)
    x = x.reshape(B * C, 1, x.shape[2], x.shape[3])
    x = torch.nn.functional.conv2d(torch.nn.functional.conv2d(x, f.view(1, 1, 1, -1)), f.view(1, 1, -1, 1))
    x = x[:, :, ::down, ::down]
    return x.reshape(B, C, x.shape[2], x.shape[3])


def _ada_pipeline(x, G_inv, f):
    """ADA's batch geometry (AugmentPipe, the general-geometry part) restated: the batch margin from the image corners, an
    asymmetric reflect pad with its origin fix, upsample2d, affine_grid / grid_sample (align_corners=False, zeros) on the (N + 6) * 2
    grid, downsample2d with flip_filter=True and padding -2 * Hz_pad.  G_inv [B, 3, 3] in centred pixel coordinates.  Returns the
    image and the margins (mx0, mx1, my0, my1)."""
    B, C, H, W = x.shape
    T = lambda tx, ty: torch.tensor([[1, 0, tx], [0, 1, ty], [0, 0, 1]], dtype=F64)
    S = lambda sx, sy: torch.tensor([[sx, 0, 0], [0, sy, 0], [0, 0, 1]], dtype=F64)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    cp = torch.tensor([[-cx, -cy, 1], [cx, -cy, 1], [cx, cy, 1], [-cx, cy, 1]], dtype=F64)
    cp = G_inv @ cp.t()
    hz = 12 // 4
    margin = cp[:, :2, :].permute(1, 0, 2).flatten(1)
    margin = torch.cat([-margin, margin]).max(dim=1).values
    margin = margin + torch.tensor([hz * 2 - cx, hz * 2 - cy] * 2, dtype=F64)
    margin = margin.max(torch.zeros(4, dtype=F64)).min(torch.tensor([W - 1, H - 1] * 2, dtype=F64))
    mx0, my0, mx1, my1 = [int(v) for v in margin.ceil()]
    img = torch.nn.functional.pad(x, [mx0, mx1, my0, my1], mode="reflect")
    G = T((mx0 - mx1) / 2, (my0 - my1) / 2) @ G_inv
    img = _upfirdn(img, f, up=2, pad=(6, 5, 6, 5), gain=4.0)
    G = S(2, 2) @ G @ S(0.5, 0.5)
    G = T(-0.5, -0.5) @ G @ T(0.5, 0.5)
    shape = [B, C, (H + hz * 2) * 2, (W + hz * 2) * 2]
    G = S(2 / img.shape[3], 2 / img.shape[2]) @ G @ S(shape[3] / 2, shape[2] / 2)
    grid = torch.nn.functional.affine_grid(G[:, :2, :], shape, align_corners=False)
    img = torch.nn.functional.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    img = _upfirdn(img, f, down=2, pad=(-1, -1, -1, -1), flip_filter=True)
    return img, (mx0, mx1, my0, my1)


def _dihedral(code, H, W):
    code &= 7
    if H != W:
        code &= 5
    fl = -1.0 if code & 1 else 1.0
    R = [[[1, 0], [0, 1]], [[0, 1], [-1, 0]], [[-1, 0], [0, -1]], [[0, -1], [1, 0]]][code >> 1]
    return torch.tensor(R, dtype=F64) @ torch.diag(torch.tensor([fl, 1.0], dtype=F64))


@pytest.mark.parametrize("H,W", [(8, 8), (9, 7), (16, 12)])
def test_definition_against_adas_batch_pipeline(H, W):
    """ADA's pipeline on G_inv = T(-t) D F^-1 (the blit composed with the fractional map, as in include/gf_ops.h) agrees with the
    definition to fp64 round-off on every output pixel whose support lies inside ADA's batch margin: each bilinear tap of its 144
    samples lands on ADA's 2x grid and the up filter of that tap reads only ADA's padded rows and columns.  Elsewhere ADA reads the
    zeros beyond its margin where the definition reads one full reflection (SURVEY A.4 item 16)."""
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(H * 31 + W)
    c, s = math.cos(0.4), math.sin(0.4)
    rows = [([0, 0, 0, 0], [0.9 * c, -0.9 * s, 0.3, 0.9 * s, 0.9 * c, -0.7]),
            ([1, 1, -1, 0], [1.2, 0.1, -0.4, -0.2, 0.8, 0.25]),
            ([6 if H == W else 4, -2, 1, 0], [0.7, -0.3, 1.1, 0.35, 1.05, 0.0])]
    geom = torch.tensor([r[0] for r in rows], dtype=torch.int32)
    frac = torch.tensor([r[1] for r in rows])
    B = len(rows)
    x = torch.randn(B, 2, H, W, dtype=F64, generator=g)
    G_inv = torch.zeros(B, 3, 3, dtype=F64)
    for b, (gm, fr) in enumerate(rows):
        D = _dihedral(gm[0], H, W)
        A = torch.cat([frac[b].double().reshape(2, 3), torch.tensor([[0.0, 0.0, 1.0]], dtype=F64)])
        M = torch.eye(3, dtype=F64)
        M[:2, :2] = D
        G_inv[b] = torch.tensor([[1, 0, -gm[1]], [0, 1, -gm[2]], [0, 0, 1]], dtype=F64) @ M @ A
    ada, (mx0, mx1, my0, my1) = _ada_pipeline(x, G_inv, ops.sym6_filter())
    ours = ops.augment_ref(x, geom, None, frac)
    # the support test, per output pixel: nu = L q + e of its 144 points (q = 2o + 1 .. 2o + 12 per axis)
    L, e = ops.resample_map(geom, frac, H, W)
    k = torch.arange(1, 13, dtype=F64)
    qx = (2 * torch.arange(W, dtype=F64)[:, None] + k)[None, None, :, None, :, None]      # [1, 1, W, 1, 12, 1] ...
    qy = (2 * torch.arange(H, dtype=F64)[:, None] + k)[None, :, None, :, None, None]
    bl = lambda v: v[:, None, None, None, None, None]

    def inside(nu, N, m0, m1):                       # ADA's padded indices m in [-m0, N - 1 + m1]; its 2x grid nu + 2 m0 in [0, 2(N + m0 + m1))
        n0 = nu.floor()
        ok = torch.ones_like(nu, dtype=torch.bool)
        for n in (n0, n0 + 1):
            ok &= (torch.ceil((n - 6) / 2) >= -m0) & (torch.floor((n + 5) / 2) <= N - 1 + m1)
            ok &= (n + 2 * m0 >= 0) & (n + 2 * m0 <= 2 * (N + m0 + m1) - 1)
        return ok
    nux = bl(L[:, 0, 0]) * qx + bl(L[:, 0, 1]) * qy + bl(e[:, 0])
    nuy = bl(L[:, 1, 0]) * qx + bl(L[:, 1, 1]) * qy + bl(e[:, 1])
    okx = inside(nux, W, mx0, mx1)
    oky = inside(nuy, H, my0, my1)
    mask = (okx & oky).flatten(3).all(dim=3)                                             # [B, H, W]
    assert mask.float().mean() > 0.25, mask.float().mean()
    diff = (ada - ours).abs().amax(dim=1)
    assert diff[mask].max() < 1e-12, diff[mask].max()


def test_identity_map_is_the_blit_bit_for_bit():
    ops = import_module(OPS)
    x = torch.randn(5, 3, 6, 7, dtype=F64)
    geom = torch.tensor([[c, c - 2, 1 - c, 0] for c in range(5)], dtype=torch.int32)
    color = torch.randn(5, 12, dtype=F64)
    frac = torch.tensor([I6] * 5)
    assert torch.equal(ops.augment_ref(x, geom, color, frac), ops.augment_ref(x, geom, color))
    assert torch.equal(ops.augment(x, geom, color, frac), ops.augment(x, geom, color))
    assert torch.equal(ops.augment_adjoint_ref(x, geom, color, frac), ops.augment_adjoint_ref(x, geom, color))


@pytest.mark.parametrize("H,W", [(3, 3), (8, 8), (5, 9)])
def test_adjoint_identity(H, W):
    ops, tr = import_module(OPS), import_module(TRAIN)
    torch.manual_seed(H + W)
    B = 8
    geom, color = tr.sample_augment(("xflip", "xint", "hue"), 1.0, B, H, W, "cpu")
    frac = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, B, H, W, "cpu")
    frac[1] = torch.tensor(I6)
    lin = ops._linear_part(color.double())
    x, gy = torch.randn(B, 3, H, W, dtype=F64), torch.randn(B, 3, H, W, dtype=F64)
    lhs = (ops.augment_ref(x, geom, lin, frac) * gy).sum(dim=(1, 2, 3))
    rhs = (x * ops.augment_adjoint_ref(gy, geom, color.double(), frac)).sum(dim=(1, 2, 3))
    assert (lhs - rhs).abs().max() < 1e-12 * max(1.0, lhs.abs().max().item())


def test_out_of_domain_images_are_nan():
    ops = import_module(OPS)
    x = torch.randn(3, 1, 5, 5, dtype=F64)
    frac = torch.tensor([[0.5, 0, 0, 0, 0.5, 0], [17.0, 0, 0, 0, 1, 0], [1, 0, 0, 0, 1, 64 * 5 + 0.5]])
    y = ops.augment_ref(x, torch.zeros(3, 4, dtype=torch.int32), None, frac)
    assert torch.isfinite(y[0]).all() and torch.isnan(y[1:]).all()


def test_sym6_properties():
    h = torch.tensor(import_module(OPS).SYM6, dtype=F64)
    assert abs(h.sum().item() - math.sqrt(2)) < 1e-12
    for j in range(6):
        assert abs((h[: 12 - 2 * j] * h[2 * j:]).sum().item() - (1.0 if j == 0 else 0.0)) < 1e-12, j
    hi = h.flip(0) * torch.tensor([(-1.0) ** k for k in range(12)], dtype=F64)   # the high-pass: six vanishing moments
    k = torch.arange(12, dtype=F64)
    for p in range(6):
        assert abs((hi * k ** p).sum().item()) < 1e-9 * 11 ** p, p


@pytest.fixture
def host_kernels(monkeypatch):
    ops = import_module(OPS)
    calls = []

    def native(name, x, geom, color, frac):
        calls.append(name)
        f = ops.augment_ref if name == "gf_augment_resample_nchw" else ops.augment_adjoint_ref
        return f(x.detach(), geom, color, frac)
    monkeypatch.setattr(ops, "_augment_resample_native", native)
    return ops, calls


@pytest.mark.parametrize("colour", [False, True])
def test_autograd_functions_gradcheck_and_gradgradcheck(host_kernels, colour):
    ops, calls = host_kernels
    g = torch.Generator().manual_seed(7)
    geom = torch.tensor([[5, 2, -3, 0], [2, -1, 1, 0]], dtype=torch.int32)
    frac = torch.tensor([[0.9, 0.3, 0.2, -0.3, 1.1, -0.6], I6])
    color = torch.randn(2, 12, dtype=F64, generator=g) if colour else None
    x = torch.randn(2, 3, 5, 5, dtype=F64, generator=g, requires_grad=True)
    f = lambda t: ops._AugmentResample.apply(t, geom, color, frac)
    assert torch.autograd.gradcheck(f, (x,))
    assert torch.autograd.gradgradcheck(f, (x,))
    assert "gf_augment_resample_adjoint_nchw" in calls


# ------------------------------------------------------------------------------------------------ the sampler and the spec
def test_sampler_identity_at_p_zero_and_laws_at_p_one():
    tr, ops = import_module(TRAIN), import_module(OPS)
    assert tr.sample_augment_frac(tr.AUGMENT_OPS, 1.0, 4, 8, 8, "cpu") is None
    torch.manual_seed(0)
    B, H, W = 20000, 32, 24
    f0 = tr.sample_augment_frac(tr.GEOM_OPS, 0.0, B, H, W, "cpu")
    assert torch.equal(f0, torch.tensor(I6).expand(B, 6))
    assert torch.equal(tr.sample_augment_frac(tr.GEOM_OPS, torch.zeros(()), 8, H, W, "cpu"), torch.tensor(I6).expand(8, 6))
    s = tr.sample_augment_frac(("scale",), 1.0, B, H, W, "cpu").double()
    assert abs(torch.log2(1 / s[:, 0]).std().item() - 0.2) < 0.01 and torch.equal(s[:, 0], s[:, 4]) and not s[:, [1, 2, 3, 5]].any()
    a = tr.sample_augment_frac(("aniso",), 1.0, B, H, W, "cpu").double()
    assert abs(torch.log2(a[:, 4]).std().item() - 0.2) < 0.01 and (a[:, 0] * a[:, 4] - 1).abs().max() < 1e-6
    t = tr.sample_augment_frac(("xfrac",), 1.0, B, H, W, "cpu").double()
    assert abs(t[:, 2].std().item() / W - 0.125) < 0.005 and abs(t[:, 5].std().item() / H - 0.125) < 0.005
    r = tr.sample_augment_frac(("rotate",), 1.0, B, H, W, "cpu").double()
    th = torch.atan2(r[:, 3], r[:, 0])                                   # the sum of two U(-pi, pi) angles, mod 2 pi: uniform
    assert abs(th.std().item() - math.pi / math.sqrt(3)) < 0.03
    for p in (0.3, 0.7):
        rp = tr.sample_augment_frac(("rotate",), p, B, H, W, "cpu")
        rotated = (rp != torch.tensor(I6)).any(dim=1).double().mean().item()
        assert abs(rotated - p) < 0.015, p
    big = tr.sample_augment_frac(tr.GEOM_OPS, 1.0, 200000, 256, 256, "cpu")
    assert ops.frac_flags(big, 256, 256)[1].all()


def test_parse_augment_bgc():
    tr = import_module(TRAIN)
    assert tr.parse_augment("bc") == tr.AUGMENT_OPS and len(tr.AUGMENT_OPS) == 8
    assert tr.parse_augment("bgc") == tr.AUGMENT_OPS[:3] + tr.GEOM_OPS + tr.AUGMENT_OPS[3:]
    assert tr.parse_augment("hue,xfrac, xflip,rotate") == ("xflip", "rotate", "xfrac", "hue")
    with pytest.raises(ValueError):
        tr.parse_augment("scale,cutout")


def test_bad_frac_raises():
    ops = import_module(OPS)
    x, g = torch.zeros(2, 3, 4, 4), torch.zeros(2, 4, dtype=torch.int32)
    for bad in (torch.zeros(2, 5), torch.zeros(3, 6), torch.zeros(2, 3, 2)):
        with pytest.raises(ValueError):
            ops.augment(x, g, None, bad)


_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A = 0x10000
out = []
for name in ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"):
    fn = getattr(lib, name)
    for args in ([A, A, A, A, A, 2, 3, 8, 8, None], [A, A, A, A, None, 2, 1, 8, 8, None],
                 [None, A, A, A, A, 2, 3, 8, 8, None], [A, None, A, A, A, 2, 3, 8, 8, None], [A, A, None, A, A, 2, 3, 8, 8, None],
                 [A, A, A, None, A, 2, 3, 8, 8, None], [A, A, A, A, A, 0, 3, 8, 8, None], [A, A, A, A, A, 2, 3, 8, 1, None],
                 [A, A, A, A, A, 2, 4, 8, 8, None], [A, A, A, A, None, 2, 3, 40000, 8, None]):
        out.append([name, fn(*args), lib.gf_last_error().decode()])
print(json.dumps(out))
"""


def test_entry_points_refuse_bad_arguments():
    gf = import_module("gansformer_b200")
    assert {"gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"} <= set(gf._lib.OPS_EXPORTS)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    want = [-3, -3, -1, -1, -1, -1, -1, -2, -2, -2]
    for name in ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"):
        got = [(rc, msg) for n, rc, msg in out if n == name]
        assert [rc for rc, _ in got] == want, (name, got)
        assert all(name in msg for rc, msg in got if rc != -3)
        assert "frac" in got[5][1] and "C == 3" in got[8][1]


def test_trainer_bgc_with_r1(gf):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", d_reg_interval=2, augment="bgc", augment_p=0.8, ada_target=0.6,
                                              ada_interval=1))
    g = torch.Generator().manual_seed(3)
    z, reals = torch.randn(4, 5, 16, generator=g), torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    seen = []
    d_fwd = D.forward
    D.forward = lambda img, c=None: seen.append(img) or d_fwd(img)
    stats = [trainer.step(z, reals) for _ in range(2)]
    assert stats[0].r1 > 0 and stats[1].r1 == 0
    assert all(math.isfinite(v) for s in stats for v in (s.loss_d, s.loss_g, s.r1, s.augment_p))
    assert len(seen) == 6 and seen[0].requires_grad and torch.isfinite(seen[0]).all()
