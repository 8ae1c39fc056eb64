"""ADA's fractional resampler on an H100, bit for bit (``pytest -m gpu``; DESIGN 4.12).

gf_augment_resample_nchw and gf_augment_resample_adjoint_nchw through the C ABI, outputs between NaN guards, against
oracle/augment_resample.py, which restates both kernels' fp32 arithmetic (rounding, the tile plan and the adjoint's chunk partition
included).  Every comparison is assert_exact; an image outside the domain must be NaN in every element.  The maps are chosen so
that the oracle's host check passes (every product in res_map and the adjoint's det exact in fp32, whatever nvcc contracts): dyadic
2 x 2 parts, any fp32 translation.
"""
from importlib import import_module

import numpy as np
import pytest
import torch

from oracle import augment_resample as oar
from tests.guards import Guarded, assert_exact
from tests.test_gpu_ops_exact import _call, _stream

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
FWD, ADJ = "gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"
BGC_NO_R90 = ("xflip", "xint", "scale", "rotate", "aniso", "xfrac", "brightness", "contrast", "lumaflip", "hue", "saturation")


def run(gf, name, x, geom, frac, color, dev):
    B, C, H, W = x.shape
    out = Guarded((B, C, H, W), dev)
    xd, gd, fd = (t.contiguous().to(dev) for t in (x.float(), geom.to(torch.int32), frac.float()))
    cd = None if color is None else color.float().contiguous().to(dev)
    _call(gf, name, xd.data_ptr(), out.ptr(), gd.data_ptr(), fd.data_ptr(), None if cd is None else cd.data_ptr(), B, C, H, W,
          _stream(dev))
    return out.check(name).cpu()


def check(gf, dev, what, x, geom, frac, color=None, adjoint=True, fstats=None, astats=None):
    """Both kernels against the oracle, bit for bit (NaN exactly where the oracle has NaN)."""
    x, geom, frac = x.float(), geom.to(torch.int32), frac.float()
    color = None if color is None else color.float()
    pairs = [(FWD, oar.forward, fstats)] + ([(ADJ, oar.adjoint, astats)] if adjoint else [])
    for name, fn, st in pairs:
        want = torch.from_numpy(fn(x, geom, frac, color, stats=st))
        got = run(gf, name, x, geom, frac, color, dev)
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan), f"{what} {name}: NaN pattern"
        assert_exact(got[~nan], want[~nan], f"{what} {name}")


def images(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, H, W, generator=g)


def quantised(frac):
    """A sampled map with its 2 x 2 part rounded to multiples of 2^-8 (entries below 4 in magnitude: at most 10 significant bits,
    so every product res_map and det form is exact in fp32); the translation stays as drawn."""
    f = frac.clone().double()
    f[:, [0, 1, 3, 4]] = torch.round(f[:, [0, 1, 3, 4]] * 256) / 256
    return f.float()


def maps(rows):
    return torch.tensor(rows, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ dyadic maps
@pytest.mark.parametrize("k", [-3, -2, -1, 1, 2, 3])
def test_dyadic_zooms(gf, cuda_dev, k):
    """Zooms by 2^k, isotropic and anisotropic (2^k x 2^-1 and 2^-k x 2), with sub-pixel and dyadic translations.  k = 3 is a
    zoom-out by 8 (the direct per-pixel path), k = -3 a zoom-in by 8 (the adjoint in many chunks)."""
    z = 2.0 ** k
    B, C, H, W = 4, 2, 40, 36
    frac = maps([[z, 0, 0.0, 0, z, 0.0], [z, 0, 0.25, 0, z, -0.375], [z, 0, 1.5, 0, 0.5, -2.0], [1 / z, 0, -0.125, 0, 2, 0.75]])
    geom = torch.tensor([[0, 0, 0, 0], [1, 3, -2, 0], [4, -1, 5, 0], [5, 0, 1, 0]], dtype=torch.int32)
    fs, as_ = {}, {}
    check(gf, cuda_dev, f"zoom 2^{k}", images(B, C, H, W, 10 + k), geom, frac, fstats=fs, astats=as_)
    if k == 3:
        assert fs["direct"] > 0
    if k == -3:
        assert as_["chunks"] > 1


def test_zoom_in_by_8_in_many_chunks(gf, cuda_dev):
    B, C, H, W = 2, 1, 64, 64
    frac = maps([[0.125, 0, 0.5, 0, 0.125, -0.25], [0.125, 0, 0, 0, 0.25, 3.0]])
    geom = torch.tensor([[0, 0, 0, 0], [6, 5, -7, 0]], dtype=torch.int32)
    st = {}
    check(gf, cuda_dev, "zoom-in 8, 64x64", images(B, C, H, W, 1), geom, frac, astats=st)
    assert st["chunks"] >= 9 and st["chunk_adds"] >= 2, st


def test_both_forward_paths_and_the_threshold(gf, cuda_dev):
    """A zoom-out by 3.75 at 48 x 48: some tiles fit the shared-memory plan and others take the direct path; one plan tile asks for
    between RS_CAP - 256 and RS_CAP floats, so a threshold off by one tile changes its bits."""
    B, C, H, W = 2, 3, 48, 48
    frac = maps([[3.75, 0, 0.3, 0, 3.75, -0.2]] * B)
    geom = torch.tensor([[0, 0, 0, 0], [0, 0, 0, 0]], dtype=torch.int32)
    m = oar.ResMap(frac[0].numpy(), geom[0].numpy(), H, W)
    plan, foot = oar.tile_plan(m, H, W, footprint=True)
    assert (plan == "plan").any() and (plan == "direct").any()
    assert ((plan == "plan") & (foot > oar.CAP - 256)).any()
    color = torch.randn(B, 12, generator=torch.Generator().manual_seed(2))
    st = {}
    check(gf, cuda_dev, "zoom-out 3.75", images(B, C, H, W, 2), geom, frac, color, fstats=st)
    assert st["plan"] > 0 and st["direct"] > 0


@pytest.mark.parametrize("H,W", [(2, 2), (3, 3), (5, 7), (20, 18), (37, 23), (16, 48)])
def test_general_dyadic_maps(gf, cuda_dev, H, W):
    """2 x 2 parts with det = +-2^k, so that the preimages are parallelograms; odd sizes, tiny images, non-square grids.  The tiny
    images caught the adjoint's transposed down filter summing past the image's last column and row (DESIGN 4.12)."""
    check(gf, cuda_dev, f"general {H}x{W}", *_general(H, W))


def _general(H, W):
    rows = [[1, 1, 0.5, -1, 1, -0.25],            # det 2
            [1, 1, 0, 1, -1, 0.125],              # det -2
            [0.75, 0.5, -0.3, 0.5, 1, 0.6],       # det 0.5
            [2, 1, 1.0, 1, 1, -1.0],              # det 1
            [0.25, -0.5, 0.0, 0.5, 0.5, 0.0],     # det 0.375 = 3 / 8: still exact (dyadic inverse not needed)
            [-1.5, 0.5, 0.1, 0.25, 0.75, 0.2]]    # det -1.25
    B = len(rows)
    frac = maps(rows)
    geom = torch.tensor([[i, (-1) ** i * i, i - 2, 0] for i in range(B)], dtype=torch.int32)
    return images(B, 1, H, W, H * 100 + W), geom, frac


@pytest.mark.parametrize("square", [True, False])
def test_every_dihedral_code_and_translations(gf, cuda_dev, square):
    """All 8 codes and codes above 7 (masked to 3 bits; bit 1 cleared on a non-square grid), integer translations 0, +-1,
    +-(N - 1) and beyond (clamped), with a fractional map that keeps the image in the resampler."""
    H, W = (24, 24) if square else (20, 28)
    codes = list(range(8)) + [9, 14, 255, -1]
    ts = [(0, 0), (1, -1), (W - 1, -(H - 1)), (-(W - 1), H - 1), (W + 3, -(H + 5)), (-100, 100)]
    geom = torch.tensor([[c, ts[i % len(ts)][0], ts[i % len(ts)][1], 0] for i, c in enumerate(codes)], dtype=torch.int32)
    B = len(codes)
    frac = maps([[1, 0.5, 0.25, -0.5, 1, -0.5] if i % 2 else [0.5, 0, -3.25, 0, 1.25, 2.5] for i in range(B)])
    color = torch.randn(B, 12, generator=torch.Generator().manual_seed(3))
    check(gf, cuda_dev, f"codes {H}x{W}", images(B, 3, H, W, 3), geom, frac, color)


def test_fractional_translations_at_and_beyond_the_edge(gf, cuda_dev):
    """Sub-pixel translations, translations that move the whole image out of U's extent (every tile reads zeros) and ones at the
    domain's limit 64 max(H, W)."""
    H, W = 18, 22
    rows = [[1, 0, 0.5, 0, 1, 0.0], [1, 0, -0.25, 0, 1, 0.75], [1, 0, 21.0, 0, 1, 0.0], [1, 0, 23.5, 0, 1, -17.25],
            [1, 0, -60.0, 0, 1, 30.0], [0.5, 0, 64.0 * W, 0, 0.5, -64.0 * W], [2, 0, 0.0625, 0, 2, -0.0625]]
    frac = maps(rows)
    geom = torch.zeros(len(rows), 4, dtype=torch.int32)
    st = {}
    check(gf, cuda_dev, "translations", images(len(rows), 2, H, W, 4), geom, frac, fstats=st)
    assert st["empty"] > 0


@pytest.mark.parametrize("C,colour", [(1, False), (2, False), (3, False), (3, True)])
def test_channels_and_colour(gf, cuda_dev, C, colour):
    B, H, W = 3, 33, 17
    frac = maps([[0.75, 0.25, 0.3, -0.25, 0.75, -0.7], [1.5, 0, 0, 0, 0.5, 0.125], [1, -0.5, 2.0, 0.5, 1, 0.0]])
    geom = torch.tensor([[1, 2, 0, 0], [2, -3, 4, 0], [0, 0, 0, 0]], dtype=torch.int32)
    color = torch.randn(B, 12, generator=torch.Generator().manual_seed(5)) if colour else None
    check(gf, cuda_dev, f"C={C} colour={colour}", images(B, C, H, W, 5 + C), geom, frac, color)


def test_batch_beyond_the_grid(gf, cuda_dev):
    """300 single-tile images: more tiles than the grid's 2 x SMs CTAs, so every CTA loops."""
    B, C, H, W = 300, 1, 16, 16
    g = torch.Generator().manual_seed(6)
    frac = torch.round(torch.randn(B, 6, generator=g) * 16) / 64
    frac[:, [0, 4]] += 1
    geom = torch.stack([torch.randint(0, 8, (B,), generator=g), torch.randint(-3, 4, (B,), generator=g),
                        torch.randint(-3, 4, (B,), generator=g), torch.zeros(B, dtype=torch.int64)], 1).to(torch.int32)
    check(gf, cuda_dev, "300 images", images(B, C, H, W, 6), geom, frac.float())


def test_mixed_batch_with_identity_and_out_of_domain_images(gf, cuda_dev):
    B, H, W = 8, 24, 20
    frac = maps([[1, 0, 0, 0, 1, 0], [0.5, 0.25, 0.1, 0, 1, 0], [float("nan"), 0, 0, 0, 1, 0], [1, -0.0, 0.0, 0, 1, -0.0],
                 [20.0, 0, 0, 0, 1, 0], [1, 0, 0, 0, 1 / 32, 0], [1, 0, 64 * 24 + 1, 0, 1, 0], [2, 0, -0.5, 0, 0.5, 0.5]])
    geom = torch.tensor([[i % 8, i - 4, 3 - i, 0] for i in range(B)], dtype=torch.int32)
    color = torch.randn(B, 12, generator=torch.Generator().manual_seed(7))
    for col in (None, color):
        check(gf, cuda_dev, f"mixed colour={col is not None}", images(B, 3, H, W, 7), geom, frac, col)


# ------------------------------------------------------------------------------------------------ sampled "bgc", quantised
@pytest.mark.parametrize("B,H,W,adjoint", [(16, 16, 16, True), (4, 64, 64, True), (2, 256, 256, False), (4, 40, 72, True)],
                         ids=lambda v: str(v))
def test_bgc_quantised(gf, cuda_dev, B, H, W, adjoint):
    tr = import_module(TRAIN)
    torch.manual_seed(B * 7 + H + W)
    spec = tr.parse_augment("bgc") if H == W else BGC_NO_R90
    geom, color = tr.sample_augment(spec, 1.0, B, H, W, "cpu")
    frac = quantised(tr.sample_augment_frac(spec, 1.0, B, H, W, "cpu"))
    for b in range(B):
        assert oar.ResMap(frac[b].numpy(), geom[b].numpy(), H, W).ok
    check(gf, cuda_dev, f"bgc {B}x{H}x{W}", images(B, 3, H, W, H + W), geom, frac, color, adjoint=adjoint)
