"""Minimal G/D training step around the attention hot path (SURVEY row f2, BASELINE configs[3]).

What the reference does (expected upstream ``src/training/training_loop.py``, ``src/training/loss.py``,
``src/training/network.py: D_Stylegan2``; none of them is in the checkout -- /root/reference/.SUBMODULES.json:2):
non-saturating logistic losses, R1 gradient penalty on the reals with lazy regularisation, Adam(beta1 = 0,
beta2 = 0.99), an exponential moving average of the generator weights, data parallelism over GPUs with a summed
gradient all-reduce.  Here: one process per GPU, gradients averaged through ONE flat fp32 buffer per network
(``dist.allreduce_gradients``: NCCL over NVLink/NVSwitch, gloo in the CPU tests).  The only other collective is the two-float sum of
the ADA accumulators below.

The attention layers run their CUDA forward.  Their backward (``autograd.py``) is the hand-written stage-T backward kernel for
simplex layers, the same kernel plus the pass-A backward kernels for duplex layers with attention dropout, and the torch
composite for the rest (duplex layers without dropout, instance / batch norm, multi-head).  The discriminator is PyTorch plumbing
(cuDNN convolutions, the native FIR); with ``transformer=True`` it also has the paper's bipartite attention: duplex layers
aggregating the image into learned latents that are carried from layer to layer and concatenated to the final features.  Those
layers run the CUDA forward and the duplex kernel backward (``BipartiteAttention.kernel_backward``), and by default the torch
composite in the R1 pass, which needs their second derivative; with ``Discriminator(r1_kernels=True)`` the R1 pass runs them on the
kernels too, differentiated twice through the double-backward kernels (``BipartiteAttention.kernel_double_backward``).

``TrainConfig.pl_weight > 0`` adds StyleGAN2's path-length regularisation of the generator, lazily, every ``g_reg_interval``-th
step after the G update: on the first B // pl_batch_shrink latents, the gradient of <G.synthesis(ws), noise / sqrt(H W)> with respect
to the dlatents ws [B, k+1, D], its length over the k+1 latent components (SURVEY A.4 item 12), and the squared distance of that
length to its running mean.  The backward of that gradient needs the generator's second derivative: the attention layers give it
through the double-backward kernels (``gf_attn_simplex_bwd_vjp_ex``, with the forward's dropout mask) or, on the composite route, torch
autograd.  Off by default.

``TrainConfig.style_mixing > 0`` adds StyleGAN2's style mixing (SURVEY A.4 item 13): each generator forward of the D and G phases
maps z and a second draw z2, and feeds the synthesis per-layer latents that switch from the first to the second at a cutoff drawn
per minibatch on the device (``mixing_cutoff``, ``mix_latents``).  The path-length phase, the w_avg update and inference do not
mix.  Off by default: with 0 the step makes the same calls and draws the same random numbers as without the option.

Class-conditional training (SURVEY A.4 item 14): a generator and a discriminator built with the same ``c_dim > 0`` take labels.
``step(z, reals, gen_c, real_c)``: the fakes of both phases, the path-length phase (on gen_c[:B']), both style-mixing draws and the
w_avg update use gen_c, the discriminator's real logits and R1 use real_c.  The labels are sharded like z and reals.  With
``c_dim = 0`` the labels are ignored and the step makes the same calls as before.

``TrainConfig.augment`` adds adaptive discriminator augmentation (ADA, Karras et al. 2020; SURVEY A.4 item 15): every image batch
the discriminator sees -- the reals of the D phase (R1 included: the gradient is taken with respect to the un-augmented reals,
through the augmentation), the fakes of the D phase and the fakes of the G phase -- goes through ``ops.augment`` with per-image
parameters of its own (``sample_augment``): integer blits (x flips, 90-degree rotations, integer translations with mirror padding)
and a colour matrix, on the gf_augment_nchw kernel and its adjoint.  The strength p is a device tensor (``Trainer.augment_p``); with
``ada_target`` it adapts to the sign of the real logits, summed over ranks, every ``ada_interval`` steps, without a host sync.  Not
in the path-length phase, the w_avg update or inference.  Off by default: with "" the step makes the same calls and draws the same
random numbers as without the option.  "bgc" adds ADA's fractional geometry (``sample_augment_frac``, SURVEY A.4 item 16); "bgcf" and
"bgcfn" add, after it, ADA's image-space filtering and additive noise (``sample_augment_filter``, ``ops.augment_filter``, SURVEY A.4
item 17).
"""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, dist as gdist
from .attention import BipartiteAttention
from .autograd import _e, composite_forward
from .networks import FullyConnected, nf
from ._state import bump_weights_epoch
from .self_attention import ImageSelfAttention
from .ops import IMGFILTER_HALO, augment, augment_filter, fir4, fir_filter, upfirdn2d_ref

SQRT2 = math.sqrt(2.0)


class EqConv2d(nn.Module):
    """Equalised-LR convolution (+ optional FIR-blurred stride-2 downsampling, + bias + leaky-ReLU * sqrt 2)."""

    def __init__(self, in_ch: int, out_ch: int, kernel: int, down: bool = False, bias: bool = True, act: str = "lrelu"):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_ch, in_ch, kernel, kernel))
        self.bias = nn.Parameter(torch.zeros(out_ch)) if bias else None
        self.wgain = 1.0 / math.sqrt(in_ch * kernel * kernel)
        self.down, self.act, self.kernel = down, act, kernel
        self.register_buffer("fir", fir_filter(), persistent=False)

    def forward(self, x):
        w = self.weight * self.wgain
        if self.down:
            p = (self.fir.shape[0] - 2) + (self.kernel - 1)          # upfirdn padding of StyleGAN2's conv_downsample_2d
            if p % 2 == 0:
                x = fir4(x, self.fir, p // 2)                          # native FIR (forward, backward, double backward for R1)
            else:
                x = upfirdn2d_ref(x, self.fir.to(x.dtype), pad=((p + 1) // 2, p // 2, (p + 1) // 2, p // 2))
            x = F.conv2d(x, w, stride=2)
        else:
            x = F.conv2d(x, w, padding=self.kernel // 2)
        if self.bias is not None:
            x = x + self.bias[None, :, None, None]
        return F.leaky_relu(x, 0.2) * SQRT2 if self.act == "lrelu" else x


def _d_attention(C: int, resolution: int, att: dict) -> BipartiteAttention:
    """One duplex attention layer of the discriminator (SURVEY A.4 item 11).  The shape is checked against the library here, so an
    unsupported one raises at construction with the library's own message."""
    if att["norm"] not in ("layer", None, "none"):
        raise ValueError(f"discriminator attention runs the duplex kernel backward: norm 'layer' or None, got {att['norm']!r}")
    k, D = att["components_num"], att["latent_dim"]
    _lib.workspace_bytes(_lib.make_desc(1, resolution, resolution, C, k, D, norm=att["norm"], integration=att["integration"],
                                        pos_dim=D if att["use_pos"] else 0, duplex=1, flags=_lib.FLAG_IMG2LTNT))
    m = BipartiteAttention(C, D, k, integration=att["integration"], norm=att["norm"], kmeans=True, kmeans_iters=1, img2ltnt=True,
                           use_pos=att["use_pos"], exact_fp32=att["exact_fp32"])
    m.kernel_backward = True          # no generator gradients to preserve: the duplex kernel backward from the start
    m.kernel_double_backward = att.get("r1_kernels", False)
    return m


def _attend(att: BipartiteAttention, x: torch.Tensor, y: torch.Tensor, composite: bool):
    """x [B,C,H,W] (channels-last memory), Y [B,k,D] -> (attended x, the Y carried to the next attention layer).

    The carry is the layer's own value input, Y <- LN(Y) (1 + Cen Wi2l_e + bi2l), with Cen the layer's centroids.  ``composite``
    (the R1 pass) runs the layer as torch ops (``composite_forward``), which can be differentiated twice, unless the layer's
    kernel backward has a derivative of its own (``kernel_double_backward``)."""
    xt = x.permute(0, 2, 3, 1).contiguous()                            # [B,H,W,C]: a view of a channels-last activation
    if composite and not att.kernel_double_backward:
        out, cen = composite_forward(xt, y, att.param_dict(), integration=att.integration, norm=att.norm, duplex=True,
                                     use_pos=att.use_pos, img2ltnt=True)
    else:
        out, _, cen = att(xt, y)
    ym = y.mean(dim=2, keepdim=True)
    yn = (y - ym) * torch.rsqrt(((y - ym) ** 2).mean(dim=2, keepdim=True) + 1e-8)
    y = (yn * (1.0 + cen @ _e(att.wi2l) + att.bi2l)).contiguous()
    return out.permute(0, 3, 1, 2), y


class DiscriminatorBlock(nn.Module):
    """Residual block; with ``attention`` (a dict of the discriminator's attention options) a duplex attention layer follows conv0
    and another follows conv1, on the main path before the residual sum."""

    def __init__(self, in_ch: int, out_ch: int, resolution: Optional[int] = None, attention: Optional[dict] = None):
        super().__init__()
        self.conv0 = EqConv2d(in_ch, in_ch, 3)
        self.conv1 = EqConv2d(in_ch, out_ch, 3, down=True)
        self.skip = EqConv2d(in_ch, out_ch, 1, down=True, bias=False, act="linear")
        self.att0 = _d_attention(in_ch, resolution, attention) if attention else None
        self.att1 = _d_attention(out_ch, resolution // 2, attention) if attention else None

    def forward(self, x, y=None, composite: bool = False):
        """x [B,C,H,W], Y [B,k,D] | None -> (x', Y')."""
        if self.att0 is None:
            return (self.skip(x) + self.conv1(self.conv0(x))) * (1.0 / SQRT2), y
        h, y = _attend(self.att0, self.conv0(x), y, composite)
        h, y = _attend(self.att1, self.conv1(h), y, composite)
        return (self.skip(x) + h) * (1.0 / SQRT2), y


class Discriminator(nn.Module):
    """StyleGAN2 residual discriminator (config f channel schedule), images [B,3,R,R] -> logits [B].

    ``transformer=True`` adds the GANsformer discriminator's bipartite attention (SURVEY A.4 item 11): learned aggregator latents
    ``latents`` [k, D] are broadcast to Y [B,k,D]; every block whose input resolution lies in [d_start_res, d_end_res] runs a
    duplex layer (one k-means iteration, g_img2ltnt) after conv0 and after conv1; Y is carried from layer to layer and fc0 takes
    [flatten(x), flatten(Y)].  The layers run the CUDA forward and the duplex kernel backward; when the image and the parameters
    both require grad under grad mode (the R1 pass), they run ``composite_forward`` instead, which has a second derivative.
    ``r1_kernels=True`` keeps the R1 pass on the kernels: the kernel backward, run with create_graph=True, is differentiated by
    the double-backward kernels, and only each layer's input and incoming gradient are kept for the second pass instead of the
    composite's [B,n,C] projections.  The R1 gradients then differ from the default route by round-off.

    ``c_dim > 0`` (SURVEY A.4 item 14, StyleGAN2's projection discriminator): fc1 has c_dim outputs and ``D(img, c)`` returns the
    sum over them weighted by the labels c [B, c_dim].  ``c_dim = 0`` (the default) is the unconditional network, and ignores c.

    ``img2img = r`` (SURVEY A.4 item 18): image self-attention (``ImageSelfAttention``, with the discriminator's integration, norm and
    use_pos, positional width latent_dim) on the activation entering the block of input resolution r, in 8 .. resolution.  Its R1
    pass differentiates the layer's backward through the torch composite, which holds n x n tensors; with ``r1_kernels=True`` it
    runs on the double-backward kernel instead (``ImageSelfAttention.kernel_double_backward``), which holds none."""

    def __init__(self, resolution: int = 256, fmap_base: int = 16384, fmap_max: int = 512, mbstd_group: int = 4,
                 transformer: bool = False, components_num: int = 16, latent_dim: int = 32, d_start_res: int = 8,
                 d_end_res: Optional[int] = None, integration: str = "mul", norm: Optional[str] = "layer", use_pos: bool = True,
                 exact_fp32: bool = False, r1_kernels: bool = False, c_dim: int = 0, img2img: int = 0):
        super().__init__()
        if c_dim < 0:
            raise ValueError(f"c_dim must be >= 0, got {c_dim}")
        if img2img and not (8 <= img2img <= resolution and img2img & (img2img - 1) == 0):
            raise ValueError(f"img2img must be 0 (off) or a block resolution in 8 .. {resolution}, got {img2img}")
        self.resolution, self.mbstd_group, self.transformer, self.c_dim = resolution, mbstd_group, transformer, int(c_dim)
        log2 = int(math.log2(resolution))
        d_end_res = resolution if d_end_res is None else d_end_res
        att = dict(components_num=components_num, latent_dim=latent_dim, integration=integration, norm=norm, use_pos=use_pos,
                   exact_fp32=exact_fp32, r1_kernels=r1_kernels) if transformer else None
        self.fromrgb = EqConv2d(3, nf(resolution, fmap_base, fmap_max), 1)
        self.block_resolutions = [2 ** i for i in range(log2, 2, -1)]                    # input resolution of each block
        self.blocks = nn.ModuleList([DiscriminatorBlock(nf(2 ** i, fmap_base, fmap_max), nf(2 ** (i - 1), fmap_base, fmap_max), 2 ** i,
                                                        att if d_start_res <= 2 ** i <= d_end_res else None)
                                     for i in range(log2, 2, -1)])
        c4 = nf(4, fmap_base, fmap_max)
        self.conv4 = EqConv2d(c4 + 1, c4, 3)
        self.fc0 = FullyConnected(c4 * 16 + (components_num * latent_dim if transformer else 0), c4, act="lrelu")
        self.fc1 = FullyConnected(c4, max(c_dim, 1))
        if transformer:
            self.latents = nn.Parameter(torch.randn(components_num, latent_dim))
        self.img2img_res = int(img2img)
        if img2img:
            self.img2img = ImageSelfAttention(nf(img2img, fmap_base, fmap_max), latent_dim, integration=integration, norm=norm,
                                              use_pos=use_pos, exact_fp32=exact_fp32)
            self.img2img.kernel_double_backward = bool(r1_kernels)

    def forward(self, img, c: Optional[torch.Tensor] = None):
        if self.c_dim > 0:
            if c is None:
                raise ValueError(f"this discriminator is conditional (c_dim={self.c_dim}): labels c [B, {self.c_dim}] are required")
            c = torch.as_tensor(c)
            if c.dim() != 2 or c.shape[0] != img.shape[0] or c.shape[1] != self.c_dim:
                raise ValueError(f"c must be [{img.shape[0]}, {self.c_dim}], got {tuple(c.shape)}")
        x = self.fromrgb(img.contiguous(memory_format=torch.channels_last))
        y, composite = None, False
        if self.transformer:
            y = self.latents[None].expand(img.shape[0], -1, -1).contiguous()
            composite = torch.is_grad_enabled() and img.requires_grad and any(p.requires_grad for p in self.parameters())
        for blk, res in zip(self.blocks, self.block_resolutions):
            if res == self.img2img_res:
                x = self.img2img(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2)
            x, y = blk(x, y, composite)
        B, C, H, W = x.shape                                            # minibatch standard deviation, one feature map
        G = min(self.mbstd_group, B)
        while B % G:
            G -= 1
        s = x.reshape(G, B // G, C, H, W)
        s = (s - s.mean(dim=0, keepdim=True)).square().mean(dim=0).add(1e-8).sqrt().mean(dim=[1, 2, 3])
        s = s.reshape(1, B // G, 1, 1).expand(G, -1, H, W).reshape(B, 1, H, W)
        x = self.conv4(torch.cat([x, s], dim=1)).reshape(B, -1)
        if y is not None:
            x = torch.cat([x, y.reshape(B, -1)], dim=1)
        out = self.fc1(self.fc0(x))
        if self.c_dim > 0:                                              # projection onto the labels
            return (out * c.to(device=out.device, dtype=out.dtype)).sum(dim=1)
        return out.reshape(B)


@dataclass
class TrainConfig:
    lr: float = 0.002
    r1_gamma: float = 10.0
    d_reg_interval: int = 16            # lazy R1: every 16th discriminator step
    ema_kimg: float = 10.0
    noise_mode: str = "random"
    bucket_mb: float = 32.0             # gradient all-reduce bucket size (MB of fp32 gradients)
    w_avg_beta: float = 0.995           # decay of the running mean of the mapping outputs (truncation trick)
    pl_weight: float = 0.0              # path-length regularisation of G (StyleGAN2: 2); 0 = off
    g_reg_interval: int = 4             # lazy path-length regularisation: every 4th generator step
    pl_batch_shrink: int = 2            # the path-length phase runs on the first B // 2 latents
    pl_decay: float = 0.01              # decay of the running mean of the path lengths
    style_mixing: float = 0.0           # probability of style mixing per generator forward (StyleGAN2 / GANsformer: 0.9); 0 = off
    augment: str = ""                   # discriminator augmentation: "" = off, "bc" = all of AUGMENT_OPS, "bgc" = those and GEOM_OPS,
                                        # "bgcf" / "bgcfn" = those and "imgfilter" / both FILTER_OPS, or a comma list of names
    augment_p: float = 0.0              # starting augmentation strength p
    ada_target: Optional[float] = None  # adaptive p: target of the mean sign of the real logits (ADA: 0.6); None = p stays put
    ada_interval: int = 4               # steps between updates of p
    ada_kimg: float = 500.0             # p can go from 0 to 1 in this many thousand images


AUGMENT_OPS = ("xflip", "rotate90", "xint", "brightness", "contrast", "lumaflip", "hue", "saturation")
GEOM_OPS = ("scale", "rotate", "aniso", "xfrac")                     # ADA's general geometry (SURVEY A.4 item 16)
_ADA_ORDER = AUGMENT_OPS[:3] + GEOM_OPS + AUGMENT_OPS[3:]
FILTER_OPS = ("imgfilter", "noise")                                  # ADA's image-space filtering and noise (SURVEY A.4 item 17)
_ALL_OPS = _ADA_ORDER + FILTER_OPS
_PRESETS = {"bc": AUGMENT_OPS, "bgc": _ADA_ORDER, "bgcf": _ADA_ORDER + FILTER_OPS[:1], "bgcfn": _ALL_OPS}
IMGFILTER_EXPECTED_POWER = (10.0, 1.0, 1.0, 1.0)                     # ADA's 1/f power spectrum of the four bands, over 13
NOISE_STD = 0.1


def parse_augment(spec: str) -> tuple:
    """TrainConfig.augment -> the enabled transforms, in ADA's order: "" none, "bc" the eight of AUGMENT_OPS, "bgc" those and
    GEOM_OPS, "bgcf" those and "imgfilter", "bgcfn" those and "noise", else a comma list of names from all of them."""
    if not spec:
        return ()
    if spec in _PRESETS:
        return _PRESETS[spec]
    names = {s.strip() for s in spec.split(",")}
    unknown = sorted(names - set(_ALL_OPS))
    if unknown:
        raise ValueError(f"unknown augmentation(s) {unknown}: use one of {tuple(_PRESETS)} or a comma list of {_ALL_OPS}")
    return tuple(n for n in _ALL_OPS if n in names)


def sample_augment_frac(ops_: tuple, p, B: int, H: int, W: int, device):
    """Per-image fractional inverse maps F^-1 [B, 6] for ops.augment (row-major 2x3, centred pixel coordinates), or None when no
    GEOM_OPS transform is enabled (then no random number is drawn).  Drawn on ``device`` without a host sync (capturable), the same
    random numbers whatever p is; a transform that does not apply contributes exactly the identity, so p = 0 gives the identity.

    F^-1 = S^-1 R_pre^-1 A^-1 R_post^-1 T^-1 (ADA's order): scale s = exp2(N(0, 0.2^2)), S^-1 = diag(1/s, 1/s); rotate: two
    rotations by U(-pi, pi), each applying with p_rot = 1 - sqrt(1 - p), so that at least one applies with probability p; aniso
    a = exp2(N(0, 0.2^2)), A^-1 = diag(1/a, a); xfrac t = N(0, 0.125^2) * (W, H) pixels, T^-1 a translation by -t."""
    if not any(n in ops_ for n in GEOM_OPS):
        return None
    eye = torch.eye(3, device=device).expand(B, 3, 3)
    G = eye

    def applies(q):
        return torch.rand(B, device=device) < q

    def then(T, a):                                  # G <- G T^-1 where the transform applies, else G I (exact)
        T = torch.where(a[:, None, None], T, eye)    # products and sums, not a matmul: TF32 matmuls would round the maps
        return (G[:, :, :, None] * T[:, None, :, :]).sum(dim=2)

    def diag(sx, sy):
        T = eye.clone()
        T[:, 0, 0], T[:, 1, 1] = sx, sy
        return T

    def rot():
        th = (torch.rand(B, device=device) * 2 - 1) * math.pi
        T = eye.clone()
        c, s = torch.cos(th), torch.sin(th)
        T[:, 0, 0], T[:, 0, 1], T[:, 1, 0], T[:, 1, 1] = c, -s, s, c
        return T
    p_rot = 1 - (1 - p) ** 0.5
    if "scale" in ops_:
        a = applies(p)
        s = torch.exp2(torch.randn(B, device=device) * 0.2)
        G = then(diag(1 / s, 1 / s), a)
    if "rotate" in ops_:
        a = applies(p_rot)
        G = then(rot(), a)
    if "aniso" in ops_:
        a = applies(p)
        s = torch.exp2(torch.randn(B, device=device) * 0.2)
        G = then(diag(1 / s, s), a)
    if "rotate" in ops_:
        a = applies(p_rot)
        G = then(rot(), a)
    if "xfrac" in ops_:
        a = applies(p)
        t = torch.randn(B, 2, device=device) * 0.125
        T = eye.clone()
        T[:, 0, 2], T[:, 1, 2] = -t[:, 0] * W, -t[:, 1] * H
        G = then(T, a)
    return G[:, :2, :].reshape(B, 6).contiguous()


def sample_augment(ops_: tuple, p, B: int, H: int, W: int, device):
    """Per-image augmentation parameters for ops.augment, drawn on ``device`` from torch's RNG without a host sync (capturable):
    (geom int32 [B, 4], color float32 [B, 12] or None when no colour transform is enabled).  ``p`` (a float or a 0-d device tensor)
    is the probability that each enabled transform applies to each image; a transform that does not apply contributes exactly the
    identity, so p = 0 gives identity parameters.  Every enabled transform draws the same random numbers whatever p is.

    Geometry (ADA's integer "pixel blitting"): xflip = a flip uniform in {none, flip}; rotate90 = k * 90 degrees, k uniform in 0..3
    (H == W only); xint = t = round(U(-0.125, 0.125) * (W, H)).  Colour, composed in this order on (r, g, b, 1): brightness + N(0, 0.2);
    contrast * lognormal(0, 0.5 ln 2); lumaflip I - 2 i v v^T, i uniform in {0, 1}, v = (1, 1, 1) / sqrt 3; hue = rotation about v
    by U(-pi, pi); saturation v v^T + s (I - v v^T), s lognormal(0, ln 2)."""
    if "rotate90" in ops_ and H != W:
        raise ValueError(f"the rotate90 augmentation needs square images, got {H}x{W}")

    def applies():
        return torch.rand(B, device=device) < p

    zero = torch.zeros(B, dtype=torch.int64, device=device)
    code, tx, ty = zero, zero, zero
    if "xflip" in ops_:
        code = code + torch.where(applies(), torch.randint(0, 2, (B,), device=device), zero)
    if "rotate90" in ops_:
        code = code + 2 * torch.where(applies(), torch.randint(0, 4, (B,), device=device), zero)
    if "xint" in ops_:
        a = applies()
        u = torch.rand(B, 2, device=device) * 2 - 1
        tx = torch.where(a, torch.round(u[:, 0] * (0.125 * W)).long(), zero)
        ty = torch.where(a, torch.round(u[:, 1] * (0.125 * H)).long(), zero)
    geom = torch.stack([code, tx, ty, zero], dim=1).to(torch.int32)
    if not any(n in ops_ for n in AUGMENT_OPS[3:]):
        return geom, None
    eye4 = torch.eye(4, device=device).expand(B, 4, 4)
    v = torch.full((3,), 1.0 / math.sqrt(3.0), device=device)
    vv = torch.outer(v, v)
    eye3 = torch.eye(3, device=device)
    M = eye4

    def then(T, a):                                  # M <- T M where transform T applies, else I M (exact)
        return torch.where(a[:, None, None], T, eye4) @ M

    def lin(T3):                                     # [B, 3, 3] -> [B, 4, 4] with no offset
        T = eye4.clone()
        T[:, :3, :3] = T3
        return T
    if "brightness" in ops_:
        a = applies()
        T = eye4.clone()
        T[:, :3, 3] = (torch.randn(B, device=device) * 0.2)[:, None]
        M = then(T, a)
    if "contrast" in ops_:
        a = applies()
        c = torch.exp2(torch.randn(B, device=device) * 0.5)
        M = then(lin(c[:, None, None] * eye3), a)
    if "lumaflip" in ops_:
        a = applies()
        i = torch.randint(0, 2, (B,), device=device).float()
        M = then(lin(eye3 - 2 * i[:, None, None] * vv), a)
    if "hue" in ops_:
        a = applies()
        th = (torch.rand(B, device=device) * 2 - 1) * math.pi
        P = eye3.roll(1, dims=0)
        K = (P - P.t()) / math.sqrt(3.0)              # the cross-product matrix [v]x of v = (1, 1, 1) / sqrt 3
        cs, sn = torch.cos(th)[:, None, None], torch.sin(th)[:, None, None]
        M = then(lin(cs * eye3 + sn * K + (1 - cs) * vv), a)
    if "saturation" in ops_:
        a = applies()
        s = torch.exp2(torch.randn(B, device=device))[:, None, None]
        M = then(lin(vv + s * (eye3 - vv)), a)
    return geom, M[:, :3, :].reshape(B, 12).contiguous()


def sample_augment_filter(ops_: tuple, p, B: int, C: int, H: int, W: int, device):
    """Per-image parameters for ops.augment_filter: (gains [B, 4] or None, sigma [B] or None, noise [B, C, H, W] or None), None where
    the transform is not enabled (then no random number is drawn for it).  Drawn on ``device`` without a host sync (capturable), in
    ADA's order and the same random numbers whatever p is.

    imgfilter: g = (1, 1, 1, 1); for each band i, t_i = exp2(N(0, 1)) (randn(B)), applying with probability p (rand(B)); where it
    applies, t = (1, .., t_i, .., 1) and g <- g * t / sqrt(sum_j ep_j t_j^2), ep = (10, 1, 1, 1) / 13; where it does not, g is left
    exactly unchanged, so p = 0 gives exactly (1, 1, 1, 1).  noise: sigma = |N(0, 1)| * 0.1 (randn(B)), applying with probability p
    (rand(B)), else 0; then the field n = randn(B, C, H, W)."""
    gains = sigma = noise = None
    if "imgfilter" in ops_:
        ep = torch.cat([torch.full((1,), IMGFILTER_EXPECTED_POWER[0] / 13, device=device),      # fills, no host copy: capturable
                        torch.full((3,), IMGFILTER_EXPECTED_POWER[1] / 13, device=device)])
        gains = torch.ones(B, 4, device=device)
        for i in range(4):
            t_i = torch.exp2(torch.randn(B, device=device))
            a = torch.rand(B, device=device) < p
            t = torch.ones(B, 4, device=device)
            t[:, i] = t_i
            t = t / (ep * t.square()).sum(dim=1, keepdim=True).sqrt()
            gains = torch.where(a[:, None], gains * t, gains)
    if "noise" in ops_:
        s = torch.randn(B, device=device).abs() * NOISE_STD
        a = torch.rand(B, device=device) < p
        sigma = torch.where(a, s, torch.zeros_like(s))
        noise = torch.randn(B, C, H, W, device=device)
    return gains, sigma, noise


def mixing_cutoff(p: float, num_ws: int, device) -> torch.Tensor:
    """The style-mixing cutoff of one minibatch as a 0-d int64 tensor on ``device``, drawn without a host sync: with probability
    ``p`` uniform in [1, num_ws - 1], else num_ws (no mixing).  ``p == 0`` draws no random number and returns num_ws."""
    no_mix = torch.full((), num_ws, dtype=torch.int64, device=device)
    if p <= 0.0:
        return no_mix
    return torch.where(torch.rand((), device=device) < p, torch.randint(1, num_ws, (), device=device), no_mix)


def mix_latents(ws1: torch.Tensor, ws2: torch.Tensor, cutoff: torch.Tensor, num_ws: int) -> torch.Tensor:
    """Per-layer latents [B, num_ws, k+1, D] from two mapping outputs [B, k+1, D]: index i takes ws1 where i < cutoff, else ws2."""
    first = torch.arange(num_ws, device=ws1.device) < cutoff
    return torch.where(first[None, :, None, None], ws1[:, None], ws2[:, None])


@dataclass
class StepStats:
    loss_g: float = 0.0
    loss_d: float = 0.0
    r1: float = 0.0
    allreduce_bytes: float = 0.0
    allreduce_ms: float = 0.0
    extra: Dict[str, float] = field(default_factory=dict)
    pl_penalty: float = 0.0             # mean squared deviation of the path lengths from their running mean (a path-length step)
    pl_mean: float = 0.0                # the running mean of the path lengths (this rank's)
    augment_p: float = 0.0              # the augmentation strength p after the step (the same on every rank)


class Trainer:
    """One process per GPU.  ``step(z, reals)`` = one discriminator update + one generator update on this rank's shard."""

    def __init__(self, G: nn.Module, D: nn.Module, cfg: Optional[TrainConfig] = None, world: int = 1):
        self.G, self.D, self.cfg, self.world = G, D, cfg or TrainConfig(), world
        self.c_dim = getattr(G, "c_dim", 0)
        if getattr(D, "c_dim", 0) != self.c_dim:
            raise ValueError(f"G and D must have the same c_dim, got {self.c_dim} and {getattr(D, 'c_dim', 0)}")
        if not 0.0 <= self.cfg.style_mixing <= 1.0:
            raise ValueError(f"style_mixing must be in [0, 1], got {self.cfg.style_mixing}")
        if self.cfg.style_mixing > 0 and not (hasattr(G, "mapping") and hasattr(G, "synthesis")):
            raise ValueError("style_mixing needs a generator with `mapping` and `synthesis`")
        self.augment_ops = parse_augment(self.cfg.augment)
        self._check_augment()
        self.G_ema = copy.deepcopy(G).eval().requires_grad_(False)
        c = self.cfg.d_reg_interval / (self.cfg.d_reg_interval + 1.0)  # lazy regularisation: rescale lr and betas
        cap = next(G.parameters()).is_cuda                              # capturable: the step can be replayed from a CUDA graph
        cg = self.cfg.g_reg_interval / (self.cfg.g_reg_interval + 1.0) if self.cfg.pl_weight > 0 else 1.0
        self.opt_g = torch.optim.Adam(G.parameters(), lr=self.cfg.lr * cg, betas=(0.0 ** cg, 0.99 ** cg), eps=1e-8, capturable=cap)
        # running mean of the path lengths: a device tensor updated in place (capturable), per rank as upstream
        self.pl_mean = torch.zeros((), device=next(G.parameters()).device) if self.cfg.pl_weight > 0 else None
        self.opt_d = torch.optim.Adam(D.parameters(), lr=self.cfg.lr * c, betas=(0.0 ** c, 0.99 ** c), eps=1e-8, capturable=cap)
        self.it = 0
        # data parallel: gradients live in one flat buffer per network, reduced bucket by bucket while backward still runs
        self.buckets_g = gdist.GradBuckets(G.parameters(), world, self.cfg.bucket_mb) if world > 1 else None
        self.buckets_d = gdist.GradBuckets(D.parameters(), world, self.cfg.bucket_mb) if world > 1 else None
        # augmentation (SURVEY A.4 item 15): the strength p and, with ada_target, the accumulators of the adaptive update -- device
        # tensors updated in place (capturable); callers may save and restore them
        dev = next(G.parameters()).device
        self.augment_p = torch.full((), float(self.cfg.augment_p), device=dev) if self.augment_ops else None
        self.ada_stats = torch.zeros(2, device=dev) if self.cfg.ada_target is not None else None     # (sum of signs, count)
        self.ada_steps = torch.zeros((), dtype=torch.int64, device=dev) if self.cfg.ada_target is not None else None

    def _check_augment(self):
        cfg = self.cfg
        if not 0.0 <= cfg.augment_p <= 1.0:
            raise ValueError(f"augment_p must be in [0, 1], got {cfg.augment_p}")
        if cfg.ada_target is not None:
            if not self.augment_ops:
                raise ValueError("ada_target adapts the augmentation strength: it needs augment to be set")
            if not -1.0 <= cfg.ada_target <= 1.0:
                raise ValueError(f"ada_target is a mean sign and must be in [-1, 1], got {cfg.ada_target}")
            if cfg.ada_interval < 1 or not cfg.ada_kimg > 0:
                raise ValueError(f"need ada_interval >= 1 and ada_kimg > 0, got {cfg.ada_interval} and {cfg.ada_kimg}")
        res = getattr(self.D, "resolution", None)
        if "imgfilter" in self.augment_ops and res is not None and res <= IMGFILTER_HALO:
            raise ValueError(f"the imgfilter augmentation needs images of at least 22x22 (its 43-tap filter reflects a 21-pixel "
                             f"border once), got a {res}x{res} discriminator")

    def _augment(self, img: torch.Tensor) -> torch.Tensor:
        """One image batch on its way into D, augmented with parameters of its own (no call and no random number when off)."""
        if not self.augment_ops:
            return img
        B, C, H, W = img.shape
        if any(n in self.augment_ops for n in _ADA_ORDER):
            geom, color = sample_augment(self.augment_ops, self.augment_p, B, H, W, img.device)
            frac = sample_augment_frac(self.augment_ops, self.augment_p, B, H, W, img.device)
            img = augment(img, geom, color) if frac is None else augment(img, geom, color, frac)
        if any(n in self.augment_ops for n in FILTER_OPS):
            gains, sigma, noise = sample_augment_filter(self.augment_ops, self.augment_p, B, C, H, W, img.device)
            img = augment_filter(img, gains, sigma, noise)
        return img

    def _ada_accumulate(self, logit_real: torch.Tensor):
        """Adds (sum of the signs, count) of this step's real logits, summed over ranks, to the ADA accumulators."""
        l = logit_real.detach()
        inc = torch.stack([l.sign().sum(), torch.ones_like(l).sum()]).float()
        if self.world > 1:
            gdist.allreduce_sum(inc)
        self.ada_stats.add_(inc)

    def _ada_update(self, batch: int):
        """Every ada_interval-th step: p <- clamp(p + sign(mean sign - target) * B_global * interval / (kimg * 1000), 0, 1), then the
        accumulators reset.  Decided on the device from a step counter, so a replayed graph does the same."""
        cfg = self.cfg
        step = batch * self.world * cfg.ada_interval / (cfg.ada_kimg * 1000.0)
        with torch.no_grad():
            boundary = torch.remainder(self.ada_steps + 1, cfg.ada_interval) == 0
            mean = self.ada_stats[0] / self.ada_stats[1].clamp(min=1.0)
            p_new = (self.augment_p + torch.sign(mean - cfg.ada_target) * step).clamp(0.0, 1.0)
            self.augment_p.copy_(torch.where(boundary, p_new, self.augment_p))
            self.ada_stats.copy_(torch.where(boundary, torch.zeros_like(self.ada_stats), self.ada_stats))
            self.ada_steps.add_(1)

    def _zero(self, opt, buckets):
        if buckets is not None:
            buckets.begin()                # one memset of the flat buffer; the .grad views stay attached
        else:
            opt.zero_grad(set_to_none=True)

    def _allreduce(self, buckets, stats: StepStats):
        if buckets is not None:
            stats.allreduce_bytes += buckets.finish()      # joins the communication stream (the buckets overlapped backward)

    def _labels(self, z: torch.Tensor, reals: torch.Tensor, gen_c, real_c):
        """(gen_c, real_c) checked against the batch and moved to z's device and dtype: both required iff c_dim > 0; (None, None) for
        an unconditional pair."""
        if self.c_dim == 0:
            return None, None
        for name, c, n in (("gen_c", gen_c, z.shape[0]), ("real_c", real_c, reals.shape[0])):
            if c is None:
                raise ValueError(f"conditional training (c_dim={self.c_dim}) needs {name} [{n}, {self.c_dim}]")
            if c.dim() != 2 or c.shape[0] != n or c.shape[1] != self.c_dim:
                raise ValueError(f"{name} must be [{n}, {self.c_dim}], got {tuple(c.shape)}")
        return gen_c.to(device=z.device, dtype=z.dtype), real_c.to(device=z.device, dtype=z.dtype)

    def _step_tensors(self, z: torch.Tensor, reals: torch.Tensor, do_r1: bool, stats: Optional[StepStats] = None,
                      do_pl: bool = False, gen_c: Optional[torch.Tensor] = None, real_c: Optional[torch.Tensor] = None):
        """One D update + one G update (+ the path-length update with ``do_pl``); returns (loss_d, loss_g, r1, pl_penalty, cutoffs) as
        device tensors without synchronising (capturable); pl_penalty is None without ``do_pl``; cutoffs maps the StepStats.extra
        names of the style-mixing cutoffs of the D and G phases to them (empty without style mixing).  gen_c / real_c: the labels
        of the fakes and of the reals (None for an unconditional pair: the calls then pass no labels)."""
        G, D, cfg = self.G, self.D, self.cfg
        gc = () if gen_c is None else (gen_c,)                          # label arguments of the calls on fakes / reals
        rc = () if real_c is None else (real_c,)
        stats = stats if stats is not None else StepStats()
        cutoffs: Dict[str, torch.Tensor] = {}
        # ---- discriminator: logistic loss (+ lazy R1 on the reals)
        G.requires_grad_(False); D.requires_grad_(True)
        self._zero(self.opt_d, self.buckets_d)
        with torch.no_grad():
            fakes = self._generate(z, cutoffs, "d", gc)
        reals_in = reals.detach().requires_grad_(do_r1)
        logit_real, logit_fake = D(self._augment(reals_in), *rc), D(self._augment(fakes), *gc)
        loss_d = F.softplus(logit_fake).mean() + F.softplus(-logit_real).mean()
        if self.ada_stats is not None:
            self._ada_accumulate(logit_real)
        r1 = torch.zeros((), device=z.device)
        if do_r1:
            (grad,) = torch.autograd.grad(logit_real.sum(), reals_in, create_graph=True)
            r1 = grad.square().sum(dim=[1, 2, 3]).mean()
            loss_d = loss_d + r1 * (cfg.r1_gamma * 0.5 * cfg.d_reg_interval)
        loss_d.backward()
        self._allreduce(self.buckets_d, stats)
        self.opt_d.step()
        # ---- generator: non-saturating logistic loss
        if z.is_cuda:
            from .attention import advance_dropout
            advance_dropout(z.device)                 # attention dropout: fresh masks for the G phase (device-side, capturable)
        G.requires_grad_(True); D.requires_grad_(False)
        self._zero(self.opt_g, self.buckets_g)
        loss_g = F.softplus(-D(self._augment(self._generate(z, cutoffs, "g", gc)), *gc)).mean()
        loss_g.backward()
        self._allreduce(self.buckets_g, stats)
        self.opt_g.step()
        if z.is_cuda:
            advance_dropout(z.device)                 # ... and for the next step
        pl_penalty = self._pl_phase(z, stats, gc) if do_pl else None
        # ---- moving average of the generator (and of the mapping outputs: the truncation trick's w_avg)
        with torch.no_grad():
            if hasattr(G, "mapping") and hasattr(G.mapping, "w_avg"):
                ws = G.mapping(z, *gc)
                k_ = G.mapping.components_num
                cur = torch.stack([ws[:, :k_].mean(dim=(0, 1)), ws[:, k_:].mean(dim=(0, 1))])
                G.mapping.w_avg.lerp_(cur, 1.0 - cfg.w_avg_beta)
            beta = 0.5 ** (z.shape[0] * self.world / (cfg.ema_kimg * 1000.0))
            for pe, p in zip(self.G_ema.parameters(), G.parameters()):
                pe.lerp_(p.detach(), 1.0 - beta)
            for be, b in zip(self.G_ema.buffers(), G.buffers()):
                be.copy_(b)
        if self.ada_stats is not None:
            self._ada_update(z.shape[0])
        return loss_d.detach(), loss_g.detach(), r1.detach(), pl_penalty, cutoffs

    def _generate(self, z: torch.Tensor, cutoffs: Dict[str, torch.Tensor], phase: str, gc=()) -> torch.Tensor:
        """The fakes of one phase: G(z), or with style mixing (SURVEY A.4 item 13) the synthesis of per-layer latents that switch
        from G.mapping(z) to the mapping of a second draw at a cutoff of their own.  gc: () or (the labels,), which both draws take.
        Device-side throughout (capturable)."""
        G, cfg = self.G, self.cfg
        if cfg.style_mixing <= 0.0:
            return G(z, *gc, noise_mode=cfg.noise_mode)
        num_ws = G.synthesis.num_ws
        z2 = torch.randn_like(z)
        ws1, ws2 = G.mapping(z, *gc), G.mapping(z2, *gc)
        cutoff = mixing_cutoff(cfg.style_mixing, num_ws, z.device)
        cutoffs["style_mixing_cutoff_" + phase] = cutoff
        return G.synthesis(mix_latents(ws1, ws2, cutoff, num_ws), noise_mode=cfg.noise_mode)

    def _pl_phase(self, z: torch.Tensor, stats: StepStats, gc=()) -> torch.Tensor:
        """The lazy path-length update of G (StyleGAN2): returns the penalty as a device tensor (capturable: no host sync, the
        noise is drawn on the device).  gc: () or (the labels of z,), cut to the same first B' rows."""
        G, cfg = self.G, self.cfg
        if z.is_cuda:
            from .attention import advance_dropout
            advance_dropout(z.device)                 # fresh attention-dropout masks; the backward regenerates the same ones
        self._zero(self.opt_g, self.buckets_g)
        nb = max(1, z.shape[0] // cfg.pl_batch_shrink)
        ws = G.mapping(z[:nb], *[c[:nb] for c in gc])
        img = G.synthesis(ws, noise_mode=cfg.noise_mode)
        pl_noise = torch.randn_like(img) / math.sqrt(img.shape[2] * img.shape[3])
        (pl_grads,) = torch.autograd.grad((img * pl_noise).sum(), ws, create_graph=True)
        pl_lengths = pl_grads.square().sum(dim=2).mean(dim=1).sqrt()          # [B']: over D, then over the k+1 latent components
        with torch.no_grad():
            self.pl_mean.lerp_(pl_lengths.mean(), cfg.pl_decay)
        pl_penalty = (pl_lengths - self.pl_mean).square().mean()
        (pl_penalty * (cfg.pl_weight * cfg.g_reg_interval)).backward()
        self._allreduce(self.buckets_g, stats)
        self.opt_g.step()
        if z.is_cuda:
            advance_dropout(z.device)
        return pl_penalty.detach()

    def _do_pl(self) -> bool:
        return self.cfg.pl_weight > 0 and self.it % self.cfg.g_reg_interval == 0

    def _finish_stats(self, stats: StepStats, loss_d, loss_g, r1, pl_penalty, cutoffs) -> StepStats:
        stats.loss_d, stats.loss_g, stats.r1 = float(loss_d), float(loss_g), float(r1)
        for name, cutoff in cutoffs.items():
            stats.extra[name] = float(cutoff)
        if pl_penalty is not None:
            stats.pl_penalty = float(pl_penalty)
        if self.pl_mean is not None:
            stats.pl_mean = float(self.pl_mean)
        if self.augment_p is not None:
            stats.augment_p = float(self.augment_p)
        return stats

    def _snapshot(self, device) -> tuple:
        """Clones of everything ``_step_tensors`` writes: the parameters and buffers of G, D and G_ema, both Adams' states, pl_mean,
        the ADA tensors, the attention-dropout state and the RNG state of ``device``.  For ``_restore``."""
        live = [t for m in (self.G, self.D, self.G_ema) for t in (*m.parameters(), *m.buffers())]
        live += [t for t in (self.pl_mean, self.augment_p, self.ada_stats, self.ada_steps) if t is not None]
        cuda = torch.device(device).type == "cuda"
        if cuda:
            from .attention import dropout_state
            live.append(dropout_state(device))
        adam = [{p: {k: v.clone() for k, v in s.items()} for p, s in opt.state.items()} for opt in (self.opt_g, self.opt_d)]
        rng = torch.cuda.get_rng_state(device) if cuda else torch.get_rng_state()
        return [(t, t.detach().clone()) for t in live], adam, rng

    def _restore(self, snap: tuple, device) -> None:
        """Copies a ``_snapshot`` back in place (captured graphs keep pointers: no tensor is replaced).  An Adam state created since
        the snapshot is zeroed, which is how a fresh Adam starts, and kept, so that a capture finds it instead of creating it."""
        live, adam, rng = snap
        with torch.no_grad():
            for t, saved in live:
                t.copy_(saved)
            for opt, states in zip((self.opt_g, self.opt_d), adam):
                for p, s in opt.state.items():
                    for k, v in s.items():
                        if p in states:
                            v.copy_(states[p][k])
                        else:
                            v.zero_()
        if torch.device(device).type == "cuda":
            torch.cuda.set_rng_state(rng, device)
        else:
            torch.set_rng_state(rng)

    def step(self, z: torch.Tensor, reals: torch.Tensor, gen_c: Optional[torch.Tensor] = None,
             real_c: Optional[torch.Tensor] = None) -> StepStats:
        """gen_c [B, c_dim]: the labels of the fakes (one per z); real_c: those of the reals.  Required iff c_dim > 0."""
        gen_c, real_c = self._labels(z, reals, gen_c, real_c)
        stats = StepStats()
        do_r1 = self.cfg.r1_gamma > 0 and self.it % self.cfg.d_reg_interval == 0
        outs = self._step_tensors(z, reals, do_r1, stats, self._do_pl(), gen_c, real_c)
        self._finish_stats(stats, *outs)
        bump_weights_epoch()
        self.it += 1
        return stats

    def step_graphed(self, z: torch.Tensor, reals: torch.Tensor, gen_c: Optional[torch.Tensor] = None,
                     real_c: Optional[torch.Tensor] = None) -> StepStats:
        """The same step replayed from a CUDA graph (one graph per combination of the lazy R1 term and the lazy path-length
        phase that occurs, at most three with the default intervals): the eager step is bound by the host launching ~5000 small
        kernels.  Shapes are fixed by the first call.  Before it captures, the first call runs the step eagerly once per graph
        (cuDNN autotuning, workspaces), then puts back everything those runs wrote (``_snapshot``, ``_restore``), so that it takes
        one step like every later call.  The labels, like z and reals, go through static buffers."""
        from . import attention as _att, networks as _nets
        cfg = self.cfg
        gen_c, real_c = self._labels(z, reals, gen_c, real_c)
        do_r1 = cfg.r1_gamma > 0 and self.it % cfg.d_reg_interval == 0
        st = self.__dict__.setdefault("_graphs", {})
        _nets.CACHE_BYPASS = _att.FORCE_REFOLD = True                  # weight-derived tensors are recomputed inside the graph
        try:
            return self._step_graphed(z, reals, (do_r1, self._do_pl()), st, gen_c, real_c)
        finally:
            _nets.CACHE_BYPASS = _att.FORCE_REFOLD = False

    def _step_graphed(self, z, reals, key, st, gen_c=None, real_c=None) -> StepStats:
        cfg = self.cfg
        if "z" not in st:
            st["z"], st["reals"] = torch.empty_like(z), torch.empty_like(reals)
            st["z"].copy_(z); st["reals"].copy_(reals)
            st["gen_c"] = st["real_c"] = None
            if gen_c is not None:
                st["gen_c"], st["real_c"] = gen_c.clone(), real_c.clone()
            lab = dict(gen_c=st["gen_c"], real_c=st["real_c"])
            snap = self._snapshot(z.device)
            side = torch.cuda.Stream(device=z.device)                 # warm-up off the capture stream: cuDNN autotune, workspaces
            side.wait_stream(torch.cuda.current_stream(z.device))
            with torch.cuda.stream(side):
                for r in ([True, False] if cfg.r1_gamma > 0 else [False]):
                    self._step_tensors(st["z"], st["reals"], r, **lab)
                if cfg.pl_weight > 0:
                    self._step_tensors(st["z"], st["reals"], False, do_pl=True, **lab)
            torch.cuda.current_stream(z.device).wait_stream(side)
            self._restore(snap, z.device)                             # the warm-up steps leave no trace: the first call is one step
            del snap
            torch.cuda.synchronize(z.device)
        st["z"].copy_(z); st["reals"].copy_(reals)
        if gen_c is not None:
            st["gen_c"].copy_(gen_c); st["real_c"].copy_(real_c)
        if key not in st:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outs = self._step_tensors(st["z"], st["reals"], key[0], do_pl=key[1], gen_c=st["gen_c"], real_c=st["real_c"])
            st[key] = (graph, outs)
            # (capture does not execute: fall through to the replay below)
        graph, outs = st[key]
        graph.replay()
        bump_weights_epoch()          # the replay moved G / D / G_ema weights without touching their version counters
        self.it += 1
        return self._finish_stats(StepStats(), *outs)
