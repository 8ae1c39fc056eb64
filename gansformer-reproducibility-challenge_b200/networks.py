"""GANsformer generator host code around the bipartite-attention hot path.

Mirrors the reference's model API (expected ``src/training/network.py`` upstream -- ``G_GANsformer`` /
``G_mapping`` / ``G_synthesis`` -- not present in the reference checkout, see SURVEY.md section 0; kwarg names
follow SURVEY.md section 8b): ``Generator(z[B,k+1,D], c=None, truncation_psi=1.0, noise_mode=..., return_att=False)
-> img[B,3,R,R]`` with ``.mapping`` / ``.synthesis`` sub-modules, plus a ``Gs.run``-style ``run(...)`` wrapper.

Everything here except the attention block is plain PyTorch plumbing (cuDNN convolutions, channels-last
memory format); the attention block -- the hot path -- is the C-ABI call in ``attention.py``.  Architecture
choices the reference source cannot arbitrate are frozen in SURVEY.md A.4 ([SPEC] items 1-9).
"""
from __future__ import annotations

import math
import os
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .attention import BipartiteAttention, _Plan, prologue_batch, tc_eligible
from . import ops
from .self_attention import ImageSelfAttention
from ._state import weights_epoch, bump_weights_epoch
from .ops import fir_filter

SQRT2 = math.sqrt(2.0)


def _inference(*params) -> bool:
    """True when no autograd graph is needed: derived tensors (scaled weights, ...) may then be cached."""
    return not (torch.is_grad_enabled() and any(p.requires_grad for p in params))


# Output resolutions whose upsampling layer runs on the fused kernel (gf_upconv3x3_blur_nhwc_tf32): those where tools/upconv_probe.py
# measured it at least 20 % faster than the cuDNN polyphase path, judged against cuDNN's fastest run (DESIGN §6, batch 32, H100
# 80GB HBM3 at 400 W: 0.058 vs 0.099-0.134 ms at 8^2, 2.14 vs 4.69 ms at 256^2); 512^2 is not timed and takes the kernel, whose lead
# grows with the layer.  16^2 .. 128^2 keep cuDNN (0.126 vs 0.111-0.188 ms at 16^2, 1.86 vs 1.70 ms at 128^2).
def upconv_fused(res: int) -> bool:
    return res == 8 or res >= 256

CACHE_BYPASS = False      # set by training.Trainer while it captures a CUDA graph: weight-derived tensors must be recomputed
                          # inside the graph on every replay (a replay runs no Python, so a version-keyed cache would go stale)


def _cached(module: nn.Module, key: str, params, fn):
    """Cache `fn()` on `module` until one of `params` changes (version counter / storage / device)."""
    if CACHE_BYPASS:
        with torch.no_grad():
            return fn()
    ver = (weights_epoch(),) + tuple((p.data_ptr(), p._version, str(p.device), p.dtype) for p in params)
    store = module.__dict__.setdefault("_icache", {})
    ent = store.get(key)
    if ent is None or ent[0] != ver:
        with torch.no_grad():
            ent = (ver, fn())
        store[key] = ent
    return ent[1]


RUNTIME_KEYS = ("_icache", "_graphs", "_side_stream", "_copy_stream")


def drop_runtime_state(module: nn.Module) -> nn.Module:
    """Remove everything derived from the weights or bound to a device context (caches, captured graphs, streams, staging
    buffers, attention plans) from `module` and its children -- after a deep copy, a device move or a weight load."""
    for m in module.modules():
        for key in [k for k in m.__dict__ if k in RUNTIME_KEYS or (isinstance(k, tuple) and k and k[0] == "_staging")]:
            del m.__dict__[key]
        if isinstance(m, BipartiteAttention):
            m._plan = _Plan()
    return module


def nf(res: int, fmap_base: int = 16384, fmap_max: int = 512) -> int:
    """StyleGAN2 config-f channel schedule (SURVEY A.4 item 7)."""
    return int(min(fmap_base // (2 ** (int(math.log2(res)) - 1)), fmap_max))


def modulated_conv2d(x: torch.Tensor, weight: torch.Tensor, styles: torch.Tensor, *, demodulate: bool = True,
                     up: int = 1, f: Optional[torch.Tensor] = None, w_eff: Optional[torch.Tensor] = None,
                     wsq: Optional[torch.Tensor] = None, prescaled: bool = False, defer_demod: bool = False,
                     d: Optional[torch.Tensor] = None, phases=None, wt_packed: Optional[torch.Tensor] = None):
    """StyleGAN2 modulated convolution in its activation-scaling form: (x * s) conv w, then * demod.

    Identical in exact arithmetic to modulating the weights per sample (the reference's grouped-conv form);
    avoids B separate weight tensors.  weight [O, I, kh, kw]; styles [B, I].  The two scalings and the FIR blur of the
    upsampling path are the native ops of ops.py (gf_ops.h).  The stride-1 3x3 convolution runs on the library's own wgmma
    implicit-GEMM kernel (wt_packed, row f1) when TF32 convolutions are allowed and the shape is eligible, else on cuDNN; with
    wt_packed the upsampling convolution, its blur and the demodulation are one kernel of the library, otherwise the polyphase
    up-convolutions are cuDNN (the fp32 path).
    w_eff / wsq: optional cached equalised-LR weight (already transposed for up=2) and its squared sum over the taps.
    prescaled: x already carries the style scale (fused into the producer's store).  defer_demod (up == 1 only): return
    (conv output, d) and let the consumer (the attention kernel's load side) apply the demodulation."""
    O, I, kh, kw = weight.shape
    if w_eff is None:
        w_eff = weight * (1.0 / math.sqrt(I * kh * kw))
        if up != 1:
            w_eff = w_eff.transpose(0, 1)
    if demodulate and d is None:
        if wsq is None:
            wsq = (weight * (1.0 / math.sqrt(I * kh * kw))).square().sum(dim=[2, 3])    # [O, I]
        d = ops.demod_coef(styles, wsq)                                                  # [B, O]
    if not prescaled:
        x = ops.chan_scale(x, styles)
    if up == 1:
        if wt_packed is not None:
            x = ops.conv3x3_native(x, wt_packed)                      # row f1: own wgmma implicit-GEMM kernel (TF32)
        else:
            x = F.conv2d(x, w_eff, padding=kh // 2)
        if defer_demod:
            return x, d
        if d is not None:
            x = ops.chan_scale(x, d)
    elif wt_packed is not None and d is not None and ops._use_cuda(x, d):
        x = ops.upconv_blur_native(x, wt_packed, scale=d, gain=4.0)    # row f1: convolution + blur + demodulation in one kernel (TF32)
    elif phases is not None and ops._use_cuda(x, d) and O % 4 == 0 and not os.environ.get("GF_NO_PHASES"):
        x = ops.upconv_blur_phases(x, phases, scale=d, gain=4.0)       # four polyphase stride-1 convolutions + blur
    else:
        x = F.conv_transpose2d(x, w_eff, stride=2)                    # [B, O, 2H+1, 2W+1]
        x = ops.blur_up(x, f, scale=d, gain=4.0)                       # -> [B, O, 2H, 2W], demodulated
    return x


class FullyConnected(nn.Module):
    def __init__(self, in_features: int, out_features: int, bias_init: float = 0.0, lr_mul: float = 1.0, act: str = "linear"):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_features, in_features) / lr_mul)
        self.bias = nn.Parameter(torch.full((out_features,), float(bias_init)))
        self.wgain = lr_mul / math.sqrt(in_features)
        self.bgain = lr_mul
        self.act = act

    def effective(self):
        """(W^T [in,out], b [out]) with the equalised-LR gains folded in (and sqrt(2) for lrelu: lrelu(z)*g == lrelu(g*z))."""
        g = SQRT2 if self.act == "lrelu" else 1.0
        return (self.weight * (self.wgain * g)).t().contiguous(), self.bias * (self.bgain * g)

    def forward(self, x):
        if _inference(self.weight, self.bias):
            wt, b = _cached(self, "eff", (self.weight, self.bias), self.effective)
            y = torch.addmm(b, x.reshape(-1, x.shape[-1]), wt).reshape(*x.shape[:-1], wt.shape[1])
            return F.leaky_relu(y, 0.2) if self.act == "lrelu" else y
        x = F.linear(x, self.weight * self.wgain, self.bias * self.bgain)
        return F.leaky_relu(x, 0.2) * SQRT2 if self.act == "lrelu" else x


class MappingNetwork(nn.Module):
    """G_mapping: z [B, k+1, D] -> w [B, k+1, D]; the k local components share one MLP, the global latent has its own.

    ``ltnt2ltnt=True`` (upstream's latent-to-latent option, SURVEY 2.2 / row f4): after every fully connected layer the k local
    latents attend to each other -- the same bipartite block as in the synthesis network (``BipartiteAttention`` with the
    latents as both the "grid" [B, k, 1, D] and the attended set, no positional encoding, integration / norm as given), so it runs
    on the same C-ABI kernels (C = D = 32: the CUDA-core kernel).  Off by default, as in the benchmarked configurations.

    ``c_dim > 0`` makes the mapping class-conditional (SURVEY A.4 item 14, StyleGAN2's label concatenation): a label embedding
    ``embed`` [c_dim, D] (N(0, 1), no equalised-LR gain), e_b = c_b embed concatenated to every latent of image b before the pixel
    norm, and layer 0 of both MLPs with fan-in 2D.  Truncation keeps the one label-agnostic w_avg.  ``c_dim = 0`` (the default)
    builds exactly the unconditional network and ignores ``c``."""

    def __init__(self, latent_dim: int, components_num: int, num_layers: int = 8, lr_mul: float = 0.01, ltnt2ltnt: bool = False,
                 integration: str = "mul", norm: Optional[str] = "layer", exact_fp32: bool = False, c_dim: int = 0):
        super().__init__()
        if c_dim < 0:
            raise ValueError(f"c_dim must be >= 0, got {c_dim}")
        self.latent_dim, self.components_num, self.c_dim = latent_dim, components_num, int(c_dim)
        fan0 = 2 * latent_dim if c_dim > 0 else latent_dim           # layer 0 reads [z || e] when conditional
        self.local = nn.ModuleList([FullyConnected(fan0 if i == 0 else latent_dim, latent_dim, lr_mul=lr_mul, act="lrelu")
                                    for i in range(num_layers)])
        self.glob = nn.ModuleList([FullyConnected(fan0 if i == 0 else latent_dim, latent_dim, lr_mul=lr_mul, act="lrelu")
                                   for i in range(num_layers)])
        self.register_buffer("w_avg", torch.zeros(2, latent_dim))
        self.self_att = None
        if ltnt2ltnt and components_num > 1:
            self.self_att = nn.ModuleList([BipartiteAttention(latent_dim, latent_dim, components_num, pos_dim=latent_dim, use_pos=False,
                                                              integration=integration, norm=norm, exact_fp32=exact_fp32)
                                           for _ in range(num_layers)])
        if c_dim > 0:
            self.embed = nn.Parameter(torch.randn(c_dim, latent_dim))

    def labels(self, c: Optional[torch.Tensor], batch: int, like: torch.Tensor) -> Optional[torch.Tensor]:
        """The labels of a call as a [batch, c_dim] tensor of `like`'s dtype, or None for an unconditional network (which ignores c).
        Raises ValueError when the network is conditional and c is missing or has the wrong shape."""
        if self.c_dim == 0:
            return None
        if c is None:
            raise ValueError(f"this network is conditional (c_dim={self.c_dim}): labels c [B, {self.c_dim}] are required")
        c = torch.as_tensor(c)
        if c.dim() != 2 or c.shape[0] != batch or c.shape[1] != self.c_dim:
            raise ValueError(f"c must be [{batch}, {self.c_dim}], got {tuple(c.shape)}")
        return c.to(device=like.device, dtype=like.dtype)

    def forward(self, z: torch.Tensor, c: Optional[torch.Tensor] = None, truncation_psi: float = 1.0) -> torch.Tensor:
        k = self.components_num
        if z.dim() != 3 or z.shape[1] != k + 1 or z.shape[2] != self.latent_dim:
            raise ValueError(f"z must be [B, {k + 1}, {self.latent_dim}], got {tuple(z.shape)}")
        c = self.labels(c, z.shape[0], z)
        params = [t for fc in list(self.local) + list(self.glob) for t in (fc.weight, fc.bias)]
        if c is not None and (self.self_att is None and z.is_cuda and z.dtype == torch.float32 and _inference(*params, self.embed)
                              and self.latent_dim <= 128 and len(self.local) * self.latent_dim ** 2 * 8 <= 200 * 1024
                              and not os.environ.get("GF_NO_MAPPING_KERNEL")):
            # inference: the conditional mapping network is ONE kernel too (gf_mapping_fwd_cond): layer 0 [2, 2D, D], the rest
            # [2, L-1, D, D]; cached until a parameter (the embedding included) changes
            def stack_cond():
                wl, bl = zip(*[fc.effective() for fc in self.local])
                wg, bg = zip(*[fc.effective() for fc in self.glob])
                w0 = torch.stack([wl[0], wg[0]]).contiguous()
                rest = torch.stack([torch.stack(wl[1:]), torch.stack(wg[1:])]).contiguous() if len(wl) > 1 else None
                return w0, rest, torch.stack([torch.stack(bl), torch.stack(bg)]).contiguous()
            w0, w_rest, b_eff = _cached(self, "stack_cond", params + [self.embed], stack_cond)
            return ops.mapping_fwd(z, w_rest, b_eff, self.w_avg, float(truncation_psi), k, c=c, embed=self.embed, w0=w0)
        if (c is None and self.self_att is None and z.is_cuda and z.dtype == torch.float32 and _inference(*params) and self.latent_dim <= 128
                and len(self.local) * self.latent_dim ** 2 * 8 <= 200 * 1024 and not os.environ.get("GF_NO_MAPPING_KERNEL")):
            # inference: the whole mapping network is ONE kernel (gf_mapping_fwd); effective weights cached until a parameter changes
            def stack():
                wl, bl = zip(*[fc.effective() for fc in self.local])
                wg, bg = zip(*[fc.effective() for fc in self.glob])
                return (torch.stack([torch.stack(wl), torch.stack(wg)]).contiguous(), torch.stack([torch.stack(bl), torch.stack(bg)]).contiguous())
            w_eff, b_eff = _cached(self, "stack", params, stack)
            return ops.mapping_fwd(z, w_eff, b_eff, self.w_avg, float(truncation_psi), k)
        if c is not None:                           # [z || c embed], normalised over its 2D entries
            e = c @ self.embed
            z = torch.cat([z, e[:, None].expand(-1, k + 1, -1)], dim=2)
        z = z * torch.rsqrt(z.square().mean(dim=2, keepdim=True) + 1e-8)
        loc, glo = z[:, :k], z[:, k:]
        for i, fc in enumerate(self.local):
            loc = fc(loc)
            if self.self_att is not None:           # latents attend to latents: grid = [B, k, 1, D] (H = k, W = 1), attended set = the same latents
                loc = loc.contiguous()
                loc, _, _ = self.self_att[i](loc.reshape(loc.shape[0], k, 1, self.latent_dim), loc)
                loc = loc.reshape(-1, k, self.latent_dim)
        for fc in self.glob:
            glo = fc(glo)
        if truncation_psi != 1.0:
            loc = self.w_avg[0].lerp(loc, truncation_psi)
            glo = self.w_avg[1].lerp(glo, truncation_psi)
        return torch.cat([loc, glo], dim=1)


class SynthesisLayer(nn.Module):
    """mod-conv -> bipartite attention (the hot path) -> noise -> bias + lrelu (SURVEY A.4 item 8)."""

    def __init__(self, in_ch: int, out_ch: int, w_dim: int, resolution: int, up: bool, components_num: int,
                 use_attention: bool, attn_kwargs: dict):
        super().__init__()
        self.resolution, self.up = resolution, up
        self.affine = FullyConnected(w_dim, in_ch, bias_init=1.0)
        self.weight = nn.Parameter(torch.randn(out_ch, in_ch, 3, 3))
        self.bias = nn.Parameter(torch.zeros(out_ch))
        self.register_buffer("noise_const", torch.randn(resolution, resolution))
        self.noise_strength = nn.Parameter(torch.zeros([]))
        self.register_buffer("fir", fir_filter())
        self.attention = BipartiteAttention(out_ch, w_dim, components_num, **attn_kwargs) if use_attention else None

    def _conv_weights(self):
        O, I, kh, kw = self.weight.shape
        w = self.weight * (1.0 / math.sqrt(I * kh * kw))
        wsq = w.square().sum(dim=[2, 3])
        phases = ops.upconv_phase_weights(w) if self.up else None
        packed = None
        if w.is_cuda and kh == 3 and I % 32 == 0 and O % 64 == 0 and (not self.up or upconv_fused(self.resolution)):
            packed = ops.conv3x3_pack(w)      # [9, O, I], TF32-rounded: operand of gf_conv3x3_nhwc_tf32 / gf_upconv3x3_blur_nhwc_tf32
        if self.up:
            w = w.transpose(0, 1)
        return w.contiguous(memory_format=torch.channels_last), wsq.contiguous(), phases, packed

    def fusable(self, x) -> bool:
        """Inference on CUDA with an attention block whose norm the kernels can fuse around."""
        a = self.attention
        return (a is not None and x.is_cuda and a.norm in ("layer", None, "none")
                and _inference(self.weight, self.bias, self.noise_strength, *a.parameters()))

    def forward(self, x, w_glob, y, noise_mode="const", centroids=None, return_att=False, styles=None,
                prescaled=False, post_scale=None, prepared=None, rgb=None, centroids_init=None, demod=None):
        """prescaled: x already carries this layer's style scale.  post_scale [B,C]: the NEXT convolution's style scale,
        folded into this layer's store (only honoured -- and only passed by SynthesisNetwork -- when `fusable`).
        rgb: dict(rgb_w [B,3,C], rgb_bias [3], rgb_out [B,3,H,W]) -- the block's tRGB computed by the attention kernel's store side
        from the layer output (fused path on the wgmma kernel only; SynthesisNetwork checks)."""
        if styles is None:
            styles = self.affine(w_glob)
        w_eff = wsq = phases = packed = None
        if _inference(self.weight) and x.is_cuda:
            w_eff, wsq, phases, packed = _cached(self, "conv", (self.weight,), self._conv_weights)
            # own convolution kernels: TF32 only (the parity tests run true-fp32 convolutions); the stride-1 kernel takes patches of
            # 8 x 16 pixels and can be switched to cuDNN (GF_CUDNN_CONV), the upsampling kernel any size (packed where upconv_fused)
            if packed is not None and not (torch.backends.cudnn.allow_tf32 and x.dtype == torch.float32
                                           and (self.up or (x.shape[2] % 8 == 0 and x.shape[3] % 16 == 0
                                                            and not os.environ.get("GF_CUDNN_CONV")))):
                packed = None
        fused = self.fusable(x)
        in_scale = None
        # prepared = (event | None, demod): SynthesisNetwork already ran this layer's stage I (batched launch)
        if prepared is not None and not fused:
            raise RuntimeError("internal: prepared prologue for a layer that does not take the fused path")
        if fused and not self.up:      # demodulation rides on the attention kernel's load side (folded into K')
            x, in_scale = modulated_conv2d(x, self.weight, styles, up=1, f=self.fir, w_eff=w_eff, wsq=wsq,
                                           prescaled=prescaled, defer_demod=True, d=prepared[1] if prepared is not None else demod,
                                           wt_packed=packed)
        else:
            x = modulated_conv2d(x, self.weight, styles, up=2 if self.up else 1, f=self.fir, w_eff=w_eff, wsq=wsq,
                                 prescaled=prescaled, phases=phases, wt_packed=packed, d=demod)
        if noise_mode == "const":
            noise = self.noise_const
        elif noise_mode == "random":
            noise = torch.randn(x.shape[0], 1, self.resolution, self.resolution, device=x.device, dtype=x.dtype)
        else:
            noise = None
        att = None
        if self.attention is not None:
            xl = x.permute(0, 2, 3, 1)                                  # channels-last storage -> [B,H,W,C] view
            if not xl.is_contiguous():
                xl = xl.contiguous()
            if fused:   # demod (load side) + noise + bias + leaky-ReLU + next style (store side) ride on the attention kernel
                post = dict(bias=self.bias, noise=noise, strength=self.noise_strength, act="lrelu", gain=SQRT2,
                            in_scale=in_scale, post_scale=post_scale)
                if rgb is not None:
                    post.update(rgb)
                post.update(self.attention.dropout_postop(x.device))     # training-mode forward under no_grad (the D step's fakes)
                if prepared is not None and prepared[0] is not None:
                    torch.cuda.current_stream(x.device).wait_event(prepared[0])
                xo, att, centroids = self.attention(xl, y, centroids=centroids, return_att=return_att, postop=post,
                                                    stage="token" if prepared is not None else "all",
                                                    need_centroids=self.attention.iterative,     # read back only to carry them on
                                                    centroids_init=centroids_init)
                return xo.permute(0, 3, 1, 2), att, centroids
            xo, att, centroids = self.attention(xl, y, centroids=centroids, return_att=return_att, centroids_init=centroids_init)
            x = xo.permute(0, 3, 1, 2)                                  # back to an NCHW view of channels-last data
        x = ops.bias_act(x, self.bias, "lrelu", noise=noise, strength=self.noise_strength)
        if post_scale is not None:
            x = ops.chan_scale(x, post_scale)
        return x, att, centroids


class ToRGB(nn.Module):
    def __init__(self, in_ch: int, w_dim: int, img_channels: int = 3):
        super().__init__()
        self.affine = FullyConnected(w_dim, in_ch, bias_init=1.0)
        self.weight = nn.Parameter(torch.randn(img_channels, in_ch, 1, 1))
        self.bias = nn.Parameter(torch.zeros(img_channels))

    def forward(self, x, w_glob, styles=None, next_styles=None):
        """1x1 modulated conv without demodulation: the style is folded into per-sample [3, C] weights, so the
        activations are read once and no styled copy is written.  next_styles: also return x * next_styles (the next
        block's modulated input) from the same read."""
        if styles is None:
            styles = self.affine(w_glob)                                # [B, C]
        return ops.torgb(x, self.weight, styles, self.bias, next_styles=next_styles)


class SynthesisNetwork(nn.Module):
    """G_synthesis, skip architecture.  Attention on both conv layers of every resolution in [start_res, end_res]."""

    def __init__(self, resolution: int, latent_dim: int, components_num: int, fmap_base: int = 16384, fmap_max: int = 512,
                 g_start_res: int = 8, g_end_res: Optional[int] = None, transformer: bool = True, attn_kwargs: Optional[dict] = None,
                 img2img: int = 0):
        super().__init__()
        assert resolution >= 4 and resolution & (resolution - 1) == 0
        if img2img and not (8 <= img2img <= resolution and img2img & (img2img - 1) == 0):
            raise ValueError(f"img2img must be 0 (off) or a block resolution in 8 .. {resolution}, got {img2img}")
        self.resolution, self.components_num = resolution, components_num
        g_end_res = resolution if g_end_res is None else g_end_res
        self.block_resolutions = [2 ** i for i in range(2, int(math.log2(resolution)) + 1)]
        attn_kwargs = dict(attn_kwargs or {})
        self.const = nn.Parameter(torch.randn(nf(4, fmap_base, fmap_max), 4, 4))
        self.layers = nn.ModuleList()
        self.torgbs = nn.ModuleList()
        self.layer_res: List[int] = []
        # `iterative` (SURVEY A.3, [SPEC]): a duplex layer's centroids initialise the k-means of the NEXT attention layer when the
        # channel width is the same (both layers of a block; consecutive blocks of equal width): that layer's first queries come
        # from the carried centroids (through wcq) instead of from the latents.  Across a change of width nothing is carried.
        self.iterative = bool(attn_kwargs.get("iterative", False)) and bool(attn_kwargs.get("kmeans", False))
        for res in self.block_resolutions:
            out_ch = nf(res, fmap_base, fmap_max)
            use_att = transformer and components_num > 0 and g_start_res <= res <= g_end_res
            if res > 4:
                in_ch = nf(res // 2, fmap_base, fmap_max)
                self.layers.append(SynthesisLayer(in_ch, out_ch, latent_dim, res, True, components_num, use_att, attn_kwargs))
                self.layer_res.append(res)
            self.layers.append(SynthesisLayer(out_ch, out_ch, latent_dim, res, False, components_num, use_att, attn_kwargs))
            self.layer_res.append(res)
            self.torgbs.append(ToRGB(out_ch, latent_dim))
        self.register_buffer("fir", fir_filter())
        # img2img (SURVEY A.4 item 18): image self-attention on the output of block `img2img`, before its tRGB
        self.img2img_res = int(img2img)
        self.img2img = None
        if img2img:
            a = attn_kwargs
            self.img2img = ImageSelfAttention(nf(img2img, fmap_base, fmap_max), a.get("pos_dim") or latent_dim,
                                              integration=a.get("integration", "mul"), norm=a.get("norm", "layer"),
                                              use_pos=a.get("use_pos", True), exact_fp32=a.get("exact_fp32", False))
        self.num_attention_layers = sum(1 for l in self.layers if l.attention is not None)
        # index into per-layer latents [B, num_ws, k+1, D] of every style affine (conv layers, then tRGBs): conv layer i reads
        # index i, the tRGB of a block reads the index after its block's last conv layer (SURVEY A.4 item 13)
        ends = list(np.cumsum([1 if res == 4 else 2 for res in self.block_resolutions]))
        self.ws_index: List[int] = list(range(len(self.layers))) + [int(e) for e in ends]

    @property
    def num_ws(self) -> int:
        """Number of per-layer latent sets ``forward`` accepts: one per conv layer, plus one for the last tRGB."""
        return len(self.layers) + 1

    def forward(self, ws: torch.Tensor, noise_mode: str = "const", return_att: bool = False, return_features: bool = False):
        """ws: [B, k+1, D] (every layer reads the same latents) or per-layer [B, num_ws, k+1, D] (style mixing: conv layer i
        takes its attention latents ws[:, i, :k] and its style from ws[:, i, k]; a block's tRGB takes the index after its last
        conv layer).  return_features: also return, per attention layer, the layer's activation after noise + bias + leaky-ReLU and
        before the next convolution's style scale, as NCHW views (parity checks against oracle.generator, which returns the
        same quantity).  The store-side fusion of the NEXT layer's style scale is switched off for such a call, so that the
        captured activations are exactly the layer outputs; everything else takes the same kernels."""
        k = self.components_num
        B = ws.shape[0]
        per_layer = ws.dim() == 4
        if per_layer:
            if ws.shape[1] != self.num_ws or ws.shape[2] != k + 1:
                raise ValueError(f"per-layer ws must be [B, {self.num_ws}, {k + 1}, D], got {tuple(ws.shape)}")
            wsl = ws.transpose(0, 1)                                    # [L, B, k+1, D]
            ys = list(wsl[:, :, :k].contiguous().unbind(0))             # one copy for all layers; each [B, k, D] contiguous
            wgs = wsl[:, :, k]                                          # [L, B, D]
        else:
            y = ws[:, :k].contiguous()
            w_glob = ws[:, k]
            ys, wgs = [y] * self.num_ws, [w_glob] * self.num_ws
        x = self.const[None].expand(B, -1, -1, -1).contiguous(memory_format=torch.channels_last)
        # all style affines (one per conv layer and per tRGB) read the same global latent: one batched GEMM at inference; with
        # per-layer latents, the same GEMM once per latent set, of which each affine keeps its own columns (the same operand shapes
        # as the shared-latent GEMM, so equal latent sets give its result bit for bit)
        mods = list(self.layers) + list(self.torgbs)
        aff = [m.affine for m in mods]
        aff_params = [t for a in aff for t in (a.weight, a.bias)]
        styles_all = [None] * len(mods)
        if _inference(*aff_params):
            def cat_affines():
                ws_, bs_ = zip(*[a.effective() for a in aff])
                return torch.cat(ws_, dim=1).contiguous(), torch.cat(bs_)
            wt_cat, b_cat = _cached(self, "affines", aff_params, cat_affines)
            widths = [a.weight.shape[0] for a in aff]
            if per_layer:
                per_set = [torch.addmm(b_cat, wgs[i], wt_cat).split(widths, dim=1) for i in range(self.num_ws)]
                styles_all = [per_set[i][m] for m, i in enumerate(self.ws_index)]
            else:
                styles_all = torch.addmm(b_cat, w_glob, wt_cat).split(widths, dim=1)
        # Stage I of every attention layer (keys / V^T / positional tables of a simplex layer, pass-A query tables + V^T of a
        # duplex layer) depends only on the latents and the styles: ONE batched launch for the whole network
        # (gf_attn_prologue_batch) instead of two small launches in front of every layer's token pass.
        prepared = [None] * len(self.layers)
        demods = [None] * len(self.layers)
        if x.is_cuda and styles_all[0] is not None and _inference(*[l.weight for l in self.layers]):
            # every layer's demodulation coefficients depend on the styles only: one launch for the network (gf_demod_coef_batch)
            demods = ops.demod_coef_batch([(styles_all[li_], _cached(l, "conv", (l.weight,), l._conv_weights)[1])
                                           for li_, l in enumerate(self.layers)])
        if x.is_cuda and styles_all[0] is not None and not os.environ.get("GF_NO_BATCH_PROLOGUE"):
            items = []
            for li_, layer in enumerate(self.layers):
                if not layer.fusable(x):
                    continue
                d_ = None
                if not layer.up:        # the demodulation of a stride-1 convolution rides on the attention kernel's load side
                    d_ = demods[li_]
                    if d_ is None:
                        _, wsq_, _, _ = _cached(layer, "conv", (layer.weight,), layer._conv_weights)
                        d_ = ops.demod_coef(styles_all[li_], wsq_)
                C_ = layer.weight.shape[0]
                items.append((layer.attention, ys[li_], (B, layer.resolution, layer.resolution, C_), d_))
                prepared[li_] = (None, d_)
            prologue_batch(items)
        img = None
        atts = []
        feats = []
        li = 0
        block_prescaled = False
        cen_prev = None
        for bi, res in enumerate(self.block_resolutions):
            nl = 1 if res == 4 else 2
            prescaled = block_prescaled
            # the tRGB pass reads x anyway: it can also write the next block's style-modulated input (inference only)
            nxt = styles_all[li + nl] if (li + nl < len(self.layers) and styles_all[li + nl] is not None and x.is_cuda and not return_features
                                          and not os.environ.get("GF_NO_TORGB_FUSE")) else None
            rgb = None
            for j in range(nl):
                layer = self.layers[li]
                cen_init = None                     # iterative: carry the previous attention layer's centroids when the widths match
                if self.iterative and layer.attention is not None and cen_prev is not None and cen_prev.shape[2] == layer.weight.shape[0] \
                        and _inference(*layer.attention.parameters()):
                    cen_init = cen_prev
                # conv0 -> conv1 inside a block has a single consumer: conv1's style scale is folded into conv0's store
                post_scale = None
                if j == 0 and nl == 2 and styles_all[li + 1] is not None and layer.fusable(x) and not return_features:
                    post_scale = styles_all[li + 1]
                rgb_args = None
                if j == nl - 1 and layer.fusable(x) and not return_features and res != self.img2img_res \
                        and not os.environ.get("GF_NO_TORGB_EPILOGUE"):
                    # last layer of the block on the wgmma path (C <= 256, or 512 with k <= 16): the attention kernel's store side computes the
                    # tRGB planes from the layer output and writes x * (next block's style): the tRGB pass disappears
                    C_ = layer.weight.shape[0]
                    tg = self.torgbs[bi]
                    if (C_ <= 256 or (k <= 16 and not os.environ.get("GF_TORGB_EPILOGUE_C256"))) and _inference(tg.weight, tg.bias) \
                            and tc_eligible(layer.attention, (B, res, res, C_), k):
                        st_rgb = styles_all[len(self.layers) + bi]
                        rgb_w = (tg.weight.reshape(1, 3, C_) * st_rgb[:, None, :] * (1.0 / math.sqrt(C_))).contiguous()
                        rgb = torch.empty((B, 3, res, res), device=x.device, dtype=torch.float32)
                        rgb_args = dict(rgb_w=rgb_w, rgb_bias=tg.bias, rgb_out=rgb)
                        post_scale = nxt
                x, att, cen_out = layer(x, wgs[li], ys[li], noise_mode=noise_mode, return_att=return_att, styles=styles_all[li],
                                        prescaled=prescaled, post_scale=post_scale, prepared=prepared[li], rgb=rgb_args,
                                        centroids_init=cen_init, demod=demods[li])
                if layer.attention is not None:
                    cen_prev = cen_out if self.iterative else None
                prescaled = post_scale is not None
                li += 1
                if att is not None:
                    atts.append(att)
                if return_features and layer.attention is not None:
                    feats.append(x)
            if res == self.img2img_res:        # the block's activation is attended, then read by its tRGB (and scaled for the next block)
                x = self.img2img(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2)
            if rgb is not None:
                block_prescaled = nxt is not None
            else:
                rgb = self.torgbs[bi](x, wgs[self.ws_index[len(self.layers) + bi]], styles=styles_all[len(self.layers) + bi], next_styles=nxt)
                block_prescaled = nxt is not None
                if block_prescaled:
                    rgb, x = rgb
            img = rgb if img is None else ops.upsample2x(img, self.fir, add=rgb)
        out = (img,) + ((atts,) if return_att else ()) + ((feats,) if return_features else ())
        return out[0] if len(out) == 1 else out


class Generator(nn.Module):
    """G_GANsformer.  ``G(z, c=None, truncation_psi=1.0, noise_mode='const', return_att=False) -> img [B,3,R,R]``.

    ``c_dim > 0``: class-conditional (SURVEY A.4 item 14).  Every call then takes labels c [B, c_dim] (one-hot or any real weights),
    which act through the mapping network's label embedding only; with the default ``c_dim = 0`` c is ignored.

    ``img2img = r`` (SURVEY A.4 item 18): image self-attention (``ImageSelfAttention``, with the generator's integration, norm and
    use_pos) on the output of block r, after its last synthesis layer and before its tRGB; r is a block resolution in 8 .. resolution.
    The layer has no latent input: num_ws, style mixing and the latent routing are unchanged.  0 (the default) builds exactly the
    network without it.

    ``pl_kernels=True`` runs the img2img layer's part of the path-length penalty on the double-backward kernel
    (``ImageSelfAttention.kernel_double_backward``) instead of the torch composite, which holds n x n tensors.  It changes only that
    layer: the bipartite attention layers run their path-length pass on kernels already.  The gradients then differ from the
    default route by TF32 round-off."""

    def __init__(self, resolution: int = 256, components_num: int = 16, latent_size: int = 512, latent_dim: Optional[int] = None,
                 transformer: bool = True, g_start_res: int = 8, g_end_res: Optional[int] = None, kmeans: bool = False,
                 kmeans_iters: int = 1, iterative: bool = False, integration: str = "mul", norm: Optional[str] = "layer",
                 use_pos: bool = True, pos_dim: Optional[int] = None, num_heads: int = 1, mapping_layers: int = 8,
                 fmap_base: int = 16384, fmap_max: int = 512, exact_fp32: bool = False, ltnt2ltnt: bool = False, g_img2ltnt: bool = False,
                 att_dp: float = 0.0, c_dim: int = 0, img2img: int = 0, pl_kernels: bool = False):
        super().__init__()
        # SURVEY A.4 item 1: D = latent_size // components_num unless given
        self.latent_dim = latent_dim if latent_dim is not None else max(latent_size // max(components_num, 1), 1)
        self.components_num, self.resolution = components_num, resolution
        attn_kwargs = dict(pos_dim=pos_dim, num_heads=num_heads, integration=integration, norm=norm, kmeans=kmeans,
                           kmeans_iters=kmeans_iters, use_pos=use_pos, exact_fp32=exact_fp32, iterative=iterative,
                           img2ltnt=bool(g_img2ltnt and kmeans), att_dp=att_dp)
        self.mapping = MappingNetwork(self.latent_dim, components_num, num_layers=mapping_layers, ltnt2ltnt=ltnt2ltnt,
                                      integration=integration, norm=norm, exact_fp32=exact_fp32, c_dim=c_dim)
        self.c_dim = int(c_dim)
        self.synthesis = SynthesisNetwork(resolution, self.latent_dim, components_num, fmap_base=fmap_base, fmap_max=fmap_max,
                                          g_start_res=g_start_res, g_end_res=g_end_res, transformer=transformer,
                                          attn_kwargs=attn_kwargs, img2img=img2img)
        if self.synthesis.img2img is not None:
            self.synthesis.img2img.kernel_double_backward = bool(pl_kernels)

    def forward(self, z: torch.Tensor, c=None, truncation_psi: float = 1.0, noise_mode: str = "const", return_att: bool = False,
                return_features: bool = False):
        ws = self.mapping(z, c, truncation_psi=truncation_psi)
        return self.synthesis(ws, noise_mode=noise_mode, return_att=return_att, return_features=return_features)

    def __deepcopy__(self, memo):
        """Copies parameters and buffers only: caches, captured graphs, streams and attention plans stay with the original
        (a copied graph closure would replay the ORIGINAL module's weights)."""
        import copy as _copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k_, v_ in self.__dict__.items():
            if k_ in RUNTIME_KEYS or isinstance(k_, tuple):
                continue
            new.__dict__[k_] = _copy.deepcopy(v_, memo)
        return drop_runtime_state(new)

    def load_state_dict(self, *args, **kwargs):
        res = super().load_state_dict(*args, **kwargs)
        bump_weights_epoch()
        drop_runtime_state(self)
        return res

    # ------------------------------------------------------------------------------------------------------------
    # CUDA-graph replay of the whole forward (the step is ~370 small launches; graphs remove the launch overhead)
    # ------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def graphed(self, batch_size: int, truncation_psi: float = 1.0, noise_mode: str = "const"):
        """Returns ``fn(z_device, c_device=None) -> img`` replaying a captured CUDA graph of ``self(z, c)`` for this batch size (the
        labels go through a static buffer of their own; an unconditional generator ignores them).

        The returned image tensor is a static buffer overwritten by the next replay.  Weight-derived tensors (folded
        attention weights, scaled conv weights) are baked at capture, so the graph is keyed on the parameters' storage,
        version counters and the process-wide weights epoch: any weight update re-captures."""
        key = (batch_size, float(truncation_psi), noise_mode, weights_epoch(), bool(torch.backends.cudnn.allow_tf32), bool(os.environ.get("GF_CUDNN_CONV")),
               tuple((p.data_ptr(), p._version) for p in self.parameters()))
        cache = self.__dict__.setdefault("_graphs", {})
        if key in cache:
            return cache[key]
        cache.clear()                                   # a stale graph holds a full set of activations: drop it
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("CUDA graphs need the generator on a CUDA device")
        static_z = torch.zeros(batch_size, self.components_num + 1, self.latent_dim, device=dev)
        static_c = torch.zeros(batch_size, self.c_dim, device=dev) if self.c_dim > 0 else None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(3):                      # warm-up: cuDNN autotune, weight folding, workspace allocation
                self(static_z, static_c, truncation_psi=truncation_psi, noise_mode=noise_mode)
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_img = self(static_z, static_c, truncation_psi=truncation_psi, noise_mode=noise_mode)

        labels = self.mapping.labels        # not `self`: the cached closure must not keep the generator (and its graphs) alive

        def replay(z: torch.Tensor, c: Optional[torch.Tensor] = None) -> torch.Tensor:
            if static_c is not None:
                static_c.copy_(labels(c, batch_size, static_c), non_blocking=True)
            static_z.copy_(z, non_blocking=True)
            graph.replay()
            return static_img

        cache[key] = replay
        return replay

    @torch.no_grad()
    def run(self, latents, labels=None, truncation_psi: float = 1.0, randomize_noise: bool = False, minibatch_size: int = 32,
            cuda_graph: bool = False, out: Optional[torch.Tensor] = None):
        """``Gs.run``-shaped convenience wrapper (reference: dnnlib/tflib/network.py Network.run): host numpy/tensor
        latents in, host images out, processed in minibatches on this module's device.  ``cuda_graph=True`` replays a
        captured graph for full minibatches; ``out`` may be a (pinned) host tensor to receive the images.  ``labels`` [N, c_dim]
        go with the latents, minibatch by minibatch (required iff c_dim > 0; ignored otherwise)."""
        dev = next(self.parameters()).device
        lat = torch.as_tensor(np.asarray(latents) if not torch.is_tensor(latents) else latents, dtype=torch.float32)
        n = lat.shape[0]
        lab = None
        if self.c_dim > 0:
            lab = self.mapping.labels(labels if labels is None or torch.is_tensor(labels) else np.asarray(labels), n, lat)
        cs = lambda i, m: None if lab is None else lab[i:i + m].to(dev, non_blocking=True)
        noise_mode = "random" if randomize_noise else "const"
        res = out if out is not None else torch.empty((n, 3, self.resolution, self.resolution), dtype=torch.float32)
        if dev.type != "cuda":
            for i in range(0, n, minibatch_size):
                z = lat[i:i + minibatch_size].to(dev)
                res[i:i + z.shape[0]].copy_(self(z, cs(i, z.shape[0]), truncation_psi=truncation_psi, noise_mode=noise_mode))
            return res
        # CUDA: the device->host copy of minibatch i runs on a copy stream while minibatch i+1 computes (two staging buffers;
        # effective with pinned `out` / latents)
        main = torch.cuda.current_stream(dev)
        copy_stream = self.__dict__.get("_copy_stream")
        if copy_stream is None or copy_stream.device != dev:
            copy_stream = self.__dict__["_copy_stream"] = torch.cuda.Stream(device=dev)
        skey = ("_staging", minibatch_size)
        staging = self.__dict__.get(skey)
        if staging is None or staging[0].device != dev:
            staging = self.__dict__[skey] = [torch.empty((minibatch_size, 3, self.resolution, self.resolution), device=dev) for _ in range(2)]
        d2h_done = [None, None]
        for idx, i in enumerate(range(0, n, minibatch_size)):
            z = lat[i:i + minibatch_size].to(dev, non_blocking=True)
            m = z.shape[0]
            c = cs(i, m)
            if cuda_graph and m == minibatch_size:
                img = self.graphed(minibatch_size, truncation_psi, noise_mode)(z, c)
            else:
                img = self(z, c, truncation_psi=truncation_psi, noise_mode=noise_mode)
            sidx = idx & 1
            if d2h_done[sidx] is not None:
                main.wait_event(d2h_done[sidx])                 # the copy that last read this staging buffer has finished
            staging[sidx][:m].copy_(img)
            ready = torch.cuda.Event()
            ready.record(main)
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(ready)
                res[i:i + m].copy_(staging[sidx][:m], non_blocking=True)
                d2h_done[sidx] = torch.cuda.Event()
                d2h_done[sidx].record(copy_stream)
        copy_stream.synchronize()
        main.synchronize()
        return res
