"""fp64 restatement of the generator and the discriminator with an image self-attention layer (img2img, SURVEY A.4 item 18), for
tests/test_host_cpu_img2img.py and tests/test_gpu_img2img.py.

Test infrastructure only, beside oracle/generator.py and oracle/discriminator.py, which have no img2img layer.  Built from the
oracle's own blocks in their order, with ``oracle.self_attention.self_attention_layer`` inserted:
* generator: on the output of block r (after its last layer's noise, bias and leaky ReLU), before the block's tRGB;
* discriminator: on the activation entering the block of input resolution r.
The state dict and inputs are used as given (no detach, no cast); ``cast`` prepares a product state dict.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle.bipartite import transformer_layer
from oracle.discriminator import _attention, _conv
from oracle.discriminator import _fc as _dfc
from oracle.generator import SQRT2, _fc, _fir, _modconv, _upfirdn
from oracle.self_attention import self_attention_layer


def cast(sd: Dict[str, torch.Tensor], dtype=torch.float64) -> Dict[str, torch.Tensor]:
    return {n: t.detach().to("cpu", dtype) if t.is_floating_point() else t.detach().cpu() for n, t in sd.items()}


def _img2img_weights(sd, pre):
    return {n[len(pre):]: t for n, t in sd.items() if n.startswith(pre)}


def generator_forward(sd, z, *, resolution: int, components_num: int, latent_dim: int, img2img: int, mapping_layers: int = 8,
                      integration="mul", norm="layer", use_pos=True, g_start_res: int = 8, noise_mode: str = "const"):
    """z [B, k+1, D] -> img [B, 3, R, R] of a simplex generator (every layer reads the same latents) with img2img at block r."""
    k, D = components_num, latent_dim
    B = z.shape[0]
    z = z * torch.rsqrt(z.square().mean(dim=2, keepdim=True) + 1e-8)
    loc, glo = z[:, :k], z[:, k:]
    for i in range(mapping_layers):
        loc = _fc(loc, sd, f"mapping.local.{i}", D, lr_mul=0.01, act="lrelu")
        glo = _fc(glo, sd, f"mapping.glob.{i}", D, lr_mul=0.01, act="lrelu")
    y, w_glob = loc, glo[:, 0]
    f = _fir(z.dtype)
    x = sd["synthesis.const"][None].expand(B, -1, -1, -1)
    img = None
    li = 0
    for bi, res in enumerate([2 ** i for i in range(2, int(math.log2(resolution)) + 1)]):
        for j in range(1 if res == 4 else 2):
            pre = f"synthesis.layers.{li}"
            li += 1
            styles = _fc(w_glob, sd, pre + ".affine", D)
            x = _modconv(x, sd[pre + ".weight"], styles, up=2 if (res > 4 and j == 0) else 1, f=f)
            if (pre + ".attention.wq") in sd and g_start_res <= res:
                w = {n[len(pre) + 11:]: t for n, t in sd.items() if n.startswith(pre + ".attention.")}
                x, _, _ = transformer_layer(x, y, w, integration=integration, norm=norm, use_pos=use_pos)
            if noise_mode == "const":
                x = x + sd[pre + ".noise_const"] * sd[pre + ".noise_strength"]
            x = F.leaky_relu(x + sd[pre + ".bias"][None, :, None, None], 0.2) * SQRT2
        if res == img2img:
            x = self_attention_layer(x, _img2img_weights(sd, "synthesis.img2img."), integration=integration, norm=norm, use_pos=use_pos)
        pre = f"synthesis.torgbs.{bi}"
        styles = _fc(w_glob, sd, pre + ".affine", D)
        rgb = _modconv(x, sd[pre + ".weight"], styles, demodulate=False) + sd[pre + ".bias"][None, :, None, None]
        img = rgb if img is None else _upfirdn(img, f, up=2, pad=(2, 1, 2, 1), gain=4.0) + rgb
    return img


def discriminator_forward(sd, img, *, img2img: int, mbstd_group: int = 4, integration: str = "mul", norm: Optional[str] = "layer",
                          use_pos: bool = True):
    """img [B, 3, R, R] -> logits [B] of an unconditional discriminator (with or without bipartite attention) with img2img."""
    x = img
    B, _, R, _ = x.shape
    y = sd["latents"][None].expand(B, -1, -1) if "latents" in sd else None
    x = _conv(x, sd, "fromrgb")
    i, res = 0, R
    while f"blocks.{i}.conv0.weight" in sd:
        if res == img2img:
            x = self_attention_layer(x, _img2img_weights(sd, "img2img."), integration=integration, norm=norm, use_pos=use_pos)
        pre = f"blocks.{i}"
        t = _conv(x, sd, pre + ".conv0")
        if pre + ".att0.wq" in sd:
            t, y = _attention(t, y, sd, pre + ".att0", integration, norm, use_pos)
        t = _conv(t, sd, pre + ".conv1", down=True)
        if pre + ".att1.wq" in sd:
            t, y = _attention(t, y, sd, pre + ".att1", integration, norm, use_pos)
        x = (_conv(x, sd, pre + ".skip", down=True, act="linear") + t) * (1.0 / SQRT2)
        i, res = i + 1, res // 2
    _, C, H, W = x.shape
    G = min(mbstd_group, B)
    while B % G:
        G -= 1
    s = x.reshape(G, B // G, C, H, W)
    s = torch.sqrt(((s - s.mean(dim=0, keepdim=True)) ** 2).mean(dim=0) + 1e-8).mean(dim=[1, 2, 3])
    s = s.reshape(1, B // G, 1, 1).expand(G, -1, H, W).reshape(B, 1, H, W)
    x = _conv(torch.cat([x, s], dim=1), sd, "conv4").reshape(B, -1)
    if y is not None:
        x = torch.cat([x, y.reshape(B, -1)], dim=1)
    return _dfc(_dfc(x, sd, "fc0", act="lrelu"), sd, "fc1").reshape(B)
