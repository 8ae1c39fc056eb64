"""CPU oracle of the discriminator forward (StyleGAN2 residual discriminator + the GANsformer discriminator's attention), NCHW,
direct op order.

TEST INFRASTRUCTURE ONLY; PARITY UNPINNED -- see oracle/bipartite.py.  Like oracle/generator.py it consumes the *state_dict* of
the product ``Discriminator`` but none of its code: equalised-LR convolutions, FIR downsampling as upfirdn (pad, then the 4x4
[1,3,3,1] filter as a depthwise convolution, then the strided convolution), minibatch standard deviation, and the attention
through ``oracle.bipartite.transformer_layer(duplex=True, img2ltnt=True)`` with its two transposes.  SURVEY A.4 item 11: the
learned aggregator latents are broadcast to Y; after each attention layer Y <- LN(Y) (1 + dense(Cen, wi2l) + bi2l), the values
that layer used; fc0 takes [flatten(x), flatten(Y)].  Which layers have attention follows from the state dict.

Tensors already in the requested dtype on the CPU are used as they are, so float64 leaves that require grad give the
oracle's first and second derivatives (the R1 penalty) through plain autograd.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .bipartite import _dense, att_norm, transformer_layer

SQRT2 = math.sqrt(2.0)


def _fir(dtype):
    f = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64)
    f = torch.outer(f, f)
    return (f / f.sum()).to(dtype)


def _conv(x, sd, pre, down=False, act="lrelu"):
    w = sd[pre + ".weight"]
    O, I, kh, kw = w.shape
    w = w * (1.0 / math.sqrt(I * kh * kw))
    if down:
        p = (4 - 2) + (kh - 1)                                           # StyleGAN2 conv_downsample_2d: FIR taps - stride + kernel - 1
        x = F.pad(x, [(p + 1) // 2, p // 2, (p + 1) // 2, p // 2])
        C = x.shape[1]
        x = F.conv2d(x, _fir(x.dtype)[None, None].expand(C, 1, 4, 4), groups=C)
        x = F.conv2d(x, w, stride=2)
    else:
        x = F.conv2d(x, w, padding=kh // 2)
    b = sd.get(pre + ".bias")
    if b is not None:
        x = x + b[None, :, None, None]
    return F.leaky_relu(x, 0.2) * SQRT2 if act == "lrelu" else x


def _fc(x, sd, pre, act="linear"):
    w = sd[pre + ".weight"]
    x = x @ (w * (1.0 / math.sqrt(w.shape[1]))).t() + sd[pre + ".bias"]
    return F.leaky_relu(x, 0.2) * SQRT2 if act == "lrelu" else x


def _attention(x, y, sd, pre, integration, norm, use_pos):
    w = {n[len(pre) + 1:]: t for n, t in sd.items() if n.startswith(pre + ".")}
    x, _, cen = transformer_layer(x, y, w, integration=integration, norm=norm, duplex=True, use_pos=use_pos, img2ltnt=True)
    return x, att_norm(y, "layer") * (1.0 + _dense(cen, w["wi2l"], w["bi2l"]))


def discriminator_forward(sd: Dict[str, torch.Tensor], img: torch.Tensor, *, mbstd_group: int = 4, integration: str = "mul",
                          norm: Optional[str] = "layer", use_pos: bool = True, dtype=torch.float64, return_latents: bool = False):
    """img [B, 3, R, R] -> logits [B] (and, with return_latents, the list of Y: the broadcast latents, then Y after every attention
    layer).  `sd` = product Discriminator.state_dict()."""
    cast = lambda t: t if (t.dtype == dtype and t.device.type == "cpu") else t.detach().to("cpu", dtype)
    sd = {n: cast(t) for n, t in sd.items() if t.is_floating_point()}
    x = cast(img)
    B = x.shape[0]
    ys = []
    y = None
    if "latents" in sd:
        y = sd["latents"][None].expand(B, -1, -1)
        ys.append(y)
    x = _conv(x, sd, "fromrgb")
    i = 0
    while f"blocks.{i}.conv0.weight" in sd:
        pre = f"blocks.{i}"
        t = _conv(x, sd, pre + ".conv0")
        if pre + ".att0.wq" in sd:
            t, y = _attention(t, y, sd, pre + ".att0", integration, norm, use_pos)
            ys.append(y)
        t = _conv(t, sd, pre + ".conv1", down=True)
        if pre + ".att1.wq" in sd:
            t, y = _attention(t, y, sd, pre + ".att1", integration, norm, use_pos)
            ys.append(y)
        x = (_conv(x, sd, pre + ".skip", down=True, act="linear") + t) * (1.0 / SQRT2)
        i += 1
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
    out = _fc(_fc(x, sd, "fc0", act="lrelu"), sd, "fc1").reshape(B)
    return (out, ys) if return_latents else out
