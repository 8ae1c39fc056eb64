"""fp64 restatement of the synthesis network with per-layer latents (style mixing, SURVEY A.4 item 13), for
tests/test_host_cpu_style_mixing.py and tests/test_gpu_style_mixing.py.

Test infrastructure only, beside oracle/generator.py, whose ``generator_forward`` gives every layer the same latents: here conv
layer i takes its attention latents ws_l[:, i, :k] and its style from ws_l[:, i, k], and the tRGB of a block the index after the
block's last conv layer.  The state dict and the latents are used as given (no detach, no cast), so fp64 leaves that require grad
give gradients.  Built from the oracle's own blocks (fully connected layer, reference-style modulated convolution, FIR,
``oracle.bipartite.transformer_layer``), in the same order as ``generator_forward``.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle.bipartite import transformer_layer
from oracle.generator import SQRT2, _fc, _fir, _modconv, _upfirdn


def mix_latents(ws1: torch.Tensor, ws2: torch.Tensor, cutoff: int, num_ws: int) -> torch.Tensor:
    """The index rule of style mixing: ws_l[:, i] = ws1 for i < cutoff, ws2 from the cutoff on.  -> [B, num_ws, k+1, D]."""
    return torch.stack([ws1 if i < cutoff else ws2 for i in range(num_ws)], dim=1)


def synthesis_forward(sd: Dict[str, torch.Tensor], ws_l: torch.Tensor, *, resolution: int, components_num: int,
                      integration="mul", norm="layer", duplex=False, use_pos=True, num_heads=1, g_start_res: int = 8,
                      g_end_res: Optional[int] = None, noise_mode: str = "const", kmeans_iters: int = 1, img2ltnt: bool = False,
                      iterative: bool = False, return_att: bool = False,
                      lrelu_pos: Optional[List[Optional[torch.Tensor]]] = None):
    """G_synthesis of ``generator_forward`` from per-layer latents ws_l [B, L, k+1, D] (L = conv layers + 1).  lrelu_pos: per
    attention layer (in order), a boolean [B, C, H, W] choosing the slope of its leaky ReLU (1 where True, 0.2 elsewhere) instead of
    the sign of the fp64 pre-activation (see tests/generator_path_length_ref.py).  -> img [B, 3, R, R] (, attention maps)."""
    k = components_num
    g_end_res = resolution if g_end_res is None else g_end_res
    B, L, _, D = ws_l.shape
    f = _fir(ws_l.dtype)
    x = sd["synthesis.const"][None].expand(B, -1, -1, -1)
    img = None
    atts: List[torch.Tensor] = []
    li = ai = 0
    cen_prev = None
    for bi, res in enumerate([2 ** i for i in range(2, int(math.log2(resolution)) + 1)]):
        for j in range(1 if res == 4 else 2):
            pre = f"synthesis.layers.{li}"
            y, w_glob = ws_l[:, li, :k], ws_l[:, li, k]
            li += 1
            styles = _fc(w_glob, sd, pre + ".affine", D)
            x = _modconv(x, sd[pre + ".weight"], styles, up=2 if (res > 4 and j == 0) else 1, f=f)
            pos = None
            if (pre + ".attention.wq") in sd and g_start_res <= res <= g_end_res:
                w = {n[len(pre) + 11:]: t for n, t in sd.items() if n.startswith(pre + ".attention.")}
                cen_init = cen_prev if (iterative and duplex and cen_prev is not None and cen_prev.shape[2] == x.shape[1]) else None
                pos = lrelu_pos[ai] if lrelu_pos is not None else None
                ai += 1
                x, att, cen_prev = transformer_layer(x, y, w, integration=integration, norm=norm, duplex=duplex,
                                                     num_heads=num_heads, use_pos=use_pos, return_att=return_att,
                                                     kmeans_iters=kmeans_iters, img2ltnt=img2ltnt, centroids_init=cen_init)
                if att is not None:
                    atts.append(att)
            if noise_mode == "const":
                x = x + sd[pre + ".noise_const"] * sd[pre + ".noise_strength"]
            elif noise_mode != "none":
                raise ValueError("the oracle supports noise_mode 'const' or 'none' (random noise is not reproducible)")
            x = x + sd[pre + ".bias"][None, :, None, None]
            x = (F.leaky_relu(x, 0.2) if pos is None else torch.where(pos, x, 0.2 * x)) * SQRT2
        pre = f"synthesis.torgbs.{bi}"
        styles = _fc(ws_l[:, li, k], sd, pre + ".affine", D)          # the index after the block's last conv layer
        rgb = _modconv(x, sd[pre + ".weight"], styles, demodulate=False) + sd[pre + ".bias"][None, :, None, None]
        img = rgb if img is None else _upfirdn(img, f, up=2, pad=(2, 1, 2, 1), gain=4.0) + rgb
    if li + 1 != L:
        raise ValueError(f"ws_l has {L} latent sets, the network reads {li + 1}")
    return (img, atts) if return_att else img
