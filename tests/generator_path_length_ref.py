"""Differentiable fp64 restatement of the generator from its dlatents, for the gradients of the path-length penalty
(tests/test_gpu_generator_path_length.py).

Test infrastructure only, beside oracle/generator.py, whose ``generator_forward`` detaches its inputs: these two entries use the
state dict and the latents as given, so fp64 leaves that require grad give the penalty's gradient of every generator weight, and
the synthesis takes per-layer attention-dropout multipliers (oracle/philox.py).  They reuse the oracle's own building blocks
(fully connected layer, reference-style modulated convolution, FIR, ``oracle.bipartite.transformer_layer``).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle.bipartite import transformer_layer
from oracle.generator import SQRT2, _fc, _fir, _modconv, _upfirdn




def mapping_forward(sd: Dict[str, torch.Tensor], z: torch.Tensor, *, components_num: int, latent_dim: int,
                    mapping_layers: int = 8) -> torch.Tensor:
    """G_mapping of ``generator_forward`` (without ltnt2ltnt and truncation), differentiable: ``sd`` and ``z`` are used as given
    (no detach, no cast), so fp64 leaves that require grad give the gradients of every mapping weight.  -> ws [B, k+1, D]."""
    k, D = components_num, latent_dim
    z = z * torch.rsqrt(z.square().mean(dim=2, keepdim=True) + 1e-8)
    loc, glo = z[:, :k], z[:, k:]
    for i in range(mapping_layers):
        loc = _fc(loc, sd, f"mapping.local.{i}", D, lr_mul=0.01, act="lrelu")
        glo = _fc(glo, sd, f"mapping.glob.{i}", D, lr_mul=0.01, act="lrelu")
    return torch.cat([loc, glo], dim=1)


def synthesis_forward(sd: Dict[str, torch.Tensor], ws: torch.Tensor, *, resolution: int, components_num: int,
                      integration="mul", norm="layer", duplex=False, use_pos=True, num_heads=1, g_start_res: int = 8,
                      g_end_res: Optional[int] = None, noise_mode: str = "const", img2ltnt: bool = False,
                      att_mults: Optional[List[Optional[torch.Tensor]]] = None,
                      lrelu_pos: Optional[List[Optional[torch.Tensor]]] = None) -> torch.Tensor:
    """G_synthesis of ``generator_forward`` from the dlatents ws [B, k+1, D], differentiable (``sd`` and ``ws`` used as given), for
    the path-length penalty's gradients.  att_mults: per attention layer (in order), the attention-dropout multipliers [B, H*W, k]
    (oracle/philox.py) or None -- the training-mode forward of a generator with att_dp > 0.  One k-means iteration, no carried
    centroids.  lrelu_pos: per attention layer (in order), a boolean [B, C, H, W] choosing the slope of the layer's leaky ReLU (1 where
    True, 0.2 elsewhere) instead of the sign of the fp64 pre-activation: the branch another evaluation took, so that both compare
    derivatives of the same piece of a function that is not differentiable at its kinks.  -> img [B, 3, R, R]."""
    k = components_num
    g_end_res = resolution if g_end_res is None else g_end_res
    B = ws.shape[0]
    y, w_glob = ws[:, :k], ws[:, k]
    f = _fir(ws.dtype)
    x = sd["synthesis.const"][None].expand(B, -1, -1, -1)
    img = None
    li = ai = 0
    for bi, res in enumerate([2 ** i for i in range(2, int(math.log2(resolution)) + 1)]):
        for j in range(1 if res == 4 else 2):
            pre = f"synthesis.layers.{li}"
            li += 1
            D = ws.shape[2]
            styles = _fc(w_glob, sd, pre + ".affine", D)
            x = _modconv(x, sd[pre + ".weight"], styles, up=2 if (res > 4 and j == 0) else 1, f=f)
            pos = None
            if (pre + ".attention.wq") in sd and g_start_res <= res <= g_end_res:
                w = {n[len(pre) + 11:]: t for n, t in sd.items() if n.startswith(pre + ".attention.")}
                mult = att_mults[ai] if att_mults is not None else None
                pos = lrelu_pos[ai] if lrelu_pos is not None else None
                ai += 1
                x, _, _ = transformer_layer(x, y, w, integration=integration, norm=norm, duplex=duplex, num_heads=num_heads,
                                            use_pos=use_pos, img2ltnt=img2ltnt, att_mult=mult)
            if noise_mode == "const":
                x = x + sd[pre + ".noise_const"] * sd[pre + ".noise_strength"]
            elif noise_mode != "none":
                raise ValueError("the oracle supports noise_mode 'const' or 'none' (random noise is not reproducible)")
            x = x + sd[pre + ".bias"][None, :, None, None]
            x = (F.leaky_relu(x, 0.2) if pos is None else torch.where(pos, x, 0.2 * x)) * SQRT2
        pre = f"synthesis.torgbs.{bi}"
        styles = _fc(w_glob, sd, pre + ".affine", ws.shape[2])
        rgb = _modconv(x, sd[pre + ".weight"], styles, demodulate=False) + sd[pre + ".bias"][None, :, None, None]
        img = rgb if img is None else _upfirdn(img, f, up=2, pad=(2, 1, 2, 1), gain=4.0) + rgb
    return img
