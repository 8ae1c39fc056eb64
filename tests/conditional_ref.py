"""fp64 restatement of the class-conditional generator and discriminator (SURVEY A.4 item 14), for
tests/test_host_cpu_conditional.py and tests/test_gpu_conditional.py.

Test infrastructure only, beside oracle/generator.py and oracle/discriminator.py, whose forwards are unconditional.  Built from the
oracle's own blocks, in the same order:
* the mapping concatenates e_b = c_b embed to every latent of image b before the pixel norm, so layer 0 of both MLPs has fan-in 2D;
  the rest (ltnt2ltnt, truncation with the one w_avg) is ``generator_forward``'s;
* the synthesis is tests/generator_style_mixing_ref.py's with every layer reading the same latents (``generator_forward``'s order);
* the discriminator is ``oracle.discriminator.discriminator_forward`` itself, run once per class with fc1 cut to that class's
  row; the labels weight the per-class logits (the projection).
The state dict, latents, images and labels are used as given (no detach, no cast), so fp64 leaves that require grad give gradients;
``cast`` prepares a product state dict for a plain forward.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle.bipartite import transformer_layer
from oracle import discriminator as od
from oracle.generator import _fc
from tests import generator_style_mixing_ref as sref


def cast(sd: Dict[str, torch.Tensor], dtype=torch.float64) -> Dict[str, torch.Tensor]:
    return {n: t.detach().to("cpu", dtype) if t.is_floating_point() else t.detach().cpu() for n, t in sd.items()}


def num_ws(resolution: int) -> int:
    return 2 * (int(math.log2(resolution)) - 2) + 2


def mapping_forward(sd, z, c: Optional[torch.Tensor], *, components_num: int, latent_dim: int, mapping_layers: int = 8,
                    truncation_psi: float = 1.0, integration="mul", norm="layer", num_heads: int = 1) -> torch.Tensor:
    """G_mapping with labels c [B, c_dim] (None: the unconditional mapping).  -> ws [B, k+1, D]."""
    k, D = components_num, latent_dim
    B = z.shape[0]
    if c is not None:
        e = c @ sd["mapping.embed"]
        z = torch.cat([z, e[:, None].expand(-1, k + 1, -1)], dim=2)
    z = z * torch.rsqrt(z.square().mean(dim=2, keepdim=True) + 1e-8)
    loc, glo = z[:, :k], z[:, k:]
    for i in range(mapping_layers):
        fan = z.shape[2] if i == 0 else D
        loc = _fc(loc, sd, f"mapping.local.{i}", fan, lr_mul=0.01, act="lrelu")
        glo = _fc(glo, sd, f"mapping.glob.{i}", fan, lr_mul=0.01, act="lrelu")
        pre = f"mapping.self_att.{i}."
        if (pre + "wq") in sd:
            w = {n[len(pre):]: t for n, t in sd.items() if n.startswith(pre)}
            xl, _, _ = transformer_layer(loc.transpose(1, 2).reshape(B, D, k, 1), loc, w, integration=integration, norm=norm,
                                         duplex=False, num_heads=num_heads, use_pos=False)
            loc = xl.reshape(B, D, k).transpose(1, 2)
    if truncation_psi != 1.0:
        loc = sd["mapping.w_avg"][0].lerp(loc, truncation_psi)
        glo = sd["mapping.w_avg"][1].lerp(glo, truncation_psi)
    return torch.cat([loc, glo], dim=1)


def generator_forward(sd, z, c, *, resolution: int, components_num: int, latent_dim: int, mapping_layers: int = 8,
                      truncation_psi: float = 1.0, return_att: bool = False, **synth):
    """img [B, 3, R, R] (, attention maps) of the conditional generator: ``synth`` takes the options of
    generator_style_mixing_ref.synthesis_forward (integration, norm, duplex, ...)."""
    ws = mapping_forward(sd, z, c, components_num=components_num, latent_dim=latent_dim, mapping_layers=mapping_layers,
                         truncation_psi=truncation_psi, integration=synth.get("integration", "mul"), norm=synth.get("norm", "layer"))
    ws_l = ws[:, None].expand(-1, num_ws(resolution), -1, -1)
    return sref.synthesis_forward(sd, ws_l, resolution=resolution, components_num=components_num, return_att=return_att, **synth)


def discriminator_forward(sd, img, c: Optional[torch.Tensor], *, mbstd_group: int = 4, integration: str = "mul",
                          norm: Optional[str] = "layer", use_pos: bool = True) -> torch.Tensor:
    """Logits [B] of the discriminator whose fc1 [c_dim, C] is projected onto c [B, c_dim] (None: the unconditional head).

    The projection is linear in fc1's rows: logit_b = sum_j c_bj (fc1_j . h_b + b_j).  So this runs oracle.discriminator_forward
    once per class, with fc1 cut to that class's row, and sums the per-class logits weighted by c: the whole trunk is the oracle's."""
    kw = dict(mbstd_group=mbstd_group, integration=integration, norm=norm, use_pos=use_pos)
    if c is None:
        return od.discriminator_forward(sd, img, **kw)
    logits = []
    for j in range(c.shape[1]):
        sd_j = dict(sd)
        sd_j["fc1.weight"], sd_j["fc1.bias"] = sd["fc1.weight"][j:j + 1], sd["fc1.bias"][j:j + 1]
        logits.append(od.discriminator_forward(sd_j, img, **kw))
    return (torch.stack(logits, dim=1) * c).sum(dim=1)
