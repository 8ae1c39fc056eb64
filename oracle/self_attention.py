"""CPU oracle of image self-attention (upstream GANsformer's ``img2img``; SURVEY A.4 item 18, [SPEC]).

TEST INFRASTRUCTURE ONLY.  ``transformer_layer(from = X, to = X)`` in the direct form: the bipartite layer of
``oracle.bipartite`` with the image itself as the key / value source, materialising the n x n probabilities.  Heads
h = max(1, C // 64) of d = C / h channels; the grid's positional table enters the queries and the keys when use_pos.
Runs in the dtype of its inputs (float64 = truth).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .bipartite import _dense, _split_heads, grid_pos_table, integrate

Tensor = torch.Tensor


def heads_of(C: int) -> int:
    return max(1, C // 64)


def init_params(C: int, pos_dim: int, integration: str = "mul", seed: int = 0, dtype=torch.float64, bias_std: float = 0.0,
                use_pos: bool = True) -> Dict[str, Tensor]:
    """N(0, 1) weights [fan_in, fan_out], biases N(0, bias_std), in the product's parameter order."""
    cout = 2 * C if integration == "both" else C
    shapes = {"wq": (C, C), "bq": (C,), "wk": (C, C), "bk": (C,), "wv": (C, C), "bv": (C,), "wo": (C, cout), "bo": (cout,)}
    if use_pos:
        shapes.update({"wpq": (pos_dim, C), "wpk": (pos_dim, C)})
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shp in shapes.items():
        t = torch.randn(shp, generator=g, dtype=torch.float64)
        out[name] = (t * bias_std if name.startswith("b") else t).to(dtype)
    return out


def attention(q: Tensor, k: Tensor, v: Tensor, heads: int):
    """The n x n part, direct: q, k, v [B,n,C] -> (concat_h(P_h V_h) [B,n,C], lse [B,h,n] = log2 sum_keys 2^(S log2 e)),
    S = Q_h K_h^T / sqrt(d), P_h = softmax over the keys of S."""
    B, n, C = q.shape
    S = (_split_heads(q, heads) @ _split_heads(k, heads).transpose(2, 3)) * (1.0 / math.sqrt(C / heads))   # [B,h,n,n]
    P = torch.softmax(S, dim=3)
    o = (P @ _split_heads(v, heads)).permute(0, 2, 1, 3).reshape(B, n, C)
    return o, torch.logsumexp(S, dim=3) / math.log(2.0)


def self_attention_layer(x_nchw: Tensor, w: Dict[str, Tensor], *, integration: str = "mul", norm: Optional[str] = "layer",
                         use_pos: bool = True) -> Tensor:
    """x [B,C,H,W] -> x' [B,C,H,W]."""
    B, C, H, W = x_nchw.shape
    X = x_nchw.reshape(B, C, H * W).permute(0, 2, 1)
    Q, K, V = _dense(X, w["wq"], w["bq"]), _dense(X, w["wk"], w["bk"]), _dense(X, w["wv"], w["bv"])
    if use_pos:
        Pg = grid_pos_table(H, W, w["wpq"].shape[0], x_nchw.dtype)
        Q = Q + _dense(Pg, w["wpq"])[None]
        K = K + _dense(Pg, w["wpk"])[None]
    ctrl, _ = attention(Q, K, V, heads_of(C))
    Xo = integrate(X, _dense(ctrl, w["wo"], w["bo"]), integration, norm)
    return Xo.permute(0, 2, 1).reshape(B, C, H, W)
