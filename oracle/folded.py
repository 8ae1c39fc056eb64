"""Folded restatement of the bipartite attention block -- the algebra the CUDA path executes.

TEST INFRASTRUCTURE ONLY (see oracle/bipartite.py header; parity unpinned).

``oracle/bipartite.py`` is the direct op order (what the reference's graph runs).  This file is the
three-stage *folded* form of SURVEY.md A.2/A.3 -- exact in real arithmetic, different rounding:

  stage W  fold_weights():   weights only            -> small matrices (once per weight update)
  stage I  prologue():       per image, from Y/Xbar  -> Kp [B,KP,C], Vt [B,Cout,KP], Rt [B,H,KP], Ct [B,W,KP]
  stage T  per_token():      one read of x, one write of x'

The CUDA library (gansformer-reproducibility-challenge_b200/csrc) implements exactly these three
stages with exactly these buffer layouts; ``tests/test_folded_algebra.py`` proves stage W+I+T equals
the direct oracle in float64, so a CUDA-vs-direct-oracle mismatch can only come from the kernels.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .bipartite import LN_EPS, sinusoidal_axis

Tensor = torch.Tensor


def _e(w: Tensor) -> Tensor:
    """equalised-LR effective weight"""
    return w * (1.0 / math.sqrt(w.shape[0]))


def pad_k(k: int) -> int:
    return 16 if k <= 16 else 32


def fold_weights(w: Dict[str, Tensor], *, C: int, k: int, integration: str, duplex: bool,
                 use_pos: bool = True, num_heads: int = 1) -> Dict[str, Tensor]:
    """Stage W.  Column layout of the key-side matrices: [K' (C) | kappa_p (p) | kappa_0 (1) | pad (3)]."""
    assert num_heads == 1
    p = w["pos_latent"].shape[1]
    s = 1.0 / math.sqrt(C)
    dt = w["wq"].dtype
    wq, wpq = _e(w["wq"]), _e(w["wpq"])
    # query-side fold target: Q-space vector t  ->  [t Wq^T s | t Wpq^T s | t.bq s | 0 0 0]
    qfold = torch.cat([wq.t() * s,
                       (wpq.t() * s) if use_pos else torch.zeros(C, p, dtype=dt),
                       (w["bq"] * s)[:, None],
                       torch.zeros(C, 3, dtype=dt)], dim=1)            # [C, C+p+4]
    kconst = w["bk"][None, :].expand(k, C)
    if use_pos:
        kconst = kconst + w["pos_latent"] @ _e(w["wpk"])                # [k, C]
    out = {}
    if duplex:
        akcen = _e(w["wkc"]) @ qfold                                    # centroid -> key -> folded
        out["AK"] = akcen                                               # [C, C+p+4], applied to Cen
        out["CK"] = kconst @ qfold                                      # [k, C+p+4]
        out["WV2"] = _e(w["wv2"])                                       # Cen = Xbar @ WV2 + bv2
        out["BV2"] = w["bv2"]
        s2 = 1.0 / math.sqrt(C)
        wk2, wpk2 = _e(w["wk2"]), _e(w["wpk2"])
        m_fold = torch.cat([wk2.t() * s2,
                            (wpk2.t() * s2) if use_pos else torch.zeros(C, p, dtype=dt),
                            torch.zeros(C, 4, dtype=dt)], dim=1)        # bk2 term is constant over n: dropped
        qconst = w["bq2"][None, :].expand(k, C)
        if use_pos:
            qconst = qconst + w["pos_latent"] @ _e(w["wpq2"])
        out["AM"] = _e(w["wq2"]) @ m_fold                               # [D, C+p+4]
        out["CM"] = qconst @ m_fold                                     # [k, C+p+4]
    else:
        out["AK"] = _e(w["wk"]) @ qfold                                 # [D, C+p+4]
        out["CK"] = kconst @ qfold
    wo = _e(w["wo"])
    out["AV"] = _e(w["wv"]) @ wo                                        # [D, Cout]
    cv = w["bv"] @ wo + w["bo"]
    if integration in ("mul", "both"):
        cv = cv.clone()
        cv[:C] += 1.0                                                   # the "1 +" of x*(1+gain)
    out["CV"] = cv                                                      # [Cout]
    return out


def _pos_tables(kp_all: Tensor, C: int, p: int, H: int, W: int, KP: int, use_pos: bool):
    """kp_all [B,k,C+p+4] -> Rt [B,H,KP], Ct [B,W,KP] (kappa_0 folded into Rt, padded latents = -inf)."""
    B, k, _ = kp_all.shape
    dt = kp_all.dtype
    kap0 = kp_all[:, :, C + p]                                          # [B,k]
    Rt = torch.full((B, H, KP), -math.inf, dtype=dt)
    Ct = torch.zeros((B, W, KP), dtype=dt)
    if use_pos:
        half = p // 2
        row = sinusoidal_axis(H, half, dt)
        col = sinusoidal_axis(W, half, dt)
        kap = kp_all[:, :, C:C + p]
        Rt[:, :, :k] = torch.einsum("hp,bjp->bhj", row, kap[:, :, :half]) + kap0[:, None, :]
        Ct[:, :, :k] = torch.einsum("wp,bjp->bwj", col, kap[:, :, half:])
    else:
        Rt[:, :, :k] = kap0[:, None, :].expand(B, H, k)
    return Rt, Ct


def prologue(y: Tensor, f: Dict[str, Tensor], *, C: int, H: int, W: int, p: int, use_pos: bool = True,
             key_source: Optional[Tensor] = None):
    """Stage I.  key_source = centroids [B,k,C] for duplex pass B, else the latents y."""
    B, k, _ = y.shape
    KP = pad_k(k)
    z = y if key_source is None else key_source
    kp_all = z @ f["AK"] + f["CK"][None]                                # [B,k,C+p+4]
    Kp = torch.zeros(B, KP, C, dtype=y.dtype)
    Kp[:, :k] = kp_all[:, :, :C]
    Rt, Ct = _pos_tables(kp_all, C, p, H, W, KP, use_pos)
    v = y @ f["AV"] + f["CV"][None, None]                               # [B,k,Cout]
    Vt = torch.zeros(B, v.shape[2], KP, dtype=y.dtype)
    Vt[:, :, :k] = v.transpose(1, 2)
    return Kp, Vt, Rt, Ct


def per_token(X: Tensor, Kp: Tensor, Vt: Tensor, Rt: Tensor, Ct: Tensor, *, H: int, W: int,
              integration: str, norm: Optional[str], return_att: bool = False, k: Optional[int] = None,
              att_mult: Optional[Tensor] = None, cb: Optional[Tensor] = None, retain: Optional[dict] = None):
    """Stage T.  X [B,n,C] channels-last tokens.

    att_mult [B,n,KP] (or [B,n,k]) and cb [Cout] (attention dropout, the form the kernels use): q = p * mult weights the
    values, and the constants cb (bo, +1 on the gain half) that dropout leaves unscaled are re-added,
    ctl = sum_j q_j (Vt_j - cb) + cb.  retain (a dict) receives the logits "S", the probabilities "P", the dropped
    probabilities "Q" and the control signal "ctl", so that a caller can take gradients with respect to them."""
    B, n, C = X.shape
    S = X @ Kp.transpose(1, 2)                                          # [B,n,KP]
    S = S + (Rt[:, :, None, :] + Ct[:, None, :, :]).reshape(B, n, -1)
    P = torch.softmax(S, dim=2)
    if att_mult is None:
        Q = P
        GB = P @ Vt.transpose(1, 2)                                     # [B,n,Cout]
    else:
        mult = att_mult.to(P.dtype)
        if mult.shape[2] < P.shape[2]:                                  # the padded latents have p = 0: any multiplier
            mult = torch.nn.functional.pad(mult, (0, P.shape[2] - mult.shape[2]), value=1.0)
        Q = P * mult
        GB = Q @ (Vt - cb[None, :, None]).transpose(1, 2) + cb
    if retain is not None:
        retain.update(S=S, P=P, Q=Q, ctl=GB)
    if norm == "layer":
        mu = X.mean(dim=2, keepdim=True)
        var = ((X - mu) ** 2).mean(dim=2, keepdim=True)
        Xn = (X - mu) / torch.sqrt(var + LN_EPS)
    elif norm in (None, "none"):
        Xn = X
    else:
        dims = {"instance": (1,), "batch": (0, 1)}[norm]
        mu = X.mean(dim=dims, keepdim=True)
        var = ((X - mu) ** 2).mean(dim=dims, keepdim=True)
        Xn = (X - mu) / torch.sqrt(var + LN_EPS)
    if integration == "mul":
        out = Xn * GB
    elif integration == "add":
        out = Xn + GB
    else:
        out = Xn * GB[..., :C] + GB[..., C:]
    att = P[:, :, :k] if return_att else None
    return out, att


def centroid_pass(X: Tensor, y: Tensor, f: Dict[str, Tensor], *, H: int, W: int, p: int, use_pos: bool = True):
    """Duplex pass A folded: stream X once, softmax over n, Xbar = A X, Cen = Xbar Wv2 + bv2."""
    B, n, C = X.shape
    k = y.shape[1]
    KP = pad_k(k)
    m_all = y @ f["AM"] + f["CM"][None]                                 # [B,k,C+p+4]
    M = m_all[:, :, :C]
    Rt, Ct = _pos_tables(m_all, C, p, H, W, KP, use_pos)
    _, xbar, _ = centroid_softmax(X, M, Rt, Ct, k=k)
    cen = xbar @ f["WV2"] + f["BV2"]
    return cen, xbar


def centroid_softmax(X: Tensor, M: Tensor, Rt2: Tensor, Ct2: Tensor, *, k: Optional[int] = None,
                     retain: Optional[dict] = None):
    """Pass A on its tables (the layout of gf_attn_centroid_stats): the logit of token (h, w) for latent j is
    x.M_j + Rt2[h,j] + Ct2[w,j]; the softmax runs over the n tokens.  Only the first k latents are used (default: all rows
    of M; the padded ones have Rt2 = -inf).  Returns A [B,n,k], Xbar = A^T X [B,k,C] and lse [B,k], the log of each
    latent's softmax denominator.  retain (a dict) receives the logits "L"."""
    B, n, C = X.shape
    k = M.shape[1] if k is None else k
    L = X @ M[:, :k].transpose(1, 2) + (Rt2[:, :, None, :k] + Ct2[:, None, :, :k]).reshape(B, n, k)   # [B,n,k]
    A = torch.softmax(L, dim=1)                                         # over n
    xbar = A.transpose(1, 2) @ X                                        # [B,k,C]
    if retain is not None:
        retain.update(L=L)
    return A, xbar, torch.logsumexp(L, dim=1)


def transformer_layer_folded(x_nhwc: Tensor, y: Tensor, w: Dict[str, Tensor], *, integration="mul", norm="layer",
                             duplex=False, use_pos=True, return_att=False, centroids_in=None):
    """Channels-last end-to-end folded path (what BipartiteAttention.forward does on the GPU)."""
    B, H, W, C = x_nhwc.shape
    k = y.shape[1]
    p = w["pos_latent"].shape[1]
    f = fold_weights(w, C=C, k=k, integration=integration, duplex=duplex, use_pos=use_pos)
    X = x_nhwc.reshape(B, H * W, C)
    cen = None
    if duplex:
        cen = centroids_in if centroids_in is not None else centroid_pass(X, y, f, H=H, W=W, p=p, use_pos=use_pos)[0]
    Kp, Vt, Rt, Ct = prologue(y, f, C=C, H=H, W=W, p=p, use_pos=use_pos, key_source=cen)
    out, att = per_token(X, Kp, Vt, Rt, Ct, H=H, W=W, integration=integration, norm=norm,
                         return_att=return_att, k=k)
    if att is not None:
        att = att.permute(0, 2, 1).reshape(B, k, H, W)
    return out.reshape(B, H, W, C), att, cen
