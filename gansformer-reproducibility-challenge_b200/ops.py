"""Host wrappers of the memory-bound companion ops (include/gf_ops.h): the sm_90a equivalents of the
reference's native ops ``dnnlib/tflib/ops/upfirdn_2d.cu`` and ``fused_bias_act.cu`` (expected upstream; not in the
checkout) in the forms the generator uses, plus channel scaling (style modulation / demodulation).

Inference on CUDA fp32 tensors goes through libgf_attn.so.  The plain-torch forms below are the *definition* of each
op (and serve autograd / float64 / CPU plumbing tests of the surrounding host code -- none of this is the attention
hot path, which has no CPU form at all).
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional

import torch
import torch.nn.functional as F

from . import _lib

SQRT2 = math.sqrt(2.0)


def _use_cuda(*tensors) -> bool:
    ts = [t for t in tensors if t is not None]
    if not all(t.is_cuda and t.dtype == torch.float32 for t in ts):
        return False
    return not (torch.is_grad_enabled() and any(t.requires_grad for t in ts))


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def fir_filter(device=None, dtype=torch.float32) -> torch.Tensor:
    f = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64)
    f = torch.outer(f, f)
    return (f / f.sum()).to(device=device, dtype=dtype)


def upfirdn2d_ref(x: torch.Tensor, f: torch.Tensor, up: int = 1, pad=(0, 0, 0, 0), gain: float = 1.0) -> torch.Tensor:
    """Definition: zero-insert upsample by `up`, pad (x0, x1, y0, y1), correlate with the symmetric FIR filter `f`."""
    B, C, H, W = x.shape
    if up > 1:
        x = x.reshape(B, C, H, 1, W, 1)
        x = F.pad(x, [0, up - 1, 0, 0, 0, up - 1])
        x = x.reshape(B, C, H * up, W * up)
    x = F.pad(x, [pad[0], pad[1], pad[2], pad[3]])
    w = (f * gain).to(x.dtype)[None, None].expand(C, 1, *f.shape)
    return F.conv2d(x, w, groups=C)


def _nhwc_view(x: torch.Tensor) -> torch.Tensor:
    """NCHW-shaped tensor -> contiguous [B,H,W,C] view (free when x is channels_last)."""
    v = x.permute(0, 2, 3, 1)
    return v if v.is_contiguous() else v.contiguous()


def _aligned(t: torch.Tensor) -> torch.Tensor:
    """t as a contiguous tensor starting on a 16-byte boundary, as the float4 kernels of gf_ops.h require: a contiguous view
    that starts inside its storage (e.g. b[1:1 + C]) is copied."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _rows(s: torch.Tensor):
    """(tensor, row stride in floats) of a [B, C] matrix that may be a column slice of a wider contiguous matrix."""
    if s.dim() == 2 and s.stride(1) == 1 and s.stride(0) % 4 == 0 and s.data_ptr() % 16 == 0 and s.stride(0) >= s.shape[1]:
        return s, s.stride(0)
    s = _aligned(s)
    return s, s.shape[1]


def chan_scale(x: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """x [B,C,H,W] * s [B,C] (style modulation / demodulation as activation scaling)."""
    if _use_cuda(x, s) and x.shape[1] % 4 == 0:
        xv = _aligned(_nhwc_view(x))
        B, H, W, C = xv.shape
        y = torch.empty_like(xv)
        sr, ld = _rows(s)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_chan_scale_nhwc(xv.data_ptr(), sr.data_ptr(), ld, y.data_ptr(), B, H * W, C,
                                                      _stream(x.device)), "gf_chan_scale_nhwc")
        return y.permute(0, 3, 1, 2)
    return x * s[:, :, None, None].to(x.dtype)


class _Fir4(torch.autograd.Function):
    """Native [1,3,3,1]^2/64 FIR with symmetric padding (gf_fir4_nhwc), differentiable to any order: the filter is symmetric,
    so the gradient of a pad-p blur is the pad-(3-p) blur of the incoming gradient -- the same op again."""

    @staticmethod
    def forward(ctx, x, pad, gain):
        ctx.pad, ctx.gain = pad, gain
        xv = _aligned(_nhwc_view(x.detach()))
        B, H, W, C = xv.shape
        y = torch.empty((B, H + 2 * pad - 3, W + 2 * pad - 3, C), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_fir4_nhwc(xv.data_ptr(), y.data_ptr(), B, H, W, C, pad, ctypes.c_float(gain), _stream(x.device)),
                       "gf_fir4_nhwc")
        return y.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, gy):
        return _Fir4.apply(gy, 3 - ctx.pad, ctx.gain), None, None


def fir4(x: torch.Tensor, f: torch.Tensor, pad: int, gain: float = 1.0) -> torch.Tensor:
    """Stride-1 FIR blur with the [1,3,3,1] filter and symmetric padding `pad`: x [B,C,H,W] -> [B,C,H+2p-3,W+2p-3].
    CUDA fp32 tensors use the native kernel in both directions (autograd included); anything else the torch definition."""
    if x.is_cuda and x.dtype == torch.float32 and x.shape[1] % 4 == 0 and 0 <= pad <= 3 and min(x.shape[2:]) + 2 * pad > 3:
        return _Fir4.apply(x, int(pad), float(gain))
    return upfirdn2d_ref(x, f.to(x.dtype), pad=(pad, pad, pad, pad), gain=gain)


def blur_up(x: torch.Tensor, f: torch.Tensor, scale: Optional[torch.Tensor] = None, gain: float = 4.0) -> torch.Tensor:
    """FIR blur after a stride-2 transposed conv: x [B,C,2H+1,2W+1] -> [B,C,2H,2W] (pad 1), optional * scale [B,C]."""
    if _use_cuda(x, scale) and x.shape[1] % 4 == 0:
        xv = _aligned(_nhwc_view(x))
        B, Hin, Win, C = xv.shape
        y = torch.empty((B, Hin - 1, Win - 1, C), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_blur_up_nhwc(xv.data_ptr(), y.data_ptr(), None if scale is None else _aligned(scale).data_ptr(),
                                                   B, Hin - 1, Win - 1, C, float(gain), _stream(x.device)), "gf_blur_up_nhwc")
        return y.permute(0, 3, 1, 2)
    y = fir4(x, f, 1, gain=gain)                                        # training: native FIR both ways, scale in torch
    return y if scale is None else y * scale[:, :, None, None].to(y.dtype)


def upconv_phase_weights(w: torch.Tensor):
    """w [O,I,3,3] (already equalised-LR scaled) -> the four (kernel, padding) pairs whose stride-1 convolutions of the
    low-resolution input give the polyphase components T[2i+a, 2j+b] of conv_transpose2d(x, w^T, stride=2)."""
    out = []
    for a in (0, 1):
        for b in (0, 1):
            wy = w[:, :, 0::2].flip(2) if a == 0 else w[:, :, 1:2]        # taps (2, 0) / (1,) -- slices, no host index tensors
            wk = wy[:, :, :, 0::2].flip(3) if b == 0 else wy[:, :, :, 1:2]   # (capturable in a CUDA graph)
            out.append((wk.contiguous(memory_format=torch.channels_last), (1 - a, 1 - b)))
    return out


def upconv_blur_phases(x: torch.Tensor, phases, scale: Optional[torch.Tensor] = None, gain: float = 4.0) -> torch.Tensor:
    """Stride-2 transposed 3x3 convolution + FIR blur (+ demodulation scale) of the upsampling layers, inference on CUDA:
    four stride-1 convolutions (cuDNN fprop) feeding the polyphase blur kernel.  x [B,I,H,W] -> [B,O,2H,2W]."""
    ps = [_nhwc_view(F.conv2d(x, wk, padding=pad)) for wk, pad in phases]
    B, H, W, C = ps[3].shape
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().gf_blur_up_phases_nhwc(ps[0].data_ptr(), ps[1].data_ptr(), ps[2].data_ptr(), ps[3].data_ptr(), y.data_ptr(),
                                                      None if scale is None else _aligned(scale).data_ptr(), B, 2 * H, 2 * W, C,
                                                      float(gain), _stream(x.device)), "gf_blur_up_phases_nhwc")
    return y.permute(0, 3, 1, 2)


def upsample2x(x: torch.Tensor, f: torch.Tensor, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    """2x FIR upsampling of an NCHW image (tRGB skip connection), optionally + add."""
    if _use_cuda(x, add):
        xc = x.contiguous()
        B, C, H, W = xc.shape
        y = torch.empty((B, C, 2 * H, 2 * W), dtype=torch.float32, device=x.device)
        ac = None if add is None else add.contiguous()
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_upsample2x_nchw(xc.data_ptr(), None if ac is None else ac.data_ptr(), y.data_ptr(), B, C, H, W,
                                                      _stream(x.device)), "gf_upsample2x_nchw")
        return y
    y = upfirdn2d_ref(x, f, up=2, pad=(2, 1, 2, 1), gain=4.0)
    return y if add is None else y + add


def _bias_act_native(x, bias, act, noise, strength, gain):
    xv = _aligned(_nhwc_view(x))
    B, H, W, C = xv.shape
    y = torch.empty_like(xv)
    nz = None if noise is None else noise.contiguous()
    bstride = H * W if (nz is not None and nz.numel() == B * H * W and B > 1) else 0
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().gf_bias_act_nhwc(xv.data_ptr(), y.data_ptr(), None if bias is None else _aligned(bias).data_ptr(),
                                                None if nz is None else nz.data_ptr(),
                                                None if strength is None else strength.data_ptr(), bstride, B, H * W, C,
                                                1 if act == "lrelu" else 0, float(gain), _stream(x.device)), "gf_bias_act_nhwc")
    return y.permute(0, 3, 1, 2)


class _BiasAct(torch.autograd.Function):
    """Training form of bias_act on CUDA: native forward; backward = one masked scaling of the incoming gradient (the sign of
    the pre-activation is the sign of the output) plus the bias / noise-strength reductions -- instead of autograd through
    five separate elementwise ops with their saved tensors."""

    @staticmethod
    def forward(ctx, x, bias, noise, strength, act, gain):
        y = _bias_act_native(x.detach(), None if bias is None else bias.detach(), act, noise,
                             None if strength is None else strength.detach(), gain)
        ctx.act, ctx.gain = act, gain
        ctx.has_bias, ctx.has_strength = bias is not None, strength is not None and noise is not None
        ctx.save_for_backward(y, noise if noise is not None else y.new_empty(0))
        return y

    @staticmethod
    def backward(ctx, gy):
        y, noise = ctx.saved_tensors
        g = gy * ctx.gain if ctx.act != "lrelu" else gy * torch.where(y > 0, ctx.gain, 0.2 * ctx.gain)
        gb = g.sum(dim=(0, 2, 3)) if ctx.has_bias else None
        gs = None
        if ctx.has_strength:
            gs = (g.sum(dim=1, keepdim=True) * noise.reshape((-1, 1) + tuple(g.shape[2:]))).sum()
        return g, gb, None, gs, None, None


def bias_act(x: torch.Tensor, bias: Optional[torch.Tensor], act: str = "lrelu", noise: Optional[torch.Tensor] = None,
             strength: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act(x + noise * strength + bias[c]) * gain; x [B,C,H,W]; noise [H,W] (shared) or [B,1,H,W]; lrelu gain sqrt(2)."""
    gain = SQRT2 if act == "lrelu" else 1.0
    cuda32 = all(t is None or (t.is_cuda and t.dtype == torch.float32) for t in (x, bias, noise, strength))
    if cuda32 and x.shape[1] % 4 == 0 and torch.is_grad_enabled() and (noise is None or not noise.requires_grad) \
            and any(t is not None and t.requires_grad for t in (x, bias, strength)):
        return _BiasAct.apply(x, bias, noise, strength, act, gain)
    if _use_cuda(x, bias, noise, strength) and x.shape[1] % 4 == 0:
        xv = _aligned(_nhwc_view(x))
        B, H, W, C = xv.shape
        y = torch.empty_like(xv)
        nz = None if noise is None else noise.contiguous()
        bstride = H * W if (nz is not None and nz.numel() == B * H * W and B > 1) else 0
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_bias_act_nhwc(xv.data_ptr(), y.data_ptr(), None if bias is None else _aligned(bias).data_ptr(),
                                                    None if nz is None else nz.data_ptr(),
                                                    None if strength is None else strength.data_ptr(), bstride, B, H * W, C,
                                                    1 if act == "lrelu" else 0, float(gain), _stream(x.device)), "gf_bias_act_nhwc")
        return y.permute(0, 3, 1, 2)
    if noise is not None:
        x = x + noise.to(x.dtype) * (1.0 if strength is None else strength.to(x.dtype))
    if bias is not None:
        x = x + bias.to(x.dtype).reshape(1, -1, 1, 1)
    if act == "lrelu":
        x = F.leaky_relu(x, 0.2) * SQRT2
    return x


def demod_coef(styles: torch.Tensor, wsq: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """d[b,o] = rsqrt(sum_i styles[b,i]^2 wsq[o,i] + eps) (StyleGAN2 demodulation, activation-scaling form)."""
    if _use_cuda(styles, wsq):
        B, I = styles.shape
        O = wsq.shape[0]
        d = torch.empty((B, O), dtype=torch.float32, device=styles.device)
        sr, ld = _rows(styles)
        with torch.cuda.device(styles.device):
            _lib.check(_lib.load().gf_demod_coef(sr.data_ptr(), ld, wsq.contiguous().data_ptr(), d.data_ptr(), B, O, I,
                                                 float(eps), _stream(styles.device)), "gf_demod_coef")
        return d
    return torch.rsqrt(styles.square() @ wsq.t() + eps)


def demod_coef_batch(pairs, eps: float = 1e-8):
    """[(styles [B,I_l], wsq [O_l,I_l]), ...] -> [d_l [B,O_l], ...]: every layer's demodulation coefficients in one launch
    (gf_demod_coef_batch).  CUDA fp32 only; the per-layer call serves everything else."""
    if not pairs:
        return []
    if len(pairs) > _lib.DEMOD_MAX_JOBS or not all(_use_cuda(s_, w_) for s_, w_ in pairs):
        return [demod_coef(s_, w_, eps) for s_, w_ in pairs]
    dev = pairs[0][0].device
    B = pairs[0][0].shape[0]
    total = sum(w_.shape[0] for _, w_ in pairs)
    d_all = torch.empty((B * total,), dtype=torch.float32, device=dev)       # one allocation, one [B, O_l] block per layer
    jobs = (_lib.GfDemodJob * len(pairs))()
    outs, keep, off = [], [], 0
    for i, (s_, w_) in enumerate(pairs):
        if s_.shape[0] != B or s_.shape[1] != w_.shape[1]:
            raise ValueError("demod_coef_batch: styles [B, I] / wsq [O, I] mismatch")
        sr, ld = _rows(s_)
        wc = w_.contiguous()
        O, I = wc.shape
        d = d_all[off:off + B * O].view(B, O)
        off += B * O
        jobs[i].styles, jobs[i].wsq, jobs[i].d = sr.data_ptr(), wc.data_ptr(), d.data_ptr()
        jobs[i].s_ld, jobs[i].O, jobs[i].I = ld, O, I
        outs.append(d)
        keep += [sr, wc]
    with torch.cuda.device(dev):
        _lib.check(_lib.load().gf_demod_coef_batch(ctypes.cast(jobs, ctypes.c_void_p), len(pairs), B, float(eps), _stream(dev)),
                   "gf_demod_coef_batch")
    return outs


def torgb(x: torch.Tensor, weight: torch.Tensor, styles: torch.Tensor, bias: Optional[torch.Tensor],
          next_styles: Optional[torch.Tensor] = None):
    """tRGB: 1x1 modulated convolution without demodulation.  x [B,C,H,W], weight [3,C,1,1] (raw; equalised-LR scale
    1/sqrt(C) applied here), styles [B,C], bias [3] -> [B,3,H,W] (planar).  With next_styles [B,C] (inference on CUDA) the same
    read of x also produces x * next_styles (the next block's modulated input) and the call returns (rgb, x_scaled)."""
    O, I = weight.shape[:2]
    wscale = 1.0 / math.sqrt(I)
    if _use_cuda(x, weight, styles, bias, next_styles) and O == 3 and I % 4 == 0 and I <= 512:
        xv = _aligned(_nhwc_view(x))
        B, H, W, C = xv.shape
        y = torch.empty((B, O, H, W), device=x.device, dtype=torch.float32)
        sr, ld = _rows(styles)
        wv = _aligned(weight.reshape(O, I))
        xs = s2 = None
        ld2 = 0
        if next_styles is not None:
            s2, ld2 = _rows(next_styles)
            xs = torch.empty_like(xv)
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().gf_torgb_scale_nhwc(xv.data_ptr(), wv.data_ptr(), sr.data_ptr(), ld,
                                                       bias.data_ptr() if bias is not None else None, ctypes.c_float(wscale),
                                                       y.data_ptr(), None if s2 is None else s2.data_ptr(), ld2,
                                                       None if xs is None else xs.data_ptr(), B, H * W, C, _stream(x.device)),
                       "gf_torgb_scale_nhwc")
        return y if next_styles is None else (y, xs.permute(0, 3, 1, 2))
    wm = weight.reshape(1, O, I).to(x.dtype) * styles[:, None, :].to(x.dtype) * wscale           # [B, 3, C]
    B, C, H, W = x.shape
    xl = x.permute(0, 2, 3, 1).reshape(B, H * W, C)
    rgb = torch.matmul(xl, wm.transpose(1, 2))
    if bias is not None:
        rgb = rgb + bias.to(x.dtype)
    rgb = rgb.transpose(1, 2).reshape(B, O, H, W)
    return rgb if next_styles is None else (rgb, x * next_styles[:, :, None, None].to(x.dtype))


def mapping_fwd(z: torch.Tensor, w_eff: torch.Tensor, b_eff: torch.Tensor, w_avg: Optional[torch.Tensor], psi: float, k: int,
                c: Optional[torch.Tensor] = None, embed: Optional[torch.Tensor] = None, w0: Optional[torch.Tensor] = None) -> torch.Tensor:
    """G_mapping in one launch (gf_mapping_fwd): z [B, k+1, D]; w_eff [2, L, D, D] ([in, out], gains folded), b_eff [2, L, D];
    w_avg [2, D] (applied with psi when psi != 1).  CUDA fp32 inference only -- the module keeps the torch form for autograd.

    With labels c [B, c_dim] (gf_mapping_fwd_cond): embed [c_dim, D] is the label embedding, w0 [2, 2D, D] the effective layer 0
    and w_eff [2, L-1, D, D] the layers after it (L = b_eff.shape[1])."""
    B, kp1, D = z.shape
    out = torch.empty_like(z)
    wa = w_avg.contiguous() if (w_avg is not None and psi != 1.0) else None
    if c is not None:
        if embed is None or w0 is None:
            raise ValueError("mapping_fwd with labels needs the label embedding and the layer-0 weight w0")
        L = b_eff.shape[1]
        cc, ec = c.contiguous(), embed.contiguous()
        with torch.cuda.device(z.device):
            _lib.check(_lib.load().gf_mapping_fwd_cond(z.contiguous().data_ptr(), cc.data_ptr(), cc.shape[1], ec.data_ptr(), w0.data_ptr(),
                                                       w_eff.data_ptr() if L > 1 else None, b_eff.data_ptr(),
                                                       wa.data_ptr() if wa is not None else None, float(psi), out.data_ptr(), B, k, D, L,
                                                       _stream(z.device)), "gf_mapping_fwd_cond")
        return out
    L = w_eff.shape[1]
    with torch.cuda.device(z.device):
        _lib.check(_lib.load().gf_mapping_fwd(z.contiguous().data_ptr(), w_eff.data_ptr(), b_eff.data_ptr(), wa.data_ptr() if wa is not None else None,
                                              float(psi), out.data_ptr(), B, k, D, L, _stream(z.device)), "gf_mapping_fwd")
    return out


def _augment_args(x: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor], frac: Optional[torch.Tensor] = None):
    """Checks of ops.augment (the same refusals as gf_augment_nchw); returns geom as int32 [B, 4] and color as [B, 12] on x's device,
    and with ``frac`` given (geom, color, frac) with frac as float32 [B, 6] on x's device."""
    if frac is not None:
        geom, color = _augment_args(x, geom, color)
        B = x.shape[0]
        if frac.dim() < 2 or frac.shape[0] != B or tuple(frac.shape[1:]) not in ((6,), (2, 3)):
            raise ValueError(f"augment: frac must be [{B}, 6] or [{B}, 2, 3], got {tuple(frac.shape)}")
        return geom, color, frac.reshape(B, 6).to(device=x.device, dtype=torch.float32).contiguous()
    if x.dim() != 4:
        raise ValueError(f"augment: x must be [B, C, H, W], got {tuple(x.shape)}")
    B, C, H, W = x.shape
    if H < 2 or W < 2:
        raise ValueError(f"augment: H and W must be at least 2, got {H}x{W}")
    if tuple(geom.shape) != (B, 4):
        raise ValueError(f"augment: geom must be [{B}, 4], got {tuple(geom.shape)}")
    geom = geom.to(device=x.device, dtype=torch.int32).contiguous()
    if color is not None:
        if C != 3:
            raise ValueError(f"augment: a colour matrix needs C == 3, got C = {C}")
        if color.numel() != B * 12 or color.shape[0] != B:
            raise ValueError(f"augment: color must be [{B}, 12] or [{B}, 3, 4], got {tuple(color.shape)}")
        color = color.reshape(B, 12).to(device=x.device, dtype=torch.float32 if x.is_cuda and x.dtype == torch.float32 else x.dtype)
        color = color.contiguous()
    return geom, color


def augment_index(geom: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Definition of the blit: the flat source index sy * W + sx [B, H * W] of every output pixel, (sx, sy) = R(D_b(x, y) - t_b),
    with the parameter rules of gf_augment_nchw (code masked to 3 bits, bit 1 cleared when H != W, |t| clamped to N - 1)."""
    g = geom.to(torch.int64)
    code = g[:, 0] & 7
    if H != W:
        code = code & 5
    tx = g[:, 1].clamp(-(W - 1), W - 1)[:, None, None]
    ty = g[:, 2].clamp(-(H - 1), H - 1)[:, None, None]
    yy, xx = torch.meshgrid(torch.arange(H, device=geom.device), torch.arange(W, device=geom.device), indexing="ij")
    c = code[:, None, None]
    xx = torch.where((c & 1) == 1, W - 1 - xx[None], xx[None])
    yy = yy[None].expand_as(xx)
    k = c >> 1
    u = torch.where(k == 0, xx, torch.where(k == 1, yy, torch.where(k == 2, W - 1 - xx, H - 1 - yy)))
    v = torch.where(k == 0, yy, torch.where(k == 1, W - 1 - xx, torch.where(k == 2, H - 1 - yy, xx)))

    def mirror(i, N):
        return torch.where(i < 0, -i, torch.where(i >= N, 2 * (N - 1) - i, i))
    return (mirror(v - ty, H) * W + mirror(u - tx, W)).reshape(geom.shape[0], H * W)


def augment_ref(x: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor] = None,
                frac: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Definition of ops.augment: an index gather (the blit) -- or, with ``frac``, the band-limited resampler for every image whose
    fractional map is not the identity (resample_ref) -- then the colour matrix per pixel.  Any dtype and device; torch autograd
    differentiates it to any order."""
    if frac is not None:
        geom, color, frac = _augment_args(x, geom, color, frac)
    else:
        geom, color = _augment_args(x, geom, color)
    B, C, H, W = x.shape
    idx = augment_index(geom, H, W)
    y = x.reshape(B, C, H * W).gather(2, idx[:, None].expand(B, C, H * W)).reshape(B, C, H, W)
    if frac is not None:
        y = _frac_select(y, resample_ref(x, geom, frac), frac, H, W)
    if color is None:
        return y
    M = color.reshape(B, 3, 4).to(x.dtype)
    return torch.einsum("bij,bjhw->bihw", M[:, :, :3], y) + M[:, :, 3, None, None]


def augment_adjoint_ref(gy: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor] = None,
                        frac: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Definition of the adjoint of ops.augment's linear part: the transposed 3x3 colour matrix (no offset), then a scatter-add
    of every output pixel onto its source pixel (the blit), or with ``frac`` the adjoint of the resampler (torch autograd's
    vector-Jacobian product of resample_ref) for every image whose fractional map is not the identity."""
    if frac is not None:
        geom, color, frac = _augment_args(gy, geom, color, frac)
    else:
        geom, color = _augment_args(gy, geom, color)
    B, C, H, W = gy.shape
    if color is not None:
        gy = torch.einsum("bij,bihw->bjhw", color.reshape(B, 3, 4).to(gy.dtype)[:, :, :3], gy)
    idx = augment_index(geom, H, W)
    gx = gy.new_zeros(B, C, H * W).scatter_add(2, idx[:, None].expand(B, C, H * W), gy.reshape(B, C, H * W))
    gx = gx.reshape(B, C, H, W)
    if frac is not None:
        with torch.enable_grad():
            x0 = gy.new_zeros(gy.shape).requires_grad_(True)
            (gr,) = torch.autograd.grad(resample_ref(x0, geom, frac), x0, gy, create_graph=gy.requires_grad)
        gx = _frac_select(gx, gr, frac, H, W)
    return gx


# ------------------------------------------------------------------------------------------------ ADA's fractional geometry
# The 12 taps of the Daubechies symlet sym6: orthonormal under even shifts (sum sqrt 2), six vanishing moments.  ADA's geometric
# low-pass; the resampler uses it normalised to sum 1.
SYM6 = (0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
        0.787641141030194, 0.3379294217276218, -0.07263752278646252, -0.021060292512300564, 0.04472490177066578,
        0.0017677118642428036, -0.007800708325034148)
FRAC_SV_MAX = 16.0          # domain of a fractional map: singular values of its 2x2 part in [1/16, 16] ...
FRAC_T_MAX = 64             # ... and |translation| <= 64 * max(H, W) in each coordinate


def sym6_filter(device=None, dtype=torch.float64) -> torch.Tensor:
    f = torch.tensor(SYM6, dtype=torch.float64)
    return (f / f.sum()).to(device=device, dtype=dtype)


def frac_flags(frac: torch.Tensor, H: int, W: int):
    """(identity [B], in_domain [B]) of fractional maps [B, 6]: exactly [1, 0, 0; 0, 1, 0]; finite, both singular values of the 2x2
    part in [1/16, 16] and |translation| <= 64 * max(H, W) in each coordinate."""
    f = frac.reshape(-1, 6).double()
    ident = (f == f.new_tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0])).all(dim=1)
    a, b, c, d = f[:, 0], f[:, 1], f[:, 3], f[:, 4]
    s2 = a * a + b * b + c * c + d * d
    det = (a * d - b * c).abs()
    smax2 = (s2 + (s2 * s2 - 4 * det * det).clamp(min=0).sqrt()) / 2
    smin2 = det * det / smax2
    ok = (torch.isfinite(f).all(dim=1) & (smax2 <= FRAC_SV_MAX ** 2) & (smin2 >= FRAC_SV_MAX ** -2)
          & (f[:, [2, 5]].abs() <= FRAC_T_MAX * max(H, W)).all(dim=1))
    return ident, ok


def _frac_select(blit: torch.Tensor, res: torch.Tensor, frac: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Per image: the blit where the fractional map is the identity, else the resampled image, NaN outside the domain."""
    ident, ok = frac_flags(frac, H, W)
    ident, ok = ident.to(blit.device)[:, None, None, None], ok.to(blit.device)[:, None, None, None]
    return torch.where(ident, blit, torch.where(ok, res, torch.full_like(res, float("nan"))))


def resample_map(geom: torch.Tensor, frac: torch.Tensor, H: int, W: int, dtype=torch.float64):
    """(L [B, 2, 2], e [B, 2]): the point q = (qx, qy) of the 2x output grid (q = 1 .. 2N + 10 per axis; output pixel o sits at
    q = 2o + 6) reads the 2x source grid at nu = L q + e, nu = 2 * (source pixel index).  The composition of the fractional map
    F^-1 = frac[b] (centred pixel coordinates) and then the blit B^-1(v) = D v - t of geom[b] (code and t under gf_augment_nchw's
    rules)."""
    B = geom.shape[0]
    g = geom.to(torch.int64)
    code = g[:, 0] & 7
    if H != W:
        code = code & 5
    flip = (1 - 2 * (code & 1)).to(dtype)
    k = code >> 1
    cs = torch.where(k == 0, 1, torch.where(k == 2, -1, 0)).to(dtype)
    sn = torch.where(k == 1, 1, torch.where(k == 3, -1, 0)).to(dtype)
    D = torch.stack([torch.stack([cs * flip, sn], 1), torch.stack([-sn * flip, cs], 1)], 1)        # (u, v) = R_k (flip * x, y)
    t = torch.stack([g[:, 1].clamp(-(W - 1), W - 1), g[:, 2].clamp(-(H - 1), H - 1)], 1).to(dtype)
    A = frac.reshape(B, 2, 3).to(dtype=dtype, device=geom.device)
    L = D @ A[:, :, :2]
    cen = torch.tensor([(W - 1) / 2, (H - 1) / 2], dtype=dtype, device=geom.device)
    off = (D @ (A[:, :, 2] - A[:, :, :2] @ cen)[:, :, None])[:, :, 0] - t + cen
    return L, 2 * off - 6 * L.sum(dim=2)


def resample_ref(x: torch.Tensor, geom: torch.Tensor, frac: torch.Tensor, taps: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Definition of the resampler (SURVEY A.4 item 16), every image, in x's dtype: (1) mirror-extend the source by R_N to
    [-(N-1), 2(N-1)] per axis, zeros beyond; (2) upsample 2x with the normalised sym6 taps as a convolution, gain 2 per axis, pads
    (6, 5); (3) sample that grid bilinearly, zeros outside it, at nu = L q + e (resample_map) for the (2N + 10)^2 points of the 2x output
    grid that (4) the 2x downsampling reads: the same taps as a correlation, pads (-1, -1).  ``taps`` replaces the 12 taps (the
    tests' magnitude companion runs |taps|)."""
    B, C, H, W = x.shape
    dev, dt = x.device, x.dtype
    f = sym6_filter(dev, dt) if taps is None else taps.to(device=dev, dtype=dt)
    fl = f.flip(0)

    def mirror(N):
        i = torch.arange(-(N - 1), 2 * N - 1, device=dev)
        return torch.where(i < 0, -i, torch.where(i >= N, 2 * (N - 1) - i, i))
    E = x[:, :, mirror(H)][:, :, :, mirror(W)].reshape(B * C, 1, 3 * H - 2, 3 * W - 2)
    Z = E.new_zeros(B * C, 1, 6 * H - 4, 6 * W - 4)
    Z[:, :, ::2, ::2] = E
    Z = F.pad(Z, [6, 5, 6, 5])
    U = F.conv2d(F.conv2d(Z, 2 * fl.reshape(1, 1, 1, 12)), 2 * fl.reshape(1, 1, 12, 1))       # [B*C, 1, 6H-4, 6W-4]
    UH, UW = 6 * H - 4, 6 * W - 4
    ok = frac_flags(frac, H, W)[1].to(frac.device)[:, None]                                     # outside the domain: any finite map
    frac = torch.where(ok, frac.reshape(B, 6), frac.new_tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0]))
    L, e = resample_map(geom.to(dev), frac, H, W, dt)
    qx = torch.arange(1, 2 * W + 11, device=dev, dtype=dt)[None, None, :]
    qy = torch.arange(1, 2 * H + 11, device=dev, dtype=dt)[None, :, None]
    bl = lambda v: v[:, None, None]
    nx = bl(L[:, 0, 0]) * qx + bl(L[:, 0, 1]) * qy + bl(e[:, 0]) + 2 * (W - 1)                      # index into U
    ny = bl(L[:, 1, 0]) * qx + bl(L[:, 1, 1]) * qy + bl(e[:, 1]) + 2 * (H - 1)
    x0, y0 = nx.floor(), ny.floor()
    ax, ay = nx - x0, ny - y0
    Uf = U.reshape(B, C, UH * UW)
    V = 0
    for dy, wy in ((0, 1 - ay), (1, ay)):
        for dx, wx in ((0, 1 - ax), (1, ax)):
            ix, iy = x0 + dx, y0 + dy
            inside = (ix >= 0) & (ix < UW) & (iy >= 0) & (iy < UH)
            idx = (iy.clamp(0, UH - 1) * UW + ix.clamp(0, UW - 1)).long().reshape(B, 1, -1).expand(B, C, -1)
            w = torch.where(inside, wx * wy, torch.zeros_like(wx)).reshape(B, 1, -1)
            V = V + w * Uf.gather(2, idx)
    V = V.reshape(B * C, 1, 2 * H + 10, 2 * W + 10)
    y = F.conv2d(F.conv2d(V, f.reshape(1, 1, 1, 12), stride=(1, 2)), f.reshape(1, 1, 12, 1), stride=(2, 1))
    return y.reshape(B, C, H, W)


def _augment_native(name: str, x: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor]) -> torch.Tensor:
    xc = x.detach().contiguous()
    B, C, H, W = xc.shape
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        _lib.check(getattr(_lib.load(), name)(xc.data_ptr(), y.data_ptr(), geom.data_ptr(), None if color is None else color.data_ptr(),
                                              B, C, H, W, _stream(x.device)), name)
    return y


def _linear_part(color: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """The colour matrices [B, 12] with their offset column zeroed: the linear part of the map, whose derivative it is."""
    if color is None:
        return None
    return torch.cat([color.reshape(-1, 3, 4)[:, :, :3], color.new_zeros(color.shape[0], 3, 1)], dim=2).reshape(-1, 12)


class _Augment(torch.autograd.Function):
    """gf_augment_nchw, differentiable to any order: the map is linear apart from the colour offset, so its gradient is the adjoint
    (_AugmentAdjoint), whose gradient is the linear part of the map again."""

    @staticmethod
    def forward(ctx, x, geom, color):
        ctx.save_for_backward(geom, color)
        return _augment_native("gf_augment_nchw", x, geom, color)

    @staticmethod
    def backward(ctx, gy):
        geom, color = ctx.saved_tensors
        return _AugmentAdjoint.apply(gy, geom, color), None, None


class _AugmentAdjoint(torch.autograd.Function):
    """gf_augment_adjoint_nchw: gx = A^T gy (the offset does not take part)."""

    @staticmethod
    def forward(ctx, gy, geom, color):
        ctx.save_for_backward(geom, color)
        return _augment_native("gf_augment_adjoint_nchw", gy, geom, color)

    @staticmethod
    def backward(ctx, ggx):
        geom, color = ctx.saved_tensors
        return _Augment.apply(ggx, geom, _linear_part(color)), None, None


def _augment_resample_native(name: str, x: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor],
                             frac: torch.Tensor) -> torch.Tensor:
    xc = x.detach().contiguous()
    B, C, H, W = xc.shape
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        _lib.check(getattr(_lib.load(), name)(xc.data_ptr(), y.data_ptr(), geom.data_ptr(), frac.data_ptr(),
                                              None if color is None else color.data_ptr(), B, C, H, W, _stream(x.device)), name)
    return y


class _AugmentResample(torch.autograd.Function):
    """gf_augment_resample_nchw, differentiable to any order like _Augment: its gradient is _AugmentResampleAdjoint, whose gradient
    is the linear part of the map again."""

    @staticmethod
    def forward(ctx, x, geom, color, frac):
        ctx.save_for_backward(geom, color, frac)
        return _augment_resample_native("gf_augment_resample_nchw", x, geom, color, frac)

    @staticmethod
    def backward(ctx, gy):
        geom, color, frac = ctx.saved_tensors
        return _AugmentResampleAdjoint.apply(gy, geom, color, frac), None, None, None


class _AugmentResampleAdjoint(torch.autograd.Function):
    """gf_augment_resample_adjoint_nchw: gx = A^T gy (the offset does not take part)."""

    @staticmethod
    def forward(ctx, gy, geom, color, frac):
        ctx.save_for_backward(geom, color, frac)
        return _augment_resample_native("gf_augment_resample_adjoint_nchw", gy, geom, color, frac)

    @staticmethod
    def backward(ctx, ggx):
        geom, color, frac = ctx.saved_tensors
        return _AugmentResample.apply(ggx, geom, _linear_part(color), frac), None, None, None


def augment(x: torch.Tensor, geom: torch.Tensor, color: Optional[torch.Tensor] = None,
            frac: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Adaptive discriminator augmentation of a batch (SURVEY A.4 items 15, 16): x [B, C, H, W] -> the same shape, image b blitted by
    its geom[b] = (dihedral code, tx, ty, unused) and, with color [B, 12] (row-major 3x4 matrices on (r, g, b, 1), C == 3), recoloured.
    With frac [B, 6] (row-major 2x3 inverse maps F_b^-1 in centred pixel coordinates) every image whose F_b^-1 is not exactly the
    identity is resampled through the composition of F_b^-1 and its blit instead (ADA's general geometry, band-limited).
    See include/gf_ops.h for the exact map.  CUDA fp32 tensors run gf_augment_nchw (gf_augment_resample_nchw with frac), and its
    adjoint in the backward (to any order); anything else runs the definition augment_ref."""
    if frac is not None:
        geom, color, frac = _augment_args(x, geom, color, frac)
        if x.is_cuda and x.dtype == torch.float32:
            return _AugmentResample.apply(x, geom, color, frac)
        return augment_ref(x, geom, color, frac)
    geom, color = _augment_args(x, geom, color)
    if x.is_cuda and x.dtype == torch.float32:
        return _Augment.apply(x, geom, color)
    return augment_ref(x, geom, color)


def conv3x3_pack(weight: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """weight [O, I, 3, 3] -> the tap-major, TF32-rounded [9, O, I] layout gf_conv3x3_nhwc_tf32 consumes (gf_conv3x3_pack_weights)."""
    O, I = weight.shape[:2]
    wt = torch.empty((9, O, I), dtype=torch.float32, device=weight.device)
    with torch.cuda.device(weight.device):
        _lib.check(_lib.load().gf_conv3x3_pack_weights(weight.detach().contiguous().data_ptr(), wt.data_ptr(), O, I, ctypes.c_float(scale),
                                                       _stream(weight.device)), "gf_conv3x3_pack_weights")
    return wt


def conv3x3_native(x: torch.Tensor, wt: torch.Tensor) -> torch.Tensor:
    """3x3 stride-1 zero-padded convolution on the wgmma implicit-GEMM kernel (row f1, TF32): x [B, I, H, W] (channels-last
    storage), wt from conv3x3_pack -> [B, O, H, W] (channels-last storage).  CUDA fp32 inference only."""
    xv = _nhwc_view(x)
    B, H, W, I = xv.shape
    O = wt.shape[1]
    y = torch.empty((B, H, W, O), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().gf_conv3x3_nhwc_tf32(xv.data_ptr(), wt.data_ptr(), y.data_ptr(), B, H, W, I, O, _stream(x.device)),
                   "gf_conv3x3_nhwc_tf32")
    return y.permute(0, 3, 1, 2)


def upconv_blur_native(x: torch.Tensor, wt: torch.Tensor, scale: torch.Tensor, gain: float = 4.0) -> torch.Tensor:
    """Stride-2 transposed 3x3 convolution + FIR blur + demodulation (scale [B, O]) of the upsampling layers in ONE wgmma kernel
    (row f1, TF32): x [B, I, H, W] (channels-last storage), wt = conv3x3_pack of the un-transposed w [O, I, 3, 3] -> [B, O, 2H, 2W]
    (channels-last storage).  Same result as upconv_blur_phases up to TF32 rounding.  CUDA fp32 inference only."""
    xv = _nhwc_view(x)
    B, H, W, I = xv.shape
    O = wt.shape[1]
    y = torch.empty((B, 2 * H, 2 * W, O), dtype=torch.float32, device=x.device)
    sc = scale.contiguous()
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().gf_upconv3x3_blur_nhwc_tf32(xv.data_ptr(), wt.data_ptr(), sc.data_ptr(), y.data_ptr(),
                                                           B, H, W, I, O, ctypes.c_float(gain), _stream(x.device)), "gf_upconv3x3_blur_nhwc_tf32")
    return y.permute(0, 3, 1, 2)
