"""Bit-level TF32 conversions of float32 tensors, in torch (CPU or CUDA).

TF32 keeps the sign, the 8 exponent bits and the top 10 of float32's 23 mantissa bits.  The two conversions the library
relies on (DESIGN.md section 5):
  * ``tf32_trunc``: the tensor core reads a float32 operand straight from memory and ignores its low 13 mantissa bits, i.e.
    rounds toward zero.  The 3x3 convolution streams its activations this way.
  * ``tf32_rne``: round to nearest, ties to even, the same integer trick as ``round_tf32_rn`` in csrc/gf_tc_common.cuh.  The
    packed convolution weights and the attention tables are rounded this way before they reach the tensor core.
  * ``tf32_rna``: round to nearest, ties away from zero: what ``cvt.rna.tf32.f32`` (``cvt_tf32`` in the attention kernels) does
    to the probabilities before they become the second GEMM's operand.
Both work on the raw bits, so they are exact whatever the value; infinities and NaNs are outside their use here.
"""
from __future__ import annotations

import torch

_LOW13 = 0x1FFF
_KEEP = -0x2000                      # 0xFFFFE000 as a signed 32-bit value


def _bits(x: torch.Tensor) -> torch.Tensor:
    if x.dtype != torch.float32:
        raise TypeError(f"TF32 conversion takes float32 tensors, got {x.dtype}")
    return x.contiguous().view(torch.int32)


def tf32_trunc(x: torch.Tensor) -> torch.Tensor:
    """Clear the low 13 mantissa bits (round toward zero to TF32)."""
    return (_bits(x) & _KEEP).view(torch.float32).reshape(x.shape)


def tf32_rne(x: torch.Tensor) -> torch.Tensor:
    """Round to the nearest TF32 value, ties to even: add 0xFFF plus the lowest kept bit, then clear the low 13 bits.  A carry out
    of the mantissa moves into the exponent, which is the correct rounding.  The sum is formed in int64 so it cannot wrap."""
    b = _bits(x).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32).reshape(x.shape)


def tf32_rna(x: torch.Tensor) -> torch.Tensor:
    """Round to the nearest TF32 value, ties away from zero: add half a TF32 ulp (0x1000) to the magnitude bits, then clear the low
    13 bits.  The sign bit is untouched, so the rounding is symmetric about zero."""
    b = _bits(x).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0x1000) & 0xFFFFE000
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32).reshape(x.shape)


def tf32_low_bits(x: torch.Tensor) -> torch.Tensor:
    """The 13 mantissa bits TF32 drops (0 exactly when x is a TF32 value)."""
    return _bits(x) & _LOW13
