"""The image self-attention kernels on an H100, exactly (``pytest -m gpu``; DESIGN 4.14).

gf_self_attn_fwd and gf_self_attn_bwd through the C ABI, every output (O, lse, the Delta scratch, dQ, dK, dV) between NaN guards,
checked for writes outside it and for elements left unwritten.  The transposed copies are made as the wrappers make them.
* Tied cases (oracle/self_attention_exact.py: tied_case, proved exact by tests/test_host_cpu_img2img_exact.py): every logit is
  1024 or 0, ties of 2^k winning keys spread over the key tiles, and uniform rows where they are exact.  O, lse, Delta, dQ, dK and
  dV equal the float64 definition with dS rounded to fp32 and then TF32 (RNE), bit for bit.  Here dS, dQ and dK are not zero, and
  where uniform rows exist the TF32 rounding of dS changes values, so RNE and truncation give different bits.
* N(0, 1) inputs against the TF32-faithful restatement of the kernels (run in float64 on the device): max error over max reference
  for O, dQ, dK and dV, absolute error for lse, under bounds frozen from a logged run.
"""
import math

import pytest
import torch

from oracle import self_attention_exact as sx
from tests.guards import Guarded, assert_exact
from tests.test_gpu_ops_exact import _call, _stream

pytestmark = pytest.mark.gpu

# Worst cases over test_against_restatement, measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (1980 MHz maximum SM
# clock): O 1.03e-4, lse 1.91e-6 (absolute), dQ 2.73e-4, dK 2.08e-4, dV 2.40e-4; frozen at about 3x.  They are set by the TF32
# rounding of P and dS, not by fp32 accumulation: see DESIGN 4.14.
RESTATED_BOUNDS = {"O": 3e-4, "lse": 6e-6, "dQ": 8e-4, "dK": 6e-4, "dV": 7e-4}


def run(gf, q, k, v, do, heads, dev):
    """Both entry points on fp32 [B,n,C] inputs; -> dict of fp32 outputs (CUDA), every guard and every element checked."""
    B, n, C = q.shape
    d = C // heads
    scale = 1.0 / math.sqrt(d)
    q, k, v, do = (t.float().contiguous().to(dev) for t in (q, k, v, do))
    vt, qt, kt, dot = (t.transpose(1, 2).contiguous() for t in (v, q, k, do))
    out = {"O": Guarded((B, n, C), dev), "lse": Guarded((B, heads, n), dev), "Delta": Guarded((B, heads, n), dev),
           "dQ": Guarded((B, n, C), dev), "dK": Guarded((B, n, C), dev), "dV": Guarded((B, n, C), dev)}
    o, lse = out["O"], out["lse"]
    _call(gf, "gf_self_attn_fwd", q.data_ptr(), k.data_ptr(), vt.data_ptr(), o.ptr(), lse.ptr(), B, n, C, d, scale, _stream(dev))
    o.check("O")
    lse.check("lse")
    _call(gf, "gf_self_attn_bwd", q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), o.ptr(), lse.ptr(),
          do.data_ptr(), dot.data_ptr(), out["Delta"].ptr(), out["dQ"].ptr(), out["dK"].ptr(), out["dV"].ptr(), B, n, C, d, scale,
          _stream(dev))
    return {name: g.check(name) for name, g in out.items()}


# (B, n, C, d): 1 to 64 tiles, odd tile counts (3 and 9: the forward's last CTA has one warpgroup), the wrap of every ring, h = 1
# to 8, both head sizes, and a batch beyond the grid's first wave
TIED = [(2, 64, 64, 64), (3, 192, 128, 32), (2, 256, 512, 64), (2, 576, 64, 64), (1, 1024, 32, 32), (1, 4096, 64, 64),
        (1, 4096, 128, 32), (130, 64, 64, 64)]


@pytest.mark.parametrize("B,n,C,d", TIED)
def test_tied_cases_exact(gf, cuda_dev, B, n, C, d):
    case = sx.tied_case(B, n, C, d, seed=B + n + C + d)
    q, k, v, do, h = (case[x] for x in ("q", "k", "v", "do", "heads"))
    got = run(gf, q, k, v, do, h, cuda_dev)
    want = sx.exact_reference(*(t.to(cuda_dev) for t in (q, k, v, do)), h)
    for name, w in zip(("O", "lse", "Delta", "dQ", "dK", "dV"), want):
        assert_exact(got[name], w, f"{name} (B={B} n={n} C={C} d={d})")
    assert (got["dQ"] != 0).any() and (got["dK"] != 0).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("h", [1, 4])
@pytest.mark.parametrize("d", [32, 64])
@pytest.mark.parametrize("n", [64, 192, 256, 1024, 4096])
def test_against_restatement(gf, cuda_dev, n, d, h, B):
    """The kernels against their own roundings restated in float64: what is left is fp32 accumulation order, exp2f / log2f
    against the correctly rounded functions, and the rare TF32 rounding of P or dS that those move across a midpoint."""
    g = torch.Generator().manual_seed(7 * n + d + 3 * h + B)
    q, k, v, do = (torch.randn(B, n, h * d, generator=g).to(cuda_dev) for _ in range(4))
    got = run(gf, q, k, v, do, h, cuda_dev)
    o, lse = sx.forward(q, k, v, h)
    grads = sx.backward(q, k, v, got["O"], got["lse"], do, h)
    rel = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    errs = {"O": rel(got["O"], o), "lse": (got["lse"].double() - lse).abs().max().item()}
    errs.update({name: rel(got[name], r) for name, r in zip(("dQ", "dK", "dV"), grads)})
    print(f"[img2img restated] n={n} d={d} h={h} B={B} " + " ".join(f"{k_}={v_:.3e}" for k_, v_ in errs.items()))
    assert all(errs[x] <= RESTATED_BOUNDS[x] for x in errs), errs
