"""The exact cases and the TF32-faithful restatement of the image self-attention kernels, without a GPU (DESIGN 4.14).

* Every tied case of tests/test_gpu_img2img_exact.py is proved exact, element by element (oracle.self_attention_exact.prove_exact),
  and covers what it is there for: ties of 2^0 to 2^5 keys, alpha = 0 resets and alpha = 1 across tiles, and (with uniform rows)
  dS values whose RNE and truncation to TF32 differ.
* On those cases the restatement with its roundings equals the exact reference bit for bit; without its roundings it equals the
  float64 oracle, forward and backward.
"""
import pytest
import torch

from oracle import self_attention as osa
from oracle import self_attention_exact as sx
from tests.test_gpu_img2img_exact import TIED


@pytest.mark.parametrize("B,n,C,d", TIED)
def test_tied_case_is_exact(B, n, C, d):
    case = sx.tied_case(B, n, C, d, seed=B + n + C + d)
    st = sx.prove_exact(case)
    assert st["ties"] == [0, 1, 2, 3, 4, 5], st
    if n > 64:
        assert st["alpha_reset"] > 0 and st["alpha_one"] > 0, st
    assert st["ds_nonzero"] > 0, st
    if sx.uniform_rows_allowed(n) == "full":
        assert st["uniform"] > 0 and st["ds_rne_ne_trunc"] > 0, st


@pytest.mark.parametrize("B,n,C,d", [c for c in TIED if c[1] <= 1024])
def test_restatement_is_exact_on_tied_cases(B, n, C, d):
    case = sx.tied_case(B, n, C, d, seed=B + n + C + d)
    q, k, v, do, h = (case[x] for x in ("q", "k", "v", "do", "heads"))
    O, lse, _, dQ, dK, dV = sx.exact_reference(q, k, v, do, h)
    o, l = sx.forward(q, k, v, h)
    assert torch.equal(o.float(), O) and torch.equal(l.float(), lse)
    for a, b in zip(sx.backward(q, k, v, O, lse, do, h), (dQ, dK, dV)):
        assert torch.equal(a.float(), b)


@pytest.mark.parametrize("n,C", [(64, 32), (192, 64), (256, 128), (1024, 64)])
def test_restatement_without_roundings_is_the_oracle(n, C):
    g = torch.Generator().manual_seed(n + C)
    q, k, v, do = (torch.randn(2, n, C, generator=g, dtype=torch.float64) * 3 for _ in range(4))
    h = osa.heads_of(C)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    o, lse = osa.attention(*leaves, h)
    ref = torch.autograd.grad(o, leaves, do)
    o2, lse2 = sx.forward(q, k, v, h, rounded=False)
    assert torch.allclose(o2, o, rtol=1e-12, atol=1e-12) and torch.allclose(lse2, lse, rtol=1e-12, atol=1e-12)
    for a, r in zip(sx.backward(q, k, v, o2, lse2, do, h, rounded=False), ref):
        assert torch.allclose(a, r, rtol=1e-12, atol=1e-12)


def test_restatement_roundings():
    """The rounded restatement differs from the plain one by TF32-level amounts only, and its x is the kernels' fp32 product."""
    g = torch.Generator().manual_seed(5)
    q, k, v, do = (torch.randn(1, 128, 64, generator=g) for _ in range(4))
    o, lse = sx.forward(q, k, v, 1)
    o64, lse64 = sx.forward(q, k, v, 1, rounded=False)
    err = ((o - o64).abs().max() / o64.abs().max()).item()
    assert 1e-5 < err < 1e-2 and torch.equal(o, o.float().double())
    scale, sl2 = sx.kernel_scales(32)
    assert scale == float(torch.tensor(32.0 ** -0.5, dtype=torch.float32)) and sl2 != scale / 0.6931471805599453
