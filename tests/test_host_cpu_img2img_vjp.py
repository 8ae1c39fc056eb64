"""The image self-attention double backward without a GPU: the fp64 restatement of gf_self_attn_bwd_vjp's algebra
(oracle/self_attention_vjp.py) against torch's double autograd, the entry point's argument checks through ctypes, and the options
that put the R1 and path-length passes of the img2img layer on it."""
import json
import os
import subprocess
import sys
from importlib import import_module

import pytest
import torch

from oracle import self_attention_vjp as ov

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = "gansformer-reproducibility-challenge_b200.training"


@pytest.mark.parametrize("h", [1, 4])
@pytest.mark.parametrize("n,d", [(37, 8), (64, 16)])
def test_restatement_is_the_double_autograd(n, d, h):
    g = torch.Generator().manual_seed(n + d + h)
    q, k, v, do, a, bk, cv = (torch.randn(2, n, h * d, generator=g, dtype=torch.float64) for _ in range(7))
    got = ov.vjp(q, k, v, do, a, bk, cv, h)
    want = ov.vjp_autograd(q, k, v, do, a, bk, cv, h)
    for name, x, y in zip(("gQ", "gK", "gV", "gdO"), got, want):
        assert torch.allclose(x, y, rtol=1e-12, atol=1e-12), (name, (x - y).abs().max().item())


_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A = 0x10000
out = []
def vjp(*a):
    out.append(["gf_self_attn_bwd_vjp", lib.gf_self_attn_bwd_vjp(*a), lib.gf_last_error().decode()])
P = [A] * 22
vjp(*P, 2, 256, 128, 64, 0.125, None)                  # valid: reaches the launch
vjp(*P[:10], None, *P[11:], 2, 256, 128, 64, 0.125, None)
vjp(*P[:16], A + 4, *P[17:], 2, 256, 128, 64, 0.125, None)
vjp(*P, 2, 256, 128, 128, 0.125, None)
vjp(*P, 2, 256, 128, 16, 0.125, None)
vjp(*P, 2, 96, 128, 64, 0.125, None)
vjp(*P, 70000, 64, 64, 64, 0.125, None)
vjp(*P, 2, 256, 128, 64, 0.0, None)
vjp(*P, 2, 256, 128, 64, float("inf"), None)
vjp(*P, 2, 256, 96, 64, 0.125, None)
print(json.dumps(out))
"""


def test_entry_point_refuses_bad_arguments(gf):
    """Refusals come before the device is touched; a valid call reaches the launch, which fails without a GPU (-3)."""
    assert "gf_self_attn_bwd_vjp" in gf._lib.OPS_EXPORTS
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    assert [rc for _, rc, _ in out] == [-3, -1, -1, -2, -2, -2, -2, -1, -1, -1], out
    assert all(name in msg for name, rc, msg in out if rc != -3)
    msgs = [msg for _, _, msg in out]
    assert "(a)" in msgs[1] and "row_r" in msgs[2] and "aligned" in msgs[2] and "d=128" in msgs[3] and "d=16" in msgs[4]
    assert "multiple of 64" in msgs[5] and "65535" in msgs[6] and "scale" in msgs[7] and "scale" in msgs[8]
    assert "multiple of the head size" in msgs[9]


def test_options_set_the_flag(gf):
    """r1_kernels and pl_kernels reach the img2img layer; the defaults leave it off, with today's state_dict keys."""
    tr = import_module(TRAIN)
    gkw = dict(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2, img2img=16)
    dkw = dict(fmap_base=1024, fmap_max=128, img2img=16)
    torch.manual_seed(0)
    g0 = gf.Generator(**gkw)
    torch.manual_seed(0)
    g1 = gf.Generator(pl_kernels=True, **gkw)
    assert not g0.synthesis.img2img.kernel_double_backward and g1.synthesis.img2img.kernel_double_backward
    s0, s1 = g0.state_dict(), g1.state_dict()
    assert list(s0) == list(s1) and all(torch.equal(s0[n], s1[n]) for n in s0)
    assert not gf.ImageSelfAttention.kernel_double_backward
    gf.Generator(pl_kernels=True, **{**gkw, "img2img": 0})          # no img2img layer: nothing to set
    for transformer in (False, True):
        torch.manual_seed(0)
        d0 = tr.Discriminator(32, transformer=transformer, components_num=4, latent_dim=16, **dkw)
        torch.manual_seed(0)
        d1 = tr.Discriminator(32, transformer=transformer, components_num=4, latent_dim=16, r1_kernels=True, **dkw)
        assert not d0.img2img.kernel_double_backward and d1.img2img.kernel_double_backward
        s0, s1 = d0.state_dict(), d1.state_dict()
        assert list(s0) == list(s1) and all(torch.equal(s0[n], s1[n]) for n in s0)
