"""Image self-attention (img2img, SURVEY A.4 item 18) without a GPU: the oracle against the kernels' online softmax (restated in
oracle/self_attention_exact.py with its roundings off), the argument
checks of gf_self_attn_fwd / gf_self_attn_bwd through ctypes, and the construction of G and D with and without the layer."""
import json
import os
import subprocess
import sys
from importlib import import_module

import pytest
import torch

from oracle import self_attention as osa
from oracle import self_attention_exact as sx
from tests import img2img_ref as iref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN = "gansformer-reproducibility-challenge_b200.training"


@pytest.mark.parametrize("n,C", [(64, 32), (256, 128), (1024, 64)])
def test_oracle_against_online_softmax(n, C):
    g = torch.Generator().manual_seed(n)
    q, k, v = (torch.randn(2, n, C, generator=g, dtype=torch.float64) * 3 for _ in range(3))
    h = osa.heads_of(C)
    o, lse = osa.attention(q, k, v, h)
    o2, lse2 = sx.forward(q, k, v, h, rounded=False)              # the kernels' 64-key streaming in float64
    assert torch.allclose(o, o2, rtol=1e-12, atol=1e-12)
    assert torch.allclose(lse, lse2, rtol=1e-12, atol=1e-12)


def test_oracle_layer_is_the_product_composite(gf):
    """The product's composite route (CPU tensors run the torch ops the CUDA route recomputes in its backward) against the oracle."""
    sa = import_module("gansformer-reproducibility-challenge_b200.self_attention")
    ag = import_module("gansformer-reproducibility-challenge_b200.autograd")
    w = osa.init_params(64, 16, "both", seed=1, bias_std=0.3)
    x = torch.randn(2, 64, 8, 8, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    ref = osa.self_attention_layer(x, w, integration="both", norm="layer")
    X = x.reshape(2, 64, 64).transpose(1, 2)
    Pg = ag.grid_pos_table(8, 8, 16, x.device, x.dtype)
    Q = X @ ag._e(w["wq"]) + w["bq"] + Pg @ ag._e(w["wpq"])
    K = X @ ag._e(w["wk"]) + w["bk"] + Pg @ ag._e(w["wpk"])
    V = X @ ag._e(w["wv"]) + w["bv"]
    out = ag.integrate(X, sa.attention_composite(Q, K, V, 1) @ ag._e(w["wo"]) + w["bo"], "both", "layer")
    assert torch.allclose(out.transpose(1, 2).reshape(2, 64, 8, 8), ref, rtol=1e-12, atol=1e-12)


def test_layer_refuses_cpu_and_bad_widths(gf):
    m = gf.ImageSelfAttention(64, 16)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.zeros(1, 8, 8, 64))
    for C in (16, 48, 96, 100):
        with pytest.raises(ValueError, match="multiple of 64"):
            gf.ImageSelfAttention(C, 16)
    assert (gf.ImageSelfAttention(32, 16).heads, gf.ImageSelfAttention(512, 16).heads) == (1, 8)
    assert [n for n, _ in m.named_parameters()] == ["wq", "bq", "wk", "bk", "wv", "bv", "wo", "bo", "wpq", "wpk"]
    assert all(p.abs().sum() == 0 for n, p in m.named_parameters() if n.startswith("b"))


def test_construction_checks_resolution(gf):
    tr = import_module(TRAIN)
    kw = dict(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2)
    for r in (4, 12, 64, -8):
        with pytest.raises(ValueError, match="img2img"):
            gf.Generator(img2img=r, **kw)
        with pytest.raises(ValueError, match="img2img"):
            tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=r)
    for r in (8, 16, 32):
        gf.Generator(img2img=r, **kw)
        tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=r)


def test_state_dict_keys(gf):
    """img2img=0 builds exactly today's networks (same keys, same draws); img2img=r adds the layer's parameters only."""
    tr = import_module(TRAIN)
    kw = dict(resolution=32, components_num=4, latent_dim=16, fmap_base=1024, fmap_max=128, mapping_layers=2)
    torch.manual_seed(0)
    g0 = gf.Generator(**kw).state_dict()
    torch.manual_seed(0)
    g1 = gf.Generator(img2img=0, **kw).state_dict()
    assert list(g0) == list(g1) and all(torch.equal(g0[n], g1[n]) for n in g0)
    g2 = gf.Generator(img2img=16, **kw).state_dict()
    assert sorted(set(g2) - set(g0)) == sorted(f"synthesis.img2img.{n}" for n in ("wq", "bq", "wk", "bk", "wv", "bv", "wo", "bo", "wpq", "wpk"))
    assert set(g0) <= set(g2) and g2["synthesis.img2img.wq"].shape == (128, 128)
    for transformer in (False, True):
        dk = dict(fmap_base=1024, fmap_max=128, transformer=transformer, components_num=4, latent_dim=16)
        torch.manual_seed(0)
        d0 = tr.Discriminator(32, **dk).state_dict()
        torch.manual_seed(0)
        d1 = tr.Discriminator(32, img2img=0, **dk).state_dict()
        assert list(d0) == list(d1) and all(torch.equal(d0[n], d1[n]) for n in d0)
        d2 = tr.Discriminator(32, img2img=8, use_pos=False, **dk).state_dict()
        assert sorted(set(d2) - set(d0)) == sorted(f"img2img.{n}" for n in ("wq", "bq", "wk", "bk", "wv", "bv", "wo", "bo"))


def test_references_run_on_the_host(gf):
    """The tests-side references with an all-zero gain control reduce to the networks without the layer where that is exact."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    D = tr.Discriminator(32, fmap_base=1024, fmap_max=128, img2img=16, norm=None)
    sd = iref.cast(D.state_dict())
    sd["img2img.wo"].zero_()                                     # ctrl = 0: "mul" with no norm is the identity
    from oracle import discriminator as od
    x = torch.randn(2, 3, 32, 32, dtype=torch.float64)
    assert torch.allclose(iref.discriminator_forward(sd, x, img2img=16, norm=None), od.discriminator_forward(sd, x, norm=None),
                          rtol=1e-12, atol=1e-12)


_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A = 0x10000
out = []
def fwd(*a):
    out.append(["gf_self_attn_fwd", lib.gf_self_attn_fwd(*a), lib.gf_last_error().decode()])
def bwd(*a):
    out.append(["gf_self_attn_bwd", lib.gf_self_attn_bwd(*a), lib.gf_last_error().decode()])
P5 = [A] * 5
for sz in ([2, 256, 128, 64], [0, 256, 128, 64], [2, 256, 96, 64], [2, 256, 128, 128], [2, 96, 128, 64], [70000, 64, 64, 64],
           [1024, 4096, 1024, 64], [2, 256, 64, 16]):
    fwd(*P5, *sz, 0.125, None)
fwd(A, None, A, A, A, 2, 256, 128, 64, 0.125, None)
fwd(A, A, A + 4, A, A, 2, 256, 128, 64, 0.125, None)
fwd(*P5, 2, 256, 128, 64, 0.0, None)
P13 = [A] * 13
bwd(*P13, 2, 256, 128, 32, 0.125, None)
bwd(*P13[:9], None, *P13[10:], 2, 256, 128, 32, 0.125, None)
bwd(*P13, 2, 100, 128, 32, 0.125, None)
bwd(*P13, 2, 256, 100, 32, 0.125, None)
print(json.dumps(out))
"""


def test_entry_points_refuse_bad_arguments(gf):
    """Refusals come before the device is touched; a valid call reaches the launch, which fails without a GPU (-3)."""
    assert {"gf_self_attn_fwd", "gf_self_attn_bwd"} <= set(gf._lib.OPS_EXPORTS)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    assert [rc for _, rc, _ in out] == [-3, -1, -1, -2, -2, -2, -2, -2, -1, -1, -1, -3, -1, -2, -1], out
    assert all(name in msg for name, rc, msg in out if rc != -3)
    msgs = [msg for _, _, msg in out]
    assert "multiple of the head size" in msgs[2] and "d=128" in msgs[3] and "multiple of 64" in msgs[4] and "65535" in msgs[5]
    assert "int32" in msgs[6] and "(k)" in msgs[8] and "aligned" in msgs[9] and "scale" in msgs[10] and "(delta)" in msgs[12]
