"""GPU tests of stage T's launch configuration (run on an H100: ``pytest -m gpu``).

``token_tc_kernel`` runs with one or two CTAs per SM, chosen from the shape (C, KP, integration) by the library's schedule
rule.  The per-tile arithmetic does not depend on it, so the rule must not change a bit of the output: every case here runs the
same layer under schedule rule 1 (one CTA per SM with the deepest ring, the configuration before the rule existed) and under the
library's rule 0, and the attention output, the attention map and the fused tRGB planes must be ``torch.equal``.  The batches
give more tiles than two per SM, not a multiple of the CTA count, so every CTA walks a contiguous tile range that crosses images.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

D = 32


def _lib(gf):
    return gf._lib.load()


def schedule(gf, desc, rule):
    """{two_pass, ctas, stages, grid} of the layer under `rule`, which then serves this thread's following stage-T launches."""
    out = (ctypes.c_int * 4)()
    gf._lib.check(_lib(gf).gf_attn_debug_tc_schedule(ctypes.byref(desc), rule, out, 4), "gf_attn_debug_tc_schedule")
    return dict(zip(("two_pass", "ctas", "stages", "grid"), (int(v) for v in out)))


@pytest.fixture
def rule_reset(gf):
    yield
    schedule(gf, gf._lib.make_desc(1, 16, 16, 64, 16, D), 0)


def _batch(sms, n):
    tpi = max(1, n // 128)
    B = (2 * sms + 5) // tpi + 1                  # more tiles than two CTAs per SM can take in one round, not a multiple of it
    assert B * tpi > 2 * sms and (B * tpi) % (2 * sms) != 0
    return B


def run_both_rules(gf, dev, attn, x, y, post_fn, desc, training=False):
    """The layer's outputs under rule 1 and rule 0 (same inputs, same weights, same dropout state)."""
    res, scheds = [], []
    attn.train(training)
    for rule in (1, 0):
        scheds.append(schedule(gf, desc, rule))
        post = post_fn()
        o = torch.full_like(x, float("nan"))
        with torch.no_grad():
            _, att, _ = attn(x, y, out=o, postop=post, return_att=True, need_centroids=False)
        torch.cuda.synchronize()
        assert gf._lib.last_path() == "wgmma_tf32"
        res.append({"Xout": o, "att": att, **({"rgb": post["rgb_out"]} if post and "rgb_out" in post else {})})
    return res, scheds


def _postop(B, H, W, C, dev, g, rgb=True):
    def make():
        p = dict(bias=torch.randn(C, generator=g).to(dev), noise=torch.randn(B, 1, H, W, generator=g).to(dev),
                 strength=torch.tensor(0.1).to(dev), act="lrelu", gain=2 ** 0.5,
                 in_scale=(torch.rand(B, C, generator=g) + 0.5).to(dev), post_scale=(torch.rand(B, C, generator=g) + 0.5).to(dev))
        if rgb:
            p.update(rgb_w=torch.randn(B, 3, C, generator=g).to(dev), rgb_bias=torch.randn(3, generator=g).to(dev),
                     rgb_out=torch.full((B, 3, H, W), float("nan"), device=dev))
        return p
    return make


def check_equal(a, b):
    assert a.keys() == b.keys()
    for name in a:
        if a[name] is None:
            assert b[name] is None
            continue
        assert torch.isfinite(a[name]).all(), name
        assert torch.equal(a[name], b[name]), f"{name}: max |diff| {(a[name] - b[name]).abs().max().item()}"


# (C, k, integration): every NS of the single-pass kernel, KP 16 and 32, the three integrations
SHAPES = [(64, 16, "mul"), (64, 27, "both"), (128, 16, "mul"), (128, 16, "both"), (128, 16, "add"), (128, 27, "mul"), (128, 27, "add"),
          (256, 16, "mul"), (256, 27, "add")]


@pytest.mark.parametrize("C,k,integration", SHAPES, ids=str)
def test_schedules_equal_with_postop_and_trgb(gf, cuda_dev, rule_reset, C, k, integration):
    """The generator's fused post-op (demodulation scales, noise, bias, leaky-ReLU, next style) and tRGB under both rules."""
    H = W = 32
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    B = _batch(sms, H * W)
    g = torch.Generator().manual_seed(C * 100 + k)
    torch.manual_seed(C + k)
    attn = gf.BipartiteAttention(C, D, k, integration=integration).to(cuda_dev)
    x = torch.randn(B, H, W, C, generator=g).to(cuda_dev)
    y = torch.randn(B, k, D, generator=g).to(cuda_dev)
    desc = gf._lib.make_desc(B, H, W, C, k, D, integration=integration)
    post_seed = C * 7 + k

    def post():
        return _postop(B, H, W, C, cuda_dev, torch.Generator().manual_seed(post_seed))()
    (r1, r0), (s1, s0) = run_both_rules(gf, cuda_dev, attn, x, y, post, desc)
    check_equal(r1, r0)
    assert s1["ctas"] == 1 and s0["grid"] <= s0["ctas"] * sms
    if C <= 128 and (k <= 16 or integration != "both"):
        assert s0["ctas"] == 2, s0                # an H100 holds two of these CTAs per SM
    if C == 256:
        assert s0 == s1                           # a whole C = 256 tile does not fit in half an SM: unchanged


@pytest.mark.parametrize("case", ["duplex", "dropout", "heads"])
def test_schedules_equal_duplex_dropout_heads(gf, cuda_dev, rule_reset, case):
    """Duplex attention (stage T behind the centroid pass), attention dropout in training mode and multi-head segments."""
    C, k, H, W = 128, 16, 32, 32
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    B = _batch(sms, H * W)
    g = torch.Generator().manual_seed(7)
    torch.manual_seed(11)
    kw = dict(duplex={"kmeans": True}, dropout={"att_dp": 0.12}, heads={"num_heads": 2})[case]
    attn = gf.BipartiteAttention(C, D, k, **kw).to(cuda_dev)
    x = torch.randn(B, H, W, C, generator=g).to(cuda_dev)
    y = torch.randn(B, k, D, generator=g).to(cuda_dev)
    desc = gf._lib.make_desc(B, H, W, C, k, D)
    (r1, r0), (_, s0) = run_both_rules(gf, cuda_dev, attn, x, y, lambda: None, desc, training=case == "dropout")
    check_equal(r1, r0)
    assert s0["ctas"] == 2, s0


def test_schedule_respects_ring_cap(gf, cuda_dev, rule_reset, monkeypatch):
    """GF_TC_MAX_STAGES still caps the per-CTA ring of the two-CTA launch (down to one tile, no prefetch)."""
    C, k, H, W = 128, 16, 32, 32
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    desc = gf._lib.make_desc(_batch(sms, H * W), H, W, C, k, D)
    assert schedule(gf, desc, 0)["stages"] > C // 32
    monkeypatch.setenv("GF_TC_MAX_STAGES", str(C // 32))
    s = schedule(gf, desc, 0)
    assert s["ctas"] == 2 and s["stages"] == C // 32
