"""Style mixing on an H100 (``pytest -m gpu``; SURVEY A.4 item 13).

* The synthesis of mixed per-layer latents on the fused inference path, eager and replayed from a captured CUDA graph, against the
  fp64 per-layer restatement (tests/generator_style_mixing_ref.py) with the same latents: simplex, and duplex with the iterative
  carry, two k-means iterations and g_img2ltnt; exact fp32 and TF32 attention.  Bounds: tolerances.json "e2e".
* A mixed call runs the same library kernels as an unmixed one: the same launch count and the same kernel path.
* The gradients of a fixed-cutoff loss with respect to every mapping and synthesis parameter of an exact-fp32 64^2 generator
  against fp64.
* ``Trainer(style_mixing=0.9)``, eager and graphed: finite losses, and the cutoffs of every phase (StepStats.extra) vary from step
  to step, also between replays of one graph.
"""
import json
import math
import os
from importlib import import_module

import pytest
import torch

from tests import generator_path_length_ref as gref
from tests import generator_style_mixing_ref as sref

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
with open(os.path.join(os.path.dirname(__file__), "tolerances.json")) as _f:
    E2E = json.load(_f)["e2e"]
EXT = dict(kmeans=True, iterative=True, kmeans_iters=2, g_img2ltnt=True)
VARIANTS = {"simplex": {}, "duplex-ext": EXT}
TOL_GRAD = 3e-5           # relative error of each parameter's gradient, exact-fp32 generator against fp64


def _generator(gf, dev, exact, **kw):
    """64^2, K = 8, D = 32 with live biases and noise strengths (as the end-to-end parity tests build it)."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     exact_fp32=exact, **kw)
    with torch.no_grad():
        for n, prm in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo", "bq2", "bk2", "bv2"):
                prm.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                prm.fill_(0.1)
    return G.to(dev).eval()


def _mixed(G, dev, cutoff, B=3, seed=1):
    """Per-layer latents of two mapping draws switched at `cutoff`, and the first draw's latents."""
    tr = import_module(TRAIN)
    g = torch.Generator().manual_seed(seed)
    z1, z2 = (torch.randn(B, G.components_num + 1, G.latent_dim, generator=g).to(dev) for _ in range(2))
    with torch.no_grad():
        ws1, ws2 = G.mapping(z1), G.mapping(z2)
    return tr.mix_latents(ws1, ws2, torch.tensor(cutoff, device=dev), G.synthesis.num_ws), ws1


def check_image(img, ref64, mode, what, scale=1.0):
    """The end-to-end image bound of tests/test_gpu_parity.py: max-abs and RMS relative to the reference's peak, PSNR."""
    e2e = E2E["simt_fp32" if mode == "fp32" else "wgmma_tf32"]
    got, ref64 = img.detach().double().cpu(), ref64.detach().double().cpu()
    assert got.shape == ref64.shape and torch.isfinite(got).all()
    err = (got - ref64).abs()
    peak = max(1.0, ref64.abs().max().item())
    rmse = err.pow(2).mean().sqrt().item()
    rel_rms = rmse / ref64.pow(2).mean().sqrt().item()
    psnr = 20.0 * math.log10(peak / max(rmse, 1e-300))
    print(f"[style mixing] {what} mode={mode} max_abs/peak={err.max().item() / peak:.3e} rel_rms={rel_rms:.3e} psnr={psnr:.1f} dB")
    assert err.max().item() <= scale * e2e["max_abs_rel_peak"] * peak, what
    assert rel_rms <= scale * e2e["rel_rms"], what
    assert psnr >= e2e["psnr_db"] - 20.0 * math.log10(scale), what


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "tf32"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_mixed_image_against_fp64(gf, cuda_dev, variant, exact):
    kw = VARIANTS[variant]
    G = _generator(gf, cuda_dev, exact, **kw)
    ws_l, ws1 = _mixed(G, cuda_dev, cutoff=4)
    ws_l2, _ = _mixed(G, cuda_dev, cutoff=7, seed=2)
    with torch.no_grad():
        img, atts = G.synthesis(ws_l, return_att=True)
        img_fused = G.synthesis(ws_l).clone()                          # every fusion on
        img_plain = G.synthesis(ws1).clone()
        # captured as Generator.graphed captures G(z): warm-up on a side stream, then one graph replayed for new latents
        static_ws = ws_l.clone()
        side = torch.cuda.Stream(device=cuda_dev)
        side.wait_stream(torch.cuda.current_stream(cuda_dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                G.synthesis(static_ws)
        torch.cuda.current_stream(cuda_dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_img = G.synthesis(static_ws)
        graph.replay()
        img_graph = static_img.clone()
        static_ws.copy_(ws_l2)
        graph.replay()
        img_graph2 = static_img.clone()
    opts = dict(duplex=bool(kw), **(dict(kmeans_iters=2, img2ltnt=True, iterative=True) if kw else {}))
    sd = {n: t.detach().cpu().double() for n, t in G.state_dict().items()}
    ref, ratts = sref.synthesis_forward(sd, ws_l.double().cpu(), resolution=64, components_num=8, return_att=True, **opts)
    ref2 = sref.synthesis_forward(sd, ws_l2.double().cpu(), resolution=64, components_num=8, **opts)
    # duplex-ext: the k-means loop and the carried centroids amplify errors; the scales of test_generator_duplex_extensions_end_to_end
    sc = 1.0 if not kw else (3.0 if exact else 6.0)
    mode = "fp32" if exact else "tf32"
    for what, got, want in (("eager", img, ref), ("fused", img_fused, ref), ("graph", img_graph, ref), ("graph-replay-2", img_graph2, ref2)):
        check_image(got, want, mode, f"{variant}/{what}", scale=sc)
    for a, r in zip(atts, ratts):
        assert (a.double().cpu() - r).abs().max() <= sc * E2E["simt_fp32" if exact else "wgmma_tf32"]["att_abs"]
    assert len(atts) == len(ratts) == G.synthesis.num_attention_layers
    # the mixing is visible: the image of the first draw alone is far outside the bound
    d_plain = ((img_plain.cpu().double() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert d_plain > 5 * sc * E2E["wgmma_tf32"]["rel_rms"], d_plain


@pytest.mark.parametrize("variant", ["simplex", "duplex", "config2-256"])
def test_mixed_call_runs_the_same_kernels(gf, cuda_dev, variant):
    """Mixed and unmixed inference: the same number of library launches and the same kernel path (no extra kernel, no fallback)."""
    if variant == "config2-256":                                       # bench.py's generator: 256^2, K = 16, config-f channels
        torch.manual_seed(0)
        G = gf.Generator(resolution=256, components_num=16, latent_dim=32).to(cuda_dev).eval()
    else:
        G = _generator(gf, cuda_dev, False, **(dict(kmeans=True) if variant == "duplex" else {}))
    ws_l, ws1 = _mixed(G, cuda_dev, cutoff=5, B=2)
    counts, paths = {}, {}
    with torch.no_grad():
        for name, ws in (("plain", ws1), ("mixed", ws_l)) * 2:         # the first round warms up
            torch.cuda.synchronize()
            l0 = gf._lib.launch_count()
            G.synthesis(ws)
            torch.cuda.synchronize()
            counts[name] = gf._lib.launch_count() - l0
            paths[name] = (gf._lib.last_path(), gf._lib.last_centroid_path() if variant == "duplex" else None)
    print(f"[style mixing] {variant}: launches {counts} paths {paths}")
    assert counts["plain"] == counts["mixed"] > 0
    assert paths["plain"] == paths["mixed"]
    if variant == "config2-256":
        assert paths["mixed"][0] == "wgmma_tf32"


def test_mixed_gradients_against_fp64(gf, cuda_dev):
    """loss = <G.synthesis(mix(G.mapping(z1), G.mapping(z2), cutoff 5)), n>: its gradient of every parameter against fp64."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     exact_fp32=True).to(cuda_dev).train()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():                  # every term live: biases, noise strengths and attention biases away from zero
        for n, p in G.named_parameters():
            if n.endswith("noise_strength") or n.split(".")[-1].startswith("b"):
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
    B, cutoff, L = 4, 5, G.synthesis.num_ws
    g = torch.Generator().manual_seed(3)
    z1, z2 = (torch.randn(B, 9, 32, generator=g, dtype=torch.float64) for _ in range(2))
    noise = torch.randn(B, 3, 64, 64, generator=g, dtype=torch.float64) / 64.0
    params = dict(G.named_parameters())
    ws_l = tr.mix_latents(G.mapping(z1.float().to(cuda_dev)), G.mapping(z2.float().to(cuda_dev)),
                          torch.tensor(cutoff, device=cuda_dev), L)
    img, feats = G.synthesis(ws_l, noise_mode="const", return_features=True)
    got = torch.autograd.grad((img * noise.float().to(cuda_dev)).sum(), list(params.values()), allow_unused=True)
    # the slopes of the attention layers' leaky ReLUs from the GPU forward (see test_gpu_generator_path_length.py)
    signs = [f.detach().cpu() > 0 for f in feats]

    sd = {n: t.detach().cpu().double() for n, t in G.state_dict().items()}
    for n in params:
        if n.endswith("noise_strength"):   # one leaf per pixel and image, compared as a sum against the sum of its terms' magnitudes
            hw = G.get_buffer(n.replace("noise_strength", "noise_const")).shape
            sd[n] = sd[n].expand(B, 1, *hw).clone()
        sd[n].requires_grad_(True)
    with torch.enable_grad():
        ws64 = [gref.mapping_forward(sd, z, components_num=8, latent_dim=32, mapping_layers=4) for z in (z1, z2)]
        img64 = sref.synthesis_forward(sd, sref.mix_latents(ws64[0], ws64[1], cutoff, L), resolution=64, components_num=8,
                                       lrelu_pos=signs)
        ref = torch.autograd.grad((img64 * noise).sum(), [sd[n] for n in params], allow_unused=True)
    errs = {}
    scale = max(r.norm().item() for r in ref if r is not None)
    for n, r, t in zip(params, ref, got):
        if r is None:
            assert t is None or torch.count_nonzero(t) == 0, n
            continue
        if n.endswith("noise_strength"):
            errs[n] = abs(t.item() - r.sum().item()) / r.abs().sum().item()
        elif r.norm().item() < 1e-9 * scale:   # the attention key biases: constant over what the softmax normalises
            assert t.norm().item() < 1e-5 * scale, n
        else:
            errs[n] = ((t.double().cpu() - r).norm() / r.norm()).item()
    assert len(errs) >= len(params) - G.synthesis.num_attention_layers
    assert any(n.startswith("mapping.") for n in errs) and any(n.startswith("synthesis.torgbs.") for n in errs)
    worst = sorted(errs, key=errs.get, reverse=True)
    print(f"[style mixing gradients] {len(errs)} parameters, median {errs[worst[len(errs) // 2]]:.2e}, worst "
          + " ".join(f"{n}={errs[n]:.1e}" for n in worst[:8]))
    assert errs[worst[0]] < TOL_GRAD, worst[0]


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphed"])
@pytest.mark.parametrize("kw", [dict(att_dp=0.12), dict(kmeans=True)], ids=["simplex-dropout", "duplex"])
def test_trainer_style_mixing(gf, cuda_dev, kw, graphed):
    tr = import_module(TRAIN)
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, **kw).to(cuda_dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128).to(cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(d_reg_interval=2, style_mixing=0.9))
    g = torch.Generator().manual_seed(5)
    z = torch.randn(4, 9, 32, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(cuda_dev)
    am.set_dropout_seed(7, cuda_dev)
    w0 = {n: p.detach().clone() for n, p in G.named_parameters()}
    stats = [(trainer.step_graphed if graphed else trainer.step)(z, reals) for _ in range(6)]
    L = G.synthesis.num_ws
    for i, s in enumerate(stats):
        assert math.isfinite(s.loss_g) and math.isfinite(s.loss_d), (i, s)
        assert set(s.extra) == {"style_mixing_cutoff_d", "style_mixing_cutoff_g"}, s.extra
        assert all(1 <= v <= L and v == int(v) for v in s.extra.values()), s.extra
    cuts = [(s.extra["style_mixing_cutoff_d"], s.extra["style_mixing_cutoff_g"]) for s in stats]
    print(f"[style mixing trainer] {kw} graphed={graphed} cutoffs {cuts}")
    # steps 1, 3, 5 (no R1) replay one graph: each replay draws its own cutoffs
    assert len({c for i in (1, 3, 5) for c in cuts[i]}) > 1
    assert len({c for c in cuts}) > 1
    assert all((G.get_parameter(n) - w).abs().max() > 0 for n, w in w0.items() if n.startswith("mapping."))
    if graphed:
        assert set(k for k in trainer._graphs if isinstance(k, tuple)) == {(True, False), (False, False)}
