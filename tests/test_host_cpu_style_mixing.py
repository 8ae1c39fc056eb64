"""Style mixing on the CPU (SURVEY A.4 item 13): the synthesis network's per-layer latents checked with the attention swapped for
the oracle, the fp64 per-layer restatement against the oracle generator, the cutoff sampler, and the training step's plumbing."""
from importlib import import_module

import pytest
import torch

from oracle import bipartite as ob
from oracle import generator as og
from tests import generator_path_length_ref as gref
from tests import generator_style_mixing_ref as sref

NETS = "gansformer-reproducibility-challenge_b200.networks"
TRAIN = "gansformer-reproducibility-challenge_b200.training"
EXT = dict(iterative=True, kmeans_iters=2, g_img2ltnt=True)
L32 = 8                           # 32^2: conv layers 0 | 1 2 | 3 4 | 5 6 and the last tRGB
TRGB_INDEX = [1, 3, 5, 7]         # the tRGB of each block reads the index after its last conv layer


def _small_generator(gf, **kw):
    torch.manual_seed(0)
    G = gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=512, fmap_max=64, mapping_layers=2,
                     integration="both", **kw)
    with torch.no_grad():
        for n, p in G.named_parameters():
            if n.endswith("bias") or n.endswith(".bq") or n.endswith(".bk") or n.endswith(".bv") or n.endswith(".bo"):
                p.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                p.fill_(0.1)
    return G.double()


def _variant(duplex):
    ext = duplex == "extensions"
    return bool(duplex), (EXT if ext else {})


def _patch_attention(gf, monkeypatch, seen=None):
    """BipartiteAttention.forward -> the fp64 oracle layer (the CUDA op has no CPU form); `seen` collects the latents each call got."""
    def fake_forward(self, x, y, centroids=None, return_att=False, out=None, centroids_init=None):
        if seen is not None:
            seen.append(y)
        w = {n: p.detach() for n, p in self.named_parameters(recurse=False)}
        o, att, cen = ob.transformer_layer(x.permute(0, 3, 1, 2), y, w, integration=self.integration, norm=self.norm,
                                           duplex=self.duplex, use_pos=self.use_pos, return_att=return_att,
                                           kmeans_iters=self.kmeans_iters, img2ltnt=self.img2ltnt, centroids_init=centroids_init)
        return o.permute(0, 2, 3, 1).contiguous(), att, cen

    monkeypatch.setattr(gf.BipartiteAttention, "forward", fake_forward)


def _distinct_ws(G, B=2, seed=5):
    """Per-layer latents whose L slices are all different (each a mapping output of its own draw)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B * G.synthesis.num_ws, 5, 16, generator=g, dtype=torch.float64)
    with torch.no_grad():
        return G.mapping(z).reshape(G.synthesis.num_ws, B, 5, 16).transpose(0, 1).contiguous()


def test_num_ws(gf):
    nets = import_module(NETS)
    with torch.device("meta"):
        G = gf.Generator(resolution=256, components_num=16, latent_size=512)
    assert G.synthesis.num_ws == len(G.synthesis.layers) + 1 == 14          # StyleGAN2's count at 256^2
    s = nets.SynthesisNetwork(32, 16, 4, fmap_base=512, fmap_max=64)
    assert s.num_ws == L32 and s.ws_index == list(range(7)) + TRGB_INDEX


@pytest.mark.parametrize("grad", [False, True], ids=["inference", "autograd"])
@pytest.mark.parametrize("duplex", [False, True, "extensions"])
def test_equal_slices_give_the_broadcast_result_bit_for_bit(gf, monkeypatch, duplex, grad):
    duplex, ext = _variant(duplex)
    G = _small_generator(gf, kmeans=duplex, **ext)
    _patch_attention(gf, monkeypatch)
    z = torch.randn(2, 5, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    G.requires_grad_(grad)
    with torch.set_grad_enabled(grad):
        ws = G.mapping(z)
        img, atts, feats = G.synthesis(ws, return_att=True, return_features=True)
        img4, atts4, feats4 = G.synthesis(ws[:, None].expand(-1, L32, -1, -1), return_att=True, return_features=True)
    assert torch.equal(img4, img)
    assert len(atts4) == len(atts) == 6 and all(torch.equal(a, b) for a, b in zip(atts4, atts))
    assert all(torch.equal(a, b) for a, b in zip(feats4, feats))


@pytest.mark.parametrize("grad", [False, True], ids=["inference", "autograd"])
@pytest.mark.parametrize("duplex", [False, True, "extensions"])
def test_every_layer_reads_its_own_index(gf, monkeypatch, duplex, grad):
    """Recording fakes: each conv layer gets ws_l[:, i] (its attention the local latents, its style affine the global one), each
    tRGB the index after its block; the image matches the fp64 per-layer restatement."""
    nets = import_module(NETS)
    duplex, ext = _variant(duplex)
    G = _small_generator(gf, kmeans=duplex, **ext)
    ws_l = _distinct_ws(G)
    att_y, conv_in, rgb_in = [], [], []
    _patch_attention(gf, monkeypatch, att_y)
    layer_fwd, rgb_fwd = nets.SynthesisLayer.forward, nets.ToRGB.forward

    def rec_layer(self, x, w_glob, y, *a, **kw):
        conv_in.append((w_glob, y, kw.get("styles")))
        return layer_fwd(self, x, w_glob, y, *a, **kw)

    def rec_rgb(self, x, w_glob, styles=None, next_styles=None):
        rgb_in.append((w_glob, styles))
        return rgb_fwd(self, x, w_glob, styles=styles, next_styles=next_styles)

    monkeypatch.setattr(nets.SynthesisLayer, "forward", rec_layer)
    monkeypatch.setattr(nets.ToRGB, "forward", rec_rgb)
    G.requires_grad_(grad)
    with torch.set_grad_enabled(grad):
        img, atts = G.synthesis(ws_l, return_att=True)
    k = 4
    assert len(conv_in) == L32 - 1 and len(rgb_in) == len(TRGB_INDEX) and len(att_y) == 6
    with torch.no_grad():
        for i, (w_glob, y, styles) in enumerate(conv_in):
            assert torch.equal(w_glob, ws_l[:, i, k]) and torch.equal(y, ws_l[:, i, :k]), i
            if styles is not None:                                 # inference: the batched affine GEMM's rows of this index
                assert torch.allclose(styles, G.synthesis.layers[i].affine(ws_l[:, i, k]), rtol=1e-13, atol=1e-13), i
        assert [y.data_ptr() for y in att_y] == [conv_in[i][1].data_ptr() for i in range(1, L32 - 1)]   # layers 1..6 attend
        for bi, (w_glob, styles) in enumerate(rgb_in):
            assert torch.equal(w_glob, ws_l[:, TRGB_INDEX[bi], k]), bi
            if styles is not None:
                assert torch.allclose(styles, G.synthesis.torgbs[bi].affine(ws_l[:, TRGB_INDEX[bi], k]), rtol=1e-13, atol=1e-13), bi
    # the iterative centroid carry is an inference feature: the autograd path runs those layers without it
    ref, ratts = sref.synthesis_forward({n: t.detach() for n, t in G.state_dict().items()}, ws_l, resolution=32, components_num=4,
                                        integration="both", duplex=duplex, return_att=True,
                                        **(dict(kmeans_iters=2, img2ltnt=True, iterative=not grad) if ext else {}))
    assert (img.detach() - ref).abs().max() < 1e-9 * max(1.0, ref.abs().max().item())
    for a, r in zip(atts, ratts):
        assert (a.detach() - r).abs().max() < 1e-10


@pytest.mark.parametrize("duplex", [False, True, "extensions"])
def test_per_layer_oracle_matches_broadcast_oracle(gf, duplex):
    duplex, ext = _variant(duplex)
    G = _small_generator(gf, kmeans=duplex, **ext)
    sd = {n: t.detach() for n, t in G.state_dict().items()}
    opts = dict(kmeans_iters=2, img2ltnt=True, iterative=True) if ext else {}
    z = torch.randn(3, 5, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    ref, ratts = og.generator_forward(sd, z, resolution=32, components_num=4, latent_dim=16, integration="both", duplex=duplex,
                                      mapping_layers=2, return_att=True, **opts)
    ws = gref.mapping_forward(sd, z, components_num=4, latent_dim=16, mapping_layers=2)
    img, atts = sref.synthesis_forward(sd, sref.mix_latents(ws, ws, 3, L32), resolution=32, components_num=4, integration="both",
                                       duplex=duplex, return_att=True, **opts)
    assert (img - ref).abs().max() <= 1e-12 * max(1.0, ref.abs().max().item())
    assert len(atts) == len(ratts) == 6 and all((a - r).abs().max() <= 1e-12 for a, r in zip(atts, ratts))
    with pytest.raises(ValueError, match="latent sets"):
        sref.synthesis_forward(sd, sref.mix_latents(ws, ws, 3, L32 + 1), resolution=32, components_num=4, integration="both",
                               duplex=duplex, **opts)


def test_per_layer_ws_shape_is_checked(gf):
    G = _small_generator(gf)
    with torch.no_grad(), pytest.raises(ValueError, match=r"\[B, 8, 5, D\]"):
        G.synthesis(torch.zeros(2, L32 - 1, 5, 16, dtype=torch.float64))


def test_mix_latents_index_rule():
    tr = import_module(TRAIN)
    g = torch.Generator().manual_seed(0)
    ws1, ws2 = torch.randn(3, 5, 16, generator=g), torch.randn(3, 5, 16, generator=g)
    for cutoff in range(0, L32 + 1):
        got = tr.mix_latents(ws1, ws2, torch.tensor(cutoff), L32)
        assert torch.equal(got, sref.mix_latents(ws1, ws2, cutoff, L32)), cutoff


def test_cutoff_sampler_p0_draws_nothing():
    tr = import_module(TRAIN)
    torch.manual_seed(3)
    state = torch.get_rng_state()
    for _ in range(10):
        c = tr.mixing_cutoff(0.0, 14, "cpu")
        assert c.dtype == torch.int64 and c.dim() == 0 and int(c) == 14
    assert torch.equal(torch.get_rng_state(), state)


def test_cutoff_sampler_p1_always_mixes():
    tr = import_module(TRAIN)
    torch.manual_seed(4)
    cuts = torch.stack([tr.mixing_cutoff(1.0, 14, "cpu") for _ in range(2000)])
    assert int(cuts.min()) >= 1 and int(cuts.max()) <= 13
    assert set(cuts.tolist()) == set(range(1, 14))


def test_cutoff_sampler_frequencies():
    """p = 0.9, L = 14, 20 000 draws: the mixing rate within 5 standard deviations of p, each cutoff 1..13 within 5 of uniform."""
    tr = import_module(TRAIN)
    torch.manual_seed(5)
    n, p, L = 20000, 0.9, 14
    cuts = torch.stack([tr.mixing_cutoff(p, L, "cpu") for _ in range(n)])
    mixed = (cuts < L).double().mean().item()
    assert abs(mixed - p) <= 5 * (p * (1 - p) / n) ** 0.5, mixed
    counts = torch.bincount(cuts[cuts < L], minlength=L)[1:].double()
    q = 1.0 / (L - 1)
    m = counts.sum().item()
    assert ((counts / m - q).abs() <= 5 * (q * (1 - q) / m) ** 0.5).all(), counts.tolist()


def _tiny_gan(gf, tr):
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32)
    return G, D


def test_trainer_style_mixing_step_plumbing(gf):
    tr = import_module(TRAIN)
    G, D = _tiny_gan(gf, tr)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", style_mixing=0.9))
    g = torch.Generator().manual_seed(3)
    z, reals = torch.randn(4, 5, 16, generator=g), torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    g0 = [p.detach().clone() for p in G.parameters()]
    torch.manual_seed(6)
    stats = [trainer.step(z, reals) for _ in range(4)]
    L = G.synthesis.num_ws
    for s in stats:
        assert all(v == v and abs(v) < 1e6 for v in (s.loss_g, s.loss_d, s.r1))
        assert set(s.extra) == {"style_mixing_cutoff_d", "style_mixing_cutoff_g"}
        assert all(1 <= v <= L and v == int(v) for v in s.extra.values())
    assert len({v for s in stats for v in s.extra.values()}) > 1                # each phase of each step draws its own cutoff
    assert any((a - b.detach()).abs().max() > 0 for a, b in zip(g0, G.parameters()))
    assert tr.Trainer(G, D, tr.TrainConfig()).step(z, reals).extra == {}       # off by default: no cutoffs reported


def test_trainer_style_mixing_validation(gf):
    tr = import_module(TRAIN)
    G, D = _tiny_gan(gf, tr)
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError, match="style_mixing"):
            tr.Trainer(G, D, tr.TrainConfig(style_mixing=bad))
