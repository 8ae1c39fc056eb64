"""CPU tests of the discriminator's bipartite attention (``Discriminator(transformer=True)``): the plain discriminator is unchanged
bit for bit, parameter shapes and construction errors, and the block / attention plumbing and the latent carry against
oracle/discriminator.py -- with the CUDA attention op swapped for the oracle layer, and through the torch composite the R1 pass
runs (first and second derivatives).  No kernel is launched here."""
import math
from importlib import import_module

import pytest
import torch
import torch.nn as nn

from oracle import bipartite as ob
from oracle import discriminator as od

tr = import_module("gansformer-reproducibility-challenge_b200.training")


# ---- the discriminator as it was before the attention option, kept verbatim as the yardstick of transformer=False -------------
class _OldBlock(nn.Module):
    def __init__(self, in_ch, out_ch):
        super().__init__()
        self.conv0 = tr.EqConv2d(in_ch, in_ch, 3)
        self.conv1 = tr.EqConv2d(in_ch, out_ch, 3, down=True)
        self.skip = tr.EqConv2d(in_ch, out_ch, 1, down=True, bias=False, act="linear")

    def forward(self, x):
        return (self.skip(x) + self.conv1(self.conv0(x))) * (1.0 / tr.SQRT2)


class _OldDiscriminator(nn.Module):
    def __init__(self, resolution=256, fmap_base=16384, fmap_max=512, mbstd_group=4):
        super().__init__()
        self.resolution, self.mbstd_group = resolution, mbstd_group
        log2 = int(math.log2(resolution))
        self.fromrgb = tr.EqConv2d(3, tr.nf(resolution, fmap_base, fmap_max), 1)
        self.blocks = nn.ModuleList([_OldBlock(tr.nf(2 ** i, fmap_base, fmap_max), tr.nf(2 ** (i - 1), fmap_base, fmap_max))
                                     for i in range(log2, 2, -1)])
        c4 = tr.nf(4, fmap_base, fmap_max)
        self.conv4 = tr.EqConv2d(c4 + 1, c4, 3)
        self.fc0 = tr.FullyConnected(c4 * 16, c4, act="lrelu")
        self.fc1 = tr.FullyConnected(c4, 1)

    def forward(self, img):
        x = self.fromrgb(img.contiguous(memory_format=torch.channels_last))
        for blk in self.blocks:
            x = blk(x)
        B, C, H, W = x.shape
        G = min(self.mbstd_group, B)
        while B % G:
            G -= 1
        y = x.reshape(G, B // G, C, H, W)
        y = (y - y.mean(dim=0, keepdim=True)).square().mean(dim=0).add(1e-8).sqrt().mean(dim=[1, 2, 3])
        y = y.reshape(1, B // G, 1, 1).expand(G, -1, H, W).reshape(B, 1, H, W)
        x = self.conv4(torch.cat([x, y], dim=1))
        return self.fc1(self.fc0(x.reshape(B, -1))).reshape(B)


PLAIN_KEYS_16 = [
    "fromrgb.weight", "fromrgb.bias",
    "blocks.0.conv0.weight", "blocks.0.conv0.bias", "blocks.0.conv1.weight", "blocks.0.conv1.bias", "blocks.0.skip.weight",
    "blocks.1.conv0.weight", "blocks.1.conv0.bias", "blocks.1.conv1.weight", "blocks.1.conv1.bias", "blocks.1.skip.weight",
    "conv4.weight", "conv4.bias", "fc0.weight", "fc0.bias", "fc1.weight", "fc1.bias",
]


def test_plain_discriminator_is_unchanged():
    """transformer=False (the default): same state-dict keys, same initial weights from the same seed, and a bit-identical forward,
    backward and R1 double backward compared with the discriminator as it was before the option existed."""
    torch.manual_seed(3)
    old = _OldDiscriminator(16, fmap_base=256, fmap_max=32)
    torch.manual_seed(3)
    new = tr.Discriminator(16, fmap_base=256, fmap_max=32)
    assert list(new.state_dict()) == list(old.state_dict()) == PLAIN_KEYS_16
    assert tr.Discriminator(16, fmap_base=256, fmap_max=32, transformer=False).fc0.weight.shape == (32, 32 * 16)
    for (n, a), (_, b) in zip(new.state_dict().items(), old.state_dict().items()):
        assert torch.equal(a, b), n
    with torch.no_grad():                                   # make every term live
        for (n, a), (_, b) in zip(new.named_parameters(), old.named_parameters()):
            v = torch.randn_like(a) * 0.3 if n.endswith("bias") else a
            a.copy_(v)
            b.copy_(v)
    g = torch.Generator().manual_seed(4)
    img = torch.randn(6, 3, 16, 16, generator=g)
    grads = []
    for D in (new, old):
        x = img.clone().requires_grad_(True)
        D.zero_grad(set_to_none=True)
        logits = D(x)
        (gx,) = torch.autograd.grad(logits.sum(), x, create_graph=True)
        r1 = gx.square().sum(dim=[1, 2, 3]).mean()
        (logits.square().sum() + r1).backward()
        grads.append([logits.detach(), gx.detach(), x.grad] + [p.grad for p in D.parameters()])
    for i, (a, b) in enumerate(zip(*grads)):
        assert torch.equal(a, b), i


def _att_d(**kw):
    args = dict(fmap_base=1024, fmap_max=128, transformer=True, components_num=4, latent_dim=16)
    args.update(kw)
    return tr.Discriminator(32, **args)


def test_parameter_shapes_and_layers():
    D = _att_d()
    C = [(b.att0.dim, b.att1.dim) for b in D.blocks]
    assert C == [(64, 128), (128, 128), (128, 128)]            # blocks at input resolution 32, 16, 8: both layers each
    for b in D.blocks:
        for att in (b.att0, b.att1):
            assert att.duplex and att.kmeans_iters == 1 and att.img2ltnt and att.kernel_backward and att.num_heads == 1
            want = ob.param_shapes(att.dim, 16, 4, 16, "mul", True, extras=True)
            del want["wcq"]
            assert {n: tuple(p.shape) for n, p in att.named_parameters()} == want
    assert D.latents.shape == (4, 16)
    assert D.fc0.weight.shape == (128, 128 * 16 + 4 * 16)
    assert not tr.BipartiteAttention(64, 16, 4, kmeans=True).kernel_backward           # the generator's default route
    # the attention range, in input resolutions of the blocks
    assert [b.att0 is not None for b in _att_d(d_end_res=16).blocks] == [False, True, True]
    assert [b.att0 is not None for b in _att_d(d_start_res=16, d_end_res=16).blocks] == [False, True, False]
    assert [b.att0 is not None for b in _att_d(d_start_res=64).blocks] == [False, False, False]
    assert _att_d(d_start_res=64).fc0.weight.shape == (128, 128 * 16 + 4 * 16)          # Y is still concatenated
    plain = tr.Discriminator(32, fmap_base=1024, fmap_max=128)
    assert all(b.att0 is None and b.att1 is None for b in plain.blocks) and not hasattr(plain, "latents")


def test_construction_errors():
    with pytest.raises(RuntimeError, match="C=48 unsupported"):
        _att_d(fmap_max=48)
    with pytest.raises(RuntimeError, match="k=33 unsupported"):
        _att_d(components_num=33)
    with pytest.raises(RuntimeError, match="D=300 unsupported"):
        _att_d(latent_dim=300)
    with pytest.raises(RuntimeError, match="pos_dim=18 unsupported"):
        _att_d(latent_dim=18)
    with pytest.raises(ValueError, match="norm 'layer' or None"):
        _att_d(norm="instance")
    with pytest.raises(ValueError, match="unknown integration"):
        _att_d(integration="sum")
    _att_d(latent_dim=18, use_pos=False, fmap_max=64)                # no positional encoding: D need not be a multiple of 4


def _live(D, seed=0):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in D.named_parameters():
            if n.split(".")[-1] in ("bias", "bq", "bk", "bv", "bo", "bq2", "bk2", "bv2", "bi2l"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return D.double()


@pytest.mark.parametrize("integration,norm,use_pos", [("mul", "layer", True), ("both", None, True), ("add", "layer", False)])
def test_plumbing_matches_oracle_with_patched_attention(gf, monkeypatch, integration, norm, use_pos):
    """Layer order, the channels-last layout around the layers, the Y carry and the final concatenation: the CUDA op swapped for
    the oracle layer, logits and every carried Y against oracle/discriminator.py."""
    torch.manual_seed(0)
    D = _live(_att_d(integration=integration, norm=norm, use_pos=use_pos))
    seen = []

    def fake_forward(self, x, y, centroids=None, return_att=False, out=None):
        seen.append((self.dim, tuple(x.shape), y.detach().clone()))
        w = {n: p.detach() for n, p in self.named_parameters(recurse=False)}
        o, att, cen = ob.transformer_layer(x.permute(0, 3, 1, 2), y, w, integration=self.integration, norm=self.norm, duplex=True,
                                           use_pos=self.use_pos, img2ltnt=True)
        return o.permute(0, 2, 3, 1).contiguous(), att, cen

    monkeypatch.setattr(gf.BipartiteAttention, "forward", fake_forward)
    img = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    with torch.no_grad():
        got = D(img)
    ref, ys = od.discriminator_forward(D.state_dict(), img, integration=integration, norm=norm, use_pos=use_pos, return_latents=True)
    assert [(c, s) for c, s, _ in seen] == [(64, (4, 32, 32, 64)), (128, (4, 16, 16, 128)), (128, (4, 16, 16, 128)),
                                            (128, (4, 8, 8, 128)), (128, (4, 8, 8, 128)), (128, (4, 4, 4, 128))]
    assert len(ys) == 7
    for (_, _, y), yr in zip(seen, ys):                         # each layer receives the Y the previous layer left
        assert (y - yr).abs().max() < 1e-12
    assert (ys[1] - ys[0]).abs().max() > 0.1                    # the carry moves Y
    assert (got - ref).abs().max() < 1e-10 * max(1.0, ref.abs().max().item())


def test_r1_route_matches_oracle_double_backward(gf):
    """Image and parameters both requiring grad under grad mode: the layers run composite_forward (no library call, so this runs
    on the CPU); logits, the image gradient, the R1 penalty and its parameter gradients against the oracle in float64."""
    torch.manual_seed(0)
    D = _live(_att_d(integration="both"))
    img = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    x = img.clone().requires_grad_(True)
    logits = D(x)
    (gx,) = torch.autograd.grad(logits.sum(), x, create_graph=True)
    r1 = gx.square().sum(dim=[1, 2, 3]).mean()
    r1.backward()
    sd = {n: p.detach().clone().requires_grad_(True) for n, p in D.named_parameters()}
    xr = img.clone().requires_grad_(True)
    ref = od.discriminator_forward(sd, xr, integration="both")
    (gr,) = torch.autograd.grad(ref.sum(), xr, create_graph=True)
    r1r = gr.square().sum(dim=[1, 2, 3]).mean()
    r1r.backward()
    assert (logits - ref).abs().max() < 1e-10 * max(1.0, ref.abs().max().item())
    assert (gx - gr).abs().max() < 1e-10 * max(1.0, gr.abs().max().item())
    assert abs(r1.item() - r1r.item()) < 1e-10 * r1r.item()
    checked = 0
    for n, p in D.named_parameters():
        if sd[n].grad is None:                                  # wk: duplex keys come from the centroids
            assert p.grad is None or p.grad.abs().max() == 0, n
            continue
        assert (p.grad - sd[n].grad).abs().max() <= 1e-9 * max(1.0, sd[n].grad.abs().max().item()), n
        checked += 1
    assert checked > 100 and sd["latents"].grad.abs().max() > 0 and sd["blocks.0.att0.wi2l"].grad.abs().max() > 0
