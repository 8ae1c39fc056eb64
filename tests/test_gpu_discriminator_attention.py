"""The discriminator's bipartite attention on the H100 (``pytest -m gpu``): logits against the fp64 oracle (oracle/discriminator.py)
in both forward modes, every gradient of the kernel route (CUDA forward + duplex kernel backward with the centroid cotangent)
against fp64 autograd, the R1 penalty through the torch composite against an fp64 double backward, the refusal of a second
derivative on the kernel route, determinism, the pass-A path, and graphed training steps."""
import math
from importlib import import_module

import pytest
import torch

from oracle import discriminator as od

pytestmark = pytest.mark.gpu

tr = import_module("gansformer-reproducibility-challenge_b200.training")
ag = import_module("gansformer-reproducibility-challenge_b200.autograd")

# Bounds on |logit - logit64| / max(1, max |logit64|) and on the relative L2 error of every gradient.  fp32: the CUDA-core
# attention kernels and fp32 convolutions, fp32 bounds (measured worst on an H100 80GB HBM3: logits 1.6e-6, gradients 6.3e-6,
# R1 9.0e-6).  TF32: the wgmma forward, bounds frozen at >= 1.5x the measured worst (logits 2.0e-3, gradients 3.6e-2, the
# query bias of the first layer; the image gradient 1.6e-2).  The kernel backward itself is fp32 on both routes.
LOGIT_TOL = {"fp32": 1e-5, "tf32": 3.5e-3}
GRAD_TOL = {"fp32": 1e-4, "tf32": 6e-2}
R1_TOL = 1e-4

B, RES, K, DL = 4, 32, 8, 16


def _make(dev, mode, integration="mul", norm="layer", seed=0):
    torch.manual_seed(seed)
    D = tr.Discriminator(RES, fmap_base=1024, fmap_max=128, transformer=True, components_num=K, latent_dim=DL, integration=integration,
                         norm=norm, exact_fp32=(mode == "fp32"))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():                                                   # every term live
        for n, p in D.named_parameters():
            if n.split(".")[-1] in ("bias", "bq", "bk", "bv", "bo", "bq2", "bk2", "bv2", "bi2l"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.2)
    return D.to(dev)


def _inputs(seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, RES, RES, generator=g, dtype=torch.float64), torch.randn(B, generator=g, dtype=torch.float64)


def _rel(a, b):
    return ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("integration,norm", [("mul", "layer"), ("both", None)])
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_logits_match_oracle(gf, cuda_dev, mode, integration, norm):
    D = _make(cuda_dev, mode, integration, norm)
    img, _ = _inputs()
    with torch.no_grad():
        got = D(img.float().to(cuda_dev))
    assert gf._lib.last_path() == ("simt_fp32" if mode == "fp32" else "wgmma_tf32")
    ref = od.discriminator_forward(D.state_dict(), img, integration=integration, norm=norm)
    err = (got.double().cpu() - ref).abs().max().item() / max(1.0, ref.abs().max().item())
    print(f"[d-attention] logits {mode} {integration}/{norm}: err {err:.3e} (bound {LOGIT_TOL[mode]:.1e}), max |logit| {ref.abs().max().item():.3f}")
    assert err <= LOGIT_TOL[mode]


def _kernel_route_errors(dev, mode):
    """Relative errors of every gradient of the kernel route against fp64 autograd through the oracle: the parameters and the
    latents with the image constant (the discriminator step), the image with the parameters frozen (the generator step)."""
    D = _make(dev, mode)
    img, gw = _inputs()
    x, w = img.float().to(dev), gw.float().to(dev)
    D.zero_grad(set_to_none=True)
    (D(x) * w).sum().backward()
    D.requires_grad_(False)
    xr = x.clone().requires_grad_(True)
    (D(xr) * w).sum().backward()
    D.requires_grad_(True)
    sd = {n: p.detach().double().cpu().requires_grad_(True) for n, p in D.named_parameters()}
    xd = img.clone().requires_grad_(True)
    (od.discriminator_forward(sd, xd) * gw).sum().backward()
    errs = {"image": _rel(xr.grad, xd.grad)}
    for n, p in D.named_parameters():
        if n.endswith(".bk2"):                      # constant over the tokens: cancels in pass A's softmax, exactly 0 on this route
            assert torch.count_nonzero(p.grad) == 0, n
        elif sd[n].grad is None:                    # wk: duplex keys come from the centroids
            assert p.grad is None, n
        elif sd[n].grad.norm() < 1e-9:              # bk: the same for every latent, cancels in pass B's softmax
            assert p.grad.abs().max().item() < 1e-3, n
        else:
            errs[n] = _rel(p.grad, sd[n].grad)
    return errs


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_kernel_route_gradients(gf, cuda_dev, mode):
    """Image, latents and every parameter; the centroid cotangent (the Y carry) is part of every attention layer's gradient."""
    errs = _kernel_route_errors(cuda_dev, mode)
    worst = max(errs, key=errs.get)
    print(f"[d-attention] gradients {mode}: worst {worst} {errs[worst]:.3e} (bound {GRAD_TOL[mode]:.1e}), image {errs['image']:.3e}, "
          f"latents {errs['latents']:.3e}, {len(errs)} tensors")
    assert "latents" in errs and "blocks.0.att0.wv2" in errs and "blocks.2.att1.wi2l" in errs
    assert errs[worst] <= GRAD_TOL[mode], worst


def test_kernel_route_gradients_need_the_centroid_cotangent(gf, cuda_dev, monkeypatch):
    """Without dCen (the centroids treated as constants, as for generator layers) the check above fails."""
    orig = ag._duplex_kernel_backward
    monkeypatch.setattr(ag, "_duplex_kernel_backward",
                        lambda m, names, x, y, params, g_out, dropout, centroids, g_cen: orig(m, names, x, y, params, g_out, dropout, centroids))
    errs = _kernel_route_errors(cuda_dev, "fp32")
    print(f"[d-attention] gradients without dCen: image {errs['image']:.3e}, max {max(errs.values()):.3e}")
    assert errs["image"] > 100 * GRAD_TOL["fp32"] and max(errs.values()) > 0.1


def test_r1_matches_oracle_double_backward(gf, cuda_dev, monkeypatch):
    """The lazy R1 pass: image and parameters require grad, so the layers run composite_forward (no library call); the penalty,
    the image gradient and the penalty's parameter gradients against an fp64 double backward through the oracle."""
    D = _make(cuda_dev, "tf32")
    img, _ = _inputs()

    def no_kernel(*a, **k):
        raise AssertionError("the R1 pass called the attention kernels")

    monkeypatch.setattr(gf.BipartiteAttention, "forward", no_kernel)
    x = img.float().to(cuda_dev).requires_grad_(True)
    logits = D(x)
    (gx,) = torch.autograd.grad(logits.sum(), x, create_graph=True)
    r1 = gx.square().sum(dim=[1, 2, 3]).mean()
    D.zero_grad(set_to_none=True)
    r1.backward()
    sd = {n: p.detach().double().cpu().requires_grad_(True) for n, p in D.named_parameters()}
    xd = img.clone().requires_grad_(True)
    (gr,) = torch.autograd.grad(od.discriminator_forward(sd, xd).sum(), xd, create_graph=True)
    r1r = gr.square().sum(dim=[1, 2, 3]).mean()
    r1r.backward()
    errs = {"r1": abs(r1.item() - r1r.item()) / r1r.item(), "image": _rel(gx, gr)}
    for n, p in D.named_parameters():
        if sd[n].grad is not None and sd[n].grad.norm() > 1e-9:
            errs[n] = _rel(p.grad, sd[n].grad)
    worst = max(errs, key=errs.get)
    print(f"[d-attention] R1: penalty {r1.item():.4e} err {errs['r1']:.3e}, worst {worst} {errs[worst]:.3e}, {len(errs)} tensors")
    assert "latents" in errs and "blocks.1.att1.wq2" in errs
    assert errs[worst] <= R1_TOL, worst


def test_kernel_route_refuses_a_second_derivative(gf, cuda_dev):
    D = _make(cuda_dev, "tf32").requires_grad_(False)           # parameters frozen: the image alone requires grad -> kernel route
    img, _ = _inputs()
    x = img.float().to(cuda_dev).requires_grad_(True)
    logits = D(x)
    with pytest.raises(RuntimeError, match="no derivative of its own"):
        torch.autograd.grad(logits.sum(), x, create_graph=True)
    (gx,) = torch.autograd.grad(D(x).sum(), x)                  # a first derivative is fine
    assert torch.isfinite(gx).all()


def test_kernel_backward_is_deterministic_and_pass_a_on_tensor_cores(gf, cuda_dev):
    """Two backward calls through a discriminator layer, with cotangents on both the output and the centroids, give the same bits;
    the TF32 forward runs pass A on the wgmma kernel."""
    D = _make(cuda_dev, "tf32")
    with torch.no_grad():
        D(_inputs()[0].float().to(cuda_dev))
    assert gf._lib.last_centroid_path() == "wgmma_tf32"
    att = D.blocks[0].att0                                          # C = 64, 32 x 32 tokens, k = 8, g_img2ltnt
    g = torch.Generator().manual_seed(9)
    x, y = torch.randn(B, RES, RES, 64, generator=g).to(cuda_dev), torch.randn(B, K, DL, generator=g).to(cuda_dev)
    g_out, g_cen = torch.randn(B, RES, RES, 64, generator=g).to(cuda_dev), torch.randn(B, K, 64, generator=g).to(cuda_dev)
    runs = []
    for _ in range(2):
        att.zero_grad(set_to_none=True)
        xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        out, _, cen = att(xr, yr)
        assert gf._lib.last_centroid_path() == "wgmma_tf32" and cen.requires_grad
        torch.autograd.backward([out, cen], [g_out, g_cen])
        runs.append([xr.grad, yr.grad] + [p.grad for p in att.parameters()])
    for a, b in zip(*runs):
        assert (a is None and b is None) or torch.equal(a, b)
    assert runs[0][0].abs().max() > 0 and runs[0][1].abs().max() > 0


def test_training_step_graph_replay_with_attention_discriminator(gf, cuda_dev):
    """Trainer.step_graphed with a transformer discriminator at 64x64: both graphs (with the lazy R1 term, through the composite,
    and without it, through the kernels) train; the discriminator's attention parameters and latents move on every replay."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4).to(cuda_dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, transformer=True, components_num=8, latent_dim=32).to(cuda_dev)
    assert sum(b.att0 is not None for b in D.blocks) == 4
    trainer = tr.Trainer(G, D, tr.TrainConfig(d_reg_interval=2))
    g = torch.Generator().manual_seed(5)
    z = torch.randn(4, 9, 32, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(cuda_dev)
    snaps, stats = [], []
    for _ in range(5):
        stats.append(trainer.step_graphed(z, reals))
        snaps.append((torch.cat([p.detach().reshape(-1) for n, p in D.named_parameters() if ".att" in n]).clone(), D.latents.detach().clone()))
    assert all(math.isfinite(s.loss_g) and math.isfinite(s.loss_d) and math.isfinite(s.r1) for s in stats)
    assert [s.r1 > 0 for s in stats] == [True, False, True, False, True]
    for (a, la), (b, lb) in zip(snaps, snaps[1:]):
        assert (a - b).abs().max() > 0 and (la - lb).abs().max() > 0
