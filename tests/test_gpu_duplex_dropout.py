"""Attention dropout on duplex layers (run on an H100: ``pytest -m gpu``): the forward with dropped pass-B probabilities and the
kernel backward (stage-T backward + the pass-A backward gf_attn_centroid_stats / gf_attn_centroid_bwd) against the fp64 oracle
given the same Philox mask (oracle/philox.py), and a graphed training step of a duplex generator with dropout on."""
import math
from importlib import import_module

import pytest
import torch

from oracle import bipartite as ob
from oracle import philox as ph
from tests.test_gpu_parity import check_close

pytestmark = pytest.mark.gpu

SHAPES = [  # C, H, W, k, integration, norm, img2ltnt, exact
    (64, 8, 16, 4, "both", "layer", False, True),       # KP = 16, one full tile per image
    (96, 10, 13, 20, "mul", "layer", True, True),       # KP = 32, ragged n = 130, g_img2ltnt
    (128, 16, 16, 16, "add", "none", False, True),      # no normalisation, additive integration
    (128, 16, 16, 16, "mul", "layer", False, False),    # TF32 (wgmma) forward
    (256, 16, 24, 20, "mul", "layer", True, False),     # TF32, KP = 32, g_img2ltnt
    (128, 8, 16, 8, "both", "none", False, False),      # TF32, both, no normalisation
]


def _rel(a, b):
    return ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30)).item()


def _case(gf, dev, C, H, W, k, integration, norm, img2ltnt, exact, given_centroids):
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    D = p = 16
    B, pd = 2, (0.25 if exact else 0.2)
    g = torch.Generator().manual_seed(C + k + H)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64).requires_grad_(True)
    cen64 = torch.randn(B, k, C, generator=g, dtype=torch.float64) if given_centroids else None
    nrm = None if norm == "none" else norm
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, norm=nrm, kmeans=True, img2ltnt=img2ltnt, att_dp=pd,
                                 exact_fp32=exact).to(dev)
    w0 = ob.init_params(C, D, k, p, integration, True, seed=4, bias_std=0.3, extras=img2ltnt)
    w = {n: w0[n].requires_grad_(True) for n, _ in attn.named_parameters()}
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].detach().float())
    seed, step = 987654321 + C, 3
    am.set_dropout_seed(seed, dev, step)
    KP = 16 if k <= 16 else 32
    mult = torch.from_numpy(ph.dropout_mult(pd, seed, step, attn.dp_salt, B * H * W, KP).reshape(B, H * W, KP)[:, :, :k].copy())
    ref, ratt, _ = ob.transformer_layer(x64, y64, w, integration=integration, norm=nrm, duplex=True, return_att=True, att_mult=mult,
                                        img2ltnt=img2ltnt, centroids_in=cen64)
    gout = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(gout)
    xg = x64.detach().permute(0, 2, 3, 1).contiguous().float().to(dev)
    yg = y64.detach().float().to(dev)
    cg = cen64.float().to(dev) if given_centroids else None
    gg = gout.permute(0, 2, 3, 1).contiguous().float().to(dev)
    path = "simt_fp32" if exact else "wgmma_tf32"

    # training-mode forward without autograd (the D step's fakes): dropped probabilities, map before dropout
    attn.train()
    with torch.no_grad():
        out, att, _ = attn(xg, yg, centroids=cg, return_att=True)
    assert gf._lib.last_path() == path
    check_close(out, ref.detach().permute(0, 2, 3, 1), path, "duplex-dropout/forward", tol_scale=2.0)
    assert (att.cpu().double() - ratt.detach()).abs().max() <= (1e-4 if exact else 5e-3)

    # the same forward under autograd, then the kernel backward: the three kernels run (one when the centroids are given)
    grads = []
    for _ in range(2):
        attn.zero_grad(set_to_none=True)
        xr, yr = xg.clone().requires_grad_(True), yg.clone().requires_grad_(True)
        out2, _, _ = attn(xr, yr, centroids=cg)
        assert torch.equal(out2.detach(), out)
        launches0 = gf._lib.launch_count()
        out2.backward(gg)
        torch.cuda.synchronize()
        assert gf._lib.launch_count() - launches0 == (1 if given_centroids else 4)      # simplex_bwd (+ stats: 2, centroid_bwd: 1)
        grads.append([xr.grad, yr.grad] + [prm.grad for _, prm in attn.named_parameters()])
    for a, b in zip(*grads):                                         # deterministic: bit-identical gradients from run to run
        assert (a is None and b is None) or torch.equal(a, b)

    tx, tp = (1e-4, 2e-4) if exact else (2e-3, 2e-3)
    assert _rel(xr.grad, x64.grad.permute(0, 2, 3, 1)) < tx
    assert _rel(yr.grad, y64.grad) < tx
    checked = []
    for n, prm in attn.named_parameters():
        if w[n].grad is None:                 # wk (duplex keys come from the centroids); the pass-A weights with given centroids
            assert prm.grad is None, n
            continue
        if w[n].grad.norm() < 1e-9:           # bk, bk2, and bv2 without g_img2ltnt: constant over what the softmax normalises
            assert prm.grad.norm().item() < 1e-3, n
            continue
        assert _rel(prm.grad, w[n].grad) < tp, n
        checked.append(n)
    want = {"wq", "wv", "wo", "wkc", "pos_latent", "wpq", "wpk", "bq", "bv", "bo"}
    if not given_centroids:
        want |= {"wq2", "wk2", "wv2", "wpq2", "wpk2", "bq2"}
    if img2ltnt:
        want |= {"wi2l", "bi2l"}
    assert want <= set(checked), want - set(checked)

    # eval mode: no dropout
    with torch.no_grad():
        attn.eval()
        out4, _, _ = attn(xg, yg, centroids=cg)
    ref0, _, _ = ob.transformer_layer(x64.detach(), y64.detach(), {n: t.detach() for n, t in w.items()}, integration=integration, norm=nrm,
                                      duplex=True, img2ltnt=img2ltnt, centroids_in=cen64)
    check_close(out4, ref0.permute(0, 2, 3, 1), path, "duplex-dropout/eval", tol_scale=2.0)


@pytest.mark.parametrize("C,H,W,k,integration,norm,img2ltnt,exact", SHAPES,
                         ids=lambda v: str(v))
def test_duplex_dropout_forward_and_backward(gf, cuda_dev, C, H, W, k, integration, norm, img2ltnt, exact):
    """Duplex layer with att_dp in training mode: forward, attention map and every gradient against the fp64 oracle given the same
    mask; two backward calls give bit-identical gradients; eval mode has no dropout."""
    _case(gf, cuda_dev, C, H, W, k, integration, norm, img2ltnt, exact, given_centroids=False)


@pytest.mark.parametrize("C,H,W,k,integration,norm,img2ltnt,exact", [SHAPES[1], SHAPES[2], SHAPES[4]], ids=lambda v: str(v))
def test_duplex_dropout_with_given_centroids(gf, cuda_dev, C, H, W, k, integration, norm, img2ltnt, exact):
    """centroids= passed in: pass A is skipped in the forward and the backward (one library kernel), the centroids get no gradient."""
    _case(gf, cuda_dev, C, H, W, k, integration, norm, img2ltnt, exact, given_centroids=True)


def test_duplex_dropout_kmeans_iters_2_raises(gf, cuda_dev):
    attn = gf.BipartiteAttention(64, 16, 8, kmeans=True, kmeans_iters=2, att_dp=0.12).to(cuda_dev)
    attn.train()
    x, y = torch.randn(2, 8, 8, 64, device=cuda_dev), torch.randn(2, 8, 16, device=cuda_dev)
    with pytest.raises(NotImplementedError, match="kmeans_iters == 1"):
        attn(x.requires_grad_(True), y)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="kmeans_iters == 1"):
        attn(x, y)


def test_duplex_dropout_training_step_graph_replay(gf, cuda_dev):
    """Trainer.step_graphed of a duplex generator with attention dropout (as in the paper): the captured step trains, losses stay
    finite, and the pass-A weights of the attention layers move on every replay."""
    tr = import_module("gansformer-reproducibility-challenge_b200.training")
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, kmeans=True,
                     att_dp=0.12).to(cuda_dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128).to(cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(d_reg_interval=2))
    g = torch.Generator().manual_seed(5)
    z = torch.randn(4, 9, 32, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(cuda_dev)
    layer = G.synthesis.layers[2].attention
    assert layer.duplex
    snaps, stats = [], []
    for _ in range(5):
        stats.append(trainer.step_graphed(z, reals))
        snaps.append({n: getattr(layer, n).detach().clone() for n in ("wq2", "wk2", "wv2")})
    assert all(math.isfinite(s.loss_g) and math.isfinite(s.loss_d) for s in stats)
    for a, b in zip(snaps, snaps[1:]):
        for n in a:
            assert (a[n] - b[n]).abs().max() > 0, n
