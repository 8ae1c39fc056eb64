"""Class-conditional generation and training on an H100 (``pytest -m gpu``; SURVEY A.4 item 14).

* gf_mapping_fwd_cond through the C ABI, output between NaN guards: exact cases (one-hot labels, embedding entries +-1, z = +-1,
  so every 2D concatenation normalises by exactly rsqrtf(1); weights +-5, biases in {-5, 0, 5}, psi = 1/2) equal fp64 bit for bit.
  They cover c_dim = 1, 10, 1000, k = 0, 1, 31, D = 16 to 128, batches that wrap the grid, and cases where every image has a
  class of its own.  tests/test_host_cpu_conditional.py proves each case exact on the host.  One realistic case (soft labels) is
  held to a frozen bound relative to its magnitude companion.
* A conditional generator in fp32 and TF32 against the fp64 restatement (tests/conditional_ref.py) under the end-to-end bounds of
  tolerances.json; the graphed replay and ``run`` with labels against ``G(z, c)``; a different class changes the image; batch
  independence.  The conditional discriminator against fp64, with and without attention.
* Training: after one eager step the gradients of ``mapping.embed`` and of D's fc1 against fp64 autograd; the R1, path-length and
  style-mixing phases with labels; ``step_graphed`` with labels against the eager step from the same state (losses and gradients);
  labels on the host reach the device.
"""
import copy
import math
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref
from tests.guards import Guarded, assert_exact
from tests.test_gpu_ops_exact import F64, _call, _dev, _ptr, _seed, _sms, _stream, ints, lrelu5
from tests.test_gpu_style_mixing import E2E, check_image

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
COND_PSI = 0.5
# Realistic case: max over elements of |y - y64| / companion.  Measured 1.13e-7 on an H100 80GB HBM3 at a 700 W power limit,
# frozen with a margin of at least 1.5x.
COND_REL_BOUND = 2e-7
TOL_GRAD = 1e-4           # relative error of the embedding's and fc1's gradients after one step, fp32 against fp64


# ------------------------------------------------------------------------------------------------ the kernel, exact cases
COND_CASES = [(16, 8, 0, 1), (16, 8, 31, 1000), (48, 8, 1, 10), (96, 3, 31, 10), (128, 1, 1, 1000), (128, 1, 0, 10),
              (32, 8, 16, 1000)]                                                     # (D, L, k, c_dim)


def cond_batch(k, sms):
    """Rows B (k + 1) above twice the 8 rows per CTA times the grid of sms CTAs: every warp takes more than one row."""
    return 2 * sms * 8 // (k + 1) + 1


def cond_def(z, c, E, W0, W, b, w_avg, psi, k, *, exact_norm, lrelu=None):
    """Conditional G_mapping on z [B, k+1, D], labels c [B, c_dim], embedding E [c_dim, D]; layer 0 W0 [2, 2D, D], layers 1.. W
    [2, L-1, D, D] ([in][out]), biases b [2, L, D].  exact_norm: the pixel norm is taken as 1 (entries +-1)."""
    D = z.shape[-1]
    e = c @ E
    x = torch.cat([z, e[:, None].expand(-1, k + 1, -1)], dim=2)
    x = x if exact_norm else x / torch.sqrt(x.square().mean(dim=-1, keepdim=True) + 1e-8)
    act = lrelu or (lambda v: torch.nn.functional.leaky_relu(v, 0.2))
    outs = []
    for path, sl in ((0, slice(0, k)), (1, slice(k, k + 1))):
        h = act(x[:, sl] @ W0[path] + b[path, 0])
        for l in range(1, b.shape[1]):
            h = act(h @ W[path, l - 1] + b[path, l])
        if w_avg is not None:
            h = w_avg[path] + psi * (h - w_avg[path])
        outs.append(h)
    return torch.cat(outs, dim=1).reshape(z.shape[0], k + 1, D)


def _sparse_pm5(g, n_in, D, nnz):
    """[n_in, D]: per output column nnz weights +-5 on distinct input rows."""
    W = torch.zeros(n_in, D, dtype=F64)
    rows = torch.stack([torch.randperm(n_in, generator=g)[:nnz] for _ in range(D)], dim=1)
    W.scatter_(0, rows, 5 * (2 * torch.randint(0, 2, (nnz, D), generator=g) - 1).to(F64))
    return W


def cond_case(D, L, k, c_dim, B):
    """z and E entries +-1; one-hot labels (every image its own class when B <= c_dim); per output column one weight +-5 (two when
    L <= 2), layer 0 drawing from all 2D inputs; biases in {-5, 0, 5}; w_avg integers."""
    s = _seed(D, L, k, c_dim, B)
    g = torch.Generator().manual_seed(s)
    z = 2 * ints((B, k + 1, D), 0, 1, s) - 1
    E = 2 * ints((c_dim, D), 0, 1, s + 3) - 1
    cls = torch.randperm(c_dim, generator=g)[:B] if B <= c_dim else torch.randint(0, c_dim, (B,), generator=g)
    c = torch.nn.functional.one_hot(cls, c_dim).to(F64)
    nnz = 2 if L <= 2 else 1
    W0 = torch.stack([_sparse_pm5(g, 2 * D, D, nnz) for _ in range(2)])
    W = torch.stack([torch.stack([_sparse_pm5(g, D, D, nnz) for _ in range(L - 1)]) if L > 1 else torch.zeros(0, D, D, dtype=F64)
                     for _ in range(2)])
    b = 5 * ints((2, L, D), -1, 1, s + 1)
    return z, c, E, W0, W, b, ints((2, D), -20, 20, s + 2)


def cond_want(z, c, E, W0, W, b, w_avg, k):
    return cond_def(z, c, E, W0, W, b, w_avg, COND_PSI, k, exact_norm=True, lrelu=lrelu5)


def _cond_run(gf, dev, z, c, E, W0, W, b, w_avg, psi, k):
    B, _, D = z.shape
    L = b.shape[1]
    zd, cd, Ed, W0d, Wd, bd, ad = (_dev(t, dev) for t in (z, c, E, W0, W if L > 1 else None, b, w_avg))
    out = Guarded((B, k + 1, D), dev)
    _call(gf, "gf_mapping_fwd_cond", zd.data_ptr(), cd.data_ptr(), c.shape[1], Ed.data_ptr(), W0d.data_ptr(), _ptr(Wd), bd.data_ptr(),
          _ptr(ad), psi, out.ptr(), B, k, D, L, _stream(dev))
    return out.check("conditional mapping out").double().cpu()


def cond_id(c):
    return "D{}_L{}_k{}_c{}".format(*c)


@pytest.mark.parametrize("case", COND_CASES, ids=cond_id)
def test_conditional_mapping_exact(gf, cuda_dev, case):
    """gf_mapping_fwd_cond with the exact construction, with and without w_avg."""
    D, L, k, c_dim = case
    B = cond_batch(k, _sms())
    z, c, E, W0, W, b, w_avg = cond_case(D, L, k, c_dim, B)
    for avg in (w_avg, None):
        got = _cond_run(gf, cuda_dev, z, c, E, W0, W, b, avg, COND_PSI, k)
        assert_exact(got, cond_want(z, c, E, W0, W, b, avg, k), f"conditional mapping {case} w_avg={avg is not None}")


def test_conditional_mapping_rejects_bad_calls(gf, cuda_dev):
    """Null pointers, c_dim < 1 and weights beyond shared memory come back as errors before any launch."""
    lib = gf._lib.load()
    buf = torch.zeros(2 * 8 * 64 * 64 * 2, device=cuda_dev)
    p, st = buf.data_ptr(), _stream(cuda_dev)
    assert lib.gf_mapping_fwd_cond(p, None, 4, p, p, p, p, None, 1.0, p, 1, 0, 16, 2, st) == -1
    assert "null pointer" in lib.gf_last_error().decode()
    assert lib.gf_mapping_fwd_cond(p, p, 4, p, p, None, p, None, 1.0, p, 1, 0, 16, 2, st) == -1       # L > 1 without w
    assert lib.gf_mapping_fwd_cond(p, p, 0, p, p, p, p, None, 1.0, p, 1, 0, 16, 2, st) == -1
    assert "c_dim=0" in lib.gf_last_error().decode()
    assert lib.gf_mapping_fwd_cond(p, p, 4, p, p, p, p, None, 1.0, p, 1, 0, 64, 8, st) == -2
    assert "shared memory" in lib.gf_last_error().decode()
    assert lib.gf_mapping_fwd_cond(p, p, 4, p, p, p, p, None, 1.0, p, 1, 0, 160, 1, st) == -2


def test_conditional_mapping_realistic(gf, cuda_dev):
    """Random fp32 data and soft labels against fp64, per element relative to the magnitude companion."""
    D, L, k, B, c_dim = 128, 1, 16, 64, 10
    f32 = lambda t: t.float().double()
    rnd = lambda shape, seed: torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=F64)
    z, E = f32(rnd((B, k + 1, D), 31)), f32(rnd((c_dim, D), 32))
    c = f32(torch.rand(B, c_dim, generator=torch.Generator().manual_seed(33), dtype=F64))
    W0 = f32(rnd((2, 2 * D, D), 34) * math.sqrt(1.0 / D))
    W = torch.zeros(2, 0, D, D, dtype=F64)
    b = f32(rnd((2, L, D), 35) * 0.1)
    w_avg, psi = f32(rnd((2, D), 36)), 0.7
    got = _cond_run(gf, cuda_dev, z, c, E, W0, W, b, w_avg, psi, k)
    psi32 = float(torch.tensor(psi, dtype=torch.float32))
    want = cond_def(z, c, E, W0, W, b, w_avg, psi32, k, exact_norm=False)
    # companion (L = 1): the same expression on absolute values, |c| |E| for the embedding, scaled by the row's own norm
    e = c @ E
    rn = torch.rsqrt(torch.cat([z, e[:, None].expand(-1, k + 1, -1)], dim=2).square().mean(dim=-1, keepdim=True) + 1e-8)
    ea = c.abs() @ E.abs()
    xa = torch.cat([z.abs(), ea[:, None].expand(-1, k + 1, -1)], dim=2) * rn
    comp = torch.cat([xa[:, :k] @ W0[0].abs() + b[0, 0].abs(), xa[:, k:] @ W0[1].abs() + b[1, 0].abs()], dim=1)
    a = w_avg.abs()[[0] * k + [1]]
    comp = a + psi32 * (comp + a)
    err = (got - want).abs()
    rel = (err / comp).max().item()
    print(f"[conditional mapping] realistic: max |y - y64| / companion = {rel:.3e} (bound {COND_REL_BOUND:.1e})")
    assert rel <= COND_REL_BOUND


# ------------------------------------------------------------------------------------------------ generator end to end
def _generator(gf, dev, exact, c_dim=5, **kw):
    """64^2, K = 8, D = 32, c_dim 5, with live biases, noise strengths and w_avg."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     exact_fp32=exact, c_dim=c_dim, **kw)
    with torch.no_grad():
        for n, prm in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo"):
                prm.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                prm.fill_(0.1)
        G.mapping.w_avg.normal_(0, 0.2)
    return G.to(dev).eval()


def _inputs(B, c_dim, seed=1):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 9, 32, generator=g, dtype=F64)
    c = torch.nn.functional.one_hot(torch.arange(B) % c_dim, c_dim).to(F64)
    return z, c


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "tf32"])
def test_conditional_generator_against_fp64(gf, cuda_dev, exact, monkeypatch):
    ops = import_module("gansformer-reproducibility-challenge_b200.ops")
    G = _generator(gf, cuda_dev, exact)
    z, c = _inputs(4, 5)
    calls = []
    real = ops.mapping_fwd
    monkeypatch.setattr(ops, "mapping_fwd", lambda *a, **kw: calls.append(kw.get("c") is not None) or real(*a, **kw))
    with torch.no_grad():
        img, atts = G(z.float().to(cuda_dev), c.float().to(cuda_dev), truncation_psi=0.7, return_att=True)
        ws = G.mapping(z.float().to(cuda_dev), c.float().to(cuda_dev))
    assert calls == [True, True]                                        # the inference mapping runs on gf_mapping_fwd_cond
    sd = cref.cast(G.state_dict())
    ref, ratts = cref.generator_forward(sd, z, c, resolution=64, components_num=8, latent_dim=32, mapping_layers=4,
                                        truncation_psi=0.7, return_att=True)
    ws64 = cref.mapping_forward(sd, z, c, components_num=8, latent_dim=32, mapping_layers=4)
    print(f"[conditional] mapping max |ws - ws64| = {(ws.double().cpu() - ws64).abs().max().item():.3e}")
    assert (ws.double().cpu() - ws64).abs().max() <= 1e-5 * max(1.0, ws64.abs().max().item())
    mode = "fp32" if exact else "tf32"
    check_image(img, ref, mode, "conditional")
    assert len(atts) == len(ratts) == G.synthesis.num_attention_layers
    for a, r in zip(atts, ratts):
        assert (a.double().cpu() - r).abs().max() <= E2E["simt_fp32" if exact else "wgmma_tf32"]["att_abs"]


def test_conditional_graph_run_and_batch_independence(gf, cuda_dev):
    G = _generator(gf, cuda_dev, False)
    z, c = _inputs(10, 5, seed=2)
    zd, cd = z.float().to(cuda_dev), c.float().to(cuda_dev)
    c_other = torch.roll(cd, 1, dims=1)
    with torch.no_grad():
        eager = G(zd, cd).clone()
        other = G(zd, c_other).clone()
        replay = G.graphed(4)
        r1 = replay(zd[:4], cd[:4]).clone()
        r2 = replay(zd[:4], c_other[:4]).clone()
        run = G.run(z.float().numpy(), c.float().numpy(), minibatch_size=4, cuda_graph=True)          # 4 + 4 + a ragged 2
        run_eager = G.run(z.float(), c.float(), minibatch_size=4)
        one = G(zd[7:8], cd[7:8]).clone()
        ws_all, ws_one = G.mapping(zd, cd), G.mapping(zd[7:8], cd[7:8])
    tol = 1e-3 * max(1.0, eager.abs().max().item())         # cuDNN may pick other algorithms for other batch sizes and in a graph
    for what, got, want in (("graph", r1, eager[:4]), ("graph-other-class", r2, other[:4]), ("run-graph", run.to(cuda_dev), eager),
                            ("run", run_eager.to(cuda_dev), eager), ("one image", one, eager[7:8])):
        d = (got - want).abs().max().item()
        print(f"[conditional] {what}: max diff {d:.3e} (tol {tol:.3e})")
        assert d <= tol, what
    assert torch.equal(ws_one, ws_all[7:8])                             # the mapping kernel is per row: bit for bit
    assert (other - eager).abs().amax(dim=(1, 2, 3)).min() > 20 * tol   # the same z with another class: another image
    with pytest.raises(ValueError):
        G(zd, None)
    with pytest.raises(ValueError):
        G.run(z.float().numpy(), c.float().numpy()[:9])


def test_graphed_replay_does_not_keep_the_generator_alive(gf, cuda_dev):
    """The replay closure cached on the generator holds no reference to it: dropping the generator frees it and its captured graph
    at once, not at some later garbage collection (which could fall inside another graph's capture)."""
    import weakref
    G = _generator(gf, cuda_dev, False)
    G.graphed(2)
    ref = weakref.ref(G)
    del G
    assert ref() is None


@pytest.mark.parametrize("transformer", [False, True], ids=["plain", "attention"])
def test_conditional_discriminator_against_fp64(gf, cuda_dev, transformer):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, transformer=transformer, components_num=8, latent_dim=32, exact_fp32=True,
                         c_dim=5).to(cuda_dev).eval()
    assert D.fc1.weight.shape == (5, 128)
    g = torch.Generator().manual_seed(4)
    img = torch.rand(4, 3, 64, 64, generator=g, dtype=F64) * 2 - 1
    c = torch.nn.functional.one_hot(torch.tensor([0, 3, 4, 1]), 5).to(F64)
    with torch.no_grad():
        got = D(img.float().to(cuda_dev), c.float().to(cuda_dev)).double().cpu()
    ref = cref.discriminator_forward(cref.cast(D.state_dict()), img, c)
    err = (got - ref).abs().max().item()
    print(f"[conditional D] transformer={transformer}: max |logit - fp64| = {err:.3e}, peak {ref.abs().max().item():.3e}")
    assert err <= 2e-4 * max(1.0, ref.abs().max().item())
    with pytest.raises(ValueError):
        D(img.float().to(cuda_dev))


# ------------------------------------------------------------------------------------------------ training
def _gan(gf, dev, c_dim=5, **dkw):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, exact_fp32=True,
                     c_dim=c_dim).to(dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, c_dim=c_dim, **dkw).to(dev)
    return tr, G, D


def _batch(dev, B=4, c_dim=5, seed=5):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 9, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    gen_c = torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev)
    real_c = torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev)
    return z, reals, gen_c, real_c


def test_conditional_step_gradients_against_fp64(gf, cuda_dev):
    """One eager step (no R1, constant noise): D's fc1 gradient is that of the D loss at the initial weights with fakes of the
    initial G; the embedding's gradient is that of the G loss with the updated D.  Both against fp64 autograd."""
    tr, G, D = _gan(gf, cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", r1_gamma=0.0))
    z, reals, gen_c, real_c = _batch(cuda_dev)
    sd_g0, sd_d0 = cref.cast(G.state_dict()), cref.cast(D.state_dict())
    st = trainer.step(z, reals, gen_c, real_c)
    assert math.isfinite(st.loss_d) and math.isfinite(st.loss_g)
    sd_d1 = cref.cast(D.state_dict())
    z64, r64, gc64, rc64 = (t.double().cpu() for t in (z, reals, gen_c, real_c))
    kw = dict(resolution=64, components_num=8, latent_dim=32, mapping_layers=4)
    sp = torch.nn.functional.softplus
    with torch.enable_grad():
        with torch.no_grad():
            fakes = cref.generator_forward(sd_g0, z64, gc64, **kw)
        for n in ("fc1.weight", "fc1.bias"):
            sd_d0[n].requires_grad_(True)
        loss_d = sp(cref.discriminator_forward(sd_d0, fakes, gc64)).mean() + sp(-cref.discriminator_forward(sd_d0, r64, rc64)).mean()
        gw, gb = torch.autograd.grad(loss_d, [sd_d0["fc1.weight"], sd_d0["fc1.bias"]])
        sd_g0["mapping.embed"].requires_grad_(True)
        loss_g = sp(-cref.discriminator_forward(sd_d1, cref.generator_forward(sd_g0, z64, gc64, **kw), gc64)).mean()
        (ge,) = torch.autograd.grad(loss_g, [sd_g0["mapping.embed"]])
    print(f"[conditional step] loss_d {st.loss_d:.6f} vs {loss_d.item():.6f}, loss_g {st.loss_g:.6f} vs {loss_g.item():.6f}")
    errs = {}
    for name, got, want in (("fc1.weight", D.fc1.weight.grad, gw), ("fc1.bias", D.fc1.bias.grad, gb), ("mapping.embed", G.mapping.embed.grad, ge)):
        errs[name] = ((got.double().cpu() - want).norm() / want.norm()).item()
    print("[conditional step] gradient errors " + " ".join(f"{n}={e:.2e}" for n, e in errs.items()))
    assert ge.norm() > 0 and gw.norm() > 0
    assert all(e < TOL_GRAD for e in errs.values()), errs


@pytest.mark.parametrize("dkw", [dict(), dict(transformer=True, components_num=8, latent_dim=32, r1_kernels=True)], ids=["plain", "attention-r1k"])
def test_conditional_trainer_phases(gf, cuda_dev, dkw):
    """R1, path length and style mixing with labels: finite losses and penalties over four eager steps."""
    tr, G, D = _gan(gf, cuda_dev, **dkw)
    trainer = tr.Trainer(G, D, tr.TrainConfig(d_reg_interval=2, pl_weight=2.0, g_reg_interval=2, style_mixing=0.9))
    z, reals, gen_c, real_c = _batch(cuda_dev)
    stats = [trainer.step(z, reals, gen_c, real_c) for _ in range(4)]
    for s in stats:
        assert all(math.isfinite(v) for v in (s.loss_d, s.loss_g, s.r1, s.pl_penalty, s.pl_mean)), s
    assert [s.r1 > 0 for s in stats] == [True, False, True, False] and stats[2].pl_mean > 0
    with pytest.raises(ValueError):
        trainer.step(z, reals, gen_c, None)


def _onehot(classes, dev, c_dim=5):
    return torch.nn.functional.one_hot(torch.tensor(classes), c_dim).float().to(dev)


def _assert_class_rows(grad, present, what):
    """The gradient of a [c_dim, ...] weight read only through one-hot labels: nonzero in the rows of the classes present, exactly 0
    in the others (so it shows which labels the step used)."""
    rows = grad.reshape(grad.shape[0], -1).abs().amax(dim=1)
    assert {j for j in range(grad.shape[0]) if rows[j] > 0} == present, (what, rows.tolist())


def test_conditional_step_graphed_matches_eager(gf, cuda_dev):
    """step_graphed with labels against the eager step from the same state.  The graphed trainer's first call (eager warm-up,
    capture and replay of the step with R1) uses classes {0, 1, 4}; its weights and Adam states are then copied into an eager
    trainer, and both take the next step, without R1, with classes {2, 3}: the graphed one captures and replays that graph with the
    new labels in its static buffers.  Compared: the losses, and the gradients of fc1 and of the embedding that the step's Adam
    updates applied.  Weights are not compared: Adam's first steps move each element by about lr * sign(g), so round-off that flips
    the sign of a near-zero gradient element moves a weight by 2 lr.  The rows of both gradients also show which labels each
    step used: a class absent from the step's labels has an exactly zero row."""
    tr = import_module(TRAIN)
    z, reals, _, _ = _batch(cuda_dev)
    gen_c, real_c = _onehot([0, 1, 0, 4], cuda_dev), _onehot([1, 0, 4, 4], cuda_dev)
    gen_c2, real_c2 = _onehot([2, 3, 2, 3], cuda_dev), _onehot([3, 2, 2, 3], cuda_dev)
    cfg = dict(noise_mode="const", d_reg_interval=2)
    _, G, D = _gan(gf, cuda_dev)
    tg = tr.Trainer(G, D, tr.TrainConfig(**cfg))
    s1 = tg.step_graphed(z, reals, gen_c, real_c)
    assert s1.r1 > 0
    _assert_class_rows(G.mapping.embed.grad, {0, 1, 4}, "graphed step 1 embed")
    _assert_class_rows(D.fc1.weight.grad, {0, 1, 4}, "graphed step 1 fc1")
    _, Ge, De = _gan(gf, cuda_dev)
    te = tr.Trainer(Ge, De, tr.TrainConfig(**cfg))
    Ge.load_state_dict(G.state_dict())
    De.load_state_dict(D.state_dict())
    # a deep copy: Optimizer.load_state_dict keeps the given state tensors when their device and dtype already match, and the two
    # trainers would then advance one set of Adam moments and step counts twice
    te.opt_g.load_state_dict(copy.deepcopy(tg.opt_g.state_dict()))
    te.opt_d.load_state_dict(copy.deepcopy(tg.opt_d.state_dict()))
    te.it = tg.it
    sg = tg.step_graphed(z, reals, gen_c2, real_c2)
    se = te.step(z, reals, gen_c2, real_c2)
    assert sg.r1 == se.r1 == 0
    for what, v, w in (("loss_d", se.loss_d, sg.loss_d), ("loss_g", se.loss_g, sg.loss_g)):
        print(f"[conditional graphed] {what}: eager {v:.7f} graphed {w:.7f}")
        assert abs(v - w) <= 1e-3 * max(1.0, abs(v)), what
    for what, ge, gg in (("fc1.weight", De.fc1.weight.grad, D.fc1.weight.grad), ("fc1.bias", De.fc1.bias.grad, D.fc1.bias.grad),
                         ("mapping.embed", Ge.mapping.embed.grad, G.mapping.embed.grad)):
        _assert_class_rows(gg, {2, 3}, f"graphed step 2 {what}")
        _assert_class_rows(ge, {2, 3}, f"eager step 2 {what}")
        rel = ((gg - ge).norm() / ge.norm()).item()
        print(f"[conditional graphed] {what} gradient: |graphed - eager| / |eager| = {rel:.2e}")
        assert rel <= 1e-3, what


def test_host_labels_are_moved_to_the_device(gf, cuda_dev):
    """Labels on the host, as int64 or float64, with CUDA latents and images: the trainer, D and G move them to the device."""
    tr, G, D = _gan(gf, cuda_dev)
    z, reals, gen_c, real_c = _batch(cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", d_reg_interval=2))
    gc, rc = trainer._labels(z, reals, gen_c.cpu().long(), real_c.cpu().double())
    assert gc.device == rc.device == z.device and gc.dtype == rc.dtype == z.dtype
    assert torch.equal(gc, gen_c) and torch.equal(rc, real_c)
    with torch.no_grad():
        assert torch.allclose(D(reals, real_c.cpu()), D(reals, real_c), rtol=1e-6, atol=1e-6)
        assert torch.allclose(G(z, gen_c.cpu().long()), G(z, gen_c), rtol=1e-6, atol=1e-6)
    for st in (trainer.step(z, reals, gen_c.cpu(), real_c.cpu()), trainer.step_graphed(z, reals, gen_c.cpu(), real_c.cpu())):
        assert math.isfinite(st.loss_d) and math.isfinite(st.loss_g)
