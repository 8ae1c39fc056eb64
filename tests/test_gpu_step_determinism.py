"""The whole training step on an H100 (``pytest -m gpu``): reruns bit for bit, and the G phase under augmentation against fp64.

* Rerun determinism: two trainers built from one state (weights copied, Adam states deep-copied) take the same two steps, the first
  with R1 and the second without, each from the same CUDA RNG state, at lr = 0 and with cuDNN pinned to its deterministic
  algorithms.  The losses, R1, p and every parameter gradient of G and D must be the same bits on both.  ``zero_grad(set_to_none)``
  runs at the start of each phase, so after a step D holds the D phase's gradients and G the G phase's.  The configurations:
  plain D without augmentation (the control), ``Discriminator(transformer=True)`` with no augmentation, "bc", "bgc" and "bgcfn",
  "bc" with labels and "bc" with ``r1_kernels``.
* The G phase against fp64: one eager step with the augmentation samplers recorded, with "bc" and "bgc"; the G loss and the
  gradients of a spread of G parameters are rebuilt in fp64 on the CPU from the state dicts (tests/conditional_ref.py's generator and discriminator,
  ops.augment_ref with the G phase's draws).  The gradients flow back through D's duplex kernel backward (dX), the augmentation's
  adjoint and G's training path.
"""
import contextlib
import copy
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"

# (Discriminator options, TrainConfig.augment, c_dim)
RERUN_CASES = {
    "plain-d": (dict(transformer=False), "", 0),
    "attention-d": (dict(transformer=True), "", 0),
    "bc": (dict(transformer=True), "bc", 0),
    "bgc": (dict(transformer=True), "bgc", 0),
    "bgcfn": (dict(transformer=True), "bgcfn", 0),
    "bc-labels": (dict(transformer=True), "bc", 5),
    "bc-r1-kernels": (dict(transformer=True, r1_kernels=True), "bc", 0),
}

# The G phase against fp64: relative errors (2-norm of the difference over the 2-norm of the fp64 value).  Measured on an H100 80GB
# HBM3 at a 700 W power limit: the loss 2.7e-6 ("bc") and 7.6e-7 ("bgc"); the gradients at most 3.7e-4 ("bc", wq; the others 2.1e-4
# to 3.4e-4) and 3.8e-5 ("bgc").  Frozen at about 1.6x the worst.
TOL_LOSS_G = 5e-6
TOL_GRAD = 6e-4
# The untrained generator's images (std 3.2, up to 16 in magnitude) put the attention discriminator where fp32 keeps no digit of
# the G phase: an all-fp32 restatement of the reference is 5e-2 off fp64 on the loss and 8x off on the gradients (condition number
# of the loss in the image about 1e5).  Scaling the tRGB weights by 0.3 brings the images to std 0.66, where that restatement agrees
# with fp64 to 8e-7 on the loss and 4e-4 on the gradients.
TORGB_SCALE = 0.3
G_GRADS = ("mapping.local.1.weight", "synthesis.layers.4.attention.wq", "synthesis.layers.4.attention.wk",
           "synthesis.layers.4.attention.wv", "synthesis.layers.4.attention.wo", "synthesis.layers.4.weight",
           "synthesis.layers.3.weight", "synthesis.torgbs.2.weight")


@contextlib.contextmanager
def _deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


def _gan(gf, dev, dkw, c_dim):
    """The 64x64 pair of tests/test_gpu_augment.py (exact_fp32), with the discriminator's options dkw."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, exact_fp32=True,
                     c_dim=c_dim).to(dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, components_num=8, latent_dim=32, exact_fp32=True, c_dim=c_dim,
                         **dkw).to(dev)
    return tr, G, D


def _batch(dev, B=4, c_dim=0, seed=5):
    """Latents, reals in [-1, 1] and, with c_dim, one-hot labels of the fakes and of the reals (tests/test_gpu_augment.py's batch)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 9, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    if not c_dim:
        return z, reals, None, None
    oh = lambda: torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev)
    return z, reals, oh(), oh()


def _config(augment, **kw):
    cfg = dict(lr=0.0, noise_mode="const", d_reg_interval=2, augment=augment, augment_p=0.5, **kw)
    if augment:
        cfg.update(ada_target=0.6, ada_interval=1, ada_kimg=0.2)
    return cfg


def _twin(gf, dev, dkw, augment, c_dim):
    """Two trainers in one state: the second gets the first's weights, a deep copy of its Adam states, its ADA state and step."""
    tr, G, D = _gan(gf, dev, dkw, c_dim)
    ta = tr.Trainer(G, D, tr.TrainConfig(**_config(augment)))
    _, G2, D2 = _gan(gf, dev, dkw, c_dim)
    tb = tr.Trainer(G2, D2, tr.TrainConfig(**_config(augment)))
    G2.load_state_dict(G.state_dict())
    D2.load_state_dict(D.state_dict())
    tb.opt_g.load_state_dict(copy.deepcopy(ta.opt_g.state_dict()))
    tb.opt_d.load_state_dict(copy.deepcopy(ta.opt_d.state_dict()))
    for a, b in ((tb.augment_p, ta.augment_p), (tb.ada_stats, ta.ada_stats), (tb.ada_steps, ta.ada_steps)):
        if a is not None:
            a.copy_(b)
    tb.it = ta.it
    return ta, tb


def differing_grads(ma, mb):
    """Names of the parameters of two modules of one architecture whose .grad are not the same bits (or not both None)."""
    bad = []
    for (n, p), (n2, q) in zip(ma.named_parameters(), mb.named_parameters()):
        assert n == n2
        if (p.grad is None) != (q.grad is None) or (p.grad is not None and not torch.equal(p.grad, q.grad)):
            bad.append(n)
    return bad


def assert_same_grads(ta, tb, what):
    for net, ma, mb in (("G", ta.G, tb.G), ("D", ta.D, tb.D)):
        assert any(p.grad is not None for p in ma.parameters()), (what, net)
        bad = differing_grads(ma, mb)
        assert not bad, f"{what}: {len(bad)} {net} gradients differ, first {bad[:6]}"


@pytest.mark.parametrize("case", list(RERUN_CASES))
def test_step_reruns_bit_for_bit(gf, cuda_dev, case):
    dkw, augment, c_dim = RERUN_CASES[case]
    z, reals, gen_c, real_c = _batch(cuda_dev, c_dim=c_dim)
    with _deterministic_cudnn():
        ta, tb = _twin(gf, cuda_dev, dkw, augment, c_dim)
        for i in range(2):                              # it = 0: the R1 step (d_reg_interval = 2); it = 1: a plain step
            torch.cuda.manual_seed(500 + i)
            sa = ta.step(z, reals, gen_c, real_c)
            torch.cuda.manual_seed(500 + i)
            sb = tb.step(z, reals, gen_c, real_c)
            print(f"[rerun {case}] step {i}: loss_d {sa.loss_d!r} / {sb.loss_d!r}, loss_g {sa.loss_g!r} / {sb.loss_g!r}, "
                  f"r1 {sa.r1!r} / {sb.r1!r}, p {sa.augment_p!r} / {sb.augment_p!r}")
            assert (sa.r1 > 0) == (i == 0)
            for what in ("loss_d", "loss_g", "r1", "augment_p"):
                assert getattr(sa, what) == getattr(sb, what), (case, i, what)
            assert_same_grads(ta, tb, f"{case} step {i}")


@pytest.mark.parametrize("augment", ["bc", "bgc"])
def test_g_phase_against_fp64(gf, cuda_dev, augment, monkeypatch):
    """One eager step with Discriminator(transformer=True) at lr = 0, so that D after its update is still D0, and the generator's
    tRGB weights scaled by TORGB_SCALE.  The samplers record their draws; the G phase's are the last.  The G loss and the gradients
    of G_GRADS against fp64 autograd of the reference."""
    ops = import_module(OPS)
    tr, G, D = _gan(gf, cuda_dev, dict(transformer=True), 0)
    with torch.no_grad():
        for t in G.synthesis.torgbs:
            t.weight.mul_(TORGB_SCALE)
    draws = {"sample_augment": [], "sample_augment_frac": []}
    for name, seen in draws.items():
        fn = getattr(tr, name)
        monkeypatch.setattr(tr, name, lambda *a, _fn=fn, _seen=seen, **k: _seen.append(_fn(*a, **k)) or _seen[-1])
    trainer = tr.Trainer(G, D, tr.TrainConfig(lr=0.0, noise_mode="const", r1_gamma=0.0, augment=augment, augment_p=0.8))
    z, reals, _, _ = _batch(cuda_dev)
    sd_g, sd_d = cref.cast(G.state_dict()), cref.cast(D.state_dict())
    torch.cuda.manual_seed(7)
    with _deterministic_cudnn():
        st = trainer.step(z, reals)
    assert len(draws["sample_augment"]) == 3                          # the D phase's reals and fakes, the G phase's fakes
    geom, color = (t.cpu() for t in draws["sample_augment"][-1])
    frac = draws["sample_augment_frac"][-1]
    frac = None if frac is None else frac.cpu()
    assert (frac is not None) == (augment == "bgc")
    for n in G_GRADS:
        sd_g[n].requires_grad_(True)
    img = cref.generator_forward(sd_g, z.double().cpu(), None, resolution=64, components_num=8, latent_dim=32, mapping_layers=4)
    loss64 = torch.nn.functional.softplus(-cref.discriminator_forward(sd_d, ops.augment_ref(img, geom, color.double(), frac), None)).mean()
    grads64 = torch.autograd.grad(loss64, [sd_g[n] for n in G_GRADS])
    params = dict(G.named_parameters())
    e_loss = abs(st.loss_g - loss64.item()) / abs(loss64.item())
    errs = {}
    for n, want in zip(G_GRADS, grads64):
        assert want.norm() > 0, n
        errs[n] = ((params[n].grad.double().cpu() - want).norm() / want.norm()).item()
    print(f"[G phase {augment}] loss_g {st.loss_g:.8f} vs {loss64.item():.8f}: rel {e_loss:.2e}; gradients "
          + " ".join(f"{n}={e:.2e}" for n, e in errs.items()))
    assert e_loss < TOL_LOSS_G, e_loss
    assert max(errs.values()) < TOL_GRAD, errs
