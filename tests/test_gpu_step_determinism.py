"""The whole training step on an H100 (``pytest -m gpu``): reruns bit for bit, and the G phase under augmentation against fp64.

* Rerun determinism: two trainers built from one state (weights copied, Adam states deep-copied) take the same two steps, the first
  with R1 and the second without, each from the same CUDA RNG state, at lr = 0 and with cuDNN pinned to its deterministic
  algorithms.  The losses, R1, p and every parameter gradient of G and D must be the same bits on both.  ``zero_grad(set_to_none)``
  runs at the start of each phase, so after a step D holds the D phase's gradients and G the G phase's.  The configurations:
  plain D without augmentation (the control), ``Discriminator(transformer=True)`` with no augmentation, "bc", "bgc" and "bgcfn",
  "bc" with labels, "bc" with ``r1_kernels`` and "bc" with img2img in both networks.
* The G phase against fp64: one eager step with the augmentation samplers recorded (tests/step_phase_ref.py), with "bc", "bgc",
  "bgcfn" and "bc" with labels; the G loss and the gradients of a spread of G parameters are rebuilt in fp64 on the CPU from the
  state dicts (tests/conditional_ref.py's generator and discriminator, ops.augment_ref and ops.augment_filter_ref with the G phase's
  draws).  The gradients flow back through D's duplex kernel backward (dX), the augmentation's adjoints and G's training path.
"""
import contextlib
import copy
from importlib import import_module

import pytest
import torch

from tests import conditional_ref as cref
from tests import step_phase_ref as step_ref

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"

# (Discriminator options, TrainConfig.augment, c_dim); img2img, when a case has it, goes to both networks
RERUN_CASES = {
    "plain-d": (dict(transformer=False), "", 0),
    "attention-d": (dict(transformer=True), "", 0),
    "bc": (dict(transformer=True), "bc", 0),
    "bgc": (dict(transformer=True), "bgc", 0),
    "bgcfn": (dict(transformer=True), "bgcfn", 0),
    "bc-labels": (dict(transformer=True), "bc", 5),
    "bc-r1-kernels": (dict(transformer=True, r1_kernels=True), "bc", 0),
    "img2img-bc": (dict(transformer=True, img2img=16), "bc", 0),
}

# The G phase against fp64: relative errors (2-norm of the difference over the 2-norm of the fp64 value).  Measured on an H100 80GB
# HBM3 at a 700 W power limit: the loss 2.7e-6 ("bc") and 7.6e-7 ("bgc"); the gradients at most 3.7e-4 ("bc", wq; the others 2.1e-4
# to 3.4e-4) and 3.8e-5 ("bgc").  Frozen at about 1.6x the worst.
TOL_LOSS_G = 5e-6
TOL_GRAD = 6e-4
# (TrainConfig.augment, c_dim, CUDA seed of the step, bound on the loss, bound on the gradients).  Seed 7's draws put D where fp32
# itself keeps few digits under "bgcfn" (an fp32 restatement of the definition 2.8e-3 off fp64 on the gradients) and with labels
# (7.5e-2).  Those two cases take a seed whose draws the restatement resolves, found by a sweep of seeds 1-12 on the H100 (DESIGN
# section 4.11), with bounds frozen at about 2x the larger of the kernels' and the restatement's error there: "bgcfn" at seed 5,
# kernels 1.7e-6 (loss) and 3.7e-5 (gradients), restatement 6.6e-7 and 1.3e-5; labels at seed 8, kernels 5.9e-7 and 7.6e-5,
# restatement 2.8e-8 and 1.4e-4.
G_PHASE_CASES = {
    "bc": ("bc", 0, 7, TOL_LOSS_G, TOL_GRAD),
    "bgc": ("bgc", 0, 7, TOL_LOSS_G, TOL_GRAD),
    "bgcfn": ("bgcfn", 0, 5, 3.4e-6, 7.5e-5),
    "bc-labels": ("bc", 5, 8, 1.2e-6, 3e-4),
}
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
    """The 64x64 pair of tests/test_gpu_augment.py (exact_fp32), with the discriminator's options dkw (an img2img there is given to
    the generator too)."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, exact_fp32=True,
                     c_dim=c_dim, img2img=dkw.get("img2img", 0)).to(dev)
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


def g_phase_errors(gf, dev, augment, c_dim, seed, monkeypatch):
    """One eager step with Discriminator(transformer=True) at lr = 0, so that D after its update is still D0, and the generator's
    tRGB weights scaled by TORGB_SCALE, from CUDA seed ``seed``.  The samplers record their draws (tests/step_phase_ref.StepRecorder);
    the G phase's are the last.  Returns the relative errors of the G loss and of the gradients of G_GRADS against fp64 autograd
    of the reference (labels gen_c on both networks), and those of the same definition restated in fp32 on the same draws."""
    tr, G, D = _gan(gf, dev, dict(transformer=True), c_dim)
    with torch.no_grad():
        for t in G.synthesis.torgbs:
            t.weight.mul_(TORGB_SCALE)
    filtered = bool(set(tr.parse_augment(augment)) & set(tr.FILTER_OPS))
    rec = step_ref.StepRecorder(tr, monkeypatch, filtered)
    trainer = tr.Trainer(G, D, tr.TrainConfig(lr=0.0, noise_mode="const", r1_gamma=0.0, augment=augment, augment_p=0.8))
    z, reals, gen_c, real_c = _batch(dev, c_dim=c_dim)
    sd_g, sd_d = cref.cast(G.state_dict()), cref.cast(D.state_dict())
    torch.cuda.manual_seed(seed)
    with _deterministic_cudnn():
        st = trainer.step(z, reals, gen_c, real_c)
    draw = rec.draws(0, 1)["fakes_g"]                                 # after the D phase's reals and fakes
    assert (draw[2] is not None) == (augment != "bc") and (draw[3] is not None) == filtered
    res = {}
    for dt in (torch.float64, torch.float32):                          # fp64, and the same definition restated in fp32
        sd = cref.cast(sd_g, dt)
        for n in G_GRADS:
            sd[n].requires_grad_(True)
        c = None if gen_c is None else gen_c.to("cpu", dt)
        img = cref.generator_forward(sd, z.to("cpu", dt), c, resolution=64, components_num=8, latent_dim=32, mapping_layers=4)
        logits = cref.discriminator_forward(cref.cast(sd_d, dt), step_ref.augment64(img, draw), c, dtype=dt)
        loss = torch.nn.functional.softplus(-logits).mean()
        res[dt] = (loss.item(), torch.autograd.grad(loss, [sd[n] for n in G_GRADS]))
    loss64, grads64 = res[torch.float64]
    params = dict(G.named_parameters())
    e_loss, r_loss = (abs(v - loss64) / abs(loss64) for v in (st.loss_g, res[torch.float32][0]))
    errs, restated = {}, {}
    for n, want, w32 in zip(G_GRADS, grads64, res[torch.float32][1]):
        assert want.norm() > 0, n
        errs[n], restated[n] = step_ref.rel(params[n].grad, want), step_ref.rel(w32, want)
    print(f"[G phase {augment} c_dim={c_dim} seed={seed}] loss_g {st.loss_g:.8f} vs {loss64:.8f}: rel {e_loss:.2e} (fp32 "
          f"restatement {r_loss:.2e}); gradients " + " ".join(f"{n}={e:.2e}" for n, e in errs.items())
          + f"; max {max(errs.values()):.2e} (fp32 restatement {max(restated.values()):.2e})")
    return e_loss, r_loss, errs, restated


@pytest.mark.parametrize("case", list(G_PHASE_CASES))
def test_g_phase_against_fp64(gf, cuda_dev, case, monkeypatch):
    """The G loss and the gradients of G_GRADS against fp64 under frozen bounds, on draws that fp32 itself resolves: the fp32
    restatement on the same draws must stay within the case's bounds too, so that the bounds measure the step and not the draw."""
    augment, c_dim, seed, tol_loss, tol_grad = G_PHASE_CASES[case]
    e_loss, r_loss, errs, restated = g_phase_errors(gf, cuda_dev, augment, c_dim, seed, monkeypatch)
    assert r_loss < tol_loss and max(restated.values()) < tol_grad, (r_loss, restated)
    assert e_loss < tol_loss, e_loss
    assert max(errs.values()) < tol_grad, errs
