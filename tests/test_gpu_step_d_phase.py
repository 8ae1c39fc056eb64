"""The training step's D phase on an H100 (``pytest -m gpu``) against its fp64 definition (tests/step_phase_ref.py).

Two eager steps per case at lr = 0 (so D and G stay at their initial weights), constant noise, cuDNN pinned and
``d_reg_interval = 2``: step 0 is the R1 step, where the reals' forward runs the torch composite (the double-backward kernels with
``r1_kernels``) because the reals require grad, and step 1 is a plain step, where both forwards run the CUDA attention forward and
the duplex kernel backward gives D's parameter gradients.  The fakes always take the kernel route.  The samplers and the D phase's
fakes are recorded; after each step the D loss, the R1 penalty, the ``.grad`` of every D parameter and the ADA accumulator are held
against ``d_phase64`` on the same fakes, cast to fp64 (the fakes are held against the fp64 generator on their own, so that G's
inference error does not enter the D phase's bounds).  The generator's tRGB weights are scaled by TORGB_SCALE first, as in
``test_g_phase_against_fp64``; tests/test_host_cpu_step_d_phase.py measures how many digits fp32 itself keeps on these inputs.
"""
import pytest
import torch

from tests import step_phase_ref as ref
from tests import test_gpu_step_determinism as sdet

pytestmark = pytest.mark.gpu

# (Discriminator options, TrainConfig.augment, c_dim)
CASES = {
    "attention-d": (dict(transformer=True), "", 0),
    "bc": (dict(transformer=True), "bc", 0),
    "bgc": (dict(transformer=True), "bgc", 0),
    "bgcfn": (dict(transformer=True), "bgcfn", 0),
    "bc-labels": (dict(transformer=True), "bc", 5),
    "bc-r1-kernels": (dict(transformer=True, r1_kernels=True), "bc", 0),
    "plain-d": (dict(transformer=False), "bgc", 0),
}
TORGB_SCALE = sdet.TORGB_SCALE

# Relative errors against fp64 (the loss and R1 as scalars, every gradient as a relative L2 norm), case by case: (loss, R1,
# gradients), frozen at about 2x the case's own worst over both steps as measured on an H100 80GB HBM3 at a 700 W power limit:
#   attention-d    5.2e-7  4.5e-7  6.0e-6        bgcfn          3.7e-6  4.2e-6  2.0e-4      plain-d  4.7e-8  1.0e-7  1.3e-4
#   bc             2.1e-6  2.8e-6  1.7e-4        bc-labels      1.7e-6  1.8e-6  1.9e-5
#   bgc            6.7e-5  8.6e-5  1.8e-3        bc-r1-kernels  1.4e-6  1.8e-6  1.7e-4
# "bgc" sits where an fp32 restatement of the same D phase is itself about 1e-3 off fp64 on the gradients (DESIGN section 4.11).
TOL = {
    "attention-d": (1.1e-6, 9e-7, 1.2e-5),
    "bc": (4.2e-6, 5.6e-6, 3.5e-4),
    "bgc": (1.4e-4, 1.7e-4, 3.6e-3),
    "bgcfn": (7.5e-6, 8.5e-6, 4.1e-4),
    "bc-labels": (3.4e-6, 3.7e-6, 3.8e-5),
    "bc-r1-kernels": (2.8e-6, 3.6e-6, 3.5e-4),
    "plain-d": (1e-7, 2e-7, 2.5e-4),
}
TOL_FAKES = 2.5e-6                          # measured 1.2e-6
# Gradients that are zero by structure (bk and bk2: a bias that is the same for every latent / every token cancels in its softmax),
# as a ratio of their 2-norm to the 2-norm of the same layer's bq / bq2 gradient: at most 2.5e-6 measured.
TOL_STRUCTURAL = 1e-5
LOGIT_MARGIN = 1e-4            # the smallest |real logit| in fp64, so that the signs the ADA accumulator sums are certain


def d_config(tr, augment):
    kw = dict(lr=0.0, noise_mode="const", d_reg_interval=2, augment=augment, augment_p=0.8)
    if augment:
        kw.update(ada_target=0.6, ada_interval=2)                 # step 0 accumulates, step 1 updates p and resets
    return tr.TrainConfig(**kw)


def filtered(tr, augment):
    return bool(set(tr.parse_augment(augment)) & set(tr.FILTER_OPS))


def grad_errors(D, want, *, bk2_exact):
    """Relative L2 errors of the .grad of every parameter of D against the fp64 gradients ``want``, and the ratios of the gradients
    that vanish by structure.  wk (the duplex layers' keys come from the centroids) has no gradient on either side; bk2 is exactly 0
    where every forward ran the kernel route (``bk2_exact``); bk and bk2 are otherwise at round-off."""
    errs, structural = {}, {}
    got = {n: p.grad for n, p in D.named_parameters()}
    assert set(got) == set(want)
    for n, w in want.items():
        g, leaf = got[n], n.rsplit(".", 1)[-1]
        if leaf == "wk":
            assert w is None and g is None, n
        elif leaf in ("bk", "bk2"):
            assert g is not None and w is not None, n
            if leaf == "bk2" and bk2_exact:
                assert torch.count_nonzero(g) == 0, n
            scale = want[n[:-len(leaf)] + leaf.replace("k", "q")].norm()
            assert w.norm() < 1e-9 * scale, n                 # zero in fp64, up to its round-off
            structural[n] = (g.double().cpu().norm() / scale).item()
        else:
            assert g is not None and w is not None and w.norm() > 0, n
            errs[n] = ref.rel(g, w)
    return errs, structural


@pytest.mark.parametrize("case", list(CASES))
def test_d_phase_against_fp64(gf, cuda_dev, case, monkeypatch):
    dkw, augment, c_dim = CASES[case]
    tr, G, D = sdet._gan(gf, cuda_dev, dkw, c_dim)
    with torch.no_grad():
        for t in G.synthesis.torgbs:
            t.weight.mul_(TORGB_SCALE)
    rec = ref.StepRecorder(tr, monkeypatch, filtered(tr, augment))
    cfg = d_config(tr, augment)
    trainer = tr.Trainer(G, D, cfg)
    z, reals, gen_c, real_c = sdet._batch(cuda_dev, c_dim=c_dim)
    sd_g = G.state_dict()
    sd_d = {n: p.detach().clone() for n, p in D.named_parameters()}
    fakes64 = ref.generator64(sd_g, z, gen_c)
    signs = []
    with sdet._deterministic_cudnn():
        for i in range(2):
            torch.cuda.manual_seed(500 + i)
            st = trainer.step(z, reals, gen_c, real_c)
            do_r1 = i == 0
            assert (st.r1 > 0) == do_r1
            fakes = rec.fakes[i]
            e_fakes = ref.rel(fakes, fakes64)
            want = ref.d_phase64(sd_d, reals, fakes, rec.draws(i, i + 1), gen_c, real_c, do_r1, cfg)
            errs, structural = grad_errors(D, want["grads"], bk2_exact=not do_r1)
            e_loss = abs(st.loss_d - want["loss"]) / abs(want["loss"])
            e_r1 = abs(st.r1 - want["r1"]) / want["r1"] if do_r1 else 0.0
            worst = max(errs, key=errs.get)
            print(f"[D phase {case}] step {i}: loss_d {st.loss_d:.8f} vs {want['loss']:.8f} rel {e_loss:.2e}; r1 {st.r1:.6e} vs "
                  f"{want['r1']:.6e} rel {e_r1:.2e}; gradients worst {worst} {errs[worst]:.2e} over {len(errs)}; structural "
                  + " ".join(f"{n}={v:.1e}" for n, v in structural.items() if v > 0)
                  + f" (max {max(structural.values(), default=0.0):.1e}); fakes {e_fakes:.2e}; "
                  f"min |logit_real| {want['logits_real'].abs().min().item():.3e}")
            tol_loss, tol_r1, tol_grad = TOL[case]
            assert e_fakes < TOL_FAKES, e_fakes
            assert e_loss < tol_loss, e_loss
            assert e_r1 < tol_r1, e_r1
            assert errs[worst] < tol_grad, (worst, errs[worst])
            assert max(structural.values(), default=0.0) < TOL_STRUCTURAL, structural
            assert (len(structural) > 0) == dkw["transformer"]
            if trainer.ada_stats is not None:
                check_ada(trainer, st, cfg, want["logits_real"], signs, i)


def check_ada(trainer, st, cfg, logits64, signs, i):
    """The ADA accumulator after step i of two (ada_interval = 2) against the signs of the fp64 real logits: after step 0 it holds
    exactly (sum of the signs, B); after step 1, p has moved by one increment towards the target from both steps' signs and the
    accumulator is reset.  ``signs`` collects the per-step sums."""
    assert cfg.ada_interval == 2
    B = logits64.numel()
    assert logits64.abs().min() > LOGIT_MARGIN, logits64
    signs.append(logits64.sign().sum().item())
    p0 = torch.tensor(cfg.augment_p, dtype=torch.float32)
    if i == 0:                                                  # accumulated, not yet reset
        assert trainer.ada_stats.tolist() == [signs[0], float(B)], (trainer.ada_stats, signs)
        assert st.augment_p == p0.item()
    else:                                                       # the update of p from both steps' signs, then the reset
        assert trainer.ada_stats.tolist() == [0.0, 0.0]
        inc = B * cfg.ada_interval / (cfg.ada_kimg * 1000.0)
        mean = torch.tensor(sum(signs) / (2 * B), dtype=torch.float32)
        p = (p0 + torch.sign(mean - cfg.ada_target) * inc).clamp(0.0, 1.0)
        assert st.augment_p == p.item() != p0.item(), (st.augment_p, p.item(), signs)
