"""The training step at a live learning rate on an H100 (``pytest -m gpu``): what the step does to the weights.

Every other trainer test on the GPU runs at lr = 0 or checks only that values are finite.  Here lr = 2e-3, with ``ema_kimg`` and
``w_avg_beta`` small enough that G_ema and w_avg move by a visible fraction each step, ``d_reg_interval = 2`` and
``g_reg_interval = 3``, so that six steps with path length take the four graph keys (R1 + pl, none, R1, pl, R1, none).  The pair is
the 64x64 exact-fp32 pair of tests/test_gpu_step_determinism.py, with cuDNN pinned to its deterministic algorithms.

* Graphed from its first call: ``step_graphed`` against ``step`` from one state, bit for bit after every step (every StepStats
  field, every G, D and G_ema parameter and buffer, every Adam state tensor, pl_mean, p and the dropout state).  The first call
  runs the step eagerly once per graph key before it captures; those runs must leave no trace.
* Every update against its definition (tests/step_phase_ref.py): each Adam step of D and G restated in fp64 from its recorded
  gradients and state, with the lazy rescaling of lr and both betas; G steps twice on a path-length step; G_ema is the lerp towards
  G after the step and its buffers are G's; w_avg is the lerp towards the fp64 mapping's means on G's weights after the G updates.
* Each phase sees the current weights: the D phase's fakes against fp64 G on its state after the previous step, the D loss and
  gradients against fp64 on D's state at the start of the step, the G loss against fp64 on D after this step's D update, and G_ema
  inference (truncation 0.7, eager and through ``G_ema.graphed``) against fp64 after eager and after graphed steps.
* The path-length phase against fp64 on its recorded state, noise draw and dropout masks: the lengths, the penalty, pl_mean and
  every gradient it leaves on G; the simplex route with dropout, a duplex generator with dropout, and labels.
"""
import contextlib
import copy
import dataclasses
from importlib import import_module

import pytest
import torch

from oracle import philox as ph
from tests import conditional_ref as cref
from tests import step_phase_ref as ref
from tests import test_gpu_step_d_phase as gd
from tests import test_gpu_step_determinism as sdet

pytestmark = pytest.mark.gpu

TRAIN = "gansformer-reproducibility-challenge_b200.training"
ATT = "gansformer-reproducibility-challenge_b200.attention"
LIVE = dict(lr=2e-3, ema_kimg=0.01, w_avg_beta=0.5, d_reg_interval=2, g_reg_interval=3, noise_mode="const")
STEPS = 6
# (Discriminator options, Generator options, TrainConfig options, c_dim)
CASES = {
    "attention-d-pl": (dict(transformer=True), dict(att_dp=0.12), dict(pl_weight=2.0), 0),
    "attention-d-pl-no-dropout": (dict(transformer=True), {}, dict(pl_weight=2.0), 0),
    "bc-labels": (dict(transformer=True), {}, dict(augment="bc", augment_p=0.5, ada_target=0.6, ada_interval=1, ada_kimg=0.2), 5),
    "mixing-random": (dict(transformer=True), {}, dict(style_mixing=0.9, noise_mode="random"), 0),
}

# Bounds, frozen at about 2x the worst value measured on an H100 80GB HBM3 at a 700 W power limit (measured values beside).
TOL_ADAM = 5e-6          # an update's error beyond storing p' in fp32, over the update, element-wise (2.1e-6)
TOL_ADAM_STATE = 2.5e-7  # m' and v', relative L2 (1.2e-7)
TOL_LERP = 6e-6          # G_ema and w_avg: |got - lerp| beyond one ulp, over the move, L2 (G_ema 4.5e-8, w_avg 2.8e-6)
TOL_FAKES = 2.5e-6       # the D phase's fakes against fp64 G on its state after the previous step (1.2e-6)
TOL_EMA = 2.5e-6         # G_ema(z, truncation_psi=0.7), eager and graphed, against fp64 (1.0e-6)
TOL_D = {"attention-d": (1.2e-6, 1e-6, 1.2e-3),     # D loss, R1, D gradients: (5.2e-7, 4.5e-7, 5.5e-4 blocks.1.att0.wpq)
         "bc-labels": (4e-6, 3e-6, 3e-4)}           # (1.8e-6, 1.5e-6, 1.5e-4 blocks.0.att0.wkc)
TOL_LOSS_G = 5e-6        # (2.2e-6)
# The path-length phase, worst over both calls of each case: the lengths 3.0e-5 (simplex-dropout), the penalty 4.9e-5 and pl_mean
# 1.2e-5; G's gradients 1.2e-3 simplex-dropout (synthesis.layers.8.weight), 1.2e-5 duplex-dropout, 3.7e-4 labels; the structural
# zeros 3.0e-7 of the largest gradient.
TOL_PL_LENGTHS = 6e-5
TOL_PL = 1e-4            # penalty and pl_mean
TOL_PL_GRAD = {"simplex-dropout": 2.5e-3, "duplex-dropout": 2.5e-5, "labels": 8e-4}
TOL_PL_STRUCTURAL = 6e-7
# Parameters without a gradient of the penalty, or with one that is zero by structure: the tRGB biases (an image offset), and per
# attention layer the key bias (constant over what a softmax normalises) and, in duplex layers, the keys and the biases of pass A's
# keys and values (the keys come from the centroids)
PL_NO_GRAD = ("wk", "bk", "bk2", "bv2")


@contextlib.contextmanager
def _pinned():
    with sdet._deterministic_cudnn():
        yield


def _gan(gf, dev, dkw, gkw, c_dim, live_terms=False):
    """The 64x64 exact-fp32 pair, with generator options gkw; ``live_terms`` moves the biases and noise strengths away from zero
    (tests/test_gpu_generator_path_length.py), so that every term of the path-length penalty is live.  A layer's dropout salt
    comes from a process-wide counter: each pair gets the same salts here, so that two pairs built alike draw the same masks, and
    so does every run of a case whichever tests ran before it."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, exact_fp32=True,
                     c_dim=c_dim, **gkw).to(dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128, components_num=8, latent_dim=32, exact_fp32=True, c_dim=c_dim,
                         **dkw).to(dev)
    for i, m in enumerate(m for m in (*G.modules(), *D.modules()) if hasattr(m, "dp_salt")):
        m.dp_salt = (i + 1) * 0x9E3779B1 & 0xFFFFFFFF     # the library's salts, counted from this pair, whatever was built before
    if live_terms:
        g = torch.Generator().manual_seed(1)
        with torch.no_grad():
            for n, p in G.named_parameters():
                if n.endswith("noise_strength") or n.split(".")[-1].startswith("b"):
                    p.copy_(0.2 * torch.randn(p.shape, generator=g))
    return tr, G, D


def _trainer(gf, dev, case, torgb_scale=1.0):
    dkw, gkw, ckw, c_dim = CASES[case] if isinstance(case, str) else case
    tr, G, D = _gan(gf, dev, dkw, gkw, c_dim)
    if torgb_scale != 1.0:
        with torch.no_grad():
            for t in G.synthesis.torgbs:
                t.weight.mul_(torgb_scale)
    return tr, tr.Trainer(G, D, tr.TrainConfig(**{**LIVE, **ckw})), c_dim


def _state(t):
    """Everything a step writes, by name, as a flat dict of tensors (Adam states by parameter name)."""
    am = import_module(ATT)
    out = _state_cpu(t)
    out["dropout"] = am.dropout_state(next(t.G.parameters()).device).clone()
    return out


def _state_cpu(t):
    """_state without the attention-dropout state, which only a CUDA device has."""
    out = {}
    for net, m in (("G", t.G), ("D", t.D), ("G_ema", t.G_ema)):
        for n, v in (*m.named_parameters(), *m.named_buffers()):
            out[f"{net}.{n}"] = v
    for net, opt, m in (("G", t.opt_g, t.G), ("D", t.opt_d, t.D)):
        for n, p in m.named_parameters():
            for k, v in opt.state.get(p, {}).items():
                out[f"adam.{net}.{n}.{k}"] = v
    for n in ("pl_mean", "augment_p", "ada_stats", "ada_steps"):
        if getattr(t, n) is not None:
            out[n] = getattr(t, n)
    return {n: v.detach().clone() for n, v in out.items()}


def _differing(a, b):
    assert set(a) == set(b), sorted(set(a) ^ set(b))[:6]
    return [n for n in a if not torch.equal(a[n], b[n])]


@pytest.mark.parametrize("case", list(CASES))
def test_graphed_from_first_call_matches_eager(gf, cuda_dev, case):
    """Two trainers from one state, one eager and one graphed, the graphed one from its very first call: after each of six steps
    the same StepStats and the same bits in everything the step writes."""
    am = import_module(ATT)
    _, te, c_dim = _trainer(gf, cuda_dev, case)
    _, tg, _ = _trainer(gf, cuda_dev, case)
    z, reals, gen_c, real_c = sdet._batch(cuda_dev, c_dim=c_dim)
    keys = []
    with _pinned():
        for i in range(STEPS):
            out = []
            for t, fn in ((te, te.step), (tg, tg.step_graphed)):
                torch.cuda.manual_seed(900 + i)
                am.set_dropout_seed(4321, cuda_dev, 10 * i)
                st = fn(z, reals, gen_c, real_c)
                out.append((dataclasses.asdict(st), _state(t)))
            (se, ae), (sg, ag) = out
            keys.append((se["r1"] > 0, se["pl_penalty"] > 0))
            print(f"[graphed {case}] step {i}: loss_d {se['loss_d']!r} / {sg['loss_d']!r}, loss_g {se['loss_g']!r} / "
                  f"{sg['loss_g']!r}, r1 {se['r1']!r} / {sg['r1']!r}, pl {se['pl_penalty']!r} / {sg['pl_penalty']!r}")
            assert se == sg, (case, i, {k: (se[k], sg[k]) for k in se if se[k] != sg[k]})
            bad = _differing(ae, ag)
            assert not bad, f"{case} step {i}: {len(bad)} tensors differ, first {bad[:6]}"
    if te.cfg.pl_weight > 0:
        assert keys == [(True, True), (False, False), (True, False), (False, True), (True, False), (False, False)], keys


def check_step_updates(t, st, i, d_calls, g_calls, ema0, w_avg0, z, gen_c, worst):
    """The updates of step i against their definitions: one D Adam step and one G Adam step (two on a path-length step), each
    against fp64 Adam with the lazy rescaling (G's only with pl_weight > 0); G_ema against the lerp from its state before the step
    (ema0) towards G after it, and its buffers against G's; w_avg against the lerp from w_avg0 towards the means of the fp64 mapping on
    G's weights after the step.  Accumulates the worst errors into ``worst``."""
    cfg = t.cfg
    do_pl = st.pl_penalty > 0
    assert do_pl == (cfg.pl_weight > 0 and i % cfg.g_reg_interval == 0)
    assert len(d_calls) == 1 and len(g_calls) == 1 + do_pl, (i, len(d_calls), len(g_calls))
    d_adam = ref.lazy_adam(cfg, cfg.d_reg_interval)
    g_adam = ref.lazy_adam(cfg, cfg.g_reg_interval if cfg.pl_weight > 0 else None)
    n_g, n_d = sum(1 for _ in t.G.parameters()), sum(1 for _ in t.D.parameters())
    for calls, hyper, n in ((d_calls, d_adam, n_d), (g_calls, g_adam, n_g)):
        for call in calls:
            e = ref.adam_errors(call, *hyper)
            assert e["steps"] == 0 and e["count"] >= n - len(t.G.synthesis.torgbs) - t.G.synthesis.num_attention_layers, (i, e, n)
            worst["adam"], worst["state"] = max(worst["adam"], e["update"]), max(worst["state"], e["state"])
    beta = 0.5 ** (z.shape[0] * t.world / (cfg.ema_kimg * 1000.0))
    for pe0, pe, p in zip(ema0, t.G_ema.parameters(), t.G.parameters()):
        if not torch.equal(p, pe0):
            worst["ema"] = max(worst["ema"], ref.lerp_error(pe0, p, 1.0 - beta, pe))
    for (n, be), b in zip(t.G_ema.named_buffers(), t.G.buffers()):
        assert torch.equal(be, b), n
    c = None if gen_c is None else gen_c.double().cpu()
    ws = cref.mapping_forward(cref.cast(t.G.state_dict()), z.double().cpu(), c, components_num=8, latent_dim=32, mapping_layers=4)
    cur = torch.stack([ws[:, :8].mean(dim=(0, 1)), ws[:, 8:].mean(dim=(0, 1))])
    worst["w_avg"] = max(worst["w_avg"], ref.lerp_error(w_avg0, cur, 1.0 - cfg.w_avg_beta, t.G.mapping.w_avg))


@pytest.mark.parametrize("case", ["attention-d-pl", "bc-labels", "mixing-random"])
def test_updates_against_their_definitions(gf, cuda_dev, case, monkeypatch):
    """Six eager steps with every Adam step recorded: each against Adam in fp64 with the lazy rescaling (G's only with
    pl_weight > 0), two G steps on a path-length step, G_ema and its buffers, and w_avg against the fp64 mapping."""
    am = import_module(ATT)
    _, t, c_dim = _trainer(gf, cuda_dev, case)
    cfg = t.cfg
    rd, rg = ref.OptRecorder(t.opt_d, monkeypatch), ref.OptRecorder(t.opt_g, monkeypatch)
    z, reals, gen_c, real_c = sdet._batch(cuda_dev, c_dim=c_dim)
    worst = dict(adam=0.0, state=0.0, ema=0.0, w_avg=0.0)
    with _pinned():
        for i in range(STEPS):
            ema0 = [p.detach().clone() for p in t.G_ema.parameters()]
            w_avg0 = t.G.mapping.w_avg.detach().clone()
            nd, ng = len(rd.calls), len(rg.calls)
            torch.cuda.manual_seed(900 + i)
            am.set_dropout_seed(4321, cuda_dev, 10 * i)
            st = t.step(z, reals, gen_c, real_c)
            check_step_updates(t, st, i, rd.calls[nd:], rg.calls[ng:], ema0, w_avg0, z, gen_c, worst)
    print(f"[updates {case}] worst: Adam update {worst['adam']:.2e}, state {worst['state']:.2e}; G_ema {worst['ema']:.2e}; "
          f"w_avg {worst['w_avg']:.2e}")
    assert worst["adam"] < TOL_ADAM and worst["state"] < TOL_ADAM_STATE, worst
    assert worst["ema"] < TOL_LERP and worst["w_avg"] < TOL_LERP, worst


def _g_ema_errors(t, z, gen_c):
    """G_ema(z, truncation_psi=0.7), eager and through G_ema.graphed, against fp64 on G_ema's state dict."""
    want = cref.generator_forward(cref.cast(t.G_ema.state_dict()), z.double().cpu(),
                                  None if gen_c is None else gen_c.double().cpu(), resolution=64, components_num=8,
                                  latent_dim=32, mapping_layers=4, truncation_psi=0.7)
    with torch.no_grad():
        eager = t.G_ema(z, gen_c, truncation_psi=0.7).clone()
    graphed = t.G_ema.graphed(z.shape[0], truncation_psi=0.7)(z, gen_c).clone()
    return ref.rel(eager, want), ref.rel(graphed, want)


PHASE_CASES = {
    "attention-d": ((dict(transformer=True), {}, {}, 0), ""),
    "bc-labels": ((dict(transformer=True), {}, dict(augment="bc", augment_p=0.8), 5), "bc"),
}


@pytest.mark.parametrize("case", list(PHASE_CASES))
def test_phases_see_current_weights(gf, cuda_dev, case, monkeypatch):
    """Three eager steps (R1, plain, R1), each phase against fp64 on the weights it must see; then G_ema inference after them, and
    after each of three graphed steps of a second trainer from the same state (a replay moves the weights behind their version
    counters: only the weights epoch tells G_ema's caches and captured forward that they are stale)."""
    spec, augment = PHASE_CASES[case]
    tr, t, c_dim = _trainer(gf, cuda_dev, spec, torgb_scale=sdet.TORGB_SCALE)
    _, tg, _ = _trainer(gf, cuda_dev, spec, torgb_scale=sdet.TORGB_SCALE)
    cfg = t.cfg
    rec = ref.StepRecorder(tr, monkeypatch, False)
    z, reals, gen_c, real_c = sdet._batch(cuda_dev, c_dim=c_dim)
    tol_loss, tol_r1, tol_grad = TOL_D[case]
    with _pinned():
        for i in range(3):
            sd_g = {n: v.detach().clone() for n, v in t.G.state_dict().items()}
            sd_d = {n: p.detach().clone() for n, p in t.D.named_parameters()}
            torch.cuda.manual_seed(900 + i)
            st = t.step(z, reals, gen_c, real_c)
            do_r1 = i % cfg.d_reg_interval == 0
            fakes64 = ref.generator64(sd_g, z, gen_c)
            e_fakes = ref.rel(rec.fakes[i], fakes64)
            draws = rec.draws(i, i + 1)
            want = ref.d_phase64(sd_d, reals, rec.fakes[i], draws, gen_c, real_c, do_r1, cfg)
            errs, structural = gd.grad_errors(t.D, want["grads"], bk2_exact=not do_r1)
            e_loss = abs(st.loss_d - want["loss"]) / abs(want["loss"])
            e_r1 = abs(st.r1 - want["r1"]) / want["r1"] if do_r1 else 0.0
            worst = max(errs, key=errs.get)
            line = (f"[phases {case}] step {i}: fakes {e_fakes:.2e}; loss_d {e_loss:.2e} r1 {e_r1:.2e} D gradients {errs[worst]:.2e} "
                    f"({worst}) structural {max(structural.values(), default=0.0):.1e}")
            e_g = 0.0
            if not augment:                              # G phase: G as at the start of the step, D after this step's D update
                logits = cref.discriminator_forward(cref.cast(dict(t.D.named_parameters())), fakes64, None, dtype=torch.float64)
                loss64 = torch.nn.functional.softplus(-logits).mean().item()
                e_g = abs(st.loss_g - loss64) / abs(loss64)
                line += f"; loss_g {e_g:.2e}"
            print(line)
            assert e_fakes < TOL_FAKES and e_loss < tol_loss and e_r1 < tol_r1, (e_fakes, e_loss, e_r1)
            assert errs[worst] < tol_grad, (worst, errs[worst])
            assert max(structural.values(), default=0.0) < gd.TOL_STRUCTURAL, structural
            assert e_g < TOL_LOSS_G, e_g
        e_eager = _g_ema_errors(t, z, gen_c)
        e_graphed = (0.0, 0.0)
        for i in range(3):                               # after each replay, G_ema's caches and graph from the step before are stale
            torch.cuda.manual_seed(900 + i)
            tg.step_graphed(z, reals, gen_c, real_c)
            e_graphed = tuple(map(max, e_graphed, _g_ema_errors(tg, z, gen_c)))
    print(f"[phases {case}] G_ema(truncation 0.7) after eager steps {e_eager[0]:.2e} (graphed inference {e_eager[1]:.2e}), after "
          f"graphed steps {e_graphed[0]:.2e} ({e_graphed[1]:.2e})")
    assert max(*e_eager, *e_graphed) < TOL_EMA, (e_eager, e_graphed)


# (Generator options, c_dim): B = 5 with pl_batch_shrink 2, so that the phase runs on B' = 2
PL_CASES = {
    "simplex-dropout": (dict(att_dp=0.12), 0),
    "duplex-dropout": (dict(att_dp=0.12, kmeans=True), 0),
    "labels": ({}, 5),
}


def _masks(G, att_dp, dp, nb):
    """The dropout multipliers [B', n, k] of every attention layer of G for the dropout state dp = (seed, step) the kernels read."""
    out = []
    for layer in G.synthesis.layers:
        if layer.attention is not None:
            n = layer.resolution ** 2
            out.append(torch.from_numpy(ph.dropout_mult(att_dp, dp[0], dp[1], layer.attention.dp_salt, nb * n, 16)
                                        .reshape(nb, n, 16)[:, :, :8].copy()))
    return out


@pytest.mark.parametrize("case", list(PL_CASES))
def test_pl_phase_against_fp64(gf, cuda_dev, case, monkeypatch):
    """Three eager steps at g_reg_interval = 2 (path length at steps 0 and 2, so that the second lerp starts from a nonzero mean),
    each path-length phase against pl_phase64 on its recorded state, noise and masks, with the leaky-ReLU slopes of the GPU forward
    on that state."""
    gkw, c_dim = PL_CASES[case]
    am = import_module(ATT)
    tr, G, D = _gan(gf, cuda_dev, dict(transformer=False), gkw, c_dim, live_terms=True)
    G_probe = copy.deepcopy(G).train()
    cfg = tr.TrainConfig(**{**LIVE, "g_reg_interval": 2, "pl_weight": 2.0})
    t = tr.Trainer(G, D, cfg)
    rec = ref.PlRecorder(tr, monkeypatch)
    z, reals, gen_c, real_c = sdet._batch(cuda_dev, B=5, c_dim=c_dim)
    means = []
    with _pinned():
        for i in range(3):
            torch.cuda.manual_seed(900 + i)
            am.set_dropout_seed(2468, cuda_dev, 10 * i)
            st = t.step(z, reals, gen_c, real_c)
            if i % cfg.g_reg_interval == 0:
                means.append(st.pl_mean)
    assert len(rec.calls) == 2 and rec.calls[0]["pl_mean"] == 0.0 and rec.calls[1]["pl_mean"] == means[0] > 0
    for j, r in enumerate(rec.calls):
        check_pl_call(r, means[j], G_probe, z, gen_c, cfg, gkw.get("att_dp", 0.0), bool(gkw.get("kmeans")), f"{case} call {j}",
                      (TOL_PL_LENGTHS, TOL_PL, TOL_PL_GRAD[case], TOL_PL_STRUCTURAL))


def check_pl_call(r, pl_mean, G_probe, z, gen_c, cfg, att_dp, duplex, what, tols):
    """One recorded path-length phase (step_phase_ref.PlRecorder) against pl_phase64: the lengths, the penalty, pl_mean after the
    phase and G's gradients.  Every synthesis layer's leaky-ReLU slopes are those G_probe's forward took on the recorded state and,
    on the GPU, the dropout state the phase's kernels read (unfused, as ``return_features`` runs it: one output per layer).  Taking
    them from fp64 instead can flip the slope of a pre-activation that lies within fp32 round-off of zero, and one such flip in the
    4x4 layer, which has no attention, can move the lengths by about one part in its 4096 activations.  tols: (lengths, penalty and
    pl_mean, gradients, structural)."""
    nb = z.shape[0] // cfg.pl_batch_shrink
    G_probe.load_state_dict(r["sd"])
    dp = None
    if r["dp"] is not None:
        am = import_module(ATT)
        dp = (r["dp"][0], r["dp"][1] + 1)                # the phase advances the dropout step before its forward
        am.set_dropout_seed(dp[0], z.device, dp[1])
    c = None if gen_c is None else gen_c[:nb]
    pos = []
    hooks = [layer.register_forward_hook(lambda m, a, out: pos.append(out[0].detach().cpu() > 0)) for layer in G_probe.synthesis.layers]
    try:
        with torch.no_grad():
            G_probe.synthesis(G_probe.mapping(z[:nb], c), noise_mode="const", return_features=True)
    finally:
        for h in hooks:
            h.remove()
    assert len(pos) == len(G_probe.synthesis.layers)
    want = ref.pl_phase64(r, z, gen_c, cfg, att_mults=_masks(G_probe, att_dp, dp, nb) if att_dp else None, layer_pos=pos,
                          duplex=duplex)
    e_len = ref.rel(ref.pl_lengths(r["pl_grads"]), want["lengths"])
    e_pen = abs(r["penalty"] - want["penalty"]) / want["penalty"]
    e_mean = abs(pl_mean - want["pl_mean"]) / want["pl_mean"]
    errs, structural = ref.pl_grad_errors(r["grads"], want["grads"])
    worst = sorted(errs, key=errs.get, reverse=True)
    print(f"[pl phase {what}] lengths {e_len:.2e} penalty {e_pen:.2e} pl_mean {e_mean:.2e} ({pl_mean:.6f}); {len(errs)} gradients, "
          "worst " + " ".join(f"{n}={errs[n]:.1e}" for n in worst[:4]) + f"; structural {max(structural.values(), default=0.0):.1e}")
    tol_len, tol, tol_grad, tol_structural = tols
    assert e_len < tol_len and e_pen < tol and e_mean < tol, (what, e_len, e_pen, e_mean)
    others = [n for n in r["grads"] if n not in errs]
    assert all((n.startswith("synthesis.torgbs.") and n.endswith(".bias")) or (".attention." in n and n.rsplit(".", 1)[1] in PL_NO_GRAD)
               for n in others), (what, others)
    assert errs[worst[0]] < tol_grad, (what, worst[0], errs[worst[0]])
    assert max(structural.values(), default=0.0) < tol_structural, (what, structural)
