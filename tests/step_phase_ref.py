"""The training step's phases restated in fp64, for tests/test_gpu_step_d_phase.py, tests/test_host_cpu_step_d_phase.py,
tests/test_gpu_step_determinism.py and tests/test_{gpu,host_cpu}_step_updates.py.  Test infrastructure only.

* ``StepRecorder`` wraps the three augmentation samplers of ``training`` and ``Trainer._generate``: it keeps every draw and the D
  phase's fakes.  ``Trainer._augment`` draws in the order sample_augment, sample_augment_frac, then (with "imgfilter" or "noise")
  sample_augment_filter, once per image batch; ``_step_tensors`` augments the reals, then the D phase's fakes, then the G phase's
  fakes.  ``draws(step)`` hands back the three batches' parameters by name and checks the number of draws, so that a reordering of
  the step fails loudly instead of silently pairing images with another batch's parameters.
* ``augment64`` applies one recorded draw in fp64 through the definitions ``ops.augment_ref`` and ``ops.augment_filter_ref``.
* ``d_phase64`` is the D update of ``_step_tensors`` written out from its definition on the discriminator's state dict
  (tests/conditional_ref.py's discriminator): softplus(D(A_f fakes, gen_c)) + softplus(-D(A_r reals, real_c)), and on an R1 step
  the penalty |d sum D(A_r x) / dx|^2 with respect to the un-augmented reals x, weighted by gamma / 2 * d_reg_interval.  It returns
  the loss, the penalty, the real logits and fp64 autograd gradients of every parameter.
* ``OptRecorder`` records every ``step`` of an optimiser (the parameters, gradients and Adam state before it, the parameters and
  state after it); ``adam_errors`` holds one recorded step against Adam written out in fp64 with the trainer's lazy rescaling.
* ``PlRecorder`` records the path-length phase (G's state, the dropout state and pl_mean at its start, its noise draw, the gradient
  it takes with respect to ws, and G's gradients at its end); ``pl_phase64`` restates the phase from its definition in fp64.
"""
from __future__ import annotations

from importlib import import_module
import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from tests import conditional_ref as cref

OPS = "gansformer-reproducibility-challenge_b200.ops"
BATCHES = ("reals", "fakes_d", "fakes_g")          # the image batches of one step, in the order _step_tensors augments them
F64 = torch.float64


def _cpu(t):
    return None if t is None else t.detach().cpu()


class StepRecorder:
    """Records the augmentation draws and the D phase's fakes of every step a trainer takes (monkeypatch undoes it)."""

    def __init__(self, tr, monkeypatch, filtered: bool):
        self.filtered = filtered
        self.sampled: Dict[str, List] = {"sample_augment": [], "sample_augment_frac": [], "sample_augment_filter": []}
        for name, seen in self.sampled.items():
            fn = getattr(tr, name)
            monkeypatch.setattr(tr, name, lambda *a, _fn=fn, _seen=seen, **k: _seen.append(_fn(*a, **k)) or _seen[-1])
        self.fakes: List[torch.Tensor] = []
        generate = tr.Trainer._generate

        def _generate(trainer, z, cutoffs, phase, gc=()):
            out = generate(trainer, z, cutoffs, phase, gc)
            if phase == "d":
                self.fakes.append(out.detach().clone())
            return out
        monkeypatch.setattr(tr.Trainer, "_generate", _generate)

    def draws(self, step: int, steps: int) -> Dict[str, Optional[tuple]]:
        """The draws of step ``step`` after ``steps`` steps: {batch: (geom, color, frac, gains, sigma, noise) on the CPU}, every value
        None without augmentation.  Asserts that each sampler ran exactly once per image batch and the D phase generated once per
        step."""
        n = len(self.sampled["sample_augment"])
        assert len(self.fakes) == steps, (len(self.fakes), steps)
        if n == 0:
            assert not any(self.sampled.values()), {k: len(v) for k, v in self.sampled.items()}
            return {b: None for b in BATCHES}
        assert n == len(BATCHES) * steps, (n, steps)
        assert len(self.sampled["sample_augment_frac"]) == n
        assert len(self.sampled["sample_augment_filter"]) == (n if self.filtered else 0)
        out = {}
        for j, b in enumerate(BATCHES):
            i = len(BATCHES) * step + j
            geom, color = self.sampled["sample_augment"][i]
            frac = self.sampled["sample_augment_frac"][i]
            gains = sigma = noise = None
            if self.filtered:
                gains, sigma, noise = self.sampled["sample_augment_filter"][i]
            out[b] = tuple(_cpu(t) for t in (geom, color, frac, gains, sigma, noise))
        return out


def augment64(img: torch.Tensor, draw: Optional[tuple]) -> torch.Tensor:
    """One recorded draw applied to img through the definitions, in img's dtype (Trainer._augment's order: blit or resampler and
    colour, then filter and noise)."""
    if draw is None:
        return img
    ops = import_module(OPS)
    geom, color, frac, gains, sigma, noise = draw
    img = ops.augment_ref(img, geom, color, frac)
    if gains is not None or sigma is not None:
        img = ops.augment_filter_ref(img, gains, sigma, noise)
    return img


def d_phase64(sd_d: Dict[str, torch.Tensor], reals: torch.Tensor, fakes: torch.Tensor, draws: Dict[str, Optional[tuple]],
              gen_c: Optional[torch.Tensor], real_c: Optional[torch.Tensor], do_r1: bool, cfg, dtype=F64) -> dict:
    """The D phase of one step from its definition, on the CPU in ``dtype`` (fp64 unless a test asks for the fp32 restatement).
    sd_d: the discriminator's parameters by name (any dtype and device); reals and fakes: the images as D's input before
    augmentation; draws: StepRecorder.draws; cfg: the TrainConfig (r1_gamma, d_reg_interval).  Returns dict(loss, r1, logits_real,
    grads) with grads {parameter name: gradient or None} for every entry of sd_d."""
    sd = {n: t.detach().to("cpu", dtype).requires_grad_(True) for n, t in sd_d.items()}
    cast = lambda t: None if t is None else t.detach().to("cpu", dtype)
    x = cast(reals).requires_grad_(do_r1)
    gc, rc = cast(gen_c), cast(real_c)
    logit_real = cref.discriminator_forward(sd, augment64(x, draws["reals"]), rc, dtype=dtype)
    logit_fake = cref.discriminator_forward(sd, augment64(cast(fakes), draws["fakes_d"]), gc, dtype=dtype)
    loss = F.softplus(logit_fake).mean() + F.softplus(-logit_real).mean()
    r1 = torch.zeros((), dtype=dtype)
    if do_r1:
        (gx,) = torch.autograd.grad(logit_real.sum(), x, create_graph=True)
        r1 = gx.square().sum(dim=[1, 2, 3]).mean()
        loss = loss + r1 * (cfg.r1_gamma / 2 * cfg.d_reg_interval)           # lazy regularisation: gamma / 2, every interval-th step
    names = list(sd)
    grads = torch.autograd.grad(loss, [sd[n] for n in names], allow_unused=True)
    return dict(loss=loss.item(), r1=r1.item(), logits_real=logit_real.detach(), grads=dict(zip(names, grads)))


def generator64(sd_g: Dict[str, torch.Tensor], z: torch.Tensor, gen_c: Optional[torch.Tensor]) -> torch.Tensor:
    """The 64x64 generator of tests/test_gpu_step_determinism._gan in fp64 (tests/conditional_ref.py), from its state dict."""
    c = None if gen_c is None else gen_c.detach().double().cpu()
    return cref.generator_forward(cref.cast(sd_g), z.detach().double().cpu(), c, resolution=64, components_num=8, latent_dim=32,
                                  mapping_layers=4)


def rel(got: torch.Tensor, want: torch.Tensor) -> float:
    """Relative L2 error: |got - want| / |want| in fp64 on the CPU."""
    want = want.detach().double().cpu()
    return ((got.detach().double().cpu() - want).norm() / want.norm()).item()


def lazy_adam(cfg, interval: Optional[int]) -> tuple:
    """(lr, beta1, beta2) of an Adam whose network is regularised lazily every ``interval``-th step (None: not lazily)."""
    c = 1.0 if interval is None else interval / (interval + 1.0)
    return cfg.lr * c, 0.0 ** c, 0.99 ** c


class OptRecorder:
    """Wraps ``opt.step`` on the instance: every call appends {param: (p, grad, exp_avg, exp_avg_sq, step) before, (p, exp_avg,
    exp_avg_sq, step) after}, on the CPU.  A state the step creates counts as zeros before it."""

    def __init__(self, opt, monkeypatch):
        self.calls: List[dict] = []
        step = opt.step

        def recorded(*a, **k):
            before = {}
            for g in opt.param_groups:
                for p in g["params"]:
                    if p.grad is None:
                        continue
                    s = opt.state.get(p, {})
                    z = torch.zeros_like(p).cpu()
                    before[p] = (_cpu(p).clone(), _cpu(p.grad).clone(), _cpu(s["exp_avg"]).clone() if s else z,
                                 _cpu(s["exp_avg_sq"]).clone() if s else z, float(s["step"]) if s else 0.0)
            out = step(*a, **k)
            self.calls.append({p: (b, (_cpu(p).clone(), _cpu(opt.state[p]["exp_avg"]).clone(),
                                       _cpu(opt.state[p]["exp_avg_sq"]).clone(), float(opt.state[p]["step"])))
                               for p, b in before.items()})
            return out
        monkeypatch.setattr(opt, "step", recorded)


def adam_errors(call: dict, lr: float, beta1: float, beta2: float, eps: float = 1e-8) -> dict:
    """One recorded Adam step against its definition in fp64, from the recorded gradients and state:
    m' = b1 m + (1 - b1) g, v' = b2 v + (1 - b2) g^2, t' = t + 1, p' = p - lr / (1 - b1^t') m' / (sqrt(v') / sqrt(1 - b2^t') + eps).
    Returns the worst over the parameters of: ``update`` the error of p' - p beyond the half ulp of p' that storing p' in fp32
    costs, over the fp64 update, element-wise; ``state`` the relative L2 error of m' and v'; ``steps`` the number of parameters
    whose step count is not t + 1; and ``count`` the parameters stepped."""
    worst = dict(update=0.0, state=0.0, steps=0, count=len(call))
    for (p, g, m, v, t), (p1, m1, v1, t1) in call.values():
        p, g, m, v = (x.double() for x in (p, g, m, v))
        t = t + 1
        m_ = beta1 * m + (1 - beta1) * g
        v_ = beta2 * v + (1 - beta2) * g * g
        upd = -lr / (1 - beta1 ** t) * m_ / (v_.sqrt() / math.sqrt(1 - beta2 ** t) + eps)
        half_ulp = (torch.nextafter(p1.abs(), torch.tensor(math.inf)) - p1.abs()).double() / 2
        live = upd.abs() > 0
        e = ((p1.double() - p - upd).abs() - half_ulp).clamp(min=0)[live] / upd.abs()[live]
        worst["update"] = max(worst["update"], e.max().item() if e.numel() else 0.0)
        for got, want in ((m1, m_), (v1, v_)):
            if want.norm() > 0:
                worst["state"] = max(worst["state"], rel(got, want))
        worst["steps"] += int(t1 != t)
    return worst


def lerp_error(before: torch.Tensor, target: torch.Tensor, weight: float, got: torch.Tensor) -> float:
    """|got - lerp(before, target, weight)| in fp64 beyond one ulp of got (what an fp32 lerp costs), in the L2 norm, over the size of
    the move |weight (target - before)|."""
    before, target, got = before.detach().cpu(), target.detach().double().cpu(), got.detach().cpu()
    want = before.double() + weight * (target - before.double())
    ulp = (torch.nextafter(got.abs(), torch.tensor(math.inf, dtype=got.dtype)) - got.abs()).double()
    e = ((got.double() - want).abs() - ulp).clamp(min=0)
    return (e.norm() / (weight * (target - before.double())).norm()).item()


class PlRecorder:
    """Wraps ``Trainer._pl_phase``: per call, {"sd": G's state at the start, "dp": the dropout state (seed, step) at the start or
    None on the CPU, "pl_mean": pl_mean at the start, "noise": the draw, "pl_grads": the gradient with respect to ws the phase
    takes, "grads": G's .grad at the end, "penalty": the returned penalty}."""

    def __init__(self, tr, monkeypatch):
        self.calls: List[dict] = []
        phase = tr.Trainer._pl_phase

        def recorded(trainer, z, stats, gc=()):
            G = trainer.G
            rec = dict(sd={n: t.detach().clone() for n, t in G.state_dict().items()}, pl_mean=trainer.pl_mean.item(), dp=None)
            if z.is_cuda:
                from importlib import import_module
                rec["dp"] = tuple(import_module(tr.__name__.rsplit(".", 1)[0] + ".attention").dropout_state(z.device).tolist())
            randn_like, grad = torch.randn_like, torch.autograd.grad

            def draw(t, *a, **k):
                out = randn_like(t, *a, **k)
                rec["noise"] = out.detach().clone()
                return out

            def pl_grad(outputs, inputs, *a, **k):
                out = grad(outputs, inputs, *a, **k)
                if k.get("create_graph") and torch.is_tensor(inputs) and inputs.dim() == 3:    # the phase's d<img, noise>/d ws
                    rec["pl_grads"] = out[0].detach().clone()
                return out
            monkeypatch.setattr(torch, "randn_like", draw)
            monkeypatch.setattr(torch.autograd, "grad", pl_grad)
            try:
                pen = phase(trainer, z, stats, gc)
            finally:
                monkeypatch.setattr(torch, "randn_like", randn_like)
                monkeypatch.setattr(torch.autograd, "grad", grad)
            rec["grads"] = {n: None if p.grad is None else p.grad.detach().clone() for n, p in G.named_parameters()}
            rec["penalty"] = pen.item()
            self.calls.append(rec)
            return pen
        monkeypatch.setattr(tr.Trainer, "_pl_phase", recorded)


def pl_lengths(pl_grads: torch.Tensor) -> torch.Tensor:
    """The path lengths of a gradient with respect to ws [B', k+1, D]: the norm over D, its mean square over the k+1 components."""
    return pl_grads.square().sum(dim=2).mean(dim=1).sqrt()


def pl_phase64(rec: dict, z: torch.Tensor, gen_c: Optional[torch.Tensor], cfg, *, att_mults=None, layer_pos=None,
               duplex: bool = False) -> dict:
    """The path-length phase of ``Trainer._pl_phase`` from its definition in fp64, on the recorded state and noise: the first
    B' = B // pl_batch_shrink latents and labels, ws = mapping(z, c), img = synthesis(ws) (constant noise; att_mults: the dropout
    multipliers of the step after the recorded one, layer_pos: every layer's leaky-ReLU slopes, tests/generator_path_length_ref.py), the
    lengths of d<img, noise / sqrt(H W)>/d ws, pl_mean' = lerp(pl_mean, mean length, pl_decay) taken before the penalty and held
    constant in it, penalty = mean (length - pl_mean')^2, and the gradients of penalty * pl_weight * g_reg_interval with respect to
    every G parameter, with each layer's noise strength expanded to one leaf per pixel and image.  Returns dict(lengths, pl_mean,
    penalty, grads)."""
    from tests import generator_path_length_ref as gref
    nb = max(1, z.shape[0] // cfg.pl_batch_shrink)
    sd = cref.cast(rec["sd"])
    for n in list(sd):
        if n.endswith("noise_strength"):
            sd[n] = sd[n].expand(nb, 1, *sd[n.replace("noise_strength", "noise_const")].shape).clone()
    params = [n for n in rec["grads"]]
    for n in params:
        sd[n].requires_grad_(True)
    c = None if gen_c is None else gen_c[:nb].detach().double().cpu()
    noise = rec["noise"].double().cpu()
    with torch.enable_grad():
        ws = cref.mapping_forward(sd, z[:nb].detach().double().cpu(), c, components_num=8, latent_dim=32, mapping_layers=4)
        img = gref.synthesis_forward(sd, ws, resolution=64, components_num=8, noise_mode="const", duplex=duplex,
                                     att_mults=att_mults, layer_pos=layer_pos)
        (pg,) = torch.autograd.grad((img * (noise / math.sqrt(img.shape[2] * img.shape[3]))).sum(), ws, create_graph=True)
        lengths = pl_lengths(pg)
        mean = rec["pl_mean"] + (lengths.detach().mean().item() - rec["pl_mean"]) * cfg.pl_decay
        penalty = (lengths - mean).square().mean()
        grads = torch.autograd.grad(penalty * (cfg.pl_weight * cfg.g_reg_interval), [sd[n] for n in params], allow_unused=True)
    return dict(lengths=lengths.detach(), pl_mean=mean, penalty=penalty.item(), grads=dict(zip(params, grads)))


def pl_grad_errors(got: Dict[str, Optional[torch.Tensor]], want: Dict[str, Optional[torch.Tensor]]) -> tuple:
    """G's gradients after the path-length phase against ``pl_phase64``'s, under the rules of tests/test_gpu_generator_path_length.py:
    a noise strength against the sum of the magnitudes of its per-pixel terms; the tRGB biases (no gradient in fp64) must have none or
    zeros; a gradient that is zero in fp64 up to its round-off (the attention key biases, constant over what a softmax normalises)
    is held, as a ratio to the largest fp64 gradient norm, in ``structural``; every other one as a relative L2 error.
    Returns (errors, structural)."""
    errs, structural = {}, {}
    scale = max(w.norm().item() for w in want.values() if w is not None)
    for n, w in want.items():
        g = got[n]
        if n.endswith("noise_strength"):
            errs[n] = abs(g.item() - w.sum().item()) / w.abs().sum().item()
        elif w is None:
            assert g is None or torch.count_nonzero(g) == 0, n
        elif w.norm().item() < 1e-9 * scale:
            structural[n] = (g.double().cpu().norm() / scale).item()
        else:
            errs[n] = rel(g, w)
    return errs, structural
