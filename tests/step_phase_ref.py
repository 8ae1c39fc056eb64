"""The training step's phases restated in fp64, for tests/test_gpu_step_d_phase.py, tests/test_host_cpu_step_d_phase.py and
tests/test_gpu_step_determinism.py.  Test infrastructure only.

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
"""
from __future__ import annotations

from importlib import import_module
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
