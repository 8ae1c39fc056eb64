"""CPU checks of the D-phase harness of tests/test_gpu_step_d_phase.py, and the conditioning its bounds rely on.

The trainer runs on the CPU with the torch definitions (ops.augment_ref, ops.augment_filter_ref, the composite R1 route) and the
CUDA attention forward swapped for the oracle's layer, with the parameters attached so that D's gradients flow through it.  For
every case of the GPU file, two steps (the R1 step, then a plain one) are held against ``step_phase_ref.d_phase64``:

* The harness: the recorder's draw order, the R1 weight, the labels and the ADA accumulator must agree with the fp32 trainer to
  fp32 round-off, before any GPU time is spent.
* The conditioning: the same D phase restated in fp32 (oracle.discriminator.discriminator_forward(dtype=float32)) against fp64 on
  the same inputs.  The untrained generator's images put the attention discriminator where fp32 keeps few digits (DESIGN section
  4.11).  With the tRGB weights scaled by TORGB_SCALE and no augmentation the restatement keeps the digits the GPU bounds need;
  under augmentation it records how far fp32 itself goes on these draws.  COND_LOSS and COND_GRAD hold both.
"""
import pytest
import torch

from oracle import bipartite as ob
from tests import step_phase_ref as ref
from tests import test_gpu_step_d_phase as gd
from tests import test_gpu_step_determinism as sdet

# The fp32 trainer against fp64, worst over the cases and both steps on an x86-64 CPU: loss and R1 3.4e-5 ("bgcfn", step 0),
# gradients 7.7e-3 ("bgc", step 0, blocks.0.att0.wpk), the fakes 1.2e-6; frozen at about 2x.  The harness mistakes this guards
# against move the loss by far more: on the H100, the R1 weight without d_reg_interval by 0.36-0.38, R1 taken through the augmented
# reals by 0.37-0.75, and a draw reused for the fakes fails the recorder's draw count (DESIGN section 4.11).
TOL_LOSS = 1e-4
TOL_GRAD = 1.5e-2
TOL_FAKES = 1e-5
# The fp32 restatement against fp64.  Without augmentation it keeps the digits the GPU bounds need: loss 3.6e-7, R1 3.8e-7,
# gradients 6.9e-6.  Under augmentation at p = 0.8 it does not, whatever the image scale (DESIGN section 4.11): loss and R1 up to
# 8.4e-5 ("bgcfn"), gradients up to 1.7e-3 ("bgc", "bgcfn").
COND_LOSS = {False: 2e-6, True: 2e-4}
COND_GRAD = {False: 2e-5, True: 5e-3}


def _oracle_attention(gf, monkeypatch):
    def forward(self, x, y, centroids=None, return_att=False, out=None, centroids_init=None, **kw):
        w = dict(self.named_parameters(recurse=False))              # attached: the parameter gradients flow through the layer
        o, att, cen = ob.transformer_layer(x.permute(0, 3, 1, 2), y, w, integration=self.integration, norm=self.norm,
                                           duplex=self.duplex, use_pos=self.use_pos, return_att=return_att,
                                           kmeans_iters=self.kmeans_iters, img2ltnt=self.img2ltnt, centroids_init=centroids_init)
        return o.permute(0, 2, 3, 1).contiguous(), att, cen
    monkeypatch.setattr(gf.BipartiteAttention, "forward", forward)


@pytest.mark.parametrize("case", list(gd.CASES))
def test_cpu_step_d_phase_against_fp64(gf, case, monkeypatch):
    dkw, augment, c_dim = gd.CASES[case]
    _oracle_attention(gf, monkeypatch)
    tr, G, D = sdet._gan(gf, "cpu", dkw, c_dim)
    with torch.no_grad():
        for t in G.synthesis.torgbs:
            t.weight.mul_(gd.TORGB_SCALE)
    rec = ref.StepRecorder(tr, monkeypatch, gd.filtered(tr, augment))
    cfg = gd.d_config(tr, augment)
    trainer = tr.Trainer(G, D, cfg)
    z, reals, gen_c, real_c = sdet._batch("cpu", c_dim=c_dim)
    sd_d = {n: p.detach().clone() for n, p in D.named_parameters()}
    fakes64 = ref.generator64(G.state_dict(), z, gen_c)
    signs = []
    torch.manual_seed(500)
    for i in range(2):
        st = trainer.step(z, reals, gen_c, real_c)
        do_r1 = i == 0
        assert (st.r1 > 0) == do_r1
        draws = rec.draws(i, i + 1)
        assert (draws["reals"] is None) == (not augment)
        want = ref.d_phase64(sd_d, reals, rec.fakes[i], draws, gen_c, real_c, do_r1, cfg)
        errs, structural = gd.grad_errors(D, want["grads"], bk2_exact=False)
        e_loss = abs(st.loss_d - want["loss"]) / abs(want["loss"])
        e_r1 = abs(st.r1 - want["r1"]) / want["r1"] if do_r1 else 0.0
        e_fakes = ref.rel(rec.fakes[i], fakes64)
        f32 = ref.d_phase64(sd_d, reals, rec.fakes[i], draws, gen_c, real_c, do_r1, cfg, dtype=torch.float32)
        c_loss = abs(f32["loss"] - want["loss"]) / abs(want["loss"])
        c_r1 = abs(f32["r1"] - want["r1"]) / want["r1"] if do_r1 else 0.0
        c_grads = {n: ref.rel(g, want["grads"][n]) for n, g in f32["grads"].items() if n in errs}
        worst, c_worst = max(errs, key=errs.get), max(c_grads, key=c_grads.get)
        print(f"[host D phase {case}] step {i}: trainer loss {e_loss:.2e} r1 {e_r1:.2e} gradients {errs[worst]:.2e} ({worst}) "
              f"structural {max(structural.values(), default=0.0):.1e} fakes {e_fakes:.2e}; fp32 restatement loss {c_loss:.2e} "
              f"r1 {c_r1:.2e} gradients {c_grads[c_worst]:.2e} ({c_worst}); min |logit_real| "
              f"{want['logits_real'].abs().min().item():.3e}")
        assert e_fakes < TOL_FAKES and e_loss < TOL_LOSS and e_r1 < TOL_LOSS and errs[worst] < TOL_GRAD
        assert max(structural.values(), default=0.0) < gd.TOL_STRUCTURAL
        aug = bool(augment)
        assert c_loss < COND_LOSS[aug] and c_r1 < COND_LOSS[aug] and c_grads[c_worst] < COND_GRAD[aug]
        if trainer.ada_stats is not None:
            gd.check_ada(trainer, st, cfg, want["logits_real"], signs, i)
