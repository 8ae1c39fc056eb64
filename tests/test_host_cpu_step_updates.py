"""CPU checks of the harness of tests/test_gpu_step_updates.py, and of the trainer's snapshot and restore.

The trainer runs on the CPU with the oracle's attention layer in place of the CUDA forward (tests/test_host_cpu_step_d_phase.py):

* Four steps at a live learning rate with path length (d_reg_interval 2, g_reg_interval 3: R1 + pl, none, R1, pl) through the GPU
  file's checks: every Adam step against fp64 with the lazy rescaling, two G steps on a path-length step, G_ema, its buffers and
  w_avg, and each path-length phase against ``step_phase_ref.pl_phase64`` (lengths, penalty, pl_mean, G's gradients).
* ``Trainer._snapshot`` and ``_restore`` around two eager steps: the next step is then a fresh trainer's first step, bit for bit,
  although the restored Adam states exist (zeroed) where the fresh trainer has none yet.
"""
import copy

import torch

from tests import step_phase_ref as ref
from tests import test_gpu_step_determinism as sdet
from tests import test_gpu_step_updates as gu
from tests import test_host_cpu_step_d_phase as hd

# The fp32 CPU trainer against the definitions on an x86-64 CPU, frozen at about 2x the worst measured: Adam updates 2.6e-7 and
# states 1.0e-7; G_ema 6.8e-9 and w_avg 5.8e-7 of the move; the path-length phase's lengths 3.9e-6, penalty and pl_mean 5.9e-6,
# gradients 4.7e-4 (mapping.local.0.bias, step 0) and structural zeros 9.8e-8.  The fp32 leaky-ReLU kinks the reference cannot
# take from a GPU forward here bound the gradients.
TOL_ADAM = 5e-7
TOL_ADAM_STATE = 2e-7
TOL_LERP = 1.2e-6
TOL_PL = (8e-6, 1.2e-5, 1e-3, 2e-7)      # lengths, penalty and pl_mean, gradients, structural


def test_cpu_updates_and_pl_phase_against_definitions(gf, monkeypatch):
    hd._oracle_attention(gf, monkeypatch)
    tr, G, D = gu._gan(gf, "cpu", dict(transformer=True), {}, 0, live_terms=True)
    G_probe = copy.deepcopy(G).train()
    t = tr.Trainer(G, D, tr.TrainConfig(**{**gu.LIVE, "pl_weight": 2.0}))
    rd, rg = ref.OptRecorder(t.opt_d, monkeypatch), ref.OptRecorder(t.opt_g, monkeypatch)
    rp = ref.PlRecorder(tr, monkeypatch)
    z, reals, _, _ = sdet._batch("cpu")
    worst = dict(adam=0.0, state=0.0, ema=0.0, w_avg=0.0)
    torch.manual_seed(900)
    for i in range(4):
        ema0 = [p.detach().clone() for p in t.G_ema.parameters()]
        w_avg0 = t.G.mapping.w_avg.detach().clone()
        nd, ng, npl = len(rd.calls), len(rg.calls), len(rp.calls)
        st = t.step(z, reals)
        gu.check_step_updates(t, st, i, rd.calls[nd:], rg.calls[ng:], ema0, w_avg0, z, None, worst)
        assert len(rp.calls) - npl == (i % 3 == 0)
        if i % 3 == 0:
            gu.check_pl_call(rp.calls[-1], st.pl_mean, G_probe, z, None, t.cfg, 0.0, False, f"host step {i}", TOL_PL)
    print(f"[host updates] worst: Adam update {worst['adam']:.2e}, state {worst['state']:.2e}; G_ema {worst['ema']:.2e}; "
          f"w_avg {worst['w_avg']:.2e}")
    assert worst["adam"] < TOL_ADAM and worst["state"] < TOL_ADAM_STATE, worst
    assert worst["ema"] < TOL_LERP and worst["w_avg"] < TOL_LERP, worst


def test_cpu_restore_leaves_no_trace(gf, monkeypatch):
    hd._oracle_attention(gf, monkeypatch)
    cfg = dict(gu.LIVE, pl_weight=2.0, augment="bc", augment_p=0.5, ada_target=0.6, ada_interval=1, ada_kimg=0.2)
    runs = []
    for warm in (2, 0):
        tr, G, D = gu._gan(gf, "cpu", dict(transformer=True), {}, 0)
        t = tr.Trainer(G, D, tr.TrainConfig(**cfg))
        z, reals, _, _ = sdet._batch("cpu")
        torch.manual_seed(900)
        snap = t._snapshot("cpu")
        for _ in range(warm):
            t.step(z, reals)
        t._restore(snap, "cpu")
        t.it = 0
        if warm:
            assert all(len(s) == 3 for s in t.opt_g.state.values()) and len(t.opt_d.state) > 0
        st = t.step(z, reals)
        runs.append((st, gu._state_cpu(t)))
    (sa, a), (sb, b) = runs
    assert sa == sb
    bad = [n for n in a if not torch.equal(a[n], b[n])]
    assert set(a) == set(b) and not bad, bad[:6]
