"""Cost of the generator's path-length regularisation at 256x256, K = 16, simplex, att_dp = 0.12, batch 32 (path-length batch 16),
with the plain discriminator of bench.py's train_step:

* the G regularisation phase alone (Trainer._pl_phase: mapping + synthesis of 16 images, the gradient with respect to ws with
  create_graph=True, the penalty's backward through it, the G update), eager and replayed from a CUDA graph of its own: time and
  the allocator's peak above what was allocated before;
* Trainer.step_graphed with pl_weight = 2 at a path-length step (it = 4: no R1) and at the step with both lazy terms (it = 0),
  against the same steps of a trainer with pl_weight = 0, and the plain step; when the graphed path-length step does not fit, the
  same steps eagerly (Trainer.step);
* images/s over the 16-step schedule of the default intervals (R1 every 16th step, path length every 4th), with and without it.

CUDA events, mean over --steps calls after warm-up.  The card's name and power limit are read in the same call.  One JSON line.

    python tools/pl_probe.py [--steps 10] [--reps 5] [--out FILE]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
from importlib import import_module

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gansformer_b200 as gf  # noqa: E402

tr = import_module("gansformer-reproducibility-challenge_b200.training")
att = import_module("gansformer-reproducibility-challenge_b200.attention")
nets = import_module("gansformer-reproducibility-challenge_b200.networks")

RES, B, K = 256, 32, 16


def events_ms(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / n, 3)


def guarded(fn):
    try:
        return fn()
    except torch.OutOfMemoryError as e:
        err = {"error": "out of memory: " + str(e).splitlines()[0][:160]}
    gc.collect()
    torch.cuda.empty_cache()
    return err


def make_trainer(dev, pl_weight):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=32, att_dp=0.12).to(dev)
    D = tr.Discriminator(RES).to(dev)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(B, K + 1, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(dev)
    return tr.Trainer(G, D, tr.TrainConfig(pl_weight=pl_weight)), z, reals


def pl_phase(dev, args):
    trainer, z, _ = make_trainer(dev, 2.0)
    trainer.G.requires_grad_(True)
    trainer.D.requires_grad_(False)
    run = lambda: trainer._pl_phase(z, tr.StepStats())
    out = {}
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out["eager"] = {"ms": events_ms(run, args.reps), "peak_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)}

    def graphed():
        nets.CACHE_BYPASS = att.FORCE_REFOLD = True
        try:
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            with torch.cuda.graph(graph):
                run()
            graph.replay()
            torch.cuda.synchronize()
            peak = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)
            return {"ms": events_ms(graph.replay, args.reps), "peak_gib": peak}
        finally:
            nets.CACHE_BYPASS = att.FORCE_REFOLD = False
    out["graphed"] = guarded(graphed)
    out["pl_mean"] = round(float(trainer.pl_mean), 4)
    return out


def steps(dev, args, pl_weight, graphed=True):
    trainer, z, reals = make_trainer(dev, pl_weight)
    torch.cuda.reset_peak_memory_stats()
    out = {}
    for label, it in (("it0_step", 0), ("it4_step", 4), ("plain_step", 1)):
        def one():
            trainer.it = it
            (trainer.step_graphed if graphed else trainer.step)(z, reals)
        for _ in range(2):
            one()
        out[label + "_ms"] = events_ms(one, args.steps if graphed else args.reps)
    out["peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    if graphed:
        out["graphs"] = sorted(str(k) for k in trainer._graphs if isinstance(k, tuple))
    return out


def amortised(a, b):
    """16-step schedule of the default intervals: R1 on step 0, path length on steps 0, 4, 8, 12 (a: pl_weight 2, b: 0)."""
    with_pl = a["it0_step_ms"] + 3 * a["it4_step_ms"] + 12 * a["plain_step_ms"]
    without = b["it0_step_ms"] + 15 * b["plain_step_ms"]
    return {"pl_ms_per_step": round((with_pl - without) / 16, 3), "images_per_s_with_pl": round(16 * B / (with_pl * 1e-3), 1),
            "images_per_s_without_pl": round(16 * B / (without * 1e-3), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pl_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rec = {"card": card, "res": RES, "batch": B, "pl_batch": B // 2, "K": K, "att_dp": 0.12}
    # each measurement in a clean allocator state, the largest first: a graph capture that runs out of memory keeps its pool
    for key, fn in (("step_pl_weight_2", lambda: steps(dev, args, 2.0)), ("step_pl_weight_0", lambda: steps(dev, args, 0.0))):
        rec[key] = guarded(fn)
        gc.collect()
        torch.cuda.empty_cache()
    a, b = rec["step_pl_weight_2"], rec["step_pl_weight_0"]
    if "error" in a:                  # the graphed path-length step does not fit: the eager steps, with and without the phase
        for key, pw in (("eager_step_pl_weight_2", 2.0), ("eager_step_pl_weight_0", 0.0)):
            rec[key] = guarded(lambda: steps(dev, args, pw, graphed=False))
            gc.collect()
            torch.cuda.empty_cache()
        a, b = rec["eager_step_pl_weight_2"], rec["eager_step_pl_weight_0"]
    if "error" not in a and "error" not in b:
        rec["amortised"] = amortised(a, b)
    rec["pl_phase"] = guarded(lambda: pl_phase(dev, args))
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
