"""Cost of adaptive discriminator augmentation (SURVEY A.4 item 15).

1. The kernels at 32 x 3 x 256 x 256 with sampled "bc" parameters (p = 1: every transform applies, a quarter of the images rotate
   by 90 or 270 degrees): gf_augment_nchw and gf_augment_adjoint_nchw, each timed over --iters launches with CUDA events after a
   warm-up, as microseconds per call and GB/s of one read and one write of the image.
2. ``Trainer.step_graphed`` on bench.py's train_step configuration (256x256, K = 16, simplex, att_dp = 0.12, batch 32, the plain
   discriminator, the common step without the lazy R1 term) with augmentation off and with "bc" plus ADA (target 0.6).  Both
   trainers are built first; then the two settings alternate, --reps rounds of --steps replays each, so that drift of the card and
   the host falls on both alike.

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line.

    python tools/augment_probe.py [--iters 200] [--steps 10] [--reps 5] [--out FILE]
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
ops = import_module("gansformer-reproducibility-challenge_b200.ops")

RES, B, K = 256, 32, 16
SETTINGS = {"off": dict(), "bc_ada": dict(augment="bc", augment_p=0.2, ada_target=0.6)}


def kernel_times(dev, iters):
    torch.manual_seed(0)
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, RES, RES, dev)
    x = torch.randn(B, 3, RES, RES, device=dev)
    out = {}
    for name in ("gf_augment_nchw", "gf_augment_adjoint_nchw"):
        for _ in range(10):
            ops._augment_native(name, x, geom, color)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ops._augment_native(name, x, geom, color)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1000.0 / iters
        out[name] = {"us": round(us, 2), "GBps": round(2 * x.numel() * 4 / (us * 1e-6) / 1e9, 1)}
    return out


def make_trainer(dev, cfg):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=32, att_dp=0.12).to(dev)
    D = tr.Discriminator(RES).to(dev)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(B, K + 1, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(dev)
    return tr.Trainer(G, D, tr.TrainConfig(**cfg)), z, reals


def run_steps(trainer, z, reals, n):
    for _ in range(n):
        trainer.it = 1                          # the common step: no lazy R1 term (15 of 16 steps)
        trainer.step_graphed(z, reals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rec = {"card": card, "kernels_32x3x256x256": kernel_times(dev, args.iters)}
    runs = {}
    for name, cfg in SETTINGS.items():
        runs[name] = make_trainer(dev, cfg)
        run_steps(*runs[name], 3)               # eager warm-up, capture, first replays
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()                # the warm-up's cached blocks: the second trainer's graph needs its own pool
    times = {name: [] for name in SETTINGS}
    for _ in range(args.reps):
        for name in SETTINGS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run_steps(*runs[name], args.steps)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    rec.update({"res": RES, "batch": B, "K": K, "att_dp": 0.12, "steps": args.steps, "reps": args.reps,
                "peak_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                "augment_p_after": round(float(runs["bc_ada"][0].augment_p), 5)})
    for name in SETTINGS:
        rec[f"step_{name}"] = {"mean_ms": round(sum(times[name]) / len(times[name]), 3), "best_ms": round(min(times[name]), 3),
                               "rounds_ms": [round(t, 3) for t in times[name]]}
    rec["extra_ms"] = round(rec["step_bc_ada"]["mean_ms"] - rec["step_off"]["mean_ms"], 3)
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
