"""Cost of style mixing in the training step: ``Trainer.step_graphed`` on bench.py's train_step configuration (256x256, K = 16,
simplex, att_dp = 0.12, batch 32, the plain discriminator, the common step without the lazy R1 term) at style_mixing 0 and 0.9.

Both trainers are built first; then the two settings alternate, --reps rounds of --steps replays each, timed with CUDA events, so
that drift of the card and the host falls on both alike.  The card's name, power limit and maximum SM clock are read in the same
call.  One JSON line: per setting the mean and best ms per step over the rounds, and the difference of the means.

    python tools/style_mixing_probe.py [--steps 10] [--reps 5] [--out FILE]
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

RES, B, K = 256, 32, 16
SETTINGS = (0.0, 0.9)


def make_trainer(dev, style_mixing):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=32, att_dp=0.12).to(dev)
    D = tr.Discriminator(RES).to(dev)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(B, K + 1, 32, generator=g).to(dev)
    reals = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(dev)
    return tr.Trainer(G, D, tr.TrainConfig(style_mixing=style_mixing)), z, reals


def run_steps(trainer, z, reals, n):
    for _ in range(n):
        trainer.it = 1                          # the common step: no lazy R1 term (15 of 16 steps)
        trainer.step_graphed(z, reals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("style_mixing_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    runs = {}
    for p in SETTINGS:
        runs[p] = make_trainer(dev, p)
        run_steps(*runs[p], 3)                  # eager warm-up, capture, first replays
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()                # the warm-up's cached blocks: the second trainer's graph needs its own pool
    times = {p: [] for p in SETTINGS}
    for _ in range(args.reps):
        for p in SETTINGS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run_steps(*runs[p], args.steps)
            e1.record()
            torch.cuda.synchronize()
            times[p].append(e0.elapsed_time(e1) / args.steps)
    rec = {"card": card, "res": RES, "batch": B, "K": K, "att_dp": 0.12, "steps": args.steps, "reps": args.reps,
           "peak_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    for p in SETTINGS:
        rec[f"style_mixing_{p}"] = {"mean_ms": round(sum(times[p]) / len(times[p]), 3), "best_ms": round(min(times[p]), 3),
                                    "rounds_ms": [round(t, 3) for t in times[p]]}
    rec["extra_ms"] = round(rec["style_mixing_0.9"]["mean_ms"] - rec["style_mixing_0.0"]["mean_ms"], 3)
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
