"""Cost of ADA's image-space filtering and additive noise (SURVEY A.4 item 17).

1. The filter at 32 x 3 x 256 x 256 with sampled "bgcfn" parameters at p = 1 and p = 0.6: gf_augment_filter_nchw (with the noise) and
   gf_augment_filter_adjoint_nchw, each timed over --iters launches with CUDA events after a warm-up, as microseconds per call, with
   the bytes each moves (forward: x, noise and y; adjoint: gy and gx) over that time.  Also the blit pair on the same batch.
2. ``Trainer.step_graphed`` on bench.py's train_step configuration (256x256, K = 16, simplex, att_dp = 0.12, the plain discriminator,
   the common step without the lazy R1 term) at batch 16 with "bgc" and "bgcfn" (both with ADA at p = 0.6, target 0.6).  Both
   trainers are built first; then the settings alternate, --reps rounds of --steps replays each.

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line.

    python tools/augment_filter_probe.py [--iters 200] [--steps 10] [--reps 4] [--out FILE]
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

RES, B, C, K = 256, 32, 3, 16
B_STEP = 16
SETTINGS = {"bgc_ada": dict(augment="bgc", augment_p=0.6, ada_target=0.6),
            "bgcfn_ada": dict(augment="bgcfn", augment_p=0.6, ada_target=0.6)}


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def kernel_times(dev, iters):
    out = {}
    x = torch.randn(B, C, RES, RES, device=dev)
    plane = B * C * RES * RES * 4
    for p in (1.0, 0.6):
        torch.manual_seed(0)
        gains, sigma, noise = tr.sample_augment_filter(tr.FILTER_OPS, p, B, C, RES, RES, dev)
        reads_noise = int((sigma != 0).sum())
        t = timed(lambda: ops._augment_filter_native("gf_augment_filter_nchw", x, gains, sigma, noise), iters)
        nbytes = 2 * plane + plane * reads_noise // B
        out[f"gf_augment_filter_nchw_p{p}"] = {"us": round(t, 1), "GB_s": round(nbytes / t / 1e3, 1), "images_with_noise": reads_noise}
        t = timed(lambda: ops._augment_filter_native("gf_augment_filter_adjoint_nchw", x, gains), iters)
        out[f"gf_augment_filter_adjoint_nchw_p{p}"] = {"us": round(t, 1), "GB_s": round(2 * plane / t / 1e3, 1)}
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, RES, RES, dev)
    for name in ("gf_augment_nchw", "gf_augment_adjoint_nchw"):
        out[f"{name}_us"] = round(timed(lambda: ops._augment_native(name, x, geom, color), iters), 1)
    return out


def make_trainer(dev, cfg):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=32, att_dp=0.12).to(dev)
    D = tr.Discriminator(RES).to(dev)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(B_STEP, K + 1, 32, generator=g).to(dev)
    reals = (torch.rand(B_STEP, 3, RES, RES, generator=g) * 2 - 1).to(dev)
    return tr.Trainer(G, D, tr.TrainConfig(**cfg)), z, reals


def run_steps(trainer, z, reals, n):
    for _ in range(n):
        trainer.it = 1                          # the common step: no lazy R1 term (15 of 16 steps)
        trainer.step_graphed(z, reals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_filter_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rec = {"card": card, "kernels_32x3x256x256": kernel_times(dev, args.iters)}
    print(json.dumps(rec), flush=True)
    runs = {}
    for name, cfg in SETTINGS.items():
        runs[name] = make_trainer(dev, cfg)
        run_steps(*runs[name], 3)               # eager warm-up, capture, first replays
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
    times = {name: [] for name in SETTINGS}
    for _ in range(args.reps):
        for name in SETTINGS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run_steps(*runs[name], args.steps)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    rec.update({"res": RES, "step_batch": B_STEP, "K": K, "att_dp": 0.12, "steps": args.steps, "reps": args.reps,
                "peak_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)})
    for name in SETTINGS:
        rec[f"step_{name}"] = {"mean_ms": round(sum(times[name]) / len(times[name]), 3), "min_ms": round(min(times[name]), 3),
                               "max_ms": round(max(times[name]), 3), "rounds_ms": [round(t, 3) for t in times[name]]}
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
