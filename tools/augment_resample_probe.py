"""Cost of ADA's fractional geometry (SURVEY A.4 item 16).

1. The resampler at 32 x 3 x 256 x 256 with sampled "bgc" parameters at p = 1 and p = 0.6: gf_augment_resample_nchw and its adjoint,
   each timed over --iters launches with CUDA events after a warm-up, as microseconds per call.  Also: the blit pair on the same
   batch, and two single-image extremes -- a zoom-out by 8 (every forward tile on the direct per-pixel path) and a zoom-in by 8 (the
   adjoint stages its 2x output points in many chunks).
2. ``Trainer.step_graphed`` on bench.py's train_step configuration (256x256, K = 16, simplex, att_dp = 0.12, the plain discriminator,
   the common step without the lazy R1 term) at batch 16 -- three graphed trainers of batch 32 do not fit on 80 GB together -- with
   augmentation off, "bc" and "bgc" (both with ADA at p = 0.6, target 0.6).  All trainers are built first; then the settings
   alternate, --reps rounds of --steps replays each, so that drift of the card and the host falls on all alike.

The card's name, power limit and maximum SM clock are read in the same call.  One JSON line.

    python tools/augment_resample_probe.py [--iters 50] [--steps 10] [--reps 5] [--out FILE]
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
B_STEP = 16
SETTINGS = {"off": dict(), "bc_ada": dict(augment="bc", augment_p=0.6, ada_target=0.6),
            "bgc_ada": dict(augment="bgc", augment_p=0.6, ada_target=0.6)}


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) * 1000.0 / iters, 1)


def kernel_times(dev, iters):
    out = {}
    spec = tr.parse_augment("bgc")
    x = torch.randn(B, 3, RES, RES, device=dev)
    for p in (1.0, 0.6):
        torch.manual_seed(0)
        geom, color = tr.sample_augment(spec, p, B, RES, RES, dev)
        frac = tr.sample_augment_frac(spec, p, B, RES, RES, dev)
        for name in ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"):
            out[f"{name}_p{p}_us"] = timed(lambda: ops._augment_resample_native(name, x, geom, color, frac), iters)
        if p == 1.0:
            for name in ("gf_augment_nchw", "gf_augment_adjoint_nchw"):
                out[f"{name}_us"] = timed(lambda: ops._augment_native(name, x, geom, color), iters)
    g1 = torch.zeros(1, 4, dtype=torch.int32, device=dev)
    x1 = x[:1].contiguous()
    for what, f in (("zoom_out_8", [8.0, 0.0, 0.5, 0.0, 8.0, -0.25]), ("zoom_in_8", [0.125, 0.0, 0.5, 0.0, 0.125, -0.25])):
        fr = torch.tensor([f], device=dev)
        for name in ("gf_augment_resample_nchw", "gf_augment_resample_adjoint_nchw"):
            out[f"{name}_1x3x256x256_{what}_us"] = timed(lambda: ops._augment_resample_native(name, x1, g1, None, fr), max(2, iters // 10))
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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_resample_probe needs a CUDA device")
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
