"""The discriminator's attention at 256x256, batch 32: discriminator forward + backward (the D step's route: parameters require grad,
the image does not), the R1 pass (image and parameters require grad: the attention layers run the torch composite, double
backward, or with r1_kernels=True the kernel backward differentiated by the double-backward kernels), and Trainer.step_graphed
images/s with the 256x256 K = 16 generator of bench.py's train_step, for the plain discriminator and for transformer=True with
d_end_res in {32, 64, 256} (K = 16, D = 32), each on both R1 routes, one after the other.  CUDA events, mean over --reps calls
after --warmup; peak = the allocator's peak above what was allocated before the calls.  When the R1 graph does not fit, the
plain steps are timed with a trainer without the penalty (r1_gamma = 0).  One JSON line per configuration.

    python tools/d_attention_probe.py [--reps 5] [--warmup 2] [--steps 10] [--out FILE]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
from importlib import import_module

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gansformer_b200 as gf  # noqa: E402

tr = import_module("gansformer-reproducibility-challenge_b200.training")

RES, B, K = 256, 32, 16
# each transformer configuration twice in a row, the R1 pass on the double-backward kernels and on the composite (the default):
# the kernels first, because a graph capture that runs out of memory (the composite at d_end_res=256) keeps memory in its pool
CONFIGS = [("plain", dict())] + [(f"transformer d_end_res={r}{' r1_kernels' if rk else ''}",
                                  dict(transformer=True, components_num=K, latent_dim=32, d_end_res=r, r1_kernels=rk))
                                 for r in (32, 64, 256) for rk in (True, False)]


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return {"ms": round(e0.elapsed_time(e1) / reps, 3), "peak_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)}


def guarded(fn):
    try:
        return fn()
    except torch.OutOfMemoryError as e:
        err = {"error": "out of memory: " + str(e).splitlines()[0][:160]}
    gc.collect()                                 # the failed call's frames held its tensors
    torch.cuda.empty_cache()
    return err


def probe(name, kw, dev, args):
    rec = {"config": name, "res": RES, "batch": B}
    torch.manual_seed(0)
    D = tr.Discriminator(RES, **kw).to(dev)
    rec["attention_layers"] = sum((b.att0 is not None) + (b.att1 is not None) for b in D.blocks)
    img = torch.rand(B, 3, RES, RES, device=dev) * 2 - 1

    def fwd_bwd():
        D.zero_grad(set_to_none=True)
        F.softplus(D(img)).mean().backward()

    def r1():
        D.zero_grad(set_to_none=True)
        x = img.detach().requires_grad_(True)
        logits = D(x)
        (g,) = torch.autograd.grad(logits.sum(), x, create_graph=True)
        (F.softplus(-logits).mean() + g.square().sum(dim=[1, 2, 3]).mean() * 80.0).backward()

    rec["d_fwd_bwd"] = guarded(lambda: timed(fwd_bwd, args.reps, args.warmup))
    rec["d_r1"] = guarded(lambda: timed(r1, args.reps, args.warmup))
    D.zero_grad(set_to_none=True)
    del img

    def train(r1_gamma):
        torch.manual_seed(0)
        G = gf.Generator(resolution=RES, components_num=K, latent_dim=32, att_dp=0.12).to(dev)
        trainer = tr.Trainer(G, D, tr.TrainConfig(r1_gamma=r1_gamma))
        g = torch.Generator().manual_seed(4)
        z = torch.randn(B, K + 1, 32, generator=g).to(dev)
        reals = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(dev)
        out = {}
        for label, it in (("plain_step", 1), ("r1_step", 0))[:2 if r1_gamma else 1]:    # lazy R1: 15 of 16 steps are plain
            for _ in range(2):
                trainer.it = it
                trainer.step_graphed(z, reals)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                trainer.it = it
                trainer.step_graphed(z, reals)
            e1.record()
            torch.cuda.synchronize()
            out[label + "_ms"] = round(e0.elapsed_time(e1) / args.steps, 3)
        out["images_per_s"] = round(B / (out["plain_step_ms"] * 1e-3), 1)
        if r1_gamma:
            out["images_per_s_lazy_r1"] = round(16 * B / ((15 * out["plain_step_ms"] + out["r1_step_ms"]) * 1e-3), 1)
        out["peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        return out

    torch.cuda.reset_peak_memory_stats()
    rec["step_graphed"] = guarded(lambda: train(10.0))
    if "error" in rec["step_graphed"]:          # the R1 graph did not fit: the plain steps alone (a trainer without the penalty)
        torch.cuda.reset_peak_memory_stats()
        rec["step_graphed_without_r1"] = guarded(lambda: train(0.0))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default=None, help="run the configurations whose name contains this string")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("d_attention_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    lines = [json.dumps({"card": card})]
    print(lines[-1], flush=True)
    for name, kw in CONFIGS:
        if args.only and args.only not in name:
            continue
        lines.append(json.dumps(probe(name, kw, dev, args)))
        print(lines[-1], flush=True)
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
