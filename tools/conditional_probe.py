"""Cost of class-conditional generation (SURVEY A.4 item 14), in one process:

* the mapping kernel alone: gf_mapping_fwd against gf_mapping_fwd_cond at c_dim 10 and 1000 (one-hot labels), B = 32, k = 16,
  D = 32, L = 8; CUDA events around --launches launches, the three alternating over --reps rounds;
* the config-2 generator (256x256, K = 16, D = 32, batch 32, graphed inference) at c_dim 0 and 10: images/s;
* the graphed training step on bench.py's train_step configuration (256x256, K = 16, att_dp = 0.12, batch 32, the common step without
  the lazy R1 term) at c_dim 0 and 10.
Each pair alternates over the rounds, so that drift of the card and the host falls on both alike.  The card's name, power limit and
maximum SM clock are read in the same call.  One JSON line: per setting the mean and best over the rounds.

    python tools/conditional_probe.py [--reps 5] [--steps 10] [--out FILE]
"""
import argparse
import ctypes
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

RES, B, K, D = 256, 32, 16, 32


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def summary(ts, scale=1.0):
    return {"mean": round(scale * sum(ts) / len(ts), 4), "best": round(scale * min(ts), 4), "rounds": [round(scale * t, 4) for t in ts]}


def mapping_calls(dev):
    """name -> a closure launching one mapping kernel (B = 32, k = 16, D = 32, L = 8)."""
    lib = gf._lib.load()
    L, k = 8, 16
    g = torch.Generator().manual_seed(1)
    z = torch.randn(B, k + 1, D, generator=g).to(dev)
    w = (torch.randn(2, L, D, D, generator=g) / D ** 0.5).to(dev)
    b = torch.zeros(2, L, D, device=dev)
    out = torch.empty_like(z)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    keep = [z, w, b, out]
    calls = {"c_dim_0": lambda: lib.gf_mapping_fwd(z.data_ptr(), w.data_ptr(), b.data_ptr(), None, 1.0, out.data_ptr(), B, k, D, L, st)}
    for c_dim in (10, 1000):
        c = torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev)
        E = torch.randn(c_dim, D, generator=g).to(dev)
        w0 = (torch.randn(2, 2 * D, D, generator=g) / (2 * D) ** 0.5).to(dev)
        w1 = w[:, 1:].contiguous()
        keep += [c, E, w0, w1]
        calls[f"c_dim_{c_dim}"] = (lambda c=c, E=E, w0=w0, w1=w1, c_dim=c_dim: lib.gf_mapping_fwd_cond(
            z.data_ptr(), c.data_ptr(), c_dim, E.data_ptr(), w0.data_ptr(), w1.data_ptr(), b.data_ptr(), None, 1.0, out.data_ptr(),
            B, k, D, L, st))
    for name, fn in calls.items():
        if fn() != 0:
            raise SystemExit(f"{name}: {lib.gf_last_error().decode()}")
    return calls, keep


def make_generator(dev, c_dim):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=D, c_dim=c_dim).to(dev).eval()
    g = torch.Generator().manual_seed(2)
    z = torch.randn(B, K + 1, D, generator=g).to(dev)
    c = torch.nn.functional.one_hot(torch.arange(B) % c_dim, c_dim).float().to(dev) if c_dim else None
    replay = G.graphed(B)
    return lambda: replay(z, c)


def make_trainer(dev, c_dim):
    torch.manual_seed(0)
    G = gf.Generator(resolution=RES, components_num=K, latent_dim=D, att_dp=0.12, c_dim=c_dim).to(dev)
    Dn = tr.Discriminator(RES, c_dim=c_dim).to(dev)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(B, K + 1, D, generator=g).to(dev)
    reals = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(dev)
    labels = ()
    if c_dim:
        labels = tuple(torch.nn.functional.one_hot(torch.randint(0, c_dim, (B,), generator=g), c_dim).float().to(dev) for _ in range(2))
    trainer = tr.Trainer(G, Dn)

    def step():
        trainer.it = 1                          # the common step: no lazy R1 term (15 of 16 steps)
        trainer.step_graphed(z, reals, *labels)
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--images", type=int, default=10, help="graphed generator calls per round")
    ap.add_argument("--steps", type=int, default=10, help="graphed training steps per round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conditional_probe needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rec = {"card": card, "reps": args.reps}
    with torch.no_grad():
        calls, _keep = mapping_calls(dev)
        for fn in calls.values():
            timed(fn, 200)
        ts = {n: [] for n in calls}
        for _ in range(args.reps):
            for n, fn in calls.items():
                ts[n].append(timed(fn, args.launches))
        rec["mapping_kernel_us"] = {n: summary(t, 1000.0) for n, t in ts.items()}
        rec["mapping_shape"] = {"B": B, "k": 16, "D": D, "L": 8}
        gens = {c: make_generator(dev, c) for c in (0, 10)}
        for fn in gens.values():
            timed(fn, 3)
        ts = {c: [] for c in gens}
        for _ in range(args.reps):
            for c, fn in gens.items():
                ts[c].append(timed(fn, args.images))
        rec["generator_images_per_s"] = {f"c_dim_{c}": summary([B * 1000.0 / t for t in v]) for c, v in ts.items()}
        del gens
    gc.collect()
    torch.cuda.empty_cache()
    steps = {}
    for c in (0, 10):
        steps[c] = make_trainer(dev, c)
        for _ in range(3):
            steps[c]()                          # eager warm-up, capture, first replays
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
    ts = {c: [] for c in steps}
    for _ in range(args.reps):
        for c, fn in steps.items():
            ts[c].append(timed(fn, args.steps))
    rec["train_step_ms"] = {f"c_dim_{c}": summary(v) for c, v in ts.items()}
    rec["peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
