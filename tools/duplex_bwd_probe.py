"""Forward + backward of the 12 duplex attention layers of the 256x256 generator (config 3 shapes: k = 32, D = 32) at the training
batch of bench.py's train_probe (32), for three backward routes:
    composite   torch autograd through the direct-form recomputation (what a dropout-free duplex layer uses today)
    kernel      stage-T backward kernel + pass-A backward kernels, dropout off, called through _duplex_kernel_backward directly
    kernel+dp   the same kernels with attention dropout (p = 0.12) through the public autograd route
Per layer: CUDA-event time of forward + backward after warm-up, and peak memory above what the inputs hold; the relative
gradient difference between the composite and the kernel route (dropout off).  Needs a CUDA GPU: fails without one.

    python tools/duplex_bwd_probe.py [--batch 32] [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
from importlib import import_module

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

LAYERS = [(8, 512), (16, 512), (32, 512), (64, 512), (128, 256), (256, 128)]      # (resolution, channels); each twice in the network
K, D = 32, 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        res = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, (torch.cuda.max_memory_allocated() - base) / 2 ** 30, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("duplex_bwd_probe: no CUDA device (this probe measures the H100 kernels)")
    import gansformer_b200 as gf
    ag = import_module("gansformer-reproducibility-challenge_b200.autograd")
    dev = torch.device("cuda:0")
    B = args.batch
    print(f"card: {card()}; batch {B}, k = {K}, D = {D}; forward + backward per layer call, mean of {args.reps} after warm-up", flush=True)
    rows, tot = [], {"composite": [0.0, 0.0], "kernel": [0.0, 0.0], "kernel+dp": [0.0, 0.0]}
    for res, C in LAYERS:
        torch.manual_seed(res)
        attn = gf.BipartiteAttention(C, D, K, kmeans=True).to(dev).train()
        attn_dp = gf.BipartiteAttention(C, D, K, kmeans=True, att_dp=0.12).to(dev).train()
        attn_dp.load_state_dict(attn.state_dict())
        names = tuple(n for n, _ in attn.named_parameters(recurse=False))
        params = [p for _, p in attn.named_parameters(recurse=False)]
        x = torch.randn(B, res, res, C, device=dev, requires_grad=True)
        y = torch.randn(B, K, D, device=dev, requires_grad=True)
        g = torch.randn(B, res, res, C, device=dev)

        def composite():
            out, _, _ = attn(x, y)
            return torch.autograd.grad(out, [x, y, *params], g, allow_unused=True)

        def kernel():
            with torch.no_grad():
                attn(x, y)
            return ag._duplex_kernel_backward(attn, names, x, y, params, g)

        def kernel_dp():
            out, _, _ = attn_dp(x, y)
            return torch.autograd.grad(out, [x, y, *attn_dp.parameters()], g, allow_unused=True)

        r = {}
        for name, fn in (("composite", composite), ("kernel", kernel), ("kernel+dp", kernel_dp)):
            ms, gib, grads = timed(fn, args.reps)
            r[name] = (ms, gib)
            tot[name][0] += 2 * ms
            tot[name][1] = max(tot[name][1], gib)
            if name == "composite":
                gc = grads
            elif name == "kernel":
                gk = grads
            del grads
        rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-30)).item()
        rx, ry = rel(gk[0], gc[0]), rel(gk[1], gc[1])
        # bk, bk2 and bv2 are constant over what their softmax normalises: their true gradient is 0 and both routes give round-off
        rp = max(rel(a, b) for n, a, b in zip(names, gk[2:], gc[2:]) if b is not None and a is not None and n not in ("bk", "bk2", "bv2"))
        del gc, gk
        row = dict(res=res, C=C, B=B, composite_ms=r["composite"][0], composite_gib=r["composite"][1], kernel_ms=r["kernel"][0],
                   kernel_gib=r["kernel"][1], kernel_dp_ms=r["kernel+dp"][0], kernel_dp_gib=r["kernel+dp"][1], rel_dx=rx, rel_dy=ry, rel_params=rp)
        rows.append(row)
        print(f"res {res:3d} C {C:3d}: composite {r['composite'][0]:8.2f} ms {r['composite'][1]:6.2f} GiB | kernel {r['kernel'][0]:8.2f} ms "
              f"{r['kernel'][1]:6.2f} GiB | kernel+dp {r['kernel+dp'][0]:8.2f} ms {r['kernel+dp'][1]:6.2f} GiB | rel grad diff x {rx:.1e} "
              f"y {ry:.1e} params {rp:.1e}", flush=True)
        del attn, attn_dp, x, y, g, params
        torch.cuda.empty_cache()
    print("12 layers (each shape twice): " + " | ".join(f"{n} {v[0]:.1f} ms, peak {v[1]:.2f} GiB" for n, v in tot.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), batch=B, k=K, D=D, rows=rows, total_ms={n: v[0] for n, v in tot.items()}), f, indent=1)


if __name__ == "__main__":
    main()
