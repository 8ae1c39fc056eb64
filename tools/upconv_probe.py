"""The six upsampling layers of the 256^2 generator (batch 32) on both inference paths: today's four cuDNN polyphase convolutions
(TF32) + the polyphase blur (ops.upconv_blur_phases), and the fused wgmma kernel (ops.upconv_blur_native).  Per layer: ms (CUDA
events over 10 calls after warm-up), algorithmic TFLOP/s (2 * B * (2H)^2 * Cin * Cout * 9 / 4, halo not counted) and the
algorithmic bytes (x read once + y written once), the fused kernel's MMA work issued over the algorithmic work ("issued": strips of
16 phase columns for 14 output column pairs, steps of 8 phase rows over H + 2), plus the rel-RMS difference between the two paths.

    python tools/upconv_probe.py [--paths phases,fused] [--batch 32]
"""
import argparse, math, os, sys, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import gansformer_b200  # noqa: F401  (registers the package)
from importlib import import_module
ops = import_module("gansformer-reproducibility-challenge_b200.ops")

# (input res, Cin, Cout) of the 256^2 generator's upsampling layers
LAYERS = [(4, 512, 512), (8, 512, 512), (16, 512, 512), (32, 512, 512), (64, 512, 256), (128, 256, 128)]


def issued_over_algorithmic(H, W):
    """MMA work upconv_blur_tc_kernel issues (16 x 8 phase positions per strip and step) over the H x W phase positions needed."""
    strips, steps = (W + 13) // 14, (H + 2 + 7) // 8
    return strips * 16 * steps * 8 / (H * W)


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", default="phases,fused")
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    paths = a.paths.split(",")
    B = a.batch
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"card: {q.stdout.strip()}  batch {B}")
    print(f"{'res':>4} {'Cin':>4} {'Cout':>4} {'GB':>6} {'TFLOP':>6} {'issued':>6}" + "".join(f" {p + ' ms':>11} {'TF/s':>6} {'GB/s':>6}" for p in paths)
          + ("  rel-rms" if len(paths) == 2 else ""))
    tot = {p: 0.0 for p in paths}
    g = torch.Generator(device=dev).manual_seed(0)
    for H, ci, co in LAYERS:
        x = torch.randn(B, ci, H, H, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
        w = torch.randn(co, ci, 3, 3, device=dev, generator=g) / math.sqrt(ci * 9)
        d = torch.rand(B, co, device=dev, generator=g) + 0.5
        phases = ops.upconv_phase_weights(w)
        wt = ops.conv3x3_pack(w)
        fns = {"phases": lambda: ops.upconv_blur_phases(x, phases, scale=d, gain=4.0),
               "fused": lambda: ops.upconv_blur_native(x, wt, d, gain=4.0)}
        flops = 2.0 * B * (2 * H) ** 2 * ci * co * 9 / 4
        nbytes = 4.0 * B * H * H * ci + 4.0 * B * (2 * H) ** 2 * co
        line = f"{2 * H:4d} {ci:4d} {co:4d} {nbytes / 1e9:6.3f} {flops / 1e12:6.3f} {issued_over_algorithmic(H, H):6.2f}"
        outs = []
        with torch.no_grad():
            for p in paths:
                t = timeit(fns[p])
                tot[p] += t
                outs.append(fns[p]())
                line += f" {t:11.4f} {flops / t / 1e9:6.0f} {nbytes / t / 1e6:6.0f}"
            if len(outs) == 2:
                diff = (outs[0] - outs[1]).pow(2).mean().sqrt() / outs[0].pow(2).mean().sqrt()
                line += f"  {diff.item():.2e}"
        print(line, flush=True)
        del x, w, d, phases, wt, outs
    print("total " + "  ".join(f"{p}: {tot[p]:.3f} ms" for p in paths))


if __name__ == "__main__":
    main()
