"""Where the GPU time of an eager config-2 step goes (256^2 generator, K = 16, batch 32, TF32 convolutions): torch.profiler with CUDA
activities over a few eager forwards after warm-up, kernel time grouped into the stride-1 3x3 convolutions, the upsampling path
(polyphase cuDNN convolutions + blur, or the fused kernel), the attention path and everything else.  Profiling slows the host,
so run it on its own, not together with timing runs.

    python tools/step_profile.py [--steps 3] [--top 12]
"""
import argparse, collections, os, sys, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
import gansformer_b200 as gf

GROUPS = (
    ("stride-1 conv", ("conv3x3_tc_kernel",)),
    ("upsampling", ("upconv_blur_tc_kernel", "blur_up_phases_kernel", "fprop", "conv", "cudnn", "implicit")),   # the only cuDNN convolutions left
    ("attention", ("token_", "centroid", "stage_i", "finalize", "gemm_tc", "gemm_kernel", "gemm64", "build_fold", "pos_axis",
                   "bias_rows", "scale_copy", "dropout", "img2ltnt")),
)


def group_of(name: str) -> str:
    for g, keys in GROUPS:
        if any(k in name for k in keys):
            return g
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--top", type=int, default=12)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"card: {q.stdout.strip()}")
    torch.manual_seed(0)
    G = gf.Generator(resolution=256, components_num=16, latent_dim=32).to(dev).eval()
    z = torch.randn(32, 17, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        for _ in range(3):
            G(z)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                G(z)
            torch.cuda.synchronize()
    per_kernel = collections.Counter()
    calls = collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
            per_kernel[e.name] += e.device_time
            calls[e.name] += 1
    per_group = collections.Counter()
    for n, t in per_kernel.items():
        per_group[group_of(n)] += t
    total = sum(per_group.values())
    print(f"kernel time per step: {total / a.steps / 1e3:.3f} ms")
    for g, t in per_group.most_common():
        print(f"  {g:14s} {t / a.steps / 1e3:8.3f} ms  {t / total:6.1%}")
    print("top kernels (ms per step, launches per step):")
    for n, t in per_kernel.most_common(a.top):
        print(f"  {t / a.steps / 1e3:8.3f}  {calls[n] // a.steps:4d}  [{group_of(n)}] {n[:110]}")


if __name__ == "__main__":
    main()
