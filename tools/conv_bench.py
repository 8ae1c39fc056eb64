"""Row f1: the wgmma implicit-GEMM 3x3 convolution (gf_conv3x3_nhwc_tf32) against cuDNN (TF32 and fp32) on the stride-1 convolution
shapes of the 256^2 generator (batch 32): correctness vs fp32 cuDNN, time, TFLOP/s."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import gansformer_b200 as gf
from importlib import import_module
ops = import_module("gansformer-reproducibility-challenge_b200.ops")
dev = torch.device("cuda:0")
torch.backends.cudnn.benchmark = True
B = int(os.environ.get("CB_BATCH", 32))
shapes = [(16, 512, 512), (32, 512, 512), (64, 512, 512), (128, 256, 256), (256, 128, 128)]
if os.environ.get("CB_ONLY"):
    shapes = [s for s in shapes if str(s[0]) in os.environ["CB_ONLY"].split(",")]
print(f"{'res':>4} {'Cin':>4} {'Cout':>4} {'ours ms':>9} {'TF/s':>7} {'cudnn tf32':>11} {'TF/s':>7} {'max rel err':>12}")
for res, ci, co in shapes:
    x = torch.randn(B, ci, res, res, device=dev).contiguous(memory_format=torch.channels_last)
    w = torch.randn(co, ci, 3, 3, device=dev) / (ci * 9) ** 0.5
    wt = ops.conv3x3_pack(w)
    wcl = w.contiguous(memory_format=torch.channels_last)
    flops = 2.0 * B * res * res * 9 * ci * co
    with torch.no_grad():
        torch.backends.cudnn.allow_tf32 = False
        ref = F.conv2d(x, wcl, padding=1)
        got = ops.conv3x3_native(x, wt)
        torch.cuda.synchronize()
        err = ((got - ref).abs().max() / ref.abs().max()).item()
        rms = ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
        torch.backends.cudnn.allow_tf32 = True
        for _ in range(3):
            F.conv2d(x, wcl, padding=1); ops.conv3x3_native(x, wt)
        ts = []
        for fn in (lambda: ops.conv3x3_native(x, wt), lambda: F.conv2d(x, wcl, padding=1)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 10)
    print(f"{res:4d} {ci:4d} {co:4d} {ts[0]:9.4f} {flops / ts[0] / 1e9:7.0f} {ts[1]:11.4f} {flops / ts[1] / 1e9:7.0f} {err:12.3e}  rel-rms {rms:.3e}", flush=True)
    del x, w, wt, ref, got
