"""Image self-attention (img2img) on the GPU, CUDA-event timed; prints one JSON line.

1. gf_self_attn_fwd and gf_self_attn_bwd at 32^2 (C = 512, h = 8) and 64^2 (C = 256, h = 4), batch 32: milliseconds per call (the
   entry point alone, its transposed operands prepared once) and achieved TFLOP/s from shape-computed FLOPs -- forward 4 B n^2 C
   (S = Q K^T and P V), backward 10 B n^2 C (the five n x n products of FlashAttention-2's backward: S, dP, dV, dK, dQ; the kernels
   compute S and dP twice, once per output kernel, which is not counted) -- with the share of the H100 SXM data sheet's 495 TFLOP/s
   dense TF32.
   gf_self_attn_bwd_vjp (the double backward) likewise, with 24 B n^2 C FLOPs: the twelve n x n products of its algebra (S, dP,
   GdS over 2d, dO Cv^T, P Cv, dS Bk + GS K over 2 x 64 keys, dS^T A + GS^T Q likewise, GdP^T dO, GdP V); the kernels compute S,
   dP, GdS and dO Cv^T again in each output kernel, which is not counted.
2. One R1 gradient through the discriminator's img2img layer (ImageSelfAttention with C = 512, batch 32): time and peak
   memory (torch.cuda.max_memory_allocated above the inputs) on the composite route and on the double-backward kernel, at 32^2,
   where the composite fits; then the kernel route alone at 64^2, where one n x n fp32 tensor of the composite is 17.2 GB.
3. The 256^2 generator (BASELINE configs[1] shape: K = 16, batch 32) forward + backward of mean(img^2), with and without img2img=32,
   alternated in the same run, min and median over repeats.
The card name and power limit are read in the same run.
"""
import json
import math
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                   # noqa: E402
import gansformer_b200 as gf                   # noqa: E402
from gansformer_b200 import _lib               # noqa: E402

TF32_PEAK = 495.0
dev = torch.device("cuda:0")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(dev)


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernels(res, C, B=32, iters=20):
    lib = _lib.load()
    h = C // 64
    d, n = C // h, res * res
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v, do = (torch.randn(B, n, C, device=dev, generator=g) for _ in range(4))
    qt, kt, vt, dot = (t.transpose(1, 2).contiguous() for t in (q, k, v, do))
    o, dq, dk, dv = (torch.empty_like(q) for _ in range(4))
    lse, delta = torch.empty(B, h, n, device=dev), torch.empty(B, h, n, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    scale = 1.0 / math.sqrt(d)
    fwd = lambda: _lib.check(lib.gf_self_attn_fwd(q.data_ptr(), k.data_ptr(), vt.data_ptr(), o.data_ptr(), lse.data_ptr(), B, n, C, d,
                                                  scale, st), "gf_self_attn_fwd")
    bwd = lambda: _lib.check(lib.gf_self_attn_bwd(q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                  lse.data_ptr(), do.data_ptr(), dot.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                                                  dk.data_ptr(), dv.data_ptr(), B, n, C, d, scale, st), "gf_self_attn_bwd")
    a, bk, cv = (torch.randn(B, n, C, device=dev, generator=g) for _ in range(3))
    at, bkt, cvt = (t.transpose(1, 2).contiguous() for t in (a, bk, cv))
    row_r, row_t = torch.empty_like(lse), torch.empty_like(lse)
    gq, gk, gv, gdo = (torch.empty_like(q) for _ in range(4))
    vjp = lambda: _lib.check(lib.gf_self_attn_bwd_vjp(q.data_ptr(), qt.data_ptr(), k.data_ptr(), kt.data_ptr(), v.data_ptr(), vt.data_ptr(),
                                                      do.data_ptr(), dot.data_ptr(), lse.data_ptr(), delta.data_ptr(), a.data_ptr(),
                                                      at.data_ptr(), bk.data_ptr(), bkt.data_ptr(), cv.data_ptr(), cvt.data_ptr(),
                                                      row_r.data_ptr(), row_t.data_ptr(), gq.data_ptr(), gk.data_ptr(), gv.data_ptr(),
                                                      gdo.data_ptr(), B, n, C, d, scale, st), "gf_self_attn_bwd_vjp")
    out = {}
    for name, fn, flops in (("fwd", fwd, 4.0 * B * n * n * C), ("bwd", bwd, 10.0 * B * n * n * C), ("bwd_vjp", vjp, 24.0 * B * n * n * C)):
        ms = timed(fn, iters)
        tf = flops / ms / 1e9
        out[name] = {"ms": round(ms, 3), "TFLOP_s": round(tf, 1), "share_of_495": round(tf / TF32_PEAK, 3)}
    return out


def r1_layer(res, kernel, C=512, B=32, iters=3):
    """One R1 gradient through ImageSelfAttention(C) on x [B, res, res, C]: ms per gradient and the peak memory above the inputs."""
    torch.manual_seed(0)
    m = gf.ImageSelfAttention(C, 32).to(dev)
    m.kernel_double_backward = kernel
    x = torch.randn(B, res, res, C, device=dev)

    def r1():
        xs = x.detach().requires_grad_(True)
        (gx,) = torch.autograd.grad(m(xs).sum(), xs, create_graph=True)
        torch.autograd.grad(gx.square().sum(), [xs, *m.parameters()])

    r1()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    ms = timed(r1, iters, warmup=1)
    peak = torch.cuda.max_memory_allocated(dev) - base
    return {"ms": round(ms, 2), "peak_GiB": round(peak / 2 ** 30, 2)}


def generator_steps(repeats=5, iters=3, B=32):
    gens = {}
    for r in (0, 32):
        torch.manual_seed(0)
        gens[r] = gf.Generator(resolution=256, components_num=16, latent_dim=32, img2img=r).to(dev)
    z = torch.randn(B, 17, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(1))

    def step(G):
        G.zero_grad(set_to_none=True)
        G(z).square().mean().backward()

    times = {r: [] for r in gens}
    for r, G in gens.items():
        timed(lambda: step(G), 1, warmup=2)
    for _ in range(repeats):                                      # alternated, so both see the same machine state
        for r, G in gens.items():
            times[r].append(timed(lambda: step(G), iters, warmup=0))
    return {f"img2img={r}": {"ms_min": round(min(t), 2), "ms_median": round(statistics.median(t), 2)} for r, t in times.items()}


def main():
    res = {"card": card(), "kernels": {}}
    for r, C in ((32, 512), (64, 256)):
        res["kernels"][f"{r}^2 C={C} h={C // 64} B=32"] = kernels(r, C)
    res["r1_d_layer_C512_B32"] = {"32^2 composite": r1_layer(32, False), "32^2 kernels": r1_layer(32, True),
                                  "64^2 kernels": r1_layer(64, True)}
    res["generator_256_fwd_bwd_B32"] = generator_steps()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
