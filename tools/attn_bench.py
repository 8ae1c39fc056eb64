"""Per-layer stage-T microbenchmark: the 12 attention layers of the 256^2 generator (BASELINE configs[1], B=32),
CUDA-event timed, both kernel families.  Inputs (>= 134 MB for the large layers) rotate over several buffers so no
iteration finds its input in L2.  Prints GB/s of ALGORITHMIC bytes (read X once + write X' once)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import gansformer_b200 as gf

dev = torch.device("cuda:0")
B = int(os.environ.get("AB_BATCH", 32)); k = int(os.environ.get("AB_K", 16)); D = 32
integ = os.environ.get("AB_INT", "mul")
duplex = bool(int(os.environ.get("AB_DUPLEX", "0")))
with_post = bool(int(os.environ.get("AB_POST", "0")))   # fused demod + noise + bias + lrelu + style, as inside the generator
layers = [(8, 512), (16, 512), (32, 512), (64, 512), (128, 256), (256, 128)]
if os.environ.get("AB_ONLY"):
    layers = [l for l in layers if str(l[0]) in os.environ["AB_ONLY"].split(",")]
iters = int(os.environ.get("AB_ITERS", 10))
modes = os.environ.get("AB_MODES", "default,fp32").split(",")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
try:      # HBM peak as bench.py takes it: the measured burst copy, else the H100 SXM data sheet
    with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
        peak, peak_src = float(json.load(f)["hbm_gbs"]), "MEASURED_PEAKS.json"
except Exception:
    peak, peak_src = 3350.0, "H100 SXM data sheet"
print(f"{torch.cuda.get_device_name(dev)}: HBM peak {peak:.1f} GB/s ({peak_src})", flush=True)
out = []
for res, C in layers:
    nbytes = 2 * 4 * B * res * res * C
    nbuf = max(2, min(6, int(1.0e9 // (nbytes // 2)) + 1))
    xs = [torch.randn(B, res, res, C, device=dev) for _ in range(nbuf)]
    y = torch.randn(B, k, D, device=dev)
    o = torch.empty_like(xs[0])
    post = None
    if with_post:
        post = dict(bias=torch.randn(C, device=dev), noise=torch.randn(res, res, device=dev), strength=torch.tensor(0.1, device=dev), act='lrelu', gain=2 ** 0.5,
                    in_scale=torch.rand(B, C, device=dev) + 0.5, post_scale=torch.rand(B, C, device=dev) + 0.5)
    for mode in modes:
        attn = gf.BipartiteAttention(C, D, k, integration=integ, kmeans=duplex, exact_fp32=(mode == "fp32")).to(dev)
        with torch.no_grad():
            for i in range(3):
                attn(xs[i % nbuf], y, out=o, postop=post, need_centroids=not bool(int(os.environ.get('AB_NOCEN', '1'))))
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            # time the whole call (prologue + stage T) and, separately, stage T alone via the StageTimer hook
            from importlib import import_module
            am = import_module("gansformer-reproducibility-challenge_b200.attention")
            am.STAGE_TIMER = am.StageTimer()
            e0.record()
            for i in range(iters):
                attn(xs[i % nbuf], y, out=o, postop=post, need_centroids=not bool(int(os.environ.get('AB_NOCEN', '1'))))
            e1.record()
            torch.cuda.synchronize()
            t_call = e0.elapsed_time(e1) / iters
            t_stage = sum(a.elapsed_time(b) for a, b, *_ in am.STAGE_TIMER.records) / iters
            am.STAGE_TIMER = None
        path = gf._lib.last_path()
        gbs = nbytes / (t_stage * 1e-3) / 1e9
        rec = dict(res=res, C=C, B=B, k=k, integration=integ, duplex=duplex, mode=mode, path=path, stage_ms=t_stage, call_ms=t_call,
                   alg_GB=nbytes / 1e9, GBps=gbs, frac=gbs / peak)
        out.append(rec)
        print(f"res={res:4d} C={C:4d} {mode:8s} path={path:13s} stage={t_stage:8.4f} ms call={t_call:8.4f} ms  {gbs:8.1f} GB/s  frac={gbs/peak:.3f}", flush=True)
    del xs, o
tot = {}
for r in out:
    t = tot.setdefault(r["mode"], [0.0, 0.0]); t[0] += 2 * r["stage_ms"]; t[1] += 2 * r["alg_GB"]
for m, (ms, gb) in tot.items():
    print(f"SUM over 12 layers mode={m}: {ms:.3f} ms, {gb:.3f} GB -> {gb/ms*1e3:.1f} GB/s, frac {gb/ms*1e3/peak:.3f}")
os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open(os.environ.get("AB_OUT", "gpurun_out/attn_layers.json"), "w"), indent=1)
