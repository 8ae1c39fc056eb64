"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Every call goes through the C ABI (libgf_attn.so).

Oracle = oracle/bipartite.py in float64 (in-repo restatement; reference source unavailable; PARITY UNPINNED).

Tolerances (stated here, per the task contract):
  * fp32-FMA mode (GF_FLAG_FP32_EXACT, CUDA-core kernel):   |y - y64| <= 1e-5 + 1e-4 |y64|      (SURVEY 8c)
  * TF32 tensor-core mode (wgmma tf32, default):    |y - y64| <= 1e-4 + 1.25e-3 max|y64| + 2e-3 |y64|  and  rel-RMS <= 1e-3
    (frozen in tests/tolerances.json by tools/calibrate_tolerances.py: the SURVEY 8c contract formula plus a scale term --
     measured worst need 6.4e-4 max|y64|, worst rel-RMS 5.5e-4.)
"""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import bipartite as ob
from oracle import generator as og
from tests.golden import make_golden as mg

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "attn_cases.npz")

TOL_PATH = os.path.join(os.path.dirname(__file__), "tolerances.json")
with open(TOL_PATH) as _f:
    TOLERANCES = json.load(_f)           # frozen by tools/calibrate_tolerances.py (see its docstring and DESIGN.md section 5)
TOL = {path: (t["atol"], t["rtol"], t["rel_rms"], t.get("atol_rel_peak", 0.0)) for path, t in TOLERANCES["layer"].items()}
CONTRACT = TOLERANCES["contract"]       # SURVEY 8c per-layer TF32 formula: max(4 e_ref, atol + rtol |y64|)


def _log_parity(rec):
    """GF_PARITY_LOG=<file>: one JSON line per comparison (tools/calibrate_tolerances.py reads them back)."""
    path = os.environ.get("GF_PARITY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(rec) + "\n")


def check_close(got, ref64, path, what="", tol_scale=1.0, e_ref=0.0):
    """|got - ref64| <= max(4 e_ref, atol + rtol |ref64|) element-wise, and relative RMS <= rel_rms (tolerances.json)."""
    got = got.detach().double().cpu()
    ref64 = ref64.detach().double().cpu()
    assert got.shape == ref64.shape, (got.shape, ref64.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    atol, rtol, rrms, arel = (t * tol_scale for t in TOL[path])
    err = (got - ref64).abs()
    atol = atol + arel * ref64.abs().max().item()              # scale term: see tolerances.json "_doc"
    bound = (atol + rtol * ref64.abs()).clamp_min(4.0 * e_ref)
    ratio = (err / bound).max().item()
    contract_ratio = (err / (CONTRACT["atol"] + CONTRACT["rtol"] * ref64.abs()).clamp_min(4.0 * e_ref)).max().item()
    rel_rms = (err.pow(2).mean().sqrt() / ref64.pow(2).mean().sqrt().clamp_min(1e-30)).item()
    print(f"[parity] {what} path={path} max_abs={err.max().item():.3e} max_ratio={ratio:.3f} contract_ratio={contract_ratio:.3f} rel_rms={rel_rms:.3e}")
    _log_parity(dict(what=what, path=path, max_abs=err.max().item(), ratio=ratio, contract_ratio=contract_ratio, rel_rms=rel_rms,
                     ref_absmax=ref64.abs().max().item(), numel=ref64.numel(), tol_scale=tol_scale,
                     need_atol_rtol2e3=(err - 2e-3 * ref64.abs()).max().item(), need_atol_rtol1e4=(err - 1e-4 * ref64.abs()).max().item()))
    assert ratio <= 1.0, f"{what}: path={path} max |err|/bound = {ratio:.3f} (max_abs {err.max().item():.3e})"
    assert rel_rms <= rrms, f"{what}: path={path} rel_rms {rel_rms:.3e} > {rrms}"


def make_layer(gf, dev, C, D, k, p, integration, norm, duplex, use_pos, exact, w, kmeans_iters=1, img2ltnt=False, num_heads=1):
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, norm=norm, kmeans=duplex, use_pos=use_pos,
                                 exact_fp32=exact, kmeans_iters=kmeans_iters, img2ltnt=img2ltnt, num_heads=num_heads).to(dev)
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].float())
    return attn


def run_layer(gf, dev, x64_nchw, y64, w, *, integration, norm, duplex, use_pos, exact, return_att=True, centroids=None,
              kmeans_iters=1, img2ltnt=False, num_heads=1):
    B, C, H, W = x64_nchw.shape
    k, D = y64.shape[1], y64.shape[2]
    p = w["pos_latent"].shape[1]
    attn = make_layer(gf, dev, C, D, k, p, integration, norm, duplex, use_pos, exact, w, kmeans_iters, img2ltnt, num_heads)
    x = x64_nchw.permute(0, 2, 3, 1).contiguous().float().to(dev)
    y = y64.float().to(dev)
    with torch.no_grad():
        out, att, cen = attn(x, y, return_att=return_att, centroids=centroids)
    torch.cuda.synchronize()
    return out, att, cen, gf._lib.last_path()


# ---------------------------------------------------------------------------------------------------------
# committed golden fixtures
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("idx", range(len(mg.cases())))
def test_layer_matches_golden(gf, cuda_dev, idx, exact):
    c = mg.cases()[idx]
    gold = np.load(GOLD)
    name = mg.case_name(c)
    x, y, w = mg.make_inputs(c, 100 + idx)
    norm = None if c["norm"] == "none" else c["norm"]
    out, att, cen, path = run_layer(gf, cuda_dev, x, y, w, integration=c["integration"], norm=norm, duplex=c["duplex"],
                                    use_pos=c["use_pos"], exact=exact, kmeans_iters=c.get("kmeans_iters", 1), img2ltnt=bool(c.get("img2ltnt")),
                                    num_heads=c.get("num_heads", 1))
    if exact:
        assert path == "simt_fp32"
    sel = torch.from_numpy(mg.out_sample_index(out.numel()))
    check_close(out.reshape(-1).cpu()[sel], torch.from_numpy(gold[name + "/out"]), path, name + "/out",
                tol_scale=1.5 if c.get("kmeans_iters", 1) > 1 else 1.0)
    a_atol = 1e-6 if path == "simt_fp32" else 2e-3
    assert (att.cpu().double() - torch.from_numpy(gold[name + "/att"]).double()).abs().max() <= a_atol + (1e-4 if exact else 5e-3)
    if c["duplex"]:
        check_close(cen, torch.from_numpy(gold[name + "/cen"]), gf._lib.last_centroid_path(), name + "/cen")


# ---------------------------------------------------------------------------------------------------------
# live oracle on the layer shapes of the generator (SURVEY 8a) at small batch + ragged / edge shapes
# ---------------------------------------------------------------------------------------------------------
SHAPES = [
    # (C, H, W, k, D, p, integration, norm)
    (512, 8, 8, 16, 32, 32, "mul", "layer"),       # res 8 of the 256^2 generator (n = 64 < one tile)
    (512, 16, 16, 16, 32, 32, "both", "layer"),
    (512, 32, 32, 8, 32, 32, "mul", "layer"),
    (256, 32, 16, 16, 32, 32, "mul", "layer"),      # C = 256 (res 128 layers), rectangular grid
    (256, 16, 16, 32, 32, 32, "both", "layer"),
    (128, 32, 32, 16, 32, 32, "mul", "layer"),      # C = 128 (res 256 layers)
    (128, 32, 32, 32, 32, 32, "add", "layer"),
    (64, 32, 32, 16, 32, 32, "mul", "layer"),       # C = 64 (res 512 layers)
    (64, 16, 24, 5, 16, 8, "both", "none"),
    (32, 4, 4, 3, 8, 4, "mul", "layer"),            # tiny
    (96, 10, 13, 7, 12, 12, "both", "instance"),    # ragged: n = 130 not a multiple of the tile, odd C/32
    (64, 16, 16, 1, 16, 16, "mul", "batch"),        # single latent
]


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "C%d-%dx%d-k%d-%s-%s" % (s[0], s[1], s[2], s[3], s[6], s[7]))
def test_simplex_layer_vs_oracle(gf, cuda_dev, shape, exact):
    C, H, W, k, D, p, integration, norm = shape
    B = 2
    g = torch.Generator().manual_seed(C + H + k)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.3 + 0.2
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, False, seed=7, bias_std=0.4)
    nrm = None if norm == "none" else norm
    ref, ratt, _ = ob.transformer_layer(x, y, w, integration=integration, norm=nrm, return_att=True)
    out, att, _, path = run_layer(gf, cuda_dev, x, y, w, integration=integration, norm=nrm, duplex=False, use_pos=True, exact=exact)
    e_ref = TOLERANCES.get("e_ref", {}).get("simplex/" + "C%d-%dx%d-k%d-%s-%s" % (C, H, W, k, integration, norm), 0.0)
    check_close(out, ref.permute(0, 2, 3, 1), path, "simplex", e_ref=e_ref)
    assert att.shape == (B, k, H, W)
    assert (att.cpu().double() - ratt).abs().max() <= (1e-5 if path == "simt_fp32" else 5e-3)
    assert (att.sum(dim=1) - 1).abs().max() < 1e-5


@pytest.mark.parametrize("C,H,W,k,B,integration", [(512, 64, 64, 16, 32, "mul"),    # the res-64 layer of config 2: two-pass, ~7 tiles/CTA
                                                    (512, 32, 32, 16, 40, "mul"),    # two-pass, 320 tiles: 2-3 tiles per CTA
                                                    (128, 16, 16, 8, 200, "both"),   # 2 tiles per image: K'/V reloads inside a CTA
                                                    (256, 16, 32, 32, 70, "mul"),    # ring barely larger than a tile
                                                    (64, 32, 32, 16, 37, "add")])
def test_persistent_schedule_many_tiles(gf, cuda_dev, C, H, W, k, B, integration):
    """More tiles than SMs: every CTA walks several tiles, crosses image boundaries (K'/V^T reload) and wraps the
    slab ring; checked against the fp64 oracle, with the attention map."""
    D = p = 32
    g = torch.Generator().manual_seed(C + B)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.2 + 0.1
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, False, seed=17, bias_std=0.3)
    ref, ratt, _ = ob.transformer_layer(x, y, w, integration=integration, return_att=True)
    out, att, _, path = run_layer(gf, cuda_dev, x, y, w, integration=integration, norm="layer", duplex=False, use_pos=True, exact=False)
    assert path == "wgmma_tf32"
    check_close(out, ref.permute(0, 2, 3, 1), path, "many-tiles")
    assert (att.cpu().double() - ratt).abs().max() <= 5e-3


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[1], SHAPES[2], SHAPES[3], SHAPES[5], SHAPES[6], SHAPES[8], SHAPES[10]],
                         ids=lambda s: "C%d-%dx%d-k%d-%s-%s" % (s[0], s[1], s[2], s[3], s[6], s[7]))
def test_duplex_layer_vs_oracle(gf, cuda_dev, shape, exact):
    C, H, W, k, D, p, integration, norm = shape
    B = 2
    g = torch.Generator().manual_seed(C + H + k + 1)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.3 + 0.2
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, True, seed=8, bias_std=0.4)
    nrm = None if norm == "none" else norm
    ref, ratt, rcen = ob.transformer_layer(x, y, w, integration=integration, norm=nrm, duplex=True, return_att=True)
    out, att, cen, path = run_layer(gf, cuda_dev, x, y, w, integration=integration, norm=nrm, duplex=True, use_pos=True, exact=exact)
    cpath = gf._lib.last_centroid_path()                            # pass A: wgmma TF32 where eligible, else CUDA cores
    if exact:
        assert cpath == "simt_fp32"
    check_close(cen, rcen, cpath, "duplex/centroids")
    # two chained [B*k, C] x [C, C] fp32 products sit between pass A and the keys: fp32 mode gets 2x the layer tolerance
    check_close(out, ref.permute(0, 2, 3, 1), path, "duplex/out", tol_scale=2.0 if path == "simt_fp32" else 1.0)
    # iterative=True: centroids fed back in skip pass A and reproduce the same output
    out2, _, cen2, _ = run_layer(gf, cuda_dev, x, y, w, integration=integration, norm=nrm, duplex=True, use_pos=True, exact=exact,
                                 centroids=cen.clone())
    assert torch.equal(cen2, cen)
    assert (out2 - out).abs().max() <= 1e-6 * max(1.0, out.abs().max().item())
    # need_centroids=False: keys straight from the attention-weighted means (centroid projection folded at stage W)
    attn = make_layer(gf, cuda_dev, C, D, k, p, integration, nrm, True, True, exact, w)
    with torch.no_grad():
        out3, _, cen3 = attn(x.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), y.float().to(cuda_dev), need_centroids=False)
    assert cen3 is None
    check_close(out3, ref.permute(0, 2, 3, 1), path, "duplex/no-centroids", tol_scale=2.0 if path == "simt_fp32" else 1.0)


@pytest.mark.parametrize("duplex", [False, True], ids=["simplex", "duplex"])
@pytest.mark.parametrize("C,H,W,k,B,integration", [(512, 8, 8, 32, 5, "mul"),     # res-8 layers of config 3: one 64-token image per tile
                                                    (512, 8, 8, 16, 33, "both"),    # config 2, more images than a wave of two-pass CTAs needs
                                                    (128, 4, 8, 8, 3, "add"),       # n = 32
                                                    (64, 8, 8, 16, 150, "mul")])    # more short tiles than SMs
def test_short_tiles_small_grid(gf, cuda_dev, C, H, W, k, B, integration, duplex):
    """Grids smaller than one 128-token tile (8x8, 4x8) run on the tensor path with one image per tile: rows past the
    image are never stored (stage T) / carry zero weight (pass A); the last image's box runs past the tensor (TMA zero fill)."""
    D = p = 32
    g = torch.Generator().manual_seed(C + B + k)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.2 + 0.1
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, duplex, seed=19, bias_std=0.3)
    ref, ratt, rcen = ob.transformer_layer(x, y, w, integration=integration, duplex=duplex, return_att=True)
    out, att, cen, path = run_layer(gf, cuda_dev, x, y, w, integration=integration, norm="layer", duplex=duplex, use_pos=True, exact=False)
    assert path == "wgmma_tf32"
    check_close(out, ref.permute(0, 2, 3, 1), path, "short-tiles")
    assert (att.cpu().double() - ratt).abs().max() <= 5e-3
    if duplex:
        assert gf._lib.last_centroid_path() == "wgmma_tf32"
        check_close(cen, rcen, gf._lib.last_centroid_path(), "short-tiles/centroids")


def test_prepare_then_token_stage_equals_one_call(gf, cuda_dev):
    """BipartiteAttention.prepare (stages W + I, needs only the latents) followed by stage='token' reproduces the single call
    bit for bit, including the folded load-side scale."""
    torch.manual_seed(4)
    attn = gf.BipartiteAttention(128, 32, 16).to(cuda_dev)
    x = torch.randn(3, 16, 16, 128, device=cuda_dev)
    y = torch.randn(3, 16, 32, device=cuda_dev)
    d = torch.rand(3, 128, device=cuda_dev) + 0.5
    post = dict(bias=torch.randn(128, device=cuda_dev), act="lrelu", gain=1.4, in_scale=d)
    with torch.no_grad():
        want, _, _ = attn(x, y, postop=post)
        want = want.clone()
        attn.prepare(y * 0 + 1.0, tuple(x.shape), in_scale=d)          # clobber the tables, then prepare for real
        attn.prepare(y, tuple(x.shape), in_scale=d)
        got, _, _ = attn(x, y, postop=post, stage="token")
    assert torch.equal(got, want)


def test_inplace_and_no_att(gf, cuda_dev):
    C, H, W, k, D, p = 128, 16, 16, 16, 32, 32
    g = torch.Generator().manual_seed(5)
    x64 = torch.randn(2, C, H, W, generator=g, dtype=torch.float64)
    y64 = torch.randn(2, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, "mul", False, seed=9)
    for exact in (True, False):
        attn = make_layer(gf, cuda_dev, C, D, k, p, "mul", "layer", False, True, exact, w)
        x = x64.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev)
        y = y64.float().to(cuda_dev)
        with torch.no_grad():
            ref, att, _ = attn(x, y)
            assert att is None
            xin = x.clone()
            out, _, _ = attn(xin, y, out=xin)          # Xout aliases X
        assert out.data_ptr() == xin.data_ptr()
        assert torch.equal(out, ref)


def test_functional_transformer_layer(gf, cuda_dev):
    """The reference-named functional entry point: [B, from_len, dim] tokens in, (tokens', att_probs, att_vars) out."""
    C, H, W, k, D, p = 64, 8, 16, 4, 16, 16
    g = torch.Generator().manual_seed(11)
    x64 = torch.randn(2, C, H, W, generator=g, dtype=torch.float64)
    y64 = torch.randn(2, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, "mul", True, seed=3, bias_std=0.2)
    ref, ratt, rcen = ob.transformer_layer(x64, y64, w, duplex=True, return_att=True)
    params = {n: t.float().to(cuda_dev) for n, t in w.items()}
    tokens = x64.permute(0, 2, 3, 1).reshape(2, H * W, C).contiguous().float().to(cuda_dev)
    out, att_probs, att_vars = gf.transformer_layer(C, p, tokens, y64.float().to(cuda_dev), H * W, k, params, grid_shape=(H, W),
                                                    kmeans=True, exact_fp32=True)
    check_close(out.reshape(2, H, W, C), ref.permute(0, 2, 3, 1), "simt_fp32", "functional")
    assert att_probs.shape == (2, H * W, k)
    assert (att_probs.cpu().double() - ratt.reshape(2, k, H * W).transpose(1, 2)).abs().max() < 1e-5
    check_close(att_vars["centroids"], rcen, "simt_fp32", "functional/centroids")


def test_errors_are_loud(gf, cuda_dev):
    attn = gf.BipartiteAttention(64, 16, 4).to(cuda_dev)
    x = torch.randn(1, 8, 16, 64, device=cuda_dev)
    y = torch.randn(1, 4, 16, device=cuda_dev)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="float32"):
            attn(x.half(), y)
        with pytest.raises(RuntimeError, match="contiguous"):
            attn(x.transpose(1, 2), y)
        with pytest.raises(ValueError):
            attn(x, y[:, :, :8].contiguous().reshape(2, 4, 4))
    a2 = gf.BipartiteAttention(64, 16, 4, num_heads=8).to(cuda_dev)            # 8 heads x 8 columns > 32 table columns
    with torch.no_grad(), pytest.raises(RuntimeError, match="num_heads"):
        a2(x, y)
    a3 = gf.BipartiteAttention(64, 16, 4, num_heads=2, kmeans=True).to(cuda_dev)   # multi-head duplex: not built
    with torch.no_grad(), pytest.raises(RuntimeError, match="num_heads"):
        a3(x, y)


# ---------------------------------------------------------------------------------------------------------
# full-size, size-independent properties (BASELINE config-2 layer shape: 256x256 grid, C = 128, k = 16)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
def test_full_size_properties(gf, cuda_dev, exact):
    C, H, W, k, D, p, B = 128, 256, 256, 16, 32, 32, 4
    torch.manual_seed(0)
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, exact_fp32=exact).to(cuda_dev)
    x = torch.randn(B, H, W, C, device=cuda_dev) * 1.2 + 0.1
    y = torch.randn(B, k, D, device=cuda_dev)
    with torch.no_grad():
        out, att, _ = attn(x, y, return_att=True)
        # (1) attention rows are probability vectors
        assert (att.sum(dim=1) - 1).abs().max() < 2e-5 and att.min() >= 0
        # (2) batch independence, bit for bit (basis of the data-parallel sharding)
        out1, _, _ = attn(x[2:3].contiguous(), y[2:3].contiguous())
        assert torch.equal(out1[0], out[2])
        # (3) run-to-run determinism
        out_b, _, _ = attn(x, y)
        assert torch.equal(out_b, out)
        # (4) modulation identity: x' / LN(x) is the gain; for layer norm + "mul" the gain of a token depends on x only
        #     through its attention row, so tokens with (numerically) one-hot attention on the same latent share it
        mu = x.mean(dim=3, keepdim=True)
        xn = (x - mu) * torch.rsqrt(((x - mu) ** 2).mean(dim=3, keepdim=True) + 1e-8)
        assert torch.isfinite(out).all()
        # (5) latent-permutation equivariance
        perm = torch.randperm(k, device=cuda_dev)
        attn2 = gf.BipartiteAttention(C, D, k, pos_dim=p, exact_fp32=exact).to(cuda_dev)
        attn2.load_state_dict(attn.state_dict())
        attn2.pos_latent.copy_(attn.pos_latent[perm])
        out_p, att_p, _ = attn2(x, y[:, perm].contiguous(), return_att=True)
        tol = 1e-4 if exact else 2e-2
        assert (out_p - out).abs().max() <= tol * max(1.0, out.abs().max().item())
        assert (att_p - att[:, perm]).abs().max() <= (1e-5 if exact else 5e-3)
        del xn


# ---------------------------------------------------------------------------------------------------------
# end-to-end generator vs the oracle generator
# ---------------------------------------------------------------------------------------------------------
def _small_generator(gf, dev, exact, **kw):
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4,
                     exact_fp32=exact, **kw)
    with torch.no_grad():
        for n, prm in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo", "bq2", "bk2", "bv2"):
                prm.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                prm.fill_(0.1)
    return G.to(dev).eval()


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("duplex", [False, True], ids=["simplex", "duplex"])
def test_generator_end_to_end(gf, cuda_dev, duplex, exact):
    """BASELINE config 1 shape class (64x64, k = 8, B = 4): same generator call, activations within tolerance."""
    G = _small_generator(gf, cuda_dev, exact, kmeans=duplex)
    assert G.synthesis.num_attention_layers == 8
    g = torch.Generator().manual_seed(1)
    z = torch.randn(4, 9, 32, generator=g)
    with torch.no_grad():
        img, atts = G(z.to(cuda_dev), return_att=True)
    ref, ratts, rfeats = og.generator_forward(G.state_dict(), z, resolution=64, components_num=8, latent_dim=32, duplex=duplex,
                                              mapping_layers=4, return_att=True, return_features=True)
    assert img.shape == (4, 3, 64, 64) and len(atts) == 8
    check_image(img, ref, "fp32" if exact else "tf32", f"e2e-64/duplex={duplex}")
    e2e = TOLERANCES["e2e"]["simt_fp32" if exact else "wgmma_tf32"]
    for a, r in zip(atts, ratts):
        assert (a.double().cpu() - r).abs().max() <= e2e["att_abs"]


def check_image(img, ref64, mode, what, scale=1.0):
    """End-to-end image bound of SURVEY 8c, for an image whose range is set by random weights instead of [-1, 1]: the
    bounds are relative to the reference's peak |value|.  max-abs <= max_abs_rel_peak * peak, PSNR >= psnr_db, rel-RMS."""
    e2e = TOLERANCES["e2e"]["simt_fp32" if mode == "fp32" else "wgmma_tf32"]
    got, ref64 = img.detach().double().cpu(), ref64.detach().double().cpu()
    assert got.shape == ref64.shape and torch.isfinite(got).all()
    err = (got - ref64).abs()
    peak = max(1.0, ref64.abs().max().item())
    rmse = err.pow(2).mean().sqrt().item()
    rel_rms = rmse / ref64.pow(2).mean().sqrt().item()
    psnr = 20.0 * math.log10(peak / max(rmse, 1e-300))
    print(f"[e2e] {what} mode={mode} max_abs={err.max().item():.3e} peak={peak:.3f} max_abs/peak={err.max().item() / peak:.3e} "
          f"rel_rms={rel_rms:.3e} psnr={psnr:.1f} dB")
    _log_parity(dict(what=what, path="e2e-" + mode, max_abs=err.max().item(), peak=peak, rel_rms=rel_rms, psnr=psnr))
    assert err.max().item() <= scale * e2e["max_abs_rel_peak"] * peak, what
    assert rel_rms <= scale * e2e["rel_rms"], what
    assert psnr >= e2e["psnr_db"] - 20.0 * math.log10(scale), what


def _benchmark_generator(gf, dev, resolution, k, duplex, exact=False):
    """The generator of the BENCHMARKED configs: config-f channels (fmap_base 16384, fmap_max 512), D = 32, 8 mapping layers,
    N(0,1) weights (seed 0), live biases and noise strengths."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=resolution, components_num=k, latent_dim=32, kmeans=duplex, exact_fp32=exact)
    with torch.no_grad():
        for n, prm in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo", "bq2", "bk2", "bv2"):
                prm.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                prm.fill_(0.1)
    return G.to(dev).eval()


@pytest.mark.parametrize("cfg", [dict(id="config2", res=256, k=16, duplex=False, B=2, layers=12),
                                 dict(id="config3", res=256, k=32, duplex=True, B=2, layers=12),
                                 dict(id="config5", res=512, k=32, duplex=False, B=1, layers=14)], ids=lambda c: c["id"])
def test_benchmarked_generators_vs_oracle(gf, cuda_dev, cfg):
    """The generators bench.py times (BASELINE configs[1], [2], [4]: 256^2 K=16 simplex, 256^2 K=32 duplex, 512^2 K=32) at a
    small batch against oracle/generator.py in float64: the image (max-abs / PSNR / rel-RMS of tolerances.json "e2e"), every
    attention layer's activation (return_features) and every attention map.  The layer activations are CUMULATIVE (layer l
    sees the error of layers < l), so they are held to the end-to-end relative-RMS bound, not to the per-layer one."""
    G = _benchmark_generator(gf, cuda_dev, cfg["res"], cfg["k"], cfg["duplex"])
    assert G.synthesis.num_attention_layers == cfg["layers"]
    z = torch.randn(cfg["B"], cfg["k"] + 1, 32, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        img = G(z.to(cuda_dev)).clone()                                        # the benchmarked path (all fusions on)
        assert gf._lib.last_path() == "wgmma_tf32"
        if cfg["duplex"]:
            assert gf._lib.last_centroid_path() == "wgmma_tf32"
        img2, atts, feats = G(z.to(cuda_dev), return_att=True, return_features=True)
    ref, ratts, rfeats = og.generator_forward(G.state_dict(), z, resolution=cfg["res"], components_num=cfg["k"], latent_dim=32,
                                              duplex=cfg["duplex"], return_att=True, return_features=True)
    check_image(img, ref, "tf32", cfg["id"] + "/image")
    check_image(img2, ref, "tf32", cfg["id"] + "/image-features-path")
    e2e = TOLERANCES["e2e"]["wgmma_tf32"]
    assert len(feats) == len(rfeats) == cfg["layers"] and len(atts) == cfg["layers"]
    for li, (f, r) in enumerate(zip(feats, rfeats)):
        f = f.double().cpu()
        err = (f - r).abs()
        rel_rms = (err.pow(2).mean().sqrt() / r.pow(2).mean().sqrt()).item()
        peak = r.abs().max().item()
        print(f"[e2e] {cfg['id']}/layer{li} {tuple(r.shape)} rel_rms={rel_rms:.3e} max_abs/peak={err.max().item() / peak:.3e}")
        _log_parity(dict(what=f"{cfg['id']}/layer{li}", path="e2e-feat", max_abs=err.max().item(), peak=peak, rel_rms=rel_rms))
        assert rel_rms <= e2e["rel_rms"], (cfg["id"], li, rel_rms)
        assert err.max().item() <= e2e["max_abs_rel_peak"] * peak, (cfg["id"], li)
    for li, (a, r) in enumerate(zip(atts, ratts)):
        d = (a.double().cpu() - r).abs().max().item()
        _log_parity(dict(what=f"{cfg['id']}/att{li}", path="e2e-att", max_abs=d))
        assert d <= e2e["att_abs"], (cfg["id"], li, d)


def test_native_ops_match_oracle_generator(gf, cuda_dev):
    """The native companions of the hot path (gf_ops.h: up-FIR blur, skip upsampling, activation-scaling mod-conv with deferred
    demodulation, polyphase up-convolution, tRGB) against the INDEPENDENT definitions of oracle/generator.py (_upfirdn,
    _modconv: per-sample modulated weights + grouped convolution, the reference's formulation), float64."""
    from importlib import import_module
    ops = import_module("gansformer-reproducibility-challenge_b200.ops")
    nets = import_module("gansformer-reproducibility-challenge_b200.networks")
    g = torch.Generator().manual_seed(0)
    f32 = ops.fir_filter(cuda_dev)
    f64 = og._fir(torch.float64)
    for (B, I, O, H, W) in [(2, 64, 32, 8, 8), (3, 128, 128, 16, 12), (2, 256, 512, 9, 7)]:
        x = torch.randn(B, I, H, W, generator=g)
        wt = torch.randn(O, I, 3, 3, generator=g)
        st = torch.randn(B, I, generator=g) + 1.0
        xc = x.to(cuda_dev).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            for up in (1, 2):
                phases = ops.upconv_phase_weights((wt * (1.0 / math.sqrt(I * 9))).to(cuda_dev)) if up == 2 else None
                got = nets.modulated_conv2d(xc, wt.to(cuda_dev), st.to(cuda_dev), up=up, f=f32, phases=phases)
                want = og._modconv(x.double(), wt.double(), st.double(), up=up, f=f64)
                assert got.shape == want.shape
                d = (got.double().cpu() - want).abs().max().item()
                print(f"[ops] modconv up={up} B={B} I={I} O={O} max_abs={d:.3e} peak={want.abs().max().item():.2f}")
                assert d <= 2e-5 * max(1.0, want.abs().max().item())          # fp32 cuDNN (allow_tf32 off in the fixture)
            # deferred demodulation (what the attention kernel's load side consumes): conv output * d == demodulated output
            raw, dd = nets.modulated_conv2d(xc, wt.to(cuda_dev), st.to(cuda_dev), up=1, f=f32, defer_demod=True)
            want = og._modconv(x.double(), wt.double(), st.double(), up=1, f=f64)
            assert ((raw * dd[:, :, None, None]).double().cpu() - want).abs().max() <= 2e-5 * max(1.0, want.abs().max().item())
            # skip-connection upsampling (upfirdn up=2) with the add
            img = torch.randn(B, 3, H, W, generator=g)
            add = torch.randn(B, 3, 2 * H, 2 * W, generator=g)
            got = ops.upsample2x(img.to(cuda_dev), f32, add=add.to(cuda_dev))
            want = og._upfirdn(img.double(), f64, up=2, pad=(2, 1, 2, 1), gain=4.0) + add.double()
            assert (got.double().cpu() - want).abs().max() < 1e-5
            # blur after a transposed convolution (upfirdn pad 1, gain 4) with a per-(b, c) scale
            t = torch.randn(B, O, 2 * H + 1, 2 * W + 1, generator=g)
            sc = torch.rand(B, O, generator=g) + 0.5
            got = ops.blur_up(t.to(cuda_dev).contiguous(memory_format=torch.channels_last), f32, scale=sc.to(cuda_dev))
            want = og._upfirdn(t.double(), f64, pad=(1, 1, 1, 1), gain=4.0) * sc.double()[:, :, None, None]
            assert (got.double().cpu() - want).abs().max() < 1e-5
            # tRGB = 1x1 modulated conv without demodulation + bias
            wr = torch.randn(3, I, 1, 1, generator=g)
            br = torch.randn(3, generator=g)
            got = ops.torgb(xc, wr.to(cuda_dev), st.to(cuda_dev), br.to(cuda_dev))
            want = og._modconv(x.double(), wr.double(), st.double(), demodulate=False) + br.double()[None, :, None, None]
            assert (got.double().cpu() - want).abs().max() <= 1e-5 * max(1.0, want.abs().max().item())


def test_run_wrapper_minibatches(gf, cuda_dev):
    G = _small_generator(gf, cuda_dev, True)
    z = torch.randn(5, 9, 32)
    imgs = G.run(z.numpy(), truncation_psi=1.0, randomize_noise=False, minibatch_size=2)
    with torch.no_grad():
        ref = G(z.to(cuda_dev)).cpu()
    assert imgs.shape == (5, 3, 64, 64)
    # cuDNN may pick different algorithms for minibatch 2 vs 5: equal up to fp32 rounding, not bit for bit
    assert (imgs - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())


def test_cuda_graph_replay_matches_eager(gf, cuda_dev):
    """Generator.graphed / run(cuda_graph=True): the captured graph reproduces the eager forward for new latents."""
    G = _small_generator(gf, cuda_dev, False)
    g = torch.Generator().manual_seed(3)
    z1, z2 = torch.randn(4, 9, 32, generator=g), torch.randn(4, 9, 32, generator=g)
    with torch.no_grad():
        e1, e2 = G(z1.to(cuda_dev)).clone(), G(z2.to(cuda_dev)).clone()
        replay = G.graphed(4)
        r1 = replay(z1.to(cuda_dev)).clone()
        r2 = replay(z2.to(cuda_dev)).clone()
    # cuDNN may pick a different (capture-safe) TF32 algorithm inside the graph: TF32-level tolerance, not bit equality
    tol = 1e-3 * max(1.0, e1.abs().max().item())
    print(f"[graph] d1={(r1 - e1).abs().max().item():.3e} d2={(r2 - e2).abs().max().item():.3e} d12={(r1 - r2).abs().max().item():.3e} tol={tol:.3e}")
    assert (r1 - e1).abs().max() <= tol and (r2 - e2).abs().max() <= tol
    assert (r1 - r2).abs().max() > 20 * tol                   # the graph really recomputed for the new latents
    host = G.run(z2.numpy(), minibatch_size=4, cuda_graph=True)
    assert (host - e2.cpu()).abs().max() <= tol


@pytest.mark.parametrize("C,H,W,k,D,p,integration,norm,duplex", [
    (64, 8, 16, 4, 16, 16, "both", "layer", False),       # backward kernel: KP = 16, one full tile per image
    (96, 10, 13, 20, 12, 8, "mul", "layer", False),       # KP = 32, ragged n = 130, odd C / 32
    (128, 16, 16, 16, 32, 32, "add", "none", False),      # no normalisation, additive integration
    (64, 8, 8, 8, 16, 16, "mul", "layer", True),          # duplex: composite torch-autograd backward
])
def test_autograd_matches_oracle(gf, cuda_dev, C, H, W, k, D, p, integration, norm, duplex):
    """Training path: forward = CUDA kernels; backward = gf_attn_simplex_bwd + batched GEMMs + autograd over the per-image
    tables (simplex, layer norm / none) or the torch composite (duplex); gradients vs the fp64 oracle."""
    g = torch.Generator().manual_seed(21)
    x64 = (torch.randn(2, C, H, W, generator=g, dtype=torch.float64)).requires_grad_(True)
    y64 = torch.randn(2, k, D, generator=g, dtype=torch.float64).requires_grad_(True)
    w = {n: t.requires_grad_(True) for n, t in ob.init_params(C, D, k, p, integration, duplex, seed=4, bias_std=0.3).items()}
    nrm = None if norm == "none" else norm
    ref, _, _ = ob.transformer_layer(x64, y64, w, integration=integration, norm=nrm, duplex=duplex)
    gout = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(gout)
    attn = make_layer(gf, cuda_dev, C, D, k, p, integration, nrm, duplex, True, True, {n: t.detach() for n, t in w.items()})
    x = x64.detach().permute(0, 2, 3, 1).contiguous().float().to(cuda_dev).requires_grad_(True)
    y = y64.detach().float().to(cuda_dev).requires_grad_(True)
    launches0 = gf._lib.launch_count()
    out, _, _ = attn(x, y)
    fwd_launches = gf._lib.launch_count() - launches0
    out.backward(gout.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev))
    bwd_launches = gf._lib.launch_count() - launches0 - fwd_launches
    assert bwd_launches == (0 if duplex else 1)                       # the hand-written kernel ran (simplex) / composite (duplex)
    check_close(out, ref.detach().permute(0, 2, 3, 1), "simt_fp32", "autograd/forward", tol_scale=2.0 if duplex else 1.0)

    def rel(a, b):
        return ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30)).item()
    assert rel(x.grad, x64.grad.permute(0, 2, 3, 1)) < 1e-4
    assert rel(y.grad, y64.grad) < 1e-4
    names = ("wq", "wv", "wo", "bo", "pos_latent", "wpq", "bq", "bv") + (("wkc", "wq2", "wk2", "wv2") if duplex else ("wk", "bk", "wpk"))
    for n in names:
        if w[n].grad is None:
            continue
        if w[n].grad.norm() < 1e-9:           # e.g. bk: constant over the latents, the softmax cancels it -- only round-off
            assert getattr(attn, n).grad.norm().item() < 1e-3, n
            continue
        assert rel(getattr(attn, n).grad, w[n].grad) < 2e-4, n


# ---------------------------------------------------------------------------------------------------------
# fused post-op (noise + bias + leaky-ReLU on the attention store) and the native companion ops (gf_ops.h)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("scales", [False, True], ids=["plain", "scales"])
@pytest.mark.parametrize("duplex", [False, True], ids=["simplex", "duplex"])
@pytest.mark.parametrize("C,H,W,k,random_noise", [(128, 16, 16, 16, False), (256, 16, 8, 8, True), (512, 8, 8, 4, False), (512, 16, 16, 16, False)])
def test_attention_postop(gf, cuda_dev, C, H, W, k, random_noise, exact, scales, duplex):
    """Fused load side (demodulation scale) and store side (noise + bias + lrelu + next style scale) vs the oracle."""
    D = p = 16
    B = 3
    g = torch.Generator().manual_seed(C + k)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    d_in = (torch.rand(B, C, generator=g, dtype=torch.float64) + 0.5) if scales else None
    ps = (torch.randn(B, C, generator=g, dtype=torch.float64) + 1.0) if scales else None
    x_raw = x64
    if scales:
        x64 = x64 * d_in[:, :, None, None]
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    bias = torch.randn(C, generator=g, dtype=torch.float64) * 0.5
    noise = torch.randn((B, 1, H, W) if random_noise else (H, W), generator=g, dtype=torch.float64)
    strength = torch.tensor(0.37, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, "both", duplex, seed=5, bias_std=0.3)
    ref, _, rcen = ob.transformer_layer(x64, y64, w, integration="both", duplex=duplex)
    ref = ref + noise * strength + bias[None, :, None, None]
    ref = torch.nn.functional.leaky_relu(ref, 0.2) * math.sqrt(2.0)
    if scales:
        ref = ref * ps[:, :, None, None]
    attn = make_layer(gf, cuda_dev, C, D, k, p, "both", "layer", duplex, True, exact, w)
    post = dict(bias=bias.float().to(cuda_dev), noise=noise.float().to(cuda_dev), strength=strength.float().to(cuda_dev),
                act="lrelu", gain=math.sqrt(2.0))
    if scales:   # pass them as column slices of a wider matrix, as the generator does (row stride != C)
        wide = torch.zeros(B, 2 * C + 8, device=cuda_dev)
        wide[:, 8:8 + C] = d_in.float().to(cuda_dev)
        wide[:, 8 + C:] = ps.float().to(cuda_dev)
        post.update(in_scale=wide[:, 8:8 + C], post_scale=wide[:, 8 + C:])
    with torch.no_grad():
        out, _, cen = attn(x_raw.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), y64.float().to(cuda_dev), postop=post)
    # with the per-channel scales the error of the block is multiplied by |post_scale| (up to ~4): tolerance x2
    # (x2 again for duplex in fp32 mode: two chained [B*k, C] x [C, C] products between pass A and the keys)
    check_close(out, ref.permute(0, 2, 3, 1), gf._lib.last_path(), "postop",
                tol_scale=(2.0 if scales else 1.0) * (2.0 if (duplex and exact) else 1.0))
    if duplex:                                   # the load-side scale reaches the latents' view of the image too
        check_close(cen, rcen, gf._lib.last_centroid_path(), "postop/centroids")


def test_native_ops_match_definitions(gf, cuda_dev):
    """gf_ops.h kernels vs their plain-torch definitions (ops.py *_ref / torch path), fp32, channels-last inputs."""
    from importlib import import_module
    ops = import_module("gansformer-reproducibility-challenge_b200.ops")
    g = torch.Generator().manual_seed(0)
    f = ops.fir_filter(cuda_dev)
    for (B, C, H, W) in [(2, 64, 8, 8), (3, 128, 16, 12), (1, 32, 4, 4), (2, 512, 40, 36), (2, 256, 33, 32)]:
        x = torch.randn(B, C, 2 * H + 1, 2 * W + 1, generator=g).to(cuda_dev).contiguous(memory_format=torch.channels_last)
        s = torch.rand(B, C, generator=g).to(cuda_dev) + 0.5
        with torch.no_grad():
            got = ops.blur_up(x, f, scale=s)
        want = ops.upfirdn2d_ref(x.double(), f.double(), pad=(1, 1, 1, 1), gain=4.0) * s.double()[:, :, None, None]
        assert got.shape == (B, C, 2 * H, 2 * W)
        assert (got.double() - want).abs().max() < 1e-5
        xs = torch.randn(B, C, H, W, generator=g).to(cuda_dev).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            assert torch.equal(ops.chan_scale(xs, s), xs * s[:, :, None, None])
            wide = torch.rand(B, C + 8, generator=g).to(cuda_dev)
            assert torch.equal(ops.chan_scale(xs, wide[:, 4:4 + C]), xs * wide[:, 4:4 + C, None, None])     # strided rows
            wsq = torch.rand(48, C, generator=g).to(cuda_dev)
            dd = ops.demod_coef(wide[:, 4:4 + C], wsq)
            want_d = torch.rsqrt(wide[:, 4:4 + C].double().square() @ wsq.double().t() + 1e-8)
            assert (dd.double() - want_d).abs().max() <= 1e-5 * want_d.abs().max()
            # every layer of a network in one launch: bit-identical to the per-layer call (same summation order)
            wsq2 = torch.rand(20, C, generator=g).to(cuda_dev)
            wsq3 = torch.rand(7, C + 8, generator=g).to(cuda_dev)
            batch = ops.demod_coef_batch([(wide[:, 4:4 + C], wsq), (s, wsq2), (wide, wsq3)])
            for got_d, (s_, w_) in zip(batch, [(wide[:, 4:4 + C], wsq), (s, wsq2), (wide, wsq3)]):
                assert torch.equal(got_d, ops.demod_coef(s_, w_))
            bias = torch.randn(C, generator=g).to(cuda_dev)
            nz = torch.randn(H, W, generator=g).to(cuda_dev)
            st = torch.tensor(0.3, device=cuda_dev)
            got = ops.bias_act(xs, bias, "lrelu", noise=nz, strength=st)
            want = torch.nn.functional.leaky_relu(xs + nz * st + bias[None, :, None, None], 0.2) * math.sqrt(2.0)
            assert (got - want).abs().max() < 1e-5
            # training form: native forward, masked-gradient backward (vs torch autograd through the definition)
        xg, bg, sg = xs.clone().requires_grad_(True), bias.clone().requires_grad_(True), st.clone().requires_grad_(True)
        yg = ops.bias_act(xg, bg, "lrelu", noise=nz, strength=sg)
        xr, br, sr = xs.double().clone().requires_grad_(True), bias.double().clone().requires_grad_(True), st.double().clone().requires_grad_(True)
        yr = torch.nn.functional.leaky_relu(xr + nz.double() * sr + br[None, :, None, None], 0.2) * math.sqrt(2.0)
        gyy = torch.randn(yg.shape, generator=g).to(cuda_dev)
        yg.backward(gyy); yr.backward(gyy.double())
        assert (yg.double() - yr).abs().max() < 1e-5 and (xg.grad.double() - xr.grad).abs().max() < 1e-5
        assert (bg.grad.double() - br.grad).abs().max() < 1e-3 * max(1.0, br.grad.abs().max().item())
        assert abs(sg.grad.item() - sr.grad.item()) < 1e-3 * max(1.0, abs(sr.grad.item()))
        with torch.no_grad():
            nzb = torch.randn(B, 1, H, W, generator=g).to(cuda_dev)
            got = ops.bias_act(xs, bias, "linear", noise=nzb, strength=None)
            assert (got - (xs + nzb + bias[None, :, None, None])).abs().max() < 1e-5
        with torch.no_grad():                                   # tRGB: 1x1 modulated conv, no demodulation, planar output
            wrgb = torch.randn(3, C, 1, 1, generator=g).to(cuda_dev)
            brgb = torch.randn(3, generator=g).to(cuda_dev)
            got = ops.torgb(xs, wrgb, wide[:, 4:4 + C], brgb)
            want = torch.einsum("bchw,oc,bc->bohw", xs.double(), wrgb.double().reshape(3, C), wide[:, 4:4 + C].double()) / math.sqrt(C) \
                + brgb.double()[None, :, None, None]
            assert got.shape == (B, 3, H, W) and got.is_contiguous()
            assert (got.double() - want).abs().max() <= 1e-5 * max(1.0, want.abs().max().item())
            got2, xs2 = ops.torgb(xs, wrgb, wide[:, 4:4 + C], brgb, next_styles=s)     # second output from the same read
            assert torch.equal(got2, got) and torch.equal(xs2, xs * s[:, :, None, None])
        with torch.no_grad():                                   # upsampling conv as four polyphase convolutions + blur
            wup = torch.randn(C, C, 3, 3, generator=g).to(cuda_dev) / math.sqrt(9 * C)
            got = ops.upconv_blur_phases(xs, ops.upconv_phase_weights(wup), scale=s, gain=4.0)
            T = torch.nn.functional.conv_transpose2d(xs.double(), wup.double().transpose(0, 1), stride=2)
            want = ops.upfirdn2d_ref(T, f.double(), pad=(1, 1, 1, 1), gain=4.0) * s.double()[:, :, None, None]
            assert got.shape == (B, C, 2 * H, 2 * W)
            assert (got.double() - want).abs().max() <= 2e-3 * max(1.0, want.abs().max().item())      # TF32 convolutions
        for pad in (1, 2):                                      # differentiable FIR: value, gradient and second-order term
            xf = xs.clone().requires_grad_(True)
            xr = xs.double().clone().requires_grad_(True)
            yf, yr = ops.fir4(xf, f, pad, gain=2.0), ops.upfirdn2d_ref(xr, f.double(), pad=(pad,) * 4, gain=2.0)
            assert yf.shape == yr.shape and (yf.double() - yr).abs().max() < 1e-5
            gyf = torch.randn(yf.shape, generator=g).to(cuda_dev)
            (gf1,) = torch.autograd.grad((yf * gyf).sum() + yf.square().sum(), xf, create_graph=True)
            (gr1,) = torch.autograd.grad((yr * gyf.double()).sum() + yr.square().sum(), xr, create_graph=True)
            assert (gf1.double() - gr1).abs().max() < 1e-4
            (gf2,) = torch.autograd.grad(gf1.square().sum(), xf)
            (gr2,) = torch.autograd.grad(gr1.square().sum(), xr)
            assert (gf2.double() - gr2).abs().max() < 1e-3 * max(1.0, gr2.abs().max().item())
        img = torch.randn(B, 3, H, W, generator=g).to(cuda_dev)
        add = torch.randn(B, 3, 2 * H, 2 * W, generator=g).to(cuda_dev)
        with torch.no_grad():
            got = ops.upsample2x(img, f, add=add)
        want = ops.upfirdn2d_ref(img.double(), f.double(), up=2, pad=(2, 1, 2, 1), gain=4.0) + add.double()
        assert (got.double() - want).abs().max() < 1e-5


def test_training_step_runs_on_gpu(gf, cuda_dev):
    """SURVEY row f2 / BASELINE configs[3] shape class at 64x64: one D + G update with the attention layers' CUDA forward
    and composite backward; every generator parameter (attention weights included) receives a finite gradient."""
    from importlib import import_module
    tr = import_module("gansformer-reproducibility-challenge_b200.training")
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4).to(cuda_dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128).to(cuda_dev)
    trainer = tr.Trainer(G, D)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(4, 9, 32, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(cuda_dev)
    before = {n: p.detach().clone() for n, p in G.named_parameters()}
    st = trainer.step(z, reals)
    assert math.isfinite(st.loss_g) and math.isfinite(st.loss_d) and st.r1 > 0
    moved = [n for n, p in G.named_parameters() if (p.detach() - before[n]).abs().max() > 0]
    assert any(".attention." in n for n in moved), "attention parameters did not train"
    assert all(torch.isfinite(p).all() for p in G.parameters())
    st2 = trainer.step(z, reals)
    assert math.isfinite(st2.loss_g) and st2.r1 == 0


def test_generator_512_config5_shape_class(gf, cuda_dev):
    """BASELINE configs[4] shape class: 512x512 synthesis, K = 32 latents (14 attention layers, C = 64 at the top), eager vs
    CUDA-graph replay, finite output; the last attention layer is checked against the oracle layer on its own input."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=512, components_num=32, latent_dim=32).to(cuda_dev).eval()
    assert G.synthesis.num_attention_layers == 14
    z = torch.randn(2, 33, 32, generator=torch.Generator().manual_seed(2)).to(cuda_dev)
    with torch.no_grad():
        img = G(z).clone()
        rep = G.graphed(2)(z).clone()
    assert img.shape == (2, 3, 512, 512) and torch.isfinite(img).all()
    assert gf._lib.last_path() == "wgmma_tf32"
    assert (img - rep).abs().max() <= 2e-3 * max(1.0, img.abs().max().item())
    layer = G.synthesis.layers[-1].attention                              # C = 64, 512x512 grid, k = 32
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 64, 512, 512, generator=g, dtype=torch.float64)
    y = torch.randn(1, 32, 32, generator=g, dtype=torch.float64)
    w = {n: p.detach().double().cpu() for n, p in layer.named_parameters()}
    ref, _, _ = ob.transformer_layer(x, y, w)
    with torch.no_grad():
        out, _, _ = layer(x.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), y.float().to(cuda_dev))
    check_close(out, ref.permute(0, 2, 3, 1), gf._lib.last_path(), "512/C64")


def test_training_step_graph_replay(gf, cuda_dev):
    """Trainer.step_graphed: the captured step (with and without the lazy R1 term) trains -- weights keep moving across
    replays (weight-derived tensors are recomputed inside the graph) and losses stay finite."""
    from importlib import import_module
    tr = import_module("gansformer-reproducibility-challenge_b200.training")
    torch.manual_seed(0)
    G = gf.Generator(resolution=64, components_num=8, latent_dim=32, fmap_base=2048, fmap_max=128, mapping_layers=4, att_dp=0.12).to(cuda_dev)
    D = tr.Discriminator(64, fmap_base=2048, fmap_max=128).to(cuda_dev)
    trainer = tr.Trainer(G, D, tr.TrainConfig(d_reg_interval=2))        # attention dropout on: the masks come from device state
    g = torch.Generator().manual_seed(5)
    z = torch.randn(4, 9, 32, generator=g).to(cuda_dev)
    reals = (torch.rand(4, 3, 64, 64, generator=g) * 2 - 1).to(cuda_dev)
    snaps, stats = [], []
    for i in range(5):
        stats.append(trainer.step_graphed(z, reals))
        snaps.append(torch.cat([p.detach().reshape(-1) for p in G.synthesis.layers[2].attention.parameters()]).clone())
    assert all(math.isfinite(s.loss_g) and math.isfinite(s.loss_d) for s in stats)
    assert [s.r1 > 0 for s in stats] == [True, False, True, False, True]
    for a, b in zip(snaps, snaps[1:]):
        assert (a - b).abs().max() > 0                       # every replay updates the attention weights
    # the fakes of the D step follow the updated generator: the fake logits' loss changes from replay to replay
    assert len({round(s.loss_d, 6) for s in stats}) > 1


@pytest.mark.parametrize("duplex", [False, True], ids=["simplex", "duplex"])
def test_batched_prologue_matches_per_layer(gf, cuda_dev, duplex, monkeypatch):
    """gf_attn_prologue_batch (stage I of every layer in one launch, then stage='token' per layer) produces the same bits as
    the per-layer calls: same arithmetic, same operation order."""
    G = _small_generator(gf, cuda_dev, False, kmeans=duplex)
    z = torch.randn(3, 9, 32, generator=torch.Generator().manual_seed(7)).to(cuda_dev)
    with torch.no_grad():
        G(z)                                           # warm-up: stage W (weight folding) runs once
        l0 = gf._lib.launch_count()
        a = G(z).clone()
        n_batched = gf._lib.launch_count() - l0
        monkeypatch.setenv("GF_NO_BATCH_PROLOGUE", "1")
        l0 = gf._lib.launch_count()
        b = G(z).clone()
        n_per_layer = gf._lib.launch_count() - l0
    assert torch.equal(a, b)
    assert n_batched < n_per_layer, (n_batched, n_per_layer)


def test_prologue_batch_api(gf, cuda_dev):
    """attention.prologue_batch over layers of different shapes (simplex + duplex) followed by stage='token' equals stage='all'."""
    from importlib import import_module
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    torch.manual_seed(3)
    specs = [(128, 16, 16, False), (512, 8, 8, True), (256, 16, 8, True), (64, 32, 32, False)]
    y = torch.randn(3, 16, 32, device=cuda_dev)
    layers, xs, scales, want = [], [], [], []
    with torch.no_grad():
        for C, H, W, dup in specs:
            m = gf.BipartiteAttention(C, 32, 16, kmeans=dup).to(cuda_dev)
            x = torch.randn(3, H, W, C, device=cuda_dev)
            d = torch.rand(3, C, device=cuda_dev) + 0.5
            post = dict(bias=torch.randn(C, device=cuda_dev), act="lrelu", gain=1.4, in_scale=d)
            w, _, _ = m(x, y, postop=post, need_centroids=False)
            layers.append(m); xs.append(x); scales.append((d, post)); want.append(w.clone())
        am.prologue_batch([(m, y * 0 + 1.0, tuple(x.shape), sc[0]) for m, x, sc in zip(layers, xs, scales)])   # clobber
        am.prologue_batch([(m, y, tuple(x.shape), sc[0]) for m, x, sc in zip(layers, xs, scales)])
        for m, x, sc, w in zip(layers, xs, scales, want):
            got, _, _ = m(x, y, postop=sc[1], stage="token", need_centroids=False)
            assert torch.equal(got, w), (m.dim, m.duplex)


@pytest.mark.parametrize("D,k,L,B", [(32, 16, 8, 5), (16, 4, 2, 3), (64, 3, 4, 37), (96, 1, 2, 2)])
def test_mapping_kernel_matches_definition(gf, cuda_dev, D, k, L, B):
    """gf_mapping_fwd (G_mapping as one kernel: pixel norm, L FC + leaky-ReLU layers per path, truncation lerp) against the
    module's float64 torch definition on the CPU, with and without truncation."""
    import copy
    from importlib import import_module
    nets = import_module("gansformer-reproducibility-challenge_b200.networks")
    torch.manual_seed(D + k)
    M = nets.MappingNetwork(D, k, num_layers=L)
    with torch.no_grad():
        for p in M.parameters():
            if p.dim() == 1:
                p.normal_(0, 30.0)               # biases carry lr_mul = 0.01: make them matter
        M.w_avg.normal_(0, 0.5)
    ref_mod = copy.deepcopy(M).double()
    Mg = M.to(cuda_dev).eval()
    z = torch.randn(B, k + 1, D, generator=torch.Generator().manual_seed(3))
    for psi in (1.0, 0.6):
        l0 = gf._lib.launch_count()
        with torch.no_grad():
            got = Mg(z.to(cuda_dev), truncation_psi=psi)
        assert gf._lib.launch_count() - l0 == 1                      # one launch of ours, nothing else
        want = ref_mod(z.double(), truncation_psi=psi)
        err = (got.double().cpu() - want).abs().max().item()
        assert err <= 2e-5 * max(1.0, want.abs().max().item()), (psi, err)


@pytest.mark.parametrize("C,H,W,k,duplex,integration", [(128, 16, 16, 16, False, "mul"), (256, 16, 8, 8, False, "both"), (64, 32, 32, 32, True, "mul"),
                                                          (128, 8, 8, 16, False, "add"), (256, 32, 32, 32, True, "mul"),
                                                          (512, 16, 16, 16, False, "mul"), (512, 8, 16, 8, True, "both")])
def test_fused_torgb_epilogue(gf, cuda_dev, C, H, W, k, duplex, integration):
    """Store-side fusion of the tRGB 1x1 modulated convolution (postop.rgb_*): the three planes are computed from the layer output
    BEFORE the next layer's style scale, which the stored activations carry; both against the float64 oracle."""
    D = p = 16
    B = 3
    g = torch.Generator().manual_seed(C + k + H)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    d_in = torch.rand(B, C, generator=g, dtype=torch.float64) + 0.5
    ps = torch.randn(B, C, generator=g, dtype=torch.float64) + 1.0
    bias = torch.randn(C, generator=g, dtype=torch.float64) * 0.5
    noise = torch.randn(H, W, generator=g, dtype=torch.float64)
    rgb_w = torch.randn(B, 3, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    rgb_b = torch.randn(3, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, duplex, seed=5, bias_std=0.3)
    ref, _, _ = ob.transformer_layer(x64 * d_in[:, :, None, None], y64, w, integration=integration, duplex=duplex)
    ref = torch.nn.functional.leaky_relu(ref + noise * 0.37 + bias[None, :, None, None], 0.2) * math.sqrt(2.0)
    ref_rgb = torch.einsum("bchw,boc->bohw", ref, rgb_w) + rgb_b[None, :, None, None]
    ref_out = ref * ps[:, :, None, None]
    attn = make_layer(gf, cuda_dev, C, D, k, p, integration, "layer", duplex, True, False, w)
    f = lambda t: t.float().to(cuda_dev)
    rgb_out = torch.full((B, 3, H, W), float("nan"), device=cuda_dev)
    post = dict(bias=f(bias), noise=f(noise), strength=torch.tensor(0.37, device=cuda_dev), act="lrelu", gain=math.sqrt(2.0),
                in_scale=f(d_in), post_scale=f(ps), rgb_w=f(rgb_w).contiguous(), rgb_bias=f(rgb_b), rgb_out=rgb_out)
    with torch.no_grad():
        out, _, _ = attn(x64.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), f(y64), postop=post, need_centroids=False)
    assert gf._lib.last_path() == "wgmma_tf32"
    check_close(out, ref_out.permute(0, 2, 3, 1), "wgmma_tf32", "torgb-epilogue/out", tol_scale=2.0)
    check_close(rgb_out, ref_rgb, "wgmma_tf32", "torgb-epilogue/rgb", tol_scale=2.0)
    # the CUDA-core path refuses the fusion loudly
    attn32 = make_layer(gf, cuda_dev, C, D, k, p, integration, "layer", duplex, True, True, w)
    with torch.no_grad(), pytest.raises(RuntimeError, match="tRGB"):
        attn32(x64.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), f(y64), postop=post, need_centroids=False)


def test_fused_torgb_refused_for_512_channels_and_32_latents(gf, cuda_dev):
    """C = 512 with k = 32: the two-pass ring has no room for the tRGB weights -- the call says so (SynthesisNetwork keeps the separate kernel)."""
    C, k, D = 512, 32, 16
    attn = make_layer(gf, cuda_dev, C, D, k, 16, "mul", "layer", False, True, False, ob.init_params(C, D, k, 16, "mul", False, seed=1))
    x = torch.randn(2, 8, 16, C, device=cuda_dev)
    post = dict(rgb_w=torch.randn(2, 3, C, device=cuda_dev), rgb_bias=torch.zeros(3, device=cuda_dev), rgb_out=torch.empty(2, 3, 8, 16, device=cuda_dev))
    with torch.no_grad(), pytest.raises(RuntimeError, match="tRGB"):
        attn(x, torch.randn(2, k, D, device=cuda_dev), postop=post, need_centroids=False)


def test_torgb_epilogue_matches_torgb_kernel(gf, cuda_dev, monkeypatch):
    """Generator with the tRGB fused into the attention store (default) vs the separate tRGB kernel: same image up to fp32 summation order."""
    G = _benchmark_generator(gf, cuda_dev, 128, 16, False)
    z = torch.randn(2, 17, 32, generator=torch.Generator().manual_seed(5)).to(cuda_dev)
    with torch.no_grad():
        G(z)
        l0 = gf._lib.launch_count(); a = G(z).clone(); n_fused = gf._lib.launch_count() - l0
        monkeypatch.setenv("GF_NO_TORGB_EPILOGUE", "1")
        l0 = gf._lib.launch_count(); b = G(z).clone(); n_sep = gf._lib.launch_count() - l0
    assert n_fused < n_sep
    assert (a - b).abs().max() <= 2e-5 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
def test_mapping_latent_self_attention(gf, cuda_dev, exact):
    """ltnt2ltnt=True: latent-to-latent attention after every mapping layer (the bipartite block on [B, k, 1, D]) -- mapping output
    and the generated image against the oracle generator."""
    torch.manual_seed(0)
    G = gf.Generator(resolution=32, components_num=8, latent_dim=32, fmap_base=1024, fmap_max=128, mapping_layers=3, ltnt2ltnt=True,
                     exact_fp32=exact)
    with torch.no_grad():
        for n, prm in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo"):
                prm.normal_(0, 0.3)
            if n.startswith("mapping.") and n.endswith("bias"):
                prm.normal_(0, 30.0)                     # lr_mul = 0.01
    G = G.to(cuda_dev).eval()
    assert len(G.mapping.self_att) == 3
    z = torch.randn(3, 9, 32, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ws = G.mapping(z.to(cuda_dev))
        assert gf._lib.last_path() == "simt_fp32"        # C = D = 32: the CUDA-core kernel serves the latent grid
        img = G(z.to(cuda_dev))
    ref = og.generator_forward(G.state_dict(), z, resolution=32, components_num=8, latent_dim=32, mapping_layers=3)
    # reference latents: run the oracle's mapping part by asking for a 4x4-only forward is not exposed; compare the image and
    # check that the self-attention changed the latents at all
    check_image(img, ref, "fp32" if exact else "tf32", "ltnt2ltnt/image")
    G2 = gf.Generator(resolution=32, components_num=8, latent_dim=32, fmap_base=1024, fmap_max=128, mapping_layers=3).to(cuda_dev).eval()
    G2.load_state_dict({n: v for n, v in G.state_dict().items() if not n.startswith("mapping.self_att")})
    with torch.no_grad():
        ws2 = G2.mapping(z.to(cuda_dev))
    assert (ws[:, :8] - ws2[:, :8]).abs().max() > 1e-3                       # the local latents changed ...
    assert (ws[:, 8] - ws2[:, 8]).abs().max() <= 1e-5 * max(1.0, ws2[:, 8].abs().max().item())    # ... the global one did not (torch path vs the fused kernel: fp32 rounding)


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("C,H,W,k,integration,iters,i2l", [(128, 16, 16, 16, "mul", 2, False), (64, 16, 24, 5, "both", 3, True),
                                                            (256, 16, 16, 32, "mul", 1, True), (512, 16, 16, 8, "add", 2, True),
                                                            (96, 10, 13, 7, "mul", 2, True)])
def test_kmeans_iters_and_img2ltnt(gf, cuda_dev, C, H, W, k, integration, iters, i2l, exact):
    """Duplex extensions (SURVEY A.3): kmeans_iters > 1 (later iterations take their queries from the previous centroids through wcq)
    and g_img2ltnt (latents modulated by the centroids before pass B), each against the fp64 oracle; with and without the centroids output."""
    D = p = 16
    B = 2
    g = torch.Generator().manual_seed(C + k + iters)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.2 + 0.1
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, True, seed=11, bias_std=0.3, extras=True)
    ref, ratt, rcen = ob.transformer_layer(x, y, w, integration=integration, duplex=True, return_att=True, kmeans_iters=iters, img2ltnt=i2l)
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, kmeans=True, kmeans_iters=iters, img2ltnt=i2l,
                                 exact_fp32=exact).to(cuda_dev)
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].float())
        xg, yg = x.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), y.float().to(cuda_dev)
        out, att, cen = attn(xg, yg, return_att=True)
        out2, _, cen2 = attn(xg, yg, need_centroids=False)
    path, cpath = gf._lib.last_path(), gf._lib.last_centroid_path()
    scale = (2.0 if path == "simt_fp32" else 1.0) * (1.5 if iters > 1 else 1.0)      # chained [B*k, C] x [C, C] products per iteration
    check_close(cen, rcen, cpath, "kmeans/centroids", tol_scale=scale)
    check_close(out, ref.permute(0, 2, 3, 1), path, "kmeans/out", tol_scale=scale)
    assert cen2 is None
    if iters > 1 or i2l:          # explicit centroids are computed internally: identical arithmetic
        assert torch.equal(out2, out)
    else:
        check_close(out2, ref.permute(0, 2, 3, 1), path, "kmeans/out-no-centroids", tol_scale=scale)
    assert (att.cpu().double() - ratt).abs().max() <= (1e-4 if path == "simt_fp32" else 5e-3)


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
@pytest.mark.parametrize("C,H,W,k,heads,integration,norm", [(128, 16, 16, 16, 2, "mul", "layer"), (256, 16, 16, 8, 4, "both", "layer"),
                                                             (512, 8, 8, 8, 2, "mul", "layer"), (64, 32, 32, 5, 2, "add", "none"),
                                                             (96, 10, 13, 7, 2, "mul", "instance"), (128, 32, 32, 16, 2, "mul", "layer")])
def test_multi_head_simplex(gf, cuda_dev, C, H, W, k, heads, integration, norm, exact):
    """num_heads > 1 (simplex): the heads are column segments of the per-image tables, one softmax per segment; output and the
    head-averaged attention map against the fp64 oracle (direct form with split heads)."""
    D = p = 16
    B = 3
    g = torch.Generator().manual_seed(C + k + heads)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 1.2 + 0.1
    y = torch.randn(B, k, D, generator=g, dtype=torch.float64)
    w = ob.init_params(C, D, k, p, integration, False, seed=13, bias_std=0.3)
    nrm = None if norm == "none" else norm
    ref, ratt, _ = ob.transformer_layer(x, y, w, integration=integration, norm=nrm, num_heads=heads, return_att=True)
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, norm=nrm, num_heads=heads, exact_fp32=exact).to(cuda_dev)
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].float())
        out, att, _ = attn(x.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev), y.float().to(cuda_dev), return_att=True)
    path = gf._lib.last_path()
    check_close(out, ref.permute(0, 2, 3, 1), path, f"heads{heads}/out")
    assert att.shape == (B, k, H, W)
    assert (att.cpu().double() - ratt).abs().max() <= (1e-5 if path == "simt_fp32" else 5e-3)
    assert (att.sum(dim=1) - 1).abs().max() < 1e-5
    # training path: composite backward with split heads
    xg = x.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev).requires_grad_(True)
    o2, _, _ = attn(xg, y.float().to(cuda_dev))
    o2.square().mean().backward()
    assert torch.isfinite(xg.grad).all() and xg.grad.abs().max() > 0


@pytest.mark.parametrize("exact", [True, False], ids=["fp32", "default"])
def test_generator_duplex_extensions_end_to_end(gf, cuda_dev, exact):
    """Duplex generator with every duplex extension on -- iterative centroid carry between layers of equal width, two k-means
    iterations, g_img2ltnt -- against the oracle generator (image + attention maps); and the carry really changes the result."""
    kw = dict(kmeans=True, iterative=True, kmeans_iters=2, g_img2ltnt=True)
    G = _small_generator(gf, cuda_dev, exact, **kw)
    z = torch.randn(3, 9, 32, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        img, atts = G(z.to(cuda_dev), return_att=True)
        img_fused = G(z.to(cuda_dev))
    ref, ratts = og.generator_forward(G.state_dict(), z, resolution=64, components_num=8, latent_dim=32, duplex=True, mapping_layers=4,
                                      return_att=True, kmeans_iters=2, img2ltnt=True, iterative=True)
    # The k-means loop feeds its centroids back into the next iteration's (and, carried, the next layer's) queries, and those queries
    # go through a softmax over all n grid cells: errors are amplified by every iteration.  fp32 mode: 3x the e2e bound (measured
    # 2.0e-5 peak-relative); TF32 mode (pass-A logits in TF32 inside the loop; the centroid -> query products are kept in fp32):
    # 6x (measured max-abs 5.2e-3 of the peak, rel-RMS 2.6e-3, 67.6 dB against 4.7e-4 / 78 dB for the plain duplex generator).
    sc = 3.0 if exact else 6.0
    check_image(img, ref, "fp32" if exact else "tf32", "duplex-ext/image", scale=sc)
    check_image(img_fused, ref, "fp32" if exact else "tf32", "duplex-ext/image-fused", scale=sc)
    e2e = TOLERANCES["e2e"]["simt_fp32" if exact else "wgmma_tf32"]
    for a, r in zip(atts, ratts):
        assert (a.double().cpu() - r).abs().max() <= sc * e2e["att_abs"]
    ref_nocarry = og.generator_forward(G.state_dict(), z, resolution=64, components_num=8, latent_dim=32, duplex=True, mapping_layers=4,
                                       kmeans_iters=2, img2ltnt=True, iterative=False)
    assert (ref - ref_nocarry).abs().max() > 1e-3 * ref.abs().max()


def _dropout_mask(gf, dev, B, H, W, C, k, D, p, salt, seed, step):
    """gf_attn_dropout_mask -> [B, n, KP] float32 on the CPU."""
    import ctypes
    from importlib import import_module
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    am.set_dropout_seed(seed, dev, step)
    desc = gf._lib.make_desc(B, H, W, C, k, D, pos_dim=0)
    KP = 16 if k <= 16 else 32
    mask = torch.empty(B, H * W, KP, device=dev)
    gf._lib.check(gf._lib.load().gf_attn_dropout_mask(ctypes.byref(desc), ctypes.c_float(p), salt, am.dropout_state(dev).data_ptr(), mask.data_ptr(),
                                                      ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "gf_attn_dropout_mask")
    torch.cuda.synchronize()
    return mask.cpu()


def test_dropout_mask_matches_philox_oracle(gf, cuda_dev):
    """The kernels' attention-dropout mask (Philox4x32-10, csrc/gf_common.cuh) is reproduced bit for bit by oracle/philox.py, whose
    Philox matches the published Random123 known-answer vectors; the keep rate is 1 - p."""
    from oracle import philox as ph
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(int(x) for x in ph.philox4x32_10(*ctr, *key)) == want
    for (B, H, W, k, p, salt, seed, step) in [(2, 10, 13, 7, 0.12, 5, 1234567890123, 0), (3, 16, 16, 20, 0.5, 0xdeadbeef, 42, 300), (1, 64, 64, 16, 0.12, 1, 7, 70000000)]:
        got = _dropout_mask(gf, cuda_dev, B, H, W, 64, k, 16, p, salt, seed, step)
        want = ph.dropout_mult(p, seed, step, salt, B * H * W, got.shape[2]).reshape(got.shape)
        assert np.array_equal(got.numpy(), want)
        keep = (got > 0).float().mean().item()
        assert abs(keep - (1 - p)) < 4 * math.sqrt(p * (1 - p) / got.numel()) + 1e-3
        assert torch.all((got == 0) | ((got - 1 / (1 - p)).abs() < 1e-6))


@pytest.mark.parametrize("C,H,W,k,integration,norm", [(64, 8, 16, 4, "both", "layer"), (96, 10, 13, 20, "mul", "layer"), (128, 16, 16, 16, "add", "none")])
def test_attention_dropout_forward_and_backward(gf, cuda_dev, C, H, W, k, integration, norm):
    """att_dp (training mode): forward and gradients of a simplex layer with dropped probabilities against the oracle given the SAME
    mask (oracle/philox.py); eval mode and a bumped step behave as expected."""
    from importlib import import_module
    from oracle import philox as ph
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    D = p = 16
    B, pd = 2, 0.25
    g = torch.Generator().manual_seed(C + k)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64).requires_grad_(True)
    w = {n: t.requires_grad_(True) for n, t in ob.init_params(C, D, k, p, integration, False, seed=4, bias_std=0.3).items()}
    nrm = None if norm == "none" else norm
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, norm=nrm, att_dp=pd, exact_fp32=True).to(cuda_dev)
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].detach().float())
    seed, step = 987654321, 3
    am.set_dropout_seed(seed, cuda_dev, step)
    KP = 16 if k <= 16 else 32
    mult = torch.from_numpy(ph.dropout_mult(pd, seed, step, attn.dp_salt, B * H * W, KP).reshape(B, H * W, KP)[:, :, :k].copy())
    ref, ratt, _ = ob.transformer_layer(x64, y64, w, integration=integration, norm=nrm, return_att=True, att_mult=mult)
    gout = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(gout)
    xg = x64.detach().permute(0, 2, 3, 1).contiguous().float().to(cuda_dev)
    yg = y64.detach().float().to(cuda_dev)
    attn.train()
    with torch.no_grad():                                            # training-mode forward without autograd (the D step's fakes)
        out, att, _ = attn(xg, yg, return_att=True)
    check_close(out, ref.detach().permute(0, 2, 3, 1), "simt_fp32", "dropout/forward", tol_scale=2.0)
    assert (att.cpu().double() - ratt.detach()).abs().max() <= 1e-5   # the map is the probabilities BEFORE dropout
    xr, yr = xg.clone().requires_grad_(True), yg.clone().requires_grad_(True)
    out2, _, _ = attn(xr, yr)
    assert torch.equal(out2.detach(), out)
    out2.backward(gout.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev))
    rel = lambda a, b: ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30)).item()
    assert rel(xr.grad, x64.grad.permute(0, 2, 3, 1)) < 1e-4 and rel(yr.grad, y64.grad) < 1e-4
    for n in ("wq", "wv", "wo", "wk", "pos_latent", "bo", "bv", "bq"):
        assert rel(getattr(attn, n).grad, w[n].grad) < 2e-4, n
    with torch.no_grad():
        am.advance_dropout(cuda_dev)                                 # next step: another mask
        out3, _, _ = attn(xg, yg)
        attn.eval()                                                  # eval: no dropout
        out4, _, _ = attn(xg, yg)
    assert (out3 - out).abs().max() > 1e-3
    ref0, _, _ = ob.transformer_layer(x64.detach(), y64.detach(), {n: t.detach() for n, t in w.items()}, integration=integration, norm=nrm)
    check_close(out4, ref0.permute(0, 2, 3, 1), "simt_fp32", "dropout/eval")


_DROPOUT_TC_CASES = [pytest.param(*c, 3, 0.2, False, id="-".join(map(str, c))) for c in
                     [(128, 16, 16, 16, "mul", "layer"), (256, 16, 24, 20, "mul", "layer"), (128, 8, 16, 8, "both", "layer"),
                      (512, 8, 16, 8, "add", "none"), (64, 8, 8, 4, "mul", "layer")]]
# the six attention layers of the 256^2 K = 16 training generator (bench.py train_probe: mul, layer norm, att_dp = 0.12), with the
# token reductions and the autograd through the tables as TF32 GEMMs (allow_tf32 = True, as the benchmarked step sets) and without
_DROPOUT_TC_CASES += [pytest.param(C, R, R, 16, "mul", "layer", 2 if R == 256 else 3, 0.12, tf32,
                                   id=f"train-{C}-{R}x{R}-{'tf32' if tf32 else 'fp32'}")
                      for C, R in ((512, 8), (512, 16), (512, 32), (512, 64), (256, 128), (128, 256)) for tf32 in (False, True)]


# the mask of a layer depends on its salt, which counts the layers constructed so far: each case fixes its own so that the masks
# (and the TF32 forward's worst element at 131,072 tokens) do not depend on which tests ran before
_DROPOUT_TC_CASES = [pytest.param(*c.values, i + 1, id=c.id) for i, c in enumerate(_DROPOUT_TC_CASES)]


@pytest.mark.parametrize("C,H,W,k,integration,norm,B,pd,tf32,salt_no", _DROPOUT_TC_CASES)
def test_attention_dropout_on_the_tensor_path(gf, cuda_dev, C, H, W, k, integration, norm, B, pd, tf32, salt_no):
    """att_dp on the wgmma kernel (training forward of the default path): against the oracle given the SAME Philox mask, with the
    fused post-op around it; and the gradients through that forward (stage-T backward kernel, same mask) against the oracle's.
    With tf32, torch.backends.cuda.matmul.allow_tf32 is on during the backward, as in the benchmarked training step."""
    from importlib import import_module
    from oracle import philox as ph
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    D = p = 16
    g = torch.Generator().manual_seed(C + k)
    x64 = torch.randn(B, C, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    y64 = torch.randn(B, k, D, generator=g, dtype=torch.float64).requires_grad_(True)
    w = {n: t.requires_grad_(True) for n, t in ob.init_params(C, D, k, p, integration, False, seed=4, bias_std=0.3).items()}
    nrm = None if norm == "none" else norm
    attn = gf.BipartiteAttention(C, D, k, pos_dim=p, integration=integration, norm=nrm, att_dp=pd).to(cuda_dev)
    attn.dp_salt = salt_no * 0x9E3779B1 & 0xFFFFFFFF
    with torch.no_grad():
        for n, prm in attn.named_parameters():
            prm.copy_(w[n].detach().float())
    seed, step = 123456789, 11
    am.set_dropout_seed(seed, cuda_dev, step)
    KP = 16 if k <= 16 else 32
    mult = torch.from_numpy(ph.dropout_mult(pd, seed, step, attn.dp_salt, B * H * W, KP).reshape(B, H * W, KP)[:, :, :k].copy())
    ref, ratt, _ = ob.transformer_layer(x64, y64, w, integration=integration, norm=nrm, return_att=True, att_mult=mult)
    xg = x64.detach().permute(0, 2, 3, 1).contiguous().float().to(cuda_dev)
    yg = y64.detach().float().to(cuda_dev)
    attn.train()
    with torch.no_grad():
        out, att, _ = attn(xg, yg, return_att=True)
    assert gf._lib.last_path() == "wgmma_tf32"
    check_close(out, ref.detach().permute(0, 2, 3, 1), "wgmma_tf32", "dropout-tc/forward", tol_scale=2.0)
    assert (att.cpu().double() - ratt.detach()).abs().max() <= 2e-3           # pre-dropout probabilities, TF32 logits
    gout = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(gout)
    xr, yr = xg.clone().requires_grad_(True), yg.clone().requires_grad_(True)
    out2, _, _ = attn(xr, yr)
    assert torch.equal(out2.detach(), out)
    try:
        torch.backends.cuda.matmul.allow_tf32 = tf32
        out2.backward(gout.permute(0, 2, 3, 1).contiguous().float().to(cuda_dev))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    rel = lambda a, b: ((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30)).item()
    errs = {"x": rel(xr.grad, x64.grad.permute(0, 2, 3, 1)), "y": rel(yr.grad, y64.grad)}
    errs.update({n: rel(getattr(attn, n).grad, w[n].grad) for n in ("wq", "wv", "wo", "wk")})
    print(f"[dropout-tc/grad] C={C} {H}x{W} k={k} B={B} tf32={tf32}: " + " ".join(f"{n}={v:.2e}" for n, v in errs.items()))
    assert errs["x"] < 2e-3 and errs["y"] < 2e-3                    # fp32 backward of a TF32 forward
    for n in ("wq", "wv", "wo", "wk"):
        assert errs[n] < 2e-3, n
    if pd == 0.12:        # the training layers: the backward's GEMMs stay fp32 under allow_tf32 (measured <= 4.8e-6, DESIGN.md 5)
        assert max(errs.values()) < 1e-5, errs
    # fused post-op + dropout, as the D step's fake images run (training-mode forward under no_grad)
    bias = torch.randn(C, generator=g, dtype=torch.float64) * 0.5
    d_in = torch.rand(B, C, generator=g, dtype=torch.float64) + 0.5
    refp, _, _ = ob.transformer_layer(x64.detach() * d_in[:, :, None, None], y64.detach(), {n: t.detach() for n, t in w.items()},
                                      integration=integration, norm=nrm, att_mult=mult)
    refp = torch.nn.functional.leaky_relu(refp + bias[None, :, None, None], 0.2) * math.sqrt(2.0)
    post = dict(bias=bias.float().to(cuda_dev), act="lrelu", gain=math.sqrt(2.0), in_scale=d_in.float().to(cuda_dev))
    post.update(attn.dropout_postop(cuda_dev))
    with torch.no_grad():
        outp, _, _ = attn(xg, yg, postop=post, need_centroids=False)
    assert gf._lib.last_path() == "wgmma_tf32"
    check_close(outp, refp.permute(0, 2, 3, 1), "wgmma_tf32", "dropout-tc/postop", tol_scale=2.0)


def test_generator_with_own_tf32_convolutions(gf, cuda_dev, monkeypatch):
    """The benchmarked path end to end: TF32 convolutions allowed, so the five stride-1 3x3 convolutions of the 256^2 generator run on
    the library's own wgmma implicit-GEMM kernel (row f1) and the rest on cuDNN TF32 -- image vs the fp64 oracle within the
    SURVEY 8c end-to-end bound (5e-3 of the peak, 60 dB), and against the same network with cuDNN TF32 convolutions everywhere."""
    G = _benchmark_generator(gf, cuda_dev, 256, 16, False)
    z = torch.randn(2, 17, 32, generator=torch.Generator().manual_seed(1))
    try:
        torch.backends.cudnn.allow_tf32 = True
        with torch.no_grad():
            l0 = gf._lib.launch_count(); G(z.to(cuda_dev)); 
            l0 = gf._lib.launch_count(); img = G(z.to(cuda_dev)).clone(); n_own = gf._lib.launch_count() - l0
            monkeypatch.setenv("GF_CUDNN_CONV", "1")
            l0 = gf._lib.launch_count(); img_c = G(z.to(cuda_dev)).clone(); n_cudnn = gf._lib.launch_count() - l0
    finally:
        torch.backends.cudnn.allow_tf32 = False
    assert n_own == n_cudnn + 5                                    # res 16 .. 256: five convolutions on the own kernel
    ref = og.generator_forward(G.state_dict(), z, resolution=256, components_num=16, latent_dim=32)
    for name, im in (("own-conv", img), ("cudnn-tf32", img_c)):
        err = (im.double().cpu() - ref).abs()
        peak = ref.abs().max().item()
        rmse = err.pow(2).mean().sqrt().item()
        psnr = 20 * math.log10(peak / rmse)
        print(f"[e2e-tf32conv] {name}: max_abs/peak={err.max().item() / peak:.3e} rel_rms={rmse / ref.pow(2).mean().sqrt().item():.3e} psnr={psnr:.1f} dB")
        _log_parity(dict(what="tf32conv/" + name, path="e2e-tf32conv", max_abs=err.max().item(), peak=peak, psnr=psnr))
        assert err.max().item() <= 5e-3 * peak and psnr >= 60.0
