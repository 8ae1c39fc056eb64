"""GPU tests of the attention backward kernels at their C boundary (csrc/gf_bwd.cu; run on an H100: ``pytest -m gpu``).

The three entries are called directly through ``_lib`` with synthetic fp32 tables, so a case can plant -inf padding, ties and
any ``r``, and no TF32 forward takes part:

* ``gf_attn_simplex_bwd_ex`` (``token_bwd_kernel``, stage T): dX, dS, P and dCtl (with its bias half for "both");
* ``gf_attn_centroid_stats`` (``centroid_simt_kernel`` split-n partials, then ``centroid_merge_kernel``): Xbar and lse;
* ``gf_attn_centroid_bwd`` (``centroid_bwd_kernel``): dS, and dX added in place to what the buffer held.

Every output is written between NaN guards; the tests check that the guards are intact and that every element was written.
The reference is fp64 autograd through the folded oracle (``oracle/attn_bwd.py``).

* Exact cases check the indexing, the 32-channel chunks, the batch offsets, the ragged last tile and the padded latents: every
  probability is 0, 1/2 or 1 and every intermediate an exact fp32 value (``tests/test_host_cpu_attn_backward.py`` checks that on
  the host), so the outputs must equal the reference bit for bit.  Layer norm cannot be exact (rsqrtf): it is covered by the
  tolerance cases.
* Tolerance cases run realistic tables, x with mean 0 and 30, with and without layer norm and dropout, and the six layer
  shapes of the benchmarked 256^2 training generator.  The error of every element is bounded relative to its magnitude
  companion (the same expression on absolute values), by the frozen bounds below.
* Determinism, batch independence and CUDA-graph replay, bit for bit.
"""
import ctypes

import pytest
import torch

from oracle import attn_bwd as ab
from oracle.folded import pad_k
from tests.guards import Guarded, assert_exact as _assert_exact

pytestmark = pytest.mark.gpu

# Per-element bounds of |kernel - fp64 reference| / companion, per output.  Measured worst cases over the tolerance cases below on
# an H100 80GB HBM3 (700 W power limit), frozen at 1.5x or more (DESIGN.md section 5).
BOUND = {"dX": 1.2e-7, "dS": 1.5e-8, "P": 8e-7, "dCtl": 3e-6, "Xbar": 8e-8, "lse": 6e-8, "cen_dX": 1.1e-6, "cen_dS": 1.3e-7}
D_LATENT = 16                    # the latent width only sizes the tables of stages W and I: no entry here reads it

# B, H, W, C, k, integration, dropout (p = 0.5) -- norm none
EXACT_T = [
    (1, 1, 1, 32, 1, "mul", False),          # one token, one latent, one chunk
    (3, 8, 8, 32, 4, "add", True),
    (1, 1, 128, 96, 16, "both", False),      # one full tile, three chunks
    (3, 128, 1, 96, 17, "mul", True),        # KP = 32 with 15 padded latents
    (3, 10, 13, 512, 31, "both", True),      # ragged n = 130 (two tiles, the second with 2 tokens), Cout = 1024
    (1, 64, 64, 512, 32, "add", False),      # KP full, 32 tiles
    (3, 10, 13, 1024, 32, "mul", False),     # 32 chunks, the largest C
    (1, 8, 8, 1024, 17, "both", True),       # Cout = 2048
    (300, 5, 7, 32, 16, "mul", True),        # B in the hundreds, n < 128
    (3, 10, 13, 96, 4, "add", False),
    (1, 8, 8, 32, 31, "both", False),
    (3, 64, 64, 32, 1, "mul", True),
]
# B, H, W, C, k, integration, norm, att_dp, mean
TOL_T = [
    (3, 10, 13, 96, 20, "mul", "layer", 0.12, 30.0),
    (3, 10, 13, 96, 20, "mul", "layer", 0.0, 0.0),
    (1, 8, 8, 1024, 32, "both", "layer", 0.5, 30.0),
    (1, 8, 8, 1024, 32, "both", "none", 0.0, 0.0),
    (3, 128, 1, 32, 1, "add", "layer", 0.12, 0.0),
    (1, 1, 128, 512, 17, "add", "none", 0.5, 30.0),
    (300, 5, 7, 32, 4, "mul", "layer", 0.12, 30.0),
    (3, 64, 64, 96, 16, "both", "layer", 0.12, 0.0),
    (1, 1, 1, 32, 31, "mul", "none", 0.12, 30.0),
    (3, 10, 13, 512, 16, "add", "layer", 0.0, 30.0),
    # the six attention layers of the 256^2 K = 16 training generator (bench.py train_probe): mul, layer norm, att_dp = 0.12
    (2, 8, 8, 512, 16, "mul", "layer", 0.12, 0.0),
    (2, 16, 16, 512, 16, "mul", "layer", 0.12, 0.0),
    (2, 32, 32, 512, 16, "mul", "layer", 0.12, 0.0),
    (2, 64, 64, 512, 16, "mul", "layer", 0.12, 0.0),
    (2, 128, 128, 256, 16, "mul", "layer", 0.12, 0.0),
    (1, 256, 256, 128, 16, "mul", "layer", 0.12, 0.0),
]
# B, H, W, C, k: n = 4186 is 33 tiles, several splits with a partial last one (the test asserts that regime)
EXACT_A = [
    (1, 46, 91, 32, 1),
    (3, 46, 91, 96, 16),
    (1, 46, 91, 512, 17),
    (3, 46, 91, 96, 32),
    (1, 46, 91, 32, 32),
    (3, 10, 13, 512, 16),                    # one split
    (2, 1, 1, 32, 4),                        # one token
]
# B, H, W, C, k, mean
TOL_A = [
    (3, 46, 91, 96, 20, 0.0),
    (1, 46, 91, 512, 32, 30.0),
    (3, 10, 13, 32, 1, 30.0),
    (2, 64, 64, 512, 16, 0.0),
]


def _lib(gf):
    return gf._lib.load()


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t, dev):
    return t.float().contiguous().to(dev)


def stage_t(gf, dev, case, *, H, W, k, integration, norm):
    """gf_attn_simplex_bwd_ex on the case's tables; returns the checked outputs on the CPU as fp64."""
    X = _f32(case["X"], dev)
    B, n, C = X.shape
    KP = pad_k(k)
    Cout = case["Vt"].shape[1]
    tabs = [_f32(case[name], dev) for name in ("dOut", "Kp", "Vt", "Rt", "Ct")]
    outs = {"dX": Guarded((B, n, C), dev), "dS": Guarded((B, n, KP), dev), "P": Guarded((B, n, KP), dev),
            "dCtl": Guarded((B, n, Cout), dev)}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm=norm, integration=integration, pos_dim=0, duplex=False)
    state = cb = None
    if case["att_dp"]:
        state = torch.tensor([case["dp_seed"], case["step"]], dtype=torch.int64, device=dev)
        cb = _f32(case["cb"], dev)
    gf._lib.check(_lib(gf).gf_attn_simplex_bwd_ex(
        ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs), *(outs[o].ptr() for o in ("dX", "dS", "P", "dCtl")),
        ctypes.c_float(case["att_dp"]), case["salt"], None if state is None else state.data_ptr(), None if cb is None else cb.data_ptr(),
        _stream(dev)), "gf_attn_simplex_bwd_ex")
    torch.cuda.synchronize()
    return {name: g.check(name).double().cpu() for name, g in outs.items()}


def pass_a(gf, dev, case, *, H, W, k):
    """gf_attn_centroid_stats, then gf_attn_centroid_bwd on top of the preloaded dX; returns the checked outputs as fp64."""
    X = _f32(case["X"], dev)
    B, n, C = X.shape
    KP = pad_k(k)
    M, Rt2, Ct2, dXbar, r = (_f32(case[name], dev) for name in ("M", "Rt2", "Ct2", "dXbar", "r"))
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    ws = torch.empty(gf._lib.workspace_bytes(desc), dtype=torch.uint8, device=dev)
    xbar, lse = Guarded((B, k, C), dev), Guarded((B, KP), dev)
    gf._lib.check(_lib(gf).gf_attn_centroid_stats(ctypes.byref(desc), X.data_ptr(), M.data_ptr(), Rt2.data_ptr(), Ct2.data_ptr(),
                                                  xbar.ptr(), lse.ptr(), ws.data_ptr(), _stream(dev)), "gf_attn_centroid_stats")
    dX, dS = Guarded((B, n, C), dev, init=_f32(case["dX0"], dev)), Guarded((B, n, KP), dev)
    gf._lib.check(_lib(gf).gf_attn_centroid_bwd(ctypes.byref(desc), X.data_ptr(), M.data_ptr(), Rt2.data_ptr(), Ct2.data_ptr(),
                                                lse.t.data_ptr(), dXbar.data_ptr(), r.data_ptr(), dX.ptr(), dS.ptr(), _stream(dev)),
                  "gf_attn_centroid_bwd")
    torch.cuda.synchronize()
    return {"Xbar": xbar.check("Xbar").double().cpu(), "lse": lse.check("lse").double().cpu(),
            "cen_dX": dX.check("dX", written=False).double().cpu(), "cen_dS": dS.check("dS").double().cpu()}


def nsplit_of(gf, B, H, W, C, k):
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    out = (ctypes.c_longlong * 8)()
    gf._lib.check(_lib(gf).gf_attn_debug_layout(ctypes.byref(desc), out, 8), "gf_attn_debug_layout")
    return int(out[2])


def split_ranges(n, nsplit):
    """The token range of every non-empty split of centroid_simt_kernel: contiguous runs of ceil(tiles / nsplit) 128-token tiles."""
    tiles = (n + 127) // 128
    per = (tiles + nsplit - 1) // nsplit
    return [(s * per * 128, min(n, (s + 1) * per * 128)) for s in range(nsplit) if s * per < tiles]


def place_winners(B, n, k, ranges, seed):
    """One winning token per (image, latent), cycling through the first, a middle and the last split."""
    g = torch.Generator().manual_seed(seed)
    picks = [ranges[0], ranges[len(ranges) // 2], ranges[-1]]
    w = torch.empty(B, k, dtype=torch.long)
    for b in range(B):
        for j in range(k):
            lo, hi = picks[(b + j) % 3]
            w[b, j] = torch.randint(lo, hi, (1,), generator=g)
    return w


def _worst(got, want, comp, name):
    """max |got - want| / comp over the elements; elements with comp == 0 must be exact (want == got, e.g. padded latents)."""
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin) and torch.equal(got[~fin], want[~fin]), f"{name}: non-finite elements differ"
    err = (got - want).abs()[fin]
    c = comp.expand_as(want)[fin]
    assert (err[c == 0] == 0).all(), f"{name}: nonzero error where the companion is 0"
    return (err[c > 0] / c[c > 0]).max().item() if (c > 0).any() else 0.0


def _id(v):
    return str(v)


@pytest.mark.parametrize("B,H,W,C,k,integration,dropout", EXACT_T, ids=_id)
def test_stage_t_exact(gf, cuda_dev, B, H, W, C, k, integration, dropout):
    """token_bwd_kernel on exact integer tables: dX, dS, P and dCtl equal the fp64 reference bit for bit."""
    case = ab.exact_stage_t_case(B, H, W, C, k, integration, dropout=dropout, seed=B * 1000 + C + k)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, norm="none")
    want = ab.stage_t_backward(case["X"], case["dOut"], case["Kp"], case["Vt"], case["Rt"], case["Ct"], H=H, W=W,
                               integration=integration, norm="none", mult=case["mult"], cb=case["cb"])
    p = want["P"] if case["mult"] is None else None
    if p is not None:                                   # both outcomes of a pair happen: one-hot rows and ties
        real = p[:, :, :k]
        assert (real == 1.0).any() and ((real == 0.5).any() or k == 1)
    for name in ("dX", "dS", "P", "dCtl"):
        _assert_exact(got[name], want[name], name)


@pytest.mark.parametrize("B,H,W,C,k,integration,norm,att_dp,mean", TOL_T, ids=_id)
def test_stage_t_tolerance(gf, cuda_dev, B, H, W, C, k, integration, norm, att_dp, mean):
    """token_bwd_kernel on realistic tables: every element of dX, dS, P and dCtl within the frozen bound of its companion."""
    case = ab.random_stage_t_case(B, H, W, C, k, integration, att_dp=att_dp, mean=mean, seed=B + H * W + C + k)
    got = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, norm=norm)
    args = (case["X"], case["dOut"], case["Kp"], case["Vt"], case["Rt"], case["Ct"])
    want = ab.stage_t_backward(*args, H=H, W=W, integration=integration, norm=norm, mult=case["mult"], cb=case["cb"])
    comp = ab.stage_t_companions(*args, H=H, W=W, k=k, integration=integration, norm=norm, mult=case["mult"], cb=case["cb"])
    worst = {name: _worst(got[name], want[name], comp[name], name) for name in ("dX", "dS", "P", "dCtl")}
    print(f"[attn-bwd] stage T {B}x{H}x{W} C={C} k={k} {integration} {norm} p={att_dp} mean={mean}: "
          + " ".join(f"{n}={v:.3e}" for n, v in worst.items()))
    for name, v in worst.items():
        assert v <= BOUND[name], f"{name}: {v:.3e} > {BOUND[name]:.1e}"


@pytest.mark.parametrize("B,H,W,C,k", EXACT_A, ids=_id)
def test_pass_a_exact(gf, cuda_dev, B, H, W, C, k):
    """centroid_simt_kernel + centroid_merge_kernel and centroid_bwd_kernel on exact tables: one winning token per latent, placed
    in the first, a middle and the last (partial) split, so A is one-hot, Xbar_j = x_{t_j} and lse_j = s_{t_j}; Xbar, lse, dX (added
    to the preloaded values) and dS equal the fp64 reference bit for bit."""
    n = H * W
    nsplit = nsplit_of(gf, B, H, W, C, k)
    ranges = split_ranges(n, nsplit)
    if n > 4096:                                           # the regime these shapes are for: several splits, the last one partial
        assert len(ranges) >= 3 and ranges[-1][1] - ranges[-1][0] < ranges[0][1] - ranges[0][0], ranges
    case = ab.exact_centroid_case(B, H, W, C, k, winners=place_winners(B, n, k, ranges, seed=C + k), seed=B * 100 + C + k)
    got = pass_a(gf, cuda_dev, case, H=H, W=W, k=k)
    args = (case["X"], case["M"], case["Rt2"], case["Ct2"])
    want = {**ab.centroid_stats(*args, k=k), **{"cen_" + a: b for a, b in
                                                ab.centroid_backward(*args, case["dXbar"], case["r"], case["dX0"], k=k).items()}}
    for name in ("Xbar", "lse", "cen_dX", "cen_dS"):
        _assert_exact(got[name], want[name], name)
    assert (got["cen_dX"] != case["dX0"]).any(), "dX was not added to"


@pytest.mark.parametrize("B,H,W,C,k,mean", TOL_A, ids=_id)
def test_pass_a_tolerance(gf, cuda_dev, B, H, W, C, k, mean):
    """The pass-A kernels on realistic tables (r = dXbar . Xbar, as the layer passes it): every element of Xbar, lse, dX and dS
    within the frozen bound of its companion; dX is the preloaded values plus the pass-A part."""
    case = ab.random_centroid_case(B, H, W, C, k, mean=mean, seed=B + H + C + k)
    got = pass_a(gf, cuda_dev, case, H=H, W=W, k=k)
    args = (case["X"], case["M"], case["Rt2"], case["Ct2"])
    want = {**ab.centroid_stats(*args, k=k), **{"cen_" + a: b for a, b in
                                                ab.centroid_backward(*args, case["dXbar"], case["r"], case["dX0"], k=k).items()}}
    comp = {"cen_" + a if a in ("dX", "dS") else a: b for a, b in
            ab.centroid_companions(*args, case["dXbar"], case["r"], case["dX0"], k=k).items()}
    worst = {name: _worst(got[name], want[name], comp[name], name) for name in ("Xbar", "lse", "cen_dX", "cen_dS")}
    print(f"[attn-bwd] pass A {B}x{H}x{W} C={C} k={k} mean={mean}: " + " ".join(f"{n}={v:.3e}" for n, v in worst.items()))
    for name, v in worst.items():
        assert v <= BOUND[name], f"{name}: {v:.3e} > {BOUND[name]:.1e}"


def test_properties_determinism_batch_independence_graph_replay(gf, cuda_dev):
    """Two calls give bit-identical outputs; each image of a batch equals the same image run alone (dropout off: the mask is keyed
    by the global token index); a CUDA-graph replay equals the eager call -- for stage T and for both pass-A entries."""
    H, W, C, k = 10, 13, 96, 20
    for integration, norm in (("both", "layer"), ("mul", "none")):
        case = ab.random_stage_t_case(3, H, W, C, k, integration, att_dp=0.0, mean=1.0, seed=5)
        a = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, norm=norm)
        b = stage_t(gf, cuda_dev, case, H=H, W=W, k=k, integration=integration, norm=norm)
        one = {n: case[n][1:2] for n in ("X", "dOut", "Kp", "Vt", "Rt", "Ct")}
        c = stage_t(gf, cuda_dev, {**case, **one}, H=H, W=W, k=k, integration=integration, norm=norm)
        for name in a:
            assert torch.equal(a[name], b[name]), name
            assert torch.equal(a[name][1:2], c[name]), name
    cen = ab.random_centroid_case(3, H, W, C, k, mean=1.0, seed=6)
    a = pass_a(gf, cuda_dev, cen, H=H, W=W, k=k)
    b = pass_a(gf, cuda_dev, cen, H=H, W=W, k=k)
    one = {n: cen[n][1:2] for n in ("X", "M", "Rt2", "Ct2", "dXbar", "r", "dX0")}
    c = pass_a(gf, cuda_dev, {**cen, **one}, H=H, W=W, k=k)
    for name in a:
        assert torch.equal(a[name], b[name]), name
        assert torch.equal(a[name][1:2], c[name]), name

    # graph replay: stage T with dropout (the state is read at run time) and the two pass-A calls, captured together
    case = ab.random_stage_t_case(2, H, W, C, k, "mul", att_dp=0.12, mean=0.0, seed=7)
    B, n = 2, H * W
    KP = pad_k(k)
    dev = cuda_dev
    ins = {name: _f32(case[name], dev) for name in ("X", "dOut", "Kp", "Vt", "Rt", "Ct", "cb")}
    state = torch.tensor([case["dp_seed"], case["step"]], dtype=torch.int64, device=dev)
    outs = [torch.empty(s, device=dev) for s in ((B, n, C), (B, n, KP), (B, n, KP), (B, n, C))]
    cins = {name: _f32(cen[name], dev) for name in ("X", "M", "Rt2", "Ct2", "dXbar", "r")}
    Bc = cen["X"].shape[0]
    tdesc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=False)
    cdesc = gf._lib.make_desc(Bc, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=1)
    ws = torch.empty(gf._lib.workspace_bytes(cdesc), dtype=torch.uint8, device=dev)
    xbar, lse = torch.empty(Bc, k, C, device=dev), torch.empty(Bc, KP, device=dev)
    cdX0 = _f32(cen["dX0"], dev)
    cdX, cdS = torch.empty_like(cdX0), torch.empty(Bc, n, KP, device=dev)
    lib = _lib(gf)

    def run():
        s = _stream(dev)
        gf._lib.check(lib.gf_attn_simplex_bwd_ex(ctypes.byref(tdesc), *(ins[nm].data_ptr() for nm in ("X", "dOut", "Kp", "Vt", "Rt", "Ct")),
                                                 *(o.data_ptr() for o in outs), ctypes.c_float(0.12), case["salt"], state.data_ptr(),
                                                 ins["cb"].data_ptr(), s), "gf_attn_simplex_bwd_ex")
        gf._lib.check(lib.gf_attn_centroid_stats(ctypes.byref(cdesc), *(cins[nm].data_ptr() for nm in ("X", "M", "Rt2", "Ct2")),
                                                 xbar.data_ptr(), lse.data_ptr(), ws.data_ptr(), s), "gf_attn_centroid_stats")
        cdX.copy_(cdX0)
        gf._lib.check(lib.gf_attn_centroid_bwd(ctypes.byref(cdesc), *(cins[nm].data_ptr() for nm in ("X", "M", "Rt2", "Ct2")),
                                               lse.data_ptr(), cins["dXbar"].data_ptr(), cins["r"].data_ptr(), cdX.data_ptr(),
                                               cdS.data_ptr(), s), "gf_attn_centroid_bwd")

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (*outs, xbar, lse, cdX, cdS)]
    for t in (*outs, xbar, lse, cdX, cdS):
        t.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    graph.replay()
    torch.cuda.synchronize()
    for i, (e, t) in enumerate(zip(eager, (*outs, xbar, lse, cdX, cdS))):
        assert torch.equal(e, t), i
