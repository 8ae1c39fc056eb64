"""GPU tests of the dropout-aware stage-T double backward at its C boundary (csrc/gf_bwd.cu: gf_attn_simplex_bwd_vjp_ex,
``token_bwd_vjp_kernel<KP, true>``; run on an H100: ``pytest -m gpu``).

The entry is called through ``_lib`` with synthetic fp32 tables, cotangents and a device dropout state.  Every output sits between
NaN guards; the tests check the guards and that every element was written.  The reference is fp64 autograd differentiated twice
through the folded oracle with the Philox multipliers of oracle/philox.py (``tests/attn_double_backward_dropout_ref.py``).  Errors
are measured as in tests/test_gpu_attn_double_backward.py: per-token outputs max |kernel - reference| / max |reference|, the
reductions the caller forms (in fp64 here) relative to their magnitude companion.  Cases: every integration, norm layer and none, x
with mean 0 and 30, KP = 16 and 32 with padded latents, ragged tiles, 1 to 32 channel chunks, B = 300, the simplex layers of the
256^2 generator (K = 16), att_dp 0.12 and 0.5.  Then att_dp = 0 against the dropout-free entry, the mask against
gf_attn_dropout_mask, determinism, batch independence and CUDA-graph replay, bit for bit.
"""
import ctypes
import math

import pytest
import torch

from oracle.folded import pad_k
from tests import attn_double_backward_dropout_ref as dr
from tests.guards import Guarded
from tests.test_gpu_attn_double_backward import D_LATENT, _err, _f32, _stream, reduce_stage_t, run_stage_t, stage_t_case

pytestmark = pytest.mark.gpu

# Bound on max |kernel - fp64| / max |fp64| per output tensor, frozen at >= 1.5x the measured worst on an H100 80GB HBM3 (1.11e-5,
# Xg of the 32-chunk case; DESIGN.md section 4.8).
BOUND = 2e-5
SALT = 0x2545F491

# B, H, W, C, k, integration, norm, mean, att_dp
CASES = [
    (1, 1, 1, 32, 1, "mul", "none", 0.0, 0.5),              # one token, one latent, one chunk
    (3, 8, 8, 32, 4, "add", "layer", 30.0, 0.12),
    (1, 1, 128, 96, 16, "both", "layer", 0.0, 0.5),         # one full tile, three chunks
    (3, 128, 1, 96, 17, "mul", "layer", 30.0, 0.12),        # KP = 32 with 15 padded latents
    (3, 10, 13, 512, 31, "both", "none", 30.0, 0.5),        # ragged n = 130, Cout = 1024
    (1, 10, 13, 1024, 32, "mul", "layer", 30.0, 0.12),      # 32 chunks
    (1, 8, 8, 1024, 20, "both", "layer", 0.0, 0.12),        # Cout = 2048
    (300, 5, 7, 32, 16, "mul", "layer", 30.0, 0.5),         # B in the hundreds, n < 128
    (2, 10, 13, 96, 4, "add", "none", 0.0, 0.5),
    (2, 9, 11, 64, 8, "mul", "none", 0.0, 0.12),
    # the simplex attention layers of Generator(256, components_num=16) (mul, layer norm), small B
    (1, 256, 256, 64, 16, "mul", "layer", 0.0, 0.12),
    (1, 128, 128, 128, 16, "mul", "layer", 0.0, 0.12),
    (2, 64, 64, 256, 16, "mul", "layer", 0.0, 0.12),
    (2, 32, 32, 512, 16, "mul", "layer", 0.0, 0.5),
    (2, 16, 16, 512, 16, "mul", "layer", 0.0, 0.12),
    (2, 8, 8, 512, 16, "mul", "layer", 0.0, 0.12),
]


def dropout_case(B, H, W, C, k, integration, mean, seed):
    ins, cots = stage_t_case(B, H, W, C, k, integration, mean, seed)
    g = torch.Generator().manual_seed(seed + 7)
    Cout = ins[3].shape[1]
    cb = 0.3 * torch.randn(Cout, generator=g, dtype=torch.float64)
    if integration != "add":
        cb[:C] += 1.0                                             # bo + 1 on the gain half, as the layers pass it
    return ins, cb, cots, torch.randn(Cout, generator=g, dtype=torch.float64)


def run_ex(gf, dev, ins, cb, cots, cbg, *, H, W, k, integration, norm, att_dp, state, guards=True):
    X = _f32(ins[0], dev)
    B, n, C = X.shape
    KP, Cout = pad_k(k), ins[3].shape[1]
    tabs = [_f32(t, dev) for t in ins[1:]]
    cg = [_f32(t, dev) for t in cots]
    cbd, cbgd = _f32(cb, dev), _f32(cbg, dev)
    shapes = {"Xg": (B, n, C), "dOutg": (B, n, C), "Sg": (B, n, KP), "dPg": (B, n, KP), "Ctlg": (B, n, Cout), "dS": (B, n, KP),
              "P": (B, n, KP), "dCtl": (B, n, Cout)}
    outs = {nm: Guarded(s, dev) for nm, s in shapes.items()}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm=norm, integration=integration, pos_dim=0, duplex=False)
    gf._lib.check(gf._lib.load().gf_attn_simplex_bwd_vjp_ex(
        ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs + cg), *(o.ptr() for o in outs.values()),
        ctypes.c_float(att_dp), SALT, state.data_ptr(), cbd.data_ptr(), cbgd.data_ptr(), _stream(dev)), "gf_attn_simplex_bwd_vjp_ex")
    torch.cuda.synchronize(dev)
    return {nm: (o.check(nm) if guards else o.t).clone() for nm, o in outs.items()}


def reduce_ex(o, ins, cots, companion=False):
    """The caller's reductions in fp64: those of the dropout-free entry (P = q) and cb: (1 - sum P) Ctlg - (sum dPg) dCtl.  With
    ``companion`` (o, ins and cots are absolute values) the magnitude companions: 1 - sum P becomes 1 + sum P, the size of the
    terms whose difference it is."""
    H, W = ins[4].shape[1], ins[5].shape[1]
    red = reduce_stage_t(o, ins, cots, H, W)
    d = {nm: t.double().cpu() for nm, t in o.items()}
    qdef = 1.0 + d["P"].sum(dim=2, keepdim=True) if companion else 1.0 - d["P"].sum(dim=2, keepdim=True)
    red["cb"] = (qdef * d["Ctlg"] + (1 if companion else -1) * d["dPg"].sum(dim=2, keepdim=True) * d["dCtl"]).sum(dim=(0, 1))
    return red


def _state(dev, seed, step):
    return torch.tensor([seed, step], dtype=torch.int64, device=dev)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c[:5])) + f"-{c[5]}-{c[6]}-m{int(c[7])}-p{c[8]}")
def test_stage_t_vjp_dropout_against_fp64(gf, cuda_dev, case):
    B, H, W, C, k, integration, norm, mean, att_dp = case
    seed = B * 7 + C + k
    ins, cb, cots, cbg = dropout_case(B, H, W, C, k, integration, mean, seed)
    dseed, step = 0x1234567 + seed, 5
    got = run_ex(gf, cuda_dev, ins, cb, cots, cbg, H=H, W=W, k=k, integration=integration, norm=norm, att_dp=att_dp,
                 state=_state(cuda_dev, dseed, step))
    mult = dr.philox_mult(att_dp, dseed, step, SALT, B, H * W, pad_k(k))
    assert 0 < torch.count_nonzero(mult[..., :k]) < mult[..., :k].numel() or B * H * W * k < 4
    ref = dr.stage_t_vjp_dropout(*ins, cb, mult, *cots, cbg, H=H, W=W, integration=integration, norm=norm)
    red = reduce_ex(got, ins, cots)
    comp = reduce_ex({nm: t.abs() for nm, t in got.items()}, [t.abs() for t in ins], [t.abs() for t in cots], companion=True)
    errs = {nm: _err(got[nm], ref[nm]) for nm in ("Xg", "dOutg", "Sg", "dS", "P", "dCtl")}
    errs.update({nm: _err(red[nm], ref[nm], comp[nm]) for nm in ("Kp", "Vt", "Rt", "Ct", "cb")})
    if integration == "add":                                      # ctl does not enter the first-order backward
        assert torch.count_nonzero(got["Ctlg"]) == 0
    else:
        errs["Ctlg"] = _err(got["Ctlg"], ref["Ctlg"])
        if integration == "both":
            assert torch.count_nonzero(got["Ctlg"][..., C:]) == 0
    assert torch.count_nonzero(got["Sg"][..., k:]) == 0 and torch.count_nonzero(got["dPg"][..., k:]) == 0
    dropped = mult.to(cuda_dev) == 0
    assert torch.count_nonzero(got["P"][dropped]) == 0 and torch.count_nonzero(got["dPg"][dropped]) == 0
    worst = max(errs, key=errs.get)
    print(f"[vjp stage T dropout] {case}: worst {worst} {errs[worst]:.2e}  " + " ".join(f"{a}={b:.1e}" for a, b in errs.items()))
    assert errs[worst] <= BOUND, worst


def test_att_dp_zero_is_the_dropout_free_entry(gf, cuda_dev):
    """att_dp = 0 through _ex (cb and cbg given, and ignored) equals gf_attn_simplex_bwd_vjp bit for bit."""
    H, W, C, k = 10, 13, 96, 20
    for integration, norm in (("both", "layer"), ("mul", "none"), ("add", "layer")):
        ins, cb, cots, cbg = dropout_case(3, H, W, C, k, integration, 30.0, seed=4)
        a = run_stage_t(gf, cuda_dev, ins, cots, H=H, W=W, k=k, integration=integration, norm=norm)
        b = run_ex(gf, cuda_dev, ins, cb, cots, cbg, H=H, W=W, k=k, integration=integration, norm=norm, att_dp=0.0,
                   state=_state(cuda_dev, 1, 2))
        for nm in a:
            assert torch.equal(a[nm], b[nm]), (integration, nm)


def test_mask_is_gf_attn_dropout_mask(gf, cuda_dev):
    """The multipliers the kernel applies are those of gf_attn_dropout_mask (and of the host Philox draw): q = p * mask, with p
    from the dropout-free call, bit for bit."""
    B, H, W, C, k = 2, 10, 13, 64, 20
    ins, cb, cots, cbg = dropout_case(B, H, W, C, k, "mul", 0.0, seed=6)
    st = _state(cuda_dev, 987654321, 11)
    for att_dp in (0.12, 0.5):
        got = run_ex(gf, cuda_dev, ins, cb, cots, cbg, H=H, W=W, k=k, integration="mul", norm="layer", att_dp=att_dp, state=st)
        p0 = run_ex(gf, cuda_dev, ins, cb, cots, cbg, H=H, W=W, k=k, integration="mul", norm="layer", att_dp=0.0, state=st)["P"]
        desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, pos_dim=0)
        mask = torch.empty(B, H * W, pad_k(k), device=cuda_dev)
        gf._lib.check(gf._lib.load().gf_attn_dropout_mask(ctypes.byref(desc), ctypes.c_float(att_dp), SALT, st.data_ptr(),
                                                          mask.data_ptr(), _stream(cuda_dev)), "gf_attn_dropout_mask")
        torch.cuda.synchronize(cuda_dev)
        assert torch.equal(mask.cpu().double(), dr.philox_mult(att_dp, 987654321, 11, SALT, B, H * W, pad_k(k)))
        assert torch.equal(got["P"], p0 * mask)


def test_vjp_dropout_deterministic_batch_independent_and_graph_replay(gf, cuda_dev):
    """Two calls give the same bits, image 0 of a batch of 3 equals a batch of 1 (the mask is keyed by the token index b n + t, so
    the batch of 1 is image 0), and a CUDA-graph replay equals the eager call; a replay after the device step moved draws the new
    mask."""
    H, W, C, k = 10, 13, 96, 20
    kw = dict(H=H, W=W, k=k, integration="both", norm="layer", att_dp=0.12)
    ins, cb, cots, cbg = dropout_case(3, H, W, C, k, "both", 30.0, seed=1)
    st = _state(cuda_dev, 42, 3)
    a = run_ex(gf, cuda_dev, ins, cb, cots, cbg, state=st, **kw)
    b = run_ex(gf, cuda_dev, ins, cb, cots, cbg, state=st, **kw)
    one = run_ex(gf, cuda_dev, [t[:1] for t in ins], cb, [t[:1] for t in cots], cbg, state=st, **kw)
    for nm in a:
        assert torch.equal(a[nm], b[nm]), nm
        assert torch.equal(a[nm][:1], one[nm]), nm

    dev = cuda_dev
    X = _f32(ins[0], dev)
    B, n, _ = X.shape
    KP, Cout = pad_k(k), ins[3].shape[1]
    tabs = [_f32(t, dev) for t in ins[1:] + cots]
    cbd, cbgd = _f32(cb, dev), _f32(cbg, dev)
    o = {nm: torch.empty(a[nm].shape, device=dev) for nm in a}
    desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, heads=1, norm="layer", integration="both", pos_dim=0, duplex=False)
    lib = gf._lib.load()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            gf._lib.check(lib.gf_attn_simplex_bwd_vjp_ex(ctypes.byref(desc), X.data_ptr(), *(t.data_ptr() for t in tabs),
                                                         *(t.data_ptr() for t in o.values()), ctypes.c_float(0.12), SALT,
                                                         st.data_ptr(), cbd.data_ptr(), cbgd.data_ptr(), _stream(dev)), "capture")
    torch.cuda.current_stream(dev).wait_stream(side)
    for t in o.values():
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize(dev)
    for nm in o:
        assert torch.equal(o[nm], a[nm]), nm
    st[1] += 1                                                     # the state is read at run time: the replay draws a new mask
    graph.replay()
    c = run_ex(gf, cuda_dev, ins, cb, cots, cbg, state=st, **kw)
    torch.cuda.synchronize(dev)
    assert not torch.equal(o["P"], a["P"])
    for nm in o:
        assert torch.equal(o[nm], c[nm]), nm


def test_ex_refuses_dropout_without_cb(gf, cuda_dev):
    lib = gf._lib.load()
    desc = gf._lib.make_desc(1, 4, 4, 32, 4, D_LATENT, heads=1, norm="layer", integration="mul", pos_dim=0, duplex=False)
    t = torch.zeros(4096, device=cuda_dev)
    st = _state(cuda_dev, 1, 1)
    rc = lib.gf_attn_simplex_bwd_vjp_ex(ctypes.byref(desc), *([t.data_ptr()] * 19), ctypes.c_float(0.12), 0, st.data_ptr(), t.data_ptr(),
                                        None, _stream(cuda_dev))
    assert rc != 0 and b"cbg" in lib.gf_last_error()
