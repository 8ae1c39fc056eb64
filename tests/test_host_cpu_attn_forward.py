"""CPU checks behind tests/test_gpu_attn_forward.py: every exact case of the forward kernels really is exact.

The GPU tests demand bit-for-bit equality between both stage-T kernel families, the pass-A kernel and the fp64 references.  That
is only fair if every probability is 0, 1/2 or 1 and every partial sum an fp32 value in any order.  These tests build each exact
case on the host and check it, as tests/test_host_cpu_attn_backward.py does for the backward: every partial sum of an intermediate
(logits, probabilities, control signal, modulation, noise and bias, activation, tRGB, post_scale) is a multiple of its grain with
a magnitude below 2^24 grains, and the fp64 reference's outputs round-trip through float32 unchanged.
"""
import torch

from oracle import attn_fwd as af
from tests.test_gpu_attn_forward import D_LATENT, EPILOGUES, EXACT_A, INSTANCES, POS, TILES, layout, plant, reference
from tests.test_host_cpu_attn_backward import _check_exact, _roundtrips


def _check_case(case, *, H, W, k, integration, post=None):
    items, p = af.stage_t_exactness(case, k=k, integration=integration, post=post)
    _check_exact(items)
    real = p[p > 0]
    assert ((real == 0.5) | (real == 1.0)).all(), "a probability other than 0, 1/2 or 1"
    want = reference(case, H=H, W=W, k=k, integration=integration, post=post)
    _roundtrips({name: t for name, t in want.items() if t is not None})


def test_stage_t_instantiation_cases_are_exact():
    for k, C, integration in INSTANCES:
        _check_case(af.exact_stage_t_case(3, 8, 32, C, k, integration, seed=C + k), H=8, W=32, k=k, integration=integration)


def test_stage_t_tile_dropout_and_multi_head_cases_are_exact():
    for H, W in TILES:
        for k, C, integration in ((16, 128, "mul"), (27, 64, "both")):
            _check_case(af.exact_stage_t_case(5, H, W, C, k, integration, seed=H * W + k), H=H, W=W, k=k, integration=integration)
    for H, W, C, k, integration in [(8, 16, 128, 16, "mul"), (8, 9, 64, 7, "add"), (4, 32, 512, 27, "add"), (8, 32, 256, 31, "mul")]:
        case = af.exact_stage_t_case(3, H, W, C, k, integration, dropout=True, seed=C + k + 1)
        assert set(case["mult"].unique().tolist()) == {0.0, 2.0}
        _check_case(case, H=H, W=W, k=k, integration=integration)
    for heads, k, C in [(2, 5, 128), (2, 12, 256), (4, 7, 64), (4, 8, 512)]:
        _check_case(af.exact_stage_t_case(3, 8, 16, C, k, "mul", heads=heads, seed=heads * 100 + k), H=8, W=16, k=k, integration="mul")


def test_stage_t_epilogue_cases_are_exact():
    """Includes the fp32 claims the epilogue relies on: 0.6f * 5 == 3 and 0.4f * 5 == 2."""
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    assert (f(0.6) * f(5.0)).item() == 3.0 and (f(0.4) * f(5.0)).item() == 2.0
    B, H, W = 3, 8, 16
    for integration, C, k, act, rgb, per_image, scales in EPILOGUES:
        for with_rgb, a in {(False, 0), (rgb, act)}:
            case = af.exact_stage_t_case(B, H, W, C, k, integration, dropout=(C == 256), seed=C + k + act)
            post = af.exact_postop(B, H * W, C, seed=C + k, act=a, rgb=with_rgb, per_image_noise=per_image, scales=scales)
            _check_case(case, H=H, W=W, k=k, integration=integration, post=post)
            if with_rgb and scales:                        # tRGB before and after post_scale differ: the test pins the order
                want = reference(case, H=H, W=W, k=k, integration=integration, post=post)
                late = reference(case, H=H, W=W, k=k, integration=integration, post={**post, "rgb_w": None})
                after = torch.einsum("btc,boc->bot", late["Xout"], post["rgb_w"]) + post["rgb_bias"][None, :, None]
                assert not torch.equal(after, want["rgb"])


def test_pass_a_cases_are_exact(gf):
    """Every logit is an integer below 2^24, the planted tokens carry weights 1 or 1/2 (runners-up present), and the reference
    Xbar is what fp32 gives for f32(acc * 1.000352220f) merged in split order.  The split ranges are derived as the GPU test
    derives them: the count from gf_attn_debug_layout (without a device the library sizes it for 132 SMs, the H100 SXM figure;
    the GPU test reads the count for the device it runs on), and 4 for the empty-split cases, which force that count."""
    cases = [(B, H, W, C, k, None, B * 1000 + C + k) for B, H, W, C, k, _ in EXACT_A]
    cases += [(2, 9, 64, 256, 20, 4, 77), (1, 9, 64, 512, 13, 4, 78)]          # test_pass_a_exact_empty_last_split
    for B, H, W, C, k, forced, seed in cases:
        n = H * W
        desc = gf._lib.make_desc(B, H, W, C, k, D_LATENT, norm="layer", integration="mul", pos_dim=POS, duplex=1)
        nsplit = forced or layout(gf, desc)["nsplit"]
        ranges = af.pass_a_split_ranges(n, nsplit)
        if forced:
            assert ranges[-1][0] == ranges[-1][1]
        win, run, tie = plant(B, H, W, k, ranges, seed=seed)
        tabs, L, wts = af.exact_pass_a_case(B, H, W, C, k, winners=win, runners_up=run, ties=tie, seed=seed)
        fin = torch.isfinite(L)
        assert torch.equal(L[fin].round(), L[fin]) and (L[fin].abs() < 2.0 ** 24).all()
        assert (L[:, :, k:] == -float("inf")).all()
        live = wts[wts > 0]
        assert ((live == 1.0) | (live == 0.5)).all()
        if n >= 4 * 64:
            assert ((wts == 0.5).sum(dim=2) == 2).any() and ((wts == 1.0).sum(dim=2) == 2).any()
        # the next planted token is at least 2^20 log2 units below: 2^(-2^20) is 0 in fp32
        top = L[:, :, :k].transpose(1, 2)
        below = top.amax(dim=2, keepdim=True) - top
        assert (below[wts == 0] > 2.0 ** 20).all()
        acc = (wts @ tabs["X"]).float()
        assert torch.equal(acc.double(), wts @ tabs["X"])
