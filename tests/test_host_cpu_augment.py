"""CPU checks of adaptive discriminator augmentation (SURVEY A.4 item 15): the fp64 definition of ops.augment, its adjoint and its
derivatives, the parameter sampler, the refusals of the two gf_ops.h entry points, and the trainer's augmentation and ADA controller.

The custom autograd functions that run the kernels on CUDA are checked here too, with the kernels swapped for the definition: their
first and second derivatives (the adjoint, then the linear part of the map again) must pass gradcheck and gradgradcheck.
"""
import json
import math
import multiprocessing as mp
import os
import subprocess
import sys
from importlib import import_module

import pytest
import torch

TRAIN = "gansformer-reproducibility-challenge_b200.training"
OPS = "gansformer-reproducibility-challenge_b200.ops"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
V = torch.full((3,), 1 / math.sqrt(3), dtype=F64)
VV = torch.outer(V, V)


def _geom(rows):
    return torch.tensor(rows, dtype=torch.int32)


def _color(M3x4):
    if isinstance(M3x4, (list, tuple)) and torch.is_tensor(M3x4[0]):
        return torch.stack(list(M3x4)).to(F64).reshape(-1, 12)
    return torch.as_tensor(M3x4, dtype=F64).reshape(-1, 12)


def _spec_index(code, tx, ty, H, W):
    """The blit of include/gf_ops.h written out pixel by pixel: source (row, col) of every output pixel."""
    code &= 7
    if H != W:
        code &= 5
    tx, ty = max(-(W - 1), min(W - 1, tx)), max(-(H - 1), min(H - 1, ty))
    R = lambda i, N: -i if i < 0 else (2 * (N - 1) - i if i >= N else i)
    out = {}
    for y in range(H):
        for x in range(W):
            xf = W - 1 - x if code & 1 else x
            u, v = [(xf, y), (y, W - 1 - xf), (W - 1 - xf, H - 1 - y), (H - 1 - y, xf)][code >> 1]
            out[(y, x)] = (R(v - ty, H), R(u - tx, W))
    return out


# ------------------------------------------------------------------------------------------------ the definition, fp64
def test_identity_parameters_give_the_identity():
    ops = import_module(OPS)
    x = torch.randn(3, 3, 5, 7, dtype=F64)
    I = _color([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]] * 3)
    assert torch.equal(ops.augment(x, torch.zeros(3, 4, dtype=torch.int32)), x)
    assert torch.equal(ops.augment(x, torch.zeros(3, 4, dtype=torch.int32), I), x)


@pytest.mark.parametrize("H,W", [(2, 2), (3, 3), (6, 6), (4, 7), (3, 2)])
def test_dihedral_codes_are_bijections_and_match_the_spec(H, W):
    ops = import_module(OPS)
    seen = set()
    for code in range(16):                                              # codes above 7 are masked to 3 bits
        idx = ops.augment_index(_geom([[code, 0, 0, 0]]), H, W)[0]
        assert sorted(idx.tolist()) == list(range(H * W)), code          # a permutation of the grid
        spec = _spec_index(code, 0, 0, H, W)
        assert idx.tolist() == [spec[(y, x)][0] * W + spec[(y, x)][1] for y in range(H) for x in range(W)]
        seen.add(tuple(idx.tolist()))
    assert len(seen) == (8 if H == W else 4)                            # non-square: the transposing codes fall back


@pytest.mark.parametrize("H,W", [(2, 2), (3, 3), (5, 5), (4, 6)])
def test_mirror_indices_at_the_edges(H, W):
    ops = import_module(OPS)
    for code in range(8):
        for tx in (-(W + 3), -(W - 1), -1, 0, 1, W - 1, W + 3):            # beyond N - 1: clamped
            for ty in (-(H - 1), -1, 0, 2, H - 1, 2 * H):
                idx = ops.augment_index(_geom([[code, tx, ty, 0]]), H, W)[0].tolist()
                spec = _spec_index(code, tx, ty, H, W)
                assert idx == [spec[(y, x)][0] * W + spec[(y, x)][1] for y in range(H) for x in range(W)], (code, tx, ty)
    idx = ops.augment_index(_geom([[0, W - 1, 0, 0]]), H, W)[0].reshape(H, W)   # a maximal shift: column x reads R(x - (W-1))
    assert idx[0].tolist() == [W - 1 - x for x in range(W)]
    idx = ops.augment_index(_geom([[0, -(W - 1), 0, 0]]), H, W)[0].reshape(H, W)
    assert idx[0].tolist() == [2 * (W - 1) - (x + W - 1) if x > 0 else W - 1 for x in range(W)]


def test_lumaflip_is_an_involution_and_saturation_one_is_the_identity():
    ops = import_module(OPS)
    x = torch.randn(2, 3, 4, 4, dtype=F64)
    g0 = torch.zeros(2, 4, dtype=torch.int32)
    L = torch.cat([torch.eye(3, dtype=F64) - 2 * VV, torch.zeros(3, 1, dtype=F64)], dim=1)
    twice = ops.augment(ops.augment(x, g0, _color([L, L])), g0, _color([L, L]))
    assert (twice - x).abs().max() < 1e-14
    S = torch.cat([VV + 1.0 * (torch.eye(3, dtype=F64) - VV), torch.zeros(3, 1, dtype=F64)], dim=1)
    assert (ops.augment(x, g0, _color([S, S])) - x).abs().max() < 1e-15


def test_geometry_and_colour_commute():
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 3, 6, 6, dtype=F64, generator=g)
    geom = _geom([[3, 2, -1, 0], [6, -5, 5, 0], [1, 0, 0, 0], [7, 1, 3, 0]])
    color = torch.randn(4, 12, dtype=F64, generator=g)
    g0 = torch.zeros(4, 4, dtype=torch.int32)
    both = ops.augment(x, geom, color)
    assert torch.equal(both, ops.augment(ops.augment(x, g0, color), geom))
    assert torch.equal(both, ops.augment(ops.augment(x, geom), g0, color))


@pytest.mark.parametrize("H,W", [(2, 2), (3, 3), (8, 8), (5, 9)])
@pytest.mark.parametrize("colour", [False, True])
def test_adjoint_identity(H, W, colour):
    """<L x, g> = <x, L^T g> for the linear part L of the map, over every code and maximal, negative and zero translations."""
    ops = import_module(OPS)
    g = torch.Generator().manual_seed(H * 100 + W)
    rows = [[c, t, s, 0] for c in range(8) for t, s in ((W - 1, H - 1), (-(W - 1), -(H - 1)), (0, 0), (1, -1))]
    B, C = len(rows), 3 if colour else 2
    geom = _geom(rows)
    color = torch.randn(B, 12, dtype=F64, generator=g) if colour else None
    lin = ops._linear_part(color)
    x, gy = torch.randn(B, C, H, W, dtype=F64, generator=g), torch.randn(B, C, H, W, dtype=F64, generator=g)
    lhs = (ops.augment_ref(x, geom, lin) * gy).sum(dim=(1, 2, 3))
    rhs = (x * ops.augment_adjoint_ref(gy, geom, color)).sum(dim=(1, 2, 3))
    assert (lhs - rhs).abs().max() < 1e-12 * max(1.0, lhs.abs().max().item())
    if colour:                                                          # the offset is the affine part: A x - A 0 = L x
        assert (ops.augment_ref(x, geom, color) - ops.augment_ref(torch.zeros_like(x), geom, color) - ops.augment_ref(x, geom, lin)).abs().max() < 1e-12


@pytest.fixture
def host_kernels(monkeypatch):
    """The CUDA autograd functions with the kernels replaced by the definition (fp64 on the CPU)."""
    ops = import_module(OPS)
    calls = []

    def native(name, x, geom, color):
        calls.append(name)
        f = ops.augment_ref if name == "gf_augment_nchw" else ops.augment_adjoint_ref
        return f(x.detach(), geom, color)
    monkeypatch.setattr(ops, "_augment_native", native)
    return ops, calls


@pytest.mark.parametrize("colour", [False, True])
def test_autograd_functions_gradcheck_and_gradgradcheck(host_kernels, colour):
    ops, calls = host_kernels
    g = torch.Generator().manual_seed(7)
    geom = _geom([[5, 2, -3, 0], [2, -4, 4, 0]])
    color = torch.randn(2, 12, dtype=F64, generator=g) if colour else None
    x = torch.randn(2, 3, 5, 5, dtype=F64, generator=g, requires_grad=True)
    f = lambda t: ops._Augment.apply(t, geom, color)
    assert torch.autograd.gradcheck(f, (x,))
    assert torch.autograd.gradgradcheck(f, (x,))
    assert "gf_augment_adjoint_nchw" in calls
    # the custom functions agree with torch autograd of the definition, to the second order
    xr = x.detach().clone().requires_grad_(True)
    w = torch.randn(2, 3, 5, 5, dtype=F64, generator=g)
    for fn, t in ((f, x), (lambda t: ops.augment_ref(t, geom, color), xr)):
        (gr,) = torch.autograd.grad((fn(t) * w).square().sum(), t, create_graph=True)
        (gg,) = torch.autograd.grad(gr.square().sum(), t)
        if fn is f:
            got = (gr.detach(), gg)
        else:
            want = (gr.detach(), gg)
    assert all((a - b).abs().max() < 1e-10 * max(1.0, b.abs().max().item()) for a, b in zip(got, want))


def test_plain_torch_gradcheck_of_the_definition():
    ops = import_module(OPS)
    geom = _geom([[4, 1, 1, 0]])
    color = torch.randn(1, 12, dtype=F64)
    x = torch.randn(1, 3, 3, 3, dtype=F64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: ops.augment(t, geom, color), (x,))
    assert torch.autograd.gradgradcheck(lambda t: ops.augment(t, geom, color), (x,))


def test_bad_arguments_raise():
    ops = import_module(OPS)
    x = torch.zeros(2, 3, 4, 4)
    with pytest.raises(ValueError):
        ops.augment(torch.zeros(2, 3, 1, 4), torch.zeros(2, 4, dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.augment(torch.zeros(2, 1, 4, 4), torch.zeros(2, 4, dtype=torch.int32), torch.zeros(2, 12))
    with pytest.raises(ValueError):
        ops.augment(x, torch.zeros(2, 3, dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.augment(x, torch.zeros(2, 4, dtype=torch.int32), torch.zeros(2, 9))


# ------------------------------------------------------------------------------------------------ the sampler
def test_sampler_p_zero_gives_identity_parameters():
    tr = import_module(TRAIN)
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 0.0, 64, 16, 16, "cpu")
    assert torch.equal(geom, torch.zeros(64, 4, dtype=torch.int32))
    assert torch.equal(color, torch.eye(4)[:3].reshape(1, 12).expand(64, 12))
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, torch.zeros(()), 8, 16, 16, "cpu")      # p as a tensor
    assert not geom.any() and torch.equal(color, torch.eye(4)[:3].reshape(1, 12).expand(8, 12))
    assert tr.sample_augment(("xflip", "xint"), 1.0, 4, 8, 8, "cpu")[1] is None


def test_sampler_p_one_frequencies_and_bounds():
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    B, H, W = 20000, 32, 24
    geom, _ = tr.sample_augment(("xflip", "xint"), 1.0, B, H, W, "cpu")
    assert abs((geom[:, 0] & 1).float().mean().item() - 0.5) < 0.02
    assert geom[:, 1].abs().max() <= round(0.125 * W) and geom[:, 2].abs().max() <= round(0.125 * H)
    assert geom[:, 1].abs().max() == 3 and geom[:, 2].abs().max() == 4 and not geom[:, 3].any()
    geom, color = tr.sample_augment(tr.AUGMENT_OPS, 1.0, B, 16, 16, "cpu")
    k = (geom[:, 0] >> 1).long()
    assert all(abs((k == j).float().mean().item() - 0.25) < 0.02 for j in range(4))
    assert geom[:, 1:3].abs().max() <= 2
    M = color.reshape(B, 3, 4).double()
    assert abs(M[:, :, 3].mean().item()) < 0.02                          # brightness offsets: mean 0 ...
    geom, _ = tr.sample_augment(("xflip",), 0.5, B, 16, 16, "cpu")       # p = 1/2: a flip applies to 1/2 of 1/2 of the images
    assert abs((geom[:, 0] & 1).float().mean().item() - 0.25) < 0.02
    # each colour transform alone, p = 1: its law
    b = tr.sample_augment(("brightness",), 1.0, B, 8, 8, "cpu")[1].reshape(B, 3, 4)
    assert abs(b[:, 0, 3].std().item() - 0.2) < 0.01 and torch.equal(b[:, :, :3], torch.eye(3).expand(B, 3, 3))
    c = tr.sample_augment(("contrast",), 1.0, B, 8, 8, "cpu")[1].reshape(B, 3, 4)[:, 0, 0]
    assert abs(torch.log2(c).std().item() - 0.5) < 0.02
    l = tr.sample_augment(("lumaflip",), 1.0, B, 8, 8, "cpu")[1].reshape(B, 3, 4)[:, :, :3].double()
    flipped = (l - (torch.eye(3, dtype=F64) - 2 * VV)).abs().amax(dim=(1, 2)) < 1e-6
    assert abs(flipped.double().mean().item() - 0.5) < 0.02
    h = tr.sample_augment(("hue",), 1.0, B, 8, 8, "cpu")[1].reshape(B, 3, 4)[:, :, :3].double()
    assert (h @ V - V).abs().max() < 1e-6 and (h @ h.transpose(1, 2) - torch.eye(3, dtype=F64)).abs().max() < 1e-5
    s = tr.sample_augment(("saturation",), 1.0, B, 8, 8, "cpu")[1].reshape(B, 3, 4)[:, :, :3].double()
    sat = torch.einsum("bij,i,j->b", s, torch.tensor([1.0, -1.0, 0.0], dtype=F64), torch.tensor([1.0, -1.0, 0.0], dtype=F64)) / 2
    assert abs(torch.log2(sat).std().item() - 1.0) < 0.03


def test_parse_augment_and_square_check():
    tr = import_module(TRAIN)
    assert tr.parse_augment("") == () and tr.parse_augment("bc") == tr.AUGMENT_OPS
    assert tr.parse_augment("hue, xflip") == ("xflip", "hue")
    with pytest.raises(ValueError):
        tr.parse_augment("xflip,cutout")
    with pytest.raises(ValueError):
        tr.sample_augment(("rotate90",), 1.0, 2, 8, 16, "cpu")


# ------------------------------------------------------------------------------------------------ the entry points refuse bad calls
_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import gansformer_b200 as gf
lib = gf._lib.load()
A = 0x10000
out = []
for name in ("gf_augment_nchw", "gf_augment_adjoint_nchw"):
    fn = getattr(lib, name)
    for args in ([A, A, A, A, 2, 3, 8, 8, None], [A, A, A, None, 2, 1, 8, 8, None],      # valid: fail at the launch (no device)
                 [None, A, A, A, 2, 3, 8, 8, None], [A, None, A, A, 2, 3, 8, 8, None], [A, A, None, A, 2, 3, 8, 8, None],
                 [A, A, A, A, 0, 3, 8, 8, None], [A, A, A, None, 2, 0, 8, 8, None], [A, A, A, A, 2, 3, -8, 8, None],
                 [A, A, A, A, 2, 3, 8, 1, None], [A, A, A, A, 2, 3, 1, 8, None], [A, A, A, A, 2, 4, 8, 8, None],
                 [A, A, A, A, 2, 1, 8, 8, None], [A, A, A, None, 2, 3, 40000, 8, None], [A, A, A, None, 2, 3000, 1000, 1000, None]):
        out.append([name, args, fn(*args), lib.gf_last_error().decode()])
print(json.dumps(out))
"""


def test_entry_points_refuse_bad_arguments():
    """Both entry points are exported, and refuse bad calls before touching the device: the child sees no GPU, so only a valid call
    gets as far as the launch (GF_ERR_CUDA)."""
    gf = import_module("gansformer_b200")
    assert {"gf_augment_nchw", "gf_augment_adjoint_nchw"} <= set(gf._lib.OPS_EXPORTS)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    want = [-3, -3, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2, -2, -2]
    for name in ("gf_augment_nchw", "gf_augment_adjoint_nchw"):
        got = [(rc, msg) for n, _, rc, msg in out if n == name]
        assert [rc for rc, _ in got] == want, (name, got)
        assert all(name in msg for rc, msg in got if rc != -3)
        assert "C == 3" in got[10][1] and "at least 2" in got[8][1] and "too large" in got[13][1]


# ------------------------------------------------------------------------------------------------ the trainer
def _gan(gf, **dkw):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32, **dkw)
    return tr, G, D


def _data(B=4, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 5, 16, generator=g), torch.rand(B, 3, 16, 16, generator=g) * 2 - 1


def _flat(m):
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()])


def test_augmentation_off_is_the_step_without_it(gf):
    """augment = "" (with the other new fields set): the same weights, bit for bit, as a trainer built without the new fields, over
    steps with and without R1."""
    tr = import_module(TRAIN)
    z, reals = _data()
    runs = []
    for cfg in (tr.TrainConfig(noise_mode="const", d_reg_interval=2),
                tr.TrainConfig(noise_mode="const", d_reg_interval=2, augment="", augment_p=0.7, ada_interval=1, ada_kimg=1.0)):
        _, G, D = _gan(gf)
        trainer = tr.Trainer(G, D, cfg)
        torch.manual_seed(11)
        stats = [trainer.step(z, reals) for _ in range(3)]
        assert trainer.augment_p is None and trainer.ada_stats is None
        runs.append((_flat(G), _flat(D), [(s.loss_d, s.loss_g, s.r1) for s in stats], torch.rand(3)))
    (g0, d0, s0, r0), (g1, d1, s1, r1) = runs
    assert torch.equal(g0, g1) and torch.equal(d0, d1) and s0 == s1 and torch.equal(r0, r1)   # the same random numbers drawn


@pytest.mark.parametrize("spec", ["bc", "xflip,rotate90,xint", "hue,saturation"])
def test_augmentation_on_runs_with_r1(gf, spec):
    tr = import_module(TRAIN)
    _, G, D = _gan(gf)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", d_reg_interval=2, augment=spec, augment_p=0.8, ada_target=0.6,
                                              ada_interval=1))
    z, reals = _data()
    seen = []
    d_fwd = D.forward
    D.forward = lambda img, c=None: seen.append(img) or d_fwd(img)
    stats = [trainer.step(z, reals) for _ in range(2)]
    assert stats[0].r1 > 0 and stats[1].r1 == 0
    assert all(math.isfinite(v) for s in stats for v in (s.loss_d, s.loss_g, s.r1, s.augment_p))
    assert len(seen) == 6 and not torch.equal(seen[0].detach(), reals)   # reals, fakes, fakes per step; the reals arrive augmented
    assert seen[0].requires_grad                                        # R1 differentiates through the augmentation


class _StubD(torch.nn.Module):
    """A discriminator whose logits are all `sign` (one parameter, so the step has something to update)."""

    def __init__(self, sign):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(()))
        self.sign = sign

    def forward(self, img, c=None):
        return self.sign + self.w * img.mean(dim=(1, 2, 3))


@pytest.mark.parametrize("interval", [1, 3])
def test_ada_rises_by_exactly_one_increment_per_interval(gf, interval):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    B, kimg = 4, 0.5
    trainer = tr.Trainer(G, _StubD(1.0), tr.TrainConfig(noise_mode="const", r1_gamma=0.0, augment="bc", augment_p=0.25,
                                                        ada_target=0.6, ada_interval=interval, ada_kimg=kimg))
    z, reals = _data(B)
    inc = torch.tensor(B * interval / (kimg * 1000.0), dtype=torch.float32)
    p = torch.tensor(0.25, dtype=torch.float32)
    for it in range(3 * interval):
        st = trainer.step(z, reals)
        if (it + 1) % interval == 0:
            p = (p + inc).clamp(0, 1)
            assert trainer.ada_stats.eq(0).all()
        else:
            assert trainer.ada_stats.tolist() == [B * ((it + 1) % interval)] * 2
        assert st.augment_p == p.item() and trainer.augment_p.item() == p.item(), it
    assert p.item() > 0.25


def test_ada_stays_at_zero_with_negative_logits(gf):
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    trainer = tr.Trainer(G, _StubD(-1.0), tr.TrainConfig(noise_mode="const", r1_gamma=0.0, augment="bc", ada_target=0.6, ada_interval=1,
                                                         ada_kimg=0.1))
    z, reals = _data()
    assert [trainer.step(z, reals).augment_p for _ in range(4)] == [0.0] * 4


def test_augment_config_is_validated(gf):
    tr = import_module(TRAIN)
    for kw in (dict(augment="bc", augment_p=1.5), dict(ada_target=0.6), dict(augment="bc", ada_target=2.0),
               dict(augment="bc", ada_target=0.6, ada_interval=0), dict(augment="bc", ada_target=0.6, ada_kimg=0.0),
               dict(augment="xflip,nope")):
        _, G, D = _gan(gf)
        with pytest.raises(ValueError):
            tr.Trainer(G, D, tr.TrainConfig(**kw))


class _SignD(torch.nn.Module):
    """A real discriminator plus 100 * the image mean: the sign of a logit is the sign of its image's mean."""

    def __init__(self, D):
        super().__init__()
        self.D = D

    def forward(self, img, c=None):
        return self.D(img) + 100.0 * img.mean(dim=(1, 2, 3))


def _ada_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import gansformer_b200 as gf
    d = import_module("gansformer-reproducibility-challenge_b200.dist")
    tr = import_module(TRAIN)
    r, w, _ = d.init_distributed("gloo")
    torch.set_num_threads(2)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False)
    D = _SignD(tr.Discriminator(16, fmap_base=256, fmap_max=32))
    # geometric transforms only: they keep the mean of a constant image, so the signs are known
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", augment="xflip,rotate90,xint", augment_p=0.5, ada_target=0.4,
                                              ada_interval=1, ada_kimg=1.0), world=w)
    g = torch.Generator().manual_seed(3)
    z = torch.randn(8, 5, 16, generator=g)
    signs = torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, -1.0, 1.0, -1.0])      # rank 0: mean sign 1; rank 1: 0; together 0.5 > 0.4
    reals = signs[:, None, None, None] * 0.5 * torch.ones(8, 3, 16, 16)
    sh = lambda t: d.shard_batch(t, r, w)
    st = trainer.step(sh(z), sh(reals))
    q.put((r, st.augment_p, _flat(D).numpy(), _flat(G).numpy()))
    d.barrier()
    dist.destroy_process_group()


def test_ada_world2_holds_the_same_p_on_every_rank():
    """world_size-2 gloo, shards whose mean signs (1 and 0) lie on either side of the target 0.4: the summed accumulators (mean 0.5)
    raise p on both ranks by B_global / (kimg * 1000), and the replicas stay identical."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 34500 + os.getpid() % 2000
    procs = [ctx.Process(target=_ada_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    (_, p0, d0, g0), (_, p1, d1, g1) = res
    want = (torch.tensor(0.5) + torch.tensor(8 / 1000.0)).item()
    assert p0 == p1 == want
    assert (d0 == d1).all() and (g0 == g1).all()
