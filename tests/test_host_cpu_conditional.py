"""CPU checks of class-conditional generation and training (SURVEY A.4 item 14), and the host proofs behind the exact cases of
tests/test_gpu_conditional.py.

* ``c_dim = 0`` builds exactly the unconditional networks (state dict keys, shapes and initial values) and ignores labels bit for bit.
* The conditional generator's torch path (with the CUDA attention swapped for the oracle's) and the conditional discriminator
  against the fp64 restatement of tests/conditional_ref.py; labels are validated.
* The trainer hands the right labels to every call of every phase (a recording stand-in), and the data-parallel step with labels
  sharded like z keeps the replicas identical.
* Every exact case of gf_mapping_fwd_cond is exact: each partial sum a multiple of its grain below 2^24 grains, and a float32
  restatement equals the fp64 reference.
"""
import multiprocessing as mp
import os
from importlib import import_module

import pytest
import torch

from oracle import bipartite as ob
from tests import conditional_ref as cref
from tests import test_gpu_conditional as cx
from tests import test_gpu_ops_exact as ex
from tests.test_host_cpu_attn_backward import _check_exact, _roundtrips

TRAIN = "gansformer-reproducibility-challenge_b200.training"
F32, F64 = torch.float32, torch.float64
H100_SMEM_OPTIN = 232448


def _g(gf, **kw):
    torch.manual_seed(0)
    return gf.Generator(resolution=32, components_num=4, latent_dim=16, fmap_base=512, fmap_max=64, mapping_layers=2, **kw)


def _d(**kw):
    torch.manual_seed(0)
    return import_module(TRAIN).Discriminator(32, fmap_base=512, fmap_max=64, **kw)


def _live(G):
    with torch.no_grad():
        for n, p in G.named_parameters():
            if n.endswith("bias") or n.split(".")[-1] in ("bq", "bk", "bv", "bo"):
                p.normal_(0, 0.3)
            if n.endswith("noise_strength"):
                p.fill_(0.1)
        G.mapping.w_avg.normal_(0, 0.2)
    return G.double()


def _fake_attention(gf, monkeypatch):
    def fake_forward(self, x, y, centroids=None, return_att=False, out=None, centroids_init=None):
        w = {n: p.detach() for n, p in self.named_parameters(recurse=False)}
        o, att, cen = ob.transformer_layer(x.permute(0, 3, 1, 2), y, w, integration=self.integration, norm=self.norm,
                                           duplex=self.duplex, use_pos=self.use_pos, return_att=return_att,
                                           kmeans_iters=self.kmeans_iters, img2ltnt=self.img2ltnt, centroids_init=centroids_init)
        return o.permute(0, 2, 3, 1).contiguous(), att, cen
    monkeypatch.setattr(gf.BipartiteAttention, "forward", fake_forward)


# ------------------------------------------------------------------------------------------------ c_dim = 0 is unchanged
@pytest.mark.parametrize("kw", [dict(), dict(ltnt2ltnt=True, kmeans=True)], ids=["plain", "ltnt2ltnt-duplex"])
def test_c_dim_zero_generator_is_the_unconditional_one(gf, kw):
    a, b = _g(gf, **kw), _g(gf, c_dim=0, **kw)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(sa[n].shape == sb[n].shape and torch.equal(sa[n], sb[n]) for n in sa)
    assert "mapping.embed" not in sa


@pytest.mark.parametrize("transformer", [False, True])
def test_c_dim_zero_discriminator_is_the_unconditional_one(transformer):
    kw = dict(transformer=transformer, components_num=4, latent_dim=16)
    sa, sb = _d(**kw).state_dict(), _d(c_dim=0, **kw).state_dict()
    assert list(sa) == list(sb) and all(sa[n].shape == sb[n].shape and torch.equal(sa[n], sb[n]) for n in sa)
    assert sa["fc1.weight"].shape == (1, 64)


def test_c_dim_zero_ignores_labels(gf):
    G = _live(_g(gf, transformer=False))
    D = _d().double()
    z = torch.randn(3, 5, 16, dtype=F64)
    c = torch.eye(3, dtype=F64)
    img = torch.rand(3, 3, 32, 32, dtype=F64)
    with torch.no_grad():
        assert torch.equal(G(z), G(z, c)) and torch.equal(G(z, truncation_psi=0.6), G(z, c, truncation_psi=0.6))
        assert torch.equal(G.mapping(z), G.mapping(z, c))
        Gf = _g(gf, transformer=False)                                  # run() feeds float32 latents
        assert torch.equal(Gf.run(z.float()), Gf.run(z.float(), c.numpy()))
        assert torch.equal(D(img), D(img, c))


# ------------------------------------------------------------------------------------------------ against fp64
def test_conditional_generator_matches_fp64_without_attention(gf):
    G = _live(_g(gf, transformer=False, c_dim=3))
    assert G.mapping.embed.shape == (3, 16) and G.mapping.local[0].weight.shape == (16, 32) and G.mapping.glob[1].weight.shape == (16, 16)
    z = torch.randn(4, 5, 16, dtype=F64)
    c = torch.rand(4, 3, dtype=F64)                                     # soft labels: c_b E is a weighted sum of rows
    with torch.no_grad():
        img = G(z, c, truncation_psi=0.7)
    ref = cref.generator_forward(cref.cast(G.state_dict()), z, c, resolution=32, components_num=4, latent_dim=16, mapping_layers=2,
                                 truncation_psi=0.7)
    assert (img - ref).abs().max() < 1e-9 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("kw", [dict(), dict(ltnt2ltnt=True, kmeans=True)], ids=["simplex", "ltnt2ltnt-duplex"])
def test_conditional_generator_matches_fp64_with_patched_attention(gf, monkeypatch, kw):
    G = _live(_g(gf, c_dim=3, **kw))
    _fake_attention(gf, monkeypatch)
    z = torch.randn(3, 5, 16, dtype=F64)
    c = torch.nn.functional.one_hot(torch.tensor([2, 0, 1]), 3).to(F64)
    with torch.no_grad():
        img, atts = G(z, c, return_att=True)
        img_other = G(z, torch.roll(c, 1, dims=1))
    ref, ratts = cref.generator_forward(cref.cast(G.state_dict()), z, c, resolution=32, components_num=4, latent_dim=16,
                                        mapping_layers=2, return_att=True, duplex=bool(kw))
    assert (img - ref).abs().max() < 1e-9 * max(1.0, ref.abs().max().item())
    assert len(atts) == len(ratts) and all((a - r).abs().max() < 1e-10 for a, r in zip(atts, ratts))
    assert (img_other - img).abs().amax(dim=(1, 2, 3)).min() > 1e-3                 # another class, another image


def test_conditional_discriminator_matches_fp64():
    D = _d(c_dim=4).double()
    assert D.fc1.weight.shape == (4, 64)
    img = torch.rand(4, 3, 32, 32, dtype=F64) * 2 - 1
    c = torch.rand(4, 4, dtype=F64)
    with torch.no_grad():
        got = D(img, c)
    ref = cref.discriminator_forward(cref.cast(D.state_dict()), img, c)
    assert got.shape == (4,) and (got - ref).abs().max() < 1e-10 * max(1.0, ref.abs().max().item())
    # the projection: the logit is linear in the labels, the sum of the per-class logits
    with torch.no_grad():
        per_class = torch.stack([D(img, torch.eye(4, dtype=F64)[[j] * 4]) for j in range(4)], dim=1)
    assert torch.allclose((per_class * c).sum(dim=1), got, rtol=0, atol=1e-12)


def test_labels_are_validated(gf):
    tr = import_module(TRAIN)
    G, D = _g(gf, transformer=False, c_dim=3), _d(c_dim=3)
    z, img = torch.randn(2, 5, 16), torch.rand(2, 3, 32, 32)
    for bad in (None, torch.zeros(2, 4), torch.zeros(3, 3), torch.zeros(2)):
        with pytest.raises(ValueError):
            G(z, bad)
        with pytest.raises(ValueError):
            G.mapping(z, bad)
        with pytest.raises(ValueError):
            D(img, bad)
    with pytest.raises(ValueError):
        G.run(z.numpy())
    with pytest.raises(ValueError, match="same c_dim"):
        tr.Trainer(G, _d())
    with pytest.raises(ValueError, match="same c_dim"):
        tr.Trainer(_g(gf, transformer=False), D)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const"))
    with pytest.raises(ValueError, match="gen_c"):
        trainer.step(z, img)
    with pytest.raises(ValueError, match="real_c"):
        trainer.step(z, img, torch.eye(3)[:2], torch.eye(3))
    with pytest.raises(ValueError):
        gf.Generator(resolution=16, components_num=2, latent_dim=8, c_dim=-1)


# ------------------------------------------------------------------------------------------------ the trainer's labels
def test_trainer_passes_each_phase_its_labels(gf):
    """A recording stand-in around G, G.mapping and D: the D phase's fakes and logits use gen_c, the real logits and R1 real_c; the G
    phase, both style-mixing draws and the w_avg update gen_c; the path-length phase gen_c[:B'].  Every value is finite."""
    tr = import_module(TRAIN)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False,
                     c_dim=3)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32, c_dim=3)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", style_mixing=1.0, pl_weight=2.0, g_reg_interval=1, pl_batch_shrink=2))
    log = []
    m_fwd, d_fwd = G.mapping.forward, D.forward
    G.mapping.forward = lambda z, c=None, **kw: log.append(("mapping", z.shape[0], c.clone())) or m_fwd(z, c, **kw)
    D.forward = lambda img, c=None: log.append(("D", img.shape[0], c.clone())) or d_fwd(img, c)
    g = torch.Generator().manual_seed(3)
    z, reals = torch.randn(4, 5, 16, generator=g), torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    gen_c = torch.nn.functional.one_hot(torch.tensor([0, 1, 2, 0]), 3).float()
    real_c = torch.nn.functional.one_hot(torch.tensor([2, 2, 1, 0]), 3).float()
    st = trainer.step(z, reals, gen_c, real_c)
    assert all(map(lambda v: v == v and abs(v) < 1e6, (st.loss_g, st.loss_d, st.r1, st.pl_penalty, st.pl_mean)))
    assert st.r1 > 0 and st.pl_mean > 0
    seen = [(name, n, "gen" if torch.equal(c, gen_c[:n]) else "real" if torch.equal(c, real_c) else "?") for name, n, c in log]
    assert seen == [("mapping", 4, "gen"), ("mapping", 4, "gen"),         # D phase: style mixing maps z and z2
                    ("D", 4, "real"), ("D", 4, "gen"),                      # real logits (and R1 through them), fake logits
                    ("mapping", 4, "gen"), ("mapping", 4, "gen"), ("D", 4, "gen"),      # G phase
                    ("mapping", 2, "gen"),                                  # path length: the first B // 2 latents and labels
                    ("mapping", 4, "gen")], seen                            # w_avg update


def _train_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import gansformer_b200 as gf
    d = import_module("gansformer-reproducibility-challenge_b200.dist")
    tr = import_module(TRAIN)
    r, w, _ = d.init_distributed("gloo")
    torch.set_num_threads(2)
    torch.manual_seed(0)
    G = gf.Generator(resolution=16, components_num=4, latent_dim=16, fmap_base=256, fmap_max=32, mapping_layers=2, transformer=False,
                     c_dim=3)
    D = tr.Discriminator(16, fmap_base=256, fmap_max=32, c_dim=3)
    trainer = tr.Trainer(G, D, tr.TrainConfig(noise_mode="const", r1_gamma=0.0), world=w)
    g = torch.Generator().manual_seed(3)
    z, reals = torch.randn(4, 5, 16, generator=g), torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    gen_c = torch.nn.functional.one_hot(torch.tensor([0, 1, 2, 0]), 3).float()
    real_c = torch.nn.functional.one_hot(torch.tensor([2, 2, 1, 0]), 3).float()
    sh = lambda t: d.shard_batch(t, r, w)
    trainer.step(sh(z), sh(reals), sh(gen_c), sh(real_c))
    flat = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()]).numpy()
    q.put((r, flat(D), flat(G), G.mapping.embed.grad.abs().sum().item()))
    d.barrier()
    dist.destroy_process_group()


def test_conditional_step_world2_keeps_replicas_identical():
    """world_size-2 gloo with labels sharded like z and reals: both ranks end the step with identical weights."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    (_, d0, g0, e0), (_, d1, g1, e1) = res
    assert (d0 == d1).all() and (g0 == g1).all() and e0 > 0 and e0 == e1


# ------------------------------------------------------------------------------------------------ host proofs of the exact cases
@pytest.mark.parametrize("case", cx.COND_CASES, ids=cx.cond_id)
def test_conditional_mapping_cases_are_exact(case):
    """One-hot labels pick a row of E (+-1), so [z || e] has 2D entries +-1 and a pixel norm of exactly 1; every pre-activation is a
    multiple of 5 below 2^24 * 5, every activation an integer, the lerp at psi = 1/2 a multiple of 1/2; the float32 restatement
    equals the fp64 reference."""
    D, L, k, c_dim = case
    B = cx.cond_batch(k, ex.H100_SMS)
    z, c, E, W0, W, b, w_avg = cx.cond_case(D, L, k, c_dim, B)
    assert set(z.unique().tolist()) == {-1.0, 1.0} and set(E.unique().tolist()) <= {-1.0, 1.0}
    assert torch.equal(c.sum(dim=1), torch.ones(B, dtype=F64)) and set(c.unique().tolist()) <= {0.0, 1.0}
    nnz = 2 if L <= 2 else 1
    assert ((W0 != 0).sum(dim=1) == nnz).all() and ((W != 0).sum(dim=2) == nnz).all()
    assert (W0[:, D:] != 0).any(dim=1).any(dim=1).all()                     # the label half feeds layer 0 of both paths
    e = c @ E
    x = torch.cat([z, e[:, None].expand(-1, k + 1, -1)], dim=2)
    assert (x.square().mean(dim=2) == 1).all()
    items = []
    for path, sl in ((0, slice(0, k)), (1, slice(k, k + 1))):
        h, cm = x[:, sl], x[:, sl].abs()
        for l in range(L):
            Wl = W0[path] if l == 0 else W[path, l - 1]
            pre, cm = h @ Wl + b[path, l], cm @ Wl.abs() + b[path, l].abs()
            h = ex.lrelu5(pre)
            items += [(f"pre p{path} l{l}", pre, cm, 5.0), (f"act p{path} l{l}", h, cm, 1.0)]
        a = w_avg[path]
        items += [(f"lerp diff p{path}", h - a, cm + a.abs(), 1.0),
                  (f"lerp p{path}", a + cx.COND_PSI * (h - a), a.abs() + cx.COND_PSI * (cm + a.abs()), 0.5)]
    _check_exact(items)
    f02 = torch.tensor(0.2, dtype=F32)
    for avg in (w_avg, None):
        want = cx.cond_want(z, c, E, W0, W, b, avg, k)
        got32 = cx.cond_def(z.float(), c.float(), E.float(), W0.float(), W.float(), b.float(), None if avg is None else avg.float(),
                            cx.COND_PSI, k, exact_norm=True, lrelu=lambda v: torch.maximum(v, f02 * v))
        assert torch.equal(got32.double(), want)
        _roundtrips({"out": want})
    assert (torch.tensor(float(2 * D), dtype=F32) / (2 * D) + torch.tensor(1e-8, dtype=F32)).item() == 1.0


def test_conditional_cases_reach_the_edges_they_claim():
    """c_dim 1, 10, 1000; k 0, 1, 31; D 16 to 128; every batch wraps the grid of 132 CTAs; the shared memory fits; some cases give
    every image a class of its own, and the mutations each case list is meant to catch change their output."""
    assert {c[3] for c in cx.COND_CASES} == {1, 10, 1000} and {c[2] for c in cx.COND_CASES} >= {0, 1, 31}
    assert min(c[0] for c in cx.COND_CASES) == 16 and max(c[0] for c in cx.COND_CASES) == 128
    distinct = 0
    for D, L, k, c_dim in cx.COND_CASES:
        B = cx.cond_batch(k, ex.H100_SMS)
        assert B * (k + 1) > 2 * 8 * ex.H100_SMS
        assert (2 * L * D * D + 2 * L * D + 8 * 2 * D) * 4 <= H100_SMEM_OPTIN, (D, L)
        z, c, E, W0, W, b, w_avg = cx.cond_case(D, L, k, c_dim, B)
        cls = c.argmax(dim=1)
        distinct += len(cls.unique()) == B
        want = cx.cond_want(z, c, E, W0, W, b, w_avg, k)
        # the mapping b = row (mod B) instead of row / (k + 1): a different output wherever two of the images' classes differ
        if k > 0 and len(cls.unique()) > 1:
            rows = torch.arange(B * (k + 1)) % B
            c_bad = c[rows].reshape(B, k + 1, c_dim)
            e_bad = torch.einsum("bjc,cd->bjd", c_bad, E)
            x_bad = torch.cat([z, e_bad], dim=2)
            assert not torch.equal(x_bad, torch.cat([z, (c @ E)[:, None].expand(-1, k + 1, -1)], dim=2))
        assert want.abs().max() < 2 ** 24
    assert distinct >= 2
