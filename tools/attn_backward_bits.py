"""Gradients of the attention layers' backward routes on seeded inputs, written to one file, and a bitwise comparison of two such
files: a change to the Python side of the backward that must not move any gradient is run on both trees and compared.

Cases (C = 64, 8x8 tokens, B = 2, D = 16; biases away from zero so that every term is live):
    simplex        every integration (mul / add / both) x norm (layer / none), attention dropout off and on; first order
    d-duplex       discriminator duplex layers (kernel_backward, img2ltnt): cotangents on the output and on the centroids
    duplex-dp      generator duplex layers with attention dropout, computed and given centroids; first order
    pl             path-length double backward (the gradient of |d<out, gout>/d(x, y, params)|^2) of a simplex layer with and
                   without dropout and of a duplex layer with dropout
    d-step / r1    a small discriminator with attention and r1_kernels=True: first-order gradients of the logits, and the image
                   gradient with the gradients of the R1 penalty (the double-backward kernels)
    composite      an instance-norm layer (composite route), first order and path-length double backward

    python tools/attn_backward_bits.py --out grads.pt
    python tools/attn_backward_bits.py --compare a.pt b.pt       # exit status 1 unless every tensor is torch.equal
"""
import argparse
import os
import sys
from importlib import import_module

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

C, H, W, K, D, B = 64, 8, 8, 8, 16, 2


def _layer(gf, dev, seed, **kw):
    torch.manual_seed(seed)
    attn = gf.BipartiteAttention(C, D, kw.pop("k", K), pos_dim=D, **kw).to(dev).train()
    attn.dp_salt = 0x1234567 + seed                      # masks independent of how many layers were built before
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in attn.named_parameters():
            if n.startswith("b"):
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
    return attn


def _inputs(dev, seed, k=K):
    g = torch.Generator().manual_seed(1000 + seed)
    x = torch.randn(B, H, W, C, generator=g).to(dev).requires_grad_(True)
    y = torch.randn(B, k, D, generator=g).to(dev).requires_grad_(True)
    return x, y, torch.randn(B, H, W, C, generator=g).to(dev), torch.randn(B, k, C, generator=g).to(dev)


def _first(attn, x, y, gout, centroids=None, gcen=None):
    out, _, cen = attn(x, y, centroids=centroids)
    outs, cots = ([out, cen], [gout, gcen]) if gcen is not None else ([out], [gout])
    return torch.autograd.grad(outs, [x, y, *attn.parameters()], cots, allow_unused=True)


def _second(attn, x, y, gout):
    leaves = [x, y, *attn.parameters()]
    g1 = torch.autograd.grad((attn(x, y)[0] * gout).sum(), leaves, create_graph=True, allow_unused=True)
    l2 = sum(t.square().sum() for t in g1 if t is not None)
    return [None if t is None else t.detach() for t in g1] + list(torch.autograd.grad(l2, leaves, allow_unused=True))


def run(dev):
    gf = import_module("gansformer_b200")
    am = import_module("gansformer-reproducibility-challenge_b200.attention")
    tr = import_module("gansformer-reproducibility-challenge_b200.training")
    res, seed = {}, 0

    def case(name, fn):
        nonlocal seed
        seed += 1
        am.set_dropout_seed(4242 + seed, dev, seed)
        res[name] = [None if t is None else t.detach().cpu() for t in fn(seed)]

    for integration in ("mul", "add", "both"):
        for norm in ("layer", None):
            for dp in (0.0, 0.25):
                k = 20 if norm is None else K                  # both latent paddings, KP = 32 and 16
                case(f"simplex-{integration}-{norm}-dp{dp}", lambda s: _first(_layer(gf, dev, s, integration=integration, norm=norm,
                                                                                       att_dp=dp, k=k), *_inputs(dev, s, k)[:3]))

    def d_layer(s, **kw):
        attn = _layer(gf, dev, s, kmeans=True, img2ltnt=True, **kw)
        attn.kernel_backward = True
        x, y, gout, gcen = _inputs(dev, s)
        return _first(attn, x, y, gout, gcen=gcen)
    case("d-duplex-mul-layer", lambda s: d_layer(s))
    case("d-duplex-both-none", lambda s: d_layer(s, integration="both", norm=None))

    def duplex_dp(s, given, **kw):
        x, y, gout, cen = _inputs(dev, s)
        return _first(_layer(gf, dev, s, kmeans=True, att_dp=0.25, **kw), x, y, gout, centroids=cen if given else None)
    case("duplex-dp-computed", lambda s: duplex_dp(s, False))
    case("duplex-dp-computed-img2ltnt", lambda s: duplex_dp(s, False, img2ltnt=True, integration="both"))
    case("duplex-dp-given", lambda s: duplex_dp(s, True))

    case("pl-simplex", lambda s: _second(_layer(gf, dev, s, exact_fp32=True), *_inputs(dev, s)[:3]))
    case("pl-simplex-dp", lambda s: _second(_layer(gf, dev, s, att_dp=0.25, integration="both", exact_fp32=True), *_inputs(dev, s)[:3]))
    case("pl-duplex-dp", lambda s: _second(_layer(gf, dev, s, kmeans=True, att_dp=0.25, exact_fp32=True), *_inputs(dev, s)[:3]))

    def disc(s, r1):
        torch.manual_seed(s)
        Dn = tr.Discriminator(32, fmap_base=1024, fmap_max=128, transformer=True, components_num=K, latent_dim=D, r1_kernels=True).to(dev)
        g = torch.Generator().manual_seed(s)
        with torch.no_grad():
            for n, p in Dn.named_parameters():
                if n.split(".")[-1] in ("bias", "bq", "bk", "bv", "bo", "bq2", "bk2", "bv2", "bi2l"):
                    p.copy_(0.2 * torch.randn(p.shape, generator=g))
        x = torch.randn(4, 3, 32, 32, generator=g).to(dev).requires_grad_(True)
        leaves = [x, *Dn.parameters()]
        if not r1:
            return torch.autograd.grad(Dn(x).sum(), leaves, allow_unused=True)
        (gx,) = torch.autograd.grad(Dn(x).sum(), x, create_graph=True)
        return [gx.detach(), *torch.autograd.grad(gx.square().sum(dim=[1, 2, 3]).mean(), leaves, allow_unused=True)]
    case("d-step", lambda s: disc(s, False))
    case("r1-kernels", lambda s: disc(s, True))

    case("composite-instance", lambda s: _first(_layer(gf, dev, s, norm="instance"), *_inputs(dev, s)[:3]))
    case("pl-composite-instance", lambda s: _second(_layer(gf, dev, s, norm="instance", exact_fp32=True), *_inputs(dev, s)[:3]))
    return res


def compare(a, b):
    ra, rb = torch.load(a), torch.load(b)
    bad = sorted(set(ra) ^ set(rb))
    for name in sorted(set(ra) & set(rb)):
        same = len(ra[name]) == len(rb[name]) and all((u is None and v is None) or (u is not None and v is not None and torch.equal(u, v))
                                                        for u, v in zip(ra[name], rb[name]))
        n = sum(t is not None for t in ra[name])
        print(f"{name:32s} {n:3d} tensors  {'equal' if same else 'DIFFERENT'}")
        if not same:
            bad.append(name)
    print(f"{len(ra)} cases, {'all bitwise equal' if not bad else 'differ: ' + ', '.join(bad)}")
    return not bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    if not torch.cuda.is_available():
        raise SystemExit("attn_backward_bits: no CUDA device (the routes run the H100 kernels)")
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    print(torch.cuda.get_device_name(0), flush=True)
    torch.save(run(torch.device("cuda:0")), args.out)


if __name__ == "__main__":
    main()
