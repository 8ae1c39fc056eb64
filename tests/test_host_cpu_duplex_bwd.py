"""CPU tests of the duplex pass-A backward entry points (gf_attn_centroid_stats / gf_attn_centroid_bwd) and of the configurations
attention dropout refuses.  Nothing here launches a kernel: every error below is raised before the device is touched."""
import ctypes

import pytest
import torch


def _desc(gf, B=2, duplex=1, norm="layer"):
    return gf._lib.make_desc(B, 8, 8, 64, 8, 16, norm=norm, integration="mul", pos_dim=16, duplex=duplex)


def _stats(lib, desc, ptr=1):
    return lib.gf_attn_centroid_stats(ctypes.byref(desc), *([ptr] * 7), None)


def _bwd(lib, desc, ptr=1):
    return lib.gf_attn_centroid_bwd(ctypes.byref(desc), *([ptr] * 9), None)


@pytest.mark.parametrize("call", [_stats, _bwd], ids=["stats", "bwd"])
def test_centroid_entry_points_validate_before_touching_the_device(gf, call):
    lib = gf._lib.load()
    err = lambda: lib.gf_last_error().decode()
    name = "gf_attn_centroid_stats" if call is _stats else "gf_attn_centroid_bwd"
    assert call(lib, _desc(gf), ptr=None) == -1 and "null pointer" in err() and name in err()          # GF_ERR_INVALID
    assert call(lib, _desc(gf, duplex=0)) == -1 and "desc.duplex is 0" in err()
    assert call(lib, _desc(gf, duplex=2)) == -2 and "one k-means iteration" in err()                  # GF_ERR_UNSUPPORTED
    assert call(lib, _desc(gf, norm="instance")) == -2 and "norm must be layer or none" in err()
    assert call(lib, _desc(gf, norm="batch")) == -2 and "norm must be layer or none" in err()
    assert call(lib, _desc(gf, B=65536)) == -2 and "B > 65535" in err()
    bad = _desc(gf)
    bad.C = 48
    assert call(lib, bad) == -2 and "C=48" in err()                                                   # descriptor checks come first


@pytest.mark.parametrize("kwargs", [dict(kmeans_iters=2), dict(norm="instance"), dict(norm="batch"), dict(num_heads=2, kmeans=False)],
                         ids=["kmeans_iters2", "instance", "batch", "multi-head"])
def test_attention_dropout_refuses_unsupported_layers(gf, kwargs):
    """Training-mode attention dropout: kmeans_iters > 1, instance / batch norm and multi-head layers keep raising
    NotImplementedError, with and without autograd, and the message names what is supported."""
    kw = dict(kmeans=True, att_dp=0.12)
    kw.update(kwargs)
    attn = gf.BipartiteAttention(64, 16, 8, **kw)
    attn.train()
    x, y = torch.randn(1, 4, 4, 64), torch.randn(1, 8, 16)
    with pytest.raises(NotImplementedError, match="duplex with kmeans_iters == 1"):
        attn(x.requires_grad_(True), y)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="norm layer / none"):
        attn(x, y)


def test_attention_dropout_refuses_iterative_carry(gf):
    attn = gf.BipartiteAttention(64, 16, 8, kmeans=True, iterative=True, att_dp=0.12)
    attn.train()
    x, y, cen = torch.randn(1, 4, 4, 64), torch.randn(1, 8, 16), torch.randn(1, 8, 64)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="iterative centroid carry"):
        attn(x, y, centroids_init=cen)
    with pytest.raises(NotImplementedError, match="iterative centroid carry"):
        attn(x.requires_grad_(True), y, centroids_init=cen)
