"""CPU tests of the native producer layers' host side: argument checks of the C entry points, their failure
without a GPU, and how nets.torch_module places the native blocks.  No device compute is attempted here."""
import ctypes

import pytest

from conftest import gpu_count

# device pointers are never dereferenced on these paths: the calls fail in the argument check or at the launch
P = ctypes.c_void_p(0x1000)


def _lrn(L, which, size, **kw):
    hyper = dict(alpha=1e-4, beta=0.75, k=1.0)
    hyper.update(kw)
    if which == "forward":
        return L.cos_lrn_forward(P, P, 2, 8, 5, 5, size, hyper["alpha"], hyper["beta"], hyper["k"], None)
    return L.cos_lrn_backward(P, P, P, 2, 8, 5, 5, size, hyper["alpha"], hyper["beta"], hyper["k"], None)


def _pool_fwd(L, h, w, k, s, ph, pw):
    return L.cos_bias_relu_maxpool_forward(P, P, P, P, 2, 3, h, w, k, s, ph, pw, None)


def _pool_bwd(L, h, w, k, s, ph, pw):
    return L.cos_bias_relu_maxpool_backward(P, P, P, P, P, 2, 3, h, w, k, s, ph, pw, None)


@pytest.mark.parametrize("which", ["forward", "backward"])
@pytest.mark.parametrize("size", [0, 2, 4, 17])
def test_lrn_rejects_even_or_unsupported_local_size(cos, which, size):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert _lrn(L, which, size) == 0
    assert b"local_size" in L.cos_last_error()


def test_lrn_rejects_non_positive_k(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert _lrn(L, "forward", 5, k=0.0) == 0
    assert b"k > 0" in L.cos_last_error()


@pytest.mark.parametrize("fn", [_pool_fwd, _pool_bwd])
def test_pool_rejects_a_pooled_size_that_is_not_ceil_mode(cos, fn):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert fn(L, 32, 32, 3, 2, 15, 16) == 0  # CIFAR-10-quick pool1: 32 -> 16 (last window clipped)
    assert b"pooled size" in L.cos_last_error()
    assert fn(L, 55, 55, 16, 2, 20, 20) == 0
    assert b"kernel" in L.cos_last_error()
    assert fn(L, 2, 2, 3, 2, 1, 1) == 0  # input smaller than the window


def test_pooled_size_matches_the_layout(cos):
    from caffeonspark_b200 import layers, nets
    for n, k, s in [(55, 3, 2), (27, 3, 2), (13, 3, 2), (32, 3, 2), (16, 3, 2), (24, 2, 2), (8, 2, 2), (9, 3, 2),
                    (7, 3, 3), (10, 2, 3)]:
        assert layers.pooled_size(n, k, s) == min(nets._pool_out(n, k, s), -(-n // s)), (n, k, s)


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
def test_layer_entry_points_fail_loudly_without_a_gpu(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    calls = [lambda: _lrn(L, "forward", 5), lambda: _lrn(L, "backward", 5),
             lambda: _pool_fwd(L, 55, 55, 3, 2, 27, 27), lambda: _pool_bwd(L, 55, 55, 3, 2, 27, 27)]
    for call in calls:
        assert call() == 0
        assert b"no CPU path" in L.cos_last_error()


def test_torch_module_places_the_native_blocks():
    import torch.nn as nn
    from caffeonspark_b200 import layers, nets
    kinds = {name: [type(m).__name__ for m in nets.torch_module(name)] for name in nets.NETS}
    assert kinds["lenet"] == ["Conv2d", "MaxPool2d", "Conv2d", "MaxPool2d", "Flatten", "Linear", "ReLU", "Linear"]
    assert kinds["cifar10_quick"][:3] == ["ConvReluMaxPool", "Conv2d", "ReLU"]
    assert kinds["cifar10_quick"].count("AvgPool2d") == 2
    assert kinds["caffenet"][:7] == ["ConvReluMaxPool", "LRN", "ConvReluMaxPool", "LRN", "Conv2d", "ReLU", "Conv2d"]
    assert kinds["caffenet"][7:10] == ["ReLU", "ConvReluMaxPool", "Flatten"]
    assert kinds["caffenet"].count("Dropout") == 2
    blk = nets.torch_module("caffenet")[0]
    assert isinstance(blk.conv, nn.Conv2d) and (blk.kernel, blk.stride) == (3, 2)
    assert isinstance(nets.torch_module("caffenet")[1], layers.LRN)


def test_torch_module_keeps_the_seeded_initial_weights():
    """The fused blocks keep their nn.Conv2d, so parameters() and reset_parameters() run in the same order as a
    plain layer list and a seed gives the same initial weights."""
    import torch
    import torch.nn as nn
    from caffeonspark_b200 import nets

    def plain(name):
        c = nets.NETS[name]["input"][0]
        mods = []
        for L in nets.NETS[name]["layers"]:
            if L[0] == "conv":
                mods.append(nn.Conv2d(c, L[2], L[3], stride=L[4], padding=L[5], groups=L[6]))
                c = L[2]
            elif L[0] == "ip":
                mods.append(nn.LazyLinear(L[2]))
        return mods

    for name in ("cifar10_quick", "caffenet"):
        mod = nets.torch_module(name)
        ref = [m for m in plain(name) if isinstance(m, nn.Conv2d)]
        convs = [m for m in mod.modules() if isinstance(m, nn.Conv2d)]
        assert [tuple(m.weight.shape) for m in convs] == [tuple(m.weight.shape) for m in ref]
        seq = [p for p in mod.parameters()]
        torch.manual_seed(7)
        for m in mod.modules():
            if hasattr(m, "reset_parameters"):
                m.reset_parameters()
        torch.manual_seed(7)
        for m in ref:
            m.reset_parameters()
        for a, b in zip(convs, ref):
            assert torch.equal(a.weight, b.weight) and torch.equal(a.bias, b.bias)
        assert seq[0] is convs[0].weight and seq[1] is convs[0].bias
