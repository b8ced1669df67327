"""CPU tests of the bf16 producer layers' host side: the four bf16 entry points are exported, check their arguments
like the fp32 ones and fail without a GPU; layers._check accepts bf16 and nothing narrower; the producer's precision
option is validated; the native blocks stay where they were.  No device compute is attempted here."""
import ctypes
import os

import pytest

from conftest import gpu_count

# device pointers are never dereferenced on these paths: the calls fail in the argument check or at the launch
P = ctypes.c_void_p(0x1000)
BF16_ENTRIES = ["cos_lrn_forward_bf16", "cos_lrn_backward_bf16", "cos_bias_relu_maxpool_forward_bf16",
                "cos_bias_relu_maxpool_backward_bf16"]


def _lrn(L, which, size=5, ptrs=None, shape=(2, 8, 5, 5), k=1.0):
    if which == "forward":
        ptrs = ptrs or (P, P)
        return L.cos_lrn_forward_bf16(*ptrs, *shape, size, 1e-4, 0.75, k, None)
    ptrs = ptrs or (P, P, P)
    return L.cos_lrn_backward_bf16(*ptrs, *shape, size, 1e-4, 0.75, k, None)


def _pool_fwd(L, h=55, w=55, k=3, s=2, ph=27, pw=27, ptrs=None, nc=(2, 3)):
    return L.cos_bias_relu_maxpool_forward_bf16(*(ptrs or (P, P, P, P)), *nc, h, w, k, s, ph, pw, None)


def _pool_bwd(L, h=55, w=55, k=3, s=2, ph=27, pw=27, ptrs=None, nc=(2, 3)):
    return L.cos_bias_relu_maxpool_backward_bf16(*(ptrs or (P, P, P, P, P)), *nc, h, w, k, s, ph, pw, None)


def test_bf16_entry_points_are_exported(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    bound = {name for name, _, _ in _lib.SYMBOLS}
    for name in BF16_ENTRIES:
        assert name in bound
        assert getattr(L, name) is not None
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "caffedistri_b200.h")) as f:
        hdr = f.read()
    for name in BF16_ENTRIES:
        assert f"COS_API int {name}(" in hdr


@pytest.mark.parametrize("which", ["forward", "backward"])
def test_bf16_lrn_argument_checks(cos, which):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for size in (0, 2, 4, 17):
        assert _lrn(L, which, size) == 0
        assert b"local_size" in L.cos_last_error()
    assert _lrn(L, which, k=0.0) == 0
    assert b"k > 0" in L.cos_last_error()
    n = 2 if which == "forward" else 3
    for i in range(n):
        ptrs = [P] * n
        ptrs[i] = None
        assert _lrn(L, which, ptrs=tuple(ptrs)) == 0
        assert b"NULL" in L.cos_last_error()
    assert _lrn(L, which, shape=(2, 8, 0, 5)) == 0
    assert b"bad shape" in L.cos_last_error()


@pytest.mark.parametrize("fn,nptr", [(_pool_fwd, 4), (_pool_bwd, 5)])
def test_bf16_pool_argument_checks(cos, fn, nptr):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert fn(L, 32, 32, 3, 2, 15, 16) == 0  # CIFAR-10-quick pool1: 32 -> 16 (last window clipped)
    assert b"pooled size" in L.cos_last_error()
    assert fn(L, 55, 55, 16, 2, 20, 20) == 0
    assert b"kernel" in L.cos_last_error()
    assert fn(L, 2, 2, 3, 2, 1, 1) == 0  # input smaller than the window
    for i in range(nptr):
        ptrs = [P] * nptr
        ptrs[i] = None
        assert fn(L, ptrs=tuple(ptrs)) == 0
        assert b"NULL" in L.cos_last_error()
    assert fn(L, nc=(-1, 3)) == 0
    assert b"bad shape" in L.cos_last_error()


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
def test_bf16_entry_points_fail_loudly_without_a_gpu(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for call in (lambda: _lrn(L, "forward"), lambda: _lrn(L, "backward"), lambda: _pool_fwd(L),
                 lambda: _pool_bwd(L)):
        assert call() == 0
        assert b"no CPU path" in L.cos_last_error()


def test_check_accepts_bf16_and_rejects_other_dtypes():
    import torch
    from caffeonspark_b200 import layers
    from caffeonspark_b200.caffenet import CosError

    class FakeCuda:  # _check only reads these attributes; no device is needed to exercise it
        def __init__(self, dtype, dim=4, is_cuda=True):
            self.dtype, self._dim, self.is_cuda, self.shape, self.device = dtype, dim, is_cuda, (1,) * dim, "cuda:0"

        def dim(self):
            return self._dim

        def contiguous(self):
            return self

    for dt in (torch.float32, torch.bfloat16):
        t = FakeCuda(dt)
        assert layers._check(t) is t
    for bad in (FakeCuda(torch.float16), FakeCuda(torch.float64), FakeCuda(torch.bfloat16, dim=3),
                FakeCuda(torch.bfloat16, is_cuda=False)):
        with pytest.raises(CosError, match="fp32 or bf16 CUDA tensors"):
            layers._check(bad)
    with pytest.raises(CosError, match="no CPU path"):
        layers._check(torch.zeros((1, 1, 1, 1), dtype=torch.bfloat16))


@pytest.mark.parametrize("precision", ["fp16", "BF16", "tf32", "", None])
def test_unknown_precision_is_rejected(precision):
    import torch
    from caffeonspark_b200 import harness
    from caffeonspark_b200.caffenet import CosError
    with pytest.raises(CosError, match="precision"):
        harness.TorchProducer(None, torch.nn.Sequential(), precision=precision)
    with pytest.raises(CosError, match="precision"):
        harness.make_producer("lenet", None, precision=precision)


def test_default_precision_is_fp32():
    import inspect
    from caffeonspark_b200 import harness
    assert inspect.signature(harness.make_producer).parameters["precision"].default == "fp32"
    assert inspect.signature(harness.TorchProducer).parameters["precision"].default == "fp32"


def test_torch_module_places_the_native_blocks_at_the_same_layers():
    from caffeonspark_b200 import nets
    kinds = {name: [type(m).__name__ for m in nets.torch_module(name)] for name in nets.NETS}
    assert kinds["lenet"] == ["Conv2d", "MaxPool2d", "Conv2d", "MaxPool2d", "Flatten", "Linear", "ReLU", "Linear"]
    assert [i for i, k in enumerate(kinds["cifar10_quick"]) if k == "ConvReluMaxPool"] == [0]
    assert [i for i, k in enumerate(kinds["caffenet"]) if k == "ConvReluMaxPool"] == [0, 2, 8]
    assert [i for i, k in enumerate(kinds["caffenet"]) if k == "LRN"] == [1, 3]
