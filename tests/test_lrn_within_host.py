"""CPU tests of within-channel LRN and the cifar10_full net: the parser's lrn_param fields, the engine's plan of the
reference's cifar10_full files, the unchanged refusal of cross-channel LRN, the CPU composition in layers.LRN against
a float64 restatement of Caffe's layers, and the argument checks of the new C entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, gpu_count
from lrn_within_ref import SIZES, composition, lrn_within_backward_ref, lrn_within_ref
from test_native_producer_host import _check_layout, _ops

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
FULL_SOLVER = os.path.join(CONFIGS, "cifar10_full_solver.prototxt")
FULL_OPS = ["ConvBiasReLUMaxPool conv1+pool1+relu1 100x3x32x32 -> 100x32x16x16",
            "LRN(WITHIN_CHANNEL) norm1 100x32x16x16 -> 100x32x16x16",
            "Convolution conv2 100x32x16x16 -> 100x32x16x16", "ReLU relu2 100x32x16x16 -> 100x32x16x16",
            "Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8", "LRN(WITHIN_CHANNEL) norm2 100x32x8x8 -> 100x32x8x8",
            "Convolution conv3 100x32x8x8 -> 100x64x8x8", "ReLU relu3 100x64x8x8 -> 100x64x8x8",
            "Pooling(AVE) pool3 100x64x8x8 -> 100x64x4x4", "InnerProduct ip1 100x64x4x4 -> 100x10",
            "SoftmaxWithLoss loss 100x10 -> scalar"]
FULL_P = 89578

P = ctypes.c_void_p(0x1000)  # never dereferenced: the calls fail in the argument check or at the launch


def _net(tmp_path, lrn_param, bottom_shape="2 channels: 3 height: 8 width: 8"):
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "data" type: "MemoryData" top: "data" top: "label" memory_data_param '
                 f'{{ batch_size: {bottom_shape} }} }}\n'
                 f'layer {{ name: "norm" type: "LRN" bottom: "data" top: "norm" {lrn_param} }}\n'
                 'layer { name: "ip" type: "InnerProduct" bottom: "norm" top: "ip" inner_product_param '
                 '{ num_output: 4 } }\n'
                 'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')
    return str(p)


def _lrn_line(text):
    return next(line for line in text.splitlines() if " norm " in line)


@pytest.mark.parametrize("lrn_param,want", [
    ("lrn_param { norm_region: WITHIN_CHANNEL }", "n=5 alpha=1 beta=0.75"),  # caffe.proto defaults
    ("lrn_param { local_size: 3 alpha: 5e-05 beta: 0.75 norm_region: WITHIN_CHANNEL }", "n=3 alpha=5e-05 beta=0.75"),
    ("lrn_param { local_size: 15 alpha: 0.25 beta: -0.5 k: 7 norm_region: 1 }", "n=15 alpha=0.25 beta=-0.5"),
])
def test_parser_records_the_lrn_param_fields(cos, tmp_path, lrn_param, want):
    line = _lrn_line(cos.native_producer_plan(_net(tmp_path, lrn_param)))
    assert line.split()[2] == "LRN(WITHIN_CHANNEL)" and line.endswith(want + " staged-bottom")


@pytest.mark.parametrize("lrn_param", ["", "lrn_param { local_size: 3 }", "lrn_param { norm_region: ACROSS_CHANNELS }",
                                       "lrn_param { local_size: 3 norm_region: 0 }"])
def test_across_channels_lrn_keeps_its_refusal(cos, tmp_path, lrn_param):
    with pytest.raises(cos.CosError, match=r"^layer 'norm' \(LRN\): layer type not supported"):
        cos.native_producer_plan(_net(tmp_path, lrn_param))


@pytest.mark.parametrize("lrn_param,match", [
    ("lrn_param { local_size: 4 norm_region: WITHIN_CHANNEL }", "local_size 4 is not odd"),
    ("lrn_param { local_size: 17 norm_region: WITHIN_CHANNEL }", "local_size 17 is not odd and <= 15"),
])
def test_within_channel_lrn_refuses_unsupported_windows(cos, tmp_path, lrn_param, match):
    with pytest.raises(cos.CosError, match=r"layer 'norm' \(LRN\): " + match):
        cos.native_producer_plan(_net(tmp_path, lrn_param))


def test_lrn_fields_leave_the_layout_unchanged(cos, tmp_path):
    solver = tmp_path / "solver.prototxt"
    solver.write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    counts = []
    for lrn_param in ("lrn_param { local_size: 3 alpha: 2 norm_region: WITHIN_CHANNEL }", ""):
        _net(tmp_path, lrn_param)
        counts.append(cos.parse_solver(str(solver)).counts)
    assert counts == [[4 * 192, 4]] * 2


def test_plan_of_the_reference_cifar10_full_files(cos):
    text = cos.native_producer_plan(FULL_SOLVER)
    assert _ops(text) == FULL_OPS
    _check_layout(cos, text, FULL_SOLVER, FULL_P)
    lrn = [line for line in text.splitlines() if "LRN(WITHIN_CHANNEL)" in line]
    assert len(lrn) == 2 and all(line.endswith("n=3 alpha=5e-05 beta=0.75") for line in lrn)
    # the LRN top always has storage of its own, and norm1's bottom is not staged, so it takes a data gradient
    assert all("in-place" not in line and "staged-bottom" not in line for line in lrn)
    assert "blob 0 0:2400 32x3x5x5 gaussian" in text and "blob 6 79328:10240 10x1024 gaussian" in text


def test_cifar10_full_entry_matches_the_reference_files(cos, tmp_path):
    from caffeonspark_b200 import nets
    d = cos.parse_solver(FULL_SOLVER)
    counts, lm, dm, _ = nets.layout("cifar10_full")
    assert d.counts == counts and d.lr_mult == lm and d.decay_mult == dm
    assert d.param_count == nets.EXPECTED_PARAM_COUNT["cifar10_full"] == FULL_P
    assert lm == [1, 2, 1, 2, 1, 1, 1, 2] and dm == [1, 1, 1, 1, 1, 1, 250, 0]
    s = nets.NETS["cifar10_full"]["solver"]
    assert (d.lr_policy, d.max_iter, d.batch_size) == (s["lr_policy"], s["max_iter"], 100) == ("fixed", 60000, 100)
    assert (d.base_lr, d.momentum, d.weight_decay) == pytest.approx((0.001, 0.9, 0.004))
    # the generated prototxt gives the reference files' plan, fillers included
    generated = cos.native_producer_plan(nets.write_prototxts("cifar10_full", str(tmp_path)))
    assert generated == cos.native_producer_plan(FULL_SOLVER)


def test_torch_module_runs_within_channel_lrn():
    from caffeonspark_b200 import layers, nets
    mod = nets.torch_module("cifar10_full")
    lrn = [m for m in mod if isinstance(m, layers.LRN)]
    assert [(m.size, m.alpha, m.beta, m.region) for m in lrn] == [(3, 5e-05, 0.75, "WITHIN_CHANNEL")] * 2
    assert [type(m).__name__ for m in mod][:3] == ["ConvReluMaxPool", "LRN", "Conv2d"]
    assert layers.LRN(5).region == "ACROSS_CHANNELS"
    with pytest.raises(ValueError, match="region"):
        layers.LRN(3, region="WITHIN")


def _inputs(shape, seed):
    rng = np.random.RandomState(seed)
    return (rng.standard_normal(shape) * 3).astype(np.float32), rng.standard_normal(shape).astype(np.float32)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", [(2, 3, 1, 1), (1, 2, 3, 2), (2, 2, 9, 7)])
def test_cpu_composition_matches_caffes_layers_in_float64(size, shape):
    from caffeonspark_b200 import layers
    x, dy = _inputs(shape, size)
    alpha, beta = 0.5, 0.75
    want = composition(x, size, alpha, beta)
    xt = torch.from_numpy(x).double().requires_grad_()
    y = layers.LRN(size, alpha=float(np.float32(alpha)), beta=beta, region="WITHIN_CHANNEL")(xt)
    np.testing.assert_allclose(y.detach().numpy(), want, rtol=1e-12, atol=0)
    np.testing.assert_allclose(lrn_within_ref(x, size, alpha, beta)[0], want, rtol=1e-12, atol=0)
    # the reference's gradient formula is the composition's gradient
    y.backward(torch.from_numpy(dy).double())
    dx, ma, mb = lrn_within_backward_ref(x, dy, size, alpha, beta)
    assert np.all(np.abs(xt.grad.numpy() - dx) <= 1e-12 * (ma + mb))


def _within(L, which, size, num=2, ptrs=(P, P, P), bf16=False, beta=0.75):
    suffix = "_bf16" if bf16 else ""
    if which == "forward":
        return getattr(L, "cos_lrn_within_forward" + suffix)(ptrs[0], ptrs[1], num, 8, 5, 5, size, 1e-4, beta, None)
    return getattr(L, "cos_lrn_within_backward" + suffix)(*ptrs, num, 8, 5, 5, size, 1e-4, beta, None)


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("which", ["forward", "backward"])
def test_within_entry_points_reject_bad_arguments(cos, which, bf16):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for size in (0, 2, 4, 16, 17):
        assert _within(L, which, size, bf16=bf16) == 0
        assert b"local_size" in L.cos_last_error()
    assert _within(L, which, 3, ptrs=(None, P, P), bf16=bf16) == 0 and b"NULL" in L.cos_last_error()
    assert _within(L, which, 3, ptrs=(P, None, None), bf16=bf16) == 0 and b"NULL" in L.cos_last_error()
    assert _within(L, which, 3, num=-1, ptrs=(P, ctypes.c_void_p(0x100000), ctypes.c_void_p(0x200000)),
                   bf16=bf16) == 0 and b"bad shape" in L.cos_last_error()
    assert _within(L, which, 3, beta=float("nan"), ptrs=(P, ctypes.c_void_p(0x100000), ctypes.c_void_p(0x200000)),
                   bf16=bf16) == 0 and b"beta" in L.cos_last_error()
    # in place, or an output overlapping an input by one element
    elem = 2 if bf16 else 4
    last = ctypes.c_void_p(0x1000 + (2 * 8 * 5 * 5 - 1) * elem)
    far = ctypes.c_void_p(0x100000)
    cases = [(P, P, P), (P, last, last)] if which == "forward" else [(P, far, P), (far, P, P), (P, far, last)]
    for ptrs in cases:
        assert _within(L, which, 3, ptrs=ptrs, bf16=bf16) == 0, ptrs
        assert b"in place" in L.cos_last_error()


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
@pytest.mark.parametrize("bf16", [False, True])
def test_within_entry_points_fail_loudly_without_a_gpu(cos, bf16):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    apart = (ctypes.c_void_p(0x1000), ctypes.c_void_p(0x100000), ctypes.c_void_p(0x200000))
    for which in ("forward", "backward"):
        assert _within(L, which, 3, ptrs=apart, bf16=bf16) == 0
        assert b"no CPU path" in L.cos_last_error()
