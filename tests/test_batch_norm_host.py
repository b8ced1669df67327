"""CPU tests of BatchNorm support: the layout parser on the reference's BN example (tests/golden/configs), the
cifar10_full_bn net, the C entry points' argument checks and their failure without a GPU, and the producer
module's CPU composition against a float64 numpy restatement of batch_norm_layer.cpp."""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT, gpu_count
from test_caffe_proto_io import _c_blobs, _strs, pb  # noqa: F401  (pb: fixture)

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
P = ctypes.c_void_p(0x1000)  # never dereferenced: the calls fail in the argument check or at the launch

BN_P, BN_BLOBS = 89709, 14
BN_COUNTS = [2400, 32, 32, 1, 25600, 32, 32, 1, 51200, 64, 64, 1, 10240, 10]


def _memory_data_copy(tmp_path):
    """The reference's BN solver and net with the two LMDB Data layers swapped for MemoryData."""
    net = open(os.path.join(CONFIGS, "cifar10_full_sigmoid_train_test_bn.prototxt")).read()
    start = net.index("layer {")
    end = net.index('layer {\n  name: "conv1"')
    data = "".join(f'layer {{ name: "cifar" type: "MemoryData" top: "data" top: "label" include {{ phase: {ph} }} '
                   f'memory_data_param {{ batch_size: {b} channels: 3 height: 32 width: 32 }} }}\n'
                   for ph, b in (("TRAIN", 100), ("TEST", 1000)))
    (tmp_path / "net.prototxt").write_text(net[:start] + data + net[end:])
    solver = open(os.path.join(CONFIGS, "cifar10_full_sigmoid_solver_bn.prototxt")).read()
    solver = solver.replace('net: "examples/cifar10/cifar10_full_sigmoid_train_test_bn.prototxt"', 'net: "net.prototxt"')
    (tmp_path / "solver.prototxt").write_text(solver)
    return str(tmp_path / "solver.prototxt")


def test_reference_bn_example_parses_to_the_pinned_layout(cos, tmp_path):
    d = cos.parse_solver(_memory_data_copy(tmp_path))
    assert d.param_count == BN_P and len(d.counts) == BN_BLOBS
    assert d.counts == BN_COUNTS
    bn = [4 * i + k for i in range(3) for k in (1, 2, 3)]  # conv, then the layer's three BN blobs
    assert [d.lr_mult[i] for i in bn] == [0.0] * 9 and [d.decay_mult[i] for i in bn] == [1.0] * 9
    assert (d.lr_mult[-1], d.decay_mult[-1]) == (1.0, 0.0)  # ip1 bias
    assert (d.lr_mult[-2], d.decay_mult[-2]) == (1.0, 1.0)
    assert d.lr_policy == "step" and d.base_lr == pytest.approx(0.001) and d.momentum == pytest.approx(0.9)
    assert d.gamma == 1.0 and d.stepsize == 5000 and d.max_iter == 60000 and d.weight_decay == 0.0
    assert d.test_iter == 10 and d.test_interval == 1000 and d.batch_size == 100
    assert d.snapshot_prefix == "examples/cifar10_full_sigmoid_bn"


def test_generated_cifar10_full_bn_gives_the_same_layout(cos, tmp_path):
    from caffeonspark_b200 import nets
    ref = cos.parse_solver(_memory_data_copy(tmp_path))
    d = cos.parse_solver(nets.write_prototxts("cifar10_full_bn", str(tmp_path)))
    counts, lm, dm, names = nets.layout("cifar10_full_bn")
    assert d.counts == ref.counts == counts and sum(counts) == nets.STATS_NET_PARAM_COUNT["cifar10_full_bn"]
    assert d.lr_mult == ref.lr_mult == lm and d.decay_mult == ref.decay_mult == dm
    assert names[1:4] == ["bn1.mean", "bn1.variance", "bn1.scale"]
    s = nets.NETS["cifar10_full_bn"]["solver"]
    for k in ("lr_policy", "max_iter", "stepsize", "test_iter", "test_interval"):
        assert getattr(d, k) == getattr(ref, k) == s[k], k
    assert d.base_lr == ref.base_lr and d.momentum == ref.momentum and d.gamma == ref.gamma
    desc = nets.solver_desc("cifar10_full_bn")
    assert desc.counts == counts and desc.batch_size == 100


def test_batch_norm_on_a_one_axis_bottom_has_one_channel(cos, tmp_path):
    solver = tmp_path / "s.prototxt"
    solver.write_text('base_lr: 0.1 lr_policy: "fixed" net_param { input: "v" input_shape { dim: 7 } '
                      'layer { name: "bn" type: "BatchNorm" bottom: "v" top: "v" } '
                      'layer { name: "ip" type: "InnerProduct" bottom: "v" top: "o" inner_product_param '
                      '{ num_output: 2 axis: 0 } } }')
    d = cos.parse_solver(str(solver))
    assert d.counts == [1, 1, 1, 14, 2] and d.lr_mult[:3] == [1.0] * 3  # ParamSpec defaults: lr_mult 1


def test_lstm_is_still_not_understood(cos, tmp_path):
    solver = tmp_path / "s.prototxt"
    solver.write_text('base_lr: 0.1 lr_policy: "fixed" net_param { input: "v" input_shape { dim: 2 dim: 3 } '
                      'layer { name: "l" type: "LSTM" bottom: "v" top: "o" } }')
    with pytest.raises(cos.CosError, match="of type 'LSTM' is not understood by the layout parser"):
        cos.parse_solver(str(solver))


def test_torch_module_registers_the_three_blobs_in_layout_order():
    from caffeonspark_b200 import layers, nets
    mod = nets.torch_module("cifar10_full_bn")
    counts, _, _, _ = nets.layout("cifar10_full_bn")
    assert [p.numel() for p in mod.parameters()] == counts
    kinds = [type(m).__name__ for m in mod]
    assert kinds == ["Conv2d", "MaxPool2d", "BatchNorm", "Sigmoid", "Conv2d", "BatchNorm", "Sigmoid", "AvgPool2d",
                     "Conv2d", "BatchNorm", "Sigmoid", "AvgPool2d", "Flatten", "Linear"]
    bn = [m for m in mod if isinstance(m, layers.BatchNorm)]
    assert all(not p.requires_grad for m in bn for p in m.parameters())
    for m in bn:
        for p in m.parameters():
            p.data.fill_(3.0)
        m.reset_parameters()
        assert all(float(p.abs().sum()) == 0.0 for p in m.parameters())


def test_cpu_forward_backward_trains_only_the_conv_and_ip_blobs():
    import torch
    from caffeonspark_b200 import nets
    mod = nets.torch_module("cifar10_full_bn")
    x = torch.rand(4, 3, 32, 32)
    torch.nn.CrossEntropyLoss()(mod(x), torch.tensor([1, 3, 0, 9])).backward()
    grads = [p.grad is not None for p in mod.parameters()]
    assert grads == [True, False, False, False] * 3 + [True, True]
    assert float(mod[2].scale_factor) == 1.0 and mod[2].mean.abs().sum() > 0


# ------------------------------------------------------------------ numpy restatement of batch_norm_layer.cpp

def numpy_bn_forward(x, mean_b, var_b, s, f=0.999, eps=1e-5, global_stats=False):
    """float64 restatement -> (y, mean, var, (mean_b', var_b', s'))"""
    n, c = x.shape[0], x.shape[1]
    xf = x.reshape(n, c, -1).astype(np.float64)
    if global_stats:
        sf = 0.0 if s == 0 else 1.0 / s
        mean, var = sf * mean_b, sf * var_b
        blobs = (mean_b, var_b, s)
    else:
        m = xf.shape[0] * xf.shape[2]
        mean = xf.mean((0, 2))
        var = ((xf - mean[None, :, None]) ** 2).mean((0, 2))
        corr = m / (m - 1) if m > 1 else 1.0
        blobs = (mean + f * mean_b, corr * var + f * var_b, s * f + 1)
    sd = np.sqrt(var + eps)
    y = (xf - mean[None, :, None]) / sd[None, :, None]
    return y.reshape(x.shape), mean, var, blobs


def numpy_bn_backward(x, dy, mean, var, eps=1e-5, global_stats=False):
    n, c = x.shape[0], x.shape[1]
    xf, g = x.reshape(n, c, -1).astype(np.float64), dy.reshape(n, c, -1).astype(np.float64)
    sd = np.sqrt(var + eps)[None, :, None]
    if global_stats:
        return (g / sd).reshape(x.shape)
    xh = (xf - mean[None, :, None]) / sd
    m = xf.shape[0] * xf.shape[2]
    s1, s2 = g.sum((0, 2))[None, :, None], (g * xh).sum((0, 2))[None, :, None]
    return ((g - s1 / m - xh * s2 / m) / sd).reshape(x.shape)


@pytest.mark.parametrize("global_stats", [False, True])
@pytest.mark.parametrize("shape", [(4, 3, 5, 7), (1, 2, 3, 3), (6, 1, 1, 1), (5, 4), (3, 2, 1, 1)])
def test_cpu_composition_matches_the_numpy_restatement(shape, global_stats):
    import torch
    from caffeonspark_b200 import layers
    rng = np.random.RandomState(sum(shape))
    x = (rng.randn(*shape) * 2 + 0.5).astype(np.float32)
    dy = rng.randn(*shape).astype(np.float32)
    c = shape[1]
    mean_b, var_b = rng.rand(c).astype(np.float32), rng.rand(c).astype(np.float32) + 0.5
    s = np.float32(3.0 if global_stats else 2.0)
    bn = layers.BatchNorm(c, use_global_stats=global_stats)
    with torch.no_grad():
        bn.mean.copy_(torch.from_numpy(mean_b))
        bn.variance.copy_(torch.from_numpy(var_b))
        bn.scale_factor.fill_(float(s))
    xt = torch.from_numpy(x).requires_grad_(True)
    y = bn(xt)
    y.backward(torch.from_numpy(dy))
    wy, mean, var, blobs = numpy_bn_forward(x, mean_b.astype(np.float64), var_b.astype(np.float64), float(s),
                                            global_stats=global_stats)
    np.testing.assert_allclose(y.detach().numpy(), wy, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(bn.mean.numpy(), blobs[0], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(bn.variance.numpy(), blobs[1], rtol=1e-5, atol=1e-6)
    assert float(bn.scale_factor) == pytest.approx(blobs[2], rel=1e-7)
    wdx = numpy_bn_backward(x, dy, mean, var, global_stats=global_stats)
    np.testing.assert_allclose(xt.grad.numpy(), wdx, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------ C entry points

def _ptrs(k):
    return [ctypes.c_void_p(0x1000 + 0x100 * i) for i in range(k)]  # distinct: no tensor aliases another


def _fwd(L, suffix="", n=2, c=3, h=4, w=5, eps=1e-5, frac=0.999, null=None):
    args = _ptrs(7)
    if null is not None:
        args[null] = None
    return getattr(L, "cos_batch_norm_forward" + suffix)(*args, n, c, h, w, 0, frac, eps, None)


def _bwd(L, suffix="", n=2, c=3, h=4, w=5, eps=1e-5, null=None):
    args = _ptrs(5)
    if null is not None:
        args[null] = None
    return getattr(L, "cos_batch_norm_backward" + suffix)(*args, n, c, h, w, 0, eps, None)


def test_batch_norm_symbols_are_exported(cos):
    from caffeonspark_b200 import _lib
    names = {s[0] for s in _lib.SYMBOLS}
    for s in ("cos_batch_norm_forward", "cos_batch_norm_backward", "cos_batch_norm_forward_bf16",
              "cos_batch_norm_backward_bf16"):
        assert s in names and getattr(_lib.lib(), s)


@pytest.mark.parametrize("suffix", ["", "_bf16"])
def test_batch_norm_checks_its_arguments(cos, suffix):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for kw in (dict(n=0), dict(c=0), dict(h=0), dict(w=-1), dict(h=1 << 16, w=1 << 15)):
        assert _fwd(L, suffix, **kw) == 0 and b"bad shape" in L.cos_last_error(), kw
        assert _bwd(L, suffix, **kw) == 0 and b"bad shape" in L.cos_last_error(), kw
    for i in range(7):
        assert _fwd(L, suffix, null=i) == 0 and b"NULL" in L.cos_last_error()
    for i in range(5):
        assert _bwd(L, suffix, null=i) == 0 and b"NULL" in L.cos_last_error()
    assert _fwd(L, suffix, eps=-1.0) == 0 and b"eps" in L.cos_last_error()
    assert _bwd(L, suffix, eps=float("nan")) == 0 and b"eps" in L.cos_last_error()
    assert _fwd(L, suffix, frac=float("inf")) == 0 and b"moving_average_fraction" in L.cos_last_error()
    other = ctypes.c_void_p(0x2000)
    # in place: y aliases x; dx aliases x or dy
    assert getattr(L, "cos_batch_norm_forward" + suffix)(P, P, other, other, other, other, other, 2, 3, 4, 5, 0,
                                                         0.999, 1e-5, None) == 0
    assert b"in place" in L.cos_last_error()
    for x, dy, dx in ((P, other, P), (other, P, P)):
        assert getattr(L, "cos_batch_norm_backward" + suffix)(x, dy, dx, other, other, 2, 3, 4, 5, 0, 1e-5,
                                                              None) == 0
        assert b"in place" in L.cos_last_error()


def test_caffemodel_of_the_bn_layout_parses_with_real_protobuf(cos, pb, tmp_path):  # noqa: F811
    """The cifar10_full_bn layout written as a .caffemodel (the blob shapes Caffe's BatchNorm gives its blobs)
    parses with the real protobuf runtime into bn1..bn3 layers of three blobs [C], [C], [1]."""
    from caffeonspark_b200 import _lib, nets
    L = _lib.lib()
    counts, _, _, names = nets.layout("cifar10_full_bn")
    shapes = {"conv1.w": (32, 3, 5, 5), "conv2.w": (32, 32, 5, 5), "conv3.w": (64, 32, 5, 5), "ip1.w": (10, 1024),
              "ip1.b": (10,)}
    arrays, layers, types = [], [], []
    for n, c in zip(names, counts):
        layer, blob = n.split(".")
        shape = shapes.get(n, (c,))
        arrays.append(np.arange(c, dtype=np.float32).reshape(shape))
        layers.append(layer)
        types.append("BatchNorm" if layer.startswith("bn") else "Convolution" if layer.startswith("conv")
                     else "InnerProduct")
    ptrs, nd, dims = _c_blobs(arrays)
    path = str(tmp_path / "bn.caffemodel")
    assert L.cos_caffemodel_write(path.encode(), b"cifar10_full_bn", len(arrays), _strs(layers), _strs(types), nd,
                                  dims, ptrs), L.cos_last_error()
    net = pb["NetParameter"]()
    net.ParseFromString(open(path, "rb").read())
    got = {l.name: l for l in net.layer}
    assert [l.name for l in net.layer] == ["conv1", "bn1", "conv2", "bn2", "conv3", "bn3", "ip1"]
    for name, c in (("bn1", 32), ("bn2", 32), ("bn3", 64)):
        assert got[name].type == "BatchNorm" and len(got[name].blobs) == 3
        assert [list(b.shape.dim) for b in got[name].blobs] == [[c], [c], [1]]


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
@pytest.mark.parametrize("suffix", ["", "_bf16"])
def test_batch_norm_fails_loudly_without_a_gpu(cos, suffix):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for call in (_fwd, _bwd):
        assert call(L, suffix) == 0
        assert b"no CPU path" in L.cos_last_error()


def test_batch_norm_function_refuses_cpu_tensors():
    import torch
    from caffeonspark_b200 import layers
    from caffeonspark_b200.caffenet import CosError
    z = torch.zeros(3)
    with pytest.raises(CosError, match="no CPU path"):
        layers.BatchNormFunction.apply(torch.zeros(2, 3, 4, 4), z, z, torch.zeros(1), False, 0.999, 1e-5)
