"""GPU tests of the native producer layers (csrc/caffe_layers.cu through layers.py) against PyTorch's fp32 ops on
the same inputs: the fused conv-bias + ReLU + MAX-pool block bit for bit (y, dx) and to 1e-5 (dbias), the LRN to
1e-6 (forward) / 1e-5 (backward) of the reference's largest magnitude; run to run and CUDA-graph replay bitwise."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from caffeonspark_b200 import layers  # noqa: E402
from caffeonspark_b200.caffenet import CosError  # noqa: E402

# (N, C, H, W) of the bias-free conv output, pool kernel, stride
POOL_CASES = {
    "caffenet_conv1_b256": ((256, 96, 55, 55), 3, 2),
    "caffenet_conv2_b256": ((256, 256, 27, 27), 3, 2),
    "caffenet_conv5_b256": ((256, 256, 13, 13), 3, 2),
    "caffenet_conv1_b4": ((4, 96, 55, 55), 3, 2),
    "caffenet_conv2_b4": ((4, 256, 27, 27), 3, 2),
    "caffenet_conv5_b4": ((4, 256, 13, 13), 3, 2),
    "cifar10_quick_conv1": ((100, 32, 32, 32), 3, 2),  # 32 -> 16: the last window is clipped
    "ragged": ((3, 3, 17, 23), 3, 2),
    "ragged_k2": ((2, 3, 9, 7), 2, 2),
    # the runtime-geometry kernels: overlapping windows (kernel > stride), stride > kernel, kernel 1, kernel 15
    "k1s1": ((2, 3, 5, 6), 1, 1),
    "k1s2": ((2, 3, 7, 6), 1, 2),
    "k2s1": ((2, 3, 9, 7), 2, 1),
    "k3s1": ((2, 3, 9, 10), 3, 1),
    "k4s3": ((2, 3, 10, 11), 4, 3),
    "k5s3_clipped": ((2, 3, 13, 12), 5, 3),
    "k7s2": ((2, 3, 15, 16), 7, 2),
    "k2s3_gaps": ((2, 3, 9, 8), 2, 3),
    "k15s1": ((1, 2, 17, 16), 15, 1),
    "k15s17": ((1, 2, 33, 40), 15, 17),
    # H*W = 33 and 257 (the backward's block sizes 64 and 256 with two strided passes), N*C > 65535, C > 128
    "hw33": ((2, 3, 3, 11), 3, 2),
    "hw257": ((2, 3, 257, 1), 1, 1),
    "planes65792": ((257, 256, 3, 3), 3, 2),
    "c257_k2s1": ((2, 257, 5, 5), 2, 1),
}
# (N, C, H, W), local_size, alpha, beta, k: every window half-width 0..7 has its own kernel instantiation
LRN_CASES = {
    "caffenet_norm1_b256": ((256, 96, 27, 27), 5, 1e-4, 0.75, 1.0),
    "caffenet_norm2_b256": ((256, 256, 13, 13), 5, 1e-4, 0.75, 1.0),
    "caffenet_norm1_b4": ((4, 96, 27, 27), 5, 1e-4, 0.75, 1.0),
    "caffenet_norm2_b4": ((4, 256, 13, 13), 5, 1e-4, 0.75, 1.0),
    "ragged": ((3, 3, 7, 9), 5, 1e-4, 0.75, 1.0),
    "ragged_size3_strong": ((2, 37, 5, 11), 3, 5e-2, 0.75, 1.0),
    "size7": ((2, 40, 6, 6), 7, 1e-3, 0.5, 1.0),
    "size1": ((2, 20, 3, 7), 1, 1e-2, 0.75, 1.0),
    "size9": ((2, 40, 6, 6), 9, 1e-3, 0.75, 1.0),
    "size11": ((3, 35, 5, 7), 11, 1e-3, 0.75, 1.0),
    "size13": ((2, 40, 4, 9), 13, 1e-3, 0.6, 1.0),
    "size15": ((2, 33, 4, 5), 15, 1e-3, 0.75, 1.0),
    "k2": ((2, 33, 5, 7), 5, 1e-4, 0.75, 2.0),
    "k1e-3_size3": ((2, 17, 3, 43), 3, 1e-4, 0.75, 1e-3),
    "size15_k2": ((1, 16, 8, 16), 15, 1e-3, 0.5, 2.0),
    "size7_k1e-3": ((3, 31, 1, 43), 7, 1e-3, 1.0, 1e-3),
}


def _pool_inputs(shape, seed, ties=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    if ties:  # many equal values and exact zeros: exercises first-maximum-wins and the <= 0 cut
        x = torch.round(x * 2)
    b = torch.randn(shape[1], device="cuda", generator=g) * (0.0 if ties else 0.3)
    return x, b


def _pool_ref(x, b, dy, k, s, relu_first=True):
    xr, br = x.clone().requires_grad_(), b.clone().requires_grad_()
    z = xr + br.view(1, -1, 1, 1)
    y = F.max_pool2d(F.relu(z), k, s, ceil_mode=True) if relu_first else F.relu(F.max_pool2d(z, k, s, ceil_mode=True))
    y.backward(dy)
    return y.detach(), xr.grad, br.grad


def _pool_native(x, b, dy, k, s):
    xn, bn = x.clone().requires_grad_(), b.clone().requires_grad_()
    y = layers.BiasReluMaxPoolFunction.apply(xn, bn, k, s)
    y.backward(dy)
    return y.detach(), xn.grad, bn.grad


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("case", list(POOL_CASES))
def test_bias_relu_maxpool_matches_pytorch_bitwise(case, ties):
    shape, k, s = POOL_CASES[case]
    x, b = _pool_inputs(shape, 11, ties)
    n, c, h, w = shape
    ph, pw = layers.pooled_size(h, k, s), layers.pooled_size(w, k, s)
    dy = torch.randn((n, c, ph, pw), device="cuda", generator=torch.Generator(device="cuda").manual_seed(12))
    y, dx, db = _pool_native(x, b, dy, k, s)
    for relu_first in (True, False):  # conv -> relu -> pool (CaffeNet) and conv -> pool -> relu (CIFAR-10-quick)
        yr, dxr, dbr = _pool_ref(x, b, dy, k, s, relu_first)
        assert y.shape == yr.shape
        assert torch.equal(y, yr), f"{case}: y differs in {(y != yr).sum().item()} elements"
        assert torch.equal(dx, dxr), f"{case}: dx differs in {(dx != dxr).sum().item()} elements"
        routed = (dy.abs() * (yr > 0)).sum(dim=(0, 2, 3))
        assert torch.all((db - dbr).abs() <= 1e-5 * routed + 1e-30), f"{case}: dbias"


def _lrn_inputs(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.relu(torch.randn(shape, device="cuda", generator=g)) * 30  # post-ReLU/pool magnitudes: s well above k
    dy = torch.randn(shape, device="cuda", generator=g)
    return x, dy


def _rel(a, ref):
    return ((a - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("case", list(LRN_CASES))
def test_lrn_matches_pytorch(case):
    shape, size, alpha, beta, k = LRN_CASES[case]
    x, dy = _lrn_inputs(shape, 21)
    xr = x.clone().requires_grad_()
    yr = nn.LocalResponseNorm(size, alpha=alpha, beta=beta, k=k)(xr)
    yr.backward(dy)
    xn = x.clone().requires_grad_()
    y = layers.LRN(size, alpha=alpha, beta=beta, k=k)(xn)
    y.backward(dy)
    assert _rel(y, yr.detach()) <= 1e-6, case
    assert _rel(xn.grad, xr.grad) <= 1e-5, case


def test_lrn_rejects_an_even_local_size():
    x = torch.rand((2, 8, 3, 3), device="cuda")
    with pytest.raises(ValueError, match="odd"):
        layers.LRN(4)
    with pytest.raises(CosError, match="odd"):
        layers.LRNFunction.apply(x, 4, 1e-4, 0.75, 1.0)


def _both_layers(xp, bp, xl, dyp, dyl):
    """forward + backward of conv1's pool block and norm1 on static buffers -> (y, dx, db, y_lrn, dx_lrn)"""
    xp.grad = bp.grad = xl.grad = None
    y = layers.BiasReluMaxPoolFunction.apply(xp, bp, 3, 2)
    yl = layers.LRNFunction.apply(xl, 5, 1e-4, 0.75, 1.0)
    torch.autograd.backward([y, yl], [dyp, dyl])
    return [y.detach(), xp.grad, bp.grad, yl.detach(), xl.grad]


def test_layers_are_deterministic_and_graph_capturable():
    shape, k, s = POOL_CASES["caffenet_conv1_b4"]
    x, b = _pool_inputs(shape, 31)
    xp, bp = x.requires_grad_(), b.requires_grad_()
    dyp = torch.randn((shape[0], shape[1], 27, 27), device="cuda")
    xl, dyl = _lrn_inputs((4, 96, 27, 27), 32)
    xl.requires_grad_()
    first = [t.clone() for t in _both_layers(xp, bp, xl, dyp, dyl)]
    second = [t.clone() for t in _both_layers(xp, bp, xl, dyp, dyl)]
    for a, c in zip(first, second):
        assert torch.equal(a, c)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _both_layers(xp, bp, xl, dyp, dyl)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    xp.grad = bp.grad = xl.grad = None
    with torch.cuda.graph(g):
        y = layers.BiasReluMaxPoolFunction.apply(xp, bp, 3, 2)
        yl = layers.LRNFunction.apply(xl, 5, 1e-4, 0.75, 1.0)
        gx, gb, gl = torch.autograd.grad([y, yl], [xp, bp, xl], [dyp, dyl])
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for a, c in zip(first, [y, gx, gb, yl, gl]):
            assert torch.equal(a, c.detach())
