"""GPU tests of the bf16 producer layers (the *_bf16 entry points through layers.py).

The contract is that a bf16 kernel computes what the fp32 kernel computes on the upcast inputs and rounds each output
element once to bf16 (round to nearest even); index and the fp32 bias gradient are the fp32 kernel's bit for bit.
That is checked at the shapes of test_gpu_layers.py plus LRN windows up to 15.  Against PyTorch's fp32 composition on
the upcast inputs, rounded to bf16: the pool block is bitwise (y, dx), LRN within one bf16 ulp.  Run to run and
CUDA-graph replay are bitwise."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import torch.nn as nn  # noqa: E402

from caffeonspark_b200 import layers  # noqa: E402
from test_gpu_layers import LRN_CASES, POOL_CASES, _lrn_inputs, _pool_inputs, _pool_ref  # noqa: E402

# every window half-width 0..7 has its own kernel instantiation; CaffeNet uses 2, LRN_CASES also 1 and 3
LRN_BF16_CASES = dict(LRN_CASES, size1=((2, 20, 3, 7), 1, 1e-2, 0.75), size9=((2, 40, 6, 6), 9, 1e-3, 0.75),
                      size11=((3, 35, 5, 7), 11, 1e-3, 0.75), size13=((2, 40, 4, 9), 13, 1e-3, 0.6),
                      size15=((2, 33, 4, 5), 15, 1e-3, 0.75))


def _bits(t):
    """float tensors as their bit patterns (so -0.0 and 0.0, or two NaNs, are told apart); others as they are"""
    return {torch.bfloat16: lambda: t.view(torch.int16), torch.float32: lambda: t.view(torch.int32)}.get(
        t.dtype, lambda: t)()


def _assert_bits(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    diff = (_bits(a) != _bits(b)).sum().item()
    assert diff == 0, f"{what}: {diff} elements differ"


def _bf16_pair(t):
    """-> (t rounded to bf16, that bf16 tensor upcast back to fp32)"""
    tb = t.to(torch.bfloat16)
    return tb, tb.float()


def _pool_forward_raw(x, b, k, s):
    """the forward entry point directly, so the index is visible"""
    n, c, h, w = x.shape
    ph, pw = layers.pooled_size(h, k, s), layers.pooled_size(w, k, s)
    y = torch.empty((n, c, ph, pw), dtype=x.dtype, device=x.device)
    index = torch.empty((n, c, ph, pw), dtype=torch.uint8, device=x.device)
    layers._call(layers._entry("cos_bias_relu_maxpool_forward", x.dtype), x.data_ptr(), b.data_ptr(), y.data_ptr(),
                 index.data_ptr(), n, c, h, w, k, s, ph, pw, layers._stream())
    return y, index


def _pool_native(x, b, dy, k, s):
    xn, bn = x.clone().requires_grad_(), b.clone().requires_grad_()
    y = layers.BiasReluMaxPoolFunction.apply(xn, bn, k, s)
    y.backward(dy)
    return y.detach(), xn.grad, bn.grad


def _pool_case(case, ties):
    shape, k, s = POOL_CASES[case]
    x, b = _pool_inputs(shape, 11, ties)
    n, c, h, w = shape
    ph, pw = layers.pooled_size(h, k, s), layers.pooled_size(w, k, s)
    dy = torch.randn((n, c, ph, pw), device="cuda", generator=torch.Generator(device="cuda").manual_seed(12))
    return x, b, dy, k, s


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("case", list(POOL_CASES))
def test_bf16_pool_equals_the_fp32_kernel_rounded(case, ties):
    x, b, dy, k, s = _pool_case(case, ties)
    xb, xu = _bf16_pair(x)
    dyb, dyu = _bf16_pair(dy)
    y32, i32 = _pool_forward_raw(xu, b, k, s)
    yb, ib = _pool_forward_raw(xb, b, k, s)
    _assert_bits(yb, y32.to(torch.bfloat16), f"{case}: y")
    _assert_bits(ib, i32, f"{case}: index")
    _, dx32, db32 = _pool_native(xu, b, dyu, k, s)
    yb2, dxb, dbb = _pool_native(xb, b, dyb, k, s)
    _assert_bits(yb2, yb, f"{case}: y through autograd")
    assert dxb.dtype == torch.bfloat16 and dbb.dtype == torch.float32
    _assert_bits(dxb, dx32.to(torch.bfloat16), f"{case}: dx")
    _assert_bits(dbb, db32, f"{case}: dbias")


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("case", list(POOL_CASES))
def test_bf16_pool_matches_pytorch_on_upcast_inputs(case, ties):
    x, b, dy, k, s = _pool_case(case, ties)
    xb, xu = _bf16_pair(x)
    dyb, dyu = _bf16_pair(dy)
    y, dx, db = _pool_native(xb, b, dyb, k, s)
    for relu_first in (True, False):
        yr, dxr, dbr = _pool_ref(xu, b, dyu, k, s, relu_first)
        _assert_bits(y, yr.to(torch.bfloat16), f"{case}: y")
        _assert_bits(dx, dxr.to(torch.bfloat16), f"{case}: dx")
        routed = (dyu.abs() * (yr > 0)).sum(dim=(0, 2, 3))  # the fp32 layer's dbias tolerance (test_gpu_layers)
        assert torch.all((db - dbr).abs() <= 1e-5 * routed + 1e-30), f"{case}: dbias"


def _lrn_native(x, dy, size, alpha, beta):
    xn = x.clone().requires_grad_()
    y = layers.LRN(size, alpha=alpha, beta=beta, k=1.0)(xn)
    y.backward(dy)
    return y.detach(), xn.grad


@pytest.mark.parametrize("case", list(LRN_BF16_CASES))
def test_bf16_lrn_equals_the_fp32_kernel_rounded(case):
    shape, size, alpha, beta = LRN_BF16_CASES[case]
    x, dy = _lrn_inputs(shape, 21)
    xb, xu = _bf16_pair(x)
    dyb, dyu = _bf16_pair(dy)
    y32, dx32 = _lrn_native(xu, dyu, size, alpha, beta)
    yb, dxb = _lrn_native(xb, dyb, size, alpha, beta)
    _assert_bits(yb, y32.to(torch.bfloat16), f"{case}: y")
    _assert_bits(dxb, dx32.to(torch.bfloat16), f"{case}: dx")


def _ordered(t):
    """bf16 bit patterns mapped to integers in the order of the values they encode (+0 and -0 both to 0)"""
    i = t.view(torch.int16).int()
    return torch.where(i < 0, -(i & 0x7FFF), i)


@pytest.mark.parametrize("case", list(LRN_BF16_CASES))
def test_bf16_lrn_matches_pytorch_within_one_ulp(case):
    shape, size, alpha, beta = LRN_BF16_CASES[case]
    x, dy = _lrn_inputs(shape, 21)
    xb, xu = _bf16_pair(x)
    dyb, dyu = _bf16_pair(dy)
    xr = xu.clone().requires_grad_()
    yr = nn.LocalResponseNorm(size, alpha=alpha, beta=beta, k=1.0)(xr)
    yr.backward(dyu)
    yb, dxb = _lrn_native(xb, dyb, size, alpha, beta)
    ulps = (_ordered(yb) - _ordered(yr.detach().to(torch.bfloat16))).abs()
    assert ulps.max().item() <= 1, f"{case}: y off by {ulps.max().item()} bf16 ulp"
    # dx_c is a difference of two terms: where they cancel, the fp32 kernel's rounding difference from PyTorch
    # (bounded at 1e-5 of max|dx| in test_gpu_layers.py) can exceed an ulp of the small result.  So one bf16 ulp,
    # or that fp32 bound for the elements it covers.
    ref = xr.grad
    ulps = (_ordered(dxb) - _ordered(ref.to(torch.bfloat16))).abs()
    outside = (ulps > 1) & ((dxb.float() - ref).abs() > 1e-5 * ref.abs().max())
    assert not outside.any(), f"{case}: {outside.sum().item()} dx elements beyond one bf16 ulp"


def _both_layers(xp, bp, xl, dyp, dyl):
    xp.grad = bp.grad = xl.grad = None
    y = layers.BiasReluMaxPoolFunction.apply(xp, bp, 3, 2)
    yl = layers.LRNFunction.apply(xl, 5, 1e-4, 0.75, 1.0)
    torch.autograd.backward([y, yl], [dyp, dyl])
    return [y.detach(), xp.grad, bp.grad, yl.detach(), xl.grad]


def test_bf16_layers_are_deterministic_and_graph_capturable():
    shape, k, s = POOL_CASES["caffenet_conv1_b4"]
    x, b = _pool_inputs(shape, 31)
    xp, bp = x.to(torch.bfloat16).requires_grad_(), b.requires_grad_()
    dyp = torch.randn((shape[0], shape[1], 27, 27), device="cuda").to(torch.bfloat16)
    xl, dyl = (t.to(torch.bfloat16) for t in _lrn_inputs((4, 96, 27, 27), 32))
    xl.requires_grad_()
    first = [t.clone() for t in _both_layers(xp, bp, xl, dyp, dyl)]
    assert [t.dtype for t in first] == [torch.bfloat16, torch.bfloat16, torch.float32, torch.bfloat16,
                                        torch.bfloat16]
    second = [t.clone() for t in _both_layers(xp, bp, xl, dyp, dyl)]
    for a, c in zip(first, second):
        _assert_bits(a, c, "run to run")

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
            _assert_bits(a, c.detach(), "graph replay")


def test_bf16_pool_rejects_a_bf16_bias():
    from caffeonspark_b200.caffenet import CosError
    x = torch.randn((2, 3, 9, 9), device="cuda").to(torch.bfloat16)
    with pytest.raises(CosError, match="fp32"):
        layers.BiasReluMaxPoolFunction.apply(x, torch.zeros(3, device="cuda", dtype=torch.bfloat16), 3, 2)
    with pytest.raises(CosError, match="fp32 or bf16"):
        layers.LRNFunction.apply(x.half(), 5, 1e-4, 0.75, 1.0)
