"""The within-channel LRN kernels on the GPU (DESIGN.md section 10): y and dx within the documented error bounds of the
float64 reference for every local_size and plane shapes around the 32 x 8 tile, non-finite and subnormal inputs in the
float64 composition's value classes, bf16 as the fp32 kernel rounded once, and bitwise-repeatable output, eagerly and
under CUDA-graph replay."""
import numpy as np
import pytest
import torch

from lrn_within_ref import (SIZES, backward_bound, composition, forward_bound, lrn_within_backward_ref,
                            lrn_within_ref, value_class)

pytestmark = pytest.mark.gpu

# 1x1, planes smaller than every window, and sizes that are not multiples of the 32 x 8 tile on either axis
SHAPES = [(2, 3, 1, 1), (1, 2, 2, 3), (2, 2, 5, 7), (1, 3, 8, 32), (1, 2, 9, 33), (2, 1, 17, 65), (1, 1, 31, 30)]
HYPER = [(5e-05, 0.75), (1.0, 0.75), (0.3, 2.0), (2.0, -0.5), (0.5, 0.0)]


def _native(x, dy, size, alpha, beta):
    from caffeonspark_b200 import layers
    xt = torch.from_numpy(x).cuda().requires_grad_()
    y = layers.LRN(size, alpha=alpha, beta=beta, region="WITHIN_CHANNEL")(xt)
    y.backward(torch.from_numpy(dy).cuda())
    return y.detach().cpu().numpy(), xt.grad.cpu().numpy()


def _first(bad, *arrays):
    i = np.argwhere(bad)[0]
    return f"{bad.sum()} elements, first at {tuple(i)}: " + ", ".join(f"{a[tuple(i)]!r}" for a in arrays)


def check(x, dy, size, alpha, beta, what):
    y, dx = _native(x, dy, size, alpha, beta)
    y64, mag = lrn_within_ref(x, size, alpha, beta)
    bound = forward_bound(mag, size, beta)
    bad = ~(np.abs(y - y64) <= bound)
    assert not bad.any(), f"{what}: y outside the bound in " + _first(bad, y, y64, bound)
    dx64, ma, mb = lrn_within_backward_ref(x, dy, size, alpha, beta)
    bound = backward_bound(ma, mb, size, beta)
    bad = ~(np.abs(dx - dx64) <= bound)
    assert not bad.any(), f"{what}: dx outside the bound in " + _first(bad, dx, dx64, bound)
    return y, dx


def _inputs(shape, seed, scale=3.0):
    rng = np.random.RandomState(seed)
    return (rng.standard_normal(shape) * scale).astype(np.float32), rng.standard_normal(shape).astype(np.float32)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES)
def test_every_local_size_and_plane_shape(shape, size):
    x, dy = _inputs(shape, size * 7 + shape[2])
    check(x, dy, size, 1.0, 0.75, f"{shape} n={size}")


@pytest.mark.parametrize("alpha,beta", HYPER)
def test_alpha_and_beta(alpha, beta):
    for size in (3, 7):
        x, dy = _inputs((2, 3, 13, 40), size)
        check(x, dy, size, alpha, beta, f"alpha={alpha} beta={beta} n={size}")


@pytest.mark.parametrize("shape", [(100, 32, 16, 16), (100, 32, 8, 8), (4, 16, 128, 200)])
def test_cifar10_full_and_larger_planes(shape):
    x, dy = _inputs(shape, 5, scale=40.0)  # pixel-scale activations: alpha s is far from 0
    check(x, dy, 3, 5e-05, 0.75, f"{shape}")


def test_subnormal_inputs_are_not_flushed():
    rng = np.random.RandomState(3)
    x = (rng.choice([1, -1], (2, 2, 9, 11)) * rng.randint(1, 1 << 20, (2, 2, 9, 11)) * 2.0 ** -149).astype(np.float32)
    assert (x != 0).all() and (np.abs(x) < np.finfo(np.float32).tiny).all()
    dy = np.ones_like(x)
    y, dx = check(x, dy, 5, 1.0, 0.75, "subnormal x")
    assert (y == x).all() and (dx == x * 0 + 1).all()  # s rounds to 1: y = x and dx = dy, bit for bit


@pytest.mark.parametrize("size", [1, 3, 5, 15])
def test_non_finite_inputs_give_the_float64_value_classes(size):
    rng = np.random.RandomState(size)
    x, dy = _inputs((2, 3, 12, 37), size + 1)
    specials = np.array([np.nan, np.inf, -np.inf, 2.0 ** -140, -(2.0 ** -149), 0.0, -0.0, 1e15], np.float32)
    mask = rng.rand(*x.shape) < 0.04
    x[mask] = rng.choice(specials, mask.sum())
    dy[rng.rand(*x.shape) < 0.02] = np.nan
    y, dx = _native(x, dy, size, 0.5, 0.75)
    want = composition(x, size, 0.5, 0.75)
    assert (value_class(y) == value_class(want)).all(), _first(value_class(y) != value_class(want), y, want, x)
    dx64 = lrn_within_backward_ref(x, dy, size, 0.5, 0.75)[0]
    assert (value_class(dx) == value_class(dx64)).all(), _first(value_class(dx) != value_class(dx64), dx, dx64)
    assert (value_class(y) != 0).any() and (value_class(dx) != 0).any()


@pytest.mark.parametrize("size", [1, 3, 9, 15])
@pytest.mark.parametrize("shape", [(2, 3, 1, 1), (2, 3, 9, 33), (100, 32, 16, 16)])
def test_bf16_is_the_fp32_kernel_rounded_once(shape, size):
    from caffeonspark_b200 import layers
    x, dy = _inputs(shape, size)
    xb, dyb = torch.from_numpy(x).cuda().bfloat16(), torch.from_numpy(dy).cuda().bfloat16()
    lrn = layers.LRN(size, alpha=0.5, beta=0.75, region="WITHIN_CHANNEL")
    xt, xf = xb.clone().requires_grad_(), xb.float().requires_grad_()
    yb, yf = lrn(xt), lrn(xf)
    yb.backward(dyb)
    yf.backward(dyb.float())
    assert yb.dtype == xt.grad.dtype == torch.bfloat16
    assert torch.equal(yb.view(torch.int16), yf.bfloat16().view(torch.int16))
    assert torch.equal(xt.grad.view(torch.int16), xf.grad.bfloat16().view(torch.int16))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bitwise_repeatable_and_graph_capturable(dtype):
    from caffeonspark_b200 import layers
    x, dy = _inputs((100, 32, 16, 16), 9, scale=40.0)
    xs, dys = torch.from_numpy(x).cuda().to(dtype), torch.from_numpy(dy).cuda().to(dtype)
    xt = xs.detach().requires_grad_()

    def run():
        y = layers.LRNWithinFunction.apply(xt, 3, 5e-05, 0.75)
        (dx,) = torch.autograd.grad([y], [xt], [dys])
        return y.detach(), dx

    eager = [tuple(t.clone() for t in run()) for _ in range(2)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        run()  # warm up on the capture stream
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = run()
    replays = []
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        replays.append(tuple(t.clone() for t in out))
    bits = torch.int32 if dtype == torch.float32 else torch.int16
    for a, b in [(eager[0], eager[1]), (eager[0], replays[0]), (eager[0], replays[1])]:
        for u, v in zip(a, b):
            assert torch.equal(u.view(bits), v.view(bits))
