"""GPU tests of the native LRN and bias + ReLU + MAX-pool kernels (fp32) against the independent references of
tests/layer_ref.py, across the geometries the C entry points accept.

* Pool: y, index and dx bit for bit against pool_ref; dbias within gamma_d * sum |routed dy|, gamma_d = d u / (1 - d u),
  d the summation depth of the kernels for the shape (pool_dbias_depth).  Every kernel 1..15 with every stride
  1..kernel+2, the CaffeNet b256 shapes, the backward's block-size thresholds, more than 65,535 planes, C > 128, and
  ties, all-negative windows, -0.0, NaN and +-Inf.
* LRN: per element against the float64 reference, |y - y64| <= c u |y64| + 2^-149 and the backward's two-term
  bound (layer_ref.lrn_forward_bound / lrn_backward_bound), for every local_size, several k and beta, channel
  counts on the 16-channel chunk boundaries and pixel counts on the 128-thread block boundaries; subnormal inputs
  (no flush to zero); the NaN / Inf classes of fp32 F.local_response_norm.  Mutated references fall outside the
  bounds on most elements, so the bounds can fail.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import torch.nn.functional as F  # noqa: E402

from caffeonspark_b200 import layers  # noqa: E402
from layer_ref import (LRN_BETAS, LRN_KS, LRN_SIZES, MUTATIONS, NO_GRAD, POOL_GEOMETRIES,  # noqa: E402
                       POOL_VALUE_KINDS, U, lrn_backward_bound, lrn_backward_ref, lrn_forward_bound, lrn_inputs,
                       lrn_ref, mutated_lrn_refs, outside_fraction, pool_inputs, pool_plane_sizes, pool_ref,
                       pooled_size, value_class)
from test_gpu_bf16_layers import _pool_forward_raw  # noqa: E402
from test_gpu_layers import POOL_CASES  # noqa: E402


def f32(v):
    return float(np.float32(v))


def _host(t):
    return t.detach().cpu().numpy()


def _same_bits(a, b):
    """elementwise: the same fp32 bit pattern, or both NaN (the GPU's NaN results carry no payload)"""
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


def _first(mask, *arrays):
    i = tuple(int(v) for v in np.argwhere(mask)[0])
    return f"{int(mask.sum())} of {mask.size} elements, first at {i}: " + ", ".join(
        repr(a[i].item()) for a in arrays)


# ---------------------------------------------------------------- bias + ReLU + MAX pool


def pool_dbias_depth(n, h, w, kernel, stride):
    """The most fp32 additions any routed dy passes through on its way into dbias: the windows that can route to
    one element, the per-thread strided sum over the plane, 5 shuffle levels, the warp sums of a block, the sum
    over n (pool_backward_kernel, bias_grad_kernel)."""
    hw = h * w
    block = 256 if hw >= 256 else (hw + 31) // 32 * 32
    nw = -(-kernel // stride)
    return nw * nw + -(-hw // block) + 5 + block // 32 + n


def check_pool(x, b, k, s, what, dy_seed=12):
    n, c, h, w = x.shape
    ph, pw = pooled_size(h, k, s), pooled_size(w, k, s)
    dy = np.random.default_rng(dy_seed).standard_normal((n, c, ph, pw), dtype=np.float32)
    xt, bt, dyt = (torch.from_numpy(a).cuda() for a in (x, b, dy))
    y_raw, index = _pool_forward_raw(xt, bt, k, s)
    xg, bg = xt.clone().requires_grad_(), bt.clone().requires_grad_()
    y = layers.BiasReluMaxPoolFunction.apply(xg, bg, k, s)
    y.backward(dyt)
    y, y_raw, index, dx, db = (_host(t) for t in (y, y_raw, index, xg.grad, bg.grad))
    ref = pool_ref(x, b, k, s, dy)
    assert np.array_equal(y_raw.view(np.int32), y.view(np.int32)), f"{what}: y of the raw entry point"
    bad = ~_same_bits(y, ref.y)
    assert not bad.any(), f"{what}: y differs in " + _first(bad, y, ref.y)
    bad = index != ref.index
    assert not bad.any(), f"{what}: index differs in " + _first(bad, index, ref.index)
    bad = dx.view(np.int32) != ref.dx.view(np.int32)
    assert not bad.any(), f"{what}: dx differs in " + _first(bad, dx, ref.dx)
    d = pool_dbias_depth(n, h, w, k, s)
    bound = d * U / (1 - d * U) * ref.dbias_abs
    bad = ~(np.abs(db.astype(np.float64) - ref.dbias) <= bound)
    assert not bad.any(), f"{what}: dbias outside gamma_{d} in " + _first(bad, db, ref.dbias, bound)
    return ref


@pytest.mark.parametrize("k,s", POOL_GEOMETRIES)
def test_pool_every_geometry(k, s):
    for j, (h, w) in enumerate(pool_plane_sizes(k, s)):
        x, b = pool_inputs("randn", (2, 3, h, w), seed=k * 100 + s * 10 + j)
        check_pool(x, b, k, s, f"kernel {k} stride {s} plane {h}x{w}")


@pytest.mark.parametrize("case", [c for c in POOL_CASES if c.endswith("_b256")])
def test_pool_caffenet_b256(case):
    shape, k, s = POOL_CASES[case]
    x, b = pool_inputs("randn", shape, seed=3)
    check_pool(x, b, k, s, case)


# (N, C, H, W), kernel, stride: the pool backward's block is 32 up to H*W = 32, 64 at 33, 256 from 255 (one strided
# pass) and 257 (two); more than 65,535 planes; bias_grad_kernel over more than one 128-channel block
POOL_EDGES = {
    "hw31_k1s1": ((2, 3, 31, 1), 1, 1),
    "hw31_k1s2": ((2, 3, 1, 31), 1, 2),
    "hw32_k3s2": ((2, 3, 4, 8), 3, 2),
    "hw32_k2s1": ((2, 3, 8, 4), 2, 1),
    "hw33_k3s2": ((2, 3, 3, 11), 3, 2),
    "hw33_k3s1": ((2, 3, 11, 3), 3, 1),
    "hw255_k3s2": ((2, 3, 15, 17), 3, 2),
    "hw255_k4s3": ((2, 3, 17, 15), 4, 3),
    "hw256_k3s2": ((2, 3, 16, 16), 3, 2),
    "hw256_k5s2": ((2, 3, 16, 16), 5, 2),
    "hw257_k1s1": ((2, 3, 257, 1), 1, 1),
    "hw257_k1s3": ((2, 3, 1, 257), 1, 3),
    "hw3025_k5s1": ((2, 3, 55, 55), 5, 1),
    "planes65792_k3s2": ((257, 256, 3, 3), 3, 2),
    "planes65792_k2s1": ((257, 256, 3, 3), 2, 1),
    "c257_k3s2": ((2, 257, 5, 5), 3, 2),
    "c257_k2s1": ((3, 257, 4, 6), 2, 1),
}


@pytest.mark.parametrize("case", list(POOL_EDGES))
def test_pool_shape_edges(case):
    shape, k, s = POOL_EDGES[case]
    x, b = pool_inputs("randn", shape, seed=5)
    check_pool(x, b, k, s, case)


@pytest.mark.parametrize("kind", POOL_VALUE_KINDS)
@pytest.mark.parametrize("k,s", [(3, 2), (3, 1), (2, 2), (5, 3), (1, 1), (2, 3)])
def test_pool_special_values(kind, k, s):
    x, b = pool_inputs(kind, (2, 4, 11, 13), seed=7)
    ref = check_pool(x, b, k, s, f"{kind}, kernel {k} stride {s}")
    if kind == "negative_zero":  # -0.0 + -0.0 passes no gradient and pools to +0.0
        assert np.all(ref.index == NO_GRAD) and np.all(ref.y.view(np.int32) == 0)
    if kind == "bias_ties":  # the test has teeth only if fl32(x + b) ties where x does not
        x_first = pool_ref(x, np.zeros_like(b), k, s).index
        assert np.mean(x_first != ref.index) > 0.1


# ---------------------------------------------------------------- LRN


def _lrn_native(x, dy, size, alpha, beta, k):
    xt = torch.from_numpy(x).cuda().requires_grad_()
    y = layers.LRNFunction.apply(xt, size, alpha, beta, k)
    y.backward(torch.from_numpy(dy).cuda())
    return _host(y), _host(xt.grad)


def check_lrn(x, dy, size, alpha, beta, k, what, chunk=32):
    """-> the kernels' (y, dx), checked against the float64 reference within the bounds (the parameters are the
    fp32 values the entry points receive); the reference runs over chunk images at a time"""
    alpha, beta, k = f32(alpha), f32(beta), f32(k)
    y, dx = _lrn_native(x, dy, size, alpha, beta, k)
    for i in range(0, x.shape[0], chunk):
        sl = slice(i, i + chunk)
        y64, mag = lrn_ref(x[sl], size, alpha, beta, k)
        bound = lrn_forward_bound(mag, size, beta)
        bad = ~(np.abs(y[sl] - y64) <= bound)
        assert not bad.any(), f"{what}: y outside the bound in " + _first(bad, y[sl], y64, bound)
        dx64, ma, mb = lrn_backward_ref(x[sl], dy[sl], size, alpha, beta, k)
        bound = lrn_backward_bound(ma, mb, size, beta)
        bad = ~(np.abs(dx[sl] - dx64) <= bound)
        assert not bad.any(), f"{what}: dx outside the bound in " + _first(bad, dx[sl], dx64, bound)
    return y, dx


LRN_CHANNELS = [1, 2, 7, 15, 16, 17, 31, 32, 33, 96, 257]


@pytest.mark.parametrize("channels", LRN_CHANNELS)
@pytest.mark.parametrize("size", LRN_SIZES)
def test_lrn_every_local_size_and_channel_count(size, channels):
    x, dy = lrn_inputs((1, channels, 3, 43), 1e-4, 2.0, seed=size * 1000 + channels)  # 129 pixels
    check_lrn(x, dy, size, 1e-4, 0.75, 2.0, f"size {size}, C {channels}")


@pytest.mark.parametrize("beta", LRN_BETAS)
@pytest.mark.parametrize("k", LRN_KS)
def test_lrn_k_and_beta(k, beta):
    x, dy = lrn_inputs((2, 33, 5, 13), 1e-4, k, seed=[LRN_KS.index(k), LRN_BETAS.index(beta)])
    check_lrn(x, dy, 5, 1e-4, beta, k, f"k {k}, beta {beta}")


# N*H*W = 1, 127, 128, 129 around the 128-pixel thread block
LRN_PIXELS = {"npix1": (1, 17, 1, 1), "npix127": (1, 17, 1, 127), "npix128": (2, 17, 8, 8), "npix129": (3, 17, 1, 43)}


@pytest.mark.parametrize("size", [1, 5, 15])
@pytest.mark.parametrize("case", list(LRN_PIXELS))
def test_lrn_pixel_counts(case, size):
    x, dy = lrn_inputs(LRN_PIXELS[case], 1e-4, 1e-3, seed=size)
    check_lrn(x, dy, size, 1e-4, 0.75, 1e-3, f"{case}, size {size}")


@pytest.mark.parametrize("shape", [(256, 96, 27, 27), (256, 256, 13, 13)], ids=["norm1_b256", "norm2_b256"])
def test_lrn_caffenet_b256(shape):
    x, dy = lrn_inputs(shape, 1e-4, 1.0, seed=9)
    check_lrn(x, dy, 5, 1e-4, 0.75, 1.0, f"CaffeNet {shape}")


@pytest.mark.parametrize("beta", [0.75, 2.0, -0.5])
@pytest.mark.parametrize("k", LRN_KS)
def test_lrn_keeps_subnormal_inputs(k, beta):
    """x of both signs in [2^-140, 2^-127): x^2 underflows, so y = x k^-beta.  A build that flushes subnormals to
    zero returns 0."""
    rng = np.random.default_rng(4)
    shape = (2, 17, 3, 5)
    x = (np.exp2(rng.uniform(-140, -127, shape)) * rng.choice([-1.0, 1.0], shape)).astype(np.float32)
    assert np.all((x != 0) & (np.abs(x) < 2.0 ** -126))
    dy = rng.standard_normal(shape, dtype=np.float32)
    y, _ = check_lrn(x, dy, 5, 1e-4, beta, k, f"subnormal x, k {k}, beta {beta}")
    expect = x.astype(np.float64) * f32(k) ** -f32(beta)
    bound = lrn_forward_bound(np.abs(expect), 5, beta)
    bad = ~(np.abs(y - expect) <= bound)
    assert not bad.any(), "y != x k^-beta in " + _first(bad, x, y, expect)
    assert np.all(y != 0), f"{int((y == 0).sum())} subnormal inputs flushed to zero"


@pytest.mark.parametrize("size", [1, 5, 15])
def test_lrn_non_finite_inputs_match_pytorch_classes(size):
    x, dy = lrn_inputs((2, 19, 4, 5), 1e-4, 1.0, seed=6)
    u = np.random.default_rng(7).random(x.shape)
    x[u < 0.03] = np.nan
    x[u > 0.97] = np.inf
    x[(u > 0.5) & (u < 0.53)] = -np.inf
    for beta in (0.75, 0.5, -0.5, 2.0):
        y, _ = _lrn_native(x, dy, size, f32(1e-4), beta, 1.0)
        yt = F.local_response_norm(torch.from_numpy(x), size, f32(1e-4), beta, 1.0).numpy()
        bad = value_class(y) != value_class(yt)
        assert not bad.any(), f"size {size}, beta {beta}: class differs in " + _first(bad, x, y, yt)


@pytest.mark.parametrize("size,k,beta", [(5, 2.0, 0.75), (3, 1e-3, 0.5), (15, 2.0, 2.0), (7, 1e-3, -0.5)])
def test_lrn_bounds_reject_mutated_references(size, k, beta):
    alpha = f32(1e-4)
    x, dy = lrn_inputs((2, 33, 5, 7), alpha, k, seed=size)
    check_lrn(x, dy, size, alpha, beta, k, f"size {size}, k {k}, beta {beta}")
    for m in MUTATIONS:
        # what a kernel computing the mutated function would return, rounded to fp32, against the true bound
        my, mdx = mutated_lrn_refs(x, dy, size, alpha, f32(beta), f32(k), m)
        fy, fdx = outside_fraction(my.astype(np.float32), mdx.astype(np.float32), x, dy, size, alpha, f32(beta),
                                   f32(k))
        assert fy > 0.5 and fdx > 0.5, f"{m}: only {fy:.2f} of y and {fdx:.2f} of dx outside the bound"
