"""CPU checks of tests/layer_ref.py against PyTorch, so that a reference bug never shows up as a kernel failure:
lrn_ref / lrn_backward_ref against F.local_response_norm and its autograd in float64 to 1e-12; pool_ref's y, index
and dx bit for bit against F.max_pool2d(F.relu(x + b), k, s, ceil_mode=True) and its autograd over every geometry
the GPU tests run.  An fp32 evaluation in the LRN kernels' operation order falls inside the stated error bounds, and
the mutated references the GPU tests use to show those bounds can fail fall outside them."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.nn.functional as F  # noqa: E402

from layer_ref import (LRN_BETAS, LRN_KS, LRN_SIZES, MUTATIONS, NO_GRAD, POOL_GEOMETRIES,  # noqa: E402
                       POOL_VALUE_KINDS, U, lrn_backward_bound, lrn_backward_ref, lrn_forward_bound, lrn_inputs,
                       lrn_ref, mutated_lrn_refs, outside_fraction, pool_inputs, pool_plane_sizes, pool_ref,
                       pooled_size, value_class)


def f32(v):
    return float(np.float32(v))


def _torch_lrn64(x, dy, size, alpha, beta, k):
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    y = F.local_response_norm(xt, size, alpha, beta, k)
    y.backward(torch.from_numpy(dy.astype(np.float64)))
    return y.detach().numpy(), xt.grad.numpy()


@pytest.mark.parametrize("size", LRN_SIZES)
@pytest.mark.parametrize("k", LRN_KS)
def test_lrn_ref_matches_torch_float64(size, k):
    for beta in LRN_BETAS:
        alpha = f32(1e-4)
        for c in (1, 2, 17):
            x, dy = lrn_inputs((2, c, 3, 5), alpha, k, seed=size * 100 + c)
            y, ymag = lrn_ref(x, size, alpha, beta, k)
            dx, ma, mb = lrn_backward_ref(x, dy, size, alpha, beta, k)
            yt, dxt = _torch_lrn64(x, dy, size, alpha, beta, k)
            assert np.all(np.abs(y - yt) <= 1e-12 * ymag), (size, k, beta, c)
            assert np.all(np.abs(dx - dxt) <= 1e-12 * (ma + mb)), (size, k, beta, c)


def test_lrn_ref_non_finite_classes_match_torch():
    x, _ = lrn_inputs((2, 9, 4, 4), 1e-4, 1.0, seed=5)
    rng = np.random.default_rng(6)
    u = rng.random(x.shape)
    x[u < 0.04] = np.nan
    x[u > 0.97] = np.inf
    x[(u > 0.5) & (u < 0.52)] = -np.inf
    for size in (1, 5, 15):
        for beta in (0.75, -0.5, 2.0):
            y, _ = lrn_ref(x, size, 1e-4, beta, 1.0)
            yt = F.local_response_norm(torch.from_numpy(x.astype(np.float64)), size, 1e-4, beta, 1.0).numpy()
            assert np.array_equal(value_class(y), value_class(yt)), (size, beta)


def _lrn_fp32(x, dy, size, alpha, beta, k):
    """the LRN kernels' arithmetic in fp32, operation by operation (numpy's powf in place of CUDA's)"""
    h, c = size // 2, x.shape[1]
    f = np.float32
    aon, beta32, k32 = f(f(alpha) / f(size)), f(beta), f(k)
    coef = f(f(f(2.0) * f(alpha)) * beta32) / f(size)
    xp = np.zeros((x.shape[0], c + 4 * h) + x.shape[2:], np.float32)
    xp[:, 2 * h:2 * h + c] = x
    dp = np.zeros_like(xp)
    dp[:, 2 * h:2 * h + c] = dy
    s = np.zeros_like(xp)  # s at padded channel i, for i in [h, c + 3h)
    for i in range(h, c + 3 * h):
        ss = np.zeros_like(x[:, 0])
        for j in range(-h, h + 1):
            if 0 <= i + j < xp.shape[1]:
                ss = ss + xp[:, i + j] * xp[:, i + j]
        s[:, i] = k32 + aon * ss
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        sb = np.power(s, -beta32)
        y = xp[:, 2 * h:2 * h + c] * sb[:, 2 * h:2 * h + c]
        r = dp * xp * sb / np.where(s == 0, f(1), s)  # s is only 0 outside [h, c + 3h), where r is not used
        r[:, :h] = 0
        r[:, h + c + 2 * h:] = 0
        acc = np.zeros_like(x)
        for j in range(-h, h + 1):
            acc = acc + r[:, 2 * h + j:2 * h + j + c]
        dx = dp[:, 2 * h:2 * h + c] * sb[:, 2 * h:2 * h + c] - coef * xp[:, 2 * h:2 * h + c] * acc
    return y, dx


@pytest.mark.parametrize("size", [3, 5, 15])
@pytest.mark.parametrize("k", [2.0, 1e-3])
def test_lrn_bounds_admit_fp32_and_reject_mutations(size, k):
    for beta in LRN_BETAS:
        alpha = f32(1e-4)
        x, dy = lrn_inputs((2, 33, 5, 7), alpha, k, seed=size + int(k * 10) + int(beta * 4))
        y, dx = _lrn_fp32(x, dy, size, alpha, beta, k)
        assert outside_fraction(y, dx, x, dy, size, alpha, beta, f32(k)) == (0.0, 0.0), (size, k, beta)
        if beta == 0:
            continue  # y = x and dx = dy whatever the window: nothing for a mutation to change
        for m in MUTATIONS:
            my, mdx = mutated_lrn_refs(x, dy, size, alpha, beta, f32(k), m)
            fy, fdx = outside_fraction(my.astype(np.float32), mdx.astype(np.float32), x, dy, size, alpha, beta,
                                       f32(k))
            assert fy > 0.5 and fdx > 0.5, (size, k, beta, m, fy, fdx)


def test_lrn_bound_constants():
    # n = 5, beta = 0.75: 0.75 * 9 + 8 + 2 units of u, about 1e-6 relative
    assert lrn_forward_bound(1.0, 5, 0.75) == pytest.approx(16.75 * U, rel=1e-9)
    assert lrn_backward_bound(1.0, 0.0, 5, 0.75) == pytest.approx(16.75 * U, rel=1e-6)


def _torch_pool(x, b, dy, k, s):
    xt = torch.from_numpy(x).requires_grad_()
    z = F.relu(xt + torch.from_numpy(b).view(1, -1, 1, 1))
    y, idx = F.max_pool2d(z, k, s, ceil_mode=True, return_indices=True)
    y.backward(torch.from_numpy(dy))
    return y.detach().numpy(), idx.numpy(), xt.grad.numpy()


def assert_pool_ref_matches_torch(x, b, k, s, seed, what):
    n, c, h, w = x.shape
    ph, pw = pooled_size(h, k, s), pooled_size(w, k, s)
    dy = np.random.default_rng(seed).standard_normal((n, c, ph, pw), dtype=np.float32)
    ref = pool_ref(x, b, k, s, dy)
    yt, it, dxt = _torch_pool(x, b, dy, k, s)
    assert ref.y.shape == yt.shape, what
    # bitwise, except that PyTorch's relu keeps -0.0 where the kernels store +0.0, and NaN payloads
    nan = np.isnan(ref.y)
    assert np.array_equal(nan, np.isnan(yt)), what
    zero = ref.y == 0
    assert np.array_equal(ref.y[zero], yt[zero]) and np.all(ref.y.view(np.int32)[zero] == 0), what
    other = ~nan & ~zero
    assert np.array_equal(ref.y.view(np.int32)[other], yt.view(np.int32)[other]), what
    flows = ref.index != NO_GRAD
    assert np.array_equal(flows, ~zero | nan), what
    i = ref.index.astype(np.int64)
    rows = np.arange(ph).reshape(1, 1, -1, 1) * s + i // k
    cols = np.arange(pw).reshape(1, 1, 1, -1) * s + i % k
    assert np.array_equal((rows * w + cols)[flows], it[flows]), f"{what}: index"
    assert np.array_equal(ref.dx.view(np.int32), dxt.view(np.int32)), f"{what}: dx"
    routed = np.where(flows, dy, 0).astype(np.float64)
    assert np.allclose(ref.dbias, routed.sum(axis=(0, 2, 3)), rtol=0, atol=1e-12)
    assert np.allclose(ref.dbias, dxt.astype(np.float64).sum(axis=(0, 2, 3)), rtol=0,
                       atol=1e-5 * ref.dbias_abs.max() + 1e-30)


@pytest.mark.parametrize("k,s", POOL_GEOMETRIES)
def test_pool_ref_matches_torch_on_every_geometry(k, s):
    for j, (h, w) in enumerate(pool_plane_sizes(k, s)):
        x, b = pool_inputs("randn", (2, 3, h, w), seed=k * 100 + s * 10 + j)
        assert_pool_ref_matches_torch(x, b, k, s, seed=j, what=(k, s, h, w))


@pytest.mark.parametrize("kind", POOL_VALUE_KINDS)
@pytest.mark.parametrize("k,s", [(3, 2), (3, 1), (2, 2), (5, 3), (1, 1), (2, 3)])
def test_pool_ref_matches_torch_on_special_values(kind, k, s):
    x, b = pool_inputs(kind, (2, 4, 11, 13), seed=7)
    assert_pool_ref_matches_torch(x, b, k, s, seed=8, what=(kind, k, s))


def test_pool_ref_special_value_rules():
    # -0.0 + -0.0: no gradient flows, y is +0.0
    x, b = pool_inputs("negative_zero", (1, 2, 5, 5), seed=1)
    r = pool_ref(x, b, 3, 2)
    assert np.all(r.index == NO_GRAD) and np.all(r.y.view(np.int32) == 0)
    # two NaNs in one window: the last one wins; a later finite value does not replace it
    x = np.zeros((1, 1, 3, 3), np.float32) + 1
    x[0, 0, 0, 1] = x[0, 0, 1, 0] = np.nan
    x[0, 0, 2, 2] = 5
    r = pool_ref(x, np.zeros(1, np.float32), 3, 1)
    assert r.index[0, 0, 0, 0] == 3 and np.isnan(r.y[0, 0, 0, 0])
    # a tie that only exists after fl32(x + b): 2^23 + 1, 2^23 + 1.25 and 2^23 + 0.75 all round to 2^23 + 1, so
    # the first of them wins although 1.25 is the largest x
    x = np.zeros((1, 1, 3, 3), np.float32)
    x[0, 0, 0] = [1.0, 1.25, 0.75]
    r = pool_ref(x, np.float32([2.0 ** 23]), 3, 3)
    assert r.index[0, 0, 0, 0] == 0 and r.y[0, 0, 0, 0] == 2.0 ** 23 + 1
