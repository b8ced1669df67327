"""CPU checks of tests/bn_ref.py, the BatchNorm references and bounds the -m gpu file test_gpu_batch_norm_reference.py
holds the kernels to: the fp32 restatement in the kernels' operation order stays inside the bounds, each plausible
kernel mistake of MUTATIONS falls outside them, and the dyadic input family makes the statistics exactly
predictable."""
from fractions import Fraction

import numpy as np
import pytest

import bn_ref as B

F32 = np.float32

# small enough for the CPU, with the features the bounds must survive: M = 1, a 2-D bottom, H*W = 1, planes past a
# warp and per-channel scales over six decades
SHAPES = [(1, 3, 1, 1), (2, 7), (7, 9, 3, 3), (3, 11, 5, 7), (2, 6, 33, 33), (32, 5, 4, 4)]


@pytest.mark.parametrize("eps", [1e-5, 1e-3])
@pytest.mark.parametrize("shape", SHAPES)
def test_restatement_stays_inside_the_bounds(shape, eps):
    rng = np.random.default_rng(sum(shape))
    x, dy = B.gaussian(rng, shape)
    out = B.kernel_model(x, dy, eps)
    fr = B.outside_fractions(x, dy, out, eps)
    assert all(v == 0 for v in fr.values()), fr


@pytest.mark.parametrize("shape", SHAPES)
def test_restatement_stays_inside_the_bounds_with_eps_0(shape):
    """eps = 0 needs var > 0 everywhere: no constant channel, M > 1"""
    if np.prod(shape) // shape[1] == 1:
        pytest.skip("M = 1 has var = 0")
    rng = np.random.default_rng(3 + sum(shape))
    x, dy = B.gaussian(rng, shape, constant=False)
    fr = B.outside_fractions(x, dy, B.kernel_model(x, dy, 0.0), 0.0)
    assert all(v == 0 for v in fr.values()), fr


def _case_for(mutation):
    """(x, dy, eps): an input on which `mutation` shows"""
    rng = np.random.default_rng(11)
    shape = (4, 6, 3, 3)
    if mutation == "one_pass_var":  # a large channel offset: E[x^2] and mean^2 cancel in fp32
        x = (F32(1e4) + rng.standard_normal(shape, dtype=F32)).astype(F32)
        return x, rng.standard_normal(shape, dtype=F32), 1e-5
    if mutation == "eps_after_sqrt":  # small variances: sqrt(var) + eps is far from sqrt(var + eps)
        x = (rng.standard_normal(shape, dtype=F32) * F32(1e-2)).astype(F32)
        return x, rng.standard_normal(shape, dtype=F32), 1e-3
    x = (rng.standard_normal(shape, dtype=F32) * F32(1.5) + F32(2)).astype(F32)
    # dy with a mean and a component along x^: S1 and S2 are far from 0
    xh = (x - x.mean((0, 2, 3), keepdims=True)) / x.std((0, 2, 3), keepdims=True)
    dy = (F32(1) + F32(0.5) * xh + rng.standard_normal(shape, dtype=F32) * F32(0.1)).astype(F32)
    return x, dy, 1e-5


@pytest.mark.parametrize("mutation", B.MUTATIONS)
def test_every_mutation_falls_outside_the_bounds(mutation):
    x, dy, eps = _case_for(mutation)
    assert all(v == 0 for v in B.outside_fractions(x, dy, B.kernel_model(x, dy, eps), eps).values())
    fr = B.outside_fractions(x, dy, B.kernel_model(x, dy, eps, mutation), eps)
    print(mutation, {k: round(float(v), 3) for k, v in fr.items()})
    assert max(fr.values()) > 0.5, fr


@pytest.mark.parametrize("mutation", B.MUTATIONS)
def test_every_mutation_changes_the_gaussian_family(mutation):
    """On the family the GPU sweep uses, each mutation puts some channel or element outside the bounds."""
    rng = np.random.default_rng(5)
    x, dy = B.gaussian(rng, (5, 12, 4, 4))
    if mutation in ("k_over_m_minus_1", "no_s2"):  # dy correlated with x: S1 and S2 are large
        dy = (x - x.mean((0, 2, 3), keepdims=True)) + dy
    fr = B.outside_fractions(x, dy, B.kernel_model(x, dy, 1e-5, mutation), 1e-5)
    assert max(fr.values()) > 0, fr


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (3, 4, 5, 7), (2, 3, 1, 1), (5, 2), (4, 2, 112, 112),
                                   (1, 2, 3, 5)])
def test_dyadic_family_is_exactly_predictable(shape):
    """mean = the centre; var = fl32(fl64(sum d^2 / M)); S1 = sum dy; the blobs follow from those in fp32.  All are
    computed here from integers, apart from the restatement's summation order."""
    rng = np.random.default_rng(sum(shape))
    x, dy = B.dyadic(rng, shape)
    xp, g = B.planes(x).astype(np.float64), B.planes(dy).astype(np.float64)
    n, c, hw = xp.shape
    m = n * hw
    assert np.array_equal(xp * 256, np.round(xp * 256)) and np.abs(xp).max() <= 4 and np.abs(g).max() <= 2
    ints = (xp * 256).astype(np.int64)
    centre = [Fraction(int(v), 256 * m) for v in ints.sum((0, 2))]
    blobs = (rng.standard_normal(c).astype(F32), rng.random(c).astype(F32) + F32(1), F32([7.25]))
    _, mean, var, nb = B.restate_forward(x, blobs)
    for ch in range(c):
        assert Fraction(float(mean[ch])) == centre[ch]  # the mean is exact
    # x - mean and its square are exact in float64, and so is their sum: one double division, one rounding to fp32
    want_var = np.array([F32(((xp[:, ch] - float(mean[ch])) ** 2).sum() / m) for ch in range(c)], F32)
    np.testing.assert_array_equal(var.view(np.uint32), want_var.view(np.uint32))
    f = F32(0.999)
    corr = F32(m) / F32(m - 1) if m > 1 else F32(1)
    for got, want in zip(nb, (mean + f * blobs[0], corr * var + f * blobs[1], blobs[2] * f + F32(1))):
        np.testing.assert_array_equal(np.asarray(got, F32).view(np.uint32), np.asarray(want, F32).view(np.uint32))
    _, s1, _ = B.restate_backward(x, dy, mean, var)
    want_s1 = np.array([F32(Fraction(int((g[:, ch] * 256).sum()), 256)) for ch in range(c)], F32)
    np.testing.assert_array_equal(s1.view(np.uint32), want_s1.view(np.uint32))
    # the order of the sums does not matter on this family: a reversed order gives the same bits
    rev = B.restate_forward(x[::-1].copy(), blobs)[1:3]
    assert np.array_equal(rev[0], mean) and np.array_equal(rev[1], var)


def test_restatement_y_from_given_statistics_is_libm_powf():
    """y from given statistics uses powf(fl(var + eps), 0.5f), not sqrtf: on an input where the two differ, y does."""
    v = np.arange(0x3f800000, 0x3f800000 + (1 << 15), dtype=np.uint32).view(F32)  # [1, 1 + 2^15 ulp)
    p = B.powf_half(v)
    s = np.sqrt(v)
    k = int(np.nonzero(p != s)[0][0])  # glibc's powf rounds a double approximation: some of these differ
    x = np.array([[p[k]], [-p[k]]], F32)  # N = 2, C = 1
    y, _, _, _ = B.restate_forward(x, (F32([0]), F32([0]), F32([0])), eps=0.0, stats=(F32([0]), F32([v[k]])))
    assert y[0, 0] == 1.0 and y[1, 0] == -1.0


def test_oracle_powf_half_fill_is_libm_powf():
    """The threaded fill the device powf sweep compares against gives libm's powf(x, 0.5f), subnormals, +-0, +inf
    and NaN included."""
    from oracle import adam
    adam.build()
    for lo, hi in ((0, 5000), (0x3f800000, 0x3f800000 + 40000), (0x7f7ff000, 0x7f800010), (0x80000000, 0x80000010)):
        got = adam.powf_half_fill(lo, hi, threads=3)
        want = B.powf_half(np.arange(lo, hi, dtype=np.uint64).astype(np.uint32).view(F32))
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        np.testing.assert_array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32))
