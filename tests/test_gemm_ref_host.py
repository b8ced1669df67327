"""Host checks of gemm_ref.py, the fp32 restatement of the built-in engine's GEMM core that test_gpu_gemm_order.py
compares the GPU with bit for bit: fma32 against exact rational arithmetic, the restatement against producer_ops_ref's
float64 references and bounds, its teeth (each plausible wrong order or rounding changes most outputs at the GPU
test's own shapes, so bit equality there means something), and the edges of the split-K chunking."""
import math
from fractions import Fraction

import numpy as np
import pytest

import gemm_ref as G
import producer_ops_ref as R
from autoencoder_ops_ref import deconv_backward, deconv_bounds, deconv_forward
from test_gpu_gemm_order import CONV_CASES, DECONV_CASES, IP_CASES, conv_inputs, deconv_inputs, ip_inputs

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)


def _round_f32(v, zero_sign):
    """the fp32 value nearest the rational v, ties to even, with subnormals and overflow to +-inf; `zero_sign` is the
    sign of an exact zero (IEEE: +0 unless both addends are -0)"""
    if v == 0:
        return math.copysign(0.0, zero_sign)
    neg, a = v < 0, abs(v)
    e = a.numerator.bit_length() - a.denominator.bit_length()  # 2^e <= a < 2^(e + 2)
    if Fraction(2) ** (e + 1) <= a:
        e += 1
    elif Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)  # the quantum of a's binade (the subnormal one below 2^-126)
    n = a / q
    f = n.numerator // n.denominator
    rem = n - f
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and f % 2):
        f += 1
    r = f * q
    out = math.inf if r >= Fraction(2) ** 128 else float(r)
    return -out if neg else out


def _exact_fma(a, b, c):
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        with np.errstate(invalid="ignore", over="ignore"):
            return float(np.float64(a) * np.float64(b) + np.float64(c))  # the product is exact in float64
    p = Fraction(a) * Fraction(b)
    p_neg = math.copysign(1, a) * math.copysign(1, b) < 0
    zero_sign = -1.0 if (p == 0 and p_neg and c == 0 and math.copysign(1, c) < 0) else 1.0
    return _round_f32(p + Fraction(c), zero_sign)


def _bits(v):
    return np.asarray(v, F32).view(np.uint32)


def _agree(a, b, c, what):
    got = G.fma32(a, b, c)
    for i in range(len(a)):
        want = F32(_exact_fma(a[i], b[i], c[i]))
        ok = (np.isnan(want) and np.isnan(got[i])) or _bits(want) == _bits(got[i])
        assert ok, f"{what} {i}: fma({a[i]!r}, {b[i]!r}, {c[i]!r}) = {got[i]!r}, exact rounding {want!r}"


def _f32(v):
    with np.errstate(over="ignore"):
        return np.asarray(v, np.float64).astype(F32)


# --------------------------------------------------------------------------- fma32 against exact rationals
def test_fma32_random_triples_across_exponents():
    rng = np.random.default_rng(1)
    n = 100_000
    a = _f32(rng.standard_normal(n) * np.exp2(rng.integers(-70, 64, n)))
    b = _f32(rng.standard_normal(n) * np.exp2(rng.integers(-70, 64, n)))
    c = _f32(rng.standard_normal(n) * np.exp2(rng.integers(-150, 128, n)))
    # half of them cancel into the low bits: c is minus the product rounded to fp32 (or to fewer bits)
    k = n // 2
    p = a[:k].astype(np.float64) * b[:k]
    c[:k] = _f32(-p)
    c[: k // 2] = _f32(-np.round(p[: k // 2] * 2.0 ** 10) * 2.0 ** -10)
    _agree(a, b, c, "triple")


def test_fma32_exact_ties_and_tails():
    u = 2.0 ** -23
    a = [1 + 2 ** -12, 1 + 2 ** -12 + u, 1 + 2 ** -12 + u, 1 + 2 ** -12, 1 + 2 ** -12, 3 * (1 + 2 ** -12)]
    b = [1 + 2 ** -12, 1 + 2 ** -12, 1 + 2 ** -12, 1 + 2 ** -12, 1 + 2 ** -12, 1 + 2 ** -12]
    c = [0.0, 0.0, -2.0 ** -40, 2.0 ** -60, -2.0 ** -60, 0.0]
    # a * b = 1 + 2^-11 + 2^-24 exactly: halfway, so the tail (or ties-to-even) decides
    a, b, c = _f32(a), _f32(b), _f32(c)
    _agree(a, b, c, "tie")
    assert G.fma32(a[3:5], b[3:5], c[3:5])[0] != G.fma32(a[3:5], b[3:5], c[3:5])[1]  # the tail's sign decides
    # constructed ties across binades: p exact in 48 bits, c moves p + c onto a midpoint plus or minus a tail
    rng = np.random.default_rng(2)
    n = 4000
    a = _f32(rng.uniform(1, 2, n) * np.exp2(rng.integers(-20, 20, n)))
    b = _f32(rng.uniform(1, 2, n) * np.exp2(rng.integers(-20, 20, n)))
    p = a.astype(np.float64) * b
    r = p.astype(F32).astype(np.float64)
    mid = r + np.spacing(r.astype(F32)).astype(np.float64) / 2
    tail = np.choose(rng.integers(0, 3, n), [np.zeros(n), np.spacing(mid) * 4, -np.spacing(mid) * 4])
    c = _f32(mid + tail - p)  # rounding c to fp32 keeps most of these on or next to the tie
    _agree(a, b, c, "constructed tie")


def test_fma32_subnormals():
    rng = np.random.default_rng(3)
    n = 20000
    tiny = 2.0 ** -149
    a = _f32(rng.integers(-2 ** 23, 2 ** 23, n) * tiny)  # subnormal operands
    b = _f32(rng.standard_normal(n) * np.exp2(rng.integers(-2, 30, n)))
    c = _f32(rng.integers(-2 ** 24, 2 ** 24, n) * tiny)  # subnormal or smallest-normal addends
    _agree(a, b, c, "subnormal operand")
    # normal operands whose product and sum land in or under the subnormal range, ties at 2^-150 included
    a = _f32(rng.uniform(1, 2, n) * np.exp2(rng.integers(-90, -60, n)))
    b = _f32(rng.uniform(-2, 2, n) * np.exp2(rng.integers(-90, -60, n)))
    c = _f32(rng.integers(-64, 64, n) * tiny)
    _agree(a, b, c, "subnormal result")
    h = _f32([2.0 ** -75] * 4)
    _agree(h, h, _f32([0.0, -0.0, tiny, -tiny]), "2^-150 tie")
    _agree(h, -h, _f32([0.0, -0.0, tiny, -tiny]), "-2^-150 tie")


def test_fma32_overflow_inf_nan_and_signed_zeros():
    big = FLT_MAX
    # 18631 * 1801 = 2^25 - 1: with 2^103 the product is exactly FLT_MAX + ulp / 2, the overflow tie
    a = _f32([big, big, -big, 2.0 ** 100, 18631 * 2.0 ** 50, 18631 * 2.0 ** 50, 18631 * 2.0 ** 50, 1.0])
    b = _f32([2.0, 1.0, 2.0, 2.0 ** 100, 1801 * 2.0 ** 53, 1801 * 2.0 ** 53, 1801 * 2.0 ** 53, big])
    c = _f32([0.0, big, 0.0, 0.0, 0.0, -1.0, 1.0, 2.0 ** 103])
    _agree(a, b, c, "overflow")
    r = G.fma32(a, b, c)
    assert r[4] == np.inf and r[5] == F32(big) and r[6] == np.inf
    inf, nan = np.inf, np.nan
    a = _f32([inf, inf, -inf, 0.0, nan, 1.0, inf, 2.0, 1.0])
    b = _f32([1.0, 0.0, 2.0, inf, 1.0, nan, 1.0, 3.0, 1.0])
    c = _f32([1.0, 1.0, inf, 0.0, 0.0, 0.0, -inf, nan, -inf])
    _agree(a, b, c, "inf/nan")
    assert np.array_equal(np.isnan(G.fma32(a, b, c)), [False, True, True, True, True, True, True, True, False])
    # signed zeros: -0 only when the product and the addend are both -0
    z = np.array([[0.0, 0.0, 0.0], [-0.0, 1.0, -0.0], [0.0, -1.0, -0.0], [-0.0, 1.0, 0.0], [1.0, 1.0, -1.0],
                  [-1.0, 1.0, 1.0], [2.0 ** -100, -2.0 ** -100, 0.0], [2.0 ** -100, 2.0 ** -100, -0.0]])
    a, b, c = _f32(z[:, 0]), _f32(z[:, 1]), _f32(z[:, 2])
    _agree(a, b, c, "signed zero")
    assert list(np.signbit(G.fma32(a, b, c))) == [False, True, True, False, False, False, True, False]


# --------------------------------------------------------------------------- the restatement against float64
def _within(got, ref, bound, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    assert np.all(err <= bound), f"{what}: {np.max(err - bound):.3e} outside the bound"


@pytest.mark.parametrize("case", [c for c in CONV_CASES if c[-1] == "gaussian" and c[0] <= 2], ids=str)
def test_conv_restatement_is_within_the_float64_bounds(case):
    x, w, b, geo = conv_inputs(*case[:-1], family="gaussian")
    y = G.conv_forward(x, w, b, geo)
    by, bw, bb, bx = R.conv_bounds(x, w, b, y, geo)
    _within(y, R.conv_forward(x, w, b, geo), by, "y")
    dw, db, dx = R.conv_backward(x, w, y, geo)
    _within(G.conv_weight_grad(x, y, geo), dw, bw, "dW")
    _within(G.bias_grad(y, y.shape[0], y.shape[1], y.shape[2] * y.shape[3]), db, bb, "db")
    _within(G.conv_data_grad(y, w, None, x.shape, geo), dx, bx, "dx")


@pytest.mark.parametrize("case", [c for c in IP_CASES if c[-1] == "gaussian" and c[0][0] < 10 ** 5], ids=str)
def test_ip_restatement_is_within_the_float64_bounds(case):
    x, w, b = ip_inputs(*case[:-1], family="gaussian")
    y = G.ip_forward(x, w, b)
    by, bw, bb, bx = R.ip_bounds(x, w, b, y)
    _within(y, R.ip_forward(x, w, b), by, "y")
    dw, db, dx = R.ip_backward(x, w, y)
    _within(G.ip_weight_grad(x, y), dw, bw, "dW")
    _within(G.bias_grad(y, y.shape[0], y.shape[1], 1), db, bb, "db")
    _within(G.ip_data_grad(y, w, x.shape), dx, bx, "dx")


@pytest.mark.parametrize("case", [c for c in DECONV_CASES if c[-1] == "gaussian" and c[0] <= 2], ids=str)
def test_deconv_restatement_is_within_the_float64_bounds(case):
    x, w, b, geo = deconv_inputs(*case[:-1], family="gaussian")
    y64 = deconv_forward(x, w, b, geo)
    y = G.deconv_forward(x, w, b, geo, y64.shape[2:])
    by, bw, bb, bx = deconv_bounds(x, w, b, y, geo)
    _within(y, y64, by, "y")
    dw, db, dx = deconv_backward(x, w, y, geo)
    _within(G.deconv_weight_grad(x, y, geo), dw, bw, "dW")
    _within(G.bias_grad(y, y.shape[0], y.shape[1], y.shape[2] * y.shape[3]), db, bb, "db")
    _within(G.deconv_data_grad(y, w, geo), dx, bx, "dx")


# --------------------------------------------------------------------------- teeth
def _differs(ref, mut):
    return float(np.mean(_bits(ref) != _bits(mut)))


# the GPU test's Gaussian cases deep enough for each mutation: chains of at least 64 products for the two chain
# mutations, at least 7 partials for the two reduction mutations
CHAIN_TEETH = [("conv", (2, 57, 5, 5, 3, (3, 3, 1, 1, 1, 1), True)), ("conv", (2, 3, 40, 40, 4, (3, 3, 1, 1, 1, 1), True)),
               ("ip", ((65, 1000), 129, True)), ("ip", ((4, 9216), 64, True))]
SPLIT_TEETH = [("conv", (2, 3, 40, 40, 4, (3, 3, 1, 1, 1, 1), True)), ("conv", (1, 2, 3, 43691, 3, (1, 1, 1, 1, 0, 0), True)),
               ("ip", ((131073, 5), 3, True))]


def _teeth_run(op, case, mutation):
    """the one restated product of the case that the mutation touches: the forward for the chain mutations, the
    weight gradient (of the restated y as the top gradient) for the reduction ones"""
    if op == "conv":
        x, w, b, geo = conv_inputs(*case, family="gaussian")
        if mutation in ("mul_add", "reversed"):
            return G.conv_forward(x, w, b, geo), G.conv_forward(x, w, b, geo, mutation)
        y = G.conv_forward(x, w, b, geo)
        return G.conv_weight_grad(x, y, geo), G.conv_weight_grad(x, y, geo, mutation)
    x, w, b = ip_inputs(*case, family="gaussian")
    if mutation in ("mul_add", "reversed"):
        return G.ip_forward(x, w, None), G.ip_forward(x, w, None, mutation)
    y = G.ip_forward(x, w, b)
    return G.ip_weight_grad(x, y), G.ip_weight_grad(x, y, mutation)


@pytest.mark.parametrize("mutation", ["mul_add", "reversed"])
@pytest.mark.parametrize("op,case", CHAIN_TEETH, ids=str)
def test_chain_mutations_change_most_outputs(op, case, mutation):
    ref, mut = _teeth_run(op, case, mutation)
    assert _differs(ref, mut) > 0.5, _differs(ref, mut)


@pytest.mark.parametrize("mutation", ["partials_reversed", "unsplit"])
@pytest.mark.parametrize("op,case", SPLIT_TEETH, ids=str)
def test_reduction_mutations_change_most_outputs(op, case, mutation):
    ref, mut = _teeth_run(op, case, mutation)
    assert _differs(ref, mut) > 0.5, _differs(ref, mut)


def test_teeth_cases_are_the_gpu_tests_own():
    for op, case in CHAIN_TEETH + SPLIT_TEETH:
        assert case + ("gaussian",) in {"conv": CONV_CASES, "ip": IP_CASES}[op]


# --------------------------------------------------------------------------- split_chunk's edges
@pytest.mark.parametrize("k,chunk,splits,last", [(511, 512, 1, 511), (512, 512, 1, 512), (513, 512, 2, 1),
                                                 (3200, 512, 7, 128), (131072, 512, 256, 512),
                                                 (131073, 528, 249, 129), (262144, 1024, 256, 1024),
                                                 (774400, 3040, 255, 2240)])
def test_split_chunk_edges(k, chunk, splits, last):
    assert (R.split_chunk(k), R.splits_of(k)) == (chunk, splits)
    assert k - (splits - 1) * chunk == last
    assert chunk % R.BK == 0 and splits <= R.MAX_SPLITS


def test_split_chunk_never_exceeds_256_partials():
    for k in list(range(1, 3000)) + list(range(131000, 132000)) + [2 ** 31 - 1]:
        c, s = R.split_chunk(k), R.splits_of(k)
        assert c % 16 == 0 and 1 <= s <= 256 and (s - 1) * c < k <= s * c
