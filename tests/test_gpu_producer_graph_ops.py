"""The built-in producer's graph and loss ops, Slice, Concat, Split, Eltwise, Scale, EuclideanLoss and ContrastiveLoss,
and its BatchNorm and within-channel LRN (DESIGN.md section 14), on the GPU, element by element against the references
of producer_ops_ref.py, test_gpu_batch_norm.py and lrn_within_ref.py, through the injector harness of
test_gpu_producer_ops.py: every bottom comes from an injector of its own, so each op's inputs and data gradients are
read exactly.  An op with several tops (Slice, Split) has them gathered into the one probe by a Concat, itself checked
here first, whose bottoms are listed in another order than the tops.

The copies (Slice, Concat, Split's forward) and Eltwise MAX are compared by value, NaN, infinities and subnormals
included; the rest by value on dyadic inputs and against the per-element bounds on Gaussian ones."""
import numpy as np
import pytest

import producer_ops_ref as R
import test_gpu_batch_norm as BN
from gpu_util import assert_bits_equal
from lrn_within_ref import backward_bound, forward_bound, lrn_within_backward_ref, lrn_within_ref
from test_batch_norm_host import numpy_bn_forward
from test_gpu_producer_ops import F32, _check, _close, _engine, _equal, _probe, _same

pytestmark = pytest.mark.gpu


def _specials(rng, shape):
    """Gaussian values with NaN, +-inf, subnormals and zeros spread through them"""
    x = R.gaussian(rng, shape).ravel()
    k = rng.choice(x.size, size=min(x.size, 10), replace=False)
    x[k] = np.array([np.nan, np.inf, -np.inf, 1e-40, -3e-42, R.TINY, 0.0, -0.0, 3e38, -1e-45], F32)[:k.size]
    return x.reshape(shape)


def _gather(name, tops, axis, out="y"):
    """Concat of `tops` (in the order given) into `out`"""
    return (f'layer {{ name: "{name}" type: "Concat" ' + " ".join(f'bottom: "{t}"' for t in tops) +
            f' top: "{out}" concat_param {{ axis: {axis} }} }}\n')


# --------------------------------------------------------------------------- Concat (checked first: it gathers below)
CONCAT_CASES = [  # (bottom shapes, concat_param, canonical axis, index of a staged bottom or None)
    ([(3, 4, 5, 6), (2, 4, 5, 6)], "axis: 0", 0, None),
    ([(2, 3, 5, 6), (2, 1, 5, 6), (2, 4, 5, 6)], "", 1, None),
    ([(2, 3, 2, 6), (2, 3, 5, 6), (2, 3, 1, 6), (2, 3, 3, 6)], "axis: 2", 2, None),
    ([(2, 3, 4, 1), (2, 3, 4, 5), (2, 3, 4, 2), (2, 3, 4, 7), (2, 3, 4, 3)], "axis: 3", 3, None),
    ([(2, 3, 4, 5), (2, 3, 4, 2)], "axis: -1", 3, None),
    ([(2, 3, 4, 5), (2, 3, 2, 5), (2, 3, 3, 5)], "axis: -2", 2, 1),
    ([(5, 3), (5, 7)], "concat_dim: 1", 1, None),
    ([(2, 6), (4, 6), (1, 6)], "concat_dim: 0", 0, 0),
    ([(2, 3, 7), (2, 5, 7)], "axis: 1", 1, 1),
]


def concat_body(n_injected, staged, param):
    names = [f"x{i}" for i in range(n_injected)]
    if staged is not None:
        names.insert(staged, "st")
    return ('layer { name: "cat" type: "Concat" ' + " ".join(f'bottom: "{b}"' for b in names) +
            f' top: "y" concat_param {{ {param} }} }}\n')


@pytest.mark.parametrize("shapes,param,axis,staged", CONCAT_CASES)
def test_concat(cos, tmp_path, shapes, param, axis, staged):
    rng = np.random.RandomState(sum(int(np.prod(s)) for s in shapes) + axis)
    xs = [_specials(rng, s) for s in shapes]
    injected = [x for i, x in enumerate(xs) if i != staged]
    y = np.concatenate(xs, axis=axis)
    body = concat_body(len(injected), staged, param)
    st = {} if staged is None else {"st": xs[staged]}
    r = _engine(cos, tmp_path, injected, body, (), y.shape, np.zeros(y.shape, F32), staged=st)
    _same(r["d"], y, "y")  # B = 0: the probe returns y, and y is the top gradient
    for i, (dx, x) in enumerate(zip(r["dx"], injected)):
        _same(dx, x, f"dx{i}")  # its own range of the top gradient, that is its own values


# --------------------------------------------------------------------------- Slice
SLICE_CASES = [  # (bottom shape, slice_param, canonical axis, [begin, end) per top, unread top or None)
    ((6, 3, 4, 5), "axis: 0 slice_point: 1 slice_point: 4", 0, R.slice_bounds(6, [1, 4]), None),
    ((2, 7, 4, 5), "slice_point: 2 slice_point: 3 slice_point: 6", 1, R.slice_bounds(7, [2, 3, 6]), 1),
    ((2, 3, 8, 5), "axis: 2", 2, R.slice_bounds(8, tops=2), None),
    ((2, 3, 4, 9), "axis: 3 slice_point: 4", 3, R.slice_bounds(9, [4]), None),
    ((2, 3, 4, 9), "axis: -1", 3, R.slice_bounds(9, tops=3), 2),
    ((3, 6, 5), "slice_dim: 2 slice_point: 1 slice_point: 2", 2, R.slice_bounds(5, [1, 2]), 0),
    ((3, 12), "slice_dim: 1", 1, R.slice_bounds(12, tops=4), None),
    ((10, 3), "axis: 0 slice_point: 7", 0, R.slice_bounds(10, [7]), None),
]


def slice_body(param, ntops, unread, axis):
    tops = [f"s{t}" for t in range(ntops)]
    read = [t for t in tops if t != (f"s{unread}" if unread is not None else None)]
    return ('layer { name: "sl" type: "Slice" bottom: "x0" ' + " ".join(f'top: "{t}"' for t in tops) +
            f' slice_param {{ {param} }} }}\n' + _gather("gather", read[::-1], axis)), read[::-1]


@pytest.mark.parametrize("shape,param,axis,ranges,unread", SLICE_CASES)
def test_slice(cos, tmp_path, shape, param, axis, ranges, unread):
    rng = np.random.RandomState(int(np.prod(shape)) + len(param))
    x = _specials(rng, shape)
    parts = R.slice_forward(x, axis, ranges)
    body, gathered = slice_body(param, len(ranges), unread, axis)
    y = np.concatenate([parts[int(t[1:])] for t in gathered], axis=axis)
    r = _engine(cos, tmp_path, [x], body, (), y.shape, np.zeros(y.shape, F32))
    _same(r["d"], y, "y")
    want = x.copy()  # the read tops' gradients are their own values; the unread top's range gets exactly 0
    if unread is not None:
        idx = [slice(None)] * x.ndim
        idx[axis] = slice(*ranges[unread])
        want[tuple(idx)] = 0
    _same(r["dx"][0], want, "dx")


# --------------------------------------------------------------------------- Split
SPLIT_CASES = [  # (tops, unread top or None, the top with an in-place ReLU)
    (2, None, 1), (3, 1, 2), (4, 1, 3), (4, None, 0),
]


def split_body(ntops, unread, relu):
    tops = [f"s{t}" for t in range(ntops)]
    read = [t for t in range(ntops) if t != unread]
    return ('layer { name: "sp" type: "Split" bottom: "x0" ' + " ".join(f'top: "{t}"' for t in tops) + " }\n" +
            f'layer {{ name: "r" type: "ReLU" bottom: "s{relu}" top: "s{relu}" }}\n' +
            _gather("gather", [f"s{t}" for t in read[::-1]], 0)), read


@pytest.mark.parametrize("ntops,unread,relu", SPLIT_CASES)
def test_split(cos, tmp_path, ntops, unread, relu):
    rng = np.random.RandomState(10 * ntops + relu)
    shape = (4, 3, 5, 6)
    x = R.gaussian(rng, shape) * np.exp2(rng.randint(-12, 12, size=shape)).astype(F32)  # spread: the order shows
    body, read = split_body(ntops, unread, relu)
    # the in-place ReLU has storage of its own (a Split top): the siblings read x, not relu(x) (DESIGN.md section 14)
    tops = {t: (np.maximum(x, 0) if t == relu else x) for t in read}
    y = np.concatenate([tops[t] for t in read[::-1]], axis=0)
    B = _probe(y.astype(np.float64), rng, "gaussian")
    r = _engine(cos, tmp_path, [x], body, (), y.shape, B)
    _same(r["d"], y - B, "y")
    d = dict(zip(read[::-1], np.split(r["d"], len(read), axis=0)))
    g = [np.where(x > 0, d[t], F32(0)) if t == relu else d[t] for t in read]
    _close(r["dx"][0], sum(v.astype(np.float64) for v in g), R.split_backward_bound(g), "dx")
    if len(g) > 2:
        assert np.any(R.split_backward32(g) != R.split_backward32(g, reverse=True)), "the order must show"
    _same(r["dx"][0], R.split_backward32(g), "dx (fp32, top order)")


# --------------------------------------------------------------------------- Eltwise
ELT_SHAPES = [(4, 3, 5, 6), (7, 33)]


def eltwise_body(k, op, extra=""):
    return ('layer { name: "e" type: "Eltwise" ' + " ".join(f'bottom: "x{i}"' for i in range(k)) +
            f' top: "y" eltwise_param {{ operation: {op} {extra} }} }}\n')


@pytest.mark.parametrize("shape", ELT_SHAPES)
@pytest.mark.parametrize("coeffs", [(1, 1), (1, -1.5), (1, 0, -1.5, 0.1), (0.1, 1, 1)])
@pytest.mark.parametrize("family", ["dyadic", "gaussian"])
def test_eltwise_sum(cos, tmp_path, shape, coeffs, family):
    exact = family == "dyadic" and 0.1 not in coeffs
    rng = np.random.RandomState(len(coeffs) * 10 + len(shape))
    xs = [R.dyadic(rng, shape) if family == "dyadic" else R.gaussian(rng, shape) for _ in coeffs]
    y64, by = R.eltwise_sum(xs, coeffs)
    B = _probe(y64, rng, family)
    extra = " ".join(f"coeff: {c}" for c in coeffs)
    r = _engine(cos, tmp_path, xs, eltwise_body(len(xs), "SUM", extra), (), y64.shape, B)
    if exact:
        _same(r["d"], np.asarray(y64, F32) - B, "y")
    else:
        _close(r["d"], y64 - B.astype(np.float64), by + R.ulp(r["d"]) / 2, "y")
    for i, c in enumerate(coeffs):
        _same(r["dx"][i], R.eltwise_sum_backward32(r["d"], c), f"dx{i}")


@pytest.mark.parametrize("shape", ELT_SHAPES)
@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("stable", [True, False], ids=["stable", "y-over-x"])
def test_eltwise_prod(cos, tmp_path, shape, k, stable):
    rng = np.random.RandomState(k * 10 + len(shape) + stable)
    xs = [R.gaussian(rng, shape) for _ in range(k)]
    for x in xs:
        x.ravel()[rng.choice(x.size, size=x.size // 10, replace=False)] = 0  # zeros: y / x is 0 / 0 there
    y64, by = R.eltwise_prod(xs)
    B = _probe(y64, rng, "gaussian")
    r = _engine(cos, tmp_path, xs, eltwise_body(k, "PROD", f"stable_prod_grad: {str(stable).lower()}"), (), y64.shape, B)
    _close(r["d"], y64 - B.astype(np.float64), by + R.ulp(r["d"]) / 2, "y")
    for i, (g, b) in enumerate(R.eltwise_prod_backward(xs, r["d"], stable)):
        _close(r["dx"][i], g, b, f"dx{i}")
        if not stable:
            assert np.isnan(g).any()


@pytest.mark.parametrize("shape", ELT_SHAPES)
@pytest.mark.parametrize("k", [2, 3, 4, 5])
def test_eltwise_max(cos, tmp_path, shape, k):
    rng = np.random.RandomState(k + len(shape))
    xs = [R.dyadic(rng, shape, top=2) for _ in range(k)]  # 5 values: ties everywhere
    for x in xs:
        idx = rng.choice(x.size, size=x.size // 8, replace=False)
        x.ravel()[idx[: idx.size // 2]] = np.nan
        x.ravel()[idx[idx.size // 2:]] = -np.inf
    y, win = R.eltwise_max(xs)
    B = R.dyadic(rng, shape)
    r = _engine(cos, tmp_path, xs, eltwise_body(k, "MAX"), (), y.shape, B)
    _same(r["d"], y - B, "y")
    for i, want in enumerate(R.eltwise_max_backward(r["d"], win, k)):
        _same(r["dx"][i], want, f"dx{i}")


@pytest.mark.parametrize("op", ["SUM", "PROD", "MAX"])
def test_eltwise_of_two_split_tops(cos, tmp_path, op):
    """x + 0.5 x, x * x and max(x, x) from two tops of one blob (the same memory); the Split adds both gradients"""
    rng = np.random.RandomState(len(op))
    x = R.gaussian(rng, (4, 3, 5, 6))
    body = ('layer { name: "sp" type: "Split" bottom: "x0" top: "a" top: "b" }\n'
            f'layer {{ name: "e" type: "Eltwise" bottom: "a" bottom: "b" top: "y" eltwise_param {{ operation: {op} '
            f'{"coeff: 1 coeff: 0.5" if op == "SUM" else ""} }} }}\n')
    y = {"SUM": x + F32(0.5) * x, "PROD": x * x, "MAX": x}[op]
    B = _probe(y.astype(np.float64), rng, "gaussian")
    r = _engine(cos, tmp_path, [x], body, (), y.shape, B)
    _same(r["d"], y - B, "y")
    d = r["d"]
    ga, gb = {"SUM": (d, F32(0.5) * d), "PROD": (x * d, x * d), "MAX": (np.zeros_like(d), d)}[op]
    _same(r["dx"][0], ga + gb, "dx")


# --------------------------------------------------------------------------- Scale
SCALE_CASES = [  # (bottom shape, scale_param (without bias_term), axis, num_axes)
    ((4, 3, 5, 6), "", 1, 1),
    ((8, 16, 32, 32), "num_axes: 0", 1, 0),  # a scalar over 131072 elements
    ((4, 3, 5, 6), "num_axes: -1", 1, -1),
    ((4, 3, 5, 6), "axis: 2 num_axes: 2", 2, 2),
    ((4, 3, 5, 6), "axis: -1", 3, 1),
    ((4, 3, 5, 6), "axis: 0 num_axes: -1", 0, -1),  # dim = count
    ((7, 33), "", 1, 1),
    ((7, 33), "num_axes: 0", 1, 0),
    ((7, 33), "axis: 0 num_axes: -1", 0, -1),
    ((256, 3), "", 1, 1),  # outer * inner = 256: one product per thread
    ((257, 3), "", 1, 1),  # 257: thread 0 adds two
    ((4, 3, 40, 40), "", 1, 1),  # 6400
]


def scale_body(param, bias, in_place):
    top = "x0" if in_place else "y"
    return (f'layer {{ name: "sc" type: "Scale" bottom: "x0" top: "{top}" scale_param {{ {param} '
            f'bias_term: {str(bias).lower()} }} }}\n'), top


@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in-place"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no-bias"])
@pytest.mark.parametrize("family", ["dyadic", "gaussian"])
@pytest.mark.parametrize("shape,param,axis,num_axes", SCALE_CASES)
def test_scale(cos, tmp_path, shape, param, axis, num_axes, family, bias, in_place):
    rng = np.random.RandomState(int(np.prod(shape)) + axis * 7 + num_axes)
    exact = family == "dyadic"
    view = R.scale_view(shape, axis, num_axes)
    sshape = shape[axis:len(shape) if num_axes == -1 else axis + num_axes]
    # dyadic values of at most top / 8: y is a multiple of 2^-6 and each x * y of 2^-9, so every partial sum of ds
    # is exact while n * max|x * y| stays below 2^24 units of 2^-9
    n = view[0] * view[2]
    top = next(t for t in (4, 2, 1) if n * (t / 8) * (t * t / 64 + t / 8) * 2 ** 9 < 2 ** 24)
    draw = (lambda s: R.dyadic(rng, s, top=top)) if exact else (lambda s: R.gaussian(rng, s))
    x, s = draw(shape), draw(sshape)
    b = draw(sshape) if bias else None
    y64, by = R.scale_forward(x, s, b, view)
    body, top = scale_body(param, bias, in_place)
    r = _engine(cos, tmp_path, [x], body, [s] + ([b] if bias else []), shape, np.zeros(shape, F32), top=top)
    y32 = r["d"]  # B = 0: the probe returns y itself, and the op's top gradient is y
    if exact:
        _equal(y32, y64, "y")
    else:
        _close(y32, y64, by, "y")
    ds, bs, db, bb, dx = R.scale_backward(x, s, y32, view)
    _check(r["grads"][0].ravel(), ds, bs, "ds", exact)
    if bias:
        _check(r["grads"][1].ravel(), db, bb, "db", exact)
    _same(r["dx"][0], dx, "dx")


# --------------------------------------------------------------------------- EuclideanLoss
EUCLID_CASES = [  # (a shape, b shape, loss_weight, staged b, with a top)
    ((4, 5), (4, 5), 1.0, False, True),  # count < 256
    ((8, 32), (8, 32), 0.5, False, True),  # = 256
    ((1, 257), (1, 257), 3.0, False, True),  # 257, num = 1
    ((7, 3, 20, 20), (7, 3, 20, 20), 1.0, False, True),  # 8400, num 7: loss_weight / num rounds
    ((6, 12), (6, 3, 2, 2), 3.0, False, True),  # equal count(1), different shapes
    ((7, 9), (7, 9), 0.5, True, True),  # a staged second bottom
    ((5, 3), (5, 3), 1.0, False, False),  # no top
]


def euclid_body(staged, lw, with_top):
    second = "st" if staged else "x1"
    top = 'top: "l" ' if with_top else ""
    return f'layer {{ name: "loss" type: "EuclideanLoss" bottom: "x0" bottom: "{second}" {top}loss_weight: {lw} }}\n'


@pytest.mark.parametrize("family", ["dyadic", "gaussian"])
@pytest.mark.parametrize("sa,sb,lw,staged,with_top", EUCLID_CASES)
def test_euclidean_loss(cos, tmp_path, sa, sb, lw, staged, with_top, family):
    rng = np.random.RandomState(int(np.prod(sa)) + int(lw * 4))
    draw = (lambda s: R.dyadic(rng, s)) if family == "dyadic" else (lambda s: R.gaussian(rng, s))
    a, b = draw(sa), draw(sb)
    loss, bound = R.euclidean_loss(a, b, lw)
    r = _engine(cos, tmp_path, [a] if staged else [a, b], euclid_body(staged, lw, with_top),
                staged={"st": b} if staged else None)
    assert abs(r["loss"] - loss) <= bound, (r["loss"], loss, bound)
    da, db = R.euclidean_grads32(a, b, lw)
    _same(r["dx"][0], da, "da")
    if not staged:
        _same(r["dx"][1], db, "db")


def test_euclidean_loss_nan_reaches_the_loss(cos, tmp_path):
    rng = np.random.RandomState(11)
    a, b = R.gaussian(rng, (5, 7)), R.gaussian(rng, (5, 7))
    a[2, 3] = np.nan
    r = _engine(cos, tmp_path, [a, b], euclid_body(False, 1.0, True))
    assert np.isnan(r["loss"])
    da, db = R.euclidean_grads32(a, b)
    _same(r["dx"][0], da, "da")
    _same(r["dx"][1], db, "db")


# --------------------------------------------------------------------------- ContrastiveLoss
SIMS = np.array([0, 1, 0.5, 0.999, 1.5, -0.5, 2, -1], F32)  # static_cast<int>: 0 0 0 0 1 0 2 -1


def contrastive_body(margin, legacy, lw=1.0):
    return ('layer { name: "loss" type: "ContrastiveLoss" bottom: "x0" bottom: "x1" bottom: "sim" top: "l" '
            f'loss_weight: {lw} contrastive_loss_param {{ margin: {margin} legacy_version: {str(legacy).lower()} }} }}\n')


def _contrastive_check(cos, tmp_path, a, b, sim, margin, legacy, lw=1.0):
    r = _engine(cos, tmp_path, [a, b], contrastive_body(margin, legacy, lw), staged={"sim": sim})
    loss, da, db, mdist = R.contrastive_loss(a, b, sim, margin, legacy, lw)
    lb, gb, _ = R.contrastive_bounds(a, b, sim, margin, legacy, lw)
    _close(r["dx"][0], da, gb, "da")
    _close(r["dx"][1], db, gb, "db")
    if np.isnan(loss):
        assert np.isnan(r["loss"]), r["loss"]
    else:
        assert abs(r["loss"] - loss) <= lb, (r["loss"], loss, lb)
    return r, mdist


@pytest.mark.parametrize("legacy", [False, True], ids=["sqrt", "legacy"])
@pytest.mark.parametrize("n,c", [(1, 1), (7, 2), (256, 64), (257, 2), (1000, 2), (7, 300), (1000, 64), (257, 1)])
def test_contrastive_loss(cos, tmp_path, n, c, legacy):
    rng = np.random.RandomState(n + c + legacy)
    margin = 1.0 if legacy else 2.0
    sd = np.sqrt(margin / (2 * c)) if legacy else margin / np.sqrt(2 * c)  # dist near the margin: both sides taken
    a, b = R.gaussian(rng, (n, c), sd), R.gaussian(rng, (n, c), sd)
    sim = SIMS[np.arange(n) % SIMS.size]
    _, _, e_md = R.contrastive_bounds(a, b, sim, margin, legacy)
    _, _, _, mdist = R.contrastive_loss(a, b, sim, margin, legacy)
    dissimilar = np.trunc(sim) == 0
    assert np.all(np.abs(mdist[dissimilar]) > e_md[dissimilar]), "a mdist > 0 decision within rounding of the edge"
    _contrastive_check(cos, tmp_path, a, b, sim, margin, legacy, lw=0.5 if n == 7 else 1.0)


@pytest.mark.parametrize("legacy", [False, True], ids=["sqrt", "legacy"])
def test_contrastive_loss_at_the_margin(cos, tmp_path, legacy):
    """Dyadic pairs with mdist exactly 0 (d = (3/8, 4/8): dist_sq 25/64, dist 5/8): no loss and an exact 0 gradient;
    pairs inside and outside the margin around them, every value exact."""
    d = np.array([[0.375, 0.5], [0.25, 0.25], [1.0, 0.5], [0.375, 0.5], [0.0, 0.125]], F32)
    b = np.array([[0.5, -0.25]] * 5, F32)
    a = b + d
    margin = 25 / 64 if legacy else 5 / 8
    sim = np.array([0, 0, 0, 1, 0], F32)
    r, mdist = _contrastive_check(cos, tmp_path, a, b, sim, margin, legacy)
    assert mdist[0] == 0 and mdist[3] == 0 and mdist[1] > 0 > mdist[2]
    assert not r["dx"][0][0].any() and not r["dx"][1][0].any()


def test_contrastive_loss_equal_embeddings(cos, tmp_path):
    """non-legacy dissimilar pairs with a = b: dist 0, beta = -alpha * margin / 1e-4, gradient beta * 0; and one pair
    2^-20 apart, whose gradient shows beta: alpha * (margin - 2^-20) / (2^-20 + 1e-4) * 2^-20"""
    rng = np.random.RandomState(5)
    a = R.gaussian(rng, (6, 4))
    b = a.copy()
    b[4:] = R.gaussian(rng, (2, 4))
    a[2] = [0.5, 0.25, -0.5, 0.125]
    b[2] = a[2]
    b[2, 0] = 0.5 + 2.0 ** -20  # d = -2^-20, exact
    sim = np.array([0, 0, 0, 0, 1, 0], F32)
    r, _ = _contrastive_check(cos, tmp_path, a, b, sim, 1.0, False)
    assert not r["dx"][0][[0, 1, 3]].any() and not r["dx"][1][[0, 1, 3]].any()
    want = (1 / 6) * (1 - 2.0 ** -20) / (2.0 ** -20 + R.EPS_DIST) * 2.0 ** -20
    assert r["dx"][0][2, 0] == pytest.approx(want, rel=1e-5) and r["dx"][1][2, 0] == -r["dx"][0][2, 0]


@pytest.mark.parametrize("legacy", [False, True], ids=["sqrt", "legacy"])
def test_contrastive_loss_non_finite_embeddings(cos, tmp_path, legacy):
    """NaN and +-inf components on similar and dissimilar pairs: a dissimilar pair's NaN reaches the loss and its
    gradient is an exact 0, as is an infinite one's (mdist = -inf); a similar pair passes alpha * d through"""
    rng = np.random.RandomState(6 + legacy)
    a, b = R.gaussian(rng, (8, 3), 0.3), R.gaussian(rng, (8, 3), 0.3)
    sim = np.array([0, 1, 0, 1, 0, 0, 1, 0], F32)
    a[0, 1] = np.nan  # dissimilar, NaN
    a[1, 2] = np.nan  # similar, NaN
    b[2, 0] = np.inf  # dissimilar, inf
    a[3, 0] = -np.inf  # similar, -inf
    r, _ = _contrastive_check(cos, tmp_path, a, b, sim, 1.0, legacy)
    assert np.isnan(r["loss"])
    for g in r["dx"]:
        assert not g[0].any() and not g[2].any(), "a dissimilar pair's gradient is an exact 0"


def test_contrastive_loss_infinite_dissimilar_pair(cos, tmp_path):
    """an infinite dissimilar pair alone: mdist = -inf adds 0, so the loss stays finite, and its gradient is 0"""
    rng = np.random.RandomState(9)
    a, b = R.gaussian(rng, (4, 3), 0.3), R.gaussian(rng, (4, 3), 0.3)
    a[1, 1] = np.inf
    sim = np.array([1, 0, 0, 1], F32)
    for legacy in (False, True):
        r, _ = _contrastive_check(cos, tmp_path, a, b, sim, 1.0, legacy)
        assert np.isfinite(r["loss"])
        assert not r["dx"][0][1].any() and not r["dx"][1][1].any()


# --------------------------------------------------------------------------- BatchNorm and within-channel LRN
BN_SHAPES = [(6, 5), (4, 3, 7), (3, 4, 5, 6), (2, 3, 9, 11)]


@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in-place"])
@pytest.mark.parametrize("global_stats", [False, True], ids=["batch", "global"])
@pytest.mark.parametrize("shape", BN_SHAPES)
def test_batch_norm(cos, tmp_path, shape, global_stats, in_place):
    """The engine's BatchNorm against the restatement of batch_norm_layer.cpp in test_gpu_batch_norm.py, with the
    statistics its kernels save (read back through the kernels' C entry points on the same input): y, the three
    statistics blobs left in the weights and, with global statistics, dx bit for bit.  With batch statistics dx holds
    two channel sums whose fp32 order the restatement does not follow: it is held to the restatement's tolerance and
    must equal the C entry point's dx bit for bit."""
    x, _, blobs = BN._inputs(shape, sum(shape) + global_stats)
    y64 = numpy_bn_forward(x, blobs[0].astype(np.float64), blobs[1].astype(np.float64), float(blobs[2][0]),
                           global_stats=global_stats)[0]
    B = _probe(y64, np.random.RandomState(len(shape)), "gaussian")
    top = "x0" if in_place else "y"
    body = (f'layer {{ name: "bn" type: "BatchNorm" bottom: "x0" top: "{top}" '
            f'batch_norm_param {{ use_global_stats: {str(global_stats).lower()} }} }}\n')
    r = _engine(cos, tmp_path, [x], body, list(blobs), shape, B, top=top)
    d = r["d"]
    _, save, _, dx_c = BN.run_native(x, blobs, global_stats, d)
    save, c = save.cpu().numpy(), shape[1]
    mean, var = save[:c], save[c:]
    if global_stats:
        sf = np.float32(1) / blobs[2][0]
        assert_bits_equal(save, np.concatenate([sf * blobs[0], sf * blobs[1]]), "global statistics")
    wy, wblobs = BN.restate_forward(x, mean, var, blobs, global_stats)
    assert_bits_equal(d, wy - B, "y (through the probe: fl(y - B))")
    for k, what in enumerate(("mean blob", "variance blob", "scale factor")):
        assert_bits_equal(r["data"][k], wblobs[k], what)
    if global_stats:
        assert_bits_equal(r["dx"][0], BN.restate_backward(x, d, mean, var, True), "dx")
    else:
        wdx, _, _ = BN.restate_backward(x, d, mean, var, False)
        np.testing.assert_allclose(r["dx"][0], wdx, rtol=0, atol=2e-6 * (np.abs(wdx).max() + 1e-30))
        assert_bits_equal(r["dx"][0], dx_c.cpu().numpy(), "dx (the C entry point's)")


LRN_CASES = [  # (shape, local_size, alpha, beta)
    ((2, 3, 8, 8), 3, 0.0001, 0.75), ((1, 2, 5, 7), 5, 1.0, 0.75), ((2, 2, 9, 9), 1, 0.5, 0.5),
    ((2, 2, 12, 10), 7, 2.0, 1.25), ((1, 1, 17, 16), 15, 1.0, 0.75),
]


@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in-place"])
@pytest.mark.parametrize("shape,size,alpha,beta", LRN_CASES)
def test_lrn_within_channel(cos, tmp_path, shape, size, alpha, beta, in_place):
    rng = np.random.RandomState(int(np.prod(shape)) + size)
    x = R.gaussian(rng, shape, 3.0)
    y64, mag = lrn_within_ref(x, size, alpha, beta)
    B = _probe(y64, rng, "gaussian")
    top = "x0" if in_place else "y"
    body = (f'layer {{ name: "n" type: "LRN" bottom: "x0" top: "{top}" lrn_param {{ local_size: {size} '
            f'alpha: {alpha} beta: {beta} norm_region: WITHIN_CHANNEL }} }}\n')
    r = _engine(cos, tmp_path, [x], body, (), shape, B, top=top)
    d = r["d"]
    _close(d, y64 - B.astype(np.float64), forward_bound(mag, size, beta) + R.ulp(d) / 2, "y")
    dx64, ma, mb = lrn_within_backward_ref(x, d, size, alpha, beta)
    _close(r["dx"][0], dx64, backward_bound(ma, mb, size, beta), "dx")
