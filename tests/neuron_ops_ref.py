"""Float64 references, with Caffe's rules, of the built-in producer's TanH, ELU, AbsVal, BNLL, Power, Exp, Log,
Threshold, PReLU, Softmax, MultinomialLogisticLoss and HingeLoss ops (DESIGN.md section 14), and per-element error
bounds in producer_ops_ref.py's terms: one rounding (U = 2^-24 relative) per fp32 operation of the kernel, CUDA's
documented maximum ulp errors for tanhf (2), expf (2), logf (1) and powf (4), and the error each input of an operation
carries in, propagated by the operation's derivative.  Where Caffe's formula cancels (BNLL's log(1 + exp(x)) for
x << 0, Log near scale * x + shift = 0, the Softmax sums) the bound is absolute.  No bound is fitted to GPU output."""
import numpy as np

import producer_ops_ref as R
from producer_ops_ref import TINY, U

F32 = np.float32
POWF_ULP = 4  # CUDA C Programming Guide: powf's maximum ulp error
LOG_THRESHOLD = 1e-20  # loss_layer.hpp kLOG_THRESHOLD
BNLL_THRESHOLD = 50.0  # bnll_layer.cu kBNLL_THRESHOLD
PRELU_CHUNK = 8192  # native_producer.cu kPreluChunk


def _f(v):
    return np.asarray(v, np.float64)


def _err(fn):
    with np.errstate(all="ignore"):
        return fn()


# ------------------------------------------------------------------ TanH, ELU, AbsVal, BNLL, Threshold
def tanh(x, dy):
    y = np.tanh(_f(x))
    return y, _f(dy) * (1 - y * y)


def tanh_bounds(x, dy):
    y, dx = tanh(x, dy)
    ey = R.TANHF_ULP * R.ulp(y) + TINY
    return ey, np.abs(_f(dy)) * (2 * np.abs(y) * ey + U * y * y + U * np.abs(1 - y * y)) + U * np.abs(dx) + TINY


def elu(x, dy, alpha):
    x = _f(x)
    y = _err(lambda: np.where(x > 0, x, alpha * np.expm1(x)))
    return y, _err(lambda: np.where(x > 0, _f(dy), _f(dy) * (y + alpha)))


def elu_bounds(x, dy, alpha):
    x = _f(x)
    y, dx = elu(x, dy, alpha)
    e = np.exp(np.minimum(x, 0))
    ey = np.where(x > 0, 0.0, abs(alpha) * (R.EXPF_ULP * R.ulp(e) + U * np.abs(e - 1)) + U * np.abs(y)) + TINY
    edx = np.where(x > 0, 0.0, np.abs(_f(dy)) * (ey + U * np.abs(y + alpha)) + U * np.abs(dx))
    return ey, edx + TINY


def absval(x, dy):
    x = _f(x)
    return np.abs(x), _f(dy) * np.sign(np.nan_to_num(x))  # sign(0) = sign(NaN) = 0


def bnll(x, dy):
    x = _f(x)
    y = _err(lambda: np.where(x > 0, x + np.log1p(np.exp(-x)), np.log1p(np.exp(x))))
    e = _err(lambda: np.exp(np.where(np.isnan(x), BNLL_THRESHOLD, np.minimum(x, BNLL_THRESHOLD))))
    return y, _err(lambda: _f(dy) * e / (e + 1))


def bnll_bounds(x, dy):
    """y: the exp's 2 ulp and the rounding of 1 + e reach the log as a relative error of its argument, which the log
    turns into an absolute one; then the log's ulp and the rounding of x + log.  dx: 4U for e (it cancels to first
    order in e / (e + 1), but not beyond), three roundings."""
    x = _f(x)
    y, dx = bnll(x, dy)
    e = np.exp(-np.abs(x))
    ey = (R.EXPF_ULP * R.ulp(e) + U * (1 + e)) / (1 + e) + R.LOGF_ULP * R.ulp(np.log1p(e)) + U * np.abs(y)
    return ey + TINY, 8 * U * np.abs(dx) + TINY


def threshold(x, t):
    return (_f(x) > t).astype(np.float64)


# ------------------------------------------------------------------ Power, Exp, Log
def _scale_shift(x, scale, shift):
    return _f(x) * scale + shift


def power(x, dy, p, scale, shift):
    """power_layer.cpp: the constant shift^p (1 for p = 0) when p * scale == 0, with dx = 0 exactly; else
    v^p with v = shift + scale x, and dx = dy * p scale v^(p-1), which Caffe's shift == 0 branch (p y / x) makes NaN at
    x = 0 for any p other than 1 and 2."""
    x, dy = _f(x), _f(dy)
    ds = F32(F32(p) * F32(scale))
    if ds == 0:
        return np.full(x.shape, 1.0 if p == 0 else float(F32(F32(shift) ** F32(p)))), np.zeros(x.shape)
    v = _scale_shift(x, scale, shift)
    y = _err(lambda: v ** p)
    if p == 1:
        return y, dy * float(ds)
    if p == 2:
        return y, dy * 2 * scale * v
    g = _err(lambda: p * scale * v ** (p - 1))
    if shift == 0:
        g = np.where(x == 0, np.nan, g)
    return y, _err(lambda: dy * g)


def power_bounds(x, dy, p, scale, shift):
    x = _f(x)
    y, dx = power(x, dy, p, scale, shift)
    if F32(p) * F32(scale) == 0:
        return np.zeros(x.shape), np.zeros(x.shape)
    v = _scale_shift(x, scale, shift)
    ev = U * np.abs(scale * x) + U * np.abs(v)  # the two roundings of v
    with np.errstate(all="ignore"):
        rel_v = np.where(v != 0, ev / np.abs(v), 0.0)
        ey = np.abs(p) * np.abs(y) * rel_v + (POWF_ULP * R.ulp(y) if p != 1 else 0) + TINY
        rel_y = np.where(y != 0, ey / np.abs(y), 0.0)
        if p == 2:  # (ds scale) x + ds shift: four roundings of terms bounded by |2 scale v| scale terms
            edx = np.abs(_f(dy)) * 2 * abs(scale) * (3 * U * np.abs(scale * x) + 2 * U * abs(shift)) + U * np.abs(dx)
        else:
            edx = np.abs(dx) * (rel_y + rel_v + 6 * U)
    return ey, np.where(np.isnan(dx), 0.0, edx) + TINY


def exp_consts(base, scale, shift):
    """exp_layer.cpp LayerSetUp in float: inner = log(base) scale, outer = base^shift (e^shift for base -1)."""
    log_base = F32(1) if base == -1 else F32(np.log(F32(base)))
    inner = F32(log_base * F32(scale))
    outer = F32(1) if shift == 0 else F32(np.exp(F32(shift))) if base == -1 else F32(F32(base) ** F32(shift))
    return float(inner), float(outer)


def exp_(x, dy, base, scale, shift):
    inner, outer = exp_consts(base, scale, shift)
    y = _err(lambda: outer * np.exp(inner * _f(x)))
    return y, _err(lambda: _f(dy) * y * inner)


def exp_bounds(x, dy, base, scale, shift):
    inner, _ = exp_consts(base, scale, shift)
    y, dx = exp_(x, dy, base, scale, shift)
    with np.errstate(all="ignore"):
        rel = U * np.abs(inner * _f(x)) + 2 * R.EXPF_ULP * U + 2 * U  # the exponent's rounding, expf, the outer product
        return np.abs(y) * rel + TINY, np.abs(dx) * (rel + 3 * U) + TINY


def log_consts(base, scale):
    log_base = F32(1) if base == -1 else F32(np.log(F32(base)))
    return float(F32(F32(1) / log_base)), float(F32(F32(scale) / log_base))


def log_(x, dy, base, scale, shift):
    base_scale, num_scale = log_consts(base, scale)
    v = _scale_shift(x, scale, shift)
    return _err(lambda: base_scale * np.log(v)), _err(lambda: _f(dy) * num_scale / v)


def log_bounds(x, dy, base, scale, shift):
    """Absolute near v = scale x + shift = 0: the roundings of v reach the log as ev / |v|."""
    base_scale, _ = log_consts(base, scale)
    y, dx = log_(x, dy, base, scale, shift)
    v = _scale_shift(x, scale, shift)
    ev = U * np.abs(scale * _f(x)) + U * np.abs(v)
    with np.errstate(all="ignore"):
        rel_v = ev / np.abs(v)
        ey = abs(base_scale) * (rel_v + R.LOGF_ULP * R.ulp(np.log(v))) + 2 * U * np.abs(y)
        return ey + TINY, np.abs(dx) * (rel_v + 4 * U) + TINY


# ------------------------------------------------------------------ PReLU (prelu_layer.cpp)
def prelu(x, a, dy, shared):
    """-> y, dx, da for x [N, C, ...] and slopes a [C] (or one, shared)."""
    x, dy = _f(x), _f(dy)
    ab = np.full(x.shape, float(np.ravel(a)[0])) if shared else \
        np.broadcast_to(_f(a).reshape((1, -1) + (1,) * (x.ndim - 2)), x.shape)
    y = np.maximum(x, 0) + ab * np.minimum(x, 0)
    dx = dy * np.where(x > 0, 1.0, ab)
    t = dy * x * (x <= 0)
    da = np.array([t.sum()]) if shared else t.sum(axis=tuple(i for i in range(x.ndim) if i != 1))
    return y, dx, da


def prelu_bounds(x, a, dy, shared):
    y, dx, _ = prelu(x, a, dy, shared)
    _, _, ada = prelu(-np.abs(_f(x)) * (_f(x) <= 0), a, np.abs(_f(dy)), shared)  # sum |dy x| over x <= 0
    ada = np.abs(ada)
    m = x.size if shared else x.size // x.shape[1]
    chunks = -(-m // PRELU_CHUNK)
    k = -(-min(m, PRELU_CHUNK) // R.BLOCK) + 8 + chunks + 2  # the product, a thread's run, the tree, the chunks, the add
    return U * np.abs(y) + TINY, U * np.abs(dx) + TINY, k * U * ada + TINY


# ------------------------------------------------------------------ Softmax (softmax_layer.cu)
def _axis_view(x, axis):
    return np.moveaxis(_f(x), axis, -1)


def softmax(x, dy, axis):
    xs, dys = _axis_view(x, axis), _axis_view(dy, axis)
    with np.errstate(all="ignore"):
        e = np.exp(xs - xs.max(axis=-1, keepdims=True))
        y = e / e.sum(axis=-1, keepdims=True)
        dx = (dys - (dys * y).sum(axis=-1, keepdims=True)) * y
    return np.moveaxis(y, -1, axis), np.moveaxis(dx, -1, axis)


def softmax_bounds(x, dy, axis):
    """y: each e carries the rounding of x - max (U |x - max|, relative after the exp) and expf's 2 ulp; the sum C
    roundings; the quotient one.  dx: the dot's C products and C sums plus every y's own error times |dy|, the
    difference one rounding, the product one, and y's error times |dy - dot|: absolute, for the sums cancel."""
    xs, dys = _axis_view(x, axis), _axis_view(dy, axis)
    c = xs.shape[-1]
    y, dx = (np.moveaxis(v, axis, -1) for v in softmax(x, dy, axis))
    with np.errstate(all="ignore"):
        rel_e = U * np.abs(xs - xs.max(axis=-1, keepdims=True)) + 2 * R.EXPF_ULP * U
        rel = rel_e + rel_e.max(axis=-1, keepdims=True) + (c + 1) * U
        ey = y * rel + TINY
        dot = (dys * y).sum(axis=-1, keepdims=True)
        edot = (np.abs(dys) * ey).sum(axis=-1, keepdims=True) + 2 * c * U * (np.abs(dys) * y).sum(axis=-1,
                                                                                                  keepdims=True)
        diff = np.abs(dys - dot)
        edx = diff * ey + y * (edot + U * diff) + U * np.abs(dx) + TINY
    return np.moveaxis(ey, -1, axis), np.moveaxis(edx, -1, axis)


# ------------------------------------------------------------------ MultinomialLogisticLoss, HingeLoss
def _rows(x):
    x = _f(x)
    return x.reshape(x.shape[0], -1)


def mll(x, label, loss_weight=1.0):
    """-> (loss, dx): -lw sum log(max(p_label, 1e-20)) / num; dx = -lw / num / max(p_label, 1e-20) at the label."""
    x2 = _rows(x)
    num = x2.shape[0]
    lab = np.asarray(label).astype(np.int64).ravel()
    p = np.maximum(x2[np.arange(num), lab], LOG_THRESHOLD)
    dx = np.zeros_like(x2)
    dx[np.arange(num), lab] = float(F32(-loss_weight) / F32(num)) / p
    return -loss_weight * float(np.log(p).sum()) / num, dx.reshape(np.shape(x))


def mll_bounds(x, label, loss_weight=1.0):
    x2 = _rows(x)
    num = x2.shape[0]
    lab = np.asarray(label).astype(np.int64).ravel()
    logs = np.abs(np.log(np.maximum(x2[np.arange(num), lab], LOG_THRESHOLD)))
    run = -(-num // R.BLOCK) + 8 + 2
    _, dx = mll(x, label, loss_weight)
    return abs(loss_weight) / num * (R.ulp(logs).sum() + run * U * logs.sum()) + TINY, 2 * U * np.abs(dx) + TINY


def _hinge_h(x, label):
    x2 = _rows(x)
    at = np.zeros(x2.shape, bool)
    at[np.arange(x2.shape[0]), np.asarray(label).astype(np.int64).ravel()] = True
    with np.errstate(invalid="ignore"):
        t = 1 + np.where(at, -x2, x2)
        return np.where(t > 0, t, 0.0), at  # std::max(0, t): a NaN gives 0


def hinge(x, label, norm="L1", loss_weight=1.0):
    h, at = _hinge_h(x, label)
    num = h.shape[0]
    g = np.where(at, -h, h)
    if norm == "L1":
        return loss_weight * h.sum() / num, (np.sign(g) * float(F32(loss_weight) / F32(num))).reshape(np.shape(x))
    return loss_weight * (h * h).sum() / num, (g * float(F32(F32(loss_weight) * 2) / F32(num))).reshape(np.shape(x))


def hinge_bounds(x, label, norm="L1", loss_weight=1.0):
    h, _ = _hinge_h(x, label)
    num, count = h.shape[0], h.size
    blocks = max(1, min(-(-count // R.BLOCK), 132 * 16))
    run = -(-count // (blocks * R.BLOCK)) + 8 + blocks + 2
    terms = h if norm == "L1" else h * h
    elem = U * h if norm == "L1" else 3 * U * h * h  # h's rounding (doubled by the square), the square's
    _, dx = hinge(x, label, norm, loss_weight)
    lb = abs(loss_weight) / num * (elem.sum() + run * U * (terms.sum() + elem.sum())) + TINY
    return lb, (0 if norm == "L1" else 4 * U) * np.abs(dx) + TINY
