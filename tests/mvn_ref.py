"""References for Caffe's MVN layer (mvn_layer.cu) on the built-in engine (DESIGN.md section 14).

- forward / backward: float64, in the layer's own terms (rows of a legacy 4-D blob), with Caffe's backward formula
  dx = (dy - (y * sum(y dy) + sum(dy)) / dim) / s, which is the exact derivative only where s >> eps.
- forward32 / backward32: the kernels' fp32 element operations, one rounding each, given their row sums; from the
  kernels' own sums they must reproduce y and dx bit for bit.
- bound_y / bound_dx: per-element first-order bounds (n + extra) * 2^-24 * sum|.| on the fp32 result's distance from
  float64, from the operation count: a row sum of n terms carries at most (n - 1) roundings of its partial sums'
  magnitudes whatever its order, each element operation one more.
- MUTATIONS: plausible wrong layers.  Each must fall outside the bounds (or fail the hand-worked case or the shape).
"""
import numpy as np

F32 = np.float32
U = 2.0 ** -24
MUTATIONS = ("eps_in_sqrt", "unbiased_var", "drop_y_term", "per_sample_rows", "bottom_shape_top")


def legacy_shape(shape):
    assert len(shape) <= 4
    return tuple(shape) + (1,) * (4 - len(shape))


def rows_dim(shape, across_channels, mutation=None):
    n, c = legacy_shape(shape)[:2]
    rows = n * (1 if across_channels or mutation == "per_sample_rows" else c)
    return rows, int(np.prod(shape)) // rows


def forward(x, normalize_variance=True, across_channels=False, eps=1e-9, mutation=None):
    """float64 -> (y in the top's shape, s per row [rows, 1] or None)."""
    rows, dim = rows_dim(x.shape, across_channels, mutation)
    xr = np.asarray(x, np.float64).reshape(rows, dim)
    y = xr - xr.mean(1, keepdims=True)
    s = None
    if normalize_variance:
        var = (y * y).sum(1, keepdims=True) / (dim - 1 if mutation == "unbiased_var" and dim > 1 else dim)
        s = np.sqrt(var + eps) if mutation == "eps_in_sqrt" else np.sqrt(var) + eps
        y = y / s
    shape = x.shape if mutation == "bottom_shape_top" else legacy_shape(x.shape)
    return y.reshape(shape), s


def backward(y, dy, s, across_channels=False, mutation=None):
    """float64 Caffe formula: dx [rows, dim] from the top y and its gradient dy (any shape of the same count)."""
    rows, dim = rows_dim(y.shape, across_channels, mutation)
    yr = np.asarray(y, np.float64).reshape(rows, dim)
    g = np.asarray(dy, np.float64).reshape(rows, dim)
    if s is None:
        return g - g.mean(1, keepdims=True)
    a = (yr * g).sum(1, keepdims=True)
    if mutation == "drop_y_term":
        a = 0 * a
    return (g - (yr * a + g.sum(1, keepdims=True)) / dim) / s


def forward32(x2, sx, syy, normalize_variance, eps, powf_half):
    """The kernels' fp32 forward of rows x2 [rows, dim] from their row sums sx, syy [rows]; powf_half(v) is glibc's
    powf(v, 0.5f) -> (y, s)."""
    rows, dim = x2.shape
    alpha = F32(1.0 / dim)
    mu = (sx.astype(F32) * alpha)[:, None]
    d = (x2.astype(F32) - mu).astype(F32)
    if not normalize_variance:
        return d, np.ones(rows, F32)
    var = (syy.astype(F32) * alpha).astype(F32)
    s = (np.array([powf_half(v) for v in var], F32) + F32(eps)).astype(F32)
    return (d / s[:, None]).astype(F32), s


def backward32(y2, dy2, a, b, s, normalize_variance):
    """The kernels' fp32 dx from y, dy [rows, dim] and their row sums a = sum(y dy), b = sum(dy) and s [rows]."""
    dim = y2.shape[1]
    if not normalize_variance:
        return (dy2 - (b.astype(F32) * F32(1.0 / dim))[:, None]).astype(F32)
    c = F32(-1.0 / dim)
    t = (y2 * a.astype(F32)[:, None]).astype(F32)
    t = (t + b.astype(F32)[:, None]).astype(F32)
    t = (c * t).astype(F32)
    t = (dy2 + t).astype(F32)
    return (t / s.astype(F32)[:, None]).astype(F32)


def sequential32(x2, normalize_variance=True, eps=1e-9, powf_half=None):
    """The fp32 forward with its row sums taken left to right (an order the kernels may use; the bounds hold for any)."""
    x2 = x2.astype(F32)
    sx = np.add.accumulate(x2, axis=1, dtype=F32)[:, -1]
    mu = (sx * F32(1.0 / x2.shape[1])).astype(F32)
    d = (x2 - mu[:, None]).astype(F32)
    syy = np.add.accumulate((d * d).astype(F32), axis=1, dtype=F32)[:, -1]
    powf_half = powf_half or (lambda v: np.sqrt(np.float64(v)))
    return forward32(x2, sx, syy, normalize_variance, eps, powf_half)


def bound_y(x2, y64, s64):
    """|y32 - y64| per element of rows x2 [rows, dim]: mu's sum ((dim + 2) roundings of sum|x|), x - mu, and s's
    relative error (dim + 6) u from the sum of squares, the scaling, powf, eps and the division."""
    dim = x2.shape[1]
    x2 = np.asarray(x2, np.float64)
    y2 = np.asarray(y64, np.float64).reshape(x2.shape)
    mean_abs = np.abs(x2).sum(1, keepdims=True) / dim
    dev = np.abs(x2 - x2.mean(1, keepdims=True))
    s = 1.0 if s64 is None else s64
    out = U * ((dim + 2) * mean_abs + dev) / s
    if s64 is not None:
        out = out + U * (dim + 6) * np.abs(y2)
    return out


def bound_dx(y2, dy2, s64, by):
    """|dx32 - dx64| per element, from y32's bound `by`, the row sums A and B ((dim + 2) roundings of their sums of
    magnitudes), the element operations and s's relative error."""
    dim = y2.shape[1]
    y2, g = np.asarray(y2, np.float64), np.asarray(dy2, np.float64)
    sum_g = np.abs(g).sum(1, keepdims=True)
    if s64 is None:
        return U * ((dim + 2) * sum_g / dim + np.abs(g))
    sum_yg = np.abs(y2 * g).sum(1, keepdims=True)
    a = (y2 * g).sum(1, keepdims=True)
    by = np.asarray(by, np.float64).reshape(y2.shape)
    carried = (by * np.abs(a) + np.abs(y2) * (by * np.abs(g)).sum(1, keepdims=True)) / dim
    rounding = U * ((dim + 4) * (np.abs(y2) * sum_yg + sum_g) / dim + 3 * np.abs(g))
    dx = (g - (y2 * a + g.sum(1, keepdims=True)) / dim) / s64
    return (rounding + carried) / s64 + U * (dim + 6) * np.abs(dx)


def glibc_powf_half():
    """glibc's powf(v, 0.5f) (the kernels' copy is powf_half.h), for forward32."""
    import ctypes
    f = ctypes.CDLL("libm.so.6").powf
    f.restype, f.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    return lambda v: F32(f(float(v), 0.5))
