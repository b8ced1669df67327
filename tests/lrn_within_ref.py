"""Float64 reference of the within-channel LRN kernels (csrc/caffe_layers.cu, DESIGN.md section 10), numpy only.

`composition` is Caffe's WITHIN_CHANNEL layer as lrn_layer.cpp builds it, five layers evaluated one after another:
split, square, AVE pool (n x n, pad (n-1)/2, stride 1, divisor counting the pad cells), power (shift 1, scale alpha,
power -beta), product.  `lrn_within_ref` / `lrn_within_backward_ref` state the same function and its gradient as the
DESIGN section 10 formulas, with the per-element magnitudes the kernels' error bounds are stated in.
"""
import numpy as np

from layer_ref import C_POW, TINY, U

SIZES = list(range(1, 16, 2))


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _alpha(alpha):
    return float(np.float32(alpha))  # the kernels get alpha as an fp32 argument


def window_sum(a, half):
    """sum over the (2 half + 1)^2 window centred on every (h, w) of the last two axes, zero outside the plane"""
    h, w = a.shape[-2:]
    p = np.zeros(a.shape[:-2] + (h + 2 * half, w + 2 * half), a.dtype)
    p[..., half:half + h, half:half + w] = a
    out = np.zeros_like(a)
    for i in range(2 * half + 1):
        for j in range(2 * half + 1):
            out += p[..., i:i + h, j:j + w]
    return out


def composition(x, size, alpha, beta):
    """Caffe's five-layer WITHIN_CHANNEL composition in float64 on the fp32 input."""
    x = _f64(x)
    pad = (size - 1) // 2
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        sq = x * x                                                          # split + square
        h, w = x.shape[-2:]
        padded = np.zeros(x.shape[:-2] + (h + 2 * pad, w + 2 * pad))
        padded[..., pad:pad + h, pad:pad + w] = sq
        pooled = np.zeros_like(x)                                           # AVE pool, stride 1
        for ph in range(h):
            for pw in range(w):
                hs, ws = ph, pw  # window start in the padded plane
                he, we = min(hs + size, h + 2 * pad), min(ws + size, w + 2 * pad)
                pool_size = (he - hs) * (we - ws)  # pooling_layer.cpp: counted before clipping to the plane
                pooled[..., ph, pw] = padded[..., hs:he, ws:we].sum(axis=(-2, -1)) / pool_size
        power = np.power(1.0 + _alpha(alpha) * pooled, -beta)               # power
        return x * power                                                    # product


def _scale(x, size, alpha):
    return 1.0 + _alpha(alpha) * window_sum(x * x, size // 2) / (size * size)


def lrn_within_ref(x, size, alpha, beta):
    """-> (y, |y|) in float64: y = x s^-beta, s = 1 + alpha/n^2 sum_window x^2"""
    x = _f64(x)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        y = x * np.power(_scale(x, size, alpha), -beta)
    return y, np.abs(y)


def lrn_within_backward_ref(x, dy, size, alpha, beta):
    """-> (dx, |dy s^-beta|, coef |x| sum_window |r|) in float64, r_j = dy_j x_j s_j^-beta / s_j,
    coef = 2 alpha beta / n^2; dx is the difference of the two terms, so both magnitudes are returned."""
    x, dy = _f64(x), _f64(dy)
    half, coef = size // 2, 2.0 * _alpha(alpha) * beta / (size * size)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        s = _scale(x, size, alpha)
        sb = np.power(s, -beta)
        r = dy * x * sb / s
        a = dy * sb
        b = coef * x * window_sum(r, half)
        return a - b, np.abs(a), np.abs(coef * x) * window_sum(np.abs(r), half)


def forward_coefficient(size, beta):
    """c with |y - y64| <= c u |y64| + TINY.  In units of u, first order: S is a sum of n^2 rounded squares, n per
    row and then n rows, so 1 + 2(n - 1) relative (every term >= 0); S / n^2 1; fma(alpha, A, 1) 1 (alpha A >= 0);
    +1 of slack gives s within 2n + 2.  powf(s, -beta) scales that by |beta| and adds C_POW; the multiply by x 1,
    +1 of slack."""
    return abs(beta) * (2 * size + 2) + C_POW + 2


def forward_bound(mag, size, beta):
    return forward_coefficient(size, beta) * U * mag + TINY


def backward_bound(mag_dy, mag_win, size, beta):
    """|dx - dx64| <= u (c_a |dy s^-beta| + c_b coef |x| sum |r|) + (4 n^2 + 16) TINY.  c_a: s^-beta as in the
    forward, times dy 1, the final fma 1.  c_b: r = fl(fl(fl(dy x) s^-beta) / s) carries s^-beta's error, s's own
    2n + 2 and 3 roundings; the window sum of n^2 terms (n per row, then n rows) 2(n - 1); coef = fl(fl(2 alpha beta)
    / n^2) 2; coef x 1; the final fma 1; +1 of slack."""
    base = abs(beta) * (2 * size + 2) + C_POW
    c_a = base + 2
    c_b = base + (2 * size + 2) + 3 + 2 * (size - 1) + 2 + 1 + 1 + 1
    return U * (c_a * mag_dy + c_b * mag_win) + (4 * size * size + 16) * TINY


def value_class(a):
    """0 finite, 1 NaN, 2 +Inf, 3 -Inf"""
    a = np.asarray(a, np.float64)
    return np.where(np.isnan(a), 1, np.where(np.isposinf(a), 2, np.where(np.isneginf(a), 3, 0)))
