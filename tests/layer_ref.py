"""Independent references of the native producer layers (csrc/caffe_layers.cu, DESIGN.md section 10), numpy only.

* LRN: the DESIGN section 10 formulas evaluated in float64 on the fp32 inputs, with the per-element magnitudes the
  kernels' error bounds are stated in (`lrn_forward_bound`, `lrn_backward_bound`).
* bias + ReLU + MAX pool: an exact float32 restatement of the documented semantics (v = fl32(x + b), first maximum
  by strict >, NaN always taken, y = +0.0 and index 255 when no gradient flows, dx gathered from 0.0f over windows in
  (ph, pw) order), so y, index and dx can be compared bit for bit; dbias in float64 with sum |routed dy| for its bound.

tests/test_layer_ref_host.py checks these against PyTorch on the CPU.
"""
from collections import namedtuple

import numpy as np

U = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)
# powf: 4 ulp maximum error over its full range (CUDA C++ Programming Guide, "Mathematical Functions" appendix, table
# of single-precision standard library functions with maximum ulp error).  One ulp of a normal fp32 result r is at
# most 2u|r|, so in units of u relative to the result that is 8.
C_POW = 8.0
TINY = 2.0 ** -149  # the smallest fp32 subnormal: the absolute error a result that underflows may carry


LRN_SIZES = list(range(1, 16, 2))
LRN_KS = [1.0, 2.0, 1e-3]
LRN_BETAS = [0.75, 0.5, 1.0, 2.0, 0.0, -0.5]


def _window_sum(a, half):
    """sum over c' in [c - half, c + half] along axis 1, zero outside [0, C)"""
    c = a.shape[1]
    p = np.zeros((a.shape[0], c + 2 * half) + a.shape[2:], a.dtype)
    p[:, half:half + c] = a
    out = np.zeros_like(a)
    for j in range(2 * half + 1):
        out += p[:, j:j + c]
    return out


def _lrn_scale(x, size, alpha, k):
    return k + (alpha / size) * _window_sum(x * x, size // 2)


def lrn_ref(x, size, alpha, beta, k):
    """-> (y, |y|) in float64 for fp32 x (N, C, ...): y_c = x_c * s_c^-beta, s_c = k + alpha/n * sum x_c'^2"""
    x = np.asarray(x, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        y = x * np.power(_lrn_scale(x, size, alpha, k), -beta)
    return y, np.abs(y)


def lrn_backward_ref(x, dy, size, alpha, beta, k):
    """-> (dx, |dy s^-beta|, coef |x| sum_window |r|) in float64, r_c' = dy_c' x_c' s_c'^(-beta-1),
    coef = 2 alpha beta / n.  dx is the difference of the two terms; both magnitudes are returned because it can
    cancel."""
    x = np.asarray(x, np.float32).astype(np.float64)
    dy = np.asarray(dy, np.float32).astype(np.float64)
    half, coef = size // 2, 2.0 * alpha * beta / size
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        s = _lrn_scale(x, size, alpha, k)
        sb = np.power(s, -beta)
        r = dy * x * sb / s
        a = dy * sb
        b = coef * x * _window_sum(r, half)
        return a - b, np.abs(a), np.abs(coef * x) * _window_sum(np.abs(r), half)


def lrn_forward_coefficient(size, beta):
    """c with |y - y64| <= c u |y64| + TINY.  In units of u, first order: s = fl(k + fl(fl(alpha/n) * ss)) with ss
    a sequential sum of 2h+1 rounded squares is off by (2h+1) + 3 relative (no cancellation: every term is >= 0),
    +1 of slack; powf(s, -beta) scales that by |beta| and adds its own C_POW; the final multiply 1, +1 of slack."""
    return abs(beta) * (2 * (size // 2) + 5) + C_POW + 2


def lrn_forward_bound(mag, size, beta):
    return lrn_forward_coefficient(size, beta) * U * mag + TINY


def lrn_backward_bound(mag_dy, mag_win, size, beta):
    """|dx - dx64| <= u (c_a |dy s^-beta| + c_b coef |x| sum |r|) + 16 TINY, the forward's construction applied to
    each term.  c_a: s^-beta as in the forward, times dy (1), the final subtraction (1).  c_b: r = fl(fl(fl(dy x)
    s^-beta) / s) carries s^-beta's error, s's own (2h+5) and 3 roundings; the window sum of 2h+1 r's adds 2h;
    coef = fl(fl(2 alpha beta) / n) 2; fl(fl(coef x) acc) 2; the final subtraction 1, +1 of slack."""
    h = size // 2
    base = abs(beta) * (2 * h + 5) + C_POW
    c_a = base + 2
    c_b = base + (2 * h + 5) + 3 + 2 * h + 2 + 2 + 2
    return U * (c_a * mag_dy + c_b * mag_win) + 16 * TINY


MUTATIONS = ("window_n_minus_2", "k_is_1", "channel_shift")


def mutated_lrn_refs(x, dy, size, alpha, beta, k, which):
    """-> (y, dx) of the reference under one of MUTATIONS: the window shrunk to n - 2 channels (alpha/n kept),
    k replaced by 1, or the output channels shifted by one"""
    if which == "window_n_minus_2":
        args = (size - 2, alpha * (size - 2) / size, beta, k)
    elif which == "k_is_1":
        args = (size, alpha, beta, 1.0)
    else:
        args = (size, alpha, beta, k)
    y, _ = lrn_ref(x, *args)
    dx, _, _ = lrn_backward_ref(x, dy, *args)
    if which == "channel_shift":
        y, dx = np.roll(y, 1, axis=1), np.roll(dx, 1, axis=1)
    return y, dx


def outside_fraction(y, dx, x, dy, size, alpha, beta, k):
    """-> (fraction of y, fraction of dx) elements outside the kernels' bound around the float64 reference"""
    y64, ymag = lrn_ref(x, size, alpha, beta, k)
    dx64, ma, mb = lrn_backward_ref(x, dy, size, alpha, beta, k)
    fy = np.mean(~(np.abs(y - y64) <= lrn_forward_bound(ymag, size, beta)))
    fdx = np.mean(~(np.abs(dx - dx64) <= lrn_backward_bound(ma, mb, size, beta)))
    return fy, fdx


def value_class(a):
    """0 NaN, 1 +Inf, 2 -Inf, 3 zero, 4 finite non-zero"""
    a = np.asarray(a)
    return np.select([np.isnan(a), a == np.inf, a == -np.inf, a == 0], [0, 1, 2, 3], 4)


def lrn_inputs(shape, alpha, k, seed, low=-3.0, high=2.0):
    """-> fp32 (x, dy).  x has both signs and a per-pixel scale, log-uniform, such that the window term
    (alpha/n) sum x^2 spans about 10^low .. 10^high times k: the window stays visible next to k, so a wrong halo or
    a wrong k shows."""
    rng = np.random.default_rng(seed)
    scale = np.sqrt(k * 10.0 ** rng.uniform(low, high, (shape[0], 1) + tuple(shape[2:])) / alpha)
    x = (rng.standard_normal(shape, dtype=np.float32) * scale).astype(np.float32)
    return x, rng.standard_normal(shape, dtype=np.float32)


def pooled_size(n, kernel, stride):
    """ceil mode, pad 0, the last window starting inside the input"""
    out = -(-(n - kernel) // stride) + 1
    return out - 1 if (out - 1) * stride >= n else out


NO_GRAD = 255
POOL_VALUE_KINDS = ("randn", "rounding_ties", "bias_ties", "negative", "negative_zero", "nan", "inf")


def pool_inputs(kind, shape, seed):
    """-> fp32 (x, b) for the pool block:
    randn          x ~ N(0, 1), b ~ 0.3 N(0, 1)
    rounding_ties  x = round(2 N(0, 1)) / 2, b in {-0.5, 0, 0.5}: equal values and exact zeros
    bias_ties      b = 2^23 (1 + c mod 3) and x ~ 2 N(0, 1): distinct x that only tie after fl32(x + b)
    negative       x = -|N(0, 1)| with 3 % of it positive: all-negative windows next to passing ones
    negative_zero  x = b = -0.0 everywhere
    nan            randn with 5 % NaN, and two NaNs in the first window of every plane
    inf            randn with 5 % +Inf and 5 % -Inf"""
    rng = np.random.default_rng(seed)
    n, c, h, w = shape
    x = rng.standard_normal(shape, dtype=np.float32)
    b = (0.3 * rng.standard_normal(c)).astype(np.float32)
    u = rng.random(shape)
    if kind == "rounding_ties":
        x = np.round(2 * x) / np.float32(2)
        b = rng.integers(-1, 2, c).astype(np.float32) / np.float32(2)
    elif kind == "bias_ties":
        x = 2 * x
        b = np.float32(2.0 ** 23) * (1 + np.arange(c) % 3).astype(np.float32)
    elif kind == "negative":
        x = np.where(u < 0.03, np.abs(x), -np.abs(x))
        b = np.zeros(c, np.float32)
    elif kind == "negative_zero":
        x = np.full(shape, -0.0, np.float32)
        b = np.full(c, -0.0, np.float32)
    elif kind == "nan":
        x = np.where(u < 0.05, np.float32(np.nan), x)
        x[:, :, 0, 0] = np.nan
        x[:, :, min(1, h - 1), min(1, w - 1)] = np.nan
    elif kind == "inf":
        x = np.where(u < 0.05, np.float32(np.inf), np.where(u > 0.95, np.float32(-np.inf), x))
    elif kind != "randn":
        raise ValueError(kind)
    return x.astype(np.float32), b


PoolRef = namedtuple("PoolRef", "y index dx dbias dbias_abs")


def pool_ref(x, b, kernel, stride, dy=None):
    """bias + ReLU + MAX pool of fp32 x (N, C, H, W) and fp32 b (C,): -> PoolRef.  y, index and dx are the exact
    fp32 values the documented algorithm produces; dbias (float64 sum of the routed dy) and dbias_abs (sum of their
    magnitudes) are None without dy."""
    x = np.asarray(x, np.float32)
    n, c, h, w = x.shape
    ph_n, pw_n = pooled_size(h, kernel, stride), pooled_size(w, kernel, stride)
    v = x + np.asarray(b, np.float32).reshape(1, c, 1, 1)  # fp32 + fp32: one rounding
    vmax = np.full((n, c, ph_n, pw_n), -np.inf, np.float32)
    pos = np.zeros((n, c, ph_n, pw_n), np.int64)
    ph, pw = np.arange(ph_n), np.arange(pw_n)
    with np.errstate(invalid="ignore"):
        for dh in range(kernel):
            rows = ph * stride + dh
            for dw in range(kernel):
                cols = pw * stride + dw
                inside = (rows < h)[:, None] & (cols < w)[None, :]
                cand = v[:, :, np.minimum(rows, h - 1)[:, None], np.minimum(cols, w - 1)[None, :]]
                take = inside & ((cand > vmax) | np.isnan(cand))
                vmax = np.where(take, cand, vmax)
                pos = np.where(take, dh * kernel + dw, pos)
        flows = (vmax > 0) | np.isnan(vmax)
    y = np.where(flows, vmax, np.float32(0.0))
    index = np.where(flows, pos, NO_GRAD).astype(np.uint8)
    if dy is None:
        return PoolRef(y, index, None, None, None)

    dy = np.asarray(dy, np.float32)
    planes = n * c
    idx = index.reshape(planes, ph_n, pw_n).astype(np.int64)
    g = dy.reshape(planes, ph_n, pw_n)
    dx = np.zeros((planes, h * w), np.float32)
    rows_of = np.arange(planes)
    for a in range(ph_n):  # each element receives its windows' dy in (ph, pw) order, summed in fp32 from 0.0f
        for bw in range(pw_n):
            i = idx[:, a, bw]
            ok = i != NO_GRAD
            e = (a * stride + i // kernel) * w + bw * stride + i % kernel
            dx[rows_of[ok], e[ok]] += g[ok, a, bw]
    routed = np.where(index != NO_GRAD, dy, np.float32(0.0)).astype(np.float64)
    return PoolRef(y, index, dx.reshape(n, c, h, w), routed.sum(axis=(0, 2, 3)),
                   np.abs(routed).sum(axis=(0, 2, 3)))


# every kernel 1..15 with every stride 1..kernel+2
POOL_GEOMETRIES = [(k, s) for k in range(1, 16) for s in range(1, k + 3)]


def pool_plane_sizes(k, s):
    """(H, W) pairs for one geometry: the window itself, one more, and k + s + 1 (ceil mode clips the last window
    when 1 < s <= k; with s > k some elements lie in no window)"""
    a, b, c = k, k + 1, k + s + 1
    return [(a, b), (b, c), (c, a), (c, c)]
