"""References, per-element error bounds and plausible wrong kernels for the BatchNorm kernels (csrc/batch_norm.cu,
DESIGN.md section 13), numpy only.

* `reference`: the float64 forward and backward of test_batch_norm_host.py (`numpy_bn_forward`,
  `numpy_bn_backward`) on the fp32 inputs.
* `restate_forward` / `restate_backward`: numpy fp32 in the kernels' operation order.  Each plane is summed in
  double and rounded once to fp32; the partials are added over n in double and divided by M; every element
  operation is one fp32 rounding; std is libm's powf(fl(var + eps), 0.5f).  The double sums may round in another
  order than the kernels' xor tree, so on general inputs the restatement only stays within the bounds below; on the
  `dyadic` family every sum is exact and mean, var, S1 and the blobs are reproduced bit for bit.  y given the
  kernel's saved statistics is reproduced bit for bit on any input.
* `mean_bound`, `var_bound`, `y_bound`, `dx_bound`: first-order bounds on |kernel - float64| per channel or per
  element, derived from that operation order (u = 2^-24).
* `MUTATIONS` / `kernel_model(..., mutation=...)`: the restatement with one plausible kernel mistake each; every one
  must fall outside the bounds (tests/test_bn_ref_host.py).
"""
import ctypes
import ctypes.util

import numpy as np

from test_batch_norm_host import numpy_bn_backward, numpy_bn_forward

F32 = np.float32
U = 2.0 ** -24  # unit roundoff of fp32
TINY = 2.0 ** -149  # the smallest fp32 subnormal
# glibc's powf is within one ulp (2u of the result) of powf(x, 0.5) over its whole range
C_POWF = 2.0
SLACK = 1.0 + 2.0 ** -20  # the double sums and the second-order terms the bounds drop

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype = ctypes.c_float
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]


def powf_half(v):
    """libm's powf(v, 0.5f) element by element (numpy's float32 power and sqrt are not powf)"""
    v = np.asarray(v, F32)
    return np.array([_libm.powf(float(a), 0.5) for a in v.ravel()], F32).reshape(v.shape)


def planes(a):
    """(N, C, H*W) view of Caffe's BatchNorm geometry: channels = axis 1 (1 for a 1-axis bottom)"""
    a = np.asarray(a)
    return a.reshape(a.shape[0], a.shape[1] if a.ndim > 1 else 1, -1)


def channel_sum(t, first_image_only=False):
    """float64 [C]: each (n, c) plane of t summed in double and rounded to fp32, the partials added over n in
    double (the kernels' bn_plane_sums_kernel, then bn_mean/var_update/channel_sums_kernel)"""
    part = t.astype(np.float64).sum(2).astype(F32).astype(np.float64)
    return part[:1].sum(0) if first_image_only else part.sum(0)


# ------------------------------------------------------------------ the kernels' operation order, and mutations of it

MUTATIONS = ("one_pass_var", "unbiased_var", "eps_after_sqrt", "k_over_m_minus_1", "no_s2", "channel_shift",
             "first_image_only")


def _std(var, eps, mutation=None):
    if mutation == "eps_after_sqrt":
        return powf_half(var) + F32(eps)
    return powf_half(var + F32(eps))


def _stats(xp, mutation=None):
    n, _, hw = xp.shape
    m = n * hw
    first = mutation == "first_image_only"
    mean = (channel_sum(xp, first) / m).astype(F32)
    if mutation == "one_pass_var":  # E[x^2] - mean^2 in fp32
        var = (channel_sum(xp * xp, first) / m).astype(F32) - mean * mean
    else:
        d = xp - mean[None, :, None]
        var = (channel_sum(d * d, first) / m).astype(F32)
    if mutation == "unbiased_var" and m > 1:
        var = var * (F32(m) / F32(m - 1))
    if mutation == "channel_shift":  # channel c normalised with channel c + 1's statistics
        mean, var = np.roll(mean, -1), np.roll(var, -1)
    return mean, var


def restate_forward(x, blobs, f=0.999, eps=1e-5, global_stats=False, stats=None, mutation=None):
    """-> (y, mean, var, (mean_blob', var_blob', s')) in fp32.  With `stats` = (mean, var), y is computed from those
    (the kernel's saved statistics) instead of the restated ones."""
    xp = planes(x).astype(F32)
    n, c, hw = xp.shape
    m = n * hw
    mb, vb, s = (np.asarray(b, F32).reshape(-1) for b in blobs)
    if global_stats:
        sf = F32(0) if s[0] == 0 else F32(1) / s[0]
        mean, var = sf * mb, sf * vb
        new = (mb.copy(), vb.copy(), s.copy())
    else:
        mean, var = _stats(xp, mutation)
        corr = F32(m) / F32(m - 1) if m > 1 else F32(1)
        f = F32(f)
        new = (mean + f * mb, corr * var + f * vb, s * f + F32(1))
    if stats is not None:
        mean, var = (np.asarray(a, F32) for a in stats)
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = _std(var, eps, mutation)
        y = (xp - mean[None, :, None]) / sd[None, :, None]
    return y.reshape(np.shape(x)), mean, var, new


def restate_backward(x, dy, mean, var, eps=1e-5, global_stats=False, mutation=None):
    """-> (dx, S1, S2) in fp32 from the saved statistics (S1, S2 None with global statistics)"""
    xp, g = planes(x).astype(F32), planes(dy).astype(F32)
    n, _, hw = xp.shape
    m = n * hw
    mean, var = np.asarray(mean, F32), np.asarray(var, F32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        sd = _std(var, eps, mutation)[None, :, None]
        if global_stats:
            return (g / sd).reshape(np.shape(x)), None, None
        xh = (xp - mean[None, :, None]) / sd
        first = mutation == "first_image_only"
        s1 = channel_sum(g, first).astype(F32)
        s2 = channel_sum(xh * g, first).astype(F32)
        k = F32(-1.0 / (m - 1)) if mutation == "k_over_m_minus_1" and m > 1 else F32(-1.0 / m)
        if mutation == "no_s2":
            dx = (g + k * s1[None, :, None]) / sd
        else:
            dx = (g + k * (s1[None, :, None] + xh * s2[None, :, None])) / sd
    return dx.reshape(np.shape(x)), s1, s2


def kernel_model(x, dy, eps=1e-5, mutation=None):
    """The training forward and backward in the kernels' order, optionally with one of MUTATIONS ->
    dict(mean, var, y, dx) in fp32"""
    c = planes(x).shape[1]
    zero = (np.zeros(c, F32), np.zeros(c, F32), np.zeros(1, F32))
    y, mean, var, _ = restate_forward(x, zero, eps=eps, mutation=mutation)
    dx, _, _ = restate_backward(x, dy, mean, var, eps, mutation=mutation)
    return dict(mean=mean, var=var, y=y, dx=dx)


# ------------------------------------------------------------------ float64 reference and bounds

def reference(x, eps=1e-5):
    """-> (y64, mean64, var64): the float64 forward with the float64 batch statistics"""
    c = planes(x).shape[1]
    y, mean, var, _ = numpy_bn_forward(np.asarray(x, F32), np.zeros(c), np.zeros(c), 0.0, eps=eps)
    return y, mean, var


def reference_backward(x, dy, mean, var, eps=1e-5, global_stats=False):
    """float64 dx from the given statistics (the kernel's saved ones: dx is checked apart from their error)"""
    return numpy_bn_backward(np.asarray(x, F32), np.asarray(dy, F32), np.asarray(mean, np.float64),
                             np.asarray(var, np.float64), eps=eps, global_stats=global_stats)


def mean_bound(x):
    """[C]: each plane sum rounded to fp32 (u |P_n| <= u sum_plane |x|), the sum of the partials over n divided by M
    and rounded (u |mean|): |mean - mean64| <= u (mean|x| + |mean|)"""
    xp = planes(x).astype(np.float64)
    return SLACK * U * (np.abs(xp).mean((0, 2)) + np.abs(xp.mean((0, 2)))) + TINY


def var_bound(x, var64, dmean):
    """[C]: var is (1/M) sum fl(fl(x - mean~)^2) with mean~ within dmean of the mean; the exact sum of
    (x - mean~)^2 is M (var + (mean~ - mean)^2).  Every term is >= 0, so the roundings add relatively: the
    subtraction and the square 3u, the plane partial u, the final rounding u: 5u (var + dmean^2) + dmean^2, and the
    underflow of the squares, at most TINY per term on average."""
    return SLACK * (5 * U * (var64 + dmean ** 2) + dmean ** 2) + 2 * TINY


def y_bound(y64, var64, eps, dmean, dvar, c_axis=1):
    """per element: sd~ = powf(fl(var~ + eps)) is relatively within dvar / (2 (var + eps)) + u/2 + C_POWF u of
    sqrt(var + eps); fl(x - mean~) differs from x - mean by dmean + u |x - mean~|; the division adds u.  So
    |y - y64| <= |y64| (dvar / (2 (var + eps)) + (C_POWF + 2.5) u) + dmean / sd (x - mean cancels)."""
    shape = [1] * np.ndim(y64)
    shape[c_axis] = -1
    ve = (np.asarray(var64, np.float64) + np.float64(F32(eps))).reshape(shape)
    sd = np.sqrt(ve)
    rel = 0.5 * np.asarray(dvar).reshape(shape) / ve + (C_POWF + 2.5) * U
    with np.errstate(invalid="ignore", divide="ignore"):
        return SLACK * (np.abs(y64) * rel + np.asarray(dmean).reshape(shape) / sd) + TINY


def dx_bound(x, dy, mean, var, eps=1e-5):
    """per element, given the saved (mean, var): with x^ = (x - mean) / sd and k = 1/M,
      S1 = sum dy: each plane partial rounded, then the total: |dS1| <= u (sum |dy| + |S1|);
      S2 = sum fl(x^~ dy), x^~ = x^ (1 + 5u) (subtraction, sd~ within (C_POWF + 1/2) u, division): each term is
        off by 6u |x^ dy|, the partials and the total add 2u: |dS2| <= 8u sum |x^ dy|;
      dx = fl(fl(dy + fl(k~ fl(S1 + fl(x^ S2)))) / sd~): with G = |dy| + k (|S1| + |x^| |S2|) every rounding is at most
        u G, there are 14 of them counting x^ (5), k~ and sd~ (C_POWF + 1/2) and the final division; the sums add
        k (|dS1| + |x^| |dS2|).
    dx = dy - k S1 - k x^ S2 cancels, so the bound is in terms of those magnitudes and not of |dx|."""
    xp = planes(x).astype(np.float64)
    g = planes(dy).astype(np.float64)
    n, c, hw = xp.shape
    k = 1.0 / (n * hw)
    sd = np.sqrt(np.asarray(var, np.float64) + np.float64(F32(eps)))[None, :, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        xh = (xp - np.asarray(mean, np.float64)[None, :, None]) / sd
        s1, s2 = g.sum((0, 2))[None, :, None], (g * xh).sum((0, 2))[None, :, None]
        ds1 = U * (np.abs(g).sum((0, 2))[None, :, None] + np.abs(s1))
        ds2 = 8 * U * np.abs(g * xh).sum((0, 2))[None, :, None]
        big = np.abs(g) + k * (np.abs(s1) + np.abs(xh) * np.abs(s2))
        b = SLACK * ((14 + C_POWF) * U * big + k * (ds1 + np.abs(xh) * ds2)) / sd + 16 * TINY / sd + 16 * TINY
    return b.reshape(np.shape(x))


def outside(got, want, bound):
    """boolean mask: |got - want| > bound, NaN counted as outside"""
    with np.errstate(invalid="ignore", over="ignore"):
        return ~(np.abs(np.asarray(got, np.float64) - want) <= bound)


def outside_fractions(x, dy, out, eps=1e-5):
    """fraction of the channels (mean, var) and elements (y, dx) of a kernel's `out` = dict(mean, var, y, dx)
    outside the bounds.  dx is compared with the float64 backward from out's own statistics."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):  # a mutation's variance may be negative
        y64, mean64, var64 = reference(x, eps)
        dm = mean_bound(x)
        dv = var_bound(x, var64, dm)
        c_axis = 1 if np.ndim(x) > 1 else 0
        dx64 = reference_backward(x, dy, out["mean"], out["var"], eps)
        return dict(mean=outside(out["mean"], mean64, dm).mean(), var=outside(out["var"], var64, dv).mean(),
                    y=outside(out["y"], y64, y_bound(y64, var64, eps, dm, dv, c_axis)).mean(),
                    dx=outside(out["dx"], dx64, dx_bound(x, dy, out["mean"], out["var"], eps)).mean())


# ------------------------------------------------------------------ input families

def dyadic(rng, shape):
    """(x, dy) on a 2^-8 grid.  Each channel is a dyadic centre in [-2, 2) plus deviations +-d, d on a 2^-4 grid in
    [-2, 2), in pairs (and one 0 when M is odd), shuffled over the channel's N x H x W positions.  |x| <= 4 and every
    plane sum of x, (x - mean)^2 and dy (|dy| <= 2) is exact in fp32 for H*W <= 16384, so mean = centre exactly,
    var = fl(fl64(sum d^2 / M)), S1 = sum dy exactly, whatever the summation order."""
    n, c = shape[0], (shape[1] if len(shape) > 1 else 1)
    hw = int(np.prod(shape[2:], dtype=np.int64)) if len(shape) > 2 else 1
    m = n * hw
    assert hw <= 16384
    centre = rng.integers(-512, 512, c).astype(np.float64) / 256
    half = rng.integers(-32, 32, (c, m // 2)).astype(np.float64) / 16
    dev = np.concatenate([half, -half, np.zeros((c, m % 2))], axis=1)
    dev = rng.permuted(dev, axis=1)
    x = (centre[:, None] + dev).reshape(c, n, hw).transpose(1, 0, 2)
    dy = rng.integers(-512, 512, (n, c, hw)).astype(np.float64) / 256
    return np.ascontiguousarray(x, F32).reshape(shape), np.ascontiguousarray(dy, F32).reshape(shape)


def gaussian(rng, shape, constant=True):
    """(x, dy): channel c is offset_c + scale_c N(0, 1) with scale log-uniform over [1e-3, 1e3]; every fifth channel
    sits at an offset of 1e4 scale_c; channel 1 (with `constant`) holds one value (var = 0).  dy has per-channel
    log-uniform scales of its own."""
    n, c = shape[0], (shape[1] if len(shape) > 1 else 1)
    scale = 10.0 ** rng.uniform(-3, 3, c)
    offset = np.where(np.arange(c) % 5 == 4, 1e4, rng.uniform(-2, 2, c)) * scale
    bshape = (1, c) + (1,) * (len(shape) - 2)
    x = rng.standard_normal(shape, dtype=F32) * scale.reshape(bshape).astype(F32) + offset.reshape(bshape).astype(F32)
    if constant and c > 1:
        x[:, 1] = F32(0.7) * F32(scale[1])
    dscale = (10.0 ** rng.uniform(-3, 3, c)).reshape(bshape).astype(F32)
    dy = rng.standard_normal(shape, dtype=F32) * dscale
    return np.ascontiguousarray(x, F32), np.ascontiguousarray(dy, F32)
