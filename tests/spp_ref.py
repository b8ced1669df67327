"""Caffe's SPP layer (spp_layer.cpp) restated in numpy three times:

- forward64 / backward64: float64, window by window;
- expansion32: fp32 in the order Caffe computes it, the Split, each level's Pooling (pooling_layer.cpp: MAX's first
  value > the running maximum from -FLT_MAX, AVE's row-major sum from +0 divided by the pool size), Flatten and Concat;
  backward each level's Pooling gradient from +0, then Split's sum g0 + g1, += g2, ...  Vectorised over windows, so
  it runs at the sizes the GPU tests use;
- index_map32: fp32 again, one output and one bottom element at a time, from integer maps of each bottom element to
  its window at every level (the form the engine's kernels compute).  Scalar loops: small shapes only.

infer() restates the shape rule and the refusals of the layout parser."""
import math

import numpy as np

F32 = np.float32
FLT_MAX = np.finfo(np.float32).max


def level(height, width, lv):
    """SPPLayer::GetPoolingParam: (bins, kernel_h, kernel_w, pad_h, pad_w), in its arithmetic (a double ceil)"""
    bins = int(pow(2, lv))
    kh, kw = int(math.ceil(height / float(bins))), int(math.ceil(width / float(bins)))
    return bins, kh, kw, (kh * bins - height + 1) // 2, (kw * bins - width + 1) // 2


def pooled(size, kernel, pad):
    """PoolingLayer::Reshape's pooled size with stride = kernel: ceil, then the last window clipped to start inside"""
    out = int(math.ceil(float(size + 2 * pad - kernel) / kernel)) + 1
    if pad and (out - 1) * kernel >= size + pad:
        out -= 1
    return out


def pool_size(height, width, lv, i, j):
    """AVE's divisor for window (i, j) of level lv: the window clipped to the map and its padding (pooling_layer.cpp)"""
    bins, kh, kw, ph, pw = level(height, width, lv)
    hs, ws = i * kh - ph, j * kw - pw
    return (min(hs + kh, height + ph) - hs) * (min(ws + kw, width + pw) - ws)


def infer(shape, pyramid_height):
    """-> the top's shape; ValueError with the parser's wording"""
    if len(shape) != 4:
        raise ValueError("Input must have 4 axes, corresponding to (num, channels, height, width)")
    n, c, h, w = shape
    if h <= 0 or w <= 0:
        raise ValueError("Input dimensions cannot be zero.")
    if pyramid_height < 1:
        raise ValueError("spp_param pyramid_height must be at least 1 (a pyramid of no levels pools nothing)")
    total = 0
    for lv in range(pyramid_height):
        bins, kh, kw, ph, pw = level(h, w, lv)
        at = f" at pyramid level {lv} ({bins} bins)"
        if ph >= kh:
            raise ValueError(f"Check failed: pad_h_ < kernel_h_ ({ph} vs. {kh})" + at)
        if pw >= kw:
            raise ValueError(f"Check failed: pad_w_ < kernel_w_ ({pw} vs. {kw})" + at)
        total += pooled(h, kh, ph) * pooled(w, kw, pw)
    return (n, c, 1, 1) if pyramid_height == 1 else (n, c * total)


def level_offsets(channels, pyramid_height):
    """where each level starts within a sample's top: channels * (4^l - 1) / 3"""
    return [channels * (4 ** lv - 1) // 3 for lv in range(pyramid_height + 1)]


# --------------------------------------------------------------------------- float64
def forward64(x, pyramid_height, pool):
    """y in float64: each window's largest value (NaN skipped, -FLT_MAX for none) or its sum over kernel_h * kernel_w"""
    n, c, h, w = x.shape
    x = x.astype(np.float64)
    parts = []
    for lv in range(pyramid_height):
        bins, kh, kw, ph, pw = level(h, w, lv)
        y = np.empty((n, c, bins, bins))
        for i in range(bins):
            for j in range(bins):
                win = x[:, :, max(i * kh - ph, 0):min(i * kh - ph + kh, h),
                        max(j * kw - pw, 0):min(j * kw - pw + kw, w)]
                win = win.reshape(n, c, -1)
                if pool == "MAX":
                    y[:, :, i, j] = np.where(win > -FLT_MAX, win, -FLT_MAX).max(-1)
                else:
                    y[:, :, i, j] = win.sum(-1) / pool_size(h, w, lv, i, j)
        parts.append(y.reshape(n, -1))
    return np.concatenate(parts, 1)


def backward64(dy, argmax, bottom_shape, pyramid_height, pool):
    """dx in float64: each level's gradient (dy at the argmax, or dy / size over the window), summed"""
    n, c, h, w = bottom_shape
    dx = np.zeros(bottom_shape)
    offs = level_offsets(c, pyramid_height)
    for lv in range(pyramid_height):
        bins, kh, kw, ph, pw = level(h, w, lv)
        d = dy[:, offs[lv]:offs[lv + 1]].astype(np.float64).reshape(n, c, bins, bins)
        for i in range(bins):
            for j in range(bins):
                if pool == "MAX":
                    a = argmax[:, offs[lv]:offs[lv + 1]].reshape(n, c, bins, bins)[:, :, i, j]
                    for (p, q), k in np.ndenumerate(a):
                        if k >= 0:
                            dx[p, q].flat[k] += d[p, q, i, j]
                else:
                    dx[:, :, max(i * kh - ph, 0):min(i * kh - ph + kh, h),
                       max(j * kw - pw, 0):min(j * kw - pw + kw, w)] += (d[:, :, i, j] /
                                                                          pool_size(h, w, lv, i, j))[:, :, None, None]
    return dx


# --------------------------------------------------------------------------- fp32, Caffe's expansion
def _tiles(a, lv, fill):
    """a [n, c, h, w] placed in level lv's padded frame (fill outside the map) -> [n, c, bins, bins, kh * kw], each
    window's taps in row-major order"""
    n, c, h, w = a.shape
    bins, kh, kw, ph, pw = level(h, w, lv)
    frame = np.full((n, c, bins * kh, bins * kw), fill, a.dtype)
    frame[:, :, ph:ph + h, pw:pw + w] = a  # bins * k - pad >= h: the map ends inside the frame
    return frame.reshape(n, c, bins, kh, bins, kw).transpose(0, 1, 2, 4, 3, 5).reshape(n, c, bins, bins, kh * kw)


def _pool_forward32(x, lv, pool):
    """one level's Pooling: (y [n, c, bins, bins], argmax or None)"""
    n, c, h, w = x.shape
    bins, kh, kw, _, _ = level(h, w, lv)
    if pool == "MAX":
        # the first value > the running maximum: of the values > -FLT_MAX (never NaN), the first equal to their largest
        v = _tiles(x, lv, -np.inf)
        taps = _tiles(np.broadcast_to(np.arange(h * w, dtype=np.int64).reshape(1, 1, h, w), x.shape), lv, -1)
        ok = v > -FLT_MAX
        m = np.where(ok, v, -np.inf).max(-1, keepdims=True)
        first = np.argmax(ok & (v == m), -1)[..., None]
        has = ok.any(-1)
        y = np.where(has, np.take_along_axis(v, first, -1)[..., 0], -FLT_MAX).astype(F32)
        return y, np.where(has, np.take_along_axis(taps, first, -1)[..., 0], -1).astype(np.int32)
    # +0 taps outside the map change no running sum from +0 (it is never -0), so the padded frame sums as Caffe does
    t = _tiles(x, lv, 0.0)
    s = np.zeros(t.shape[:-1], F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(t.shape[-1]):
            s = s + t[..., k]
        return s / F32(kh * kw), None  # every accepted level's pool size is the whole kernel


def _pool_backward32(d, arg, bottom_shape, lv, pool):
    """one level's Pooling gradient from +0 (pooling_layer.cpp Backward)"""
    n, c, h, w = bottom_shape
    bins, kh, kw, ph, pw = level(h, w, lv)
    with np.errstate(invalid="ignore", over="ignore"):
        if pool == "MAX":
            g = np.zeros((n * c, h * w), F32)
            planes = np.repeat(np.arange(n * c), bins * bins).reshape(n * c, -1)
            a, dd = arg.reshape(n * c, -1), d.reshape(n * c, -1)
            hit = a >= 0
            np.add.at(g, (planes[hit], a[hit]), dd[hit])
            return g.reshape(bottom_shape)
        frame = np.zeros((n, c, bins, kh, bins, kw), F32)
        frame += (d / F32(kh * kw))[:, :, :, None, :, None]  # 0 + dy / size, once per tap
        return frame.reshape(n, c, bins * kh, bins * kw)[:, :, ph:ph + h, pw:pw + w].copy()


def expansion32(x, pyramid_height, pool):
    """Split -> Pooling per level -> Flatten -> Concat: (y, argmax or None)"""
    ys, args = [], []
    for lv in range(pyramid_height):
        y, a = _pool_forward32(x, lv, pool)
        ys.append(y.reshape(x.shape[0], -1))
        args.append(None if a is None else a.reshape(x.shape[0], -1))
    if pyramid_height == 1:
        return ys[0].reshape(x.shape[0], x.shape[1], 1, 1), None if pool != "MAX" else args[0].reshape(
            x.shape[0], x.shape[1], 1, 1)
    return np.concatenate(ys, 1), None if pool != "MAX" else np.concatenate(args, 1)


def expansion32_backward(dy, argmax, bottom_shape, pyramid_height, pool):
    """Concat -> Flatten -> each level's Pooling backward -> Split: g0 (+ g1, += g2, ..)"""
    n, c, h, w = bottom_shape
    dy = dy.reshape(n, -1)
    argmax = None if argmax is None else argmax.reshape(n, -1)
    offs = level_offsets(c, pyramid_height)
    dx = None
    with np.errstate(invalid="ignore", over="ignore"):
        for lv in range(pyramid_height):
            bins = 2 ** lv
            part = slice(offs[lv], offs[lv + 1])
            d = dy[:, part].reshape(n, c, bins, bins)
            a = None if argmax is None else argmax[:, part].reshape(n, c, bins, bins)
            g = _pool_backward32(d, a, bottom_shape, lv, pool)
            dx = g if dx is None else dx + g
    return dx


# --------------------------------------------------------------------------- fp32, index maps
def bin_maps(height, width, lv):
    """each row's and each column's window at level lv (stride = kernel: windows do not overlap)"""
    bins, kh, kw, ph, pw = level(height, width, lv)
    return (np.arange(height) + ph) // kh, (np.arange(width) + pw) // kw


def index_map32(x, dy, pyramid_height, pool):
    """(y, argmax, dx) one element at a time: each output scans the bottom elements the maps send to it in (h, w)
    order; each bottom element adds its levels' terms in level order"""
    with np.errstate(invalid="ignore", over="ignore"):
        return _index_map32(x, dy, pyramid_height, pool)


def _index_map32(x, dy, pyramid_height, pool):
    n, c, h, w = x.shape
    offs = level_offsets(c, pyramid_height)
    y = np.zeros((n, offs[-1]), F32)
    arg = np.full((n, offs[-1]), -1, np.int32)
    size = {}
    for lv in range(pyramid_height):
        rows, cols = bin_maps(h, w, lv)
        bins, kh, kw, _, _ = level(h, w, lv)
        size[lv] = F32(kh * kw)
        for p in range(n):
            for q in range(c):
                for i in range(bins):
                    for j in range(bins):
                        o = offs[lv] + (q * bins + i) * bins + j
                        m, mi, s = F32(-FLT_MAX), -1, F32(0)
                        for hh in np.nonzero(rows == i)[0]:
                            for ww in np.nonzero(cols == j)[0]:
                                v = x[p, q, hh, ww]
                                if v > m:
                                    m, mi = v, hh * w + ww
                                s = F32(s + v)
                        y[p, o], arg[p, o] = (m, mi) if pool == "MAX" else (F32(s / size[lv]), -1)
    dx = np.zeros(x.shape, F32)
    dyf = dy.reshape(n, -1)
    maps = [bin_maps(h, w, lv) for lv in range(pyramid_height)]
    for p in range(n):
        for q in range(c):
            for hh in range(h):
                for ww in range(w):
                    s = F32(0)
                    for lv in range(pyramid_height):
                        bins = 2 ** lv
                        o = offs[lv] + (q * bins + maps[lv][0][hh]) * bins + maps[lv][1][ww]
                        if pool == "MAX":
                            t = F32(F32(0) + dyf[p, o]) if arg[p, o] == hh * w + ww else F32(0)
                        else:
                            t = F32(F32(0) + F32(dyf[p, o] / size[lv]))
                        s = t if lv == 0 else F32(s + t)
                    dx[p, q, hh, ww] = s
    if pyramid_height == 1:
        y, arg = y.reshape(n, c, 1, 1), arg.reshape(n, c, 1, 1)
    return y, (arg if pool == "MAX" else None), dx


def specials(rng, shape, ties=True):
    """Gaussian fp32 values with NaNs, both infinities, both zeros, -FLT_MAX and FLT_MAX spread through them; with
    `ties`, values drawn from a few levels so that windows hold equal maxima, and one plane that is all -FLT_MAX, NaN
    and -inf (a MAX window with no value > -FLT_MAX)"""
    x = rng.randn(*shape).astype(F32)
    if ties:
        x = np.round(x * 2).astype(F32) / F32(2)
    flat = x.reshape(-1)
    bits = np.array([0x7FC00000, 0xFFC00001, 0x7F800000, 0xFF800000, 0x00000000, 0x80000000, 0xFF7FFFFF, 0x7F7FFFFF,
                     0x00000001], np.uint32).view(F32)
    k = rng.choice(flat.size, size=min(flat.size, 3 * bits.size), replace=False)
    flat[k] = np.resize(bits, k.size)
    if ties and shape[0] * shape[1] > 1:
        plane = x[-1, -1].reshape(-1)
        plane[:] = np.resize(np.array([-FLT_MAX, np.nan, -np.inf], F32), plane.size)
    return x


def canonical_bits(a):
    """a's bits with every NaN as 0x7FFFFFFF, the GPU's canonical NaN (numpy carries an input's payload through an add,
    the GPU does not)"""
    b = np.ascontiguousarray(a, F32).view(np.uint32).copy()
    b[np.isnan(np.asarray(a, F32))] = 0x7FFFFFFF
    return b
