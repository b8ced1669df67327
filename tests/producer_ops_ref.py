"""Float64 references, with Caffe's rules, of the built-in producer's Convolution, Pooling, InnerProduct, ReLU, Sigmoid,
SoftmaxWithLoss, Slice, Concat, Split, Eltwise, Scale, EuclideanLoss and ContrastiveLoss ops (DESIGN.md section 14),
and per-element error bounds derived from each op's rounding count.

Every reference takes the fp32 inputs exactly (as float64) and returns float64.  A dot-product bound is
(n + extra) * 2^-24 * sum |a_i * b_i|: n is the number of FMAs of one accumulation, extra the further roundings of
its result (a bias add, the chunk-partial adds of a split-K reduction), and the absolute sum is the same op evaluated
on |a| and |b|.  Elementwise bounds use the CUDA maximum ulp errors of tanhf (2), expf (2) and logf (1) plus one
rounding per further operation.  No bound is fitted to GPU output."""
import math

import numpy as np

U = 2.0 ** -24  # unit roundoff of fp32
TINY = 2.0 ** -149  # the smallest fp32 subnormal: the absolute error floor of a rounding that underflows
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
EXPF_ULP, LOGF_ULP, TANHF_ULP = 2, 1, 2  # CUDA C Programming Guide, single-precision maximum ulp errors

# the weight-gradient split-K of native_producer.cu (kSplitK, kMaxSplits, kBK) and bias_grad_kernel's block
SPLIT_K, MAX_SPLITS, BK, BLOCK = 512, 256, 16, 256


def ulp(v):
    """fp32 ulp at |v| (of the binade above when |v| sits just below a power of two), never below a subnormal's."""
    a = np.abs(np.asarray(v, np.float64)) * (1 + 2.0 ** -20)
    e = np.floor(np.log2(np.maximum(a, FLT_MIN)))
    return np.maximum(2.0 ** (e - 23), TINY)


def split_chunk(k):
    need = -(-k // MAX_SPLITS)
    return max(SPLIT_K, -(-need // BK) * BK)


def splits_of(k):
    return -(-k // split_chunk(k))


def bias_grad_count(n):
    """Roundings of bias_grad_kernel's sum of n values: one thread's in-order run, the 8-level tree, the add into
    the gradient."""
    return -(-n // BLOCK) + 8 + 1


# ------------------------------------------------------------------ Convolution (im2col with zero padding)
def out_size(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def im2col(x, kh, kw, sh, sw, ph, pw):
    """[N, C, H, W] -> [N, C * kh * kw, OH * OW], k = (c * kh + i) * kw + j (Caffe's order)."""
    n, c, h, w = x.shape
    oh, ow = out_size(h, kh, sh, ph), out_size(w, kw, sw, pw)
    xp = np.zeros((n, c, h + 2 * ph + kh, w + 2 * pw + kw))
    xp[:, :, ph:ph + h, pw:pw + w] = x
    cols = np.empty((n, c, kh, kw, oh, ow))
    for i in range(kh):
        for j in range(kw):
            cols[:, :, i, j] = xp[:, :, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw]
    return cols.reshape(n, c * kh * kw, oh * ow), oh, ow


def col2im(cols, shape, kh, kw, sh, sw, ph, pw):
    n, c, h, w = shape
    oh, ow = out_size(h, kh, sh, ph), out_size(w, kw, sw, pw)
    cols = cols.reshape(n, c, kh, kw, oh, ow)
    xp = np.zeros((n, c, h + 2 * ph + kh, w + 2 * pw + kw))
    for i in range(kh):
        for j in range(kw):
            xp[:, :, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw] += cols[:, :, i, j]
    return xp[:, :, ph:ph + h, pw:pw + w]


def conv_forward(x, w, b, geo):
    """y[n, o, p] = sum_k w[o, k] * cols[n, k, p] + b[o]; geo = (kh, kw, sh, sw, ph, pw)."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    cols, oh, ow = im2col(x, *geo)
    y = np.einsum("ok,nkp->nop", w.reshape(w.shape[0], -1), cols)
    if b is not None:
        y = y + np.asarray(b, np.float64)[None, :, None]
    return y.reshape(x.shape[0], w.shape[0], oh, ow)


def conv_backward(x, w, dy, geo):
    """-> dW, db, dx of the convolution for top gradient dy."""
    x, w, dy = (np.asarray(v, np.float64) for v in (x, w, dy))
    cols, _, _ = im2col(x, *geo)
    d = dy.reshape(dy.shape[0], dy.shape[1], -1)
    dw = np.einsum("nop,nkp->ok", d, cols).reshape(w.shape)
    dcols = np.einsum("ok,nop->nkp", w.reshape(w.shape[0], -1), d)
    return dw, d.sum(axis=(0, 2)), col2im(dcols, x.shape, *geo)


def conv_bounds(x, w, b, dy, geo):
    """Per-element bounds of (y, dW, db, dx): each dot product's rounding count times the sum of |terms|."""
    cin, kh, kw = w.shape[1:]
    k = cin * kh * kw
    n_pix = x.shape[0] * dy.shape[2] * dy.shape[3]
    ay = conv_forward(np.abs(x), np.abs(w), None if b is None else np.abs(b), geo)
    adw, adb, adx = conv_backward(np.abs(x), np.abs(w), np.abs(dy), geo)
    return ((k + (b is not None)) * U * ay, (n_pix + splits_of(n_pix) + 1) * U * adw,
            bias_grad_count(n_pix) * U * adb, w.shape[0] * kh * kw * U * adx)


# ------------------------------------------------------------------ InnerProduct: y[B, N] = x[B, K] w[N, K]^T + b
def ip_forward(x, w, b):
    y = np.asarray(x, np.float64).reshape(x.shape[0], -1) @ np.asarray(w, np.float64).T
    return y if b is None else y + np.asarray(b, np.float64)


def ip_backward(x, w, dy):
    x2 = np.asarray(x, np.float64).reshape(x.shape[0], -1)
    dy = np.asarray(dy, np.float64)
    return dy.T @ x2, dy.sum(axis=0), (dy @ np.asarray(w, np.float64)).reshape(x.shape)


def ip_bounds(x, w, b, dy):
    bsz, k = x.shape[0], w.shape[1]
    ay = ip_forward(np.abs(x), np.abs(w), None if b is None else np.abs(b))
    adw, adb, adx = ip_backward(np.abs(x), np.abs(w), np.abs(dy))
    return ((k + (b is not None)) * U * ay, (bsz + splits_of(bsz) + 1) * U * adw, bias_grad_count(bsz) * U * adb,
            w.shape[0] * U * adx)


# ------------------------------------------------------------------ Pooling (pooling_layer.cu)
def pooled_size(h, k, s, p):
    """PoolingLayer::Reshape: ceil((H + 2p - k) / s) + 1, one fewer when pad > 0 and the last window would start
    at or past H + pad."""
    o = int(math.ceil((h + 2 * p - k) / s)) + 1
    if p and (o - 1) * s >= h + p:
        o -= 1
    return o


def _windows(h, w, kh, kw, sh, sw, ph, pw):
    """(ph, pw, hs, he, ws, we, size) of every window: `size` is the AVE divisor, the window clipped to H + pad
    before it is clipped to H."""
    for i in range(pooled_size(h, kh, sh, ph)):
        for j in range(pooled_size(w, kw, sw, pw)):
            hs, ws = i * sh - ph, j * sw - pw
            he, we = min(hs + kh, h + ph), min(ws + kw, w + pw)
            size = (he - hs) * (we - ws)
            yield i, j, max(hs, 0), min(he, h), max(ws, 0), min(we, w), size


def pool_forward(x, method, geo, last_max_wins=False, divisor_clipped_to_h=False):
    """-> y (float64) and, for MAX, the argmax (h * W + w, or -1 for an empty window).  MAX: the first maximum in
    row-major order wins; an empty window gives -FLT_MAX.  AVE: sum / size, so an empty window gives 0 / size (NaN
    for size 0).  The two flags are mutations for the bound tests."""
    x = np.asarray(x, np.float64)
    n, c, h, w = x.shape
    kh, kw, sh, sw, ph, pw = geo
    oh, ow = pooled_size(h, kh, sh, ph), pooled_size(w, kw, sw, pw)
    y = np.empty((n, c, oh, ow))
    idx = np.full((n, c, oh, ow), -1, np.int64)
    for i, j, hs, he, ws, we, size in _windows(h, w, *geo):
        win = x[:, :, hs:he, ws:we].reshape(n, c, -1)
        if method == "AVE":
            if divisor_clipped_to_h:
                size = (he - hs) * (we - ws)
            with np.errstate(invalid="ignore", divide="ignore"):
                y[:, :, i, j] = win.sum(axis=2) / size
            continue
        if win.shape[2] == 0:
            y[:, :, i, j] = -FLT_MAX
            continue
        a = win.shape[2] - 1 - np.argmax(win[:, :, ::-1], axis=2) if last_max_wins else np.argmax(win, axis=2)
        y[:, :, i, j] = np.take_along_axis(win, a[..., None], axis=2)[..., 0]
        idx[:, :, i, j] = (hs + a // (we - ws)) * w + ws + a % (we - ws)
    return y, idx


def pool_backward(dy, x_shape, method, geo, idx=None, divisor_clipped_to_h=False):
    """MAX: every dy goes to its window's argmax (none for an empty window); AVE: dy / size to every element of the
    clipped window."""
    dy = np.asarray(dy, np.float64)
    n, c, h, w = x_shape
    dx = np.zeros((n, c, h * w))
    for i, j, hs, he, ws, we, size in _windows(h, w, *geo):
        if method == "MAX":
            k = idx[:, :, i, j]
            nn, cc = np.nonzero(k >= 0)
            dx[nn, cc, k[nn, cc]] += dy[nn, cc, i, j]
            continue
        if divisor_clipped_to_h:
            size = (he - hs) * (we - ws)
        if he > hs and we > ws:
            cover = np.zeros((h, w), bool)
            cover[hs:he, ws:we] = True
            dx[:, :, cover.ravel()] += (dy[:, :, i, j] / size)[..., None]
    return dx.reshape(x_shape)


def pool_bounds(x, dy, method, geo):
    """MAX: the forward is exact, and each dx sums the dy of the windows routed to it (one rounding per window).
    AVE: a window's in-order sum then one division; each dx sums dy / size over its windows (two roundings each)."""
    kh, kw, sh, sw = geo[:4]
    nwin = -(-kh // sh) * -(-kw // sw)  # windows that can cover one element
    if method == "MAX":
        _, idx = pool_forward(x, "MAX", geo)
        return None, nwin * U * pool_backward(np.abs(dy), x.shape, "MAX", geo, idx)
    ay, _ = pool_forward(np.abs(x), "AVE", geo)
    return (kh * kw + 1) * U * np.nan_to_num(np.abs(ay)), (nwin + 1) * U * pool_backward(np.abs(dy), x.shape, "AVE", geo)


def max_decisions_hold(x, bound, geo):
    """True when every MAX window's winner beats the rest of its window by more than twice the largest error bound
    in it, so that values within their bounds pick the same argmax (a precondition of the Gaussian cases)."""
    n, c, h, w = x.shape
    for _, _, hs, he, ws, we, _ in _windows(h, w, *geo):
        win = np.sort(x[:, :, hs:he, ws:we].reshape(n * c, -1), axis=1)
        if win.shape[1] > 1 and np.any(win[:, -1] - win[:, -2] <= 2 * bound[:, :, hs:he, ws:we].max()):
            return False
    return True


# ------------------------------------------------------------------ ReLU and Sigmoid (relu_layer.cu, sigmoid_layer.cu)
def relu_forward32(x, slope):
    """Exact in fp32: x, or one rounded product."""
    x = np.asarray(x, np.float32)
    return np.where(x > 0, x, x * np.float32(slope))


def relu_backward32(bottom, dy, slope):
    """`bottom` is what the backward reads: the input, or the output itself for an in-place layer."""
    dy = np.asarray(dy, np.float32)
    return np.where(np.asarray(bottom) > 0, dy, dy * np.float32(slope))


def sigmoid_forward(x):
    return 0.5 * np.tanh(0.5 * np.asarray(x, np.float64)) + 0.5


def sigmoid_forward_bound(x):
    """0.5 * tanhf(0.5 x) + 0.5: 0.5 x and the product by 0.5 are exact for normal x; tanhf's 2 ulp, halved, and the
    rounding of the add."""
    t = np.tanh(0.5 * np.asarray(x, np.float64))
    y = 0.5 * t + 0.5
    return 0.5 * TANHF_ULP * ulp(t) + 0.5 * ulp(y)


def sigmoid_backward(y32, dy):
    """dx = dy * s * (1 - s) with s the op's fp32 output (the backward reads the top)."""
    s = np.asarray(y32, np.float64)
    return np.asarray(dy, np.float64) * s * (1 - s)


def sigmoid_backward_bound(y32, dy):
    """three roundings: dy * s, 1 - s, the product"""
    return 3 * U * np.abs(sigmoid_backward(y32, dy)) + TINY


# ------------------------------------------------------------------ SoftmaxWithLoss (softmax_loss_layer.cu)
def _rows(x, axis):
    """[outer, C, inner] view of the scores with the class axis in the middle."""
    x = np.asarray(x, np.float64)
    axis = axis % x.ndim
    outer, c = int(np.prod(x.shape[:axis], dtype=np.int64)), x.shape[axis]
    return x.reshape(outer, c, -1)


def softmax_loss(x, label, axis=1, loss_weight=1.0):
    """-> loss, dx.  p = softmax over the class axis; loss = loss_weight * mean over rows of -log(max(p[label],
    FLT_MIN)) (VALID normalisation, no ignore_label; a label is read as static_cast<int>); dx = (p - onehot) *
    loss_weight / rows."""
    v = _rows(x, axis)
    outer, c, inner = v.shape
    e = np.exp(v - v.max(axis=1, keepdims=True))
    p = e / e.sum(axis=1, keepdims=True)
    lab = np.trunc(np.asarray(label, np.float64)).astype(np.int64).reshape(outer, inner)
    pl = np.take_along_axis(p, lab[:, None, :], axis=1)[:, 0]
    rows = outer * inner
    loss = loss_weight * float(np.sum(-np.log(np.maximum(pl, FLT_MIN)))) / rows
    onehot = np.zeros_like(p)
    np.put_along_axis(onehot, lab[:, None, :], 1.0, axis=1)
    return loss, ((p - onehot) * (loss_weight / rows)).reshape(np.shape(x))


def softmax_loss_bounds(x, label, axis=1, loss_weight=1.0):
    """-> (loss bound, dx bound).  Per element of a row, in units of u = 2^-24 relative: x - m rounds once
    (|x - m| u), expf adds 2 ulp (<= 4u); the in-order row sum adds C u; p = e / sum one more; so
    rel(p) <= |x - m| u + 4u + (max over the row of the same) + C u + u, plus an absolute floor for subnormal e.
    dx = (p - onehot) * scale with scale = loss_weight / rows rounded once: |scale| (err_p + u |p - onehot|)
    + 2u |dx|.  The loss: -logf(max(p, FLT_MIN)) has err_p / max(p, FLT_MIN) + 1 ulp of the log; the rows are added
    in ceil(rows / 256) + 8 roundings, then divided and multiplied (2 more)."""
    v = _rows(x, axis)
    outer, c, inner = v.shape
    rows = outer * inner
    arg = np.abs(v - v.max(axis=1, keepdims=True))
    e = np.exp(-arg)
    rel_e = arg * U + 2 * EXPF_ULP * U
    rel_sum = (rel_e * e).sum(axis=1, keepdims=True) / e.sum(axis=1, keepdims=True) + c * U
    p = e / e.sum(axis=1, keepdims=True)
    err_p = p * (rel_e + rel_sum + U) + 4 * TINY
    lab = np.trunc(np.asarray(label, np.float64)).astype(np.int64).reshape(outer, inner)
    onehot = np.zeros_like(p)
    np.put_along_axis(onehot, lab[:, None, :], 1.0, axis=1)
    scale = abs(loss_weight) / rows
    dx = np.abs(p - onehot) * scale
    dx_bound = scale * (err_p + U * np.abs(p - onehot)) + 2 * U * dx + TINY
    pl = np.take_along_axis(p, lab[:, None, :], axis=1)[:, 0]
    epl = np.take_along_axis(err_p, lab[:, None, :], axis=1)[:, 0]
    lr = -np.log(np.maximum(pl, FLT_MIN))
    err_r = epl / np.maximum(pl - epl, FLT_MIN) + LOGF_ULP * ulp(lr)
    adds = -(-rows // BLOCK) + 8 + 2
    loss_bound = abs(loss_weight) * (err_r.sum() + adds * U * lr.sum()) / rows
    return loss_bound, dx_bound.reshape(np.shape(x))


# ------------------------------------------------------------------ Slice, Concat, Split (slice_layer, concat_layer, split_layer)
def slice_bounds(size, points=None, tops=None):
    """slice_layer.cpp Reshape: the [begin, end) of every top along the axis, from slice_points or an equal split"""
    cuts = list(points) if points else [t * (size // tops) for t in range(1, tops)]
    return list(zip([0] + cuts, cuts + [size]))


def slice_forward(x, axis, ranges):
    """pure copies: every value, NaN, infinity and subnormal, comes through unchanged"""
    idx = [slice(None)] * x.ndim
    out = []
    for b, e in ranges:
        idx[axis] = slice(b, e)
        out.append(np.asarray(x)[tuple(idx)])
    return out


def split_backward32(ds, reverse=False):
    """split_layer.cpp: the gradients of the read tops added in fp32 in top order (`reverse`: a mutation)"""
    ds = [np.asarray(d, np.float32) for d in (ds[::-1] if reverse else ds)]
    acc = ds[0].copy()
    for d in ds[1:]:
        acc = acc + d
    return acc


def split_backward_bound(ds):
    """k tops: k - 1 roundings, each at most u times the running sum's magnitude"""
    return (len(ds) - 1) * U * sum(np.abs(np.asarray(d, np.float64)) for d in ds)


def rel(n):
    """relative error of n roundings, (1 + u)^n - 1, from above"""
    return n * U * (1 + n * U)


# ------------------------------------------------------------------ Eltwise (eltwise_layer.cpp, the CPU order)
def eltwise_sum(xs, coeffs):
    """-> y (float64), its bound and the gradients' scale: y = c0 x0 rounded, then one fma per further bottom, so k
    roundings each at most u times the sum of |c_i x_i|"""
    c = [float(np.float32(v)) for v in coeffs]
    terms = [ci * np.asarray(x, np.float64) for ci, x in zip(c, xs)]
    return sum(terms), len(xs) * U * sum(np.abs(t) for t in terms) + len(xs) * TINY


def eltwise_sum_backward32(dy, coeff):
    """a copy when the coefficient is 1, else fl(c * dy)"""
    dy = np.asarray(dy, np.float32)
    return dy.copy() if np.float32(coeff) == 1 else np.float32(coeff) * dy


def eltwise_prod(xs):
    """-> y (float64) and its bound: x0 x1, then times each further bottom, k - 1 roundings"""
    y = np.prod([np.asarray(x, np.float64) for x in xs], axis=0)
    return y, rel(len(xs) - 1) * np.abs(y) + TINY


def eltwise_prod_backward(xs, dy, stable):
    """-> per-bottom (dx (float64), bound).  stable_prod_grad: the product of the other bottoms, then times dy (k - 1
    roundings).  Otherwise caffe_div(y, x_i) then times dy: y carries k - 1 roundings and the two operations add two
    more, and the division makes NaN exactly where x_i is 0 or infinite (0 / 0, inf / inf)."""
    xs = [np.asarray(x, np.float64) for x in xs]
    dy = np.asarray(dy, np.float64)
    out = []
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(len(xs)):
            g = np.prod([x for j, x in enumerate(xs) if j != i], axis=0) * dy
            if stable:
                out.append((g, rel(len(xs) - 1) * np.abs(g) + TINY))
            else:
                g = np.where((xs[i] == 0) | np.isinf(xs[i]), np.nan, g)
                out.append((g, rel(len(xs) + 1) * np.abs(g) + 2 * TINY))
    return out


def eltwise_max(xs, later_wins_ties=False):
    """-> y, winner index.  eltwise_layer.cpp Forward_cpu: bottom 0 wins over bottom 1 only when strictly greater;
    every later bottom takes over only when strictly greater than y, so a NaN wins when it is bottom 1 and is passed
    over elsewhere.  `later_wins_ties` (a later bottom taking over on >=, as in Caffe's GPU kernel) is a mutation for
    the bound tests."""
    xs = [np.asarray(x, np.float32) for x in xs]
    gt = np.greater_equal if later_wins_ties else np.greater
    first = ~np.greater(xs[0], xs[1])
    y = np.where(first, xs[1], xs[0])
    idx = first.astype(np.int64)
    for b in range(2, len(xs)):
        take = gt(xs[b], y)
        y = np.where(take, xs[b], y)
        idx = np.where(take, b, idx)
    return y, idx


def eltwise_max_backward(dy, idx, k):
    dy = np.asarray(dy, np.float32)
    return [np.where(idx == b, dy, np.float32(0)) for b in range(k)]


# ------------------------------------------------------------------ Scale (scale_layer.cu)
def scale_view(shape, axis, num_axes):
    """-> (outer, dim, inner) of scale_layer.cpp for a canonical axis and num_axes (-1: to the end)"""
    end = len(shape) if num_axes == -1 else axis + num_axes
    if end == axis:  # a scalar scale applies from axis 0 (ScaleLayer::Reshape)
        axis = end = 0
    return (int(np.prod(shape[:axis], dtype=np.int64)), int(np.prod(shape[axis:end], dtype=np.int64)),
            int(np.prod(shape[end:], dtype=np.int64)))


def scale_forward(x, s, b, view, two_roundings=False):
    """-> y (float64) and its bound: x * s + b rounded once (one fma): half an ulp, plus the float64 rounding of the
    reference itself and the subnormal floor.  `two_roundings` (the product rounded to fp32 first) is a mutation."""
    outer, dim, inner = view
    x3 = np.asarray(x, np.float64).reshape(outer, dim, inner)
    s3 = np.asarray(s, np.float64).reshape(1, dim, 1)
    p = x3 * s3
    if two_roundings:
        p = p.astype(np.float32).astype(np.float64)
    y = p if b is None else p + np.asarray(b, np.float64).reshape(1, dim, 1)
    return y.reshape(np.shape(x)), (ulp(y) / 2 + 2.0 ** -53 * np.abs(y) + TINY).reshape(np.shape(x))


def scale_backward(x, s, dy, view):
    """-> ds, db (float64) and their bounds (one fma per product in scale_grad_kernel, bias_grad_kernel's order), and
    dx = fl(dy * s) in fp32"""
    outer, dim, inner = view
    x3, dy3 = np.asarray(x, np.float64).reshape(outer, dim, inner), np.asarray(dy, np.float64).reshape(outer, dim, inner)
    n = bias_grad_count(outer * inner)
    ds, db = (x3 * dy3).sum(axis=(0, 2)), dy3.sum(axis=(0, 2))
    bs, bb = n * U * np.abs(x3 * dy3).sum(axis=(0, 2)), n * U * np.abs(dy3).sum(axis=(0, 2))
    dx = (np.asarray(dy, np.float32).reshape(outer, dim, inner) * np.asarray(s, np.float32).reshape(1, dim, 1))
    return ds, bs + TINY, db, bb + TINY, dx.reshape(np.shape(x))


# ------------------------------------------------------------------ EuclideanLoss (euclidean_loss_layer.cpp)
def euclidean_loss(a, b, loss_weight=1.0):
    """-> loss (float64) and its bound: d = a - b and d^2 round (rel(3) each), the per-thread in-order sums and the
    8-level tree add ceil(count / 256) + 8 roundings, then / num and * loss_weight one each (/ 2 is exact)."""
    num = np.shape(a)[0]
    d = np.asarray(a, np.float64).ravel() - np.asarray(b, np.float64).ravel()
    dot = float(np.sum(d * d))
    loss = loss_weight * (dot / num / 2)
    adds = -(-d.size // BLOCK) + 8
    with np.errstate(invalid="ignore"):
        bound = abs(loss_weight) / num / 2 * (rel(3) + adds * U) * dot * (1 + rel(2)) + rel(2) * abs(loss) + TINY
    return loss, bound


def euclidean_grads32(a, b, loss_weight=1.0):
    """da = fl(fl(loss_weight / num) * fl(a - b)), db = fl(-fl(loss_weight / num) * fl(a - b)), as numpy float32"""
    alpha = np.float32(loss_weight) / np.float32(np.shape(a)[0])
    d = (np.asarray(a, np.float32).reshape(np.shape(a)[0], -1) - np.asarray(b, np.float32).reshape(np.shape(a)[0], -1))
    return (alpha * d).reshape(np.shape(a)), (-alpha * d).reshape(np.shape(b))


# ------------------------------------------------------------------ ContrastiveLoss (contrastive_loss_layer.cpp)
EPS_DIST = float(np.float32(1e-4))  # Dtype(1e-4)


def contrastive_loss(a, b, sim, margin=1.0, legacy=False, loss_weight=1.0, eps=EPS_DIST, legacy_grad_without_d=False):
    """-> loss, da, db, mdist (float64) with Caffe's CPU rules: static_cast<int>(sim) truncates; a dissimilar pair adds
    std::max(mdist, 0), which keeps a NaN mdist; its gradient is beta * d while mdist > 0 and an exact 0 otherwise
    (caffe_set), beta = -alpha (legacy) or -alpha * mdist / (dist + 1e-4).  `eps` and `legacy_grad_without_d` (the
    legacy gradient written as beta alone, as Caffe's GPU kernel does) are mutations for the bound tests."""
    n = np.shape(a)[0]
    d = np.asarray(a, np.float64).reshape(n, -1) - np.asarray(b, np.float64).reshape(n, -1)
    similar = np.trunc(np.asarray(sim, np.float64).ravel()) != 0
    alpha = loss_weight / n
    with np.errstate(invalid="ignore", over="ignore"):
        dsq = np.sum(d * d, axis=1)
        dist = np.sqrt(dsq)
        mdist = margin - (dsq if legacy else dist)
        m = np.where(mdist < 0, 0.0, mdist)
        per = np.where(similar, dsq, m if legacy else m * m)
        beta = np.full(n, -alpha) if legacy else -alpha * mdist / (dist + eps)
        scale = np.where(similar, alpha, np.where(mdist > 0, beta, 0.0))
        grad = scale[:, None] * d
        if legacy and legacy_grad_without_d:
            grad = np.where((~similar & (mdist > 0))[:, None], beta[:, None] * np.ones_like(d), grad)
        grad = np.where((similar | (mdist > 0))[:, None], grad, 0.0)  # caffe_set: not 0 * NaN
    loss = loss_weight * float(np.sum(per)) / n / 2
    return loss, grad.reshape(np.shape(a)), (-grad).reshape(np.shape(b)), mdist


def contrastive_bounds(a, b, sim, margin=1.0, legacy=False, loss_weight=1.0):
    """-> (loss bound, gradient bound, mdist bound), all first order in u.  dist_sq: d and d^2 round (rel(3)) and C - 1
    in-order adds; sqrt one more (half the relative error of dist_sq, plus u); mdist one subtraction.  A dissimilar
    pair's max(mdist, 0)^2 doubles mdist's relative error and rounds once.  The loss adds ceil(N / 256) + 8 roundings,
    then / N and * loss_weight.  The gradient: alpha, d and the product one rounding each; the non-legacy beta adds
    the product and quotient roundings, dist + 1e-4 (one) and mdist's error relative to its size."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _contrastive_bounds(a, b, sim, margin, legacy, loss_weight)


def _contrastive_bounds(a, b, sim, margin, legacy, loss_weight):
    n = np.shape(a)[0]
    d = np.asarray(a, np.float64).reshape(n, -1) - np.asarray(b, np.float64).reshape(n, -1)
    c = d.shape[1]
    similar = np.trunc(np.asarray(sim, np.float64).ravel()) != 0
    dsq = np.sum(d * d, axis=1)
    e_dsq = (rel(3) + (c - 1) * U) * dsq + c * TINY
    dist = np.sqrt(dsq)
    e_dist = np.where(dsq > 0, e_dsq / (2 * np.maximum(dist, FLT_MIN)), np.sqrt(e_dsq)) + U * dist
    mdist = margin - (dsq if legacy else dist)
    e_md = (e_dsq if legacy else e_dist) + U * np.abs(mdist)
    m = np.maximum(mdist, 0)
    e_per = np.where(similar, e_dsq, np.where(mdist > 0, e_md if legacy else 2 * m * e_md + e_md ** 2 + U * m * m, 0))
    per = np.where(similar, dsq, m if legacy else m * m)
    adds = -(-n // BLOCK) + 8
    alpha = abs(loss_weight) / n
    loss_bound = alpha / 2 * (e_per.sum() + adds * U * per.sum()) * (1 + rel(2)) + rel(2) * alpha / 2 * per.sum() + TINY
    den = dist + EPS_DIST
    g_rel = np.where(similar | legacy, rel(3), rel(6) + (e_dist + U * den) / den)
    g_abs = np.where(similar | legacy, 0.0, alpha * e_md / den)
    ref_scale = np.where(similar | legacy, alpha, alpha * np.abs(mdist) / den)
    on = similar | (mdist > 0)
    bound = np.where(on[:, None], (ref_scale * g_rel + g_abs)[:, None] * np.abs(d), 0.0) + 2 * TINY
    return loss_bound, bound.reshape(np.shape(a)), e_md


# ------------------------------------------------------------------ inputs
def dyadic(rng, shape, bits=3, top=4):
    """Integers in [-top, top] times 2^-bits: ties are real ties, and every sum of a few thousand products of such
    values is exact in fp32."""
    return np.asarray(rng.randint(-top, top + 1, size=shape) * 2.0 ** -bits).astype(np.float32)


def gaussian(rng, shape, scale=1.0):
    return np.asarray(rng.randn(*shape) * scale).astype(np.float32)
