"""An fp32 restatement of the built-in engine's GEMM core (native_producer.cu, DESIGN.md section 14), bit for bit.

Every output of `gemm_kernel` is one thread's chain acc = fmaf(A[m, k], B[k, n], acc) from +0 over k in increasing
order; a weight gradient splits k into split_chunk(K) products per partial, each partial its own chain, and
`reduce_partials_kernel` adds them as s = +0 + p0 + p1 + ..., then dst + s.  A bias is added once, __fadd_rn(v, b).
`bias_grad_kernel` runs 256 threads strided over the values in index order, then a fixed 8-level tree, then adds
the result into dst.  Terms a gather zeroes (padding, taps with no window) are real terms of the chain.  The zero
padding of the last 16-deep tile is fmaf(0, 0, acc): it only turns a -0 accumulator into +0, so it is left out and
zeros are compared by value.

`fma32` rounds a * b + c once, to nearest even, with fp32's subnormals, infinities and NaNs.  Inputs are fp32 arrays;
every result is an fp32 array.  `mutation` names a plausible wrong version of the arithmetic, for the tests that show
bit equality would catch it."""
import numpy as np

from producer_ops_ref import out_size, split_chunk, splits_of

F32 = np.float32
BLOCK = 256  # bias_grad_kernel's threads


def fma32(a, b, c):
    """fp32 fmaf(a, b, c), elementwise with broadcasting: a * b is exact in float64, TwoSum splits a * b + c into
    s + e exactly, and s rounds to fp32 directly unless it lies on an fp32 midpoint, where e decides the side."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        r = s.astype(F32)
        back = r.astype(np.float64)
        # the two fp32 neighbours around s (r is one of them); nextafter of +-0 gives the smallest subnormals
        below = back > s
        lo = np.where(below, np.nextafter(r, F32(-np.inf)), r)
        hi = np.where(below, r, np.nextafter(r, F32(np.inf)))
        lo64, hi64 = lo.astype(np.float64), hi.astype(np.float64)
        # s is finite and exact as s + e; a midpoint of two finite fp32 values, or the overflow threshold
        # FLT_MAX + ulp / 2 (which rounds to inf at a tie or above, to FLT_MAX below it)
        fin = np.isfinite(s) & np.isfinite(e) & (e != 0) & (back != s)
        both = np.isfinite(lo64) & np.isfinite(hi64)
        mid = fin & both & ((lo64 + hi64) / 2 == s)
        flt_max = float(np.finfo(F32).max)
        edge = fin & ~both & (np.abs(s) == flt_max + 2.0 ** 103)
        r = np.where(mid & (e > 0), hi, np.where(mid & (e < 0), lo, r))
        r = np.where(edge & (np.sign(e) != np.sign(s)), F32(flt_max) * np.sign(s).astype(F32), r)
    return np.asarray(r, F32)


def _step(a, b, acc, mutation):
    if mutation == "mul_add":
        with np.errstate(invalid="ignore", over="ignore"):
            return (acc + a * b).astype(F32)  # fp32 product rounded, then the add rounded
    return fma32(a, b, acc)


def chain(A, B, mutation=None):
    """C[m, n] = the fmaf chain over k of A[..., m, k] * B[..., k, n] from +0, in increasing k (leading axes batch)."""
    A, B = np.asarray(A, F32), np.asarray(B, F32)
    acc = np.zeros(A.shape[:-1] + B.shape[-1:], F32)
    ks = range(A.shape[-1])
    for k in (reversed(ks) if mutation == "reversed" else ks):
        acc = _step(A[..., :, k, None], B[..., k, None, :], acc, mutation)
    return acc


def gemm(A, B, bias=None, mutation=None):
    """One launch with kchunk = K: the chain, then __fadd_rn(v, bias[m]) (a per-row bias, as StoreNCHW's channel)."""
    c = chain(A, B, mutation)
    with np.errstate(invalid="ignore", over="ignore"):
        return c if bias is None else (c + np.asarray(bias, F32)[:, None]).astype(F32)


def gemm_split(A, B, mutation=None):
    """A weight gradient: dst (+0) + (+0 + p0 + p1 + ...) with p_z the chain over k in [z * chunk, (z + 1) * chunk),
    every partial computed at once (the loop runs over one chunk's length; the last partial stops at K)."""
    A, B = np.asarray(A, F32), np.asarray(B, F32)
    M, K = A.shape
    N = B.shape[1]
    if mutation == "unsplit":
        with np.errstate(invalid="ignore", over="ignore"):
            return (F32(0) + (F32(0) + chain(A, B))).astype(F32)
    chunk, splits = split_chunk(K), splits_of(K)
    chunk = min(chunk, K)
    last = K - (splits - 1) * chunk  # the last partial's length; the padding past K is never used
    pad = splits * chunk - K
    Ap = np.concatenate([A, np.zeros((M, pad), F32)], axis=1).reshape(M, splits, chunk).transpose(1, 0, 2)
    Bp = np.concatenate([B, np.zeros((pad, N), F32)], axis=0).reshape(splits, chunk, N)
    parts = np.zeros((splits, M, N), F32)
    for k in (range(chunk - 1, -1, -1) if mutation == "reversed" else range(chunk)):
        z = splits if k < last else splits - 1
        parts[:z] = _step(Ap[:z, :, k, None], Bp[:z, k, None, :], parts[:z], mutation)
    s = np.zeros((M, N), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for z in (range(splits - 1, -1, -1) if mutation == "partials_reversed" else range(splits)):
            s = (s + parts[z]).astype(F32)
        return (F32(0) + s).astype(F32)


def bias_grad(dy, N, C, HW):
    """bias_grad_kernel: per channel c, thread t adds dy[n, c, p] for i = n * HW + p = t, t + 256, ... from +0, the
    256 sums go through the tree sh[t] += sh[t + w] for w = 128 .. 1, and the root is added into dst = +0."""
    v = np.asarray(dy, F32).reshape(N, C, HW).transpose(1, 0, 2).reshape(C, N * HW)
    rounds = -(-v.shape[1] // BLOCK)
    v = np.concatenate([v, np.zeros((C, rounds * BLOCK - v.shape[1]), F32)], axis=1).reshape(C, rounds, BLOCK)
    s = np.zeros((C, BLOCK), F32)  # a thread past the end adds nothing; +0 added to a sum that is never -0 is a no-op
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(rounds):
            s = (s + v[:, r]).astype(F32)
        w = BLOCK // 2
        while w:
            s = np.concatenate([(s[:, :w] + s[:, w:2 * w]).astype(F32), s[:, w:]], axis=1)
            w //= 2
        return (F32(0) + s[:, 0]).astype(F32)


# ------------------------------------------------------------------ the gathers, as dense fp32 operands
def im2col(x, geo):
    """Im2col's B[k, j]: k = (ci * KH + kh) * KW + kw, j = (n * OH + oh) * OW + ow, zero outside the input."""
    x = np.asarray(x, F32)
    kh, kw, sh, sw, ph, pw = geo
    n, c, h, w = x.shape
    oh, ow = out_size(h, kh, sh, ph), out_size(w, kw, sw, pw)
    xp = np.zeros((n, c, h + 2 * ph + kh, w + 2 * pw + kw), F32)
    xp[:, :, ph:ph + h, pw:pw + w] = x
    cols = np.empty((c, kh, kw, n, oh, ow), F32)
    for i in range(kh):
        for j in range(kw):
            cols[:, i, j] = xp[:, :, i:i + sh * (oh - 1) + 1:sh, j:j + sw * (ow - 1) + 1:sw].transpose(1, 0, 2, 3)
    return cols.reshape(c * kh * kw, n * oh * ow)


def chan_major(dy):
    """ChanMajor's A[c, j] = dy[n, c, p], j = n * HW + p."""
    dy = np.asarray(dy, F32)
    return dy.reshape(dy.shape[0], dy.shape[1], -1).transpose(1, 0, 2).reshape(dy.shape[1], -1)


def weight_t(w):
    """WeightT's A[ci, k2] = W[co, ci, kh, kw], k2 = (co * KH + kh) * KW + kw."""
    w = np.asarray(w, F32)
    return w.transpose(1, 0, 2, 3).reshape(w.shape[1], -1)


def col2im_gather(dy, x_shape, geo):
    """Col2imGather's B[k2, j]: dy[n, co, oh, ow] at the output whose window puts tap (kh, kw) on input pixel j = (n * H
    + h) * W + w, i.e. h + PH - kh = oh * SH and w + PW - kw = ow * SW; zero where there is none."""
    dy = np.asarray(dy, F32)
    kh, kw, sh, sw, ph, pw = geo
    n, _, h, w = x_shape
    cout, oh, ow = dy.shape[1:]
    out = np.zeros((cout, kh, kw, n, h, w), F32)
    hh, ww = np.arange(h), np.arange(w)
    for i in range(kh):
        th = hh + ph - i
        okh = (th >= 0) & (th % sh == 0) & (th // sh < oh)
        for j in range(kw):
            tw = ww + pw - j
            okw = (tw >= 0) & (tw % sw == 0) & (tw // sw < ow)
            hs, ws = np.flatnonzero(okh), np.flatnonzero(okw)
            out[:, i, j][:, :, hs[:, None], ws[None, :]] = dy.transpose(1, 0, 2, 3)[
                :, :, (th[hs] // sh)[:, None], (tw[ws] // sw)[None, :]]
    return out.reshape(cout * kh * kw, n * h * w)


def _nchw(c, n, hw_shape):
    """C[m = channel, j = (n, pixel)] -> [N, C, H, W] (StoreNCHW)"""
    return np.ascontiguousarray(c.reshape(c.shape[0], n, *hw_shape).transpose(1, 0, 2, 3))


# ------------------------------------------------------------------ the six instantiations
def conv_forward(x, w, b, geo, mutation=None):
    """y = W * im2col(x) (+ bias): A = W [Cout, Cin KH KW], B = Im2col."""
    x, w = np.asarray(x, F32), np.asarray(w, F32)
    kh, kw, sh, sw, ph, pw = geo
    oh, ow = out_size(x.shape[2], kh, sh, ph), out_size(x.shape[3], kw, sw, pw)
    c = gemm(w.reshape(w.shape[0], -1), im2col(x, geo), b, mutation)
    return _nchw(c, x.shape[0], (oh, ow))


def conv_weight_grad(x, dy, geo, mutation=None):
    """dW [Cout, Cin, KH, KW] = dy * im2col(x)^T over N OH OW, split-K: A = ChanMajor(dy), B = Im2col transposed.
    dy may hold a subset of the output channels; dW then holds theirs."""
    kh, kw = geo[:2]
    g = gemm_split(chan_major(dy), im2col(x, geo).T, mutation)
    return g.reshape(np.shape(dy)[1], np.shape(x)[1], kh, kw)


def conv_data_grad(dy, w, b, x_shape, geo, mutation=None):
    """dx = W^T * dy gathered back to the input (+ bias): A = WeightT, B = Col2imGather."""
    c = gemm(weight_t(w), col2im_gather(dy, x_shape, geo), b, mutation)
    return _nchw(c, x_shape[0], x_shape[2:])


def ip_forward(x, w, b, mutation=None):
    """y[B, N] = x[B, K] w[N, K]^T (+ bias[n]): A = DenseRM x, B = DenseCM w, StoreRM."""
    x = np.asarray(x, F32).reshape(np.shape(x)[0], -1)
    c = chain(x, np.asarray(w, F32).T, mutation)
    with np.errstate(invalid="ignore", over="ignore"):
        return c if b is None else (c + np.asarray(b, F32)[None, :]).astype(F32)


def ip_weight_grad(x, dy, mutation=None):
    """dW[N, K] = dy^T x over the rows, split-K: A = DenseCM dy, B = DenseRM x."""
    x = np.asarray(x, F32).reshape(np.shape(x)[0], -1)
    return gemm_split(np.asarray(dy, F32).T, x, mutation)


def ip_data_grad(dy, w, x_shape, mutation=None):
    """dx[B, K] = dy[B, N] w[N, K]: A = DenseRM dy, B = DenseRM w."""
    return chain(dy, w, mutation).reshape(x_shape)


# ------------------------------------------------------------------ Deconvolution: the convolution from top to bottom
def deconv_forward(x, w, b, geo, out_hw, mutation=None):
    """the convolution's data gradient of x, with the bias: w is [Cin, Cout, KH, KW], the convolution's [Cout, Cin]"""
    n = np.shape(x)[0]
    return conv_data_grad(x, w, b, (n, np.shape(w)[1]) + tuple(out_hw), geo, mutation)


def deconv_weight_grad(x, dy, geo, mutation=None):
    """the convolution's weight gradient with the top's gradient dy as its input and the bottom x as its dy"""
    return conv_weight_grad(dy, x, geo, mutation)


def deconv_data_grad(dy, w, geo, mutation=None):
    """the convolution's forward of dy, without the bias"""
    return conv_forward(dy, w, None, geo, mutation)
