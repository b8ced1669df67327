"""Float64 references, with Caffe's rules, of the built-in producer's Deconvolution and SigmoidCrossEntropyLoss ops
(DESIGN.md section 14), and per-element error bounds from each op's rounding count, in producer_ops_ref.py's terms.
No bound is fitted to GPU output."""
import numpy as np

import producer_ops_ref as R
from producer_ops_ref import U


# ------------------------------------------------------------------ Deconvolution (deconv_layer.cpp)
def deconv_out(h, k, s, p):
    return s * (h - 1) + k - 2 * p


def deconv_forward(x, w, b, geo):
    """The transpose of the convolution from the top to the bottom: w is [Cin, Cout, kh, kw], x [N, Cin, H, W]."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    kh, kw, sh, sw, ph, pw = geo
    n, cin, h, wd = x.shape
    shape = (n, w.shape[1], deconv_out(h, kh, sh, ph), deconv_out(wd, kw, sw, pw))
    cols = np.einsum("ck,ncp->nkp", w.reshape(cin, -1), x.reshape(n, cin, -1))
    y = R.col2im(cols, shape, *geo)
    if b is not None:
        y = y + np.asarray(b, np.float64)[None, :, None, None]
    return y


def deconv_backward(x, w, dy, geo):
    """-> dW, db, dx of the deconvolution for top gradient dy: dx is the convolution of dy by w, dW[ci, k] the sum over
    (n, p) of x[n, ci, p] * im2col(dy)[n, k, p]."""
    x, w, dy = (np.asarray(v, np.float64) for v in (x, w, dy))
    cols, _, _ = R.im2col(dy, *geo)
    dw = np.einsum("ncp,nkp->ck", x.reshape(x.shape[0], x.shape[1], -1), cols).reshape(w.shape)
    return dw, dy.sum(axis=(0, 2, 3)), R.conv_forward(dy, w, None, geo)


def deconv_bounds(x, w, b, dy, geo):
    """Per-element bounds of (y, dW, db, dx): the forward sums Cin kh kw products (+ the bias), the weight gradient
    N H W products in split-K chunks, the bias gradient N OH OW values, the data gradient Cout kh kw products."""
    cin, cout, kh, kw = w.shape
    n_pix = x.shape[0] * x.shape[2] * x.shape[3]
    ay = deconv_forward(np.abs(x), np.abs(w), None if b is None else np.abs(b), geo)
    adw, adb, adx = deconv_backward(np.abs(x), np.abs(w), np.abs(dy), geo)
    n_out = dy.shape[0] * dy.shape[2] * dy.shape[3]
    return ((cin * kh * kw + (b is not None)) * U * ay, (n_pix + R.splits_of(n_pix) + 1) * U * adw,
            R.bias_grad_count(n_out) * U * adb, cout * kh * kw * U * adx)


# ------------------------------------------------------------------ SigmoidCrossEntropyLoss
# (sigmoid_cross_entropy_loss_layer.cpp)
BLOCK, SMS = 256, 132  # native_producer.cu: kThreads, and grid_for's cap of kTargetSms * 16 blocks


def blocks_of(count):
    return max(1, min(-(-count // BLOCK), SMS * 16))


def sigmoid_xent(x, t, num, loss_weight=1.0):
    """-> (loss, dx): loss_weight * sum(-(x (t - [x >= 0]) - log(1 + exp(-|x|)))) / num, dx = (sigmoid(x) - t) *
    loss_weight / num."""
    x, t = np.asarray(x, np.float64), np.asarray(t, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        pos = (x >= 0).astype(np.float64)
        term = x * (t - pos) - np.log1p(np.exp(-np.abs(x)))
        return loss_weight * float(-term.sum()) / num, (R.sigmoid_forward(x) - t) * (loss_weight / num)


def sigmoid_xent_bounds(x, t, num, loss_weight=1.0):
    """(loss bound, per-element dx bound).  Per element: x (t - p) takes two roundings; exp(-|x|) is within 2 ulp, 1 +
    e one rounding, the log 1 ulp of a result below log 2 and passes the relative error of 1 + e on as an absolute one:
    under 6U in all; the difference one more rounding.  The sum: each thread's run, the 8-level tree, the block-order
    sum of the partials, the division by num and the product with loss_weight.  dx: the Sigmoid op's bound, one
    rounding for the difference, one for loss_weight / num and one for the product."""
    x, t = np.asarray(x, np.float64), np.asarray(t, np.float64)
    count = x.size
    blocks = blocks_of(count)
    with np.errstate(invalid="ignore", over="ignore"):
        pos = (x >= 0).astype(np.float64)
        b = np.abs(x * (t - pos))
        term = np.abs(x * (t - pos) - np.log1p(np.exp(-np.abs(x))))
        elem = 2 * U * b + 6 * U + U * term
        steps = -(-count // (blocks * BLOCK)) + 8 + blocks + 2
        lw = abs(loss_weight) / num
        loss_bound = lw * (elem.sum() + steps * U * (term.sum() + elem.sum()))
        s64 = R.sigmoid_forward(x)
        sb = R.sigmoid_forward_bound(x)
        d = np.abs(s64 - t) + sb
        dx_bound = lw * (sb + 4 * U * d) + R.TINY
    return loss_bound, dx_bound
