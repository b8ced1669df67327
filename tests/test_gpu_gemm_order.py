"""The built-in engine's GEMM core (DESIGN.md section 14) on the GPU, bit for bit against gemm_ref.py's fp32
restatement of its order: each output one fmaf chain over k in increasing order from +0, no TF32, weight gradients
split in split_chunk(K) products per partial with the partials added in chunk order and then once into the gradient,
bias gradients in bias_grad_kernel's order.  The float64 checks of test_gpu_producer_ops.py cannot see a changed
order or rounding, and their bounds grow with depth; this one can, down to the widened split-K chunks past 131,072
products.

Each op runs once through test_gpu_producer_ops.py's injector harness with B = 0: the probe returns y itself, and
y is also the top gradient the op receives.  y, dW, db and dx are compared with the restatement fed that very y:
equal values (the injectors return a zero up to its sign), NaN exactly where the restatement has NaN.  The deepest
cases restate a few images or output channels of what the GPU computed in full."""
import numpy as np
import pytest

import gemm_ref as G
import producer_ops_ref as R
from autoencoder_ops_ref import deconv_out
from test_gpu_producer_ops import _conv_layer, _engine, _same

pytestmark = pytest.mark.gpu

F32 = np.float32
BUDGET = 4e7  # fma32 element-steps per restated product: a few seconds on one CPU core


def _take(total, cost_each):
    """how many images (or channels) of `total` to restate within BUDGET"""
    return max(1, min(total, int(BUDGET // max(cost_each, 1))))


def _specials(rng, x, w, family):
    """specials-x: the first image (row) of x scaled into the subnormal range, the last holding NaN, +inf and -inf, and
    zeros, -0 and subnormals in x and w.  specials-w: NaN in w's first output channel, +-inf in its second, and zeros,
    -0 and subnormals in x and w.  Each special reaches only the outputs that read it."""
    tiny = 2.0 ** -149
    for a in (x, w):
        f = a.reshape(-1)
        i = rng.choice(f.size, size=max(1, f.size // 10), replace=False)
        f[i[0::3]] = 0.0
        f[i[1::3]] = -0.0
        f[i[2::3]] = (rng.integers(-2 ** 20, 2 ** 20, i[2::3].size) * tiny).astype(F32)
    if family == "specials-x":
        x[0] = (x[0].astype(np.float64) * 2.0 ** -130).astype(F32)
        last = x[-1].reshape(-1)
        j = rng.choice(last.size, size=min(3, last.size), replace=False)
        last[j] = np.array([np.nan, np.inf, -np.inf], F32)[:j.size]
    else:
        w[0].reshape(-1)[rng.integers(w[0].size)] = np.nan
        if w.shape[0] > 1:
            k = rng.choice(w[1].size, size=min(2, w[1].size), replace=False)
            w[1].reshape(-1)[k] = np.array([np.inf, -np.inf], F32)[:k.size]


def _draw(seed, x_shape, w_shape, k, nb, family):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(x_shape).astype(F32)
    w = (rng.standard_normal(w_shape) / np.sqrt(k)).astype(F32)
    b = (rng.standard_normal(nb) * 0.1).astype(F32)
    if family != "gaussian":
        _specials(rng, x, w, family)
    return x, w, b


# --------------------------------------------------------------------------- Convolution
CONV_FAMILIES = ["gaussian", "specials-x", "specials-w"]
CONV_CASES = [(*c, "gaussian") for c in [  # (N, Cin, H, W, Cout, (kh, kw, sh, sw, ph, pw), bias)
    # Cout across the 64-row tile edge
    (2, 4, 5, 5, 1, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 63, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 64, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 65, (2, 2, 1, 1, 0, 0), False),
    (2, 4, 5, 5, 130, (2, 2, 1, 1, 0, 0), True),
    # N OH OW across the 64-column tile edge
    (1, 2, 7, 9, 3, (1, 1, 1, 1, 0, 0), True),
    (1, 2, 8, 8, 3, (1, 1, 1, 1, 0, 0), True),
    (1, 2, 5, 13, 3, (1, 1, 1, 1, 0, 0), True),
    # K = Cin kh kw across the 16-deep k-step
    (2, 1, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 15, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 16, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 17, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 57, 5, 5, 3, (3, 3, 1, 1, 1, 1), True),  # K = 513
    # the gathers
    (2, 2, 6, 6, 3, (3, 3, 1, 1, 3, 3), True),  # pad >= kernel
    (2, 3, 8, 8, 4, (2, 2, 3, 3, 0, 0), True),  # stride > kernel
    (2, 3, 9, 10, 4, (3, 5, 1, 2, 1, 2), True),  # non-square kernel and strides
    (2, 3, 5, 5, 4, (5, 5, 1, 1, 0, 0), True),  # kernel = input
    (1, 3, 35, 35, 5, (11, 11, 4, 4, 0, 0), True),
    # the weight gradient's depth N OH OW: one chunk, two, seven, 256 of 512, then the widened chunks
    (1, 2, 7, 73, 3, (1, 1, 1, 1, 0, 0), True),  # 511
    (2, 2, 16, 16, 3, (1, 1, 1, 1, 0, 0), True),  # 512
    (1, 2, 27, 19, 3, (1, 1, 1, 1, 0, 0), True),  # 513
    (2, 3, 40, 40, 4, (3, 3, 1, 1, 1, 1), True),  # 3,200
    (128, 2, 32, 32, 3, (3, 3, 1, 1, 1, 1), True),  # 131,072: 256 chunks of 512
    (1, 2, 3, 43691, 3, (1, 1, 1, 1, 0, 0), True),  # 131,073: 249 chunks of 528
    (256, 3, 32, 32, 32, (5, 5, 1, 1, 2, 2), True),  # CIFAR-10-quick conv1 at batch 256: 262,144 in 256 of 1,024
    (256, 2, 55, 55, 3, (1, 1, 1, 1, 0, 0), True),  # 774,400: 255 chunks of 3,040
]] + [(2, 3, 6, 6, 4, (3, 3, 1, 1, 1, 1), True, f) for f in CONV_FAMILIES[1:]]


def conv_inputs(n, cin, h, w, cout, geo, bias, family):
    x, wt, b = _draw(n * 1000 + cin * 100 + cout + h + w + sum(geo), (n, cin, h, w), (cout, cin, geo[0], geo[1]),
                     cin * geo[0] * geo[1], cout, family)
    return x, wt, (b if bias else None), geo


@pytest.mark.parametrize("n,cin,h,w,cout,geo,bias,family", CONV_CASES)
def test_convolution_bit_for_bit(cos, tmp_path, n, cin, h, w, cout, geo, bias, family):
    x, wt, b, geo = conv_inputs(n, cin, h, w, cout, geo, bias, family)
    kh, kw, sh, sw, ph, pw = geo
    oh, ow = R.out_size(h, kh, sh, ph), R.out_size(w, kw, sw, pw)
    shape = (n, cout, oh, ow)
    r = _engine(cos, tmp_path, [x], _conv_layer("c", "x0", "y", cout, geo, bias), [wt] + ([b] if bias else []), shape,
                np.zeros(shape, F32))
    y = r["d"]
    k = cin * kh * kw
    m = _take(n, cout * oh * ow * k)
    _same(y[:m], G.conv_forward(x[:m], wt, b, geo), "y")
    c = _take(cout, k * n * oh * ow)
    _same(r["grads"][0][:c], G.conv_weight_grad(x, y[:, :c], geo), "dW")
    if bias:
        _same(r["grads"][1], G.bias_grad(y, n, cout, oh * ow), "db")
    m = _take(n, cin * h * w * cout * kh * kw)
    _same(r["dx"][0][:m], G.conv_data_grad(y[:m], wt, None, (m, cin, h, w), geo), "dx")


# --------------------------------------------------------------------------- InnerProduct
IP_CASES = [(*c, "gaussian") for c in [  # (bottom shape, num_output, bias)
    ((1, 16), 64, True), ((64, 15), 1, True), ((65, 17), 65, True), ((1100, 17), 129, True),
    ((7, 33), 64, True), ((65, 1000), 129, True), ((4, 9216), 64, True),  # CaffeNet fc6's fan-in
    ((5, 3, 4, 5), 10, False),  # a 4-D bottom: K = 60
    # the weight gradient's depth: the rows
    ((511, 7), 5, True), ((512, 7), 5, True), ((513, 7), 5, True), ((3200, 7), 5, True), ((131073, 5), 3, True),
]] + [((6, 40), 5, True, f) for f in CONV_FAMILIES[1:]]


def ip_inputs(shape, nout, bias, family):
    k = int(np.prod(shape[1:]))
    x, w, b = _draw(int(np.prod(shape)) + nout, shape, (nout, k), k, nout, family)
    return x, w, (b if bias else None)


@pytest.mark.parametrize("shape,nout,bias,family", IP_CASES)
def test_inner_product_bit_for_bit(cos, tmp_path, shape, nout, bias, family):
    x, wt, b = ip_inputs(shape, nout, bias, family)
    rows = shape[0]
    body = ('layer { name: "ip" type: "InnerProduct" bottom: "x0" top: "y" inner_product_param { '
            f'num_output: {nout} bias_term: {"true" if bias else "false"} }} }}\n')
    r = _engine(cos, tmp_path, [x], body, [wt] + ([b] if bias else []), (rows, nout), np.zeros((rows, nout), F32))
    y = r["d"]
    _same(y, G.ip_forward(x, wt, b), "y")
    _same(r["grads"][0], G.ip_weight_grad(x, y), "dW")
    if bias:
        _same(r["grads"][1], G.bias_grad(y, rows, nout, 1), "db")
    _same(r["dx"][0], G.ip_data_grad(y, wt, x.shape), "dx")


# --------------------------------------------------------------------------- Deconvolution
DECONV_CASES = [(*c, "gaussian") for c in [  # (N, Cin, H, W, Cout, (kh, kw, sh, sw, ph, pw), bias)
    (2, 4, 7, 7, 3, (4, 4, 2, 2, 1, 1), True),  # the conv autoencoder's upsampling
    (2, 3, 4, 4, 2, (2, 2, 3, 3, 0, 0), True),  # stride > kernel: some outputs are the bias alone
    (2, 3, 5, 6, 4, (2, 5, 1, 2, 0, 2), True),  # non-square kernel and strides
    (1, 5, 3, 3, 65, (2, 2, 2, 2, 0, 0), True),  # Cout across the 64-row tile edge of the forward
    (1, 65, 3, 3, 2, (1, 1, 1, 1, 0, 0), False),  # Cin across it for the data gradient
    (2, 2, 20, 20, 2, (3, 3, 1, 1, 1, 1), True),  # N H W = 800: two chunks of the weight gradient
    (128, 2, 32, 33, 2, (2, 2, 2, 2, 0, 0), True),  # N H W = 135,168: 256 widened chunks of 528
]] + [(2, 3, 5, 5, 4, (3, 3, 1, 1, 1, 1), True, f) for f in CONV_FAMILIES[1:]]


def deconv_inputs(n, cin, h, w, cout, geo, bias, family):
    x, wt, b = _draw(n * 1000 + cin * 100 + cout + h + w + sum(geo) + 7, (n, cin, h, w), (cin, cout, geo[0], geo[1]),
                     cin * geo[0] * geo[1], cout, family)
    return x, wt, (b if bias else None), geo


@pytest.mark.parametrize("n,cin,h,w,cout,geo,bias,family", DECONV_CASES)
def test_deconvolution_bit_for_bit(cos, tmp_path, n, cin, h, w, cout, geo, bias, family):
    x, wt, b, geo = deconv_inputs(n, cin, h, w, cout, geo, bias, family)
    kh, kw, sh, sw, ph, pw = geo
    oh, ow = deconv_out(h, kh, sh, ph), deconv_out(w, kw, sw, pw)
    shape = (n, cout, oh, ow)
    body = (f'layer {{ name: "dc" type: "Deconvolution" bottom: "x0" top: "y" convolution_param {{ num_output: {cout} '
            f'kernel_h: {kh} kernel_w: {kw} stride_h: {sh} stride_w: {sw} pad_h: {ph} pad_w: {pw} '
            f'bias_term: {"true" if bias else "false"} }} }}\n')
    r = _engine(cos, tmp_path, [x], body, [wt] + ([b] if bias else []), shape, np.zeros(shape, F32))
    y = r["d"]
    m = _take(n, cout * oh * ow * cin * kh * kw)
    _same(y[:m], G.deconv_forward(x[:m], wt, b, geo, (oh, ow)), "y")
    c = _take(cin, cout * kh * kw * n * h * w)
    _same(r["grads"][0][:c], G.deconv_weight_grad(x[:, :c], y, geo), "dW")
    if bias:
        _same(r["grads"][1], G.bias_grad(y, n, cout, oh * ow), "db")
    m = _take(n, cin * h * w * cout * kh * kw)
    _same(r["dx"][0][:m], G.deconv_data_grad(y[:m], wt, geo), "dx")
