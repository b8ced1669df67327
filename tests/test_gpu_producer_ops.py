"""The built-in producer's Convolution, fused conv + ReLU + MAX pool, Pooling, InnerProduct, ReLU, Sigmoid and
SoftmaxWithLoss ops (DESIGN.md section 14) on the GPU, element by element against the float64 references of
producer_ops_ref.py, on dyadic inputs (every result exact in fp32, so compared by equality, except for the ops that
divide) and on Gaussian inputs (against per-element rounding bounds).

Each case is one tiny net run once.  The op reads each bottom x0, x1, ... from an input injector of its own, an
all-zeros Input through Scale {axis: 0 num_axes: -1 bias_term: true} with scale 1 and bias X: x = fmaf(0, 1, X) = X
exactly, and the injector's bias gradient is the op's data gradient bit for bit.  The op's top y meets a second
injector of bias B in EuclideanLoss with loss_weight N = y.shape[0], so alpha = N / N = 1 and the op receives
d = fl(y - B) as its top gradient, which the second injector's bias gradient returns as -d exactly.
B = fl(y64 - e) for a chosen e, so d is small and known.  Both injectors return their values exactly up to the sign of
a zero (bias_grad_kernel starts its sums from +0), so exact results are compared by value."""
import numpy as np
import pytest
import torch

import producer_ops_ref as R
from gpu_util import assert_bits_equal, to_host

pytestmark = pytest.mark.gpu

F32 = np.float32
INJECT = "scale_param { axis: 0 num_axes: -1 bias_term: true }"


def _dims(shape):
    return "shape { " + " ".join(f"dim: {d}" for d in shape) + " }"


def _net(xs, body, weights=(), out_shape=None, B=None, staged=None, top="y"):
    """-> (prototxt, learnable blobs in layout order) of Input -> one injector per bottom (z<i> -> x<i>) -> `body`
    [-> probe + EuclideanLoss]; `staged` (name -> array) adds Input tops the body reads as they are."""
    staged = staged or {}
    shapes = [np.shape(x) for x in xs] + ([out_shape] if out_shape is not None else []) + [v.shape for v in staged.values()]
    tops = [f"z{i}" for i in range(len(xs))] + (["zo"] if out_shape is not None else []) + list(staged)
    text = ('name: "t" layer { name: "in" type: "Input" ' + " ".join(f'top: "{t}"' for t in tops) +
            " input_param { " + " ".join(_dims(s) for s in shapes) + " } }\n" +
            "".join(f'layer {{ name: "inj{i}" type: "Scale" bottom: "z{i}" top: "x{i}" {INJECT} }}\n'
                    for i in range(len(xs))) + body + "\n")
    ws = [w for x in xs for w in (np.ones(np.shape(x), F32), np.asarray(x, F32))] + [np.asarray(w, F32) for w in weights]
    if out_shape is not None:
        text += (f'layer {{ name: "probe" type: "Scale" bottom: "zo" top: "b" {INJECT} }}\n'
                 f'layer {{ name: "loss" type: "EuclideanLoss" bottom: "{top}" bottom: "b" loss_weight: {out_shape[0]} }}\n')
        ws += [np.ones(out_shape, F32), np.asarray(B, F32)]
    return text, ws


def _engine(cos, tmp_path, xs, body, weights=(), out_shape=None, B=None, staged=None, top="y"):
    """Runs Input -> injectors -> `body` (reads "x0", "x1", ..., writes `top`) [-> probe + EuclideanLoss] once on the
    engine.  -> dict(dx (one per injected bottom), grads (one per op weight), data (the op weights after the call),
    d (None without a probe), loss)."""
    staged = staged or {}
    text, ws = _net(xs, body, weights, out_shape, B, staged, top)
    inputs = [np.zeros(np.shape(x), F32) for x in xs] + ([np.zeros(out_shape, F32)] if out_shape is not None else [])
    inputs += [np.asarray(v, F32) for v in staged.values()]
    (tmp_path / "net.prototxt").write_text(text)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        flat = np.concatenate([w.ravel() for w in ws])
        assert net.param_count() == flat.size
        net.data().copy_(torch.from_numpy(flat).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(v).cuda() for v in inputs], loss.data_ptr()), net.last_error()
        assert net.synchronize(), net.last_error()
        g, w, l32 = to_host(net.diff()), to_host(net.data()), float(loss.item())
    finally:
        net.deallocate()
    parts, data, off = [], [], 0
    for v in ws:
        parts.append(g[off:off + v.size].reshape(v.shape))
        data.append(w[off:off + v.size].reshape(v.shape))
        off += v.size
    dx = parts[1:2 * len(xs):2]
    for ds, dxi in zip(parts[0:2 * len(xs):2], dx):
        assert not ds[np.isfinite(dxi)].any(), "an injector's scale gradient is dy * 0"
    op = slice(2 * len(xs), 2 * len(xs) + len(weights))
    out = dict(dx=dx, grads=parts[op], data=data[op], loss=l32, d=None)
    if out_shape is not None:
        out["d"] = -parts[-1]
        assert not parts[-2][np.isfinite(out["d"])].any(), "the probe's scale gradient is -d * 0"
    return out


def _probe(y64, rng, family):
    """B = fl(y64 - e): the top gradient the op receives is then e, up to the forward's rounding."""
    e = R.dyadic(rng, y64.shape) if family == "dyadic" else R.gaussian(rng, y64.shape)
    with np.errstate(invalid="ignore", over="ignore"):
        return (y64 - e).astype(F32)


def _close(got, ref, bound, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    nan = np.isnan(ref)
    if not np.array_equal(np.isnan(got), nan):
        i = int(np.flatnonzero(np.isnan(got) != nan)[0])
        raise AssertionError(f"{what}: NaN positions differ; first at {i}: {got.flat[i]!r}, want {ref.flat[i]!r}")
    with np.errstate(invalid="ignore"):
        err = np.where(got == ref, 0.0, np.abs(got - ref))[~nan]  # equal infinities match
    b = np.broadcast_to(bound, ref.shape)[~nan]
    if err.size and not np.all(err <= b):
        i = int(np.argmax(err - b))
        raise AssertionError(f"{what}: {int(np.sum(err > b))} of {err.size} elements outside the bound; worst "
                             f"{np.flatnonzero(~nan)[i]}: |{got[~nan][i]!r} - {ref[~nan][i]!r}| = {err[i]:.3e} > "
                             f"{b[i]:.3e}")


def _equal(got, ref, what):
    """exact results: equal values (either sign of zero), NaN where the reference has NaN"""
    ref = np.asarray(ref, np.float64)
    assert np.array_equal(np.asarray(ref, F32).astype(np.float64), ref, equal_nan=True), f"{what}: not exact in fp32"
    _close(got, ref, 0.0, what)


def _check(got, ref, bound, what, exact):
    if exact:
        _equal(got, ref, what)
    else:
        _close(got, ref, bound, what)


def _same(got, want, what):
    """equal fp32 values (either sign of zero), NaN where `want` has NaN"""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements differ; first {got[bad][0]!r} vs {want[bad][0]!r}"


def _forward(d, y64, B, bound, what, exact):
    """The probe's d = fl(y32 - B) against y64 - B: equal to fl(y64 - B) when y is exact, else within the forward
    bound plus half an ulp of d."""
    with np.errstate(invalid="ignore", over="ignore"):
        if exact:
            _same(d, np.asarray(y64, F32) - B, what)
        else:
            _close(d, y64 - B.astype(np.float64), bound + R.ulp(d) / 2, what)


FAMILIES = ["dyadic", "gaussian"]


# --------------------------------------------------------------------------- the harness itself
def test_harness_is_exact(cos, tmp_path):
    rng = np.random.RandomState(0)
    X, B = R.gaussian(rng, (3, 2, 4, 5)), R.gaussian(rng, (3, 2, 4, 5))
    r = _engine(cos, tmp_path, [X], "", out_shape=X.shape, B=B, top="x0")
    d = X - B
    assert d.all()  # no zero, so no sign of a zero to lose: bit for bit
    assert_bits_equal(r["d"], d, "the probe returns d = fl(X - B)")
    assert_bits_equal(r["dx"][0], d, "the injector returns its top's gradient")


# --------------------------------------------------------------------------- Convolution
def _conv_layer(name, bottom, top, cout, geo, bias=True):
    kh, kw, sh, sw, ph, pw = geo
    return (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{top}" convolution_param {{ '
            f'num_output: {cout} kernel_h: {kh} kernel_w: {kw} stride_h: {sh} stride_w: {sw} pad_h: {ph} pad_w: {pw} '
            f'bias_term: {"true" if bias else "false"} }} }}\n')


CONV_CASES = [  # (N, Cin, H, W, Cout, (kh, kw, sh, sw, ph, pw), bias)
    (2, 3, 8, 8, 4, (1, 1, 1, 1, 0, 0), True),
    (2, 3, 9, 9, 5, (3, 3, 1, 1, 1, 1), True),
    (2, 2, 11, 11, 3, (5, 5, 1, 1, 2, 2), True),
    (1, 3, 27, 27, 4, (11, 11, 4, 4, 0, 0), True),
    (2, 3, 9, 10, 4, (3, 5, 1, 2, 1, 2), True),
    (2, 2, 9, 9, 3, (1, 7, 1, 1, 0, 3), True),
    (2, 2, 9, 9, 3, (7, 1, 1, 1, 3, 0), True),
    (2, 3, 8, 8, 4, (2, 2, 3, 3, 0, 0), True),  # stride > kernel: some pixels get no gradient
    (2, 2, 6, 6, 3, (3, 3, 1, 1, 3, 3), True),  # pad >= kernel: whole windows in the padding
    (2, 3, 5, 5, 4, (5, 5, 1, 1, 0, 0), True),  # kernel = input
    (2, 3, 13, 7, 4, (3, 3, 2, 1, 1, 0), True),  # odd, non-square
    (2, 3, 6, 6, 5, (3, 3, 1, 1, 1, 1), False),
    # Cout across the 64-row tile edge (K = 16)
    (2, 4, 5, 5, 1, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 63, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 64, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 65, (2, 2, 1, 1, 0, 0), True),
    (2, 4, 5, 5, 130, (2, 2, 1, 1, 0, 0), True),
    # K = Cin kh kw across the 16-deep k-step
    (2, 1, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 15, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 16, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 17, 6, 6, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 57, 5, 5, 3, (3, 3, 1, 1, 1, 1), True),  # K = 513
    # N OH OW across the 64-column tile edge, and several 512-chunks of the weight gradient with a partial last one
    (1, 2, 1, 1, 3, (1, 1, 1, 1, 0, 0), True),
    (1, 2, 7, 9, 3, (1, 1, 1, 1, 0, 0), True),
    (1, 2, 8, 8, 3, (1, 1, 1, 1, 0, 0), True),
    (1, 2, 5, 13, 3, (1, 1, 1, 1, 0, 0), True),
    (2, 3, 40, 40, 4, (3, 3, 1, 1, 1, 1), True),  # N OH OW = 3200 = 6 * 512 + 128
    # past 256 chunks of 512 the chunk widens: N OH OW = 131,073 (249 chunks of 528), 774,400 (255 of 3,040)
    (1, 2, 3, 43691, 3, (1, 1, 1, 1, 0, 0), True),
    (256, 2, 55, 55, 3, (1, 1, 1, 1, 0, 0), True),
]


def _exact_depth(abs_sum, unit, what):
    """On dyadic inputs a sum is exact in fp32 in any order while sum |terms| stays below 2^24 of the terms' unit: every
    partial sum is then a multiple of the unit below 2^24 units.  The deep reductions assert it before comparing."""
    assert np.max(abs_sum) < 2 ** 24 * unit, f"{what}: sum |terms| = {np.max(abs_sum) / unit:.0f} units, not exact"


def _conv_params(rng, family, cin, cout, kh, kw, bias):
    k = cin * kh * kw
    if family == "dyadic":
        w, b = R.dyadic(rng, (cout, cin, kh, kw), bits=4), R.dyadic(rng, (cout,), bits=7)
    else:
        w, b = R.gaussian(rng, (cout, cin, kh, kw), 1 / np.sqrt(k)), R.gaussian(rng, (cout,), 0.1)
    return w, (b if bias else None)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n,cin,h,w,cout,geo,bias", CONV_CASES)
def test_convolution(cos, tmp_path, family, n, cin, h, w, cout, geo, bias):
    rng = np.random.RandomState(n * 1000 + cin * 100 + cout + h + sum(geo))
    exact = family == "dyadic"
    x = R.dyadic(rng, (n, cin, h, w)) if exact else R.gaussian(rng, (n, cin, h, w))
    wt, b = _conv_params(rng, family, cin, cout, geo[0], geo[1], bias)
    y64 = R.conv_forward(x, wt, b, geo)
    B = _probe(y64, rng, family)
    r = _engine(cos, tmp_path, [x], _conv_layer("c", "x0", "y", cout, geo, bias),
                [wt] + ([b] if bias else []), y64.shape, B)
    d = r["d"]
    if exact:  # x and d are dyadic in 2^-3, so dW's terms are in 2^-6 and db's in 2^-3
        adw, adb, _ = R.conv_backward(np.abs(x), np.abs(wt), np.abs(d), geo)
        _exact_depth(adw, 2.0 ** -6, "dW")
        _exact_depth(adb, 2.0 ** -3, "db")
    by, bw, bb, bx = R.conv_bounds(x, wt, b, d, geo)
    _forward(d, y64, B, by, "y", exact)
    dw, db, dx = R.conv_backward(x, wt, d, geo)
    _check(r["grads"][0], dw, bw, "dW", exact)
    if bias:
        _check(r["grads"][1], db, bb, "db", exact)
    _check(r["dx"][0], dx, bx, "dx", exact)
    assert np.abs(dw).max() > 0 and np.abs(dx).max() > 0


# --------------------------------------------------------------------------- fused conv + ReLU + MAX pool
def _fused_body(geo, cout, k, s, relu_first):
    pool = f'pooling_param {{ pool: MAX kernel_size: {k} stride: {s} }}'
    if relu_first:
        return (_conv_layer("c", "x0", "c", cout, geo) + 'layer { name: "r" type: "ReLU" bottom: "c" top: "c" }\n'
                f'layer {{ name: "p" type: "Pooling" bottom: "c" top: "y" {pool} }}\n')
    return (_conv_layer("c", "x0", "c", cout, geo) + f'layer {{ name: "p" type: "Pooling" bottom: "c" top: "y" {pool} }}\n'
            'layer { name: "r" type: "ReLU" bottom: "y" top: "y" }\n')


FUSED_CASES = [  # (H, W, k, s): the conv is 3x3 pad 1, so its output is H x W
    (8, 8, 1, 1), (7, 9, 1, 2), (8, 8, 2, 2), (9, 9, 3, 2), (7, 8, 3, 1), (13, 11, 5, 3), (16, 15, 15, 1),
    (6, 6, 2, 3),  # Caffe counts an empty last window: 3 pooled rows, the third starting at row 6
    (6, 6, 1, 2),  # the same on the per-element path (k = 1): 4 pooled rows
]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("relu_first", [True, False], ids=["relu-pool", "pool-relu"])
@pytest.mark.parametrize("h,w,k,s", FUSED_CASES)
def test_conv_relu_max_pool(cos, tmp_path, family, relu_first, h, w, k, s):
    rng = np.random.RandomState(h * 100 + w + 10 * k + s)
    exact = family == "dyadic"
    n, cin, cout, geo = 2, 3, 5, (3, 3, 1, 1, 1, 1)
    x = R.dyadic(rng, (n, cin, h, w)) if exact else R.gaussian(rng, (n, cin, h, w))
    wt, b = _conv_params(rng, family, cin, cout, 3, 3, True)
    b[0] = -64.0  # channel 0: every window all negative
    pgeo = (k, k, s, s, 0, 0)
    z = R.conv_forward(x, wt, b, geo)
    bz = R.conv_bounds(x, wt, b, np.zeros_like(z), geo)[0]
    if not exact:  # the Gaussian inputs were drawn so that every ReLU and MAX decision is clear of rounding
        assert np.all(np.abs(z) > bz) and R.max_decisions_hold(z, bz, pgeo)
    if relu_first:
        y64, idx = R.pool_forward(np.maximum(z, 0), "MAX", pgeo)
    else:
        p, idx = R.pool_forward(z, "MAX", pgeo)
        y64 = np.maximum(p, 0)
    B = _probe(y64, rng, family)
    r = _engine(cos, tmp_path, [x], _fused_body(geo, cout, k, s, relu_first), [wt, b], y64.shape, B)
    d = r["d"]
    by = np.maximum(R.pool_forward(bz, "MAX", pgeo)[0], 0.0)  # an empty window: -FLT_MAX, exact
    _forward(d, y64, B, by, "y", exact)
    dp = np.where(y64 > 0, d, 0.0) if not relu_first else np.asarray(d, np.float64)
    dz = R.pool_backward(dp, z.shape, "MAX", pgeo, idx)
    if relu_first:
        dz = np.where(z > 0, dz, 0.0)
    dw, db, dx = R.conv_backward(x, wt, dz, geo)
    # dz, routed back through the windows, adds up to ceil(k/s)^2 values of d (one rounding each), then the conv
    # backward rounds as in test_convolution
    nwin = (-(-k // s)) ** 2
    adz = R.pool_backward(np.abs(dp), z.shape, "MAX", pgeo, idx)
    _, bw, bb, bx = R.conv_bounds(x, wt, b, adz, geo)
    adw, adb, adx = R.conv_backward(np.abs(x), np.abs(wt), adz, geo)
    bw, bb, bx = bw + nwin * R.U * adw, bb + nwin * R.U * adb, bx + nwin * R.U * adx
    _check(r["grads"][0], dw, bw, "dW", exact)
    _check(r["grads"][1], db, bb, "db", exact)
    _check(r["dx"][0], dx, bx, "dx", exact)
    assert np.abs(dw).max() > 0


# --------------------------------------------------------------------------- Pooling
POOL_CASES = [  # (H, W, pooling_param, (kh, kw, sh, sw, ph, pw))
    (6, 6, "kernel_size: 2 stride: 2", (2, 2, 2, 2, 0, 0)),
    (8, 8, "kernel_size: 3 stride: 2", (3, 3, 2, 2, 0, 0)),  # the last window clipped
    (7, 7, "kernel_size: 3 stride: 2 pad: 1", (3, 3, 2, 2, 1, 1)),
    (5, 6, "kernel_size: 3 stride: 1 pad: 1", (3, 3, 1, 1, 1, 1)),
    (6, 6, "kernel_size: 2 stride: 3", (2, 2, 3, 3, 0, 0)),  # an empty last window
    (7, 6, "kernel_h: 3 kernel_w: 2 stride_h: 2 stride_w: 1 pad_h: 1 pad_w: 0", (3, 2, 2, 1, 1, 0)),
    (7, 5, "global_pooling: true", (7, 5, 1, 1, 0, 0)),
    (17, 20, "kernel_size: 17 stride: 1", (17, 17, 1, 1, 0, 0)),
    (4, 4, "kernel_size: 5 stride: 2", (5, 5, 2, 2, 0, 0)),  # kernel > input
]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("method", ["MAX", "AVE"])
@pytest.mark.parametrize("h,w,param,geo", POOL_CASES)
def test_pooling(cos, tmp_path, family, method, h, w, param, geo):
    rng = np.random.RandomState(h * 100 + w + len(param))
    exact = family == "dyadic"
    x = R.dyadic(rng, (2, 3, h, w), top=2) if exact else R.gaussian(rng, (2, 3, h, w))  # top 2: many ties
    y64, idx = R.pool_forward(x, method, geo)
    B = _probe(y64, rng, family)
    body = f'layer {{ name: "p" type: "Pooling" bottom: "x0" top: "y" pooling_param {{ pool: {method} {param} }} }}\n'
    r = _engine(cos, tmp_path, [x], body, (), y64.shape, B)
    d = r["d"]
    by, bx = R.pool_bounds(x, d, method, geo)
    _forward(d, y64, B, by, "y", method == "MAX")
    dx = R.pool_backward(d, x.shape, method, geo, idx)
    _check(r["dx"][0], dx, bx, "dx", exact and method == "MAX")


# --------------------------------------------------------------------------- InnerProduct
IP_CASES = [  # (bottom shape, N, bias)
    ((1, 16), 10, True), ((7, 15), 1, True), ((64, 17), 64, True), ((65, 16), 65, True), ((7, 1), 129, True),
    ((600, 1000), 10, True), ((1100, 17), 65, True), ((65, 1000), 129, True),
    ((5, 3, 4, 5), 10, True),  # a 4-D bottom: K = 60
    ((64, 15), 10, False),
    ((131073, 5), 3, True), ((774400, 3), 2, True),  # rows past 256 chunks of 512: the widened chunks
]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape,nout,bias", IP_CASES)
def test_inner_product(cos, tmp_path, family, shape, nout, bias):
    rng = np.random.RandomState(int(np.prod(shape)) + nout)
    exact = family == "dyadic"
    k = int(np.prod(shape[1:]))
    x = R.dyadic(rng, shape) if exact else R.gaussian(rng, shape)
    if exact:
        wt, b = R.dyadic(rng, (nout, k), bits=4), R.dyadic(rng, (nout,), bits=7)
    else:
        wt, b = R.gaussian(rng, (nout, k), 1 / np.sqrt(k)), R.gaussian(rng, (nout,), 0.1)
    b = b if bias else None
    y64 = R.ip_forward(x, wt, b)
    B = _probe(y64, rng, family)
    body = ('layer { name: "ip" type: "InnerProduct" bottom: "x0" top: "y" inner_product_param { '
            f'num_output: {nout} bias_term: {"true" if bias else "false"} }} }}\n')
    r = _engine(cos, tmp_path, [x], body, [wt] + ([b] if bias else []), y64.shape, B)
    d = r["d"]
    if exact:
        adw, adb, _ = R.ip_backward(np.abs(x), np.abs(wt), np.abs(d))
        _exact_depth(adw, 2.0 ** -6, "dW")
        _exact_depth(adb, 2.0 ** -3, "db")
    by, bw, bb, bx = R.ip_bounds(x, wt, b, d)
    _forward(d, y64, B, by, "y", exact)
    dw, db, dx = R.ip_backward(x, wt, d)
    _check(r["grads"][0], dw, bw, "dW", exact)
    if bias:
        _check(r["grads"][1], db, bb, "db", exact)
    _check(r["dx"][0], dx, bx, "dx", exact)


# --------------------------------------------------------------------------- ReLU and Sigmoid
@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in-place"])
@pytest.mark.parametrize("slope", [0.0, 0.1, -0.25])
def test_relu(cos, tmp_path, slope, in_place):
    rng = np.random.RandomState(7)
    x = R.gaussian(rng, (3, 4, 5, 6))
    x[:, :, ::2, ::3] = 0.0  # exact zeros: not > 0
    y = R.relu_forward32(x, slope)
    B = _probe(y.astype(np.float64), rng, "gaussian")
    top = "x0" if in_place else "y"
    body = f'layer {{ name: "r" type: "ReLU" bottom: "x0" top: "{top}" relu_param {{ negative_slope: {slope} }} }}\n'
    r = _engine(cos, tmp_path, [x], body, (), y.shape, B, top=top)
    _same(r["d"], y - B, "y")
    # relu_layer.cu reads the bottom's memory: the output itself when in place (so a negative slope passes dy)
    _same(r["dx"][0], R.relu_backward32(y if in_place else x, r["d"], slope), "dx")


@pytest.mark.parametrize("in_place", [False, True], ids=["separate", "in-place"])
def test_sigmoid(cos, tmp_path, in_place):
    rng = np.random.RandomState(8)
    x = np.concatenate([rng.uniform(-30, 30, 300), rng.randn(60) * 1e-30, [0.0, 30.0, -30.0, 8.0, -8.0]])
    x = x.astype(F32).reshape(5, 73)
    top = "x0" if in_place else "y"
    r = _engine(cos, tmp_path, [x], f'layer {{ name: "s" type: "Sigmoid" bottom: "x0" top: "{top}" }}\n', (),
                x.shape, np.zeros(x.shape, F32), top=top)
    y32 = r["d"]  # B = 0: the probe returns y itself, and the op's top gradient is y
    _close(y32, R.sigmoid_forward(x), R.sigmoid_forward_bound(x), "y")
    _close(r["dx"][0], R.sigmoid_backward(y32, y32), R.sigmoid_backward_bound(y32, y32), "dx")


# --------------------------------------------------------------------------- SoftmaxWithLoss
SOFTMAX_CASES = [  # (scores shape, softmax_param, axis, loss_weight, logit scale)
    ((1, 10), "", 1, 1.0, 3.0), ((7, 2), "", 1, 1.0, 3.0), ((256, 10), "", 1, 1.0, 3.0),
    ((257, 1000), "", 1, 1.0, 3.0), ((1000, 10), "", 1, 1.0, 3.0), ((7, 1), "", 1, 1.0, 3.0),
    ((3, 1000), "", 1, 1.0, 3.0),
    ((2, 5, 3, 4), "", 1, 1.0, 3.0),  # spatial scores: inner = 12
    ((2, 3, 5, 4), "softmax_param { axis: 2 }", 2, 1.0, 3.0),
    ((2, 3, 4, 6), "softmax_param { axis: -1 }", 3, 1.0, 3.0),
    ((40, 10), "", 1, 0.5, 3.0), ((3, 7, 2), "", 1, 3.0, 3.0),
    ((300, 10), "", 1, 1.0, 1e4),  # logits spread by 10^4: p underflows, and the FLT_MIN clamp caps the loss
]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape,param,axis,lw,spread", SOFTMAX_CASES)
def test_softmax_loss(cos, tmp_path, family, shape, param, axis, lw, spread):
    rng = np.random.RandomState(int(np.prod(shape)) + axis)
    if family == "dyadic":  # integer logits (times 4096 for the spread case)
        x = R.dyadic(rng, shape, bits=0 if spread < 1e3 else -12)
    else:
        x = R.gaussian(rng, shape, spread)
    c = shape[axis]
    lab_shape = tuple(s for i, s in enumerate(shape) if i != axis)
    label = (rng.randint(0, c, size=lab_shape) + 0.7 * (rng.rand(*lab_shape) < 0.5)).astype(F32)  # 2.7 reads as 2
    lw_text = "" if lw == 1.0 else f" loss_weight: {lw}"
    body = f'layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "x0" bottom: "label" top: "l"{lw_text} {param} }}\n'
    r = _engine(cos, tmp_path, [x], body, staged={"label": label.reshape(-1)})
    l64, dx64 = R.softmax_loss(x, label, axis, lw)
    lb, dxb = R.softmax_loss_bounds(x, label, axis, lw)
    assert abs(r["loss"] - l64) <= lb, (r["loss"], l64, lb)
    _close(r["dx"][0], dx64, dxb, "dx")
    if spread > 1e3:  # most rows' p[label] underflows: their loss is -log(FLT_MIN) = 87.3365
        assert 0.5 * -np.log(R.FLT_MIN) < l64 <= -np.log(R.FLT_MIN)
