"""Host checks of producer_ops_ref.py, the float64 references and rounding bounds that test_gpu_producer_ops.py holds
the built-in producer's ops to: the references agree with torch float64 wherever Caffe and PyTorch agree, follow
Caffe on hand-worked cases where they do not, and each bound admits an fp32 evaluation of its op while rejecting
references that are subtly wrong.  Also the plan's side of the same ops: the softmax axis, when conv + ReLU + MAX pool
fuses, and the pooling setups Caffe refuses (DESIGN.md section 14)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import producer_ops_ref as R

F32 = np.float32


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


# --------------------------------------------------------------------------- references against torch float64
@pytest.mark.parametrize("geo", [(1, 1, 1, 1, 0, 0), (3, 3, 1, 1, 1, 1), (3, 5, 1, 2, 1, 2), (2, 2, 3, 3, 0, 0),
                                 (3, 3, 1, 1, 3, 3), (11, 11, 4, 4, 0, 0), (1, 7, 1, 1, 0, 3)])
def test_convolution_reference_matches_torch(geo):
    rng = np.random.RandomState(sum(geo))
    x, w, b = R.gaussian(rng, (2, 3, 13, 15)), R.gaussian(rng, (4, 3, geo[0], geo[1])), R.gaussian(rng, (4,))
    y = R.conv_forward(x, w, b, geo)
    xt, wt, bt = _t(x), _t(w), _t(b)
    yt = F.conv2d(xt, wt, bt, stride=geo[2:4], padding=geo[4:6])
    np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-12, atol=1e-12)
    dy = rng.randn(*y.shape)
    yt.backward(torch.from_numpy(dy))
    for got, ref in zip(R.conv_backward(x, w, dy, geo), (wt.grad, bt.grad, xt.grad)):
        np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("geo", [(2, 2, 2, 2, 0, 0), (3, 3, 2, 2, 1, 1), (3, 3, 1, 1, 1, 1), (3, 2, 2, 1, 1, 0)])
def test_unclipped_pooling_matches_torch(geo):
    """Caffe's ceil rule is ceil_mode, and its AVE divisor count_include_pad, wherever no window starts past H + pad."""
    rng = np.random.RandomState(geo[0] * 10 + geo[2])
    x = R.gaussian(rng, (2, 3, 8, 7) if geo[1] == 2 and geo[3] == 1 else (2, 3, 7, 7))
    for method, fn in (("MAX", F.max_pool2d), ("AVE", F.avg_pool2d)):
        xt = _t(x)
        yt = fn(xt, geo[:2], geo[2:4], geo[4:6], ceil_mode=True)
        y, idx = R.pool_forward(x, method, geo)
        assert y.shape == yt.shape
        np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-12)
        dy = rng.randn(*y.shape)
        yt.backward(torch.from_numpy(dy))
        np.testing.assert_allclose(R.pool_backward(dy, x.shape, method, geo, idx), xt.grad.numpy(), rtol=1e-12,
                                   atol=1e-15)


@pytest.mark.parametrize("shape,axis", [((7, 10), 1), ((2, 5, 3, 4), 1), ((2, 3, 5, 4), 2), ((2, 3, 4, 6), -1)])
def test_softmax_loss_reference_matches_torch(shape, axis):
    rng = np.random.RandomState(len(shape) + axis)
    x = R.gaussian(rng, shape, 3)
    lab_shape = tuple(s for i, s in enumerate(shape) if i != axis % len(shape))
    label = rng.randint(0, shape[axis], size=lab_shape)
    loss, dx = R.softmax_loss(x, label.astype(F32) + F32(0.5), axis, 3.0)  # x.5 labels read as x
    xt = _t(x)
    lt = 3.0 * F.cross_entropy(torch.movedim(xt, axis, 1), torch.from_numpy(label))
    lt.backward()
    assert abs(loss - lt.item()) <= 1e-12 * abs(lt.item())
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-10, atol=1e-15)


def test_inner_product_reference_matches_torch():
    rng = np.random.RandomState(1)
    x, w, b = R.gaussian(rng, (5, 3, 2, 2)), R.gaussian(rng, (7, 12)), R.gaussian(rng, (7,))
    xt, wt, bt = _t(x), _t(w), _t(b)
    yt = F.linear(xt.reshape(5, -1), wt, bt)
    np.testing.assert_allclose(R.ip_forward(x, w, b), yt.detach().numpy(), rtol=1e-12)
    dy = rng.randn(5, 7)
    yt.backward(torch.from_numpy(dy))
    for got, ref in zip(R.ip_backward(x, w, dy), (wt.grad, bt.grad, xt.grad)):
        np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12)


# --------------------------------------------------------------------------- Caffe's rules, hand-worked
def test_pooled_size_is_caffes():
    assert R.pooled_size(6, 2, 3, 0) == 3  # ceil(4 / 3) + 1: the third window starts at row 6, past the edge
    assert R.pooled_size(8, 3, 2, 0) == 4  # the last window clipped to rows 6..7
    assert R.pooled_size(7, 3, 2, 1) == 4  # ceil(6 / 2) + 1 = 4; it starts at 5 < 7 + 1: kept
    assert R.pooled_size(5, 2, 2, 1) == 3  # ceil(5 / 2) + 1 = 4, but the fourth would start at 6 >= 5 + 1: clipped
    assert R.pooled_size(4, 5, 2, 0) == 1  # kernel > input: ceil(-1 / 2) + 1


def test_empty_windows_and_the_ave_divisor():
    x = np.arange(36, dtype=F32).reshape(1, 1, 6, 6) - 40  # all negative
    y, idx = R.pool_forward(x, "MAX", (2, 2, 3, 3, 0, 0))
    assert y.shape == (1, 1, 3, 3)
    assert y[0, 0, 0, 0] == -33 and idx[0, 0, 0, 0] == 7  # max of rows 0..1, cols 0..1: x[1, 1]
    assert np.all(y[0, 0, 2] == -R.FLT_MAX) and np.all(y[0, 0, :, 2] == -R.FLT_MAX) and np.all(idx[0, 0, 2] == -1)
    a, _ = R.pool_forward(x, "AVE", (2, 2, 3, 3, 0, 0))
    assert np.isnan(a[0, 0, 2, 0]) and a[0, 0, 0, 0] == (-40 - 39 - 34 - 33) / 4  # 0 / 0 for the empty window
    # k 2, s 4 on 7 rows: ceil(5 / 4) + 1 = 3 windows, the third at row 8 with divisor (7 - 8) * 2: 0 / -2 = -0
    a, _ = R.pool_forward(np.ones((1, 1, 7, 7)), "AVE", (2, 2, 4, 4, 0, 0))
    assert a.shape == (1, 1, 3, 3) and np.all(a[0, 0, :2, :2] == 1)
    assert a[0, 0, 2, 0] == 0 and np.signbit(a[0, 0, 2, 0]) and a[0, 0, 2, 2] == 0 and not np.signbit(a[0, 0, 2, 2])
    # pad 1, 3x3 stride 2 on 7x7: the corner window holds 4 pixels, divided by 9 (clipped to H + pad, not H); the
    # last holds rows 5..6 of a window that ends at H + pad = 8, so 3 x 3 = 9 too
    a, _ = R.pool_forward(np.ones((1, 1, 7, 7)), "AVE", (3, 3, 2, 2, 1, 1))
    assert a[0, 0, 0, 0] == 4 / 9 and a[0, 0, 0, 1] == 6 / 9 and a[0, 0, 3, 3] == 4 / 9
    dx = R.pool_backward(np.ones((1, 1, 4, 4)), (1, 1, 7, 7), "AVE", (3, 3, 2, 2, 1, 1))
    assert dx[0, 0, 0, 0] == 1 / 9 and dx[0, 0, 1, 1] == 4 / 9


def test_max_pool_first_maximum_wins():
    x = np.array([[[[1, 3, 3], [3, 0, 3], [2, 3, 1]]]], F32)
    y, idx = R.pool_forward(x, "MAX", (2, 2, 1, 1, 0, 0))
    assert np.all(y == 3) and idx[0, 0].tolist() == [[1, 1], [3, 5]]
    _, last = R.pool_forward(x, "MAX", (2, 2, 1, 1, 0, 0), last_max_wins=True)
    assert last[0, 0].tolist() == [[3, 5], [7, 7]]
    dx = R.pool_backward(np.array([[[[1.0, 2.0], [4.0, 8.0]]]]), x.shape, "MAX", (2, 2, 1, 1, 0, 0), idx)
    assert dx[0, 0].tolist() == [[0, 3, 0], [4, 0, 8], [0, 0, 0]]


def test_softmax_loss_clamps_and_truncates_labels():
    x = np.array([[0.0, 200.0], [5.0, 5.0]], F32)
    loss, dx = R.softmax_loss(x, np.array([0.9, 1.7], F32))  # labels 0 and 1
    assert loss == pytest.approx((-np.log(R.FLT_MIN) + np.log(2)) / 2)
    assert dx[0].tolist() == pytest.approx([-0.5, 0.5]) and dx[1].tolist() == pytest.approx([0.25, -0.25])


# --------------------------------------------------------------------------- the bounds: admit fp32, reject mutations
def _outside(got, ref, bound):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return np.abs(got - ref) > bound


def _admits(got32, ref, bound, what):
    assert not _outside(got32, ref, bound).any(), f"{what}: the bound rejects an fp32 evaluation"


def _rejects(mutated, ref, bound, what):
    """Most elements the mutation changes fall outside the bound (rounded to fp32, as a kernel would return them)."""
    m = np.asarray(np.asarray(mutated, F32), np.float64)
    changed = np.abs(m - ref) > 0
    assert changed.any(), f"{what}: the mutation changes nothing"
    frac = _outside(m, ref, bound)[changed].mean()
    assert frac > 0.5, f"{what}: only {frac:.2f} of the changed elements fall outside the bound"


def _shift(x):  # x[h + 1, w + 1]: what a kernel with the pad one too small reads
    s = np.zeros_like(x)
    s[:, :, :-1, :-1] = x[:, :, 1:, 1:]
    return s


def _overlap(a, b):
    h, w = min(a.shape[2], b.shape[2]), min(a.shape[3], b.shape[3])
    return a[:, :, :h, :w], b[:, :, :h, :w]


def test_convolution_bounds_admit_fp32_and_reject_mutations():
    rng = np.random.RandomState(3)
    geo = (3, 5, 1, 2, 1, 2)
    x, w, b = R.gaussian(rng, (3, 3, 30, 40)), R.gaussian(rng, (4, 3, 3, 5), 0.25), R.gaussian(rng, (4,), 0.1)
    y = R.conv_forward(x, w, b, geo)
    dy = R.gaussian(rng, y.shape)
    by, bw, bb, bx = R.conv_bounds(x, w, b, dy, geo)
    dw, db, dx = R.conv_backward(x, w, dy, geo)
    xt, wt, bt = (torch.tensor(v, requires_grad=True) for v in (x, w, b))
    yt = F.conv2d(xt, wt, bt, stride=geo[2:4], padding=geo[4:6])
    yt.backward(torch.from_numpy(dy))
    _admits(yt.detach().numpy(), y, by, "y")
    _admits(wt.grad.numpy(), dw, bw, "dW")
    _admits(bt.grad.numpy(), db, bb, "db")
    _admits(xt.grad.numpy(), dx, bx, "dx")
    _rejects(R.conv_forward(_shift(x), w, b, geo), y, by, "pad off by one")
    # the same weights read as a 5 x 3 kernel, and the strides exchanged: compared where the outputs overlap
    for mgeo, mw, what in (((5, 3) + geo[2:], w.reshape(4, 3, 5, 3), "kh and kw swapped"),
                           (geo[:2] + (geo[3], geo[2]) + geo[4:], w, "sh and sw swapped")):
        m, r = _overlap(R.conv_forward(x, mw, b, mgeo), y)
        _rejects(m, r, by[:, :, :r.shape[2], :r.shape[3]], what)
    n_pix = dy.shape[0] * dy.shape[2] * dy.shape[3]
    chunk = R.split_chunk(n_pix)
    assert R.splits_of(n_pix) > 2 and n_pix % chunk
    flat = dy.transpose(1, 0, 2, 3).reshape(4, -1).copy()
    flat[:, (R.splits_of(n_pix) - 1) * chunk:] = 0  # j = (n OH + oh) OW + ow past the last full chunk
    dropped = flat.reshape(4, dy.shape[0], dy.shape[2], dy.shape[3]).transpose(1, 0, 2, 3)
    _rejects(R.conv_backward(x, w, dropped, geo)[0], dw, bw, "the last k-chunk dropped")


def test_inner_product_bounds_admit_fp32_and_reject_a_dropped_chunk():
    rng = np.random.RandomState(4)
    x, w, b = R.gaussian(rng, (1100, 17)), R.gaussian(rng, (65, 17), 0.25), R.gaussian(rng, (65,), 0.1)
    dy = R.gaussian(rng, (1100, 65))
    by, bw, bb, bx = R.ip_bounds(x, w, b, dy)
    xt, wt, bt = (torch.tensor(v, requires_grad=True) for v in (x, w, b))
    yt = F.linear(xt, wt, bt)
    yt.backward(torch.from_numpy(dy))
    dw, db, dx = R.ip_backward(x, w, dy)
    _admits(yt.detach().numpy(), R.ip_forward(x, w, b), by, "y")
    for got, ref, bound, what in ((wt.grad, dw, bw, "dW"), (bt.grad, db, bb, "db"), (xt.grad, dx, bx, "dx")):
        _admits(got.numpy(), ref, bound, what)
    cut = dy.copy()
    cut[(R.splits_of(1100) - 1) * R.split_chunk(1100):] = 0
    _rejects(R.ip_backward(x, w, cut)[0], dw, bw, "the last k-chunk dropped")


def _ave32(x, geo):
    """AVE pooling evaluated in fp32 as pooling_layer.cu does: the window summed in row-major order, then divided"""
    y64, _ = R.pool_forward(x, "AVE", geo)
    y = np.zeros(y64.shape, F32)
    n, c, h, w = x.shape
    for i, j, hs, he, ws, we, size in R._windows(h, w, *geo):
        s = np.zeros((n, c), F32)
        for a in range(hs, he):
            for b in range(ws, we):
                s = s + x[:, :, a, b]
        with np.errstate(invalid="ignore", divide="ignore"):
            y[:, :, i, j] = s / F32(size)
    return y


def test_pooling_bounds_admit_fp32_and_reject_mutations():
    rng = np.random.RandomState(5)
    geo = (3, 3, 2, 2, 1, 1)
    x = R.gaussian(rng, (2, 3, 7, 7))
    y, _ = R.pool_forward(x, "AVE", geo)
    dy = R.gaussian(rng, y.shape)
    by, bx = R.pool_bounds(x, dy, "AVE", geo)
    _admits(_ave32(x, geo), y, by, "AVE y")
    _rejects(R.pool_forward(x, "AVE", geo, divisor_clipped_to_h=True)[0], y, by, "AVE divisor clipped to H")
    dx = R.pool_backward(dy, x.shape, "AVE", geo)
    _rejects(R.pool_backward(dy, x.shape, "AVE", geo, divisor_clipped_to_h=True), dx, bx,
             "AVE backward divisor clipped to H")
    xt = torch.tensor(x, requires_grad=True)
    F.avg_pool2d(xt, 3, 2, 1).backward(torch.from_numpy(dy))  # no window reaches past H + pad here
    _admits(xt.grad.numpy(), dx, bx, "AVE dx")
    # MAX on ties (dyadic inputs): the last maximum winning routes dy elsewhere
    xd = R.dyadic(rng, (2, 3, 7, 7), top=1)
    y, idx = R.pool_forward(xd, "MAX", geo)
    dy = R.gaussian(rng, y.shape)
    _, bx = R.pool_bounds(xd, dy, "MAX", geo)
    dx = R.pool_backward(dy, xd.shape, "MAX", geo, idx)
    _, last = R.pool_forward(xd, "MAX", geo, last_max_wins=True)
    _rejects(R.pool_backward(dy, xd.shape, "MAX", geo, last), dx, bx, "the last maximum wins a tie")


def test_softmax_bounds_admit_fp32_and_reject_the_wrong_axis():
    rng = np.random.RandomState(6)
    x = R.gaussian(rng, (3, 5, 5, 4), 3)
    label = rng.randint(0, 5, size=(3, 5, 4)).astype(F32)
    loss, dx = R.softmax_loss(x, label, 1, 3.0)
    lb, dxb = R.softmax_loss_bounds(x, label, 1, 3.0)
    xt = torch.tensor(x, requires_grad=True)
    lt = 3 * F.cross_entropy(xt, torch.from_numpy(label).long())
    lt.backward()
    assert abs(float(lt) - loss) <= lb
    _admits(xt.grad.numpy(), dx, dxb, "dx")
    _, wrong = R.softmax_loss(x, label, 2, 3.0)  # axes 1 and 2 both hold 5: the same labels fit either
    _rejects(wrong, dx, dxb, "softmax over axis 2 instead of 1")


def test_sigmoid_bounds_admit_fp32():
    x = np.concatenate([np.linspace(-30, 30, 1001), [1e-30, -1e-30, 0]]).astype(F32)
    y32 = F32(0.5) * np.tanh(F32(0.5) * x) + F32(0.5)  # sigmoid_layer.cu's formula in fp32
    _admits(y32, R.sigmoid_forward(x), R.sigmoid_forward_bound(x), "y")
    _rejects(0.5 * np.tanh(x.astype(np.float64)) + 0.5, R.sigmoid_forward(x), R.sigmoid_forward_bound(x),
             "tanh(x) for tanh(x / 2)")


# --------------------------------------------------------------------------- the plan
def _plan(cos, tmp_path, shape, body):
    p = tmp_path / "net.prototxt"
    dims = " ".join(f"dim: {d}" for d in shape)
    p.write_text(f'name: "t" layer {{ name: "in" type: "Input" top: "x" top: "label" input_param {{ shape {{ {dims} }} '
                 f'shape {{ dim: {shape[0]} }} }} }}\n' + body)
    return cos.native_producer_plan(str(p))


def _ops(text):
    return [" ".join(line.split()[2:4]) for line in text.splitlines() if line.startswith("op ")]


def _softmax_net(param, label_count):
    return ('layer { name: "c" type: "Convolution" bottom: "x" top: "s" convolution_param { num_output: 4 '
            'kernel_size: 1 } }\n'
            f'layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "s" bottom: "label" top: "l" {param} }}\n')


@pytest.mark.parametrize("param,axis", [("", 1), ("softmax_param { axis: 1 }", 1), ("softmax_param { axis: 2 }", 2),
                                        ("softmax_param { axis: -1 }", 3), ("softmax_param { axis: -4 }", 0)])
def test_plan_shows_the_softmax_axis(cos, tmp_path, param, axis):
    shape = (2, 3, 5, 6)
    out = (2, 4, 5, 6)
    rows = int(np.prod(out)) // out[axis]
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "in" type: "Input" top: "x" top: "label" input_param { shape { '
                 + " ".join(f"dim: {d}" for d in shape) + f' }} shape {{ dim: {rows} }} }} }}\n' + _softmax_net(param, rows))
    line = [ln for ln in cos.native_producer_plan(str(p)).splitlines() if " SoftmaxWithLoss " in ln][0]
    assert f" axis={axis} label=1 loss_weight=1" in line


@pytest.mark.parametrize("axis", [4, -5])
def test_plan_refuses_an_out_of_range_softmax_axis(cos, tmp_path, axis):
    with pytest.raises(cos.CosError, match=rf"layer 'loss' \(SoftmaxWithLoss\): axis {axis} out of range for 4-D Blob"):
        _plan(cos, tmp_path, (2, 3, 5, 6), _softmax_net(f"softmax_param {{ axis: {axis} }}", 2))


def test_plan_refuses_labels_that_do_not_match_the_axis(cos, tmp_path):
    # axis 2: 2 * 4 * 6 = 48 rows of 5 classes, but the label holds 2
    with pytest.raises(cos.CosError, match=r"label count 2 does not match the 48 rows of the scores along axis 2"):
        _plan(cos, tmp_path, (2, 3, 5, 6), _softmax_net("softmax_param { axis: 2 }", 2))


def _fusion_net(h, k, s, relu_first):
    conv = ('layer { name: "c" type: "Convolution" bottom: "x" top: "c" convolution_param { num_output: 4 '
            'kernel_size: 3 pad: 1 } }\n')
    pool = f'layer {{ name: "p" type: "Pooling" bottom: "c" top: "c2" pooling_param {{ pool: MAX kernel_size: {k} stride: {s} }} }}\n'
    relu = 'layer { name: "r" type: "ReLU" bottom: "c" top: "c" }\n'
    if relu_first:
        body = conv + relu + pool
    else:
        body = conv + pool + relu.replace('"c"', '"c2"')
    return body + ('layer { name: "ip" type: "InnerProduct" bottom: "c2" top: "ip" inner_product_param { num_output: 3 } }\n'
                   'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "l" }\n')


@pytest.mark.parametrize("relu_first", [True, False], ids=["relu-pool", "pool-relu"])
@pytest.mark.parametrize("h,k,s,fused", [
    (6, 2, 3, False),  # Caffe: ceil(4 / 3) + 1 = 3 pooled rows, the third starting at row 6: empty
    (6, 1, 2, False),  # ceil(5 / 2) + 1 = 4, the fourth starting at row 6
    (7, 2, 3, True),  # ceil(5 / 3) + 1 = 3, the third starting at row 6 < 7
    (32, 3, 2, True),  # CIFAR-10-quick's pool1
    (8, 2, 2, True), (5, 1, 2, True), (16, 15, 1, True)])
def test_plan_fuses_only_without_empty_windows(cos, tmp_path, relu_first, h, k, s, fused):
    ops = _ops(_plan(cos, tmp_path, (2, 3, h, h), _fusion_net(h, k, s, relu_first)))
    if fused:
        assert ops[0] == ("ConvBiasReLUMaxPool c+r+p" if relu_first else "ConvBiasReLUMaxPool c+p+r"), ops
        assert ops[1] == "InnerProduct ip"
    else:
        order = ["ReLU r", "Pooling(MAX) p"] if relu_first else ["Pooling(MAX) p", "ReLU r"]
        assert ops[:3] == ["Convolution c"] + order, ops


@pytest.mark.parametrize("param,match", [
    ("pool: MAX kernel_size: 3 pad: 3", r"Check failed: pad_h_ < kernel_h_ \(3 vs. 3\)"),
    ("pool: AVE kernel_h: 3 kernel_w: 2 pad_h: 1 pad_w: 2", r"Check failed: pad_w_ < kernel_w_ \(2 vs. 2\)"),
    ("pool: AVE global_pooling: true pad: 1", r"With Global_pooling: true; only pad = 0 and stride = 1"),
    ("pool: AVE global_pooling: true stride: 2", r"With Global_pooling: true; only pad = 0 and stride = 1"),
    ("pool: MAX global_pooling: true kernel_size: 3", r"With Global_pooling: true Filter size cannot specified"),
    ("pool: MAX global_pooling: true kernel_h: 3 kernel_w: 3", r"With Global_pooling: true Filter size cannot specified"),
])
def test_pooling_setups_caffe_refuses(cos, tmp_path, param, match):
    body = (f'layer {{ name: "p" type: "Pooling" bottom: "x" top: "p" pooling_param {{ {param} }} }}\n'
            'layer { name: "ip" type: "InnerProduct" bottom: "p" top: "ip" inner_product_param { num_output: 3 } }\n'
            'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "l" }\n')
    with pytest.raises(cos.CosError, match=r"layer 'p' \(Pooling\): " + match):
        _plan(cos, tmp_path, (2, 3, 8, 8), body)


def test_accepted_pooling_setups_still_plan(cos, tmp_path):
    for param in ("pool: AVE global_pooling: true", "pool: MAX kernel_size: 3 stride: 2 pad: 2",
                  "pool: AVE kernel_size: 2 stride: 3"):
        body = (f'layer {{ name: "p" type: "Pooling" bottom: "x" top: "p" pooling_param {{ {param} }} }}\n'
                'layer { name: "ip" type: "InnerProduct" bottom: "p" top: "ip" inner_product_param { num_output: 3 } }\n'
                'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "l" }\n')
        assert _ops(_plan(cos, tmp_path, (2, 3, 8, 8), body))[0] == "Pooling(" + param.split()[1] + ") p"
