"""TanH, ELU, AbsVal, BNLL, Power, Exp, Log, Threshold, PReLU, Softmax, MultinomialLogisticLoss and HingeLoss on the
built-in engine (DESIGN.md section 14), each op alone on the GPU against the float64 references of neuron_ops_ref.py
through test_gpu_producer_ops.py's injector harness: dyadic inputs compared by value where the result is exact,
Gaussian inputs held to the bounds, in place or not, the non-finite and zero inputs Caffe's rules single out, and the
bad-label status of both losses.  Every case makes three calls on one net: two from a cleared diff_ must agree bit for
bit (loss included), and a third without clearing must leave exactly twice the gradient."""
import numpy as np
import pytest
import torch

import neuron_ops_ref as N
import producer_ops_ref as R
from gpu_util import assert_bits_equal, to_host
from test_gpu_producer_ops import _check, _close, _forward, _net, _probe, _same

pytestmark = pytest.mark.gpu

F32 = np.float32
SHAPE = (4, 3, 5, 7)


def _engine(cos, tmp_path, xs, body, weights=(), out_shape=None, B=None, staged=None, top="y"):
    """test_gpu_producer_ops._engine's net and result, from three calls on it: two from a cleared diff_, which must
    agree bit for bit, and a third without clearing, which must leave exactly 2g (diff_ += g once more)."""
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
        dev = [torch.from_numpy(v).cuda() for v in inputs]
        loss = torch.zeros(1, device="cuda")
        runs = []
        for clear in (True, True, False):
            if clear:
                net.diff().zero_()
            torch.cuda.synchronize()
            assert net.forward_backward(dev, loss.data_ptr()), net.last_error()
            assert net.synchronize(), net.last_error()
            runs.append((to_host(net.diff()), float(loss.item())))
        w = to_host(net.data())
    finally:
        net.deallocate()
    g, l32 = runs[0]
    assert_bits_equal(runs[1][0], g, "diff_ of two calls")
    assert np.array_equal(np.float64(runs[1][1]), np.float64(l32), equal_nan=True), (runs[1][1], l32)
    _same(runs[2][0], F32(2) * g, "a call without clearing adds g once more")
    parts, data, off = [], [], 0
    for v in ws:
        parts.append(g[off:off + v.size].reshape(v.shape))
        data.append(w[off:off + v.size].reshape(v.shape))
        off += v.size
    dx = parts[1:2 * len(xs):2]
    op = slice(2 * len(xs), 2 * len(xs) + len(weights))
    out = dict(dx=dx, grads=parts[op], data=data[op], loss=l32, d=None)
    if out_shape is not None:
        out["d"] = -parts[-1]
    return out


def _layer(type_, param="", inplace=False):
    top = "x0" if inplace else "y"
    return f'layer {{ name: "op" type: "{type_}" bottom: "x0" top: "{top}" {param} }}\n', top


def _run(cos, tmp_path, x, type_, param="", inplace=False, weights=(), y64=None, family="gaussian", seed=0):
    body, top = _layer(type_, param, inplace)
    B = _probe(y64, np.random.RandomState(seed), family)
    return _engine(cos, tmp_path, [x], body, weights, y64.shape, B, top=top), B


ELEMENTWISE = {  # case -> (layer type, param, reference, bounds), reference(x, dy) -> (y, dx)
    "TanH": ("TanH", "", N.tanh, N.tanh_bounds),
    "ELU": ("ELU", "elu_param { alpha: 0.5 }", lambda x, d: N.elu(x, d, 0.5), lambda x, d: N.elu_bounds(x, d, 0.5)),
    "BNLL": ("BNLL", "", N.bnll, N.bnll_bounds),
    "Power": ("Power", "power_param { power: 3 scale: 0.5 shift: 4 }", lambda x, d: N.power(x, d, 3, 0.5, 4),
              lambda x, d: N.power_bounds(x, d, 3, 0.5, 4)),
    "Power2": ("Power", "power_param { power: 2 scale: 0.5 shift: 1 }", lambda x, d: N.power(x, d, 2, 0.5, 1),
               lambda x, d: N.power_bounds(x, d, 2, 0.5, 1)),
    "Exp": ("Exp", "exp_param { base: 2 scale: 0.5 shift: 1 }", lambda x, d: N.exp_(x, d, 2, 0.5, 1),
            lambda x, d: N.exp_bounds(x, d, 2, 0.5, 1)),
    "ExpE": ("Exp", "", lambda x, d: N.exp_(x, d, -1, 1, 0), lambda x, d: N.exp_bounds(x, d, -1, 1, 0)),
    "Log": ("Log", "log_param { base: 10 scale: 2 shift: 9 }", lambda x, d: N.log_(x, d, 10, 2, 9),
            lambda x, d: N.log_bounds(x, d, 10, 2, 9)),
}


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("name", sorted(ELEMENTWISE))
def test_elementwise_gaussian(cos, tmp_path, name, inplace):
    type_, param, ref, bounds = ELEMENTWISE[name]
    rng = np.random.RandomState(len(name))
    x = R.gaussian(rng, SHAPE, 2.0)
    y64, _ = ref(x, np.zeros(SHAPE))
    r, B = _run(cos, tmp_path, x, type_, param, inplace, y64=y64)
    d = r["d"]
    y64, dx64 = ref(x, d)
    by, bdx = bounds(x, d)
    _forward(d, y64, B, by, "y", False)
    _close(r["dx"][0], dx64, bdx, "dx")


@pytest.mark.parametrize("name", ["TanH", "ELU", "BNLL", "Power", "Exp", "Log"])
def test_a_large_blob_against_the_bounds(cos, tmp_path, name):
    type_, param, ref, bounds = ELEMENTWISE[name]
    rng = np.random.RandomState(7)
    x = R.gaussian(rng, (3, 200000))  # more elements than the grid's threads
    y64, _ = ref(x, np.zeros(x.shape))
    r, B = _run(cos, tmp_path, x, type_, param, y64=y64)
    y64, dx64 = ref(x, r["d"])
    by, bdx = bounds(x, r["d"])
    _forward(r["d"], y64, B, by, "y", False)
    _close(r["dx"][0], dx64, bdx, "dx")


@pytest.mark.parametrize("inplace", [False, True])
def test_absval_and_elu_are_exact_on_dyadic_inputs(cos, tmp_path, inplace):
    rng = np.random.RandomState(3)
    x = R.dyadic(rng, SHAPE)
    x.flat[:3] = [0.0, -0.0, 1.0]
    y64, _ = N.absval(x, np.zeros(SHAPE))
    if not inplace:  # AbsVal refuses to run in place
        r, B = _run(cos, tmp_path, x, "AbsVal", y64=y64, family="dyadic")
        _forward(r["d"], y64, B, 0, "y", True)
        _, dx64 = N.absval(x, r["d"])
        _check(r["dx"][0], dx64, 0, "dx", True)
        assert r["dx"][0].flat[0] == 0 and r["dx"][0].flat[1] == 0  # sign(0) = 0
    x = np.abs(x) + F32(0.5)  # ELU with x > 0 is the identity either way
    y64, _ = N.elu(x, np.zeros(SHAPE), 0.5)
    (tmp_path / "e").mkdir()
    r, B = _run(cos, tmp_path / "e", x, "ELU", "elu_param { alpha: 0.5 }", inplace, y64=y64, family="dyadic")
    _forward(r["d"], y64, B, 0, "y", True)
    _check(r["dx"][0], N.elu(x, r["d"], 0.5)[1], 0, "dx", True)


def test_power_branches_and_the_nan_at_zero(cos, tmp_path):
    rng = np.random.RandomState(4)
    x = R.gaussian(rng, (2, 50))
    x.flat[:2] = [0.0, -0.0]
    # shift 0, power 3: dx = power * y / x, NaN where x = 0, as in Caffe
    y64, _ = N.power(x, np.zeros(x.shape), 3, 1, 0)
    r, B = _run(cos, tmp_path, x, "Power", "power_param { power: 3 }", y64=y64)
    assert np.isnan(r["dx"][0].flat[:2]).all() and np.isfinite(r["dx"][0].flat[2:]).all()
    _close(r["dx"][0], N.power(x, r["d"], 3, 1, 0)[1], N.power_bounds(x, r["d"], 3, 1, 0)[1], "dx")
    # power * scale == 0: the constant shift^power and an exact 0 gradient, whatever dy is
    (tmp_path / "c").mkdir()
    y64, _ = N.power(x, np.zeros(x.shape), 2, 0, 3)
    r, B = _run(cos, tmp_path / "c", x, "Power", "power_param { power: 2 scale: 0 shift: 3 }", y64=y64, seed=1)
    assert (r["d"] == F32(9) - B).all() and not r["dx"][0].any()
    # power 1: dx = scale * dy
    (tmp_path / "p1").mkdir()
    y64, _ = N.power(x, np.zeros(x.shape), 1, 0.5, 0.25)
    r, B = _run(cos, tmp_path / "p1", x, "Power", "power_param { scale: 0.5 shift: 0.25 }", y64=y64, seed=2)
    _close(r["dx"][0], r["d"] * 0.5, R.ulp(r["d"]) / 2, "dx")


def test_non_finite_inputs(cos, tmp_path):
    x = np.array([[np.nan, np.inf, -np.inf, 0.0, -0.0, 60.0, -60.0, 1.0]], F32)
    for i, (name, ref) in enumerate([("TanH", N.tanh), ("BNLL", N.bnll), ("AbsVal", N.absval)]):
        (tmp_path / name).mkdir()
        y64, _ = ref(x, np.zeros(x.shape))
        body, _ = _layer(name)
        B = np.zeros(x.shape, F32)
        r = _engine(cos, tmp_path / name, [x], body, (), x.shape, B)
        y = r["d"] + B
        want = np.asarray(y64, F32)
        assert np.array_equal(np.isnan(y), np.isnan(want)), (name, y, want)
        fin = np.isfinite(want)
        assert np.allclose(y[fin], want[fin], rtol=1e-6, atol=1e-6), (name, y, want)  # BNLL cancels at -60


def test_threshold_binarises_a_staged_target(cos, tmp_path):
    rng = np.random.RandomState(5)
    x, t = R.gaussian(rng, (4, 6)), R.gaussian(rng, (4, 6))
    t.flat[:3] = [0.25, 0.2500001, np.nan]
    body = ('layer { name: "th" type: "Threshold" bottom: "t" top: "tb" threshold_param { threshold: 0.25 } }\n'
            'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "x0" bottom: "tb" top: "l" }')
    r = _engine(cos, tmp_path, [x], body, staged={"t": t})
    tb = N.threshold(t, F32(0.25))
    assert tb.flat[0] == 0 and tb.flat[1] == 1 and tb.flat[2] == 0
    sig = 1 / (1 + np.exp(-x.astype(np.float64)))
    _close(r["dx"][0], (sig - tb) / 4, 1e-6 * np.abs(sig - tb) / 4 + 1e-9, "dx against the binarised target")


# --------------------------------------------------------------------------- PReLU
PRELU_CASES = [((4, 3, 5, 7), False), ((4, 3, 5, 7), True), ((2, 6), False), ((2, 6), True),
               ((40, 3, 16, 16), False), ((40, 3, 16, 16), True),  # N * dim = 10240 > one chunk; shared: 30720
               ((3, 2, 100, 100), False)]  # 30000 per channel: four chunks, the last partial


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("shape,shared", PRELU_CASES)
def test_prelu(cos, tmp_path, shape, shared, inplace):
    rng = np.random.RandomState(shape[0] + shape[1] + shared)
    exact = shape[0] * shape[1] <= 12
    x = R.dyadic(rng, shape) if exact else R.gaussian(rng, shape)
    x.flat[:2] = [0.0, -0.0]
    a = np.array([0.25], F32) if shared else R.dyadic(rng, (shape[1],), bits=3)
    param = "prelu_param { channel_shared: true }" if shared else ""
    y64, _, _ = N.prelu(x, a, np.zeros(shape), shared)
    r, B = _run(cos, tmp_path, x, "PReLU", param, inplace, [a.reshape(()) if shared else a], y64,
                "dyadic" if exact else "gaussian")
    d = r["d"]
    y64, dx64, da64 = N.prelu(x, a, d, shared)
    by, bdx, bda = N.prelu_bounds(x, a, d, shared)
    _forward(d, y64, B, by, "y", exact)
    _check(r["dx"][0], dx64, bdx, "dx", exact)
    _close(r["grads"][0].ravel(), da64, bda, "da")


# --------------------------------------------------------------------------- Softmax
SOFTMAX_CASES = [((6, 10), a) for a in (0, 1, -1)] + [((4, 5, 6), a) for a in (0, 1, 2, -2)] + \
                [((3, 4, 5, 6), a) for a in (0, 1, 2, 3)]


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("shape,axis", SOFTMAX_CASES)
def test_softmax(cos, tmp_path, shape, axis, inplace):
    rng = np.random.RandomState(len(shape) * 10 + axis)
    x = R.gaussian(rng, shape, 3.0)
    y64, _ = N.softmax(x, np.zeros(shape), axis)
    r, B = _run(cos, tmp_path, x, "Softmax", f"softmax_param {{ axis: {axis} }}", inplace, y64=y64)
    y64, dx64 = N.softmax(x, r["d"], axis)
    by, bdx = N.softmax_bounds(x, r["d"], axis)
    _forward(r["d"], y64, B, by, "y", False)
    _close(r["dx"][0], dx64, bdx, "dx")


# --------------------------------------------------------------------------- the losses
def _loss_run(cos, tmp_path, x, label, type_, param="", loss_weight=1.0):
    body = (f'layer {{ name: "loss" type: "{type_}" bottom: "x0" bottom: "lab" top: "l" loss_weight: {loss_weight} '
            f'{param} }}')
    return _engine(cos, tmp_path, [x], body, staged={"lab": label})


@pytest.mark.parametrize("n,dim", [(4, 10), (64, 10), (300, 7), (1000, 3), (16, 2000)])
def test_multinomial_logistic_loss(cos, tmp_path, n, dim):
    rng = np.random.RandomState(n + dim)
    x = rng.rand(n, dim).astype(F32)
    x.flat[:3] = [0.0, 1e-30, 0.5]
    label = rng.randint(0, dim, n).astype(F32)
    label[0] = 0  # a zero probability at the label: the clamp at 1e-20
    r = _loss_run(cos, tmp_path, x, label, "MultinomialLogisticLoss", loss_weight=2.0)
    l64, dx64 = N.mll(x, label, 2.0)
    lb, dxb = N.mll_bounds(x, label, 2.0)
    assert abs(r["loss"] - l64) <= lb, (r["loss"], l64, lb)
    _close(r["dx"][0], dx64, dxb, "dx")
    off = np.ones(x.shape, bool)
    off[np.arange(n), label.astype(int)] = False
    assert not r["dx"][0][off].any()


@pytest.mark.parametrize("norm", ["L1", "L2"])
@pytest.mark.parametrize("n,dim", [(4, 10), (64, 10), (100, 1000), (3, 200000)])
def test_hinge_loss(cos, tmp_path, n, dim, norm):
    rng = np.random.RandomState(n + dim + len(norm))
    x = R.gaussian(rng, (n, dim))
    label = rng.randint(0, dim, n).astype(F32)
    x[0, :3] = [1.0, 0.5, np.nan]  # h = 0 at the margin (sign(0) = 0) and for a NaN (std::max(0, NaN) = 0)
    label[0] = 0
    r = _loss_run(cos, tmp_path, x, label, "HingeLoss", f"hinge_loss_param {{ norm: {norm} }}", loss_weight=0.5)
    l64, dx64 = N.hinge(x, label, norm, 0.5)
    lb, dxb = N.hinge_bounds(x, label, norm, 0.5)
    assert abs(r["loss"] - l64) <= lb, (r["loss"], l64, lb)
    _close(r["dx"][0], dx64, dxb, "dx")
    assert r["dx"][0][0, 0] == 0 and r["dx"][0][0, 2] == 0 and r["dx"][0][0, 1] != 0


@pytest.mark.parametrize("type_,message", [("MultinomialLogisticLoss", "MultinomialLogisticLoss: a label outside"),
                                           ("HingeLoss", "HingeLoss: a label outside")])
def test_a_bad_label_reaches_the_status_message(cos, tmp_path, type_, message):
    x = np.full((4, 5), 0.2, F32)
    label = np.array([0, 5, 2, np.nan], F32)
    body = f'layer {{ name: "loss" type: "{type_}" bottom: "x0" bottom: "lab" top: "l" }}'
    text, ws = _net([x], body, staged={"lab": label})
    (tmp_path / "net.prototxt").write_text(text)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().copy_(torch.from_numpy(np.concatenate([w.ravel() for w in ws])).cuda())
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.zeros(x.shape, device="cuda"), torch.from_numpy(label).cuda()],
                                    loss.data_ptr())
        assert not net.synchronize()
        assert message in net.last_error(), net.last_error()
        g = to_host(net.diff())[x.size:2 * x.size].reshape(x.shape)  # the injector's bias gradient: the loss's dx
        assert not g[1].any() and not g[3].any() and g[0].any()
    finally:
        net.deallocate()
