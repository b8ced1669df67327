"""CPU tests of TanH, ELU, AbsVal, BNLL, Power, Exp, Log, Threshold, PReLU, Softmax, MultinomialLogisticLoss and
HingeLoss on the built-in engine (DESIGN.md section 14): the float64 references of neuron_ops_ref.py against torch and
hand-worked Caffe cases, the bounds against an fp32 evaluation in the engine's order and a mutated reference, the plan
lines, every refusal with Caffe's wording, the Threshold rule, PReLU's layout, and both fixtures' layouts and plans."""
import os

import numpy as np
import pytest
import torch

import neuron_ops_ref as N
import producer_ops_ref as R
from conftest import ROOT
from test_autoencoder_host import _op_lines, _write
from test_native_producer_host import _check_layout

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
TANH_SOLVER = os.path.join(CONFIGS, "lenet_tanh_solver.prototxt")
PRELU_SOLVER = os.path.join(CONFIGS, "cifar10_quick_prelu_solver.prototxt")
SCE = 'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "%s" bottom: "t" top: "l" }'
SCALE = 'layer { name: "sc" type: "Scale" bottom: "x" top: "s" }\n'


def _t(v):
    return torch.from_numpy(np.asarray(v, np.float64))


# --------------------------------------------------------------------------- the references
def test_references_match_torch_float64():
    rng = np.random.RandomState(0)
    x, d = rng.randn(3, 4, 5), rng.randn(3, 4, 5)
    cases = [(N.tanh(x, d), torch.tanh), (N.elu(x, d, 0.7), lambda v: torch.nn.functional.elu(v, 0.7)),
             (N.absval(x, d), torch.abs), (N.bnll(x, d), torch.nn.functional.softplus),
             (N.power(x, d, 3, 0.5, 4), lambda v: (4 + 0.5 * v) ** 3),
             (N.log_(x, d, -1, 2, 9), lambda v: torch.log(2 * v + 9))]
    for (y, dx), fn in cases:
        v = _t(x).requires_grad_()
        out = fn(v)
        out.backward(_t(d))
        assert np.allclose(y, out.detach().numpy(), rtol=1e-12, atol=1e-12)
        assert np.allclose(dx, v.grad.numpy(), rtol=1e-9, atol=1e-12)
    for axis in (0, 1, 2, -1):
        y, dx = N.softmax(x, d, axis)
        v = _t(x).requires_grad_()
        out = torch.softmax(v, axis)
        out.backward(_t(d))
        assert np.allclose(y, out.detach().numpy()) and np.allclose(dx, v.grad.numpy())
    a = np.array([0.25, -0.5, 2.0, 0.0])
    y, dx, da = N.prelu(x, a, d, False)
    v, av = _t(x).requires_grad_(), _t(a).requires_grad_()
    torch.nn.functional.prelu(v, av).backward(_t(d))
    assert np.allclose(y, torch.nn.functional.prelu(_t(x), _t(a)).numpy())
    assert np.allclose(dx, v.grad.numpy()) and np.allclose(da, av.grad.numpy())


def test_the_torch_losses_follow_caffe():
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(1)
    p = rng.rand(6, 5)
    p[0, 2] = 0.0  # clamped at 1e-20, and the gradient still flows
    label = np.array([2, 0, 1, 4, 3, 3], np.float64)
    v = _t(p).requires_grad_()
    loss = nets.multinomial_logistic_loss(v, _t(label), 2.0)
    loss.backward()
    l64, dx = N.mll(p, label, 2.0)
    assert np.isclose(float(loss), l64) and np.allclose(v.grad.numpy(), dx)
    assert dx[0, 2] == pytest.approx(-2 / 6 / 1e-20) and l64 == pytest.approx(-2 * np.log(np.maximum(
        p[np.arange(6), label.astype(int)], 1e-20)).sum() / 6)
    s = rng.randn(6, 5)
    s[0, 2], s[1, 1] = 1.0, -1.0  # h = 0 exactly at the label and off it: sign(0) = 0
    for norm in ("L1", "L2"):
        v = _t(s).requires_grad_()
        nets.hinge_loss(v, _t(label), norm, 0.5).backward()
        l64, dx = N.hinge(s, label, norm, 0.5)
        assert np.allclose(v.grad.numpy(), dx)
        assert dx[0, 2] == 0 and dx[1, 1] == 0


def test_hand_worked_caffe_cases():
    # Power: the four branches; shift 0 and power 3 is NaN at x = 0 (power * y / x); power * scale = 0 is constant
    x = np.array([0.0, -0.0, 2.0])
    assert np.isnan(N.power(x, np.ones(3), 3, 1, 0)[1][:2]).all() and N.power(x, np.ones(3), 3, 1, 0)[1][2] == 12
    y, dx = N.power(x, np.ones(3), 2, 0, 3)
    assert (y == 9).all() and (dx == 0).all()
    y, dx = N.power(x, np.ones(3), 0, 2, 3)
    assert (y == 1).all() and (dx == 0).all()
    assert (N.power(x, np.full(3, 2.0), 1, 0.5, 7)[1] == 1).all()
    assert N.power(x, np.ones(3), 2, 0.5, 1)[1][2] == 2 * 0.5 * 2  # 2 scale (shift + scale x)
    # AbsVal: sign(0) = 0; Threshold: strictly greater
    assert (N.absval(np.array([0.0, -0.0, -3.0]), np.ones(3))[1] == [0, 0, -1]).all()
    assert (N.threshold(np.array([0.5, 0.5000001, np.nan]), 0.5) == [0, 1, 0]).all()
    # PReLU at x = +-0: y = 0, dx = a dy, no slope gradient
    y, dx, da = N.prelu(np.array([[0.0, -0.0]]).reshape(1, 2), np.array([0.25, 0.5]), np.array([[4.0, 4.0]]), False)
    assert (y == 0).all() and (dx == [1, 2]).all() and (da == 0).all()
    # MLL's clamp, Hinge's sign rule and NaN rule
    assert N.mll(np.array([[0.0, 1.0]]), [0])[0] == pytest.approx(-np.log(1e-20))
    _, dx = N.hinge(np.array([[1.0, -1.0, np.nan]]), [0])
    assert (dx == 0).all()  # h = 0 at the label (1 - 1), off it (1 + -1) and for the NaN
    # BNLL cancels for x << 0 as Caffe's formula does: the bound is absolute there
    y, _ = N.bnll(np.array([-60.0]), np.ones(1))
    assert y[0] > 0 and N.bnll_bounds(np.array([-60.0]), np.ones(1))[0][0] >= y[0]


def _fp32_softmax(x, dy, axis):
    """softmax_layer.cu's order in fp32, one rounding per operation"""
    xs, ds = np.moveaxis(x.astype(F32), axis, -1), np.moveaxis(dy.astype(F32), axis, -1)
    m = xs.max(axis=-1, keepdims=True)
    e = np.exp((xs - m).astype(F32)).astype(F32)
    s = np.zeros(m.shape, F32)
    for c in range(xs.shape[-1]):
        s = (s + e[..., c:c + 1]).astype(F32)
    y = (e / s).astype(F32)
    dot = np.zeros(m.shape, F32)
    for c in range(xs.shape[-1]):
        dot = (dot + (ds[..., c:c + 1] * y[..., c:c + 1]).astype(F32)).astype(F32)
    dx = ((ds - dot).astype(F32) * y).astype(F32)
    return np.moveaxis(y, -1, axis), np.moveaxis(dx, -1, axis)


def _admits(got, ref, bound):
    """equal NaN positions, and every other element within its bound"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    nan = np.isnan(ref)
    with np.errstate(invalid="ignore"):
        err = np.where(got == ref, 0, np.abs(got - ref))
    return bool(np.array_equal(np.isnan(got), nan) and np.all(err[~nan] <= np.broadcast_to(bound, ref.shape)[~nan]))


MUTATION = 2.0 ** -16  # a relative error of 256 roundings: every bound must reject a reference off by this much


def _fp32(fn):
    with np.errstate(all="ignore"):
        return fn()


def _f32(v):
    return np.asarray(v, F32)


def _engine_order(x, d):
    """Each elementwise op evaluated in fp32 in its kernel's order (numpy's float32 arithmetic rounds each operation
    once; its exp, log, tanh and power are at least as accurate as CUDA's), -> name -> (y, dx)."""
    one = F32(1)
    t = np.tanh(x)
    e = np.exp(x)
    elu_y = np.where(x > 0, x, _f32(F32(0.5) * _f32(e - one)))
    v3 = _f32(_f32(F32(0.5) * x) + F32(4))  # Power 3, scale 0.5, shift 4: the general branch
    p3 = _f32(np.power(v3, F32(3)))
    ds3 = F32(F32(3) * F32(0.5))
    v2 = _f32(_f32(F32(0.5) * x) + one)  # Power 2, scale 0.5, shift 1: (ds scale) x + ds shift
    ds2 = F32(F32(2) * F32(0.5))
    inner, outer = (F32(c) for c in N.exp_consts(2, 0.5, 1))
    ey = _f32(outer * np.exp(_f32(inner * x)))
    base_scale, num_scale = (F32(c) for c in N.log_consts(10, 2))
    lv = _f32(_f32(F32(2) * x) + F32(9))
    bnll_e = np.exp(np.minimum(x, F32(50)))
    return {
        "tanh": (t, _f32(d * _f32(one - _f32(t * t)))),
        "elu": (elu_y, np.where(x > 0, d, _f32(d * _f32(elu_y + F32(0.5))))),
        "bnll": (np.where(x > 0, _f32(x + np.log(_f32(one + np.exp(-x)))), np.log(_f32(one + np.exp(x)))),
                 _f32(_f32(d * bnll_e) / _f32(bnll_e + one))),
        "power3": (p3, _f32(d * _f32(ds3 * _f32(p3 / v3)))),
        "power2": (_f32(np.power(v2, F32(2))), _f32(d * _f32(_f32(ds2 * F32(0.5) * x) + ds2 * one))),
        "exp": (ey, _f32(inner * _f32(ey * d))),
        "log": (_f32(base_scale * np.log(lv)), _f32(d * _f32(num_scale * _f32(one / lv)))),
    }


REFS = {  # name -> float64 (y, dx) and bounds
    "tanh": (N.tanh, N.tanh_bounds),
    "elu": (lambda x, d: N.elu(x, d, 0.5), lambda x, d: N.elu_bounds(x, d, 0.5)),
    "bnll": (N.bnll, N.bnll_bounds),
    "power3": (lambda x, d: N.power(x, d, 3, 0.5, 4), lambda x, d: N.power_bounds(x, d, 3, 0.5, 4)),
    "power2": (lambda x, d: N.power(x, d, 2, 0.5, 1), lambda x, d: N.power_bounds(x, d, 2, 0.5, 1)),
    "exp": (lambda x, d: N.exp_(x, d, 2, 0.5, 1), lambda x, d: N.exp_bounds(x, d, 2, 0.5, 1)),
    "log": (lambda x, d: N.log_(x, d, 10, 2, 9), lambda x, d: N.log_bounds(x, d, 10, 2, 9)),
}


@pytest.mark.parametrize("name", sorted(REFS))
def test_elementwise_bounds_admit_fp32_and_reject_a_mutated_reference(name):
    rng = np.random.RandomState(2)
    x, d = R.gaussian(rng, (64, 100), 3.0), R.gaussian(rng, (64, 100))
    y32, dx32 = _fp32(lambda: _engine_order(x, d))[name]
    ref, bounds = REFS[name]
    with np.errstate(all="ignore"):
        y64, dx64 = ref(x, d)
        by, bdx = bounds(x, d)
    assert _admits(y32, y64, by) and _admits(dx32, dx64, bdx), name
    assert not _admits(y32, y64 * (1 + MUTATION), by), name
    assert not _admits(dx32, dx64 * (1 + MUTATION), bdx), name


def test_formula_mutations_are_rejected():
    """References with one of Caffe's rules dropped fall outside the bounds of the engine-order fp32 evaluation."""
    rng = np.random.RandomState(3)
    x, d = R.gaussian(rng, (64, 100), 3.0), R.gaussian(rng, (64, 100))
    ev = _fp32(lambda: _engine_order(x, d))
    # ELU's backward with alpha dropped: dy * y instead of dy * (y + alpha)
    y, _ = N.elu(x, d, 0.5)
    assert not _admits(ev["elu"][1], np.where(x > 0, d, d * y), N.elu_bounds(x, d, 0.5)[1])
    # Exp without its outer scale base^shift
    y, _ = N.exp_(x, d, 2, 0.5, 1)
    assert not _admits(ev["exp"][0], y / 2, N.exp_bounds(x, d, 2, 0.5, 1)[0])
    # Log multiplied by log(base) instead of divided
    y, _ = N.log_(x, d, 10, 2, 9)
    assert not _admits(ev["log"][0], y * np.log(10) ** 2, N.log_bounds(x, d, 10, 2, 9)[0])


def _fp32_prelu_slope(x, a_dy, shared):
    """prelu_slope_partial_kernel's order in fp32: per slope, chunks of 8192 values; in a chunk, thread t sums values
    t, t + 256, ... in order, then block_sum's tree; the partials in chunk order."""
    x, dy = x.astype(F32), a_dy.astype(F32)
    t = _f32(_f32(dy * x) * (x <= 0).astype(F32))
    rows = t.reshape(1, -1) if shared else np.moveaxis(t, 1, 0).reshape(t.shape[1], -1)
    out = []
    for row in rows:
        total = F32(0)
        for k in range(0, row.size, N.PRELU_CHUNK):
            chunk = np.zeros(N.PRELU_CHUNK, F32)
            chunk[:min(N.PRELU_CHUNK, row.size - k)] = row[k:k + N.PRELU_CHUNK]
            acc = np.zeros(R.BLOCK, F32)
            for r in chunk.reshape(-1, R.BLOCK):
                acc = _f32(acc + r)
            w = R.BLOCK // 2
            while w:
                acc[:w] = _f32(acc[:w] + acc[w:2 * w])
                w //= 2
            total = F32(total + acc[0])
        out.append(F32(F32(0) + total))
    return np.array(out, F32)


@pytest.mark.parametrize("shape,shared", [((4, 3, 5, 7), False), ((40, 3, 16, 16), False), ((40, 3, 16, 16), True),
                                          ((3, 2, 100, 100), False)])
def test_prelu_bounds_admit_fp32_and_reject_a_mutated_reference(shape, shared):
    rng = np.random.RandomState(4)
    x, d = R.gaussian(rng, shape), R.gaussian(rng, shape)
    a = np.array([0.25], F32) if shared else R.dyadic(rng, (shape[1],), bits=3)
    ab = np.full(shape, a[0], F32) if shared else np.broadcast_to(a.reshape((1, -1) + (1,) * (len(shape) - 2)), shape)
    hi, lo = np.where(x < 0, F32(0), x), np.where(0 < x, F32(0), x)
    y32 = _f32(hi + _f32(ab * lo))
    dx32 = _f32(d * _f32((x > 0).astype(F32) + _f32(ab * (x <= 0).astype(F32))))
    da32 = _fp32_prelu_slope(x, d, shared)
    y64, dx64, da64 = N.prelu(x, a, d, shared)
    by, bdx, bda = N.prelu_bounds(x, a, d, shared)
    assert _admits(y32, y64, by) and _admits(dx32, dx64, bdx) and _admits(da32, da64, bda)
    # a reduction of one chunk holds to a relative mutation; over several chunks, whose worst-case bound is loose where
    # the terms cancel, the reference must at least miss the sum without its last chunk
    t = d.astype(np.float64) * x * (x <= 0)
    rows = t.reshape(1, -1) if shared else np.moveaxis(t, 1, 0).reshape(t.shape[1], -1)
    if rows.shape[1] <= N.PRELU_CHUNK:
        assert not _admits(da32, da64 * (1 + MUTATION), bda)
    else:
        assert not _admits(da32, rows[:, :(rows.shape[1] - 1) // N.PRELU_CHUNK * N.PRELU_CHUNK].sum(axis=1), bda)
    t = d.astype(np.float64) * x * (x > 0)  # the slope gradient summed over x > 0 instead of x <= 0
    wrong = np.array([t.sum()]) if shared else t.sum(axis=tuple(i for i in range(len(shape)) if i != 1))
    assert not _admits(da32, wrong, bda)


def test_softmax_bounds_admit_fp32_and_reject_a_mutated_reference():
    rng = np.random.RandomState(2)
    x, d = R.gaussian(rng, (64, 10), 3.0), R.gaussian(rng, (64, 10))
    y32, dx32 = _fp32_softmax(x, d, 1)
    y64, dx64 = N.softmax(x, d, 1)
    by, bdx = N.softmax_bounds(x, d, 1)
    assert _admits(y32, y64, by) and _admits(dx32, dx64, bdx)
    assert not _admits(y32, y64 * (1 + MUTATION), by)
    assert not _admits(dx32, dx64 * (1 + MUTATION), bdx)


def test_loss_bounds_admit_fp32_and_reject_a_mutated_reference():
    """The fp32 sums in the kernels' order (one block's thread runs and tree for MLL at num <= 256 is one run per
    thread; the hinge's grid of one block here) against float64."""
    rng = np.random.RandomState(5)
    p, label = rng.rand(64, 10).astype(F32), rng.randint(0, 10, 64)
    l64, _ = N.mll(p, label)
    lb, _ = N.mll_bounds(p, label)
    logs = [F32(-np.log(max(p[r, label[r]], F32(1e-20)))) for r in range(64)]
    acc = np.array(logs + [F32(0)] * (R.BLOCK - 64), F32)
    w = R.BLOCK // 2
    while w:
        acc[:w] = _f32(acc[:w] + acc[w:2 * w])
        w //= 2
    l32 = float(F32(F32(1) * F32(acc[0] / F32(64))))
    assert abs(l32 - l64) <= lb and abs(l32 - l64 * (1 + MUTATION)) > lb
    x = R.gaussian(rng, (4, 10))
    label = rng.randint(0, 10, 4)
    for norm in ("L1", "L2"):
        l64, _ = N.hinge(x, label, norm)
        lb, _ = N.hinge_bounds(x, label, norm)
        h, _ = N._hinge_h(x.astype(F32), label)
        terms = h.astype(F32) if norm == "L1" else _f32(h.astype(F32) * h.astype(F32))
        acc = np.zeros(R.BLOCK, F32)
        acc[:terms.size] = terms.ravel()
        w = R.BLOCK // 2
        while w:
            acc[:w] = _f32(acc[:w] + acc[w:2 * w])
            w //= 2
        l32 = float(F32(F32(1) * F32(acc[0] / F32(4))))
        assert abs(l32 - l64) <= lb and abs(l32 - l64 * (1 + MUTATION)) > lb, norm


# --------------------------------------------------------------------------- plan lines
@pytest.mark.parametrize("layer,line", [
    ('type: "TanH"', "TanH op 2x3x6x6 -> 2x3x6x6"),
    ('type: "ELU" elu_param { alpha: 0.5 }', "ELU op 2x3x6x6 -> 2x3x6x6 alpha=0.5"),
    ('type: "AbsVal"', "AbsVal op 2x3x6x6 -> 2x3x6x6"),
    ('type: "BNLL"', "BNLL op 2x3x6x6 -> 2x3x6x6"),
    ('type: "Power" power_param { power: 2 scale: 0.5 shift: 1 }', "Power op 2x3x6x6 -> 2x3x6x6 power=2 scale=0.5 shift=1"),
    ('type: "Power"', "Power op 2x3x6x6 -> 2x3x6x6 power=1 scale=1 shift=0"),
    ('type: "Exp" exp_param { base: 2 shift: 1 }', "Exp op 2x3x6x6 -> 2x3x6x6 base=2 scale=1 shift=1"),
    ('type: "Log"', "Log op 2x3x6x6 -> 2x3x6x6 base=-1 scale=1 shift=0"),
    ('type: "Softmax"', "Softmax op 2x3x6x6 -> 2x3x6x6 axis=1"),
    ('type: "Softmax" softmax_param { axis: -1 }', "Softmax op 2x3x6x6 -> 2x3x6x6 axis=3"),
    ('type: "PReLU"', "PReLU op 2x3x6x6 -> 2x3x6x6 w=3:3"),
    ('type: "PReLU" prelu_param { channel_shared: true }', "PReLU op 2x3x6x6 -> 2x3x6x6 w=3:1 channel_shared"),
])
def test_plan_lines(cos, tmp_path, layer, line):
    body = SCALE + f'layer {{ name: "op" {layer} bottom: "s" top: "y" }}\n' + SCE % "y"
    text = cos.native_producer_plan(_write(tmp_path, body))
    assert _op_lines(text)[1] == "op 1 " + line


def test_in_place_ops_get_storage_of_their_own(cos, tmp_path):
    body = SCALE + 'layer { name: "op" type: "TanH" bottom: "s" top: "s" }\n' + SCE % "s"
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, body)))
    assert lines[1] == "op 1 TanH op 2x3x6x6 -> 2x3x6x6"  # no in-place mark: a top of its own


@pytest.mark.parametrize("loss,line", [
    ('type: "MultinomialLogisticLoss"', "MultinomialLogisticLoss loss 2x10 -> scalar label=1 loss_weight=1"),
    ('type: "HingeLoss" loss_weight: 0.5', "HingeLoss loss 2x10 -> scalar label=1 norm=L1 loss_weight=0.5"),
    ('type: "HingeLoss" hinge_loss_param { norm: L2 }', "HingeLoss loss 2x10 -> scalar label=1 norm=L2 loss_weight=1"),
])
def test_loss_plan_lines(cos, tmp_path, loss, line):
    body = SCALE + f'layer {{ name: "loss" {loss} bottom: "s" bottom: "t" top: "l" }}'
    text = cos.native_producer_plan(_write(tmp_path, body, shape=(2, 10), target=(2,)))
    assert _op_lines(text)[1] == "op 1 " + line


# --------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("body,shape,target,match", [
    (SCALE + 'layer { name: "e" type: "Exp" bottom: "s" top: "y" exp_param { base: -2 } }\n' + SCE % "y", None, None,
     r"^layer 'e' \(Exp\): base must be strictly positive\. \(native producer\)$"),
    (SCALE + 'layer { name: "g" type: "Log" bottom: "s" top: "y" log_param { base: 0 } }\n' + SCE % "y", None, None,
     r"^layer 'g' \(Log\): base must be strictly positive\. \(native producer\)$"),
    (SCALE + 'layer { name: "sm" type: "Softmax" bottom: "s" top: "y" softmax_param { axis: 4 } }\n' + SCE % "y",
     None, None, r"^layer 'sm' \(Softmax\): axis 4 out of range for 4-D Blob \(native producer\)$"),
    (SCALE + 'layer { name: "sm" type: "Softmax" bottom: "s" top: "y" softmax_param { axis: -5 } }\n' + SCE % "y",
     None, None, r"^layer 'sm' \(Softmax\): axis -5 out of range for 4-D Blob"),
    (SCALE + 'layer { name: "a" type: "AbsVal" bottom: "s" top: "s" }\n' + SCE % "s", None, None,
     r"^layer 'a' \(AbsVal\): AbsVal Layer does not allow in-place computation\. \(native producer\)$"),
    ('layer { name: "p" type: "PReLU" bottom: "x" top: "y" }\n' + SCE % "y", (6,), None,
     r"^layer 'p' \(PReLU\): Number of axes of bottom blob must be >=2\. \(native producer\)$"),
    ('layer { name: "p" type: "PReLU" bottom: "x" top: "y" }\n' + SCE % "y", (1, 65536), None,
     r"^layer 'p' \(PReLU\): 65536 channels is more than the 65535 per-channel slopes the engine supports"),
    (SCALE + 'layer { name: "p" type: "PReLU" bottom: "s" top: "y" prelu_param { filler { type: "bilinear" } } }\n' +
     SCE % "y", None, None, r"^layer 'p' \(PReLU\): filler type 'bilinear' is not supported"),
    (SCALE + 'layer { name: "loss" type: "MultinomialLogisticLoss" bottom: "s" bottom: "t" top: "l" }', (2, 10),
     (2, 3), r"^layer 'loss' \(MultinomialLogisticLoss\): Check failed: bottom\[1\]->channels\(\) == 1 \(3 vs\. 1\)"),
    (SCALE + 'layer { name: "loss" type: "MultinomialLogisticLoss" bottom: "s" bottom: "t" top: "l" }', (2, 10),
     (2, 1, 1, 4), r"^layer 'loss' \(MultinomialLogisticLoss\): Check failed: bottom\[1\]->width\(\) == 1 \(4 vs\. 1\)"),
    (SCALE + 'layer { name: "loss" type: "HingeLoss" bottom: "s" bottom: "t" top: "l" }', (2, 10), (3,),
     r"^layer 'loss' \(HingeLoss\): The data and label should have the same number\."),
    (SCALE + 'layer { name: "loss" type: "HingeLoss" bottom: "s" bottom: "t" top: "l" loss_param { normalize: false } }',
     (2, 10), (2,), r"^layer 'loss' \(HingeLoss\): loss_param is not supported"),
    (SCALE + 'layer { name: "sp" type: "Split" bottom: "s" top: "a" top: "b" }\n'
     'layer { name: "loss" type: "HingeLoss" bottom: "a" bottom: "t" top: "l" }\n'
     'layer { name: "l2" type: "MultinomialLogisticLoss" bottom: "b" bottom: "t" top: "l2" }', (2, 10), (2,),
     r"^layer 'l2' \(MultinomialLogisticLoss\): a second loss layer is not supported"),
])
def test_refusals_name_the_layer(cos, tmp_path, body, shape, target, match):
    with pytest.raises(cos.CosError, match=match):
        cos.native_producer_plan(_write(tmp_path, body, shape or (2, 3, 6, 6), target))
    assert cos.parse_solver(str(tmp_path / "solver.prototxt")) is not None  # the layout parser still accepts it


def test_threshold_runs_only_where_no_gradient_passes(cos, tmp_path):
    ok = ('layer { name: "th" type: "Threshold" bottom: "t" top: "tb" threshold_param { threshold: 0.5 } }\n' + SCALE +
          'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "s" bottom: "tb" top: "l" }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, ok)))
    assert lines[0] == "op 0 Threshold th 2x3x6x6 -> 2x3x6x6 threshold=0.5 staged-bottom no-backward"
    (tmp_path / "b").mkdir()  # on a staged input under the loss: no gradient is wanted at its bottom
    staged = ('layer { name: "th" type: "Threshold" bottom: "x" top: "xb" }\n'
              'layer { name: "sc" type: "Scale" bottom: "xb" top: "s" }\n' + SCE % "s")
    assert _op_lines(cos.native_producer_plan(_write(tmp_path / "b", staged)))[0].endswith("threshold=0 staged-bottom")
    (tmp_path / "c").mkdir()
    bad = SCALE + 'layer { name: "th" type: "Threshold" bottom: "s" top: "y" }\n' + SCE % "y"
    with pytest.raises(cos.CosError, match=r"^layer 'th' \(Threshold\): Not Implemented Yet"):
        cos.native_producer_plan(_write(tmp_path / "c", bad))


# --------------------------------------------------------------------------- PReLU in the layout
def test_prelu_layout(cos, tmp_path):
    body = ('layer { name: "c" type: "Convolution" bottom: "x" top: "c" convolution_param { num_output: 4 '
            'kernel_size: 1 } }\n'
            'layer { name: "p1" type: "PReLU" bottom: "c" top: "c" param { name: "slope" lr_mult: 2 decay_mult: 0 } }\n'
            'layer { name: "c2" type: "Convolution" bottom: "c" top: "c2" convolution_param { num_output: 4 '
            'kernel_size: 1 } }\n'
            'layer { name: "p2" type: "PReLU" bottom: "c2" top: "y" param { name: "slope" } }\n'
            'layer { name: "p3" type: "PReLU" bottom: "y" top: "z" prelu_param { channel_shared: true filler { '
            'type: "constant" value: 0.1 } } }\n'
            'layer { name: "ip" type: "InnerProduct" bottom: "z" top: "q" inner_product_param { num_output: 3 } }\n'
            'layer { name: "loss" type: "HingeLoss" bottom: "q" bottom: "t" top: "l" }')
    solver = _write(tmp_path, body, target=(2,))
    d = cos.parse_solver(solver)
    assert list(d.counts) == [12, 4, 4, 16, 4, 1, 432, 3]
    assert list(d.lr_mult) == [1, 1, 2, 1, 1, 1, 1, 1] and list(d.decay_mult) == [1, 1, 0, 1, 1, 1, 1, 1]
    text = cos.native_producer_plan(solver)
    lines = _op_lines(text)
    assert lines[1] == "op 1 PReLU p1 2x4x6x6 -> 2x4x6x6 w=16:4"
    assert lines[3] == "op 3 PReLU p2 2x4x6x6 -> 2x4x6x6 w=16:4 shares=2"
    assert lines[4] == "op 4 PReLU p3 2x4x6x6 -> 2x4x6x6 w=40:1 channel_shared"
    blobs = [line for line in text.splitlines() if line.startswith("blob ")]
    assert blobs[2] == "blob 2 16:4 4 constant" and blobs[5] == "blob 5 40:1 scalar constant"
    _check_layout(cos, text, solver, 476)
    (tmp_path / "m").mkdir()
    mism = body.replace('top: "y" param { name: "slope" }', 'top: "y" param { name: "slope" lr_mult: 3 }')
    with pytest.raises(cos.CosError, match=r"Shared param 'slope' has mismatched lr_mult\."):
        cos.parse_solver(_write(tmp_path / "m", mism, target=(2,)))


# --------------------------------------------------------------------------- the fixtures
TANH_OPS = [
    "op 0 Convolution conv1 64x1x28x28 -> 64x20x24x24 k5x5 s1x1 p0x0 w=0:500 b=500:20 staged-bottom",
    "op 1 Pooling(MAX) pool1 64x20x24x24 -> 64x20x12x12 k2x2 s2x2 p0x0",
    "op 2 TanH tanh_pool1 64x20x12x12 -> 64x20x12x12",
    "op 3 Convolution conv2 64x20x12x12 -> 64x50x8x8 k5x5 s1x1 p0x0 w=520:25000 b=25520:50",
    "op 4 Pooling(MAX) pool2 64x50x8x8 -> 64x50x4x4 k2x2 s2x2 p0x0",
    "op 5 TanH tanh_pool2 64x50x4x4 -> 64x50x4x4",
    "op 6 InnerProduct ip1 64x50x4x4 -> 64x500 w=25570:400000 b=425570:500",
    "op 7 TanH tanh1 64x500 -> 64x500",
    "op 8 InnerProduct ip2 64x500 -> 64x10 w=426070:5000 b=431070:10",
    "op 9 Softmax prob 64x10 -> 64x10 axis=1",
    "op 10 MultinomialLogisticLoss loss 64x10 -> scalar label=1 loss_weight=1",
]
PRELU_OPS = [
    "op 0 Convolution conv1 100x3x32x32 -> 100x32x32x32 k5x5 s1x1 p2x2 w=0:2400 b=2400:32 staged-bottom",
    "op 1 Pooling(MAX) pool1 100x32x32x32 -> 100x32x16x16 k3x3 s2x2 p0x0",
    "op 2 PReLU prelu1 100x32x16x16 -> 100x32x16x16 w=2432:32",
    "op 3 Convolution conv2 100x32x16x16 -> 100x32x16x16 k5x5 s1x1 p2x2 w=2464:25600 b=28064:32",
    "op 4 PReLU prelu2 100x32x16x16 -> 100x32x16x16 w=28096:32",
    "op 5 Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8 k3x3 s2x2 p0x0",
    "op 6 Convolution conv3 100x32x8x8 -> 100x64x8x8 k5x5 s1x1 p2x2 w=28128:51200 b=79328:64",
    "op 7 PReLU prelu3 100x64x8x8 -> 100x64x8x8 w=79392:64",
    "op 8 Pooling(AVE) pool3 100x64x8x8 -> 100x64x4x4 k3x3 s2x2 p0x0",
    "op 9 InnerProduct ip1 100x64x4x4 -> 100x64 w=79456:65536 b=144992:64",
    "op 10 PReLU prelu_ip1 100x64 -> 100x64 w=145056:1 channel_shared",
    "op 11 InnerProduct ip2 100x64 -> 100x10 w=145057:640 b=145697:10",
    "op 12 SoftmaxWithLoss loss 100x10 -> scalar axis=1 label=1 loss_weight=1",
]


def test_the_fixture_layouts(cos):
    from caffeonspark_b200 import nets
    d = cos.parse_solver(TANH_SOLVER)
    assert d.param_count == 431080 == nets.LENET_TANH_PARAM_COUNT == nets.EXPECTED_PARAM_COUNT["lenet"]
    assert [p.numel() for p in nets.lenet_tanh_module().parameters()] == list(d.counts)
    d = cos.parse_solver(PRELU_SOLVER)
    assert d.param_count == 145578 + 32 + 32 + 64 + 1 == nets.CIFAR10_QUICK_PRELU_PARAM_COUNT
    assert [p.numel() for p in nets.cifar10_quick_prelu_module().parameters()] == list(d.counts)
    slopes = [2, 5, 8, 11]
    assert [d.decay_mult[k] for k in slopes] == [0.0] * 4 and [d.lr_mult[k] for k in slopes] == [1.0] * 4
    assert "lenet_tanh" not in nets.NETS and "cifar10_quick_prelu" not in nets.NETS


@pytest.mark.parametrize("solver,ops,total", [(TANH_SOLVER, TANH_OPS, 431080), (PRELU_SOLVER, PRELU_OPS, 145707)])
def test_the_fixture_plans(cos, solver, ops, total):
    text = cos.native_producer_plan(solver)
    assert _op_lines(text) == ops
    _check_layout(cos, text, solver, total)
    blobs = [line.split()[-1] for line in text.splitlines() if line.startswith("blob ")]
    if solver == PRELU_SOLVER:
        assert [blobs[k] for k in (2, 5, 8, 11)] == ["constant"] * 4
        assert "blob 11 145056:1 scalar constant" in text
