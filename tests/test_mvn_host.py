"""CPU tests of Caffe's MVN layer on the built-in engine (DESIGN.md section 14): mvn_ref.py's float64 reference
against a hand-worked case, central finite differences (where s >> eps) and layers.MVN; its fp32 restatement against
its bounds, and every plausible wrong version it lists outside them; the parser's legacy 4-D tops and refusals; the
plan of in-place and staged-input MVNs; and both MVN fixtures' layouts and plans, line for line."""
import os
import re

import numpy as np
import pytest
import torch

import mvn_ref as M
from conftest import ROOT
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
EUCLID = 'layer {{ name: "loss" type: "EuclideanLoss" bottom: "{}" bottom: "t" top: "l" }}\n'
SCALE = 'layer { name: "s" type: "Scale" bottom: "x" top: "a" scale_param { axis: 0 } }\n'


def _mvn(bottom, top, param=""):
    return f'layer {{ name: "m" type: "MVN" bottom: "{bottom}" top: "{top}" mvn_param {{ {param} }} }}\n'


# --------------------------------------------------------------------------- the reference
def _hand_ok(mutation=None, eps=0.0):
    """One row x = 1, 2, 3, 4: mu 2.5, var 1.25, y = (x - mu) / sqrt(1.25); dy = e_0."""
    x = np.array([[[1.0, 2.0, 3.0, 4.0]]])
    y, s = M.forward(x, True, False, eps, mutation)
    if y.shape != (1, 1, 4, 1):
        return False
    sd = np.sqrt(1.25) + eps
    want_y = (np.array([1.0, 2.0, 3.0, 4.0]) - 2.5) / sd
    if not np.allclose(y.ravel(), want_y, rtol=1e-14):
        return False
    dx = M.backward(y, np.array([1.0, 0, 0, 0]), s, False, mutation)
    a = want_y[0]  # sum(y dy)
    want_dx = (np.array([1.0, 0, 0, 0]) - (want_y * a + 1.0) / 4) / sd
    return np.allclose(dx.ravel(), want_dx, rtol=1e-13)


def _fd_ok(mutation=None, h=1e-6):
    """Caffe's backward formula against central differences of sum(R * y) where s >> eps (eps 1e-9, s ~ 1)."""
    rng = np.random.RandomState(4)
    x, R = rng.randn(2, 3, 5), rng.randn(2, 3, 5, 1)
    y, s = M.forward(x, True, False, 1e-9, mutation)
    dx = M.backward(y, R, s, False, mutation).reshape(x.shape)
    for i in range(x.size):
        v = x.flat[i]
        x.flat[i] = v + h
        up = (M.forward(x, True, False, 1e-9, mutation)[0].reshape(R.shape) * R).sum()
        x.flat[i] = v - h
        down = (M.forward(x, True, False, 1e-9, mutation)[0].reshape(R.shape) * R).sum()
        x.flat[i] = v
        if abs((up - down) / (2 * h) - dx.flat[i]) > 1e-6 * max(1.0, abs(dx.flat[i])):
            return False
    return True


def _bounds_ok(mutation=None):
    """fp32 results (sums left to right) within the bounds (from the true float64 values) around the possibly mutated
    float64 reference, eps 1e-3, and its top of the legacy shape."""
    rng = np.random.RandomState(6)
    powf = M.glibc_powf_half()
    for shape, across in (((3, 4, 5, 6), False), ((5, 64), True), ((2, 3, 33), False)):
        x = (rng.randn(*shape) * 2 + 0.7).astype(np.float32)
        rows, dim = M.rows_dim(shape, across)
        y64, s64 = M.forward(x, True, across, 1e-3)
        ym, sm = M.forward(x, True, across, 1e-3, mutation)
        if ym.shape != M.legacy_shape(shape):
            return False
        y32, s32 = M.sequential32(x.reshape(rows, dim), True, 1e-3, powf)
        by = M.bound_y(x.reshape(rows, dim), y64, s64)
        if (np.abs(y32 - ym.reshape(rows, dim)) > by).any():
            return False
        dy = rng.randn(rows, dim).astype(np.float32)
        a = np.add.accumulate((y32 * dy).astype(np.float32), axis=1, dtype=np.float32)[:, -1]
        b = np.add.accumulate(dy, axis=1, dtype=np.float32)[:, -1]
        dx32 = M.backward32(y32, dy, a, b, s32, True)
        dxm = M.backward(ym, dy, sm, across, mutation).reshape(rows, dim)
        if (np.abs(dx32 - dxm) > M.bound_dx(y64.reshape(rows, dim), dy, s64, by)).any():
            return False
    return True


def test_reference_passes_every_check():
    assert _hand_ok()
    assert _hand_ok(eps=1e-3)
    assert _fd_ok()
    assert _bounds_ok()


# the checks each wrong version fails; every one falls outside the bounds
FAILS = {"eps_in_sqrt": {"hand_eps", "bounds"}, "unbiased_var": {"hand", "hand_eps", "fd", "bounds"},
         "drop_y_term": {"hand", "hand_eps", "fd", "bounds"}, "per_sample_rows": {"bounds"},
         "bottom_shape_top": {"hand", "hand_eps", "bounds"}}


@pytest.mark.parametrize("mutation", M.MUTATIONS)
def test_every_mutation_fails_a_check(mutation):
    passed = {"hand": _hand_ok(mutation), "hand_eps": _hand_ok(mutation, eps=1e-3), "fd": _fd_ok(mutation),
              "bounds": _bounds_ok(mutation)}
    assert {k for k, ok in passed.items() if not ok} == FAILS[mutation]


def test_a_shape_of_2_to_the_31_elements_is_refused():
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for rows, dim in ((1, 1 << 31), (2, 1 << 30), (3, (1 << 31) // 3 + 1)):
        assert not L.cos_mvn_forward(1, 1, 1, 1, rows, dim, 1, 1e-9, None)
        assert "bad shape" in L.cos_last_error().decode()
        assert not L.cos_mvn_backward(1, 1, 1, 1, 1, rows, dim, 1, None)
        assert "bad shape" in L.cos_last_error().decode()


@pytest.mark.parametrize("variance", [True, False])
@pytest.mark.parametrize("shape,across", [((2, 3, 4, 5), False), ((4, 6), True), ((3, 7, 5), False), ((6,), True)])
def test_layers_mvn_matches_the_reference(shape, across, variance):
    from caffeonspark_b200 import layers
    rng = np.random.RandomState(len(shape))
    x = torch.from_numpy(rng.randn(*shape) * 2 + 1).requires_grad_()
    y = layers.MVN.apply(x, variance, across, 1e-3)
    y64, s64 = M.forward(x.detach().numpy(), variance, across, 1e-3)
    assert tuple(y.shape) == M.legacy_shape(shape)
    np.testing.assert_allclose(y.detach().numpy(), y64, rtol=1e-13, atol=1e-14)
    dy = rng.randn(*y.shape)
    y.backward(torch.from_numpy(dy))
    want = M.backward(y64, dy, s64, across).reshape(shape)
    np.testing.assert_allclose(x.grad.numpy(), want, rtol=1e-12, atol=1e-13)


# --------------------------------------------------------------------------- the parser and the plan
def _plan(cos, tmp_path, inputs, body):
    return cos.native_producer_plan(_write(tmp_path, inputs, body))


@pytest.mark.parametrize("bottom,top", [((6, 5), (6, 5, 1, 1)), ((4, 3, 7), (4, 3, 7, 1)), ((9,), (9, 1, 1, 1)),
                                        ((2, 3, 4, 5), (2, 3, 4, 5))])
def test_the_top_is_the_legacy_4d_shape(cos, tmp_path, bottom, top):
    body = SCALE + _mvn("a", "y") + EUCLID.format("y")
    text = _plan(cos, tmp_path, {"x": bottom, "t": top}, body)
    line = [ln for ln in text.splitlines() if " MVN " in ln][0]
    assert f"{'x'.join(map(str, bottom))} -> {'x'.join(map(str, top))} " in line
    n, c = M.legacy_shape(bottom)[:2]
    assert f" rows={n * c} dim={int(np.prod(bottom)) // (n * c)} eps=1e-09" in line


def test_downstream_shape_inference_sees_the_4d_top(cos, tmp_path):
    # a Scale on axis 3 of an [N, C] bottom exists only on the 4-D top
    body = (SCALE + _mvn("a", "y", "across_channels: true") +
            'layer { name: "s3" type: "Scale" bottom: "y" top: "z" scale_param { axis: 3 } }\n' + EUCLID.format("z"))
    text = _plan(cos, tmp_path, {"x": (4, 6), "t": (4, 6, 1, 1)}, body)
    assert "op 1 MVN m 4x6 -> 4x6x1x1 rows=4 dim=6 eps=1e-09 across" in text
    assert "op 2 Scale s3 4x6x1x1 -> 4x6x1x1 w=4:1 outer=24 dim=1 inner=1" in text


@pytest.mark.parametrize("bottom,want", [
    ((2, 3, 4, 5, 6), "Cannot use legacy accessors on Blobs with > 4 axes."),
    ((2, 0, 3), "a bottom of shape 2x0x3 has no elements to normalise"),
])
def test_refusals(cos, tmp_path, bottom, want):
    body = _mvn("x", "y") + EUCLID.format("y")
    with pytest.raises(cos.CosError, match="^layer 'm' \\(MVN\\): " + re.escape(want) + "$"):
        _plan(cos, tmp_path, {"x": bottom, "t": (1,)}, body)


def test_params_mean_only_eps_and_extra_param_entries(cos, tmp_path):
    body = (SCALE + 'layer { name: "m" type: "MVN" bottom: "a" top: "y" param { lr_mult: 0 } '
            'mvn_param { normalize_variance: false across_channels: true eps: 0.5 } }\n' + EUCLID.format("y"))
    text = _plan(cos, tmp_path, {"x": (3, 4, 5), "t": (3, 4, 5, 1)}, body)
    assert "op 1 MVN m 3x4x5 -> 3x4x5x1 rows=3 dim=20 eps=0.5 across mean-only\n" in text
    assert "params 3 blobs 1" in text  # the MVN owns no blob


def test_in_place_gets_a_top_of_its_own(cos, tmp_path):
    body = SCALE + _mvn("a", "a") + EUCLID.format("a")
    text = _plan(cos, tmp_path, {"x": (2, 3, 4, 4), "t": (2, 3, 4, 4)}, body)
    line = [ln for ln in text.splitlines() if " MVN " in ln][0]
    assert line == "op 1 MVN m 2x3x4x4 -> 2x3x4x4 rows=6 dim=16 eps=1e-09"


def test_on_a_staged_input_no_data_gradient_is_computed(cos, tmp_path):
    body = (_mvn("x", "n") + 'layer { name: "c" type: "Convolution" bottom: "n" top: "y" convolution_param { '
            'num_output: 2 kernel_size: 3 } }\n' + EUCLID.format("y"))
    text = _plan(cos, tmp_path, {"x": (2, 3, 5, 5), "t": (2, 2, 3, 3)}, body)
    assert "op 0 MVN m 2x3x5x5 -> 2x3x5x5 rows=6 dim=25 eps=1e-09 staged-bottom\n" in text
    assert "op 1 Convolution c 2x3x5x5 -> 2x2x3x3 k3x3 s1x1 p0x0 w=0:54 b=54:2 no-bottom-grad\n" in text


QUICK_OPS = """\
op 0 MVN mvn_data 100x3x32x32 -> 100x3x32x32 rows=300 dim=1024 eps=1e-09 staged-bottom
op 1 ConvBiasReLUMaxPool conv1+pool1+relu1 100x3x32x32 -> 100x32x16x16 k5x5 s1x1 p2x2 pool3/2 w=0:2400 b=2400:32 no-bottom-grad
op 2 Convolution conv2 100x32x16x16 -> 100x32x16x16 k5x5 s1x1 p2x2 w=2432:25600 b=28032:32
op 3 MVN mvn2 100x32x16x16 -> 100x32x16x16 rows=3200 dim=256 eps=1e-09
op 4 Scale scale2 100x32x16x16 -> 100x32x16x16 w=28064:32 b=28096:32 outer=100 dim=32 inner=256
op 5 ReLU relu2 100x32x16x16 -> 100x32x16x16 in-place
op 6 Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8 k3x3 s2x2 p0x0
op 7 MVN mvn_pool2 100x32x8x8 -> 100x32x8x8 rows=3200 dim=64 eps=1e-09 mean-only
op 8 Convolution conv3 100x32x8x8 -> 100x64x8x8 k5x5 s1x1 p2x2 w=28128:51200 b=79328:64
op 9 ReLU relu3 100x64x8x8 -> 100x64x8x8 in-place
op 10 Pooling(AVE) pool3 100x64x8x8 -> 100x64x4x4 k3x3 s2x2 p0x0
op 11 MVN mvn3 100x64x4x4 -> 100x64x4x4 rows=6400 dim=16 eps=0.001
op 12 Scale scale3 100x64x4x4 -> 100x64x4x4 w=79392:64 b=79456:64 outer=100 dim=64 inner=16
op 13 InnerProduct ip1 100x64x4x4 -> 100x64 w=79520:65536 b=145056:64
op 14 MVN mvn_ip1 100x64 -> 100x64x1x1 rows=100 dim=64 eps=1e-09 across
op 15 InnerProduct ip2 100x64x1x1 -> 100x10 w=145120:640 b=145760:10
op 16 SoftmaxWithLoss loss 100x10 -> scalar axis=1 label=1 loss_weight=1
"""
LM_OPS = """\
op 0 Embed embed 20x32 -> 20x32x128 input_dim=2000 num_output=128 w=0:256000 staged-bottom
op 1 RNN rnn 20x32x128 -> 20x32x256 T=20 N=32 H=256 cont=0 w_xh=256000 b_h=288768 w_hh=289024 w_ho=354560 b_o=420096
op 2 MVN ln 20x32x256 -> 20x32x256x1 rows=640 dim=256 eps=1e-09
op 3 Scale ln_scale 20x32x256x1 -> 20x32x256x1 w=420352:256 b=420608:256 outer=640 dim=256 inner=1
op 4 InnerProduct predict 20x32x256x1 -> 20x32x2000 w=420864:512000 b=932864:2000
op 5 SoftmaxWithLoss loss 20x32x2000 -> scalar axis=2 label=2 loss_weight=1
"""


@pytest.mark.parametrize("name,ops,total", [("cifar10_quick_mvn", QUICK_OPS, 145770), ("rnn_lm_ln", LM_OPS, 934864)])
def test_fixture_layouts_and_plans(cos, name, ops, total):
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, f"{name}_solver.prototxt")
    text = cos.native_producer_plan(solver)
    assert "".join(ln + "\n" for ln in text.splitlines() if ln.startswith("op ")) == ops
    _check_layout(cos, text, solver, total)
    m = nets.cifar10_quick_mvn_module() if name == "cifar10_quick_mvn" else nets.rnn_lm_ln_module()
    assert [p.numel() for p in m.parameters()] == cos.parse_solver(solver).counts
    assert total == (nets.CIFAR10_QUICK_MVN_PARAM_COUNT if name == "cifar10_quick_mvn" else nets.RNN_LM_LN_PARAM_COUNT)
