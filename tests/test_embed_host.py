"""CPU tests of Embed and Reshape on the built-in engine (DESIGN.md section 14): the references of embed_ref.py against
torch and against plausible wrong versions, the parser's Reshape shapes against ReshapeLayer's inference across a table
of cases and every refusal, the Embed and Reshape plan lines and refusals, a shared Embed table, and both embedding
fixtures' layouts, counted independently, and full plans."""
import os
import re

import numpy as np
import pytest
import torch

import embed_ref as E
from conftest import ROOT
from test_autoencoder_host import _op_lines
from test_native_producer_host import _check_layout

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
TEXT_SOLVER = os.path.join(CONFIGS, "text_cnn_solver.prototxt")
LM_SOLVER = os.path.join(CONFIGS, "ngram_lm_solver.prototxt")


def _write(tmp_path, inputs, body):
    """A net of one Input layer with the tops `inputs` (name -> shape), then `body`."""
    tops = " ".join(f'top: "{n}"' for n in inputs)
    shapes = " ".join("shape { " + " ".join(f"dim: {d}" for d in s) + " }" for s in inputs.values())
    (tmp_path / "net.prototxt").write_text(
        f'name: "t" layer {{ name: "in" type: "Input" {tops} input_param {{ {shapes} }} }}\n' + body + "\n")
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / "solver.prototxt")


def _embed(name, bottom, top, input_dim, num_output, extra="", param=""):
    return (f'layer {{ name: "{name}" type: "Embed" bottom: "{bottom}" top: "{top}" {param} embed_param {{ '
            f'input_dim: {input_dim} num_output: {num_output} {extra} }} }}\n')


def _reshape(bottom, top, dims, axis=None, num_axes=None):
    p = "shape { " + " ".join(f"dim: {d}" for d in dims) + " }"
    p += f" axis: {axis}" if axis is not None else ""
    p += f" num_axes: {num_axes}" if num_axes is not None else ""
    return f'layer {{ name: "r" type: "Reshape" bottom: "{bottom}" top: "{top}" reshape_param {{ {p} }} }}\n'


EUCLID = 'layer { name: "loss" type: "EuclideanLoss" bottom: "%s" bottom: "t" top: "l" }'
SCALE = 'layer { name: "sc" type: "Scale" bottom: "x" top: "s" scale_param { axis: 0 } }\n'


# --------------------------------------------------------------------------- the references
def test_forward_reference_matches_torch():
    rng = np.random.RandomState(0)
    w, b = rng.randn(11, 5), rng.randn(5)
    ids = rng.randint(0, 11, (3, 4)).astype(F32)
    y = E.embed_forward(ids, w, b)
    want = torch.nn.functional.embedding(torch.from_numpy(ids).long(), torch.from_numpy(w)) + torch.from_numpy(b)
    assert y.shape == (3, 4, 5) and np.array_equal(y, want.numpy())
    bad = np.array([-1, 11, 0.5, np.nan, np.inf, -np.inf, 10, 0], F32)
    y = E.embed_forward(bad, w)
    assert not y[:6].any() and np.array_equal(y[6], w[10]) and np.array_equal(y[7], w[0])
    assert np.array_equal(E.embed_forward(bad, w, b)[:6], np.tile(b, (6, 1)))
    assert list(E.valid_rows(np.array([2 ** 24 - 1, 2 ** 24], F32), 2 ** 24)) == [2 ** 24 - 1, -1]


def test_backward_reference_is_torch_up_to_rounding_and_caffe_order_exactly():
    rng = np.random.RandomState(1)
    ids = rng.randint(0, 6, 200).astype(F32)
    dy = rng.randn(200, 3).astype(F32)
    w = torch.zeros(6, 3, dtype=torch.float64, requires_grad=True)
    torch.nn.functional.embedding(torch.from_numpy(ids).long(), w).backward(torch.from_numpy(dy.astype(np.float64)))
    g = E.embed_backward_cpu(ids, dy, np.zeros((6, 3), F32))
    assert np.allclose(g, w.grad.numpy(), rtol=1e-5, atol=1e-5)
    # the order by hand: row 0 of diff starts at 1, then gets 2^-24 three times: each add rounds back to 1
    ids = np.array([0, 1, 0, 0], F32)
    dy = np.array([[2.0 ** -24], [1.0], [2.0 ** -24], [2.0 ** -24]], F32)
    g = E.embed_backward_cpu(ids, dy, np.ones((2, 1), F32))
    assert g[0, 0] == 1 and g[1, 0] == 2
    assert E.embed_backward_summed_first(ids, dy, np.ones((2, 1), F32))[0, 0] > 1  # 3 * 2^-24 survives when summed first
    # invalid ids add nothing
    ids = np.array([-1, 2, 0.5, np.nan, np.inf], F32)
    assert not E.embed_backward_cpu(ids, np.ones((5, 2), F32), np.zeros((2, 2), F32)).any()


def test_backward_reference_is_not_the_summed_first_order():
    """The mutation: summing each id's rows before one add into diff differs from Caffe's order on repeated ids."""
    rng = np.random.RandomState(2)
    ids = (rng.zipf(1.5, 4096) % 50).astype(F32)
    dy = (rng.randn(4096, 16) * np.exp2(rng.randint(-8, 8, (4096, 1)))).astype(F32)
    diff = (rng.randn(50, 16) * 100).astype(F32)
    a, b = E.embed_backward_cpu(ids, dy, diff), E.embed_backward_summed_first(ids, dy, diff)
    assert (a != b).sum() > 100
    assert np.allclose(a, b, rtol=1e-4, atol=1e-3)  # both sum the same rows


# --------------------------------------------------------------------------- Reshape's shape inference
RESHAPE_CASES = [  # (bottom, dims, axis, num_axes) -> top shape, or the refusal's wording
    ((2, 3, 4, 5), [0, -1], None, None, (2, 60)),
    ((2, 3, 4, 5), [0, 0, 20], None, None, (2, 3, 20)),
    ((2, 3, 4, 5), [-1], None, None, (120,)),
    ((2, 3, 4, 5), [6, -1, 5], None, None, (6, 4, 5)),
    ((2, 3, 4, 5), [0, 0, 0, 0], None, None, (2, 3, 4, 5)),
    ((50, 32, 64), [0, 1, -1, 64], None, None, (50, 1, 32, 64)),
    ((6,), [2, -1], None, None, (2, 3)),
    ((2, 6, 4, 5), [2, 3], 1, 1, (2, 2, 3, 4, 5)),
    ((2, 3, 4, 5), [1], 2, 0, (2, 3, 1, 4, 5)),
    ((2, 3, 4, 5), [1], -1, 0, (2, 3, 4, 5, 1)),
    ((2, 3, 4, 5), [1, 1], 4, 0, (2, 3, 4, 5, 1, 1)),
    ((2, 3, 4, 5), [-1], -3, None, (2, 3, 20)),
    ((2, 3, 4, 5), [0, -1], -3, None, (2, 3, 4, 5)),
    ((2, 3, 4, 5), [0, -1], -2, 1, (2, 3, 4, 5, 1)),
    ((2, 3, 4, 5), [-1, 2], 1, 2, (2, 6, 2, 5)),
    ((2, 3, 4, 5), [3, 4, 5], -4, -1, (2, 3, 4, 5)),
    ((2, 3, 4, 5), [-1, -1], None, None, "new shape contains multiple -1 dims; at most a single (1) value of -1 may be "
                                         "specified"),
    ((2, 3, 4, 5), [-1], -6, None, "axis -6 out of range"),
    ((2, 3, 4, 5), [-1], 5, None, "axis 5 out of range for 4-D input blob"),
    ((2, 3, 4, 5), [-1], 0, -2, "num_axes must be >= 0, or -1 for all"),
    ((2, 3, 4, 5), [-1], 3, 2, "end_axis = axis + num_axes is out of range"),
    ((2, 3, 4, 5), [0, 0, 0, 0, 0], None, None, "new shape contains a 0, but there was no corresponding bottom axis to "
                                                "copy"),
    ((2, 3, 4, 5), [7, -1], None, None, "bottom count (120) must be divisible by the product of the specified "
                                        "dimensions (7)"),
    ((2, 3, 4, 5), [7, 8], None, None, "output count must match input count"),
    ((2, 3, 4, 5), [0], 4, 0, "new shape contains a 0, but there was no corresponding bottom axis to copy"),
]


def _ref(bottom, dims, axis, num_axes, start_of=None):
    try:
        return E.reshape_shape(bottom, dims, 0 if axis is None else axis, -1 if num_axes is None else num_axes,
                               start_of)
    except E.ReshapeError as e:
        return str(e)


def test_reshape_reference_follows_the_table():
    for bottom, dims, axis, num_axes, want in RESHAPE_CASES:
        assert _ref(bottom, dims, axis, num_axes) == want, (bottom, dims, axis, num_axes)


def test_reshape_reference_catches_an_axis_off_by_one():
    for start_of in (lambda a, n: a if a >= 0 else n + a, lambda a, n: a + 1 if a >= 0 else n + a + 1):
        assert any(_ref(b, d, a, k, start_of) != want for b, d, a, k, want in RESHAPE_CASES)


@pytest.mark.parametrize("case", range(len(RESHAPE_CASES)))
def test_the_parser_reshapes_as_caffe(cos, tmp_path, case):
    bottom, dims, axis, num_axes, want = RESHAPE_CASES[case]
    body = SCALE + _reshape("s", "r", dims, axis, num_axes) + EUCLID % "r"
    if isinstance(want, str):
        with pytest.raises(cos.CosError, match="^layer 'r' \\(Reshape\\): " + re.escape(want) + "$"):
            cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": (1,)}, body))
        return
    text = cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": want}, body))
    shape = "x".join(str(d) for d in bottom)
    assert _op_lines(text)[1] == f"op 1 Reshape r {shape} -> {'x'.join(str(d) for d in want)} data=bottom diff=bottom"


def test_reshape_of_a_staged_input_keeps_its_own_gradient(cos, tmp_path):
    body = _reshape("x", "r", [0, -1]) + EUCLID % "r"
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 4), "t": (2, 12)}, body)))
    assert lines[0] == "op 0 Reshape r 2x3x4 -> 2x12 data=bottom staged-bottom"


def test_reshape_refuses_in_place_and_flatten_is_unchanged(cos, tmp_path):
    body = SCALE + _reshape("s", "s", [0, -1]) + EUCLID % "s"
    with pytest.raises(cos.CosError, match=r"^layer 'r' \(Reshape\): Reshape Layer does not allow in-place "
                                           r"computation\. \(native producer\)$"):
        cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 4), "t": (2, 12)}, body))
    (tmp_path / "f").mkdir()
    body = SCALE + 'layer { name: "f" type: "Flatten" bottom: "s" top: "s" }\n' + EUCLID % "s"
    with pytest.raises(cos.CosError, match=r"^layer 'f' \(Flatten\): Flatten Layer does not allow in-place "
                                           r"computation\. \(native producer\)$"):
        cos.native_producer_plan(_write(tmp_path / "f", {"x": (2, 3, 4), "t": (2, 12)}, body))


# --------------------------------------------------------------------------- Embed
@pytest.mark.parametrize("ids,bias", [((6,), True), ((4, 6), True), ((2, 3, 4), False)])
def test_embed_plan(cos, tmp_path, ids, bias):
    extra = "" if bias else "bias_term: false"
    out = ids + (8,)
    solver = _write(tmp_path, {"ids": ids, "t": out}, _embed("e", "ids", "y", 10, 8, extra) + EUCLID % "y")
    d = cos.parse_solver(solver)
    assert d.counts == [80] + ([8] if bias else [])
    text = cos.native_producer_plan(solver)
    shape = "x".join(str(v) for v in ids)
    w = "w=0:80" + (" b=80:8" if bias else "")
    assert _op_lines(text)[0] == f"op 0 Embed e {shape} -> {shape}x8 input_dim=10 num_output=8 {w} staged-bottom"
    assert "blob 0 0:80 10x8 constant" in text and (("blob 1 80:8 8 constant" in text) == bias)
    _check_layout(cos, text, solver, 80 + 8 * bias)


def test_embed_blobs_take_fillers_multipliers_and_the_largest_input_dim(cos, tmp_path):
    extra = ('weight_filler { type: "gaussian" std: 0.5 } bias_filler { type: "constant" value: 0.25 }')
    param = "param { lr_mult: 3 decay_mult: 0 } param { lr_mult: 2 }"
    solver = _write(tmp_path, {"ids": (5,), "t": (5, 1)}, _embed("e", "ids", "y", 2 ** 24, 1, extra, param) +
                    EUCLID % "y")
    d = cos.parse_solver(solver)
    assert d.counts == [2 ** 24, 1] and d.lr_mult == [3.0, 2.0] and d.decay_mult == [0.0, 1.0]
    text = cos.native_producer_plan(solver)
    assert f"blob 0 0:{2 ** 24} {2 ** 24}x1 gaussian" in text and f"blob 1 {2 ** 24}:1 1 constant" in text


def test_a_shared_embed_table(cos, tmp_path):
    param = 'param { name: "table" }'
    body = (_embed("e1", "a", "ya", 10, 4, "bias_term: false", param) +
            _embed("e2", "b", "yb", 10, 4, "bias_term: false", param) +
            'layer { name: "cat" type: "Concat" bottom: "ya" bottom: "yb" top: "y" concat_param { axis: 0 } }\n' +
            EUCLID % "y")
    solver = _write(tmp_path, {"a": (3,), "b": (5,), "t": (8, 4)}, body)
    assert cos.parse_solver(solver).counts == [40]
    lines = _op_lines(cos.native_producer_plan(solver))
    assert lines[:2] == ["op 0 Embed e1 3 -> 3x4 input_dim=10 num_output=4 w=0:40 staged-bottom",
                         "op 1 Embed e2 5 -> 5x4 input_dim=10 num_output=4 w=0:40 shares=0 staged-bottom"]


@pytest.mark.parametrize("body,match", [
    (_embed("e", "ids", "y", 10, 0), r"^layer 'e' \(Embed\): EmbedLayer num_output must be positive\.$"),
    (_embed("e", "ids", "y", 0, 8), r"^layer 'e' \(Embed\): EmbedLayer input_dim must be positive\.$"),
    ('layer { name: "e" type: "Embed" bottom: "ids" top: "y" }\n',
     r"^layer 'e' \(Embed\): EmbedLayer num_output must be positive\.$"),
    (_embed("e", "ids", "y", 2 ** 24 + 1, 8), r"^layer 'e' \(Embed\): input_dim 16777217 is more than 2\^24"),
    ('layer { name: "sc" type: "Scale" bottom: "ids" top: "s" }\n' + _embed("e", "s", "y", 10, 8),
     r"^layer 'e' \(Embed\): Can't backpropagate to EmbedLayer input\. \(native producer\)$"),
    (_embed("e", "ids", "y", 10, 8) + _embed("e2", "ids", "y2", 10, 8),
     r"^layer 'e2' \(Embed\): bottom 'ids' already feeds layer 'e'; a blob read by two layers needs a Split"),
])
def test_embed_refusals_name_the_layer(cos, tmp_path, body, match):
    with pytest.raises(cos.CosError, match=match):
        cos.native_producer_plan(_write(tmp_path, {"ids": (4, 6), "t": (4, 6, 8)}, body + EUCLID % "y"))


def test_an_embed_off_the_loss_runs_no_backward(cos, tmp_path):
    body = (_embed("e", "ids", "y", 10, 8) + _embed("e2", "ids2", "y2", 10, 8) + EUCLID % "y" +
            '\nlayer { name: "s" type: "Silence" bottom: "y2" }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, {"ids": (4, 6), "t": (4, 6, 8), "ids2": (3,)}, body)))
    assert lines[1] == "op 1 Embed e2 3 -> 3x8 input_dim=10 num_output=8 w=88:80 b=168:8 staged-bottom no-backward"


# --------------------------------------------------------------------------- the fixtures
def _text_cnn_count():
    s = dict(vocab=5000, dim=64, widths=(3, 4, 5), filters=32, classes=2)
    convs = [(s["filters"] * k * s["dim"], s["filters"]) for k in s["widths"]]
    ip = (s["classes"] * s["filters"] * len(s["widths"]), s["classes"])
    return [s["vocab"] * s["dim"]] + [c for pair in convs + [ip] for c in pair]


def _ngram_count():
    vocab, dim, tokens, hidden = 2000, 32, 4, 128
    return [vocab * dim, dim, hidden * tokens * dim, hidden, vocab * hidden, vocab]


def test_the_fixture_layouts(cos):
    from caffeonspark_b200 import nets
    for solver, counts, total, blobs, module in (
            (TEXT_SOLVER, _text_cnn_count(), 344866, 9, nets.text_cnn_module()),
            (LM_SOLVER, _ngram_count(), 338544, 6, nets.ngram_lm_module())):
        assert sum(counts) == total and len(counts) == blobs
        d = cos.parse_solver(solver)
        assert d.param_count == total and list(d.counts) == counts
        assert [p.numel() for p in module.parameters()] == counts
        assert d.batch_size == (50 if solver == TEXT_SOLVER else 128)
    assert nets.TEXT_CNN_PARAM_COUNT == 344866 and nets.NGRAM_LM_PARAM_COUNT == 338544
    text = cos.native_producer_plan(TEXT_SOLVER)
    shapes = [line.split()[3] for line in text.splitlines() if line.startswith("blob ")]
    assert shapes == ["5000x64", "32x1x3x64", "32", "32x1x4x64", "32", "32x1x5x64", "32", "2x96", "2"]
    assert cos.parse_solver(TEXT_SOLVER).lr_mult == [1.0] + [1.0, 2.0] * 4
    text = cos.native_producer_plan(LM_SOLVER)
    blobs = [line.split()[3:] for line in text.splitlines() if line.startswith("blob ")]
    # the Embed's bias is there by default (bias_term true), a constant-0 [32]
    assert blobs == [["2000x32", "uniform"], ["32", "constant"], ["128x128", "xavier"], ["128", "constant"],
                     ["2000x128", "xavier"], ["2000", "constant"]]
    assert cos.parse_solver(LM_SOLVER).lr_mult == [1.0, 2.0] * 3


TEXT_OPS = [
    "op 0 Embed embed 50x32 -> 50x32x64 input_dim=5000 num_output=64 w=0:320000 staged-bottom",
    "op 1 Reshape reshape 50x32x64 -> 50x1x32x64 data=bottom diff=bottom",
    "op 2 Split sentence_split 50x1x32x64 -> 50x1x32x64 top=0 data=bottom",
    "op 3 Split sentence_split 50x1x32x64 -> 50x1x32x64 top=1 data=bottom",
    "op 4 Split sentence_split 50x1x32x64 -> 50x1x32x64 top=2 data=bottom",
    "op 5 Convolution conv3 50x1x32x64 -> 50x32x30x1 k3x64 s1x1 p0x0 w=320000:6144 b=326144:32",
    "op 6 ReLU relu3 50x32x30x1 -> 50x32x30x1 in-place",
    "op 7 Pooling(MAX) pool3 50x32x30x1 -> 50x32x1x1 k30x1 s1x1 p0x0",
    "op 8 Convolution conv4 50x1x32x64 -> 50x32x29x1 k4x64 s1x1 p0x0 w=326176:8192 b=334368:32",
    "op 9 ReLU relu4 50x32x29x1 -> 50x32x29x1 in-place",
    "op 10 Pooling(MAX) pool4 50x32x29x1 -> 50x32x1x1 k29x1 s1x1 p0x0",
    "op 11 Convolution conv5 50x1x32x64 -> 50x32x28x1 k5x64 s1x1 p0x0 w=334400:10240 b=344640:32",
    "op 12 ReLU relu5 50x32x28x1 -> 50x32x28x1 in-place",
    "op 13 Pooling(MAX) pool5 50x32x28x1 -> 50x32x1x1 k28x1 s1x1 p0x0",
    "op 14 Concat concat 50x32x1x1 -> 50x96x1x1 axis=1 begin=0",
    "op 15 Concat concat 50x32x1x1 -> 50x96x1x1 axis=1 begin=32",
    "op 16 Concat concat 50x32x1x1 -> 50x96x1x1 axis=1 begin=64",
    "op 17 InnerProduct ip 50x96x1x1 -> 50x2 w=344672:192 b=344864:2",
    "op 18 SoftmaxWithLoss loss 50x2 -> scalar axis=1 label=1 loss_weight=1",
]
LM_OPS = [
    "op 0 Embed embed 128x4 -> 128x4x32 input_dim=2000 num_output=32 w=0:64000 b=64000:32 staged-bottom",
    "op 1 InnerProduct hidden 128x4x32 -> 128x128 w=64032:16384 b=80416:128",
    "op 2 TanH tanh 128x128 -> 128x128",
    "op 3 InnerProduct predict 128x128 -> 128x2000 w=80544:256000 b=336544:2000",
    "op 4 SoftmaxWithLoss loss 128x2000 -> scalar axis=1 label=1 loss_weight=1",
]


@pytest.mark.parametrize("solver,ops,inputs,total", [
    (TEXT_SOLVER, TEXT_OPS, "input 0 tokens 1600\ninput 1 label 50\n", 344866),
    (LM_SOLVER, LM_OPS, "input 0 context 512\ninput 1 next 128\n", 338544)])
def test_the_fixture_plans(cos, solver, ops, inputs, total):
    text = cos.native_producer_plan(solver)
    assert text.startswith(inputs + "op 0 ")
    assert _op_lines(text) == ops
    _check_layout(cos, text, solver, total)
