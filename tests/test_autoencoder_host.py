"""CPU tests of Deconvolution, Flatten and SigmoidCrossEntropyLoss on the built-in engine (DESIGN.md section 14): their
plan lines, the two rules that let Caffe's MNIST autoencoder run as written (a loss of weight 0 does no TRAIN work;
only ops under the loss run a backward), every refusal with the layer's name and Caffe's wording, and both autoencoder
fixtures' layouts, counted independently, and full plans."""
import os

import pytest

from conftest import ROOT
from test_native_producer_host import _check_layout, _ops

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
FC_SOLVER = os.path.join(CONFIGS, "mnist_autoencoder_solver.prototxt")
CONV_SOLVER = os.path.join(CONFIGS, "mnist_conv_autoencoder_solver.prototxt")


def _write(tmp_path, body, shape=(2, 3, 6, 6), target=None):
    """A net of an Input `x` of `shape` and a target `t` of shape `target` (the same by default), then `body`."""
    dims, tdims = (" ".join(f"dim: {d}" for d in s) for s in (shape, target or shape))
    (tmp_path / "net.prototxt").write_text(
        f'name: "t" layer {{ name: "in" type: "Input" top: "x" top: "t" input_param {{ shape {{ {dims} }} '
        f'shape {{ {tdims} }} }} }}\n' + body + "\n")
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / "solver.prototxt")


def _op_lines(text):
    return [line for line in text.splitlines() if line.startswith("op ")]


def _deconv(name, bottom, top, cout, param="kernel_size: 4 stride: 2 pad: 1"):
    return (f'layer {{ name: "{name}" type: "Deconvolution" bottom: "{bottom}" top: "{top}" convolution_param {{ '
            f'num_output: {cout} {param} }} }}\n')


SCE = 'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "%s" bottom: "t" top: "l" }'


# --------------------------------------------------------------------------- Deconvolution
@pytest.mark.parametrize("param,out,geo,bias", [
    ("kernel_size: 4 stride: 2 pad: 1", "2x1x12x12", "k4x4 s2x2 p1x1", True),
    ("kernel_size: 3", "2x1x8x8", "k3x3 s1x1 p0x0", True),
    ("kernel_h: 2 kernel_w: 5 stride_h: 3 stride_w: 1 pad_h: 0 pad_w: 2", "2x1x17x6", "k2x5 s3x1 p0x2", True),
    ("kernel_size: 3 stride: 2 pad: 1 bias_term: false", "2x1x11x11", "k3x3 s2x2 p1x1", False),
])
def test_deconvolution_plan(cos, tmp_path, param, out, geo, bias):
    target = tuple(int(v) for v in out.split("x"))
    solver = _write(tmp_path, _deconv("dc", "x", "y", 1, param) + SCE % "y", target=target)
    d = cos.parse_solver(solver)
    kh, kw = (int(v) for v in geo.split()[0][1:].split("x"))
    assert d.counts == [3 * 1 * kh * kw] + ([1] if bias else [])  # [Cin, Cout, KH, KW]: the parser's layout
    text = cos.native_producer_plan(solver)
    line = _op_lines(text)[0]
    w = f"w=0:{3 * kh * kw}" + (f" b={3 * kh * kw}:1" if bias else "")
    assert line == f"op 0 Deconvolution dc 2x3x6x6 -> {out} {geo} {w} staged-bottom"
    assert f"blob 0 0:{3 * kh * kw} 3x1x{kh}x{kw} constant" in text
    _check_layout(cos, text, solver, sum(d.counts))


def test_deconvolution_is_never_fused_and_shares_like_convolution(cos, tmp_path):
    share = 'param { name: "w" } param { name: "b" } convolution_param'
    body = ('layer { name: "c" type: "Convolution" bottom: "x" top: "c" convolution_param { num_output: 4 '
            'kernel_size: 3 pad: 1 } }\n' +
            _deconv("da", "c", "a", 4, 'kernel_size: 2 stride: 2 weight_filler { type: "xavier" } '
                    'bias_filler { type: "constant" value: 0.5 }').replace("convolution_param", share) +
            'layer { name: "r" type: "ReLU" bottom: "a" top: "a" }\n'
            'layer { name: "p" type: "Pooling" bottom: "a" top: "p" pooling_param { pool: MAX kernel_size: 2 '
            'stride: 2 } }\n' +
            _deconv("db", "p", "y", 4, "kernel_size: 2 stride: 2").replace("convolution_param", share) +
            'layer { name: "f" type: "Convolution" bottom: "y" top: "z" convolution_param { num_output: 3 '
            'kernel_size: 1 } }\n' + SCE % "z")
    text = cos.native_producer_plan(_write(tmp_path, body, target=(2, 3, 12, 12)))
    lines = _op_lines(text)
    # a Deconvolution with a bias before ReLU and MAX pool stays three ops
    assert [line.split()[2] for line in lines] == ["Convolution", "Deconvolution", "ReLU", "Pooling(MAX)",
                                                   "Deconvolution", "Convolution", "SigmoidCrossEntropyLoss"]
    assert lines[1] == "op 1 Deconvolution da 2x4x6x6 -> 2x4x12x12 k2x2 s2x2 p0x0 w=112:64 b=176:4"
    assert lines[2].endswith(" in-place")
    assert lines[4] == "op 4 Deconvolution db 2x4x6x6 -> 2x4x12x12 k2x2 s2x2 p0x0 w=112:64 b=176:4 shares=2,3"
    blobs = [line.split()[-1] for line in text.splitlines() if line.startswith("blob ")]
    assert blobs[2:4] == ["xavier", "constant"]


# --------------------------------------------------------------------------- Flatten
def test_flatten_plan(cos, tmp_path):
    body = ('layer { name: "c" type: "Convolution" bottom: "x" top: "c" convolution_param { num_output: 2 '
            'kernel_size: 1 } }\n'
            'layer { name: "f" type: "Flatten" bottom: "c" top: "f" }\n'
            'layer { name: "ip" type: "InnerProduct" bottom: "f" top: "y" inner_product_param { num_output: 108 } }\n'
            'layer { name: "ft" type: "Flatten" bottom: "t" top: "tf" flatten_param { axis: -3 end_axis: 3 } }\n'
            'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "y" bottom: "tf" top: "l" }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, body)))
    # the top's gradient is the bottom's; a staged bottom's top gets a gradient buffer of its own
    assert lines[1] == "op 1 Flatten f 2x2x6x6 -> 2x72 data=bottom diff=bottom"
    assert lines[3] == "op 3 Flatten ft 2x3x6x6 -> 2x108 data=bottom staged-bottom no-backward"
    assert lines[4] == "op 4 SigmoidCrossEntropyLoss loss 2x108 -> scalar target=5 loss_weight=1"


def test_flatten_top_is_never_in_place_for_a_later_layer(cos, tmp_path):
    body = ('layer { name: "c" type: "Convolution" bottom: "x" top: "c" convolution_param { num_output: 2 '
            'kernel_size: 1 } }\n'
            'layer { name: "f" type: "Flatten" bottom: "c" top: "f" }\n'
            'layer { name: "r" type: "ReLU" bottom: "f" top: "f" }\n'
            'layer { name: "ip" type: "InnerProduct" bottom: "f" top: "y" inner_product_param { num_output: 108 } }\n'
            'layer { name: "ft" type: "Flatten" bottom: "t" top: "tf" }\n' + SCE.replace('"t"', '"tf"') % "y")
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, body)))
    assert lines[2] == "op 2 ReLU r 2x72 -> 2x72"


# --------------------------------------------------------------------------- SigmoidCrossEntropyLoss
def test_sigmoid_cross_entropy_plan(cos, tmp_path):
    body = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
            'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "y" bottom: "t" top: "l" loss_weight: 2.5 }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, body)))
    assert lines[1] == "op 1 SigmoidCrossEntropyLoss loss 2x3x6x6 -> scalar target=1 loss_weight=2.5"
    # the target is label-like: not counted as its blob's reader, so another layer may read it without a Split
    body = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n' + SCE % "y" +
            '\nlayer { name: "ip" type: "InnerProduct" bottom: "t" top: "z" inner_product_param { num_output: 2 } }')
    (tmp_path / "b").mkdir()
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path / "b", body)))
    assert lines[1].endswith("target=1 loss_weight=1") and lines[2].endswith("staged-bottom no-backward")


# --------------------------------------------------------------------------- the two rules
def test_a_zero_weight_loss_does_no_train_work(cos, tmp_path):
    body = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
            'layer { name: "sp" type: "Split" bottom: "y" top: "y0" top: "y1" }\n' + SCE % "y0" +
            '\nlayer { name: "s" type: "Sigmoid" bottom: "y1" top: "s" }\n'
            'layer { name: "l2" type: "EuclideanLoss" bottom: "s" bottom: "t" top: "l2" loss_weight: 0 }')
    text = cos.native_producer_plan(_write(tmp_path, body))
    lines = _op_lines(text)
    assert [line.split()[3] for line in lines] == ["sc", "sp", "sp", "loss", "s"]  # no l2
    assert lines[2] == "op 2 Split sp 2x3x6x6 -> 2x3x6x6 top=1 data=bottom unread"
    assert lines[4] == "op 4 Sigmoid s 2x3x6x6 -> 2x3x6x6 no-backward"
    # the zero-weight loss's bottoms are not read: `s` may feed another layer, and the second loss is not refused
    body2 = body + ('\nlayer { name: "ip" type: "InnerProduct" bottom: "s" top: "z" inner_product_param { '
                    'num_output: 2 } }')
    (tmp_path / "b").mkdir()
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path / "b", body2)))
    assert lines[-1].endswith(" no-backward") and lines[-1].split()[3] == "ip"


def test_ops_off_the_loss_run_no_backward(cos, tmp_path):
    """An op whose top only a label reads, or nothing reads, runs no backward; nor does an op that feeds only such an
    op.  Split and Slice ops keep their marks."""
    body = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
            'layer { name: "sp" type: "Split" bottom: "y" top: "a" top: "b" top: "u" }\n'
            'layer { name: "c" type: "Convolution" bottom: "b" top: "c" convolution_param { num_output: 3 '
            'kernel_size: 1 } }\n'
            'layer { name: "bn" type: "BatchNorm" bottom: "c" top: "bn" }\n'
            'layer { name: "sl" type: "Slice" bottom: "bn" top: "s0" top: "s1" slice_param { axis: 1 '
            'slice_point: 1 } }\n'
            'layer { name: "g" type: "Sigmoid" bottom: "s1" top: "g" }\n'
            'layer { name: "cat" type: "Concat" bottom: "s0" bottom: "g" top: "tt" }\n'
            'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "a" bottom: "tt" top: "l" }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path, body)))
    names = [line.split()[3] for line in lines]
    assert names == ["sc", "sp", "sp", "sp", "c", "bn", "sl", "sl", "g", "cat", "cat", "loss"]
    assert lines[1].endswith("top=0 data=bottom")
    assert lines[2].endswith("top=1 data=bottom unread") and lines[3].endswith("top=2 data=bottom unread")
    for i in (4, 5, 8, 9, 10):  # conv, BatchNorm (its forward still runs), Sigmoid, both Concat parts
        assert lines[i].endswith(" no-backward"), lines[i]
    for i in (0, 6, 7, 11):
        assert "no-backward" not in lines[i], lines[i]


def test_existing_loss_rules_hold(cos, tmp_path):
    two = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
           'layer { name: "sp" type: "Split" bottom: "y" top: "y0" top: "y1" }\n' + SCE % "y0" +
           '\nlayer { name: "l2" type: "EuclideanLoss" bottom: "y1" bottom: "t" top: "l2" loss_weight: 0.5 }')
    with pytest.raises(cos.CosError, match=r"^layer 'l2' \(EuclideanLoss\): a second loss layer is not supported"):
        cos.native_producer_plan(_write(tmp_path, two))
    (tmp_path / "b").mkdir()
    only_zero = ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n' +
                 (SCE % "y").replace('top: "l" }', 'top: "l" loss_weight: 0 }'))
    with pytest.raises(cos.CosError, match=r"^the net has no SoftmaxWithLoss, ContrastiveLoss, EuclideanLoss or "
                                           r"SigmoidCrossEntropyLoss layer with a non-zero loss_weight"):
        cos.native_producer_plan(_write(tmp_path / "b", only_zero))
    (tmp_path / "c").mkdir()
    with pytest.raises(cos.CosError, match=r"^layer 'loss' \(SigmoidCrossEntropyLoss\): loss_param"):
        cos.native_producer_plan(_write(tmp_path / "c", ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n' +
                                                         (SCE % "y").replace('top: "l" }', 'top: "l" loss_param { '
                                                                             'normalize: false } }'))))


# --------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("body,shape,match", [
    (_deconv("dc", "x", "y", 3, "kernel_size: 2 group: 3") + SCE % "y", (2, 3, 6, 6),
     r"^layer 'dc' \(Deconvolution\): group 3 > 1 is not supported"),
    (_deconv("dc", "x", "y", 3, "kernel_size: 2 dilation: 2") + SCE % "y", (2, 3, 6, 6),
     r"^layer 'dc' \(Deconvolution\): dilation other than 1 is not supported"),
    (_deconv("dc", "x", "y", 3, 'kernel_size: 4 stride: 2 weight_filler { type: "bilinear" }') + SCE % "y",
     (2, 3, 6, 6),
     r"^layer 'dc' \(Deconvolution\): filler type 'bilinear' is not supported"),
    (_deconv("dc", "x", "y", 3, 'kernel_size: 1 weight_filler { type: "xavier" sparse: 2 }') + SCE % "y", (2, 3, 6, 6),
     r"^layer 'dc' \(Deconvolution\): Sparsity not supported by this Filler\."),
    ('layer { name: "f" type: "Flatten" bottom: "x" top: "f" flatten_param { axis: 2 } }\n' + SCE % "f", (2, 3, 6, 6),
     r"^layer 'f' \(Flatten\): flatten_param axis 2, end_axis -1 is not supported"),
    ('layer { name: "f" type: "Flatten" bottom: "x" top: "f" flatten_param { end_axis: 2 } }\n' + SCE % "f",
     (2, 3, 6, 6), r"^layer 'f' \(Flatten\): flatten_param axis 1, end_axis 2 is not supported"),
    ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
     'layer { name: "f" type: "Flatten" bottom: "y" top: "y" }\n' + SCE % "y", (2, 3, 6, 6),
     r"^layer 'f' \(Flatten\): Flatten Layer does not allow in-place computation\. \(native producer\)$"),
    ('layer { name: "sl" type: "Slice" bottom: "x" top: "a" top: "b" slice_param { axis: 0 } }\n'
     'layer { name: "sc" type: "Scale" bottom: "a" top: "y" }\n' + SCE % "y" +
     '\nlayer { name: "s" type: "Silence" bottom: "b" }', (2, 3, 6, 6),
     r"^layer 'loss' \(SigmoidCrossEntropyLoss\): The data and label should have the same number\. "
     r"\(native producer\)$"),
    ('layer { name: "sl" type: "Slice" bottom: "x" top: "a" top: "b" slice_param { axis: 1 slice_point: 1 } }\n'
     'layer { name: "sc" type: "Scale" bottom: "a" top: "y" }\n' + SCE % "y" +
     '\nlayer { name: "s" type: "Silence" bottom: "b" }', (2, 3, 6, 6),
     r"^layer 'loss' \(SigmoidCrossEntropyLoss\): SIGMOID_CROSS_ENTROPY_LOSS layer inputs must have the same "
     r"count\. \(native producer\)$"),
    ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" }\n'
     'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "y" top: "l" }', (2, 3, 6, 6),
     r"^layer 'loss' \(SigmoidCrossEntropyLoss\): 2 bottom\(s\) and one top"),
])
def test_refusals_name_the_layer(cos, tmp_path, body, shape, match):
    with pytest.raises(cos.CosError, match=match):
        cos.native_producer_plan(_write(tmp_path, body, shape))


# --------------------------------------------------------------------------- the fixtures
def _fc_count():
    """The FC autoencoder from its widths alone: in * out + out per InnerProduct."""
    widths = [784, 1000, 500, 250, 30, 250, 500, 1000, 784]
    return sum(a * b + b for a, b in zip(widths, widths[1:])), 2 * (len(widths) - 1)


def test_the_fixture_layouts(cos):
    from caffeonspark_b200 import nets
    total, blobs = _fc_count()
    assert (total, blobs) == (2837314, 16) == (nets.AUTOENCODER_PARAM_COUNT, 16)
    d = cos.parse_solver(FC_SOLVER)
    assert d.param_count == total and len(d.counts) == blobs
    assert [p.numel() for p in nets.autoencoder_module().parameters()] == list(d.counts)
    assert d.lr_mult == [1.0] * 16 and d.decay_mult == [1.0, 0.0] * 8
    assert d.base_lr == pytest.approx(0.01) and d.momentum == pytest.approx(0.9) and d.lr_policy == "step"
    conv = 16 * 1 * 9 + 16, 32 * 16 * 9 + 32, 32 * 16 * 16 + 16, 16 * 1 * 16  # deconv [32, 16, 4, 4], [16, 1, 4, 4]
    assert conv == (160, 4640, 8208, 256) and sum(conv) == 13264 == nets.CONV_AUTOENCODER_PARAM_COUNT
    d = cos.parse_solver(CONV_SOLVER)
    assert d.param_count == 13264 and len(d.counts) == 7
    assert [tuple(p.shape) for p in nets.conv_autoencoder_module().parameters()] == [
        (16, 1, 3, 3), (16,), (32, 16, 3, 3), (32,), (32, 16, 4, 4), (16,), (16, 1, 4, 4)]
    assert [p.numel() for p in nets.conv_autoencoder_module().parameters()] == list(d.counts)


FC_OPS = [
    "op 0 Split data_split 100x1x28x28 -> 100x1x28x28 top=0 data=bottom unread staged-bottom",
    "op 1 Split data_split 100x1x28x28 -> 100x1x28x28 top=1 data=bottom staged-bottom",
    "op 2 Flatten flatdata 100x1x28x28 -> 100x784 data=bottom diff=bottom no-bottom-grad no-backward",
    "op 3 InnerProduct encode1 100x1x28x28 -> 100x1000 w=0:784000 b=784000:1000 no-bottom-grad",
    "op 4 Sigmoid encode1neuron 100x1000 -> 100x1000",
    "op 5 InnerProduct encode2 100x1000 -> 100x500 w=785000:500000 b=1285000:500",
    "op 6 Sigmoid encode2neuron 100x500 -> 100x500",
    "op 7 InnerProduct encode3 100x500 -> 100x250 w=1285500:125000 b=1410500:250",
    "op 8 Sigmoid encode3neuron 100x250 -> 100x250",
    "op 9 InnerProduct encode4 100x250 -> 100x30 w=1410750:7500 b=1418250:30",
    "op 10 InnerProduct decode4 100x30 -> 100x250 w=1418280:7500 b=1425780:250",
    "op 11 Sigmoid decode4neuron 100x250 -> 100x250",
    "op 12 InnerProduct decode3 100x250 -> 100x500 w=1426030:125000 b=1551030:500",
    "op 13 Sigmoid decode3neuron 100x500 -> 100x500",
    "op 14 InnerProduct decode2 100x500 -> 100x1000 w=1551530:500000 b=2051530:1000",
    "op 15 Sigmoid decode2neuron 100x1000 -> 100x1000",
    "op 16 InnerProduct decode1 100x1000 -> 100x784 w=2052530:784000 b=2836530:784",
    "op 17 Split decode1_split 100x784 -> 100x784 top=0 data=bottom",
    "op 18 Split decode1_split 100x784 -> 100x784 top=1 data=bottom unread",
    "op 19 SigmoidCrossEntropyLoss loss 100x784 -> scalar target=3 loss_weight=1",
    "op 20 Sigmoid decode1neuron 100x784 -> 100x784 no-backward",
]
CONV_OPS = [
    "op 0 Convolution conv1 100x1x28x28 -> 100x16x14x14 k3x3 s2x2 p1x1 w=0:144 b=144:16 staged-bottom",
    "op 1 ReLU relu1 100x16x14x14 -> 100x16x14x14 in-place",
    "op 2 Convolution conv2 100x16x14x14 -> 100x32x7x7 k3x3 s2x2 p1x1 w=160:4608 b=4768:32",
    "op 3 ReLU relu2 100x32x7x7 -> 100x32x7x7 in-place",
    "op 4 Deconvolution deconv1 100x32x7x7 -> 100x16x14x14 k4x4 s2x2 p1x1 w=4800:8192 b=12992:16",
    "op 5 ReLU relu3 100x16x14x14 -> 100x16x14x14 in-place",
    "op 6 Deconvolution deconv2 100x16x14x14 -> 100x1x28x28 k4x4 s2x2 p1x1 w=13008:256",
    "op 7 SigmoidCrossEntropyLoss loss 100x1x28x28 -> scalar target=0 loss_weight=1",
]


@pytest.mark.parametrize("solver,ops,total", [(FC_SOLVER, FC_OPS, 2837314), (CONV_SOLVER, CONV_OPS, 13264)])
def test_the_fixture_plans(cos, solver, ops, total):
    text = cos.native_producer_plan(solver)
    assert text.startswith("input 0 data 78400\nop 0 ")
    assert _op_lines(text) == ops
    _check_layout(cos, text, solver, total)
    blobs = [line.split()[-1] for line in text.splitlines() if line.startswith("blob ")]
    if solver == FC_SOLVER:
        assert blobs == ["gaussian", "constant"] * 8
    else:
        assert blobs == ["xavier", "constant"] * 3 + ["xavier"]
    assert sum(op.startswith("SigmoidCrossEntropyLoss loss 100x") for op in _ops(text)) == 1
