"""Host-only checks of the built-in producer's net plan (DESIGN.md section 14): the ops and shapes it derives from the
reference's prototxts, learnable offsets equal to the layout parser's, refusals that name the layer, and the new entry
points' argument checks."""
import os
import re

import pytest

from conftest import ROOT
from test_batch_norm_host import _memory_data_copy

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")

LENET_OPS = ["Convolution conv1 64x1x28x28 -> 64x20x24x24", "Pooling(MAX) pool1 64x20x24x24 -> 64x20x12x12",
             "Convolution conv2 64x20x12x12 -> 64x50x8x8", "Pooling(MAX) pool2 64x50x8x8 -> 64x50x4x4",
             "InnerProduct ip1 64x50x4x4 -> 64x500", "ReLU relu1 64x500 -> 64x500", "InnerProduct ip2 64x500 -> 64x10",
             "SoftmaxWithLoss loss 64x10 -> scalar"]
QUICK_OPS = ["ConvBiasReLUMaxPool conv1+pool1+relu1 100x3x32x32 -> 100x32x16x16",
             "Convolution conv2 100x32x16x16 -> 100x32x16x16", "ReLU relu2 100x32x16x16 -> 100x32x16x16",
             "Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8", "Convolution conv3 100x32x8x8 -> 100x64x8x8",
             "ReLU relu3 100x64x8x8 -> 100x64x8x8", "Pooling(AVE) pool3 100x64x8x8 -> 100x64x4x4",
             "InnerProduct ip1 100x64x4x4 -> 100x64", "InnerProduct ip2 100x64 -> 100x10",
             "SoftmaxWithLoss loss 100x10 -> scalar"]
BN_OPS = ["Convolution conv1 100x3x32x32 -> 100x32x32x32", "Pooling(MAX) pool1 100x32x32x32 -> 100x32x16x16",
          "BatchNorm bn1 100x32x16x16 -> 100x32x16x16", "Sigmoid Sigmoid1 100x32x16x16 -> 100x32x16x16",
          "Convolution conv2 100x32x16x16 -> 100x32x16x16", "BatchNorm bn2 100x32x16x16 -> 100x32x16x16",
          "Sigmoid Sigmoid2 100x32x16x16 -> 100x32x16x16", "Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8",
          "Convolution conv3 100x32x8x8 -> 100x64x8x8", "BatchNorm bn3 100x64x8x8 -> 100x64x8x8",
          "Sigmoid Sigmoid3 100x64x8x8 -> 100x64x8x8", "Pooling(AVE) pool3 100x64x8x8 -> 100x64x4x4",
          "InnerProduct ip1 100x64x4x4 -> 100x10", "SoftmaxWithLoss loss 100x10 -> scalar"]


def _ops(text):
    """'<kind> <name> <in> -> <out>' of every op line."""
    return [" ".join(line.split()[2:7]) for line in text.splitlines() if line.startswith("op ")]


def _check_layout(cos, text, solver, total):
    d = cos.parse_solver(solver)
    blobs = [tuple(int(v) for v in re.match(r"blob \d+ (\d+):(\d+) ", line).groups())
             for line in text.splitlines() if line.startswith("blob ")]
    offs = [sum(d.counts[:k]) for k in range(len(d.counts))]
    assert [b[0] for b in blobs] == offs and [b[1] for b in blobs] == d.counts
    assert f"params {total} blobs {len(d.counts)}" in text and d.param_count == total


@pytest.mark.parametrize("solver,ops,total", [
    ("lenet_memory_solver.prototxt", LENET_OPS, 431080),
    ("lenet_cos_solver.prototxt", LENET_OPS, 431080),
    ("lenet_dataframe_solver.prototxt", LENET_OPS, 431080),
    ("cifar10_quick_solver.prototxt", QUICK_OPS, 145578)])
def test_plan_of_reference_configs(cos, solver, ops, total):
    path = os.path.join(CONFIGS, solver)
    text = cos.native_producer_plan(path)
    assert _ops(text) == ops
    _check_layout(cos, text, path, total)
    assert "in-place" in text  # ReLU with top == bottom shares its bottom's memory


def test_plan_of_the_reference_batch_norm_example(cos, tmp_path):
    solver = _memory_data_copy(tmp_path)
    text = cos.native_producer_plan(solver)
    assert _ops(text) == BN_OPS
    _check_layout(cos, text, solver, 89709)


@pytest.mark.parametrize("name,ops,total", [("lenet", LENET_OPS, 431080), ("cifar10_quick", QUICK_OPS, 145578),
                                            ("cifar10_full_bn", BN_OPS, 89709)])
def test_plan_of_generated_prototxts(cos, tmp_path, name, ops, total):
    from caffeonspark_b200 import nets
    solver = nets.write_prototxts(name, str(tmp_path))
    text = cos.native_producer_plan(solver)
    assert _ops(text) == ops
    _check_layout(cos, text, solver, total)
    # a net prototxt gives the same plan as the solver that names it
    assert cos.native_producer_plan(os.path.join(str(tmp_path), f"{name}_net.prototxt")) == text


def test_plan_lists_fillers_and_inputs(cos):
    text = cos.native_producer_plan(os.path.join(CONFIGS, "cifar10_quick_solver.prototxt"))
    assert "input 0 data 307200" in text and "input 1 label 100" in text
    assert "blob 0 0:2400 32x3x5x5 gaussian" in text and "blob 1 2400:32 32 constant" in text


def _net(tmp_path, body):
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "data" type: "MemoryData" top: "data" top: "label" memory_data_param '
                 '{ batch_size: 2 channels: 3 height: 8 width: 8 } }\n' + body +
                 '\nlayer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')
    return str(p)


IP = 'layer { name: "ip" type: "InnerProduct" bottom: "%s" top: "ip" inner_product_param { num_output: 4 } }'


@pytest.mark.parametrize("body,match", [
    ('layer { name: "drop" type: "Dropout" bottom: "data" top: "data" }' + IP % "data",
     r"layer 'drop' \(Dropout\): layer type not supported"),
    ('layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param { num_output: 4 kernel_size: 3 '
     'group: 1 weight_filler { type: "bilinear" } } }' + IP % "c", r"layer 'c' \(Convolution\): filler type 'bilinear'"),
    ('layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param { num_output: 3 kernel_size: 3 '
     'group: 3 } }' + IP % "c", r"layer 'c' \(Convolution\): group 3 > 1"),
    ('layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param { num_output: 3 kernel_size: 3 '
     'dilation: 2 } }' + IP % "c", r"layer 'c' \(Convolution\): dilation"),
    ('layer { name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param { num_output: 4 '
     'transpose: true } }', r"layer 'ip' \(InnerProduct\): transpose"),
    ('layer { name: "p" type: "Pooling" bottom: "data" top: "p" pooling_param { pool: STOCHASTIC kernel_size: 2 } }'
     + IP % "p", r"layer 'p' \(Pooling\): pool method STOCHASTIC"),
    ('layer { name: "r" type: "ReLU" bottom: "data" top: "r" }' + IP % "data",
     r"layer 'ip' \(InnerProduct\): bottom 'data' already feeds layer 'r'"),
])
def test_refusals_name_the_layer(cos, tmp_path, body, match):
    with pytest.raises(cos.CosError, match=match):
        cos.native_producer_plan(_net(tmp_path, body))


def test_loss_param_is_refused(cos, tmp_path):
    p = _net(tmp_path, IP % "data")
    with open(p) as f:
        text = f.read().replace('top: "loss" }', 'top: "loss" loss_param { ignore_label: 3 } }')
    with open(p, "w") as f:
        f.write(text)
    with pytest.raises(cos.CosError, match=r"layer 'loss' \(SoftmaxWithLoss\): loss_param"):
        cos.native_producer_plan(p)


def test_caffenet_and_lrcn_are_refused(cos):
    for f in ("bvlc_reference_solver.prototxt", os.path.join("jni_test", "caffenet_solver.prototxt")):
        with pytest.raises(cos.CosError, match=r"layer 'norm1' \(LRN\): layer type not supported"):
            cos.native_producer_plan(os.path.join(CONFIGS, f))
    with pytest.raises(cos.CosError, match="clip_gradients"):  # the layout parser refuses LRCN already
        cos.native_producer_plan(os.path.join(CONFIGS, "lrcn_solver.prototxt"))


def test_new_entry_points_survive_null_and_garbage(cos, tmp_path):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert L.cos_net_use_native_producer(None, None, 1) == 0 and b"NULL" in L.cos_last_error()
    assert L.cos_net_forward_backward(None, 0, None, 0, None, None) == 0
    assert L.cos_native_producer_plan(None, None, 0) == -1
    assert L.cos_native_producer_plan(b"/nonexistent.prototxt", None, 0) == -1
    assert b"cannot read" in L.cos_last_error()
    junk = tmp_path / "junk.prototxt"
    junk.write_bytes(b"layer { name: \"x\" type: {{{ \x00\xff")
    assert L.cos_native_producer_plan(str(junk).encode(), None, 0) == -1
    path = os.path.join(CONFIGS, "lenet_memory_solver.prototxt").encode()
    n = L.cos_native_producer_plan(path, None, 0)
    assert n > 0
    import ctypes
    small = ctypes.create_string_buffer(8)
    assert L.cos_native_producer_plan(path, small, 8) == n and small.value == b""  # too small: length only


def test_staged_inputs_are_never_written(cos, tmp_path):
    # top == bottom on a staged input: the ReLU's top gets its own storage, and no data gradient flows into the input
    text = cos.native_producer_plan(_net(tmp_path, 'layer { name: "r" type: "ReLU" bottom: "data" top: "data" }'
                                                   + IP % "data"))
    relu = next(line for line in text.splitlines() if " ReLU r " in line)
    assert "in-place" not in relu and "staged-bottom" in relu
    # scores straight from a data layer: accepted, the loss's bottom gradient has a buffer of its own
    p = tmp_path / "scores.prototxt"
    p.write_text('name: "s" layer { name: "data" type: "Input" top: "scores" top: "label" input_param { '
                 'shape { dim: 4 dim: 5 } shape { dim: 4 } } }\n'
                 'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "scores" bottom: "label" top: "loss" }\n')
    text = cos.native_producer_plan(str(p))
    assert _ops(text) == ["SoftmaxWithLoss loss 4x5 -> scalar"] and "staged-bottom" in text
