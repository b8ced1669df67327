"""CPU tests of Caffe's N-D Convolution and Deconvolution on the built-in engine (DESIGN.md section 14): the layout
parser's shapes for 3-D and 1-D layers (isotropic and per-axis fields, stride 2 over odd sizes, pad on one axis only)
and every refusal with Caffe's wording; the plan lines and layouts of the V-Net and C3D clip fixtures; every older
fixture's plan text byte for byte as the engine printed it before N-D convolutions (tests/golden/plan_digests.json,
refusals included); the PyTorch mirrors' parameter order; and gemm3d_ref.py's fp32 restatement of the 3-D gathers
against float64, with mutations it catches."""
import glob
import hashlib
import json
import os
import re

import numpy as np
import pytest

import conv3d_ref as C3
import gemm3d_ref as G3
import gemm_ref as G
import producer_ops_ref as R
from conftest import ROOT
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
EUCLID = 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n'


def _conv(param, kind="Convolution", bottom="x"):
    return f'layer {{ name: "c" type: "{kind}" bottom: "{bottom}" top: "y" convolution_param {{ {param} }} }}\n'


# --------------------------------------------------------------------------- the parser's shapes and plan lines
SHAPE_CASES = [  # (kind, bottom, param, weight, top, plan's k/s/p)
    ("Convolution", (2, 3, 9, 9, 9), "num_output: 4 kernel_size: 3", (4, 3, 3, 3, 3), (2, 4, 7, 7, 7),
     "k3x3x3 s1x1x1 p0x0x0"),
    ("Convolution", (2, 3, 8, 9, 10), "num_output: 2 kernel_size: 1 kernel_size: 3 kernel_size: 5 stride: 1 stride: 2 "
     "stride: 3 pad: 0 pad: 1 pad: 2", (2, 3, 1, 3, 5), (2, 2, 8, 5, 4), "k1x3x5 s1x2x3 p0x1x2"),
    ("Convolution", (1, 2, 7, 9, 11), "num_output: 3 kernel_size: 3 stride: 2", (3, 2, 3, 3, 3), (1, 3, 3, 4, 5),
     "k3x3x3 s2x2x2 p0x0x0"),
    ("Convolution", (1, 2, 5, 5, 5), "num_output: 3 kernel_size: 3 pad: 1 pad: 0 pad: 0", (3, 2, 3, 3, 3),
     (1, 3, 5, 3, 3), "k3x3x3 s1x1x1 p1x0x0"),
    ("Convolution", (1, 2, 5, 6, 7), "num_output: 3 kernel_size: 2 pad: 0 pad: 0 pad: 1 bias_term: false",
     (3, 2, 2, 2, 2), (1, 3, 4, 5, 8), "k2x2x2 s1x1x1 p0x0x1"),
    ("Deconvolution", (2, 4, 3, 4, 5), "num_output: 2 kernel_size: 2 stride: 2", (4, 2, 2, 2, 2), (2, 2, 6, 8, 10),
     "k2x2x2 s2x2x2 p0x0x0"),
    ("Deconvolution", (1, 3, 3, 3, 3), "num_output: 2 kernel_size: 1 kernel_size: 3 kernel_size: 4 stride: 1 stride: 2 "
     "stride: 2 pad: 0 pad: 1 pad: 1", (3, 2, 1, 3, 4), (1, 2, 3, 5, 6), "k1x3x4 s1x2x2 p0x1x1"),
    ("Convolution", (2, 3, 11), "num_output: 4 kernel_size: 3 stride: 2 pad: 1", (4, 3, 3), (2, 4, 6), "k3 s2 p1"),
    ("Convolution", (2, 3, 10), "num_output: 4 kernel_size: 4 axis: -2", (4, 3, 4), (2, 4, 7), "k4 s1 p0"),
    ("Deconvolution", (2, 3, 5), "num_output: 2 kernel_size: 4 stride: 2 pad: 1", (3, 2, 4), (2, 2, 10), "k4 s2 p1"),
]


def _x(shape):
    return "x".join(str(v) for v in shape)


@pytest.mark.parametrize("kind,bottom,param,weight,top,ksp", SHAPE_CASES)
def test_shapes_and_plan_line(cos, tmp_path, kind, bottom, param, weight, top, ksp):
    text = cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": top}, _conv(param, kind) + EUCLID))
    blobs = [line.split()[3] for line in text.splitlines() if line.startswith("blob ")]
    bias = "bias_term: false" not in param
    assert blobs == [_x(weight)] + ([str(top[1])] if bias else [])
    wc = int(np.prod(weight))
    want = f"op 0 {kind} c {_x(bottom)} -> {_x(top)} {ksp} w=0:{wc}" + (f" b={wc}:{top[1]}" if bias else "")
    assert want + " staged-bottom" in text.splitlines()


REFUSALS = [  # (bottom, param, message), a parser refusal unless it ends with "(native producer)"
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_h: 3 kernel_w: 3", "kernel_h & kernel_w can only be used for 2D convolution."),
    ((1, 2, 5), "num_output: 2 kernel_size: 3 stride_w: 2", "stride_h & stride_w can only be used for 2D convolution."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 pad_h: 1", "pad_h & pad_w can only be used for 2D convolution."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 kernel_size: 3",
     "kernel_size must be specified once, or once per spatial dimension (kernel_size specified 2 times; 3 spatial "
     "dims)."),
    ((1, 2, 5, 5, 5), "num_output: 2",
     "kernel_size must be specified once, or once per spatial dimension (kernel_size specified 0 times; 3 spatial "
     "dims)."),
    ((1, 2, 9), "num_output: 2 kernel_size: 3 kernel_size: 3",
     "kernel_size must be specified once, or once per spatial dimension (kernel_size specified 2 times; 1 spatial "
     "dims)."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 stride: 1 stride: 2",
     "stride must be specified once, or once per spatial dimension (stride specified 2 times; 3 spatial dims)."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 pad: 1 pad: 1 pad: 1 pad: 1",
     "pad must be specified once, or once per spatial dimension (pad specified 4 times; 3 spatial dims)."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 dilation: 1 dilation: 1",
     "dilation must be specified once, or once per spatial dimension (dilation specified 2 times; 3 spatial dims)."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 kernel_size: 0 kernel_size: 3", "Filter dimensions must be nonzero."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 stride: 0", "Stride dimensions must be nonzero."),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 axis: 2",
     "convolution_param axis 2 is not supported on a 5-axis bottom (the channel axis must be 1)"),
    ((1, 2, 5), "num_output: 2 kernel_size: 3 axis: 0",
     "convolution_param axis 0 is not supported on a 3-axis bottom (the channel axis must be 1)"),
    ((1, 2, 3, 3, 3, 3), "num_output: 2 kernel_size: 1",
     "a bottom of 6 axes is not supported (at most 3 spatial axes are)"),
    ((1, 3, 5, 5, 5), "num_output: 3 kernel_size: 3 group: 3", "group 3 > 1 is not supported (native producer)"),
    ((1, 2, 5, 5, 5), "num_output: 2 kernel_size: 3 dilation: 2",
     "dilation other than 1 is not supported (native producer)"),
    ((1, 2, 9), "num_output: 2 kernel_size: 3 dilation: 2", "dilation other than 1 is not supported (native producer)"),
    ((1, 2, 5, 5, 5), 'num_output: 2 kernel_size: 3 weight_filler { type: "bilinear" }',
     "filler type 'bilinear' is not supported (constant, uniform, gaussian, xavier, msra are) (native producer)"),
    # the 3-D gathers index in 32 bits: a top of exactly 2^31 elements is refused, one 2^21 below it is not
    ((1, 1, 1024, 1024, 1024), "num_output: 2 kernel_size: 1",
     "a geometry of 2147483648 elements reaches the 2^31 the 3-D convolution kernels index in 32 bits (native "
     "producer)"),
    ((2, 1, 1024, 1024, 1024), "num_output: 1 kernel_size: 1",
     "a geometry of 2147483648 elements reaches the 2^31 the 3-D convolution kernels index in 32 bits (native "
     "producer)"),
]


@pytest.mark.parametrize("bottom,param,want", REFUSALS)
def test_refusals(cos, tmp_path, bottom, param, want):
    with pytest.raises(cos.CosError, match="^layer 'c' \\(Convolution\\): " + re.escape(want) + "$"):
        cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": (1,)}, _conv(param) + EUCLID))


def test_just_below_the_32_bit_limit_plans(cos, tmp_path):
    text = cos.native_producer_plan(_write(tmp_path, {"x": (1, 1, 1024, 1024, 1023), "t": (1, 2, 1024, 1024, 1023)},
                                           _conv("num_output: 2 kernel_size: 1") + EUCLID))
    assert "op 0 Convolution c 1x1x1024x1024x1023 -> 1x2x1024x1024x1023 k1x1x1" in text


def test_deconvolution_refusals_keep_the_2d_wording(cos, tmp_path):
    with pytest.raises(cos.CosError, match=r"^layer 'c' \(Deconvolution\): group 2 > 1 is not supported"):
        cos.native_producer_plan(_write(tmp_path, {"x": (1, 4, 3, 3, 3), "t": (1,)},
                                        _conv("num_output: 2 kernel_size: 2 group: 2", "Deconvolution") + EUCLID))


@pytest.mark.parametrize("body,want", [
    ('layer { name: "c" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 2 kernel_size: 1 } }\n',
     "layer 'c': bad Convolution"),
    ('layer { name: "p" type: "Pooling" bottom: "x5" top: "y" pooling_param { pool: MAX kernel_size: 2 } }\n',
     "layer 'p': bad Pooling"),
])
def test_a_1_axis_convolution_and_a_5_axis_pooling_are_still_refused(cos, tmp_path, body, want):
    with pytest.raises(cos.CosError, match="^" + re.escape(want) + "$"):
        cos.native_producer_plan(_write(tmp_path, {"x": (7,), "x5": (1, 2, 4, 4, 4), "t": (1,)}, body + EUCLID))


# --------------------------------------------------------------------------- the fixtures
VNET_CONVS = [
    "op 1 Convolution conv1a 2x1x32x32x32 -> 2x8x32x32x32 k3x3x3 s1x1x1 p1x1x1 w=0:216 b=216:8 no-bottom-grad",
    "op 5 Convolution conv1b 2x8x32x32x32 -> 2x8x32x32x32 k3x3x3 s1x1x1 p1x1x1 w=232:1728 b=1960:8",
    "op 10 Convolution down1 2x8x32x32x32 -> 2x16x16x16x16 k2x2x2 s2x2x2 p0x0x0 w=1976:1024 b=3000:16",
    "op 14 Convolution conv2 2x16x16x16x16 -> 2x16x16x16x16 k3x3x3 s1x1x1 p1x1x1 w=3032:6912 b=9944:16",
    "op 19 Convolution down2 2x16x16x16x16 -> 2x32x8x8x8 k2x2x2 s2x2x2 p0x0x0 w=9976:4096 b=14072:32",
    "op 23 Convolution conv3 2x32x8x8x8 -> 2x32x8x8x8 k3x3x3 s1x1x1 p1x1x1 w=14136:27648 b=41784:32",
    "op 26 Deconvolution up2 2x32x8x8x8 -> 2x16x16x16x16 k2x2x2 s2x2x2 p0x0x0 w=41848:4096 b=45944:16",
    "op 32 Convolution conv4 2x32x16x16x16 -> 2x16x16x16x16 k3x3x3 s1x1x1 p1x1x1 w=45976:13824 b=59800:16",
    "op 35 Deconvolution up1 2x16x16x16x16 -> 2x8x32x32x32 k2x2x2 s2x2x2 p0x0x0 w=59832:1024 b=60856:8",
    "op 41 Convolution conv5 2x16x32x32x32 -> 2x8x32x32x32 k3x3x3 s1x1x1 p1x1x1 w=60872:3456 b=64328:8",
    "op 44 Convolution score 2x8x32x32x32 -> 2x2x32x32x32 k1x1x1 s1x1x1 p0x0x0 w=64344:16 b=64360:2",
    "op 45 SoftmaxWithLoss loss 2x2x32x32x32 -> scalar axis=1 label=1 loss_weight=1",
]
C3D_OPS = [
    "op 0 Reshape clip 4x24x56x56 -> 4x3x8x56x56 data=bottom staged-bottom",
    "op 1 Convolution conv1 4x3x8x56x56 -> 4x16x8x28x28 k3x3x3 s1x2x2 p1x1x1 w=0:1296 b=1296:16 no-bottom-grad",
    "op 2 ReLU relu1 4x16x8x28x28 -> 4x16x8x28x28 in-place",
    "op 3 Convolution conv2 4x16x8x28x28 -> 4x32x4x14x14 k3x3x3 s2x2x2 p1x1x1 w=1312:13824 b=15136:32",
    "op 4 ReLU relu2 4x32x4x14x14 -> 4x32x4x14x14 in-place",
    "op 5 Convolution conv3 4x32x4x14x14 -> 4x32x4x7x7 k1x3x3 s1x2x2 p0x1x1 w=15168:9216 b=24384:32",
    "op 6 ReLU relu3 4x32x4x7x7 -> 4x32x4x7x7 in-place",
    "op 7 InnerProduct fc4 4x32x4x7x7 -> 4x10 w=24416:62720 b=87136:10",
    "op 8 SoftmaxWithLoss loss 4x10 -> scalar axis=1 label=1 loss_weight=1",
]


def test_vnet3d_layout_and_plan(cos):
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "vnet3d_solver.prototxt")
    text = cos.native_producer_plan(solver)
    lines = text.splitlines()
    assert all(op in lines for op in VNET_CONVS)
    assert sum(line.startswith("op ") for line in lines) == 46
    _check_layout(cos, text, solver, 64362)
    assert nets.VNET3D_PARAM_COUNT == 64362
    assert cos.parse_solver(solver).batch_size == 2
    assert "input 0 data 65536" in lines and "input 1 label 65536" in lines  # one label per voxel


def test_c3d_clip_layout_and_plan(cos):
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "c3d_clip_solver.prototxt")
    text = cos.native_producer_plan(solver)
    assert [line for line in text.splitlines() if line.startswith("op ")] == C3D_OPS
    _check_layout(cos, text, solver, 87146)
    assert nets.C3D_CLIP_PARAM_COUNT == 87146
    blobs = [line.split()[3:] for line in text.splitlines() if line.startswith("blob ")]
    assert blobs[0] == ["16x3x3x3x3", "msra"] and blobs[4] == ["32x32x1x3x3", "msra"] and blobs[6] == ["10x6272", "xavier"]


@pytest.mark.parametrize("name", ["vnet3d", "c3d_clip"])
def test_mirrors_register_parameters_in_layout_order(cos, name):
    from caffeonspark_b200 import nets
    m = nets.vnet3d_module() if name == "vnet3d" else nets.c3d_clip_module()
    text = cos.native_producer_plan(os.path.join(CONFIGS, f"{name}_solver.prototxt"))
    shapes = [line.split()[3] for line in text.splitlines() if line.startswith("blob ")]
    assert ["x".join(str(v) for v in p.shape) for p in m.parameters()] == shapes


def test_every_older_fixture_plans_byte_for_byte_as_before(cos):
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "plan_digests.json")))
    got = {}
    for path in sorted(glob.glob(os.path.join(CONFIGS, "*.prototxt"))):
        name = os.path.basename(path)
        if name not in want:
            assert name.startswith(("vnet3d_", "c3d_clip_")), f"{name}: a fixture without a recorded plan"
            continue
        try:
            text = cos.native_producer_plan(path)
        except cos.CosError as e:
            text = "refused: " + str(e)
        got[name] = hashlib.sha256(text.encode()).hexdigest()
    assert got == want


# --------------------------------------------------------------------------- the restatement against float64
def _within(got, ref, bound, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    assert np.all(err <= bound), f"{what}: {np.max(err - bound):.3e} outside the bound"


HOST_CONV = [c for c in C3.CONV3D_CASES if c[2] * c[3] * c[4] < 10 ** 4]


@pytest.mark.parametrize("case", HOST_CONV, ids=str)
def test_conv3d_restatement_is_within_the_float64_bounds(case):
    x, w, b = C3.inputs(case)
    geo3 = case[6]
    y = G3.conv3d_forward(x, w, b, geo3)
    by, bw, bb, bx = C3.conv3d_bounds(x, w, b, y, geo3)
    _within(y, C3.conv3d64(x, w, b, geo3), by, "y")
    dw, db, dx = C3.conv3d_backward64(x, w, y, geo3)
    _within(G3.conv3d_weight_grad(x, y, geo3), dw, bw, "dW")
    _within(G.bias_grad(y, y.shape[0], y.shape[1], int(np.prod(y.shape[2:]))), db, bb, "db")
    _within(G3.conv3d_data_grad(y, w, None, x.shape, geo3), dx, bx, "dx")


@pytest.mark.parametrize("case", C3.DECONV3D_CASES[:4], ids=str)
def test_deconv3d_restatement_is_within_the_float64_bounds(case):
    x, w, b = C3.inputs(case, deconv=True)
    geo3 = case[6]
    y64 = C3.deconv3d64(x, w, b, geo3)
    y = G3.deconv3d_forward(x, w, b, geo3, y64.shape[2:])
    by, bw, bb, bx = C3.deconv3d_bounds(x, w, b, y, geo3)
    _within(y, y64, by, "y")
    dw, db, dx = C3.deconv3d_backward64(x, w, y, geo3)
    _within(G3.deconv3d_weight_grad(x, y, geo3), dw, bw, "dW")
    _within(G.bias_grad(y, y.shape[0], y.shape[1], int(np.prod(y.shape[2:]))), db, bb, "db")
    _within(G3.deconv3d_data_grad(y, w, geo3), dx, bx, "dx")


def test_the_2d_restatement_is_the_3d_one_with_a_depth_of_one():
    x, w, b = C3.inputs((2, 3, 1, 7, 8, 4, (1, 3, 3, 1, 2, 1, 0, 1, 0), True))
    geo, geo3 = (3, 3, 2, 1, 1, 0), (1, 3, 3, 1, 2, 1, 0, 1, 0)
    y = G.conv_forward(x[:, :, 0], w[:, :, 0], b, geo)
    assert np.array_equal(y.view(np.uint32), G3.conv3d_forward(x, w, b, geo3)[:, :, 0].view(np.uint32))
    assert np.array_equal(G.conv_weight_grad(x[:, :, 0], y, geo).view(np.uint32),
                          G3.conv3d_weight_grad(x, y[:, :, None], geo3)[:, :, 0].view(np.uint32))
    assert np.array_equal(G.conv_data_grad(y, w[:, :, 0], None, x[:, :, 0].shape, geo).view(np.uint32),
                          G3.conv3d_data_grad(y[:, :, None], w, None, x.shape, geo3)[:, :, 0].view(np.uint32))


# --------------------------------------------------------------------------- teeth
def _outside(got, ref, bound):
    """the share of elements outside the float64 bound"""
    return float(np.mean(np.abs(np.asarray(got, np.float64) - ref) > bound))


GATHER_TEETH = [  # (case, mutation): each case's geometry tells the mutated index apart
    ((2, 3, 6, 6, 6, 4, (2, 2, 2, 2, 2, 2, 0, 0, 0), True), "depth_height_swapped"),
    ((2, 3, 5, 6, 7, 4, (3, 3, 3, 1, 1, 1, 1, 1, 1), True), "depth_height_swapped"),
    ((2, 1, 5, 5, 5, 3, (3, 3, 3, 1, 1, 1, 1, 0, 0), False), "pad_rotated"),
    ((2, 3, 4, 9, 9, 5, (1, 3, 3, 1, 2, 2, 0, 1, 1), True), "pad_rotated"),
    ((2, 3, 4, 9, 9, 5, (1, 3, 3, 1, 2, 2, 0, 1, 1), True), "stride_reversed"),
    ((1, 3, 8, 9, 10, 2, (3, 3, 3, 1, 2, 2, 1, 1, 1), True), "stride_reversed"),
]


@pytest.mark.parametrize("case,mutation", GATHER_TEETH, ids=str)
def test_gather_mutations_leave_the_float64_bounds(case, mutation):
    assert case in C3.CONV3D_CASES
    x, w, b = C3.inputs(case)
    geo3 = case[6]
    if mutation == "depth_height_swapped" and x.shape[2] != x.shape[3]:  # swap a cube cut from the case's input
        x = np.ascontiguousarray(x[:, :, :5, :5, :])
    y = G3.conv3d_forward(x, w, b, geo3)
    by, bw, _, _ = C3.conv3d_bounds(x, w, b, y, geo3)
    assert _outside(G3.conv3d_forward(x, w, b, geo3, mutation), C3.conv3d64(x, w, b, geo3), by) > 0.3
    assert _outside(G3.conv3d_weight_grad(x, y, geo3, mutation), C3.conv3d_backward64(x, w, y, geo3)[0], bw) > 0.3


def test_a_reversed_chunk_order_changes_most_weight_gradients():
    case = C3.CONV3D_CASES[-1]  # 256 widened chunks
    assert (R.split_chunk(2 * 48 ** 3), R.splits_of(2 * 48 ** 3)) == (864, 256)
    x, w, b = C3.inputs(case)
    geo3 = case[6]
    y = G3.conv3d_forward(x, w, b, geo3)
    ref, mut = G3.conv3d_weight_grad(x, y, geo3), G3.conv3d_weight_grad(x, y, geo3, "partials_reversed")
    assert float(np.mean(ref.view(np.uint32) != mut.view(np.uint32))) > 0.5


def test_a_volume_is_staged_with_its_trailing_axes_folded():
    """cos_blob holds four dims: train() and forward_backward() fold a 5-D input's axes from the fourth on into its
    width (the producers check the element count), and leave shapes of up to four axes as they were"""
    from caffeonspark_b200.caffenet import _blob_dims
    assert _blob_dims((2, 1, 32, 32, 32)) == (2, 1, 32, 1024)
    assert _blob_dims((4, 3, 8, 56, 56)) == (4, 3, 8, 3136)
    assert [_blob_dims(s) for s in [(), (5,), (5, 3), (5, 3, 7), (5, 3, 7, 2)]] == [
        (1, 1, 1, 1), (5, 1, 1, 1), (5, 3, 1, 1), (5, 3, 7, 1), (5, 3, 7, 2)]
