"""CPU tests of Caffe's Crop layer on the built-in engine (DESIGN.md section 14): crop_ref.py's slice restatement
against its index-map restatement, bit for bit on special values; the parser's shape rule for every axis and offset
form, and each of its refusals; the plan's shape-only reference (no Split with a Concat, a gradient wanted through its
other readers), its staged-bottom and no-backward marks; and the U-Net fixture's layout and plan, line for line."""
import os
import re

import numpy as np
import pytest

import crop_ref as R
from conftest import ROOT
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
SCALE = 'layer { name: "s" type: "Scale" bottom: "x" top: "a" scale_param { axis: 0 } }\n'
EUCLID = 'layer {{ name: "loss" type: "EuclideanLoss" bottom: "{}" bottom: "t" top: "l" }}\n'


def _crop(bottom="a", ref="r", top="y", param="", name="c", extra=""):
    return (f'layer {{ name: "{name}" type: "Crop" bottom: "{bottom}" bottom: "{ref}" top: "{top}" {extra}'
            f'crop_param {{ {param} }} }}\n')


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# --------------------------------------------------------------------------- the references
REF_CASES = [  # (bottom shape, top shape, offsets)
    ((7,), (3,), (2,)), ((5, 9), (5, 4), (0, 5)), ((4, 6, 9), (2, 3, 9), (1, 3, 0)),
    ((2, 3, 8, 10), (2, 3, 5, 3), (0, 0, 3, 7)),
    ((3, 4, 5, 6, 7), (1, 2, 3, 4, 5), (2, 1, 2, 1, 2)), ((2, 2, 4, 4), (2, 2, 4, 4), (0, 0, 0, 0)),
]


@pytest.mark.parametrize("bottom,top,offsets", REF_CASES)
def test_slices_equal_the_index_map_bit_for_bit(bottom, top, offsets):
    rng = np.random.RandomState(int(np.prod(bottom)))
    x, dy = R.specials(rng, bottom), R.specials(rng, top)
    y = R.forward(x, top, offsets)
    assert y.shape == top
    assert np.array_equal(_bits(y), _bits(R.forward_index_map(x, top, offsets)))
    dx = R.backward(dy, bottom, offsets)
    assert np.array_equal(_bits(dx), _bits(R.backward_index_map(dy, bottom, offsets)))
    outside = np.ones(bottom, bool)
    outside[R.window(offsets, top)] = False
    assert (_bits(dx)[outside] == 0).all()  # +0, never -0


def test_the_index_map_catches_an_offset_on_the_wrong_axis():
    x = np.arange(60, dtype=np.float32).reshape(3, 4, 5)
    assert not np.array_equal(R.forward(x, (3, 2, 2), (0, 1, 2)), R.forward_index_map(x, (3, 2, 2), (0, 2, 1)))


# --------------------------------------------------------------------------- the parser's shape rule
SHAPE_CASES = [  # (bottom, reference, crop_param)
    ((6, 5), (3, 2), "axis: 0"),
    ((6, 5), (9, 2), "axis: 1 offset: 3"),
    ((6, 5), (9, 4), "axis: -1"),
    ((4, 7, 9), (2, 3, 4), "axis: 1 offset: 2 offset: 5"),
    ((4, 7, 9), (1, 1, 9), "axis: 2"),
    ((4, 7, 9), (4, 5, 1), "axis: 0 offset: 0 offset: 1 offset: 8"),
    ((2, 3, 10, 12), (9, 9, 4, 5), ""),
    ((2, 3, 10, 12), (9, 9, 4, 5), "offset: 3"),
    ((2, 3, 10, 12), (9, 9, 4, 5), "offset: 6 offset: 7"),
    ((2, 3, 10, 12), (9, 2, 4, 5), "axis: 1 offset: 1"),
    ((2, 3, 10, 12), (9, 9, 9, 5), "axis: 3 offset: 7"),
    ((2, 3, 10, 12), (9, 9, 9, 5), "axis: -1 offset: 4"),
    ((5, 3, 10, 12), (2, 3, 4, 5, 6), "axis: 0 offset: 3 offset: 0 offset: 6 offset: 7"),
    ((2, 3, 4, 6, 8), (2, 3, 2, 3, 4), "axis: 2 offset: 1 offset: 2 offset: 3"),
    ((2, 3, 4, 6, 8), (1, 1, 1, 1, 1), "axis: -2 offset: 5"),
]


def _param(param):
    axis = re.search(r"axis: (-?\d+)", param)
    return int(axis.group(1)) if axis else 2, tuple(int(v) for v in re.findall(r"offset: (\d+)", param))


@pytest.mark.parametrize("bottom,ref,param", SHAPE_CASES)
def test_shape_inference_and_plan_line(cos, tmp_path, bottom, ref, param):
    axis, top, offs = R.infer(bottom, ref, *_param(param))
    body = SCALE + _crop(param=param) + EUCLID.format("y")
    text = cos.native_producer_plan(_write(tmp_path, {"x": bottom, "r": ref, "t": top}, body))
    shape = lambda s: "x".join(map(str, s))  # noqa: E731
    want = f"op 1 Crop c {shape(bottom)} -> {shape(top)} axis={axis} offsets={','.join(map(str, offs[axis:]))} ref=1\n"
    assert want in text
    assert f"params {bottom[0]} blobs 1" in text  # the Scale's: the Crop owns no blob


REFUSALS = [  # (bottom, reference, layer text after the bottoms, message)
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" top: "z"', "Crop Layer produces 1 top blob(s) as output."),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "a"', "Crop Layer does not allow in-place computation."),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { axis: 4 }', "axis 4 out of range for 4-D Blob"),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { axis: -5 }', "axis -5 out of range for 4-D Blob"),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { offset: 1 offset: 2 offset: 3 }',
     "number of offset values specified must be equal to the number of dimensions following axis."),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { axis: 1 offset: 1 offset: 2 }',
     "number of offset values specified must be equal to the number of dimensions following axis."),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { offset: -1 }',
     "crop_param offset -1: Expected integer, got: -"),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { offset: 5 }',
     "the crop for dimension 2 is out-of-bounds with size 4 and offset 5"),
    ((2, 3, 8, 8), (2, 3, 4, 9), 'top: "y"', "the crop for dimension 3 is out-of-bounds with size 9 and offset 0"),
    ((2, 3, 8, 8), (2, 3, 4, 4), 'top: "y" crop_param { offset: 0 offset: 6 }',
     "the crop for dimension 3 is out-of-bounds with size 4 and offset 6"),
    ((2, 3, 8, 8), (2, 9, 4, 4), 'top: "y" crop_param { axis: 1 }',
     "the crop for dimension 1 is out-of-bounds with size 9 and offset 0"),
    ((2, 3, 8, 8), (2, 3, 4), 'top: "y"', "axis 3 out of range for 3-D Blob"),
    ((2, 3, 8, 8), (2, 3), 'top: "y" crop_param { axis: 1 }', "axis 2 out of range for 2-D Blob"),
]


@pytest.mark.parametrize("bottom,ref,rest,want", REFUSALS)
def test_refusals(cos, tmp_path, bottom, ref, rest, want):
    body = SCALE + f'layer {{ name: "c" type: "Crop" bottom: "a" bottom: "r" {rest} }}\n' + EUCLID.format("y")
    with pytest.raises(cos.CosError, match="^layer 'c' \\(Crop\\): " + re.escape(want) + "$"):
        cos.native_producer_plan(_write(tmp_path, {"x": bottom, "r": ref, "t": (1,)}, body))
    if "crop_param" in rest and "offset: -1" not in rest or rest == 'top: "y"':  # a CHECK of the shapes: restated
        with pytest.raises(ValueError, match="^" + re.escape(want) + "$"):
            R.infer(bottom, ref, *_param(rest))


@pytest.mark.parametrize("bottoms", [1, 3])
def test_two_bottoms_are_required(cos, tmp_path, bottoms):
    names = " ".join(f'bottom: "{b}"' for b in ["a", "r", "x"][:bottoms])
    body = SCALE + f'layer {{ name: "c" type: "Crop" {names} top: "y" }}\n' + EUCLID.format("y")
    with pytest.raises(cos.CosError, match="^layer 'c' \\(Crop\\): Crop Layer takes 2 bottom blob\\(s\\) as input\\.$"):
        cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 3, 4, 4), "t": (1,)}, body))


def test_extra_param_entries_are_ignored(cos, tmp_path):
    body = SCALE + _crop(extra="param { lr_mult: 0 } ") + EUCLID.format("y")
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 3, 4, 4), "t": (2, 3, 4, 4)}, body))
    assert "op 1 Crop c 2x3x8x8 -> 2x3x4x4 axis=2 offsets=0,0 ref=1\n" in text and "params 2 blobs 1" in text


# --------------------------------------------------------------------------- the plan
def test_a_reference_shared_with_a_concat_needs_no_split(cos, tmp_path):
    """U-Net's pattern: the up-convolution's output is both the Concat's bottom and the Crop's reference"""
    body = (SCALE + 'layer { name: "u" type: "Scale" bottom: "r" top: "up" scale_param { axis: 0 } }\n' +
            _crop(ref="up", param="offset: 2") +
            'layer { name: "cat" type: "Concat" bottom: "y" bottom: "up" top: "cat" }\n' + EUCLID.format("cat"))
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 5, 4, 4), "t": (2, 8, 4, 4)}, body))
    assert "op 2 Crop c 2x3x8x8 -> 2x3x4x4 axis=2 offsets=2,2 ref=4\n" in text
    assert "op 3 Concat cat 2x3x4x4 -> 2x8x4x4 axis=1 begin=0\n" in text
    assert "op 4 Concat cat 2x5x4x4 -> 2x8x4x4 axis=1 begin=3\n" in text


def test_a_reference_that_wants_a_gradient_is_accepted(cos, tmp_path):
    """The reference's gradient comes from its other reader alone: Crop adds nothing to it"""
    body = (SCALE + 'layer { name: "u" type: "Scale" bottom: "r" top: "up" scale_param { axis: 0 } }\n' +
            _crop(ref="up") + 'layer { name: "e" type: "Eltwise" bottom: "y" bottom: "up" top: "sum" }\n' +
            EUCLID.format("sum"))
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 3, 4, 4), "t": (2, 3, 4, 4)}, body))
    assert "op 2 Crop c 2x3x8x8 -> 2x3x4x4 axis=2 offsets=0,0 ref=4\n" in text
    assert "op 3 Eltwise(SUM) e 2x3x4x4 -> 2x3x4x4 bottoms=2 coeff=1,1\n" in text


def test_a_crop_of_a_staged_input(cos, tmp_path):
    body = _crop(bottom="x", param="offset: 1") + EUCLID.format("y")
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 3, 6, 6), "t": (2, 3, 6, 6)}, body))
    assert "op 0 Crop c 2x3x8x8 -> 2x3x6x6 axis=2 offsets=1,1 ref=1 staged-bottom\n" in text


def test_a_label_crop_runs_its_forward_alone(cos, tmp_path):
    body = (SCALE + _crop(bottom="lab", ref="a", top="lc", param="offset: 3", name="cl") +
            'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "a" bottom: "lc" top: "l" }\n')
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 4, 4), "lab": (2, 1, 10, 10)}, body))
    assert "op 1 Crop cl 2x1x10x10 -> 2x1x4x4 axis=2 offsets=3,3 ref=2 staged-bottom no-backward\n" in text
    assert "op 2 SoftmaxWithLoss loss 2x3x4x4 -> scalar axis=1 label=3 loss_weight=1\n" in text


def test_a_crop_off_the_loss_runs_no_backward(cos, tmp_path):
    body = (SCALE + 'layer { name: "sp" type: "Split" bottom: "a" top: "a0" top: "a1" }\n' +
            _crop(bottom="a1", ref="r", top="y") + 'layer { name: "z" type: "Silence" bottom: "y" }\n' +
            EUCLID.format("a0"))
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 8, 8), "r": (2, 3, 4, 4), "t": (2, 3, 8, 8)}, body))
    assert "op 3 Crop c 2x3x8x8 -> 2x3x4x4 axis=2 offsets=0,0 ref=1 no-backward\n" in text


# --------------------------------------------------------------------------- the U-Net fixture
UNET_OPS = """\
op 0 Convolution conv1a 8x1x92x92 -> 8x16x90x90 k3x3 s1x1 p0x0 w=0:144 b=144:16 staged-bottom
op 1 ReLU relu1a 8x16x90x90 -> 8x16x90x90 in-place
op 2 Convolution conv1b 8x16x90x90 -> 8x16x88x88 k3x3 s1x1 p0x0 w=160:2304 b=2464:16
op 3 ReLU relu1b 8x16x88x88 -> 8x16x88x88 in-place
op 4 Split split1 8x16x88x88 -> 8x16x88x88 top=0 data=bottom
op 5 Split split1 8x16x88x88 -> 8x16x88x88 top=1 data=bottom
op 6 Pooling(MAX) pool1 8x16x88x88 -> 8x16x44x44 k2x2 s2x2 p0x0
op 7 Convolution conv2a 8x16x44x44 -> 8x32x42x42 k3x3 s1x1 p0x0 w=2480:4608 b=7088:32
op 8 ReLU relu2a 8x32x42x42 -> 8x32x42x42 in-place
op 9 Convolution conv2b 8x32x42x42 -> 8x32x40x40 k3x3 s1x1 p0x0 w=7120:9216 b=16336:32
op 10 ReLU relu2b 8x32x40x40 -> 8x32x40x40 in-place
op 11 Split split2 8x32x40x40 -> 8x32x40x40 top=0 data=bottom
op 12 Split split2 8x32x40x40 -> 8x32x40x40 top=1 data=bottom
op 13 Pooling(MAX) pool2 8x32x40x40 -> 8x32x20x20 k2x2 s2x2 p0x0
op 14 Convolution conv3a 8x32x20x20 -> 8x64x18x18 k3x3 s1x1 p0x0 w=16368:18432 b=34800:64
op 15 ReLU relu3a 8x64x18x18 -> 8x64x18x18 in-place
op 16 Convolution conv3b 8x64x18x18 -> 8x64x16x16 k3x3 s1x1 p0x0 w=34864:36864 b=71728:64
op 17 ReLU relu3b 8x64x16x16 -> 8x64x16x16 in-place
op 18 Deconvolution upconv2 8x64x16x16 -> 8x32x32x32 k2x2 s2x2 p0x0 w=71792:8192 b=79984:32
op 19 ReLU relu_up2 8x32x32x32 -> 8x32x32x32 in-place
op 20 Crop crop2 8x32x40x40 -> 8x32x32x32 axis=2 offsets=4,4 ref=21
op 21 Concat concat2 8x32x32x32 -> 8x64x32x32 axis=1 begin=0
op 22 Concat concat2 8x32x32x32 -> 8x64x32x32 axis=1 begin=32
op 23 Convolution conv4a 8x64x32x32 -> 8x32x30x30 k3x3 s1x1 p0x0 w=80016:18432 b=98448:32
op 24 ReLU relu4a 8x32x30x30 -> 8x32x30x30 in-place
op 25 Convolution conv4b 8x32x30x30 -> 8x32x28x28 k3x3 s1x1 p0x0 w=98480:9216 b=107696:32
op 26 ReLU relu4b 8x32x28x28 -> 8x32x28x28 in-place
op 27 Deconvolution upconv1 8x32x28x28 -> 8x16x56x56 k2x2 s2x2 p0x0 w=107728:2048 b=109776:16
op 28 ReLU relu_up1 8x16x56x56 -> 8x16x56x56 in-place
op 29 Crop crop1 8x16x88x88 -> 8x16x56x56 axis=2 offsets=16,16 ref=29
op 30 Concat concat1 8x16x56x56 -> 8x32x56x56 axis=1 begin=0
op 31 Concat concat1 8x16x56x56 -> 8x32x56x56 axis=1 begin=16
op 32 Convolution conv5a 8x32x56x56 -> 8x16x54x54 k3x3 s1x1 p0x0 w=109792:4608 b=114400:16
op 33 ReLU relu5a 8x16x54x54 -> 8x16x54x54 in-place
op 34 Convolution conv5b 8x16x54x54 -> 8x16x52x52 k3x3 s1x1 p0x0 w=114416:2304 b=116720:16
op 35 ReLU relu5b 8x16x52x52 -> 8x16x52x52 in-place
op 36 Convolution score 8x16x52x52 -> 8x2x52x52 k1x1 s1x1 p0x0 w=116736:32 b=116768:2
op 37 Crop crop_label 8x1x92x92 -> 8x1x52x52 axis=2 offsets=20,20 ref=36 staged-bottom no-backward
op 38 SoftmaxWithLoss loss 8x2x52x52 -> scalar axis=1 label=37 loss_weight=1
"""


def test_unet_layout_and_plan(cos):
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "unet_solver.prototxt")
    text = cos.native_producer_plan(solver)
    assert "input 0 data 67712\ninput 1 label 67712\n" in text  # the label has the image's height and width
    assert "".join(ln + "\n" for ln in text.splitlines() if ln.startswith("op ")) == UNET_OPS
    _check_layout(cos, text, solver, nets.UNET_PARAM_COUNT)
    d = cos.parse_solver(solver)
    assert nets.UNET_PARAM_COUNT == 116770 and len(d.counts) == 26
    m = nets.unet_module()
    assert [p.numel() for p in m.parameters()] == d.counts
    shapes = [tuple(int(v) for v in ln.split()[3].split("x")) for ln in text.splitlines() if ln.startswith("blob ")]
    assert [tuple(p.shape) for p in m.parameters()] == shapes
    # 21,632 pixel rows of SoftmaxWithLoss, and the mirror's scores on as many
    import torch
    assert m(torch.zeros(8, 1, 92, 92)).shape == (8, 2, 52, 52)
    assert m.crop_label(torch.zeros(8, 1, 92, 92)).numel() == 8 * 52 * 52 == 21632
