"""CPU tests of Caffe's Tile layer on the built-in engine (DESIGN.md section 14): tile_ref.py's fp32 restatement of
Forward_cpu and Backward_cpu against its float64 one, on ordinary and special values; three plausible mistakes (a sum
started from +0, the tiles added in reverse, outer and inner swapped) that these checks catch; the parser's shape rule
for axes 0 to 3 and -1 on 1-D to 5-D bottoms, every refusal with its wording, the plan line and the plan's refusals;
and the SE-ResNet-20 and U-Net scSE fixtures' layouts and plans."""
import os
import re

import numpy as np
import pytest

import tile_ref as R
from conftest import ROOT
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
EUCLID = 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n'
F32 = np.float32


def _tile(param="axis: 1 tiles: 3", bottom="x", top="y"):
    return f'layer {{ name: "tl" type: "Tile" bottom: "{bottom}" top: "{top}" tile_param {{ {param} }} }}\n'


# --------------------------------------------------------------------------- the references
REF_CASES = [  # (bottom, axis, tiles): both sides of the staged threshold (inner 32), odd sizes, 1-D to 5-D
    ((4, 6, 1, 1), 2, 7), ((4, 6, 7, 1), 3, 7), ((3, 1, 8, 8), 1, 5), ((2, 3, 5), 0, 4), ((5,), 0, 33),
    ((2, 3, 4, 5, 2), -1, 3), ((3, 31), 1, 40), ((2, 33), 1, 3), ((7, 3), 0, 1), ((1, 1, 1, 1), 3, 64),
]


@pytest.mark.parametrize("shape,axis,tiles", REF_CASES)
def test_fp32_is_float64_rounded(shape, axis, tiles):
    rng = np.random.RandomState(sum(shape) + tiles)
    x = rng.randn(*shape).astype(F32)
    y = R.forward32(x, axis, tiles)
    assert y.shape == R.infer(shape, axis, tiles)
    assert np.array_equal(y, R.forward64(x, axis, tiles))  # a copy
    dy = R.specials(rng, y.shape, count=0)
    dx, dx64 = R.backward32(dy, shape, axis, tiles), R.backward64(dy, shape, axis, tiles)
    # a sequential sum of `tiles` values: (tiles - 1) u of the sum of |dy| per element at most
    bound = (tiles - 1) * 2.0 ** -24 * R.backward64(np.abs(dy), shape, axis, tiles)
    assert (np.abs(dx - dx64) <= bound).all()
    if tiles == 1:
        assert np.array_equal(dx, dy.reshape(shape))


@pytest.mark.parametrize("shape,axis,tiles", REF_CASES)
def test_special_values(shape, axis, tiles):
    rng = np.random.RandomState(len(shape) * tiles)
    x = R.specials(rng, shape)
    outer, inner = R.dims(shape, axis)
    want = np.repeat(x.reshape(outer, 1, inner), tiles, axis=1)
    assert np.array_equal(R.forward32(x, axis, tiles).view(np.uint32).ravel(), want.view(np.uint32).ravel())  # NaNs too
    top = R.infer(shape, axis, tiles)
    dy = R.negative_zero_column(R.specials(rng, top), shape, axis, tiles)
    dx = R.backward32(dy, shape, axis, tiles)
    assert dx.reshape(-1)[-1].view(np.uint32) == 0x80000000, "a column of -0 stays -0"
    dx64 = R.backward64(dy, shape, axis, tiles)
    assert np.isnan(dx[np.isnan(dx64)]).all()
    finite = np.isfinite(dx64) & np.isfinite(dx)
    assert (np.abs(dx[finite] - dx64[finite]) <= tiles * 2.0 ** -24 * np.abs(dx64[finite]).max() + 1e-44).all()


# --------------------------------------------------------------------------- mistakes the checks catch
def _grad_case(seed=5):
    shape, axis, tiles = (3, 4, 1, 1), 2, 9
    rng = np.random.RandomState(seed)
    dy = R.negative_zero_column(R.specials(rng, R.infer(shape, axis, tiles), count=0), shape, axis, tiles)
    return dy, shape, axis, tiles


def test_a_sum_started_from_plus_zero_is_caught(monkeypatch):
    dy, shape, axis, tiles = _grad_case()
    want = R.canonical_bits(R.backward32(dy, shape, axis, tiles)).ravel()
    monkeypatch.setattr(R, "start", lambda col: F32(0) + col)
    got = R.canonical_bits(R.backward32(dy, shape, axis, tiles)).ravel()
    assert got[-1] == 0 and want[-1] == 0x80000000 and not np.array_equal(got, want)


def test_tiles_added_in_reverse_are_caught(monkeypatch):
    dy, shape, axis, tiles = _grad_case()
    want = R.canonical_bits(R.backward32(dy, shape, axis, tiles))
    monkeypatch.setattr(R, "tile_order", lambda t: (t - 1, range(t - 2, -1, -1)))
    assert not np.array_equal(R.canonical_bits(R.backward32(dy, shape, axis, tiles)), want)


def test_outer_and_inner_swapped_are_caught(monkeypatch):
    x = np.arange(24, dtype=F32).reshape(2, 3, 4)
    want = R.forward32(x, 1, 2)
    dy, shape, axis, tiles = _grad_case()
    want_dx = R.backward32(dy, shape, axis, tiles)
    dims = R.dims
    monkeypatch.setattr(R, "dims", lambda s, a: dims(s, a)[::-1])
    assert not np.array_equal(R.forward32(x, 1, 2), want)
    assert not np.array_equal(R.canonical_bits(R.backward32(dy, shape, axis, tiles)), R.canonical_bits(want_dx))


# --------------------------------------------------------------------------- the parser and the plan
SHAPES = [(7,), (3, 5), (2, 3, 4), (2, 3, 4, 5), (2, 1, 3, 2, 2)]


@pytest.mark.parametrize("tiles", [1, 3])
@pytest.mark.parametrize("axis", [0, 1, 2, 3, -1])
@pytest.mark.parametrize("bottom", SHAPES)
def test_shape_inference_and_plan_line(cos, tmp_path, bottom, axis, tiles):
    if not -len(bottom) <= axis < len(bottom):
        with pytest.raises(cos.CosError, match=re.escape(f"axis {axis} out of range for {len(bottom)}-D Blob")):
            cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": (1,)}, _tile(f"axis: {axis} tiles: {tiles}")
                                            + EUCLID))
        return
    top = R.infer(bottom, axis, tiles)
    a = axis % len(bottom)
    assert top == tuple(d * tiles if k == a else d for k, d in enumerate(bottom))
    if tiles == 1:
        assert top == bottom
    text = cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": top}, _tile(f"axis: {axis} tiles: {tiles}") +
                                           EUCLID))
    shape = lambda s: "x".join(map(str, s))  # noqa: E731
    inner = int(np.prod(bottom[a:]))
    assert f"op 0 Tile tl {shape(bottom)} -> {shape(top)} axis={a} tiles={tiles} inner={inner} staged-bottom\n" in text
    assert "params 0 blobs 0" in text  # Tile owns no blob


def test_axis_defaults_to_one(cos, tmp_path):
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 4), "t": (2, 12, 4)}, _tile("tiles: 4") + EUCLID))
    assert "op 0 Tile tl 2x3x4 -> 2x12x4 axis=1 tiles=4 inner=12 staged-bottom\n" in text


PARSER_REFUSALS = [  # (bottom, tile_param or None, axis, tiles, message)
    ((2, 3, 4, 5), "axis: 1", 1, None, "Number of tiles must be specified"),
    ((2, 3, 4, 5), None, 1, None, "Number of tiles must be specified"),
    ((2, 3, 4, 5), "axis: 2 tiles: 0", 2, 0, "Number of tiles must be positive."),
    ((2, 3, 4, 5), "tiles: -3", 1, -3, "Number of tiles must be positive."),
    ((2, 3, 4, 5), "axis: 4 tiles: 2", 4, 2, "axis 4 out of range for 4-D Blob"),
    ((2, 3, 4, 5), "axis: -5 tiles: 2", -5, 2, "axis -5 out of range for 4-D Blob"),
    ((6,), "tiles: 2", 1, 2, "axis 1 out of range for 1-D Blob"),
]


@pytest.mark.parametrize("bottom,param,axis,tiles,want", PARSER_REFUSALS)
def test_parser_refusals(cos, tmp_path, bottom, param, axis, tiles, want):
    layer = _tile(param) if param is not None else 'layer { name: "tl" type: "Tile" bottom: "x" top: "y" }\n'
    with pytest.raises(cos.CosError, match="^layer 'tl' \\(Tile\\): " + re.escape(want) + "$"):
        cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": (1,)}, layer + EUCLID))
    with pytest.raises(ValueError, match="^" + re.escape(want) + "$"):
        R.infer(bottom, axis, tiles)


def test_in_place_is_refused(cos, tmp_path):
    body = ('layer { name: "sc" type: "Scale" bottom: "in0" top: "x" scale_param { axis: 0 } }\n' +
            _tile("axis: 1 tiles: 1", top="x") + EUCLID.replace('"y"', '"x"'))
    with pytest.raises(cos.CosError, match="^layer 'tl' \\(Tile\\): Tile Layer does not allow in-place computation. "
                                           "\\(native producer\\)$"):
        cos.native_producer_plan(_write(tmp_path, {"in0": (2, 3), "t": (2, 3)}, body))


@pytest.mark.parametrize("bottom,tiles,refused", [((2,), 2 ** 30, True), ((1,), 2 ** 31 - 1, False),
                                                  ((3, 5), 143165577, True)])
def test_a_top_past_32_bit_indices_is_refused(cos, tmp_path, bottom, tiles, refused):
    # the kernels index the top in 32 bits: a top of 2^31 or more elements is refused by the plan (which allocates
    # nothing) rather than failing at its first forward
    top = R.infer(bottom, 0, tiles)
    path = _write(tmp_path, {"x": bottom, "t": top}, _tile(f"axis: 0 tiles: {tiles}") + EUCLID)
    if refused:
        with pytest.raises(cos.CosError, match=f"^layer 'tl' \\(Tile\\): a top of {int(np.prod(top))} elements is more "
                                               r"than the 2147483647 the Tile kernels index in 32 bits"):
            cos.native_producer_plan(path)
    else:
        assert f"op 0 Tile tl 1 -> {tiles} axis=0 tiles={tiles} inner=1" in cos.native_producer_plan(path)


# --------------------------------------------------------------------------- the fixtures
def _se_block_lines(first, name, c, hw, w_off):
    """the plan lines of one SE block of the SE-ResNet-20 fixture (batch 100), its ops numbered from `first`"""
    r = c // 4
    m = f"100x{c}x{hw}x{hw}"
    lines = [
        f"Split {name}_se_split {m} -> {m} top=0 data=bottom",
        f"Split {name}_se_split {m} -> {m} top=1 data=bottom",
        f"Pooling(AVE) {name}_se_squeeze {m} -> 100x{c}x1x1 k{hw}x{hw} s1x1 p0x0",
        f"InnerProduct {name}_se_fc1 100x{c}x1x1 -> 100x{r} w={w_off}:{c * r} b={w_off + c * r}:{r}",
        f"ReLU {name}_se_relu 100x{r} -> 100x{r} in-place",
        f"InnerProduct {name}_se_fc2 100x{r} -> 100x{c} w={w_off + c * r + r}:{c * r} b={w_off + 2 * c * r + r}:{c}",
        f"Sigmoid {name}_se_sigmoid 100x{c} -> 100x{c} in-place",
        f"Reshape {name}_se_reshape 100x{c} -> 100x{c}x1x1 data=bottom diff=bottom",
        f"Tile {name}_se_tile_h 100x{c}x1x1 -> 100x{c}x{hw}x1 axis=2 tiles={hw} inner=1",
        f"Tile {name}_se_tile_w 100x{c}x{hw}x1 -> {m} axis=3 tiles={hw} inner=1",
        f"Eltwise(PROD) {name}_se {m} -> {m} bottoms=2 stable_prod_grad",
    ]
    return [f"op {first + k} {line}" for k, line in enumerate(lines)]


def test_se_resnet20_layout_and_plan(cos):
    import torch
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "cifar10_se_resnet20_solver.prototxt")
    text = cos.native_producer_plan(solver)
    ops = [ln for ln in text.splitlines() if ln.startswith("op ")]
    _check_layout(cos, text, solver, nets.SE_RESNET20_PARAM_COUNT)
    d = cos.parse_solver(solver)
    base = cos.parse_solver(os.path.join(CONFIGS, "cifar10_resnet20_solver.prototxt"))
    assert nets.SE_RESNET20_PARAM_COUNT == 282547 == base.param_count + 8484 and len(d.counts) == len(base.counts) + 36
    assert [p.numel() for p in nets.se_resnet20_module().parameters()] == d.counts
    # every block's SE ops come right after its branch2b's Scale and before its Eltwise SUM
    blocks = [(f"res{s}{b}", c, hw) for s, c, hw in (("2", 16, 32), ("3", 32, 16), ("4", 64, 8)) for b in "abc"]
    for name, c, hw in blocks:
        k = next(i for i, ln in enumerate(ops) if f" scale_{name}_branch2b " in ln)
        w_off = int(re.search(r" b=(\d+):(\d+)", ops[k]).group(1)) + c
        assert ops[k + 1:k + 12] == _se_block_lines(k + 1, name, c, hw, w_off), name
        assert next(i for i, ln in enumerate(ops) if f" Eltwise(SUM) {name} " in ln) > k + 11
    assert sum(" Tile " in ln for ln in ops) == 18
    base_ops = [ln for ln in cos.native_producer_plan(os.path.join(CONFIGS, "cifar10_resnet20_solver.prototxt"))
                .splitlines() if ln.startswith("op ")]
    assert len(ops) == len(base_ops) + 11 * len(blocks)
    m = nets.se_resnet20_module().eval()
    assert m(torch.zeros(2, 3, 32, 32)).shape == (2, 10)


UNET_SCSE_OPS = """\
op 26 ReLU relu4b 8x32x28x28 -> 8x32x28x28 in-place
op 27 Split scse4_split 8x32x28x28 -> 8x32x28x28 top=0 data=bottom
op 28 Split scse4_split 8x32x28x28 -> 8x32x28x28 top=1 data=bottom
op 29 Split scse4_split 8x32x28x28 -> 8x32x28x28 top=2 data=bottom
op 30 Split scse4_split 8x32x28x28 -> 8x32x28x28 top=3 data=bottom
op 31 Pooling(AVE) scse4_c_squeeze 8x32x28x28 -> 8x32x1x1 k28x28 s1x1 p0x0
op 32 InnerProduct scse4_c_fc1 8x32x1x1 -> 8x8 w=107728:256 b=107984:8
op 33 ReLU scse4_c_relu 8x8 -> 8x8 in-place
op 34 InnerProduct scse4_c_fc2 8x8 -> 8x32 w=107992:256 b=108248:32
op 35 Sigmoid scse4_c_sigmoid 8x32 -> 8x32 in-place
op 36 Reshape scse4_c_reshape 8x32 -> 8x32x1x1 data=bottom diff=bottom
op 37 Tile scse4_c_tile_h 8x32x1x1 -> 8x32x28x1 axis=2 tiles=28 inner=1
op 38 Tile scse4_c_tile_w 8x32x28x1 -> 8x32x28x28 axis=3 tiles=28 inner=1
op 39 Eltwise(PROD) scse4_c 8x32x28x28 -> 8x32x28x28 bottoms=2 stable_prod_grad
op 40 Convolution scse4_s_conv 8x32x28x28 -> 8x1x28x28 k1x1 s1x1 p0x0 w=108280:32 b=108312:1
op 41 Sigmoid scse4_s_sigmoid 8x1x28x28 -> 8x1x28x28 in-place
op 42 Tile scse4_s_tile 8x1x28x28 -> 8x32x28x28 axis=1 tiles=32 inner=784
op 43 Eltwise(PROD) scse4_s 8x32x28x28 -> 8x32x28x28 bottoms=2 stable_prod_grad
op 44 Eltwise(MAX) scse4 8x32x28x28 -> 8x32x28x28 bottoms=2
op 45 Deconvolution upconv1 8x32x28x28 -> 8x16x56x56 k2x2 s2x2 p0x0 w=108313:2048 b=110361:16
op 46 ReLU relu_up1 8x16x56x56 -> 8x16x56x56 in-place
op 47 Crop crop1 8x16x88x88 -> 8x16x56x56 axis=2 offsets=16,16 ref=47
op 48 Concat concat1 8x16x56x56 -> 8x32x56x56 axis=1 begin=0
op 49 Concat concat1 8x16x56x56 -> 8x32x56x56 axis=1 begin=16
op 50 Convolution conv5a 8x32x56x56 -> 8x16x54x54 k3x3 s1x1 p0x0 w=110377:4608 b=114985:16
op 51 ReLU relu5a 8x16x54x54 -> 8x16x54x54 in-place
op 52 Convolution conv5b 8x16x54x54 -> 8x16x52x52 k3x3 s1x1 p0x0 w=115001:2304 b=117305:16
op 53 ReLU relu5b 8x16x52x52 -> 8x16x52x52 in-place
op 54 Split scse5_split 8x16x52x52 -> 8x16x52x52 top=0 data=bottom
op 55 Split scse5_split 8x16x52x52 -> 8x16x52x52 top=1 data=bottom
op 56 Split scse5_split 8x16x52x52 -> 8x16x52x52 top=2 data=bottom
op 57 Split scse5_split 8x16x52x52 -> 8x16x52x52 top=3 data=bottom
op 58 Pooling(AVE) scse5_c_squeeze 8x16x52x52 -> 8x16x1x1 k52x52 s1x1 p0x0
op 59 InnerProduct scse5_c_fc1 8x16x1x1 -> 8x4 w=117321:64 b=117385:4
op 60 ReLU scse5_c_relu 8x4 -> 8x4 in-place
op 61 InnerProduct scse5_c_fc2 8x4 -> 8x16 w=117389:64 b=117453:16
op 62 Sigmoid scse5_c_sigmoid 8x16 -> 8x16 in-place
op 63 Reshape scse5_c_reshape 8x16 -> 8x16x1x1 data=bottom diff=bottom
op 64 Tile scse5_c_tile_h 8x16x1x1 -> 8x16x52x1 axis=2 tiles=52 inner=1
op 65 Tile scse5_c_tile_w 8x16x52x1 -> 8x16x52x52 axis=3 tiles=52 inner=1
op 66 Eltwise(PROD) scse5_c 8x16x52x52 -> 8x16x52x52 bottoms=2 stable_prod_grad
op 67 Convolution scse5_s_conv 8x16x52x52 -> 8x1x52x52 k1x1 s1x1 p0x0 w=117469:16 b=117485:1
op 68 Sigmoid scse5_s_sigmoid 8x1x52x52 -> 8x1x52x52 in-place
op 69 Tile scse5_s_tile 8x1x52x52 -> 8x16x52x52 axis=1 tiles=16 inner=2704
op 70 Eltwise(PROD) scse5_s 8x16x52x52 -> 8x16x52x52 bottoms=2 stable_prod_grad
op 71 Eltwise(MAX) scse5 8x16x52x52 -> 8x16x52x52 bottoms=2
op 72 Convolution score 8x16x52x52 -> 8x2x52x52 k1x1 s1x1 p0x0 w=117486:32 b=117518:2
op 73 Crop crop_label 8x1x92x92 -> 8x1x52x52 axis=2 offsets=20,20 ref=72 staged-bottom no-backward
op 74 SoftmaxWithLoss loss 8x2x52x52 -> scalar axis=1 label=73 loss_weight=1
"""


def test_unet_scse_layout_and_plan(cos):
    import torch
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "unet_scse_solver.prototxt")
    text = cos.native_producer_plan(solver)
    ops = [ln + "\n" for ln in text.splitlines() if ln.startswith("op ")]
    assert "".join(ops[26:]) == UNET_SCSE_OPS
    # up to relu4b the plan is the U-Net's, op for op
    unet = [ln + "\n" for ln in cos.native_producer_plan(os.path.join(CONFIGS, "unet_solver.prototxt")).splitlines()
            if ln.startswith("op ")]
    assert ops[:26] == unet[:26]
    _check_layout(cos, text, solver, nets.UNET_SCSE_PARAM_COUNT)
    d = cos.parse_solver(solver)
    assert nets.UNET_SCSE_PARAM_COUNT == 117520 == nets.UNET_PARAM_COUNT + 750 and len(d.counts) == 26 + 12
    m = nets.unet_scse_module()
    assert [p.numel() for p in m.parameters()] == d.counts
    assert m(torch.zeros(2, 1, 92, 92)).shape == (2, 2, 52, 52)
