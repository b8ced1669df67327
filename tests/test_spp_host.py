"""CPU tests of Caffe's SPP layer on the built-in engine (DESIGN.md section 14): spp_ref.py's fp32 restatement of
Caffe's expansion against its index-map restatement, bit for bit on special values, and both against float64; four
plausible mistakes that these checks catch; the geometry every accepted level has, for every map side from 1 to 399;
the parser's shape rule on Caffe's own SPP test geometries, the one-level 4-D top, every refusal with its wording, the
plan line; and the SPP CIFAR-10-quick fixture's layout and plan, line for line."""
import os
import re

import numpy as np
import pytest

import spp_ref as R
from conftest import ROOT
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
EUCLID = 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n'
F32 = np.float32


def _spp(param="pyramid_height: 3", bottom="x", top="y"):
    return f'layer {{ name: "s" type: "SPP" bottom: "{bottom}" top: "{top}" spp_param {{ {param} }} }}\n'


# --------------------------------------------------------------------------- the references
REF_CASES = [  # (bottom shape, pyramid height)
    ((2, 3, 9, 8), 3), ((1, 2, 6, 6), 3), ((2, 2, 7, 7), 3), ((1, 3, 5, 11), 2), ((2, 2, 13, 13), 3),
    ((1, 1, 4, 4), 1), ((1, 2, 16, 16), 4), ((3, 1, 3, 9), 2),
]


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("shape,h", REF_CASES)
def test_expansion_equals_the_index_map_bit_for_bit(shape, h, pool):
    rng = np.random.RandomState(sum(shape) + h)
    x = R.specials(rng, shape)
    y, arg = R.expansion32(x, h, pool)
    assert y.shape == R.infer(shape, h)
    dy = R.specials(rng, y.shape, ties=False)
    dx = R.expansion32_backward(dy, arg, shape, h, pool)
    y2, arg2, dx2 = R.index_map32(x, dy, h, pool)
    assert np.array_equal(R.canonical_bits(y), R.canonical_bits(y2))
    assert pool == "AVE" or np.array_equal(arg, arg2)
    assert np.array_equal(R.canonical_bits(dx), R.canonical_bits(dx2))
    assert not (np.ascontiguousarray(dx).view(np.uint32) == 0x80000000).any(), "-0 becomes +0, as in Caffe"
    if pool == "MAX" and shape[0] * shape[1] > 1:  # the last plane has no value > -FLT_MAX: -FLT_MAX, argmax -1
        offs = R.level_offsets(shape[1], h)
        for lv in range(h):
            part = slice(offs[lv], offs[lv + 1])
            assert (arg.reshape(shape[0], -1)[-1, part].reshape(shape[1], -1)[-1] == -1).all()
            assert (y.reshape(shape[0], -1)[-1, part].reshape(shape[1], -1)[-1] == -R.FLT_MAX).all()


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("shape,h", REF_CASES)
def test_fp32_is_float64_rounded(shape, h, pool):
    rng = np.random.RandomState(sum(shape))
    x = rng.randn(*shape).astype(F32)
    y, arg = R.expansion32(x, h, pool)
    y64 = R.forward64(x, h, pool).reshape(y.shape)
    dy = rng.randn(*y.shape).astype(F32)
    dx = R.expansion32_backward(dy, arg, shape, h, pool)
    dx64 = R.backward64(dy.reshape(shape[0], -1), None if arg is None else arg.reshape(shape[0], -1), shape, h, pool)
    u = 2.0 ** -24
    if pool == "MAX":
        assert np.array_equal(y, y64)
    else:  # a sequential sum of k values: (k + 1) u of the sum of |x|, one u more for the division
        k = max(R.level(shape[2], shape[3], lv)[1] * R.level(shape[2], shape[3], lv)[2] for lv in range(h))
        assert np.abs(y - y64).max() <= (k + 2) * u * np.abs(x).max()
    assert np.abs(dx - dx64).max() <= (h + 1) * u * np.abs(dx64).max() + 1e-30


# --------------------------------------------------------------------------- mistakes the checks catch
def _agrees(x, h, pool, ref):
    try:
        y, _ = R.expansion32(x, h, pool)
        return np.array_equal(R.canonical_bits(y), R.canonical_bits(ref))
    except (ValueError, IndexError):
        return False


def test_pad_rounded_down_is_caught(monkeypatch):
    x = R.specials(np.random.RandomState(1), (2, 2, 7, 7))  # level 2: kernel 2, remainder 1, pad (1 + 1) / 2 = 1
    ref = R.index_map32(x, np.zeros((2, 2 * 21), F32), 3, "MAX")[0]
    level = R.level
    monkeypatch.setattr(R, "level", lambda h, w, lv: level(h, w, lv)[:3] + ((level(h, w, lv)[1] * 2 ** lv - h) // 2,
                                                                             (level(h, w, lv)[2] * 2 ** lv - w) // 2))
    assert not _agrees(x, 3, "MAX", ref)


def test_level_offset_is_caught(monkeypatch):
    x = R.specials(np.random.RandomState(2), (2, 3, 9, 8))
    y, arg = R.expansion32(x, 3, "MAX")
    dy = np.arange(y.size, dtype=F32).reshape(y.shape)
    want = R.expansion32_backward(dy, arg, x.shape, 3, "MAX")
    monkeypatch.setattr(R, "level_offsets", lambda c, h: [c * 4 ** lv for lv in range(h)] + [c * (4 ** h - 1) // 3])
    try:
        got = R.expansion32_backward(dy, arg, x.shape, 3, "MAX")
        assert not np.array_equal(got, want)
    except (ValueError, IndexError):
        pass


def test_ave_divisor_clipped_to_the_map_is_caught(monkeypatch):
    x = np.random.RandomState(3).rand(1, 2, 6, 6).astype(F32) + 1  # level 2 is padded
    y, _ = R.expansion32(x, 3, "AVE")
    assert np.abs(y - R.forward64(x, 3, "AVE")).max() < 1e-6
    level = R.level

    def clipped(h, w, lv, i, j):
        _, kh, kw, ph, pw = level(h, w, lv)
        return ((min(i * kh - ph + kh, h) - max(i * kh - ph, 0)) * (min(j * kw - pw + kw, w) - max(j * kw - pw, 0)))

    monkeypatch.setattr(R, "pool_size", clipped)
    assert np.abs(y - R.forward64(x, 3, "AVE")).max() > 1e-2


def test_last_maximum_winning_is_caught():
    x = R.specials(np.random.RandomState(4), (2, 3, 9, 8))  # values in steps of 0.5: ties in most windows
    _, arg = R.expansion32(x, 3, "MAX")
    last = []
    for lv in range(3):
        v = R._tiles(x, lv, -np.inf)
        taps = R._tiles(np.broadcast_to(np.arange(72).reshape(1, 1, 9, 8), x.shape), lv, -1)
        ok = v > -R.FLT_MAX
        m = np.where(ok, v, -np.inf).max(-1, keepdims=True)
        rev = np.argmax((ok & (v == m))[..., ::-1], -1)
        k = v.shape[-1] - 1 - rev
        idx = np.where(ok.any(-1), np.take_along_axis(taps, k[..., None], -1)[..., 0], -1)
        last.append(idx.reshape(2, -1))
    assert not np.array_equal(np.concatenate(last, 1), arg)


# --------------------------------------------------------------------------- every accepted level's geometry
def test_every_accepted_level_pools_bins_by_bins():
    """For every side from 1 to 399 and level up to 8: a level with pad < kernel pools exactly bins windows, each
    starting inside the map, and AVE divides every window by the whole kernel"""
    for side in range(1, 400):
        for lv in range(9):
            bins, k, _, pad, _ = R.level(side, side, lv)
            assert (bins, k, pad) == (2 ** lv, -(-side // 2 ** lv), (k * bins - side + 1) // 2)
            if pad >= k:
                continue
            assert R.pooled(side, k, pad) == bins, (side, lv)
            assert all(0 <= i * k - pad + k and i * k - pad < side for i in range(bins)), (side, lv)
            assert all(R.pool_size(side, side, lv, i, i) == k * k for i in range(bins)), (side, lv)


# --------------------------------------------------------------------------- the parser and the plan
SHAPE_CASES = [  # (bottom, pyramid height, per-sample top): Caffe's test_spp_layer.cpp geometries and the fixture's
    ((2, 3, 9, 8), 3, 63), ((4, 3, 1024, 765), 5, 1023), ((10, 3, 7, 7), 3, 63), ((100, 64, 6, 6), 3, 1344),
    ((64, 256, 13, 13), 3, 5376), ((3, 2, 5, 40), 2, 10),
]


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("bottom,h,per", SHAPE_CASES)
def test_shape_inference_and_plan_line(cos, tmp_path, bottom, h, per, pool):
    top = R.infer(bottom, h)
    assert top == (bottom[0], per)
    text = cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": top}, _spp(f"pyramid_height: {h} pool: {pool}")
                                           + EUCLID))
    levels = "".join(f" level{lv} {b}x{b} k{kh}x{kw} p{ph}x{pw}"
                     for lv, (b, kh, kw, ph, pw) in enumerate(R.level(bottom[2], bottom[3], lv) for lv in range(h)))
    shape = "x".join(map(str, bottom))
    assert f"op 0 SPP({pool}) s {shape} -> {bottom[0]}x{per}{levels} staged-bottom\n" in text
    assert "params 0 blobs 0" in text  # SPP owns no blob


def test_one_level_is_poolings_4d_top(cos, tmp_path):
    assert R.infer((2, 3, 9, 8), 1) == (2, 3, 1, 1)
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 9, 8), "t": (2, 3, 1, 1)},
                                           _spp("pyramid_height: 1 pool: AVE") + EUCLID))
    assert "op 0 SPP(AVE) s 2x3x9x8 -> 2x3x1x1 level0 1x1 k9x8 p0x0 staged-bottom\n" in text


def test_max_is_the_default_and_the_argmax_is_the_tops_size(cos, tmp_path):
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 9, 8), "t": (2, 63)}, _spp() + EUCLID))
    assert "op 0 SPP(MAX) s 2x3x9x8 -> 2x63 level0 1x1 k9x8 p0x0 level1 2x2 k5x4 p1x0 level2 4x4 k3x2 p2x0" in text


PARSER_REFUSALS = [  # (bottom, spp_param, message)
    ((2, 3, 8), "pyramid_height: 2", "Input must have 4 axes, corresponding to (num, channels, height, width)"),
    ((2, 3, 8, 8, 2), "pyramid_height: 2", "Input must have 4 axes, corresponding to (num, channels, height, width)"),
    ((2, 3, 0, 8), "pyramid_height: 2", "Input dimensions cannot be zero."),
    ((2, 3, 8, 0), "pyramid_height: 2", "Input dimensions cannot be zero."),
    ((2, 3, 8, 8), "pool: MAX", "spp_param pyramid_height must be at least 1 (a pyramid of no levels pools nothing)"),
    ((2, 3, 8, 8), "pyramid_height: 0",
     "spp_param pyramid_height must be at least 1 (a pyramid of no levels pools nothing)"),
    ((2, 256, 13, 13), "pyramid_height: 4", "Check failed: pad_h_ < kernel_h_ (2 vs. 2) at pyramid level 3 (8 bins)"),
    ((2, 3, 16, 5), "pyramid_height: 3", "Check failed: pad_w_ < kernel_w_ (2 vs. 2) at pyramid level 2 (4 bins)"),
    ((1, 1, 1, 1), "pyramid_height: 2", "Check failed: pad_h_ < kernel_h_ (1 vs. 1) at pyramid level 1 (2 bins)"),
]


@pytest.mark.parametrize("bottom,param,want", PARSER_REFUSALS)
def test_parser_refusals(cos, tmp_path, bottom, param, want):
    with pytest.raises(cos.CosError, match="^layer 's' \\(SPP\\): " + re.escape(want) + "$"):
        cos.native_producer_plan(_write(tmp_path, {"x": bottom, "t": (1,)}, _spp(param) + EUCLID))
    h = int(re.search(r"pyramid_height: (\d+)", param).group(1)) if "pyramid_height" in param else 0
    with pytest.raises(ValueError, match="^" + re.escape(want) + "$"):
        R.infer(bottom, h)


def test_thirteen_by_thirteen_takes_three_levels(cos, tmp_path):
    text = cos.native_producer_plan(_write(tmp_path, {"x": (2, 256, 13, 13), "t": (2, 5376)}, _spp() + EUCLID))
    assert "level2 4x4 k4x4 p2x2" in text


@pytest.mark.parametrize("layer,want", [
    (_spp("pyramid_height: 2 pool: STOCHASTIC"), "pool method STOCHASTIC is not supported (MAX and AVE are)"),
    (_spp("pyramid_height: 2", top="x"), "SPP Layer does not allow in-place computation."),
])
def test_plan_refusals(cos, tmp_path, layer, want):
    body = ('layer { name: "sc" type: "Scale" bottom: "in0" top: "x" scale_param { axis: 0 } }\n' + layer +
            EUCLID.replace('"y"', '"x"' if 'top: "x"' in layer else '"y"'))
    with pytest.raises(cos.CosError, match="^layer 's' \\(SPP\\): " + re.escape(want) + " \\(native producer\\)$"):
        cos.native_producer_plan(_write(tmp_path, {"in0": (2, 3, 8, 8), "t": (2, 15)}, body))


# --------------------------------------------------------------------------- the fixture
SPP_OPS = """\
op 0 ConvBiasReLUMaxPool conv1+pool1+relu1 100x3x32x32 -> 100x32x16x16 k5x5 s1x1 p2x2 pool3/2 w=0:2400 b=2400:32 \
staged-bottom
op 1 Convolution conv2 100x32x16x16 -> 100x32x16x16 k5x5 s1x1 p2x2 w=2432:25600 b=28032:32
op 2 ReLU relu2 100x32x16x16 -> 100x32x16x16 in-place
op 3 Pooling(AVE) pool2 100x32x16x16 -> 100x32x8x8 k3x3 s2x2 p0x0
op 4 Convolution conv3 100x32x8x8 -> 100x64x6x6 k5x5 s1x1 p1x1 w=28064:51200 b=79264:64
op 5 ReLU relu3 100x64x6x6 -> 100x64x6x6 in-place
op 6 SPP(MAX) spp 100x64x6x6 -> 100x1344 level0 1x1 k6x6 p0x0 level1 2x2 k3x3 p0x0 level2 4x4 k2x2 p1x1
op 7 InnerProduct ip1 100x1344 -> 100x64 w=79328:86016 b=165344:64
op 8 InnerProduct ip2 100x64 -> 100x10 w=165408:640 b=166048:10
op 9 SoftmaxWithLoss loss 100x10 -> scalar axis=1 label=1 loss_weight=1
"""


def test_fixture_layout_and_plan(cos):
    from caffeonspark_b200 import nets
    solver = os.path.join(CONFIGS, "cifar10_quick_spp_solver.prototxt")
    text = cos.native_producer_plan(solver)
    assert "".join(ln + "\n" for ln in text.splitlines() if ln.startswith("op ")) == SPP_OPS
    _check_layout(cos, text, solver, nets.CIFAR10_QUICK_SPP_PARAM_COUNT)
    d = cos.parse_solver(solver)
    assert nets.CIFAR10_QUICK_SPP_PARAM_COUNT == 166058 == 145578 - 65600 + 86080 and len(d.counts) == 10
    m = nets.cifar10_quick_spp_module()
    assert [p.numel() for p in m.parameters()] == d.counts
    import torch
    assert m(torch.zeros(2, 3, 32, 32)).shape == (2, 10)


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("shape,h", [((2, 3, 9, 8), 3), ((1, 2, 6, 6), 3), ((2, 2, 7, 5), 2), ((1, 3, 4, 4), 1)])
def test_the_pytorch_mirror_is_the_expansion(shape, h, pool):
    """nets.spp (explicit padding, one pool per level) against the float64 reference on NaN-free values"""
    import torch
    from caffeonspark_b200 import nets
    x = np.random.RandomState(h).randn(*shape)
    y = nets.spp(torch.from_numpy(x), h, pool).numpy()
    assert np.abs(y.reshape(shape[0], -1) - R.forward64(x.astype(F32), h, pool)).max() < 1e-6
