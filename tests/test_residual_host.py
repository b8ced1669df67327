"""CPU tests of Split, Eltwise and Scale on the built-in engine: Scale's learnable layout for each of its forms against
hand-computed counts, shapes, mults and fillers; the ResNet-20 fixture's layout and plan (Split tops alias their
bottom, in-place layers on a Split top and every Scale top get storage of their own); and every refusal of the three
layers, which names the layer and uses Caffe's CHECK wording."""
import os
import re

import pytest

from conftest import ROOT
from test_native_producer_host import _check_layout, _ops

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
RESNET_SOLVER = os.path.join(CONFIGS, "cifar10_resnet20_solver.prototxt")
RESNET_NET = os.path.join(CONFIGS, "cifar10_resnet20_train_test.prototxt")


def _write(tmp_path, body, shape=(2, 3, 4, 5)):
    """A net of an Input `x` of `shape` and labels, `body`, and an InnerProduct `ip` on blob `y` into SoftmaxWithLoss."""
    dims = " ".join(f"dim: {d}" for d in shape)
    (tmp_path / "net.prototxt").write_text(
        f'name: "t" layer {{ name: "in" type: "Input" top: "x" top: "label" input_param {{ shape {{ {dims} }} '
        f'shape {{ dim: {shape[0]} }} }} }}\n' + body +
        '\nlayer { name: "ip" type: "InnerProduct" bottom: "y" top: "ip" inner_product_param { num_output: 3 } }\n'
        'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / "solver.prototxt")


def _blob_lines(text):
    return [line.split()[2:] for line in text.splitlines() if line.startswith("blob ")]


# Scale on a 2x3x4x5 bottom: (scale_param, scale blob shape, bias?, plan's outer/dim/inner)
SCALE_CASES = [
    ("", "3", False, (2, 3, 20)),
    ("scale_param { bias_term: true }", "3", True, (2, 3, 20)),
    ("scale_param { num_axes: 0 bias_term: true }", "scalar", True, (1, 1, 120)),
    ("scale_param { num_axes: -1 }", "3x4x5", False, (2, 60, 1)),
    ("scale_param { axis: 2 }", "4", False, (6, 4, 5)),
    ("scale_param { axis: 2 num_axes: 2 bias_term: true }", "4x5", True, (6, 20, 1)),
    ("scale_param { axis: -3 num_axes: 1 }", "3", False, (2, 3, 20)),
]


@pytest.mark.parametrize("param,shape,bias,dims", SCALE_CASES)
def test_scale_layout_and_plan(cos, tmp_path, param, shape, bias, dims):
    solver = _write(tmp_path, f'layer {{ name: "sc" type: "Scale" bottom: "x" top: "y" {param} }}')
    d = cos.parse_solver(solver)
    n = 1
    for v in ([] if shape == "scalar" else shape.split("x")):
        n *= int(v)
    assert d.counts == [n] * (2 if bias else 1) + [3 * 60, 3]
    assert d.lr_mult == [1.0] * len(d.counts) and d.decay_mult == [1.0] * len(d.counts)
    text = cos.native_producer_plan(solver)
    sc = next(line for line in text.splitlines() if " Scale sc " in line)
    assert sc.endswith(f"w=0:{n}" + (f" b={n}:{n}" if bias else "") + " outer={} dim={} inner={} staged-bottom".format(*dims))
    blobs = _blob_lines(text)
    assert blobs[0] == [f"0:{n}", shape, "constant"]  # the default filler: constant 1
    if bias:
        assert blobs[1] == [f"{n}:{n}", shape, "constant"]
    _check_layout(cos, text, solver, sum(d.counts))


def test_scale_fillers_and_mults(cos, tmp_path):
    solver = _write(tmp_path, 'layer { name: "sc" type: "Scale" bottom: "x" top: "y" param { lr_mult: 0.5 decay_mult: 0 } '
                              'param { lr_mult: 2 decay_mult: 3 } scale_param { bias_term: true '
                              'filler { type: "uniform" min: 0.5 max: 2 } bias_filler { type: "gaussian" std: 0.1 } } }')
    d = cos.parse_solver(solver)
    assert d.counts[:2] == [3, 3] and d.lr_mult[:2] == [0.5, 2.0] and d.decay_mult[:2] == [0.0, 3.0]
    blobs = _blob_lines(cos.native_producer_plan(solver))
    assert blobs[0] == ["0:3", "3", "uniform"] and blobs[1] == ["3:3", "3", "gaussian"]


def test_two_bottom_scale_layout_and_refusal(cos, tmp_path):
    # no scale blob: the bias takes bottom[1]'s shape
    body = ('layer { name: "s" type: "Input" top: "s" input_param { shape { dim: 3 dim: 4 } } }\n'
            'layer { name: "sc" type: "Scale" bottom: "x" bottom: "s" top: "y" scale_param { bias_term: true } }')
    solver = _write(tmp_path, body)
    d = cos.parse_solver(solver)
    assert d.counts == [12, 180, 3]
    with pytest.raises(cos.CosError, match=r"^layer 'sc' \(Scale\): the two-bottom form"):
        cos.native_producer_plan(solver)
    (tmp_path / "b").mkdir()
    solver = _write(tmp_path / "b", body.replace("scale_param { bias_term: true }", ""))
    assert cos.parse_solver(solver).counts == [180, 3]


def test_named_scale_param_shares_its_owner(cos, tmp_path):
    body = ('layer { name: "sa" type: "Scale" bottom: "x" top: "a" param { name: "g" } param { name: "b" } '
            'scale_param { bias_term: true } }\n'
            'layer { name: "sb" type: "Scale" bottom: "a" top: "y" param { name: "g" } param { name: "b" } '
            'scale_param { bias_term: true } }')
    solver = _write(tmp_path, body)
    assert cos.parse_solver(solver).counts == [3, 3, 180, 3]
    lines = [line for line in cos.native_producer_plan(solver).splitlines() if " Scale " in line]
    assert "shares=" not in lines[0] and lines[0].endswith("w=0:3 b=3:3 outer=2 dim=3 inner=20 staged-bottom")
    assert lines[1].endswith("w=0:3 b=3:3 shares=0,1 outer=2 dim=3 inner=20")


@pytest.mark.parametrize("body,match", [
    ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" scale_param { num_axes: -2 } }',
     r"^layer 'sc' \(Scale\): num_axes must be non-negative, or -1 to extend to the end of bottom\[0\]$"),
    ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" scale_param { axis: 2 num_axes: 3 } }',
     r"^layer 'sc' \(Scale\): scale blob's shape extends past bottom\[0\]'s shape when applied starting with "
     r"bottom\[0\] axis = 2$"),
    ('layer { name: "sc" type: "Scale" bottom: "x" top: "y" scale_param { axis: 4 } }',
     r"^layer 'sc' \(Scale\): axis 4 out of range for 4-D Blob"),
    ('layer { name: "s" type: "Input" top: "s" input_param { shape { dim: 3 dim: 5 } } }\n'
     'layer { name: "sc" type: "Scale" bottom: "x" bottom: "s" top: "y" }',
     r"^layer 'sc' \(Scale\): dimension mismatch between bottom\[0\]->shape\(2\) and scale->shape\(1\)"),
    ('layer { name: "sp" type: "Split" bottom: "x" top: "x" top: "y" }',
     r"^layer 'sp' \(Split\): Split Layer does not allow in-place computation\.$"),
    ('layer { name: "e" type: "Eltwise" bottom: "x" top: "y" }',
     r"^layer 'e' \(Eltwise\): Eltwise Layer takes at least 2 bottom blob\(s\) as input\.$"),
    ('layer { name: "sp" type: "Split" bottom: "x" top: "a" top: "b" }\n'
     'layer { name: "e" type: "Eltwise" bottom: "a" bottom: "b" top: "y" eltwise_param { coeff: 1 } }',
     r"^layer 'e' \(Eltwise\): Eltwise Layer takes one coefficient per bottom blob\.$"),
    ('layer { name: "sp" type: "Split" bottom: "x" top: "a" top: "b" }\n'
     'layer { name: "e" type: "Eltwise" bottom: "a" bottom: "b" top: "y" eltwise_param { operation: PROD coeff: 1 '
     'coeff: 2 } }',
     r"^layer 'e' \(Eltwise\): Eltwise layer only takes coefficients for summation\.$"),
    ('layer { name: "sp" type: "Split" bottom: "x" top: "a" top: "b" }\n'
     'layer { name: "p" type: "Pooling" bottom: "b" top: "c" pooling_param { pool: MAX kernel_size: 2 stride: 2 } }\n'
     'layer { name: "e" type: "Eltwise" bottom: "a" bottom: "c" top: "y" }',
     r"^layer 'e' \(Eltwise\): bottom 1 is 2x3x2x3, bottom 0 2x3x4x5 \(Check failed: bottom\[i\]->shape\(\) == "
     r"bottom\[0\]->shape\(\)\)$"),
])
def test_refusals_name_the_layer(cos, tmp_path, body, match):
    solver = _write(tmp_path, body)
    with pytest.raises(cos.CosError, match=match):
        cos.parse_solver(solver)
    with pytest.raises(cos.CosError, match=match):
        cos.native_producer_plan(solver)


def test_eltwise_plans(cos, tmp_path):
    body = ('layer { name: "sp" type: "Split" bottom: "x" top: "a" top: "b" top: "c" top: "u" }\n'
            'layer { name: "ea" type: "Scale" bottom: "a" top: "a2" }\n'
            'layer { name: "e1" type: "Eltwise" bottom: "a2" bottom: "b" top: "s" eltwise_param { coeff: 0.5 '
            'coeff: -2 } }\n'
            'layer { name: "e2" type: "Eltwise" bottom: "s" bottom: "c" top: "p" eltwise_param { operation: PROD '
            'stable_prod_grad: false } }\n'
            'layer { name: "sq" type: "Split" bottom: "p" top: "p0" top: "q1" top: "q2" }\n'
            'layer { name: "e3" type: "Eltwise" bottom: "p0" bottom: "q1" bottom: "q2" top: "y" eltwise_param { '
            'operation: 2 } }')
    text = cos.native_producer_plan(_write(tmp_path, body))
    lines = [line for line in text.splitlines() if line.startswith("op ")]
    split = [line for line in lines if " Split sp " in line]
    assert [line.split()[-3:] for line in split] == [["top=0", "data=bottom", "staged-bottom"],
                                                    ["top=1", "data=bottom", "staged-bottom"],
                                                    ["top=2", "data=bottom", "staged-bottom"],
                                                    ["data=bottom", "unread", "staged-bottom"]]
    assert next(line for line in lines if " e1 " in line).endswith("bottoms=2 coeff=0.5,-2 no-bottom-grad")
    assert next(line for line in lines if " e2 " in line).split()[2] == "Eltwise(PROD)"
    assert next(line for line in lines if " e2 " in line).endswith("bottoms=2 top/bottom_grad no-bottom-grad")
    e3 = next(line for line in lines if " e3 " in line)
    assert e3.split()[2] == "Eltwise(MAX)" and e3.endswith("bottoms=3")  # every bottom follows the Scale
    assert [line.split()[-2:] for line in lines if " Split sq " in line] == [
        ["top=0", "data=bottom"], ["top=1", "data=bottom"], ["top=2", "data=bottom"]]


def test_in_place_layers_on_a_split_top_get_storage_of_their_own(cos, tmp_path):
    body = ('layer { name: "sc" type: "Scale" bottom: "x" top: "h" }\n'
            'layer { name: "sp" type: "Split" bottom: "h" top: "a" top: "b" }\n'
            'layer { name: "r" type: "ReLU" bottom: "a" top: "a" }\n'
            'layer { name: "g" type: "Sigmoid" bottom: "b" top: "b" }\n'
            'layer { name: "r2" type: "ReLU" bottom: "a" top: "a" }\n'
            'layer { name: "e" type: "Eltwise" bottom: "a" bottom: "b" top: "y" }')
    lines = [line for line in cos.native_producer_plan(_write(tmp_path, body)).splitlines() if line.startswith("op ")]
    kinds = {line.split()[3]: line for line in lines}
    assert "in-place" not in kinds["r"] and "in-place" not in kinds["g"]
    assert kinds["r2"].endswith(" in-place")  # r's top has storage of its own, so r2 may share it


def test_layouts_without_these_layers_are_unchanged(cos, tmp_path):
    """A Scale-free net parses as before, and Split / Eltwise add no learnable blob (the model:
    test_lrn_fields_leave_the_layout_unchanged)."""
    counts = []
    for body in ('layer { name: "r" type: "ReLU" bottom: "x" top: "y" }',
                 'layer { name: "sp" type: "Split" bottom: "x" top: "a" top: "b" }\n'
                 'layer { name: "e" type: "Eltwise" bottom: "a" bottom: "b" top: "y" eltwise_param { operation: MAX } }'):
        (tmp_path / str(len(counts))).mkdir()
        counts.append(cos.parse_solver(_write(tmp_path / str(len(counts)), body)).counts)
    assert counts == [[3 * 60, 3]] * 2


# --------------------------------------------------------------------------- the ResNet-20 fixture
def _prototxt_layers(path):
    """(name, type, body) of every layer of a prototxt, by brace matching."""
    text = re.sub(r"#[^\n]*", "", open(path).read())
    out, i = [], 0
    while True:
        i = text.find("layer {", i)
        if i < 0:
            return out
        depth, j = 0, text.index("{", i)
        while True:
            depth += {"{": 1, "}": -1}.get(text[j], 0)
            j += 1
            if depth == 0:
                break
        body = text[i:j]
        out.append((re.search(r'name: "([^"]+)"', body).group(1), re.search(r'type: "([^"]+)"', body).group(1), body))
        i = j


def _independent_count():
    """Parameters of the fixture from its layer list alone: channels and spatial size followed through the layers."""
    channels, total, stats = {}, 0, 0
    for name, kind, body in _prototxt_layers(RESNET_NET):
        bottoms = re.findall(r'bottom: "([^"]+)"', body)
        tops = re.findall(r'top: "([^"]+)"', body)
        if kind == "MemoryData":
            channels["data"] = int(re.search(r"channels: (\d+)", body).group(1))
        elif kind == "Convolution":
            k = int(re.search(r"kernel_size: (\d+)", body).group(1))
            cout = int(re.search(r"num_output: (\d+)", body).group(1))
            assert "bias_term: false" in body
            total += cout * channels[bottoms[0]] * k * k
            channels[tops[0]] = cout
        elif kind == "BatchNorm":
            c = channels[bottoms[0]]
            total += 2 * c + 1
            stats += 2 * c + 1
        elif kind == "Scale":
            assert "bias_term: true" in body
            total += 2 * channels[bottoms[0]]
        elif kind == "InnerProduct":
            nout = int(re.search(r"num_output: (\d+)", body).group(1))
            total += nout * channels[bottoms[0]] + nout  # after global pooling: one value per channel
        else:
            for t in tops:
                channels[t] = channels.get(bottoms[0], 0) if bottoms else 0
    return total, stats


def test_the_fixture_layout(cos):
    from caffeonspark_b200 import nets
    total, stats = _independent_count()
    d = cos.parse_solver(RESNET_SOLVER)
    assert d.param_count == total
    layers = _prototxt_layers(RESNET_NET)
    bn_blobs = [i for i, lr in enumerate(d.lr_mult) if lr == 0]
    assert len(bn_blobs) == 3 * sum(kind == "BatchNorm" for _, kind, _ in layers) == 3 * 21
    assert sum(d.counts[i] for i in bn_blobs) == stats
    assert [p.numel() for p in nets.resnet20_module().parameters()] == list(d.counts)
    assert d.momentum == pytest.approx(0.9) and d.weight_decay == pytest.approx(1e-4)
    assert d.lr_policy == "multistep" and d.base_lr == pytest.approx(0.1) and d.stepvalues == (32000, 48000)


def test_the_fixture_plan(cos):
    text = cos.native_producer_plan(RESNET_SOLVER)
    _check_layout(cos, text, RESNET_SOLVER, _independent_count()[0])
    lines = [line for line in text.splitlines() if line.startswith("op ")]
    layers = _prototxt_layers(RESNET_NET)
    by_kind = lambda k: [name for name, kind, _ in layers if kind == k]  # noqa: E731
    # every Split op (one per top), Eltwise and Scale op of the net, in net order
    assert [line.split()[3] for line in lines if " Split " in line] == [n for n in by_kind("Split") for _ in range(2)]
    assert [line.split()[3] for line in lines if " Eltwise(SUM) " in line] == by_kind("Eltwise")
    assert [line.split()[3] for line in lines if " Scale " in line] == by_kind("Scale")
    assert len(by_kind("Split")) == len(by_kind("Eltwise")) == 9 and len(by_kind("Scale")) == 21
    for line in lines:
        f = line.split()
        if f[2] == "Split":
            assert "data=bottom" in line and "unread" not in line and "in-place" not in line
        if f[2] == "Eltwise(SUM)":
            assert line.endswith("bottoms=2 coeff=1,1")
        if f[2] == "Scale":  # written in place in the prototxt, yet a top of its own: the scale gradient reads x
            assert "in-place" not in line and re.search(r" w=\d+:\d+ b=\d+:\d+ outer=100 dim=\d+ inner=\d+$", line)
        if f[2] == "ReLU":  # after a Scale or an Eltwise: in place
            assert line.endswith(" in-place")
    pool = next(line for line in lines if " Pooling(AVE) pool " in line)
    assert " 100x64x8x8 -> 100x64x1x1 k8x8 s1x1 p0x0" in pool
    assert "Convolution conv1 100x3x32x32 -> 100x16x32x32" in text and "staged-bottom" in lines[0]
    assert sum(" staged-bottom" in line for line in lines) == 1
    blobs = _blob_lines(text)
    kinds = [b[2] for b in blobs]
    assert kinds.count("msra") == 21 + 1  # 19 convs + 2 projections, and fc10
    from caffeonspark_b200 import nets
    names = [n for n, _ in nets.resnet20_module().named_parameters()]  # each unit: conv 0, BatchNorm 1, Scale 2
    scale_blobs = [i for i, n in enumerate(names) if n.endswith(("2.weight", "2.bias"))]
    assert len(scale_blobs) == 42 and all(kinds[i] == "constant" for i in scale_blobs)
