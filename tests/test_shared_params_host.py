"""CPU tests of named (shared) params, Slice and ContrastiveLoss: the layout of the reference's siamese MNIST example
and of a variant without its two new layer types, Caffe's sharing checks and lr_mult / decay_mult rules, the engine's
plan of the siamese net, Slice plans over several axes and slice points, and the ContrastiveLoss bottom checks."""
import os

import pytest

from conftest import ROOT
from test_native_producer_host import _check_layout, _ops

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
SIAMESE_P, SIAMESE_BLOBS = 431102, 10
SIAMESE_COUNTS = [500, 20, 25000, 50, 400000, 500, 5000, 10, 20, 2]


def _siamese_text():
    return open(os.path.join(CONFIGS, "mnist_siamese_train_test.prototxt")).read()


def _write_solver(tmp_path, net):
    (tmp_path / "net.prototxt").write_text(net)
    solver = open(os.path.join(CONFIGS, "mnist_siamese_solver.prototxt")).read()
    solver = solver.replace('net: "examples/siamese/mnist_siamese_train_test.prototxt"', 'net: "net.prototxt"')
    (tmp_path / "solver.prototxt").write_text(solver)
    return str(tmp_path / "solver.prototxt")


def memory_data_copy(tmp_path, batch=64):
    """The reference's siamese solver and net with the two LevelDB Data layers swapped for MemoryData (2x28x28)."""
    net = _siamese_text()
    start, end = net.index("layer {"), net.index('layer {\n  name: "slice_pair"')
    data = "".join(f'layer {{ name: "pair_data" type: "MemoryData" top: "pair_data" top: "sim" include {{ phase: {ph} }} '
                   f'memory_data_param {{ batch_size: {b} channels: 2 height: 28 width: 28 }} }}\n'
                   for ph, b in (("TRAIN", batch), ("TEST", 100)))
    return _write_solver(tmp_path, net[:start] + data + net[end:])


def _input_two_softmax_copy(tmp_path):
    """The siamese net with Slice replaced by an Input layer and a SoftmaxWithLoss on each branch."""
    net = _siamese_text()
    start, end = net.index("layer {"), net.index('layer {\n  name: "conv1"')
    data = ('layer { name: "input" type: "Input" top: "data" top: "data_p" top: "label" input_param { '
            'shape { dim: 64 dim: 1 dim: 28 dim: 28 } shape { dim: 64 dim: 1 dim: 28 dim: 28 } shape { dim: 64 } } }\n')
    loss = net.index('layer {\n  name: "loss"')
    losses = ('layer { name: "loss" type: "SoftmaxWithLoss" bottom: "feat" bottom: "label" top: "loss" }\n'
              'layer { name: "loss_p" type: "SoftmaxWithLoss" bottom: "feat_p" bottom: "label" top: "loss_p" }\n')
    return _write_solver(tmp_path, net[:start] + data + net[end:loss] + losses)


def test_siamese_example_parses_to_caffes_layout(cos, tmp_path):
    d = cos.parse_solver(memory_data_copy(tmp_path))
    assert d.param_count == SIAMESE_P and len(d.counts) == SIAMESE_BLOBS
    assert d.counts == SIAMESE_COUNTS
    assert d.lr_mult == [1.0, 2.0] * 5 and d.decay_mult == [1.0] * 10
    assert d.lr_policy == "inv" and d.base_lr == pytest.approx(0.01) and d.momentum == pytest.approx(0.9)
    assert d.batch_size == 64


def test_named_params_are_shared_without_the_new_layer_types(cos, tmp_path):
    # before sharing was modelled this parsed to 862,204 parameters in 20 blobs: the two branches trained apart
    d = cos.parse_solver(_input_two_softmax_copy(tmp_path))
    assert d.param_count == SIAMESE_P and d.counts == SIAMESE_COUNTS
    assert d.lr_mult == [1.0, 2.0] * 5


def _two_ip(tmp_path, p1, p2, nout2=4, bottom2_channels=3):
    """Two InnerProducts on two inputs, with the given param blocks, feeding one ContrastiveLoss (through a third
    InnerProduct to 4 outputs when the second has nout2 != 4)."""
    fix = ('layer { name: "ip_q" type: "InnerProduct" bottom: "b" top: "b4" inner_product_param { num_output: 4 } }\n'
           if nout2 != 4 else "")
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "in" type: "Input" top: "x" top: "x2" top: "sim" input_param { '
                 f'shape {{ dim: 2 dim: 3 }} shape {{ dim: 2 dim: {bottom2_channels} }} shape {{ dim: 2 }} }} }}\n'
                 f'layer {{ name: "ip" type: "InnerProduct" bottom: "x" top: "a" {p1} '
                 'inner_product_param { num_output: 4 } }\n'
                 f'layer {{ name: "ip_p" type: "InnerProduct" bottom: "x2" top: "b" {p2} '
                 f'inner_product_param {{ num_output: {nout2} }} }}\n{fix}'
                 f'layer {{ name: "loss" type: "ContrastiveLoss" bottom: "a" bottom: "{"b4" if fix else "b"}" '
                 'bottom: "sim" top: "loss" }\n')
    return str(p)


def test_sharing_a_param_with_another_shape_is_refused(cos, tmp_path):
    with pytest.raises(cos.CosError, match=r"Cannot share param 'w' owned by layer 'ip' with layer 'ip_p'; shape "
                                           r"mismatch.  Owner layer param shape is 4 3 \(12\); sharing layer expects "
                                           r"shape 6 2 \(12\)"):
        cos.native_producer_plan(_two_ip(tmp_path, 'param { name: "w" }', 'param { name: "w" }', 6, 2))


def test_permissive_sharing_needs_an_equal_count_only(cos, tmp_path):
    text = cos.native_producer_plan(_two_ip(tmp_path, 'param { name: "w" }',
                                            'param { name: "w" share_mode: PERMISSIVE }', 6, 2))
    assert "params 50 blobs 5" in text  # w 4x3, ip's bias 4, ip_p's bias 6, ip_q 4x6 + 4
    assert "shares=0" in next(line for line in text.splitlines() if " ip_p " in line)
    with pytest.raises(cos.CosError, match=r"Cannot share param 'w' owned by layer 'ip' with layer 'ip_p'; count "
                                           r"mismatch.  Owner layer param shape is 4 3 \(12\); sharing layer shape is "
                                           r"5 3 \(15\)"):
        cos.native_producer_plan(_two_ip(tmp_path, 'param { name: "w" }',
                                         'param { name: "w" share_mode: PERMISSIVE }', 5, 3))


@pytest.mark.parametrize("field", ["lr_mult", "decay_mult"])
def test_a_different_explicit_mult_is_refused(cos, tmp_path, field):
    with pytest.raises(cos.CosError, match=rf"^Shared param 'w' has mismatched {field}\.$"):
        cos.native_producer_plan(_two_ip(tmp_path, f'param {{ name: "w" {field}: 1 }}',
                                         f'param {{ name: "w" {field}: 2 }}'))


def test_the_first_explicit_mult_wins(cos, tmp_path):
    # the owner sets neither: the sharer's lr_mult becomes the blob's, and a repeat of it is accepted
    path = _two_ip(tmp_path, 'param { name: "w" } param { name: "b" decay_mult: 0 }',
                   'param { name: "w" lr_mult: 3 } param { name: "b" decay_mult: 0 }')
    solver = tmp_path / "solver.prototxt"
    solver.write_text(f'net: "{path}"\nbase_lr: 0.1\nlr_policy: "fixed"\n')
    d = cos.parse_solver(str(solver))
    assert d.counts == [12, 4] and d.lr_mult == [3.0, 1.0] and d.decay_mult == [1.0, 0.0]


def test_siamese_plan_marks_the_sharers_and_slices_the_staged_input(cos, tmp_path):
    solver = memory_data_copy(tmp_path)
    text = cos.native_producer_plan(solver)
    _check_layout(cos, text, solver, SIAMESE_P)
    lines = [line for line in text.splitlines() if line.startswith("op ")]
    assert _ops(text)[:2] == ["Slice slice_pair 64x2x28x28 -> 64x1x28x28"] * 2
    assert lines[0].endswith("axis=1 begin=0 staged-bottom") and lines[1].endswith("axis=1 begin=1 staged-bottom")
    shares = {line.split()[3]: line.split("shares=")[1].split()[0] for line in lines if "shares=" in line}
    assert shares == {"conv1_p": "0,1", "conv2_p": "2,3", "ip1_p": "4,5", "ip2_p": "6,7", "feat_p": "8,9"}
    owner = {line.split()[3]: line.split(" w=")[1].split()[:2] for line in lines if " w=" in line}
    for nm in ("conv1", "conv2", "ip1", "ip2", "feat"):
        assert owner[nm + "_p"] == owner[nm]  # the sharer reads and accumulates into the owner's offsets
    # Slice's tops come from a staged input: no data gradient flows into them, so conv1 and conv1_p compute none
    assert [line.split()[3] for line in lines if line.endswith(" no-bottom-grad")] == ["conv1", "conv1_p"]
    assert sum("-bottom" in line for line in lines) == 4
    assert _ops(text)[-1] == "ContrastiveLoss loss 64x2 -> scalar"
    assert lines[-1].endswith("margin=1 loss_weight=1")
    assert all(line.endswith(("xavier", "constant")) for line in text.splitlines() if line.startswith("blob "))


def _slice_net(tmp_path, x_shape, slice_param, ntops, a_top=0, b_top=1, sim=None, through_ip=False):
    """Input x -> Slice -> ContrastiveLoss(top a_top, top b_top, sim).  through_ip puts an InnerProduct first, so the
    Slice's bottom is not a staged input."""
    dims = " ".join(f"dim: {d}" for d in x_shape)
    tops = " ".join(f'top: "t{i}"' for i in range(ntops))
    n = sim if sim is not None else x_shape[0]
    src = "x"
    ip = ""
    if through_ip:
        ip = 'layer { name: "ip" type: "InnerProduct" bottom: "x" top: "h" inner_product_param { num_output: 6 } }\n'
        src = "h"
    p = tmp_path / "net.prototxt"
    p.write_text(f'name: "t" layer {{ name: "in" type: "Input" top: "x" top: "sim" input_param {{ shape {{ {dims} }} '
                 f'shape {{ dim: {n} }} }} }}\n{ip}'
                 f'layer {{ name: "s" type: "Slice" bottom: "{src}" {tops} {slice_param} }}\n'
                 f'layer {{ name: "loss" type: "ContrastiveLoss" bottom: "t{a_top}" bottom: "t{b_top}" bottom: "sim" '
                 'top: "loss" contrastive_loss_param { margin: 2 legacy_version: true } }\n')
    return str(p)


@pytest.mark.parametrize("shape,param,ntops,sim,outs,begins", [
    ((4, 6), "slice_param { slice_point: 2 slice_point: 4 }", 3, None, ["4x2", "4x2", "4x2"], [0, 2, 4]),
    ((4, 7), "slice_param { axis: 1 slice_point: 3 slice_point: 6 }", 3, None, ["4x3", "4x3", "4x1"], [0, 3, 6]),
    ((4, 6), "slice_param { axis: -1 }", 3, None, ["4x2", "4x2", "4x2"], [0, 2, 4]),  # equal split
    ((6, 4), "slice_param { axis: 0 slice_point: 3 }", 2, 3, ["3x4", "3x4"], [0, 3]),
    ((8, 4), "slice_param { slice_dim: 0 }", 4, 2, ["2x4"] * 4, [0, 2, 4, 6]),
    ((4, 3, 4, 1), "slice_param { axis: 2 slice_point: 1 slice_point: 2 }", 3, None,
     ["4x3x1x1", "4x3x1x1", "4x3x2x1"], [0, 1, 2]),
])
def test_slice_plans(cos, tmp_path, shape, param, ntops, sim, outs, begins):
    text = cos.native_producer_plan(_slice_net(tmp_path, shape, param, ntops, sim=sim))
    lines = [line for line in text.splitlines() if line.startswith("op ") and " Slice " in line]
    src = "x".join(str(d) for d in shape)
    assert _ops(text)[:ntops] == [f"Slice s {src} -> {o}" for o in outs]
    assert [int(line.split("begin=")[1].split()[0]) for line in lines] == begins
    assert all(line.endswith("staged-bottom") for line in lines)
    assert _ops(text)[-1] == f"ContrastiveLoss loss {outs[0]} -> scalar"
    assert "margin=2 legacy" in text and "params 0 blobs 0" in text


def test_no_data_gradient_before_the_first_learnable_blob(cos, tmp_path):
    # x -> ReLU -> Slice -> ip, ip_p -> ContrastiveLoss: nothing before the InnerProducts learns, so neither the ReLU,
    # the Slice nor the InnerProducts' data gradients are computed; the ops after them propagate as before
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "in" type: "Input" top: "x" top: "sim" input_param { shape { dim: 4 dim: 6 } '
                 'shape { dim: 4 } } }\n'
                 'layer { name: "r" type: "ReLU" bottom: "x" top: "r" }\n'
                 'layer { name: "s" type: "Slice" bottom: "r" top: "a" top: "b" slice_param { axis: 1 } }\n'
                 'layer { name: "ip" type: "InnerProduct" bottom: "a" top: "fa" inner_product_param { num_output: 5 } }\n'
                 'layer { name: "ip_p" type: "InnerProduct" bottom: "b" top: "fb" inner_product_param { num_output: 5 } }\n'
                 'layer { name: "r2" type: "ReLU" bottom: "fa" top: "fa" }\n'
                 'layer { name: "loss" type: "ContrastiveLoss" bottom: "fa" bottom: "fb" bottom: "sim" top: "loss" }\n')
    lines = [line for line in cos.native_producer_plan(str(p)).splitlines() if line.startswith("op ")]
    marks = [(line.split()[3], line.split()[-1]) for line in lines]
    assert marks == [("r", "staged-bottom"), ("s", "no-bottom-grad"), ("s", "no-bottom-grad"),
                     ("ip", "no-bottom-grad"), ("ip_p", "no-bottom-grad"), ("r2", "in-place"),
                     ("loss", "loss_weight=1")]


def test_slice_of_a_computed_blob_propagates_its_gradient(cos, tmp_path):
    text = cos.native_producer_plan(_slice_net(tmp_path, (4, 5), "slice_param { axis: 1 }", 2, through_ip=True))
    lines = [line for line in text.splitlines() if " Slice " in line]
    assert [line.split()[4:7] for line in lines] == [["4x6", "->", "4x3"]] * 2
    assert not any("staged-bottom" in line for line in lines)


@pytest.mark.parametrize("shape,param,ntops,msg", [
    ((4, 6), "slice_param { slice_point: 0 }", 2, r"slice_point 0 is not increasing inside \(0, 6\)"),
    ((4, 6), "slice_param { slice_point: 6 }", 2, r"slice_point 6 is not increasing inside \(0, 6\)"),
    ((4, 6), "slice_param { slice_point: 4 slice_point: 2 }", 3, r"slice_point 2 is not increasing"),
    ((4, 6), "slice_param { slice_point: 2 }", 3, r"1 slice_point\(s\) for 3 tops"),
    ((4, 6), "slice_param { axis: 1 }", 4, r"4 tops do not evenly divide slice axis 6"),
    ((4, 6), "slice_param { axis: 2 }", 2, r"slice axis 2 is out of range for a 2-axis bottom"),
    ((4, 6), "slice_param { axis: 1 slice_dim: 1 }", 2, r"either axis or slice_dim"),
])
def test_bad_slices_are_refused_with_the_layer_name(cos, tmp_path, shape, param, ntops, msg):
    with pytest.raises(cos.CosError, match=r"^layer 's' \(Slice\): " + msg):
        cos.native_producer_plan(_slice_net(tmp_path, shape, param, ntops))


def _loss_net(tmp_path, a, b, sim, nbottoms=3):
    dims = lambda s: " ".join(f"dim: {d}" for d in s)  # noqa: E731
    bottoms = ["a", "b", "sim"][:nbottoms]
    p = tmp_path / "net.prototxt"
    p.write_text('name: "t" layer { name: "in" type: "Input" top: "a" top: "b" top: "sim" input_param { '
                 f'shape {{ {dims(a)} }} shape {{ {dims(b)} }} shape {{ {dims(sim)} }} }} }}\n'
                 'layer { name: "loss" type: "ContrastiveLoss" '
                 + " ".join(f'bottom: "{x}"' for x in bottoms) + ' top: "loss" }\n')
    return str(p)


@pytest.mark.parametrize("a,b,sim,nbottoms,msg", [
    ((4, 2), (4, 3), (4,), 3, "a and b must have the same channels"),
    ((4, 2), (3, 2), (4,), 3, "a, b and sim must have the same first dimension"),
    ((4, 2), (4, 2), (3,), 3, "a, b and sim must have the same first dimension"),
    ((4, 2, 2, 1), (4, 2, 2, 1), (4,), 3, r"a and b must be N x C \(x 1 x 1\)"),
    ((4, 2), (4, 2, 1), (4,), 3, "bottoms must have 1 to 4 axes, a and b as many"),
    ((4, 2), (4, 2), (4, 2), 3, "sim must hold one value per pair"),
    ((4, 2), (4, 2), (4,), 2, r"needs 3 bottoms \(a, b, sim\)"),
])
def test_contrastive_loss_bottom_checks(cos, tmp_path, a, b, sim, nbottoms, msg):
    with pytest.raises(cos.CosError, match=r"^layer 'loss' \(ContrastiveLoss\): " + msg):
        cos.native_producer_plan(_loss_net(tmp_path, a, b, sim, nbottoms))


def test_contrastive_loss_accepts_nc11_bottoms(cos, tmp_path):
    text = cos.native_producer_plan(_loss_net(tmp_path, (4, 3, 1, 1), (4, 3, 1, 1), (4, 1, 1, 1)))
    assert _ops(text) == ["ContrastiveLoss loss 4x3x1x1 -> scalar"]
    assert text.splitlines()[3].endswith("margin=1 loss_weight=1 staged-bottom")
