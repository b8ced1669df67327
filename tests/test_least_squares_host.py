"""CPU tests of EuclideanLoss and Concat on the built-in engine: the plans of Caffe's least-squares solver-test net
(test_gradient_based_solver.cpp) and of its shared-weights variant, their learnable layout, Concat plans over several
axes and bottoms, and the refusals of both layers, which name the layer and use Caffe's CHECK wording."""
import pytest

from test_native_producer_host import _check_layout, _ops

N, C, H, W = 8, 3, 10, 10  # tests/golden/hdf5/solver_data.h5: data 8x3x10x10, targets 8x1
D = C * H * W
FILLER = "weight_filler { type: 'gaussian' std: 1.0 } bias_filler { type: 'gaussian' std: 1.0 }"


def least_squares_net(share=False, rows=N):
    """The net of GradientBasedSolverTest::RunLeastSquaresSolver, with an Input layer of the fixture's shapes (`rows`
    of them) in place of HDF5Data.  share: the data is sliced in two, two InnerProducts share 'weights' and 'bias', and
    a Concat joins their outputs again."""
    text = ("name: 'TestNetwork' "
            f"layer {{ name: 'data' type: 'Input' top: 'data' top: 'targets' input_param {{ "
            f"shape {{ dim: {rows} dim: {C} dim: {H} dim: {W} }} shape {{ dim: {rows} dim: 1 }} }} }} ")
    if share:
        text += ("layer { name: 'slice' type: 'Slice' bottom: 'data' top: 'data1' top: 'data2' "
                 "slice_param { axis: 0 } } ")
    text += ("layer { name: 'innerprod' type: 'InnerProduct' param { name: 'weights' } param { name: 'bias' } "
             f"inner_product_param {{ num_output: 1 {FILLER} }} "
             f"bottom: '{'data1' if share else 'data'}' top: '{'innerprod1' if share else 'innerprod'}' }} ")
    if share:
        text += ("layer { name: 'innerprod2' type: 'InnerProduct' param { name: 'weights' } param { name: 'bias' } "
                 f"inner_product_param {{ num_output: 1 {FILLER} }} bottom: 'data2' top: 'innerprod2' }} "
                 "layer { name: 'concat' type: 'Concat' bottom: 'innerprod1' bottom: 'innerprod2' top: 'innerprod' "
                 "concat_param { axis: 0 } } ")
    return text + "layer { name: 'loss' type: 'EuclideanLoss' bottom: 'innerprod' bottom: 'targets' }\n"


def write_solver(tmp_path, share=False, lr=1.0, weight_decay=0.0, momentum=0.0, solver_type=None, iter_size=1,
                 extra=""):
    """A solver over least_squares_net with the reference's fixed policy and the given constants; with iter_size k
    each pass reads N / k rows, as the reference's accumulation tests set batch_size."""
    (tmp_path / "net.prototxt").write_text(least_squares_net(share, N // iter_size))
    text = (f'net: "net.prototxt"\nbase_lr: {lr!r}\nlr_policy: "fixed"\nweight_decay: {weight_decay!r}\n'
            f'momentum: {momentum!r}\niter_size: {iter_size}\nrandom_seed: 1701\n'
            f'snapshot_prefix: "{tmp_path}/snap"\n' + (f'type: "{solver_type}"\n' if solver_type else "") + extra)
    (tmp_path / "solver.prototxt").write_text(text)
    return str(tmp_path / "solver.prototxt")


def test_plan_of_the_least_squares_net(cos, tmp_path):
    solver = write_solver(tmp_path)
    text = cos.native_producer_plan(solver)
    assert _ops(text) == [f"InnerProduct innerprod {N}x{C}x{H}x{W} -> {N}x1", f"EuclideanLoss loss {N}x1 -> scalar"]
    lines = [line for line in text.splitlines() if line.startswith("op ")]
    assert lines[0].endswith(f"w=0:{D} b={D}:1 staged-bottom")
    assert lines[1].endswith("second=1 loss_weight=1 staged-bottom")  # the targets are a staged input
    assert f"blob 0 0:{D} 1x{D} gaussian" in text and f"blob 1 {D}:1 1 gaussian" in text
    _check_layout(cos, text, solver, D + 1)
    assert cos.native_producer_plan(str(tmp_path / "net.prototxt")) == text


def test_plan_of_the_share_variant(cos, tmp_path):
    solver = write_solver(tmp_path, share=True)
    text = cos.native_producer_plan(solver)
    half = N // 2
    assert _ops(text) == [f"Slice slice {N}x{C}x{H}x{W} -> {half}x{C}x{H}x{W}"] * 2 + [
        f"InnerProduct innerprod {half}x{C}x{H}x{W} -> {half}x1",
        f"InnerProduct innerprod2 {half}x{C}x{H}x{W} -> {half}x1"] + [f"Concat concat {half}x1 -> {N}x1"] * 2 + [
        f"EuclideanLoss loss {N}x1 -> scalar"]
    lines = [line for line in text.splitlines() if line.startswith("op ")]
    assert lines[0].endswith("axis=0 begin=0 staged-bottom") and lines[1].endswith(f"axis=0 begin={half} staged-bottom")
    assert lines[2].endswith(f"w=0:{D} b={D}:1 no-bottom-grad")
    assert lines[3].endswith(f"w=0:{D} b={D}:1 shares=0,1 no-bottom-grad")  # the sharer uses the owner's offsets
    assert lines[4].endswith("axis=0 begin=0") and lines[5].endswith(f"axis=0 begin={half}")
    assert lines[6].endswith("loss_weight=1 staged-bottom")
    _check_layout(cos, text, solver, D + 1)  # 301 parameters in 2 blobs, as the plain net


def test_the_share_variant_resolves_to_the_plain_layout(cos, tmp_path):
    plain = cos.parse_solver(write_solver(tmp_path))
    (tmp_path / "s").mkdir()
    shared = cos.parse_solver(write_solver(tmp_path / "s", share=True))
    assert plain.counts == shared.counts == [D, 1] and plain.param_count == shared.param_count == 301
    assert plain.lr_mult == shared.lr_mult == [1.0, 1.0] and plain.decay_mult == shared.decay_mult == [1.0, 1.0]


def _write_concat(tmp_path, shapes, param, staged=(), target=None):
    """A Concat of one bottom per shape into a EuclideanLoss against a staged target of the given shape.  A bottom
    listed in `staged`, or of other than two axes, is a staged input; any other is the output of an InnerProduct (from
    a 3-wide input of its row count), so that it wants a gradient."""
    dims = lambda s: " ".join(f"dim: {d}" for d in s)  # noqa: E731
    tops, shapes_txt, layers, bottoms = [], [], [], []
    for i, s in enumerate(shapes):
        if i in staged or len(s) != 2:
            tops.append(f"x{i}")
            shapes_txt.append(dims(s))
            bottoms.append(f"x{i}")
        else:  # s = (rows, outputs): an InnerProduct from a 3-wide input
            tops.append(f"h{i}")
            shapes_txt.append(dims((s[0], 3)))
            layers.append(f"layer {{ name: 'ip{i}' type: 'InnerProduct' bottom: 'h{i}' top: 'y{i}' "
                          f"inner_product_param {{ num_output: {s[1]} }} }}")
            bottoms.append(f"y{i}")
    p = tmp_path / "net.prototxt"
    p.write_text("name: 't' layer { name: 'in' type: 'Input' " + " ".join(f"top: '{t}'" for t in tops) +
                 " top: 'target' input_param { " + " ".join(f"shape {{ {s} }}" for s in shapes_txt) +
                 f" shape {{ {dims(target)} }} }} }}\n" + "\n".join(layers) + "\n"
                 "layer { name: 'cat' type: 'Concat' " + " ".join(f"bottom: '{b}'" for b in bottoms) +
                 f" top: 'cat' {param} }}\n"
                 "layer { name: 'loss' type: 'EuclideanLoss' bottom: 'cat' bottom: 'target' top: 'loss' }\n")
    return str(p)


@pytest.mark.parametrize("shapes,param,staged,target,outs,begins,axis", [
    ([(2, 3), (5, 3)], "concat_param { axis: 0 }", (), (7, 3), "7x3", [0, 2], 0),
    ([(4, 2), (4, 3), (4, 1)], "", (1,), (4, 6), "4x6", [0, 2, 5], 1),  # the default axis 1, a staged middle bottom
    ([(4, 2), (4, 3)], "concat_param { axis: -1 }", (0,), (4, 5), "4x5", [0, 2], 1),
    ([(4, 2), (4, 3)], "concat_param { concat_dim: 1 }", (), (4, 5), "4x5", [0, 2], 1),
    ([(2, 3, 2), (2, 1, 2), (2, 2, 2)], "concat_param { axis: 1 }", (0, 1, 2), (2, 6, 2), "2x6x2", [0, 3, 4], 1),
])
def test_concat_plans(cos, tmp_path, shapes, param, staged, target, outs, begins, axis):
    text = cos.native_producer_plan(_write_concat(tmp_path, shapes, param, staged, target))
    lines = [line for line in text.splitlines() if line.startswith("op ") and " Concat " in line]
    assert [line.split()[4:7] for line in lines] == [["x".join(map(str, s)), "->", outs] for s in shapes]
    assert [int(line.split("begin=")[1].split()[0]) for line in lines] == begins
    assert all(f" axis={axis} " in line for line in lines)
    for i, line in enumerate(lines):  # no gradient flows into a staged bottom
        assert line.endswith("staged-bottom") == (i in staged or len(shapes[i]) != 2), line
    loss = next(line for line in text.splitlines() if " EuclideanLoss " in line)
    # the loss sends a gradient into the concat top when any bottom is learnable, never into the staged target
    assert loss.endswith("staged-bottom") != all(i in staged or len(s) != 2 for i, s in enumerate(shapes))


@pytest.mark.parametrize("shapes,param,msg", [
    ([(4, 2), (4, 3)], "concat_param { axis: 1 concat_dim: 1 }",
     r"Either axis or concat_dim should be specified; not both\."),
    ([(4, 2), (4, 3)], "concat_param { concat_dim: 2 }", r"concat_dim out of range\."),
    ([(4, 2), (4, 3)], "concat_param { axis: 2 }", r"axis 2 out of range for 2-D Blob"),
    ([(4, 2), (4, 3)], "concat_param { axis: -3 }", r"axis -3 out of range for 2-D Blob"),
    ([(4, 2), (4, 3, 1)], "", r"All inputs must have the same #axes\."),
    ([(4, 2), (5, 3)], "", r"All inputs must have the same shape, except at concat_axis\."),
    ([(4, 2, 2), (4, 2, 3)], "concat_param { axis: 1 }", r"All inputs must have the same shape, except at concat_axis\."),
])
def test_bad_concats_are_refused_with_the_layer_name(cos, tmp_path, shapes, param, msg):
    path = _write_concat(tmp_path, shapes, param, staged=tuple(range(len(shapes))), target=(4, 5))
    with pytest.raises(cos.CosError, match=r"^layer 'cat' \(Concat\): " + msg):
        cos.native_producer_plan(path)
    solver = tmp_path / "solver.prototxt"
    solver.write_text(f'net: "{path}"\nbase_lr: 0.1\nlr_policy: "fixed"\n')
    with pytest.raises(cos.CosError, match=r"layer 'cat' \(Concat\): " + msg):  # Caffe refuses the net itself
        cos.parse_solver(str(solver))


def _loss_net(tmp_path, a, b, extra_loss=False):
    dims = lambda s: " ".join(f"dim: {d}" for d in s)  # noqa: E731
    p = tmp_path / "net.prototxt"
    p.write_text("name: 't' layer { name: 'in' type: 'Input' top: 'x' top: 'b' top: 'label' input_param { "
                 f"shape {{ {dims((a[0], 3))} }} shape {{ {dims(b)} }} shape {{ dim: {a[0]} }} }} }}\n"
                 "layer { name: 'ip' type: 'InnerProduct' bottom: 'x' top: 'a' inner_product_param { "
                 f"num_output: {a[1]} }} }}\n"
                 + ("layer { name: 'ip_s' type: 'InnerProduct' bottom: 'b' top: 's' inner_product_param { "
                    "num_output: 4 } }\n"
                    "layer { name: 'soft' type: 'SoftmaxWithLoss' bottom: 's' bottom: 'label' top: 'soft' }\n"
                    if extra_loss else "")
                 + "layer { name: 'euc' type: 'EuclideanLoss' bottom: 'a' bottom: 'b' top: 'loss' }\n")
    return str(p)


@pytest.mark.parametrize("a,b,msg", [
    ((4, 2), (4, 3), r"Inputs must have the same dimension\."),
    ((4, 6), (4, 2, 2), r"Inputs must have the same dimension\."),
    ((4, 2), (3, 2), r"The data and label should have the same number\."),
    ((4, 2), (2, 4), r"The data and label should have the same number\."),  # num is checked first, as in Caffe
])
def test_euclidean_loss_bottom_checks(cos, tmp_path, a, b, msg):
    with pytest.raises(cos.CosError, match=r"^layer 'euc' \(EuclideanLoss\): " + msg):
        cos.native_producer_plan(_loss_net(tmp_path, a, b))


def test_euclidean_loss_accepts_equal_counts_of_other_shapes(cos, tmp_path):
    text = cos.native_producer_plan(_loss_net(tmp_path, (4, 6), (4, 3, 2)))  # count(1) is 6 in both
    loss = [line for line in text.splitlines() if " EuclideanLoss " in line]
    assert loss == ["op 1 EuclideanLoss euc 4x6 -> scalar second=1 loss_weight=1 staged-bottom"]


def test_euclidean_and_softmax_loss_is_a_second_loss(cos, tmp_path):
    with pytest.raises(cos.CosError, match=r"^layer 'euc' \(EuclideanLoss\): a second loss layer is not supported"):
        cos.native_producer_plan(_loss_net(tmp_path, (4, 3), (4, 3), extra_loss=True))


def test_euclidean_loss_with_a_loss_param_is_refused(cos, tmp_path):
    path = _loss_net(tmp_path, (4, 3), (4, 3))
    text = open(path).read().replace("top: 'loss' }", "top: 'loss' loss_param { normalize: false } }")
    open(path, "w").write(text)
    with pytest.raises(cos.CosError, match=r"^layer 'euc' \(EuclideanLoss\): loss_param"):
        cos.native_producer_plan(path)


def test_a_learnable_second_bottom_gets_a_gradient(cos, tmp_path):
    # both bottoms come out of InnerProducts: the loss sends +g into the first and -g into the second
    p = tmp_path / "net.prototxt"
    p.write_text("name: 't' layer { name: 'in' type: 'Input' top: 'x' top: 'z' input_param { shape { dim: 4 dim: 3 } "
                 "shape { dim: 4 dim: 5 } } }\n"
                 "layer { name: 'ip' type: 'InnerProduct' bottom: 'x' top: 'a' inner_product_param { num_output: 2 } }\n"
                 "layer { name: 'ip2' type: 'InnerProduct' bottom: 'z' top: 'b' inner_product_param { num_output: 2 } }\n"
                 "layer { name: 'euc' type: 'EuclideanLoss' bottom: 'a' bottom: 'b' loss_weight: 0.5 }\n")
    text = cos.native_producer_plan(str(p))
    loss = [line for line in text.splitlines() if " EuclideanLoss " in line]
    assert loss == ["op 2 EuclideanLoss euc 4x2 -> scalar second=3 loss_weight=0.5"]
