"""Host-only checks of the input transform (DESIGN.md, "Input transform on the device"): the parser's transform_param
record and its plan lines, mean files in both BlobProto shape encodings and their path resolution, every refusal the
plan makes, the entry points' argument checks, and the restatement's draws."""
import ctypes
import os
import re
import shutil

import numpy as np
import pytest

from conftest import ROOT
import transform_ref as T

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")


def _plan(cos, path):
    return cos.input_transform_plan(str(path))


def _copy_cifar(tmp_path, name, mean_bytes=None):
    """The golden CIFAR-10 solver and net in tmp_path, next to a test-written mean.binaryproto."""
    for f in (f"{name}_solver.prototxt", f"{name}_train_test.prototxt"):
        shutil.copy(os.path.join(CONFIGS, f), tmp_path / f)
    mean = np.arange(3 * 32 * 32, dtype=np.float32) / 7.0
    (tmp_path / "mean.binaryproto").write_bytes(mean_bytes or T.blobproto(mean, shape=(1, 3, 32, 32)))
    return tmp_path / f"{name}_solver.prototxt"


def _solver(tmp_path, net_text, name="net.prototxt"):
    (tmp_path / name).write_text(net_text)
    s = tmp_path / ("solver_" + name)
    s.write_text(f'net: "{tmp_path / name}"\nbase_lr: 0.01\nlr_policy: "fixed"\nmax_iter: 10\n')
    return s


def _net(transform, channels=3, height=32, width=32, batch=4):
    return f"""name: "t"
layer {{ name: "data" type: "MemoryData" top: "data" top: "label"
  memory_data_param {{ batch_size: {batch} channels: {channels} height: {height} width: {width} }}
  {transform} }}
layer {{ name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param {{ num_output: 10 }} }}
layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }}
"""


def test_plan_lines_of_the_golden_configs(cos, tmp_path):
    caffenet = _plan(cos, os.path.join(CONFIGS, "bvlc_reference_solver.prototxt")).splitlines()
    assert caffenet == ["input 0 data layer=data shape=2x3x227x227 scale=1 mirror=1 crop=227 mean=values:104,117,123",
                        "input 1 label layer=data shape=2 transform=none"]
    lenet = _plan(cos, os.path.join(CONFIGS, "lenet_memory_solver.prototxt")).splitlines()
    assert lenet == ["input 0 data layer=data shape=64x1x28x28 scale=0.00390625 mirror=0 crop=0 mean=none",
                     "input 1 label layer=data shape=64 transform=none"]
    cos_data = _plan(cos, os.path.join(CONFIGS, "lenet_cos_solver.prototxt")).splitlines()  # per-top CoSData
    assert cos_data == ["input 0 data layer=data shape=64x1x28x28 scale=0.00390625 mirror=0 crop=0 mean=none",
                        "input 1 label layer=data shape=64x1x1x1 transform=none"]
    for name, batch in (("cifar10_quick", 100), ("cifar10_full", 100)):
        d = tmp_path / name
        d.mkdir()
        lines = _plan(cos, _copy_cifar(d, name)).splitlines()
        assert len(lines) == 2, lines
        m = re.fullmatch(rf"input 0 data layer=\S+ shape={batch}x3x32x32 scale=1 mirror=0 crop=0 "
                         r"mean=file:(\S+)\[3x32x32\]", lines[0])
        assert m and os.path.samefile(m.group(1), d / "mean.binaryproto"), lines[0]
        assert lines[1].endswith("transform=none")


def _strip_transform(text):
    return re.sub(r"transform_param\s*\{[^{}]*\}", "", text)


@pytest.mark.parametrize("solver", ["bvlc_reference_solver", "cifar10_quick_solver", "cifar10_full_solver",
                                    "lenet_memory_solver", "lenet_cos_solver"])
def test_transform_param_leaves_the_layout_alone(cos, tmp_path, solver):
    src = os.path.join(CONFIGS, solver + ".prototxt")
    net = re.search(r'^\s*net:\s*"([^"]+)"', open(src).read(), re.M).group(1)
    text = open(os.path.join(CONFIGS, os.path.basename(net))).read()
    assert "transform_param" in text
    stripped = _strip_transform(text)
    assert "transform_param" not in stripped
    with_t = cos.parse_solver(_solver(tmp_path, text, "with.prototxt"))
    without = cos.parse_solver(_solver(tmp_path, stripped, "without.prototxt"))
    assert with_t.counts == without.counts and len(with_t.counts) > 0
    assert with_t.lr_mult == without.lr_mult and with_t.decay_mult == without.decay_mult


@pytest.mark.parametrize("encoding", ["shape", "legacy"])
def test_mean_file_in_both_shape_encodings(cos, tmp_path, encoding):
    mean = np.linspace(-3, 5, 2 * 5 * 6).astype(np.float32)
    kw = {"shape": (1, 2, 5, 6)} if encoding == "shape" else {"legacy": (1, 2, 5, 6)}
    (tmp_path / "m.binaryproto").write_bytes(T.blobproto(mean, **kw))
    s = _solver(tmp_path, _net('transform_param { mean_file: "m.binaryproto" scale: 0.5 }', 2, 5, 6))
    line = _plan(cos, s).splitlines()[0]
    assert line.endswith("scale=0.5 mirror=0 crop=0 mean=file:" + str(tmp_path / "m.binaryproto") + "[2x5x6]"), line


def test_relative_mean_file_resolution(cos, tmp_path):
    sub = tmp_path / "nets"
    sub.mkdir()
    (sub / "mean.binaryproto").write_bytes(T.blobproto(np.zeros(3 * 32 * 32, np.float32), shape=(1, 3, 32, 32)))
    # next to the net file
    s = _solver(sub, _net('transform_param { mean_file: "mean.binaryproto" }'))
    assert "mean=file:" + str(sub / "mean.binaryproto") in _plan(cos, s)
    # by its basename next to the net file
    s = _solver(sub, _net('transform_param { mean_file: "examples/cifar10/mean.binaryproto" }'), "b.prototxt")
    assert "mean=file:" + str(sub / "mean.binaryproto") in _plan(cos, s)
    # an absolute path as given
    s = _solver(tmp_path, _net(f'transform_param {{ mean_file: "{sub / "mean.binaryproto"}" }}'), "c.prototxt")
    assert "mean=file:" + str(sub / "mean.binaryproto") in _plan(cos, s)


def test_golden_cifar_configs_still_parse_without_their_mean_file(cos):
    for name in ("cifar10_quick_solver", "cifar10_full_solver"):
        path = os.path.join(CONFIGS, name + ".prototxt")
        assert len(cos.parse_solver(path).counts) > 0
        assert cos.native_producer_plan(path)
        with pytest.raises(cos.CosError,
                           match=r"layer '\w+' \(MemoryData\), top 'data': cannot open mean_file 'mean.binaryproto'"):
            _plan(cos, path)


REFUSALS = [
    ('transform_param { mean_file: "m.binaryproto" mean_value: 1 }', 3, 32, None,
     "Cannot specify mean_file and mean_value at the same time"),
    ("transform_param { mean_value: 1 mean_value: 2 }", 3, 32, None, "Specify either 1 mean_value or as many as "
     "channels: 3"),
    ('transform_param { mean_file: "missing.binaryproto" }', 3, 32, None, "cannot open mean_file"),
    ('transform_param { mean_file: "m.binaryproto" }', 3, 32, b"\xff\xff\xff\xff", "is not a BlobProto"),
    ('transform_param { mean_file: "m.binaryproto" }', 3, 32, ("legacy", (2, 3, 32, 32)), "has num 2; it must be 1"),
    ('transform_param { mean_file: "m.binaryproto" }', 3, 32, ("shape", (1, 1, 32, 32)), "has 1 channels, the top 3"),
    ("transform_param { crop_size: 28 }", 3, 32, None, "crop_size 28 must equal the top's height and width"),
]


@pytest.mark.parametrize("transform,channels,hw,mean,msg", REFUSALS)
def test_plan_refusals_name_the_layer(cos, tmp_path, transform, channels, hw, mean, msg):
    if mean is None:
        mean = ("shape", (1, 3, 32, 32))
    if isinstance(mean, bytes):
        (tmp_path / "m.binaryproto").write_bytes(mean)
    else:
        enc, shape = mean
        (tmp_path / "m.binaryproto").write_bytes(T.blobproto(np.zeros(int(np.prod(shape)), np.float32),
                                                             **{enc: shape}))
    s = _solver(tmp_path, _net(transform, channels, hw, hw))
    with pytest.raises(cos.CosError) as e:
        _plan(cos, s)
    assert "layer 'data' (MemoryData), top 'data'" in str(e.value) and msg in str(e.value), str(e.value)
    assert len(cos.parse_solver(s).counts) == 2  # never refused at parse time


def test_entry_points_survive_null_and_garbage(cos, tmp_path):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert L.cos_net_train_raw(None, 0, None, 0) == 0 and b"NULL" in L.cos_last_error()
    blob = _lib.cos_raw_blob()
    assert L.cos_net_train_raw(None, 0, ctypes.byref(blob), 1) == 0
    assert L.cos_input_transform_plan(None, None, 0) == -1
    assert L.cos_input_transform_plan(b"/nonexistent/solver.prototxt", None, 0) == -1
    garbage = tmp_path / "garbage.prototxt"
    garbage.write_bytes(b"layer { transform_param { mean_value: } \x00\xff")
    assert L.cos_input_transform_plan(str(garbage).encode(), None, 0) == -1
    mv = (ctypes.c_float * 4)(1, 2, 3, 4)
    fake = ctypes.c_void_p(16)  # never dereferenced: every call below is refused before a launch
    bad = [
        (None, 1, 1, 3, 8, 8, fake, 0, 0, None, None, 0),       # NULL input
        (fake, 1, 1, 3, 8, 8, None, 0, 0, None, None, 0),       # NULL output
        (fake, 7, 1, 3, 8, 8, fake, 0, 0, None, None, 0),       # bad format
        (fake, 0, 0, 3, 8, 8, fake, 0, 0, None, None, 0),       # num 0
        (fake, 0, 1, 3, 8, 8, fake, 9, 0, None, None, 0),       # crop > height
        (fake, 0, 1, 3, 8, 8, fake, -1, 0, None, None, 0),      # negative crop
        (fake, 0, 1, 3, 8, 8, fake, 0, 0, fake, mv, 3),         # mean and mean values
        (fake, 0, 1, 3, 8, 8, fake, 0, 0, None, mv, 2),         # 2 mean values for 3 channels
        (fake, 0, 1, 3, 8, 8, fake, 0, 0, None, None, 3),       # NULL mean values
        (fake, 1, 1, 3, 8, 20000, fake, 0, 0, None, None, 0),   # u8 row beyond shared memory
    ]
    for args in bad:
        a = list(args)
        mean = ctypes.cast(a[9], ctypes.POINTER(ctypes.c_float)) if a[9] is not None else None
        rc = L.cos_data_transform(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], mean, a[10], a[11],
                                  1.0, 0, None)
        assert rc == 0, args
        assert L.cos_last_error().startswith(b"cos_data_transform: "), (args, L.cos_last_error())


def test_draws_match_hand_computed_mix64():
    # splitmix64 from state 0: the first outputs are mix64(phi), mix64(2 phi), mix64(3 phi)
    assert T.mix64(T.PHI) == 0xE220A8397B1DCDAF
    assert T.mix64(2 * T.PHI) == 0x6E789E6AA1B965F4
    assert T.mix64(3 * T.PHI) == 0x06C45D188009454F
    assert T.mix64(0) == 0
    k = T.key(0, 0, 0, 0, 0)  # seed 0, rank 0: mix64 of 0 four times over
    assert k == 0
    assert T.key(-1, 0, 0, 0, 0) == T.key(0, 0, 0, 0, 0)  # a negative seed counts as 0, as for the fillers
    k = T.key(7, 1, 0, 3, 1)
    assert k == T.mix64(T.mix64(T.mix64(T.mix64(7 * T.PHI + 1) + 0) + 3) + 1)
    # draw (n, j) hashes key + (4n + j) phi: image 0's mirror draw of key 0 is mix64(0) >> 32 = 0
    assert T.draw(0, 0, 0, 2) == 0
    assert T.draw(0, 0, 1, 30) == (0xE220A8397B1DCDAF >> 32) % 30
    assert T.draw(0, 0, 2, 30) == (0x6E789E6AA1B965F4 >> 32) % 30
    assert T.draw(0, 1, 0, 2) == (T.mix64(4 * T.PHI) >> 32) % 2
    assert T.draws(0, 0, 32, 32, 0, False) == (False, 0, 0)  # no crop, no mirror: nothing drawn


def test_restatement_follows_caffe_on_a_hand_example():
    x = np.arange(2 * 3 * 4, dtype=np.uint8).reshape(1, 3, 4, 2)  # 1 image, H 3, W 4, C 2 interleaved
    out = T.transform(x, "u8", mean_values=[1.0], scale=2.0)
    assert out.shape == (1, 2, 3, 4)
    assert np.array_equal(out[0, 1, 2], (x[0, 2, :, 1].astype(np.float32) - 1) * 2)
    k = next(k for k in range(100) if T.draws(k, 0, 3, 4, 2, True)[0])  # a key that mirrors image 0
    m, h0, w0 = T.draws(k, 0, 3, 4, 2, True)
    out = T.transform(x, "u8", crop=2, mirror=True, k=k)
    assert np.array_equal(out[0, 0, :, 0], x[0, h0:h0 + 2, w0 + 1, 0].astype(np.float32))  # column 0 <- column 1
