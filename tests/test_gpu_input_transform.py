"""The input transform on the GPU (DESIGN.md, "Input transform on the device"): cos_data_transform bit for bit against
the numpy restatement of data_transformer.cpp, the statistics of its draws, what train_raw hands the producer
(iter_size passes, ranks, snapshot and resume), the built-in engine trained through train_raw against train() on
pre-transformed batches, and the train-time refusals."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

from conftest import ROOT
from gpu_util import Ranks, assert_bits_equal, to_host
import transform_ref as T

pytestmark = pytest.mark.gpu

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")


def _kernel(x, fmt, crop=0, mirror=False, mean=None, mean_values=None, scale=1.0, k=0):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    if fmt == "u8":
        N, H, W, C = x.shape
    else:
        N, C, H, W = x.shape
    ho, wo = (crop, crop) if crop else (H, W)
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.full((N, C, ho, wo), float("nan"), device="cuda")
    md = torch.from_numpy(np.asarray(mean, np.float32)).cuda() if mean is not None else None
    mv = (ctypes.c_float * max(1, len(mean_values or [])))(*(mean_values or []))
    rc = L.cos_data_transform(xd.data_ptr(), 1 if fmt == "u8" else 0, N, C, H, W, out.data_ptr(), crop, int(mirror),
                              ctypes.cast(md.data_ptr(), ctypes.POINTER(ctypes.c_float)) if md is not None else None,
                              mv if mean_values else None, len(mean_values or []), scale, k, None)
    assert rc == 1, L.cos_last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _input(fmt, N, C, H, W, seed):
    rng = np.random.RandomState(seed)
    if fmt == "u8":
        return rng.randint(0, 256, (N, H, W, C)).astype(np.uint8)
    return (rng.randn(N, C, H, W) * 60).astype(np.float32)


GEOMETRIES = [  # name, N, C, H, W, crop, mirror, mean kind, scale
    ("caffenet", 4, 3, 256, 256, 227, True, "values", 1.0),
    ("cifar_mean_file", 5, 3, 32, 32, 0, False, "file", 1.0),
    ("lenet_scale", 7, 1, 28, 28, 0, False, None, 0.00390625),
    ("broadcast_value", 3, 3, 20, 20, 16, True, "one", 0.5),
    ("crop_equals_h", 3, 3, 17, 17, 17, True, "values", 1.0),
    ("odd_h_ne_w", 4, 3, 37, 53, 31, True, "file", 0.017),
    ("b1", 1, 3, 40, 40, 33, True, "values", 1.0),
    ("c1", 6, 1, 30, 30, 25, True, "file", 2.0),
]


@pytest.mark.parametrize("fmt", ["u8", "f32"])
@pytest.mark.parametrize("geo", GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_kernel_equals_restatement(fmt, geo):
    name, N, C, H, W, crop, mirror, mean_kind, scale = geo
    x = _input(fmt, N, C, H, W, 11)
    rng = np.random.RandomState(5)
    mean = (rng.rand(C * H * W) * 255).astype(np.float32) if mean_kind == "file" else None
    mv = {"values": [104.0, 117.0, 123.0][:C] if C == 3 else [99.5], "one": [77.25]}.get(mean_kind)
    for k in (T.key(3, 0, 0, it, 0) for it in range(4)):
        got = _kernel(x, fmt, crop, mirror, mean, mv, scale, k)
        want = T.transform(x, fmt, crop, mirror, mean, mv, scale, k)
        assert T.same_bits(got, want), f"{name} {fmt} key {k:#x}"


def test_nonfinite_and_subnormal_inputs_propagate():
    N, C, H, W = 2, 3, 9, 11
    x = _input("f32", N, C, H, W, 2)
    flat = x.reshape(-1)
    specials = np.array([np.nan, np.inf, -np.inf, 1e-40, -1e-40, 1.4e-45, 0.0, -0.0], np.float32)
    flat[::5] = np.resize(specials, flat[::5].size)
    mean = np.full(C * H * W, 1e-39, np.float32)
    for kw in (dict(mean=mean, scale=0.5), dict(mean_values=[np.inf, 0.0, -1e-40], scale=1.0),
               dict(scale=1e-3), dict(crop=7, mirror=True, mean_values=[2.0], scale=3.0)):
        for k in (1, 2, 3):
            got = _kernel(x, "f32", k=k, **kw)
            assert T.same_bits(got, T.transform(x, "f32", k=k, **kw)), kw


def test_draw_statistics_fixed_seed():
    """Per-image draws of the u8 path, recovered from the output: pixels hold their own row and column."""
    N, H, W, crop = 4096, 8, 8, 5
    x = np.empty((N, H, W, 2), np.uint8)
    x[..., 0] = np.arange(H, dtype=np.uint8)[None, :, None]
    x[..., 1] = np.arange(W, dtype=np.uint8)[None, None, :]
    mirrors, hist_h, hist_w = 0, np.zeros(H - crop + 1), np.zeros(W - crop + 1)
    keys = [T.key(1234, r, 0, it, 0) for r in range(2) for it in range(4)]
    for k in keys:
        out = _kernel(x, "u8", crop, True, k=k)
        h_off = out[:, 0, 0, 0].astype(int)
        step = out[:, 1, 0, 1] - out[:, 1, 0, 0]
        m = step < 0
        w_off = np.where(m, out[:, 1, 0, 0] - (crop - 1), out[:, 1, 0, 0]).astype(int)
        exp = [T.draws(k, n, H, W, crop, True) for n in range(0, N, 97)]  # spot check against the formula
        assert [(bool(m[n]), h_off[n], w_off[n]) for n in range(0, N, 97)] == exp
        mirrors += m.sum()
        hist_h += np.bincount(h_off, minlength=H - crop + 1)
        hist_w += np.bincount(w_off, minlength=W - crop + 1)
    total = N * len(keys)
    # binomial: 32768 fair draws, sd 90.5; 5 sd either side
    assert abs(mirrors - total / 2) < 5 * np.sqrt(total / 4), mirrors
    # chi-square with 3 degrees of freedom: 21.1 is its 0.01 % tail
    for hist in (hist_h, hist_w):
        e = total / hist.size
        assert ((hist - e) ** 2 / e).sum() < 21.1, hist


# ----------------------------------------------------------------------------------------------- train_raw
class _DevArray:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


class Recorder:
    """A producer that copies the device inputs it is handed (and adds no gradient).  The copies go into buffers
    allocated up front, so that a call never allocates while another in-process rank's sync kernel is waiting."""

    def __init__(self, net, ncalls=8, cap=400_000):
        self.bufs = [torch.empty(cap, device="cuda") for _ in range(ncalls)]
        self.calls = []
        net.set_forward_backward(self)

    def __call__(self, solver_index, ins, loss_dev, stream):
        buf, shapes, off = self.bufs[len(self.calls)], [], 0
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            for p, s in ins:
                n = int(np.prod(s))
                buf[off:off + n].copy_(torch.as_tensor(_DevArray(p, n), device="cuda"))
                shapes.append((off, s))
                off += n
            torch.as_tensor(_DevArray(loss_dev, 1), device="cuda").zero_()
        self.calls.append(shapes)
        return 0

    def host(self, i):
        torch.cuda.synchronize()
        b = self.bufs[i].cpu().numpy()
        return [b[off:off + int(np.prod(s))].reshape(s).copy() for off, s in self.calls[i]]


SMALL_NET = """name: "small"
layer {{ name: "data" type: "MemoryData" top: "data" top: "label"
  memory_data_param {{ batch_size: {N} channels: 3 height: {crop} width: {crop} }}
  transform_param {{ crop_size: {crop} mirror: true mean_value: 104 mean_value: 117 mean_value: 123 scale: 0.5 }} }}
layer {{ name: "ip" type: "InnerProduct" bottom: "data" top: "ip"
  inner_product_param {{ num_output: 4 weight_filler {{ type: "gaussian" std: 0.01 }} }} }}
layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }}
"""


def _solver(d, net_text, seed=7, iter_size=1, extra=""):
    (d / "net.prototxt").write_text(net_text)
    s = d / "solver.prototxt"
    s.write_text(f'net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\nmax_iter: 100\nmomentum: 0.9\n'
                 f'random_seed: {seed}\niter_size: {iter_size}\nsnapshot_prefix: "{d}/snap"\n{extra}')
    return str(s)


def _net(cos, solver, model="", state=""):
    net = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    return net


def _small(N=3, crop=9):
    return SMALL_NET.format(N=N, crop=crop), N, crop


MV = [104.0, 117.0, 123.0]


@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_caffenet_shaped_batch_reaches_the_producer(cos, fmt):
    """The golden CaffeNet net (b2, 256 -> 227, mirror, three mean values), seed 0 (no random_seed)."""
    net = _net(cos, os.path.join(CONFIGS, "bvlc_reference_solver.prototxt"))
    try:
        rec = Recorder(net)
        label = np.array([3, 1], np.float32)
        for t in range(3):
            x = _input(fmt, 2, 3, 256, 256, t)
            assert net.train_raw(0, [x, label]), net.last_error()
            got = rec.host(t)
            want = T.transform(x, fmt, 227, True, None, MV, 1.0, T.key(0, 0, 0, t, 0))
            assert T.same_bits(got[0], want), t
            assert_bits_equal(got[1].reshape(-1), label, "label")
    finally:
        net.deallocate()


def _cifar_dir(d, name="cifar10_quick"):
    for f in (f"{name}_solver.prototxt", f"{name}_train_test.prototxt"):
        shutil.copy(os.path.join(CONFIGS, f), d / f)
    mean = (np.random.RandomState(9).rand(3 * 32 * 32) * 255).astype(np.float32)
    (d / "mean.binaryproto").write_bytes(T.blobproto(mean, legacy=(1, 3, 32, 32)))
    return str(d / f"{name}_solver.prototxt"), mean


def _cifar_batch(seed, N=100):
    rng = np.random.RandomState(seed)
    return rng.randint(0, 256, (N, 32, 32, 3)).astype(np.uint8), rng.randint(0, 10, N).astype(np.float32)


def test_cifar10_quick_mean_file_reaches_the_producer(cos, tmp_path):
    solver, mean = _cifar_dir(tmp_path)
    net = _net(cos, solver)
    try:
        rec = Recorder(net)
        for t in range(2):
            x, y = _cifar_batch(t)
            assert net.train_raw(0, [x, y]), net.last_error()
            got = rec.host(t)
            assert T.same_bits(got[0], T.transform(x, "u8", mean=mean)), t
            assert_bits_equal(got[1].reshape(-1), y, "label")
    finally:
        net.deallocate()


def test_iter_size_passes_draw_differently(cos, tmp_path):
    text, N, crop = _small()
    net = _net(cos, _solver(tmp_path, text, seed=11, iter_size=2))
    try:
        rec = Recorder(net)
        x = _input("u8", N, 3, 16, 16, 4)
        y = np.zeros(N, np.float32)
        for t in range(2):
            assert net.train_raw(0, [x, y]), net.last_error()
        assert len(rec.calls) == 4
        for t in range(2):
            outs = [rec.host(2 * t + p)[0] for p in range(2)]
            for p in range(2):
                assert T.same_bits(outs[p], T.transform(x, "u8", crop, True, None, MV, 0.5, T.key(11, 0, 0, t, p)))
            assert not np.array_equal(outs[0], outs[1])
    finally:
        net.deallocate()


def test_two_ranks_draw_differently(cos, tmp_path):
    text, N, crop = _small()
    R = Ranks(cos, _solver(tmp_path, text, seed=5), 2, timeout_ms=20000)
    try:
        R.connect()
        recs = [Recorder(n) for n in R.nets]
        x = _input("u8", N, 3, 16, 16, 6)
        y = np.zeros(N, np.float32)
        for t in range(2):
            for net in R.nets:
                assert net.train_raw(0, [x, y]), net.last_error()
            for net in R.nets:
                assert net.synchronize(), net.last_error()
        for t in range(2):
            outs = [recs[r].host(t)[0] for r in range(2)]
            for r in range(2):
                assert T.same_bits(outs[r], T.transform(x, "u8", crop, True, None, MV, 0.5, T.key(5, r, 0, t, 0)))
            assert not np.array_equal(outs[0], outs[1])
    finally:
        R.close()


def test_resume_from_snapshot_draws_as_the_uninterrupted_run(cos, tmp_path):
    text, N, crop = _small()
    solver = _solver(tmp_path, text, seed=3)
    xs = [_input("u8", N, 3, 16, 16, 20 + t) for t in range(4)]
    y = np.zeros(N, np.float32)
    net = _net(cos, solver)
    try:
        rec = Recorder(net)
        for t in range(4):
            assert net.train_raw(0, [xs[t], y]), net.last_error()
            if t == 1:
                assert net.synchronize()
                assert net.snapshot() >= 0, net.last_error()
        whole = [rec.host(t)[0] for t in range(4)]
    finally:
        net.deallocate()
    model, state = str(tmp_path / "snap_iter_2.caffemodel"), str(tmp_path / "snap_iter_2.solverstate")
    assert os.path.exists(model) and os.path.exists(state)
    net = _net(cos, solver, model, state)
    try:
        assert net.iter() == 2
        rec = Recorder(net)
        for t in (2, 3):
            assert net.train_raw(0, [xs[t], y]), net.last_error()
        for t in (2, 3):
            got = rec.host(t - 2)[0]
            assert T.same_bits(got, whole[t]), t
            assert T.same_bits(got, T.transform(xs[t], "u8", crop, True, None, MV, 0.5, T.key(3, 0, 0, t, 0)))
    finally:
        net.deallocate()


@pytest.mark.parametrize("which", ["cifar10_quick", "lenet_memory"])
def test_engine_trained_by_train_raw_equals_train_on_restated_batches(cos, tmp_path, which):
    if which == "cifar10_quick":
        solver, mean = _cifar_dir(tmp_path)
        batches = [_cifar_batch(10 + t) for t in range(4)]
        restate = lambda x: T.transform(x, "u8", mean=mean)  # noqa: E731
    else:
        solver = os.path.join(CONFIGS, "lenet_memory_solver.prototxt")
        rng = np.random.RandomState(1)
        batches = [(rng.randint(0, 256, (64, 28, 28, 1)).astype(np.uint8), rng.randint(0, 10, 64).astype(np.float32))
                   for _ in range(4)]
        restate = lambda x: T.transform(x, "u8", scale=0.00390625)  # noqa: E731
    nets = [_net(cos, solver), _net(cos, solver)]
    try:
        for n in nets:
            n.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        assert_bits_equal(to_host(nets[0].data()), to_host(nets[1].data()), "initial weights")
        for x, y in batches:
            assert nets[0].train_raw(0, [x, y]), nets[0].last_error()
            assert nets[1].train(0, [restate(x), y]), nets[1].last_error()
        for n in nets:
            assert n.synchronize(), n.last_error()
        w = [to_host(n.data()) for n in nets]
        assert_bits_equal(w[0], w[1], f"{which} weights after train_raw vs train")
        assert np.isfinite(w[0]).all()
    finally:
        for n in nets:
            n.deallocate()


def test_train_time_refusals_then_a_valid_call(cos, tmp_path):
    from caffeonspark_b200 import _lib, nets as N_
    L = _lib.lib()
    desc_net = cos.CaffeNet(N_.solver_desc("lenet"))
    try:
        assert desc_net.connect(desc_net.localAddresses())
        Recorder(desc_net)
        assert not desc_net.train_raw(0, [np.zeros((64, 28, 28, 1), np.uint8), np.zeros(64, np.float32)])
        assert "layout descriptor" in desc_net.last_error()
    finally:
        desc_net.deallocate()
    text = SMALL_NET.format(N=3, crop=9).replace(
        "mean_value: 104 mean_value: 117 mean_value: 123", 'mean_file: "m.binaryproto"')
    (tmp_path / "m.binaryproto").write_bytes(T.blobproto(np.ones(3 * 12 * 12, np.float32), shape=(1, 3, 12, 12)))
    net = _net(cos, _solver(tmp_path, text))
    try:
        rec = Recorder(net)
        x, y = _input("u8", 3, 3, 12, 12, 1), np.zeros(3, np.float32)
        bad = [
            ([x], "1 blobs for the net's 2 staged inputs"),
            ([x[..., :2].copy(), y], "channels == img_channels"),
            ([_input("u8", 3, 3, 8, 12, 1), y], "img_height >= crop_size"),
            ([_input("u8", 3, 3, 14, 14, 1), y], "data_mean_.height()"),
            ([x, np.zeros((3, 2), np.float32)], "without transform_param must be COS_RAW_F32_NCHW"),
            ([x, np.zeros(3, np.uint8).reshape(3, 1, 1, 1)], "without transform_param must be COS_RAW_F32_NCHW"),
        ]
        for arrays, msg in bad:
            assert not net.train_raw(0, arrays), msg
            assert msg in net.last_error() and "layer 'data'" in net.last_error() or msg.startswith("1 blobs"), \
                (msg, net.last_error())
        with pytest.raises(cos.CosError):
            net.train_raw(0, [x.astype(np.float64), y])
        blobs = (_lib.cos_raw_blob * 2)()
        for i, a in enumerate((x, y)):
            blobs[i].data, blobs[i].num, blobs[i].channels = a.ctypes.data, 3, 3 if i == 0 else 1
            blobs[i].format, blobs[i].height, blobs[i].width = (1, 12, 12) if i == 0 else (0, 1, 1)
        blobs[0].format = 5
        assert L.cos_net_train_raw(net._h, 0, blobs, 2) == 0 and b"format 5" in L.cos_last_error()
        blobs[0].format, blobs[0].data = 1, None
        assert L.cos_net_train_raw(net._h, 0, blobs, 2) == 0 and b"NULL" in L.cos_last_error()
        assert L.cos_net_train_raw(net._h, 1, blobs, 2) == 0
        assert len(rec.calls) == 0
        assert net.train_raw(0, [x, y]), net.last_error()  # a valid call after every refusal
        assert T.same_bits(rec.host(0)[0], T.transform(x, "u8", 9, True, np.ones(3 * 12 * 12), None, 0.5,
                                                       T.key(7, 0, 0, 0, 0)))
        # later calls must keep the first call's raw shapes
        x16 = _input("u8", 3, 3, 12, 12, 2).astype(np.float32).transpose(0, 3, 1, 2).copy()
        assert not net.train_raw(0, [x16, y]) and "differs from the first call's" in net.last_error()
        assert net.train_raw(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()
    finally:
        net.deallocate()
