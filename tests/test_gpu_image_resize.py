"""Ragged 8-bit images on the GPU (DESIGN.md, "Images of any size"): cos_image_transform bit for bit against the resize
restatement (resize_ref.py) followed by the transform restatement (transform_ref.py), what train_raw(list of images)
hands the recording producer, the PyTorch producer and the built-in engine, iter_size passes, snapshot and resume,
arena growth, and every train-time refusal followed by a valid call."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
import resize_ref as R
import transform_ref as T
from test_gpu_input_transform import MV, SMALL_NET, Recorder, _cifar_dir, _net, _solver

pytestmark = pytest.mark.gpu

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")


def restate(images, target=None, crop=0, mirror=False, mean=None, mean_values=None, scale=1.0, k=0, out_hw=None):
    """resize_ref then transform_ref, image by image, with image n's draws taken on its post-resize size."""
    outs = []
    for n, img in enumerate(images):
        img = img if img.ndim == 3 else img[:, :, None]
        r = R.resize(img, *target) if target else img
        Hr, Wr, C = r.shape
        m, h_off, w_off = T.draws(k, n, Hr, Wr, crop, mirror)
        ho, wo = (crop, crop) if crop else (out_hw or (Hr, Wr))
        chw = np.ascontiguousarray(r.transpose(2, 0, 1)).astype(np.float32)
        outs.append(T._one(chw, mean, mean_values, scale, h_off, w_off, ho, wo, m))
    return np.stack(outs)


def _images(sizes, C, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, (h, w, C)).astype(np.uint8) for h, w in sizes]


def _kernel(images, target=None, crop=0, mirror=False, mean=None, mean_hw=(0, 0), mean_values=None, scale=1.0, k=0,
            out_hw=None):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    N, C = len(images), images[0].shape[2]
    geom = (_lib.cos_image_geometry * N)()
    off, blobs = 0, []
    for n, img in enumerate(images):
        geom[n].offset, geom[n].height, geom[n].width = off, img.shape[0], img.shape[1]
        blobs.append(img.reshape(-1))
        off += img.size
    arena = torch.from_numpy(np.concatenate(blobs)).cuda()
    gd = torch.frombuffer(bytearray(bytes(geom)), dtype=torch.uint8).cuda()
    ho, wo = (crop, crop) if crop else (out_hw or target)
    out = torch.full((N, C, ho, wo), -7.0, device="cuda")
    md = torch.from_numpy(np.asarray(mean, np.float32)).cuda() if mean is not None else None
    mv = (ctypes.c_float * max(1, len(mean_values or [])))(*(mean_values or []))
    th, tw = target or (0, 0)
    rc = L.cos_image_transform(arena.data_ptr(), ctypes.cast(gd.data_ptr(), ctypes.POINTER(_lib.cos_image_geometry)),
                               N, C, th, tw, out.data_ptr(), ho, wo, crop, int(mirror),
                               ctypes.cast(md.data_ptr(), ctypes.POINTER(ctypes.c_float)) if md is not None else None,
                               mean_hw[0], mean_hw[1], mv if mean_values else None, len(mean_values or []), scale, k,
                               None)
    assert rc == 1, L.cos_last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy()


RAGGED = [(375, 500), (500, 375), (333, 500), (257, 300), (240, 320), (300, 241)]
KERNEL_CASES = [  # name, sizes, C, target, crop, mirror, mean kind, scale
    ("resize_crop_mirror_values", RAGGED, 3, (256, 256), 227, True, "values", 1.0),
    ("resize_to_crop", RAGGED, 3, (227, 227), 227, True, "values", 1.0),
    ("no_resize_crop", RAGGED, 3, None, 227, True, "values", 1.0),
    ("resize_mean_file", [(37, 53), (20, 20), (64, 31), (9, 9)], 3, (32, 32), 0, False, "file", 1.0),
    ("resize_crop_mean_file", [(37, 53), (20, 20), (64, 31)], 3, (32, 30), 27, True, "file", 0.017),
    ("upscale_gray", [(7, 5), (1, 1), (28, 28), (3, 40)], 1, (28, 28), 0, False, None, 0.00390625),
    ("four_channels_one_value", [(50, 60), (61, 45), (33, 33)], 4, (40, 44), 31, True, "one", 0.5),
    ("equal_size", [(32, 32), (32, 32)], 3, (32, 32), 0, True, "values", 1.0),
]


@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_kernel_equals_restatement(case):
    name, sizes, C, target, crop, mirror, mean_kind, scale = case
    images = _images(sizes, C, 11)
    post = target or sizes[0]
    mean = (np.random.RandomState(5).rand(C * post[0] * post[1]) * 255).astype(np.float32) \
        if mean_kind == "file" else None
    mv = {"values": [104.0, 117.0, 123.0][:C], "one": [77.25]}.get(mean_kind)
    for k in (T.key(3, 0, 0, it, 0) for it in range(3)):
        got = _kernel(images, target, crop, mirror, mean, post if mean is not None else (0, 0), mv, scale, k)
        want = restate(images, target, crop, mirror, mean, mv, scale, k)
        assert T.same_bits(got, want), f"{name} key {k:#x}"


def test_kernel_fills_an_image_it_cannot_take_with_nan():
    images = _images([(40, 40), (20, 40), (40, 40)], 3, 2)  # image 1 is below the crop
    got = _kernel(images, None, 31, True, mean_values=MV, k=5)
    assert np.isnan(got[1]).all() and np.isfinite(got[[0, 2]]).all()
    want = restate([images[0], images[2]], None, 31, True, None, MV, 1.0, 5)
    assert T.same_bits(got[0], want[0])


# ----------------------------------------------------------------------------------------------- train_raw
def test_caffenet_shaped_ragged_batch_reaches_the_producer(cos):
    """The golden CaffeNet net (b2, crop 227, mirror, three mean values): ImageNet-sized images resized to 256 x 256
    and, without a resize, cropped from their own sizes."""
    label = np.array([3, 1], np.float32)
    # the target repeats from call to call, so each target runs on its own net
    runs = [((256, 256), [[(375, 500), (500, 333)], [(480, 640), (256, 256)]]),
            (None, [[(227, 300), (260, 229)], [(500, 375), (240, 320)]])]
    for target, calls in runs:
        net = _net(cos, os.path.join(CONFIGS, "bvlc_reference_solver.prototxt"))
        try:
            rec = Recorder(net)
            for t, sizes in enumerate(calls):
                images = _images(sizes, 3, t)
                assert net.train_raw(0, [images, label], resize=target), net.last_error()
                got = rec.host(t)
                want = restate(images, target, 227, True, None, MV, 1.0, T.key(0, 0, 0, t, 0))
                assert T.same_bits(got[0], want), (target, t)
                assert_bits_equal(got[1].reshape(-1), label, "label")
        finally:
            net.deallocate()


def _cifar_images(seed, N=100):
    rng = np.random.RandomState(seed)
    sizes = [(int(rng.randint(8, 70)), int(rng.randint(8, 70))) for _ in range(N)]
    return _images(sizes, 3, seed), rng.randint(0, 10, N).astype(np.float32)


def test_cifar10_quick_mean_file_and_resize_reach_the_producer(cos, tmp_path):
    solver, mean = _cifar_dir(tmp_path)
    net = _net(cos, solver)
    try:
        rec = Recorder(net)
        for t in range(2):
            x, y = _cifar_images(t)
            assert net.train_raw(0, [x, y], resize=(32, 32)), net.last_error()
            got = rec.host(t)
            assert T.same_bits(got[0], restate(x, (32, 32), mean=mean)), t
            assert_bits_equal(got[1].reshape(-1), y, "label")
    finally:
        net.deallocate()


def test_iter_size_passes_draw_differently(cos, tmp_path):
    net = _net(cos, _solver(tmp_path, SMALL_NET.format(N=3, crop=9), seed=11, iter_size=2))
    try:
        rec = Recorder(net)
        x = _images([(16, 20), (31, 12), (9, 9)], 3, 4)
        y = np.zeros(3, np.float32)
        for t in range(2):
            assert net.train_raw(0, [x, y], resize=(14, 15)), net.last_error()
        assert len(rec.calls) == 4
        for t in range(2):
            outs = [rec.host(2 * t + p)[0] for p in range(2)]
            for p in range(2):
                assert T.same_bits(outs[p], restate(x, (14, 15), 9, True, None, MV, 0.5, T.key(11, 0, 0, t, p)))
            assert not np.array_equal(outs[0], outs[1])
    finally:
        net.deallocate()


def test_resume_from_snapshot_draws_as_the_uninterrupted_run(cos, tmp_path):
    solver = _solver(tmp_path, SMALL_NET.format(N=3, crop=9), seed=3)
    xs = [_images([(10 + t, 12), (9, 30 - t), (20, 11)], 3, 20 + t) for t in range(4)]
    y = np.zeros(3, np.float32)
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
    net = _net(cos, solver, str(tmp_path / "snap_iter_2.caffemodel"), str(tmp_path / "snap_iter_2.solverstate"))
    try:
        assert net.iter() == 2
        rec = Recorder(net)
        for t in (2, 3):
            assert net.train_raw(0, [xs[t], y]), net.last_error()
        for t in (2, 3):
            got = rec.host(t - 2)[0]
            assert T.same_bits(got, whole[t]), t
            assert T.same_bits(got, restate(xs[t], None, 9, True, None, MV, 0.5, T.key(3, 0, 0, t, 0)))
    finally:
        net.deallocate()


def test_a_later_larger_batch_grows_the_arena(cos, tmp_path):
    net = _net(cos, _solver(tmp_path, SMALL_NET.format(N=3, crop=9), seed=2))
    try:
        rec = Recorder(net)
        y = np.zeros(3, np.float32)
        batches = [[(9, 9), (10, 9), (9, 12)], [(200, 180), (90, 300), (9, 9)], [(12, 12), (9, 10), (11, 9)],
                   [(400, 420), (380, 390), (300, 500)]]
        for t, sizes in enumerate(batches):
            x = _images(sizes, 3, 40 + t)
            assert net.train_raw(0, [x, y], resize=(24, 24)), net.last_error()
            assert T.same_bits(rec.host(t)[0], restate(x, (24, 24), 9, True, None, MV, 0.5, T.key(2, 0, 0, t, 0))), t
        assert net.synchronize(), net.last_error()
    finally:
        net.deallocate()


def _restated_batches(which, tmp_path):
    if which == "cifar10_quick":
        solver, mean = _cifar_dir(tmp_path)
        batches = [_cifar_images(10 + t) for t in range(3)]
        return solver, batches, (32, 32), lambda x: restate(x, (32, 32), mean=mean)
    solver = os.path.join(CONFIGS, "lenet_memory_solver.prototxt")
    rng = np.random.RandomState(1)
    batches = []
    for t in range(3):
        sizes = [(int(rng.randint(5, 60)), int(rng.randint(5, 60))) for _ in range(64)]
        batches.append((_images(sizes, 1, 30 + t), rng.randint(0, 10, 64).astype(np.float32)))
    return solver, batches, (28, 28), lambda x: restate(x, (28, 28), scale=0.00390625)


@pytest.mark.parametrize("which", ["cifar10_quick", "lenet_memory"])
def test_engine_trained_by_ragged_train_raw_equals_train_on_restated_batches(cos, tmp_path, which):
    solver, batches, target, restate_x = _restated_batches(which, tmp_path)
    nets = [_net(cos, solver), _net(cos, solver)]
    try:
        for n in nets:
            n.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        for x, y in batches:
            assert nets[0].train_raw(0, [x, y], resize=target), nets[0].last_error()
            assert nets[1].train(0, [restate_x(x), y]), nets[1].last_error()
        for n in nets:
            assert n.synchronize(), n.last_error()
        w = [to_host(n.data()) for n in nets]
        assert_bits_equal(w[0], w[1], f"{which} weights after ragged train_raw vs train")
        assert np.isfinite(w[0]).all()
    finally:
        for n in nets:
            n.deallocate()


def test_pytorch_producer_sees_the_restated_inputs(cos):
    from caffeonspark_b200 import harness

    class Recording(harness.TorchProducer):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.seen = []

        def forward_backward(self, x, label):
            self.seen.append(x.detach().clone())
            return super().forward_backward(x, label)

    from caffeonspark_b200 import nets as N_
    solver = os.path.join(CONFIGS, "lenet_memory_solver.prototxt")
    _, batches, target, restate_x = _restated_batches("lenet_memory", None)
    nets = [_net(cos, solver), _net(cos, solver)]
    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        prods = [Recording(n, N_.torch_module("lenet"), seed=3, use_graph=False) for n in nets]
        for x, y in batches:
            assert nets[0].train_raw(0, [x, y], resize=target), nets[0].last_error()
            assert nets[1].train(0, [restate_x(x), y]), nets[1].last_error()
        for n in nets:
            assert n.synchronize(), n.last_error()
        assert len(prods[0].seen) == len(prods[1].seen) == len(batches)
        for t, (a, b) in enumerate(zip(prods[0].seen, prods[1].seen)):
            assert T.same_bits(a.cpu().numpy(), b.cpu().numpy()), t
            assert T.same_bits(a.cpu().numpy(), restate_x(batches[t][0])), t
        assert_bits_equal(to_host(nets[0].data()), to_host(nets[1].data()), "lenet weights, PyTorch producer")
    finally:
        torch.backends.cudnn.deterministic = prev
        for n in nets:
            n.deallocate()


def test_train_time_refusals_then_a_valid_call(cos, tmp_path):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    text = SMALL_NET.format(N=3, crop=9).replace(
        "mean_value: 104 mean_value: 117 mean_value: 123", 'mean_file: "m.binaryproto"')
    (tmp_path / "m.binaryproto").write_bytes(T.blobproto(np.ones(3 * 12 * 12, np.float32), shape=(1, 3, 12, 12)))
    net = _net(cos, _solver(tmp_path, text))
    try:
        rec = Recorder(net)
        x, y = _images([(30, 20), (12, 12), (7, 50)], 3, 1), np.zeros(3, np.float32)
        bad = [
            (([x, [np.zeros((1, 1, 1), np.uint8)] * 3], (12, 12)), "without transform_param must be COS_RAW_F32_NCHW"),
            (([x[:2], y], (12, 12)), "raw num 2 != the top's 3"),
            (([[i[..., :2].copy() for i in x], y], (12, 12)), "channels == img_channels"),
            (([x, y], (8, 12)), "image 0: Check failed: img_height >= crop_size"),
            (([x, y], None), "image 0: Check failed: img_height == data_mean_.height()"),
            (([x, y], (14, 14)), "image 0: Check failed: img_height == data_mean_.height()"),
        ]
        for (arrays, resize), msg in bad:
            assert not net.train_raw(0, arrays, resize=resize), msg
            assert msg in net.last_error() and "layer 'data'" in net.last_error(), (msg, net.last_error())
        # raw ABI: NULL image array, NULL image data, sizes <= 0, one zero in the target, an overflowing byte count
        imgs = (_lib.cos_raw_image * 3)()
        for k, a in enumerate(x):
            imgs[k].data, imgs[k].height, imgs[k].width = a.ctypes.data, a.shape[0], a.shape[1]
        blobs = (_lib.cos_raw_blob * 2)()
        blobs[0].data, blobs[0].format, blobs[0].num, blobs[0].channels = ctypes.addressof(imgs), 2, 3, 3
        blobs[0].height, blobs[0].width = 12, 12
        blobs[1].data, blobs[1].format, blobs[1].num, blobs[1].channels = y.ctypes.data, 0, 3, 1
        blobs[1].height, blobs[1].width = 1, 1

        def refused(msg):
            assert L.cos_net_train_raw(net._h, 0, blobs, 2) == 0
            err = L.cos_last_error().decode()
            assert msg in err and "layer 'data'" in err, (msg, err)

        blobs[0].data = None
        refused("data[0] is NULL")
        blobs[0].data = ctypes.addressof(imgs)
        imgs[1].data = None
        refused("image 1: data is NULL")
        imgs[1].data = x[1].ctypes.data
        imgs[2].height = 0
        refused("image 2: height and width must be positive")
        imgs[2].height, imgs[2].width = x[2].shape[0], -3
        refused("image 2: height and width must be positive")
        imgs[2].width = x[2].shape[1]
        blobs[0].width = 0
        refused("give both sides, or 0x0")
        blobs[0].width = 12
        imgs[2].height = imgs[2].width = 0x7fffffff  # never read: the count overflows first
        refused("total byte count overflows")
        imgs[2].height, imgs[2].width = x[2].shape[0], x[2].shape[1]
        assert len(rec.calls) == 0
        assert net.train_raw(0, [x, y], resize=(12, 12)), net.last_error()  # a valid call after every refusal
        want = restate(x, (12, 12), 9, True, np.ones(3 * 12 * 12), None, 0.5, T.key(7, 0, 0, 0, 0))
        assert T.same_bits(rec.host(0)[0], want)
        # later calls must keep the first call's format, num, channels and target; image sizes may change
        same = _images([(12, 12)] * 3, 3, 8)  # no target: each image passes the per-image checks on its own size
        assert not net.train_raw(0, [same, y]) and "differs from the first call's" in net.last_error()
        x2 = _images([(9, 9), (40, 41), (12, 13)], 3, 9)
        assert net.train_raw(0, [x2, y], resize=(12, 12)), net.last_error()
        assert T.same_bits(rec.host(1)[0], restate(x2, (12, 12), 9, True, np.ones(3 * 12 * 12), None, 0.5,
                                                   T.key(7, 0, 0, 1, 0)))
        assert net.synchronize(), net.last_error()
    finally:
        net.deallocate()


def test_no_crop_size_must_match_the_top(cos):
    net = _net(cos, os.path.join(CONFIGS, "lenet_memory_solver.prototxt"))
    try:
        rec = Recorder(net)
        x = _images([(28, 28)] * 63 + [(28, 27)], 1, 3)
        y = np.zeros(64, np.float32)
        assert not net.train_raw(0, [x, y])
        assert "image 63: Check failed: img_height == height (image 28x27, top 28x28)" in net.last_error()
        assert net.train_raw(0, [x[:63] + [x[0]], y]), net.last_error()
        assert T.same_bits(rec.host(0)[0], restate(x[:63] + [x[0]], scale=0.00390625))
    finally:
        net.deallocate()
