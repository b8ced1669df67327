"""Caffe's Crop layer on the built-in engine (DESIGN.md section 14), on the GPU.

The kernels alone (layers.crop_forward / crop_backward) against crop_ref.py bit for bit, compared as uint32, on values
with NaNs of several payloads, infinities, subnormals and both zeros: every geometry of the host tests' references,
U-Net's crops, odd sizes, identity, maximal offsets, a crop on axis 0, 1-D and 5-D blobs and one large map, through
both the float4 and the scalar path.  The backward writes every element of a NaN-poisoned dx: dy inside the window and
+0 outside it.  Two calls give the same bits.

The op in the engine, through the injector harness of test_gpu_producer_ops.py, with a NaN-poisoned staged reference:
the injectors carry every value but -0 (which they make +0) and NaN payloads (which they make the GPU's canonical NaN),
so non-zero values are compared as uint32, zeros by value and NaNs by position.

The U-Net fixture: per-blob gradients against float64 (branches of every ReLU and MAX pool taken from an fp32 forward)
at b8 and b3, within NET_BOUND of each blob's largest gradient.  PyTorch fp32 on the CPU reaches 2.2e-6 on these two
cases (blob 19, upconv1's bias), and NET_BOUND is 1e-5.  Training through train() alone with every update equal to the
oracle's, on one rank and two in-process ranks, and BINARYPROTO and HDF5 snapshots that resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import crop_ref as R
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_crop_host import _param
from test_gpu_producer_ops import _engine

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
NET_BOUND = 1e-5
POISON = np.uint32(0x7FBADBAD)  # a signalling NaN: an element the backward failed to write would keep it


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, F32)).view(np.uint32)


# --------------------------------------------------------------------------- the kernels
KERNEL_CASES = [  # (bottom, top, offsets)
    ((8, 32, 40, 40), (8, 32, 32, 32), (0, 0, 4, 4)),      # U-Net's crop2
    ((8, 16, 88, 88), (8, 16, 56, 56), (0, 0, 16, 16)),    # crop1
    ((8, 1, 92, 92), (8, 1, 52, 52), (0, 0, 20, 20)),      # the label crop
    ((3, 5, 17, 13), (3, 5, 9, 6), (0, 0, 3, 5)),          # odd sizes: scalar path
    ((2, 3, 8, 8), (2, 3, 8, 8), (0, 0, 0, 0)),            # identity
    ((2, 3, 9, 11), (2, 3, 4, 5), (0, 0, 5, 6)),           # maximal offsets
    ((2, 3, 12, 16), (2, 3, 1, 4), (0, 0, 11, 12)),        # maximal, float4
    ((7, 6, 5), (3, 6, 5), (4, 0, 0)),                     # axis 0 only: merged to one axis
    ((4, 6, 9), (2, 3, 9), (1, 3, 0)),                     # the innermost axis whole
    ((100,), (37,), (50,)),                                # 1-D
    ((101,), (36,), (65,)),
    ((3, 4, 5, 6, 7), (1, 2, 3, 4, 5), (2, 1, 2, 1, 2)),   # 5-D
    ((2, 3, 4, 8, 12), (2, 3, 2, 4, 8), (0, 0, 1, 4, 4)),  # 5-D, float4
    ((8, 64, 392, 392), (8, 64, 200, 200), (0, 0, 96, 96)),  # one large map
]


def _kernels(cos, x, top, offsets, dy, misalign=False):
    """-> (y, dx) from the native kernels, dx's buffer poisoned first; misalign puts every tensor one float past a
    16-byte boundary (the scalar path)"""
    from caffeonspark_b200 import layers

    def dev(a):
        buf = torch.empty(a.size + 4, dtype=torch.float32, device="cuda")
        t = buf[1:1 + a.size] if misalign else buf[:a.size]
        t.copy_(torch.from_numpy(np.ascontiguousarray(a).ravel()))
        return t.view(a.shape)

    y = layers.crop_forward(dev(x), top, offsets, out=dev(np.zeros(top, F32)))
    dx = dev(np.full(x.shape, POISON, np.uint32).view(F32))
    layers.crop_backward(dev(dy), x.shape, offsets, out=dx)
    torch.cuda.synchronize()
    return to_host(y), to_host(dx)


@pytest.mark.parametrize("bottom,top,offsets", KERNEL_CASES)
def test_kernels_bit_for_bit(cos, bottom, top, offsets):
    rng = np.random.RandomState(int(np.prod(bottom)) % 100003)
    x, dy = R.specials(rng, bottom), R.specials(rng, top)
    want_y, want_dx = R.forward(x, top, offsets), R.backward(dy, bottom, offsets)
    paths = [False, True] if np.prod(bottom) < 10 ** 6 else [False]
    runs = []
    for misalign in paths:
        y, dx = _kernels(cos, x, top, offsets, dy, misalign)
        assert np.array_equal(_bits(y), _bits(want_y)), f"forward (misaligned {misalign})"
        assert np.array_equal(_bits(dx), _bits(want_dx)), f"backward (misaligned {misalign})"
        runs.append((y, dx))
    y2, dx2 = _kernels(cos, x, top, offsets, dy)
    assert_bits_equal(y2, runs[0][0], "a second forward")
    assert_bits_equal(dx2, runs[0][1], "a second backward")


def test_a_window_outside_the_bottom_is_refused(cos):
    from caffeonspark_b200 import layers
    x = torch.zeros(2, 3, 8, 8, device="cuda")
    with pytest.raises(cos.CosError, match="the window leaves the bottom"):
        layers.crop_forward(x, (2, 3, 4, 4), (0, 0, 5, 0))


# --------------------------------------------------------------------------- the op in the engine
OP_CASES = [  # (bottom, reference, crop_param, canonical axis)
    ((2, 3, 12, 12), (1, 1, 8, 8), "offset: 2", 2),
    ((2, 3, 12, 16), (1, 1, 4, 8), "offset: 4 offset: 8", 2),
    ((3, 5, 17, 13), (1, 1, 9, 6), "offset: 3 offset: 5", 2),
    ((2, 3, 8, 8), (2, 3, 8, 8), "", 2),
    ((2, 3, 9, 11), (1, 1, 4, 5), "offset: 5 offset: 6", 2),
    ((4, 6, 5), (2, 6, 5), "axis: 0 offset: 2 offset: 0 offset: 0", 0),
    ((2, 7, 6, 6), (2, 3, 2, 2), "axis: 1 offset: 4", 1),
    ((2, 3, 8, 13), (1, 1, 1, 5), "axis: -1 offset: 8", 3),
    ((5, 9), (5, 4), "axis: 1 offset: 5", 1),
    ((3, 10, 7), (3, 4, 7), "axis: 1 offset: 6 offset: 0", 1),
]


def _harness_equal(got, want, what):
    """NaN where want has NaN; zeros equal by value; every other value bit for bit"""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    zero = want == 0
    assert (got[zero] == 0).all(), f"{what}: zeros differ"
    rest = ~nan & ~zero
    bad = _bits(got)[rest] != _bits(want)[rest]
    assert not bad.any(), f"{what}: {int(bad.sum())} of {int(rest.sum())} values differ"


@pytest.mark.parametrize("bottom,ref,param,axis", OP_CASES)
def test_op_in_the_engine(cos, tmp_path, bottom, ref, param, axis):
    rng = np.random.RandomState(int(np.prod(bottom)) + axis)
    x = R.specials(rng, bottom)
    a, top, offs = R.infer(bottom, ref, *_param(param))
    assert a == axis
    body = f'layer {{ name: "c" type: "Crop" bottom: "x0" bottom: "r" top: "y" crop_param {{ {param} }} }}\n'
    staged = {"r": np.full(ref, np.nan, F32)}  # a NaN-poisoned reference changes nothing
    results = []
    for k in range(2):
        (tmp_path / str(k)).mkdir()
        r = _engine(cos, tmp_path / str(k), [x], body, (), top, np.zeros(top, F32), staged=staged)
        _harness_equal(r["d"], R.forward(x, top, offs), "y")  # B = 0: the probe returns y, the top gradient
        _harness_equal(r["dx"][0], R.backward(R.forward(x, top, offs), bottom, offs), "dx")
        results.append(r)
    assert_bits_equal(results[1]["d"], results[0]["d"], "two calls: y")
    assert_bits_equal(results[1]["dx"][0], results[0]["dx"][0], "two calls: dx")


# --------------------------------------------------------------------------- the U-Net fixture
UNET = "unet"


def _solver(tmp_path, extra="", batch=None):
    text = open(os.path.join(CONFIGS, "unet_train_test.prototxt")).read()
    if batch is not None:
        text = text.replace("batch_size: 8\n", f"batch_size: {batch}\n")
    net = tmp_path / f"unet_b{batch}.prototxt"
    net.write_text(text)
    s = open(os.path.join(CONFIGS, "unet_solver.prototxt")).read()
    s = s.replace('net: "unet_train_test.prototxt"', f'net: "{net}"')
    s = s.replace('snapshot_prefix: "unet"', f'snapshot_prefix: "{tmp_path}/snap"')
    path = tmp_path / f"unet_{batch}_solver.prototxt"
    path.write_text(s + extra)
    return str(path)


def _net_of(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


def batch_of(seed, n):
    """n images [n, 1, 92, 92] of three bright disks on noise, and their per-pixel labels (1 inside a disk)"""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:92, 0:92]
    mask = np.zeros((n, 1, 92, 92), F32)
    for i in range(n):
        for _ in range(3):
            cy, cx, r = rng.randint(10, 82), rng.randint(10, 82), rng.randint(8, 20)
            mask[i, 0][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 1
    return [(0.7 * mask + 0.3 * rng.rand(n, 1, 92, 92)).astype(F32), mask]


def host_weights(seed):
    """Flat weights drawn on the host: each weight Gaussian with Caffe's msra deviation sqrt(2 / fan_in), each bias
    uniform in [-0.05, 0.05)"""
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(seed)
    parts = []
    for p in nets.unet_module().parameters():
        if p.dim() > 1:
            parts.append((rng.randn(p.numel()) * np.sqrt(2.0 / (p.numel() // p.shape[0]))).astype(F32))
        else:
            parts.append(rng.uniform(-0.05, 0.05, p.numel()).astype(F32))
    w = np.concatenate(parts)
    assert w.size == nets.UNET_PARAM_COUNT
    return w


def reference(w, batch, dtype, device, branches=None):
    """(loss, flat gradient, branches) of nets.unet_module on the flat weights w; branches are each ReLU's mask and
    each MAX pool's argmax, in forward order.  With `branches` (another forward's), every ReLU and MAX pool takes its
    branch from them."""
    from caffeonspark_b200 import nets
    m = nets.unet_module().to(device=device, dtype=dtype)
    _load(m, w)
    taken = []

    def relu(h):
        mask = (h > 0).cpu() if branches is None else branches[len(taken)]
        taken.append(mask)
        return h * mask.to(device=device, dtype=dtype)

    def pool(h):
        if branches is None:
            out, i = F.max_pool2d(h, 2, 2, ceil_mode=True, return_indices=True)
            taken.append(i.cpu())
            return out
        i = branches[len(taken)].to(device)
        taken.append(i.cpu())
        return h.flatten(2).gather(2, i.flatten(2)).view(i.shape)

    m.relu, m.pool = relu, pool
    label = m.crop_label(torch.from_numpy(batch[1]).to(device)).reshape(-1).long()
    scores = m(torch.from_numpy(batch[0]).to(device=device, dtype=dtype))
    loss = F.cross_entropy(scores.permute(0, 2, 3, 1).reshape(-1, 2), label)  # one row per scored pixel
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def blob_errors(g, g64, counts):
    """Per blob, the largest error relative to the blob's largest float64 gradient, or to 1% of the net's largest
    where the blob's is smaller"""
    floor = 1e-2 * np.abs(g64).max()
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / max(np.abs(g64[sl]).max(), floor))
    return errs


@pytest.mark.parametrize("n", [8, 3])
def test_unet_matches_float64_and_pytorch(cos, tmp_path, n):
    net = _net_of(cos, _solver(tmp_path, batch=n), fill=False)
    try:
        w = host_weights(21 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        b = batch_of(n, n)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(v).cuda() for v in b], loss.data_ptr())
        assert net.synchronize(), net.last_error()
        l32, g, counts = float(loss.item()), to_host(net.diff()), net.desc.counts
    finally:
        net.deallocate()
    # float64 takes each ReLU's and MAX pool's branch from an fp32 forward: PyTorch's on the CPU for PyTorch fp32, and
    # PyTorch's on the GPU (TF32 off) for the engine
    lt, gt, branches = reference(w, b, torch.float32, "cpu")
    _, g64t, _ = reference(w, b, torch.float64, "cpu", branches)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        branches = reference(w, b, torch.float32, "cuda")[2]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    l64, g64, _ = reference(w, b, torch.float64, "cpu", branches)
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    native, torch32 = blob_errors(g, g64, counts), blob_errors(gt, g64t, counts)
    report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}"
                       for k, (a, b) in enumerate(zip(native, torch32)))
    print(f"b{n}: worst native {max(native):.2e}, worst PyTorch fp32 {max(torch32):.2e}")
    assert max(native + torch32) <= NET_BOUND, f"relative to max|g64| per blob: {report}"


def _train(net, steps, seed, check=None):
    losses = []
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, batch_of(seed + t, 8)), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


def test_unet_trains_through_train_alone(cos, oracle, tmp_path):
    from caffeonspark_b200 import nets
    net = _net_of(cos, _solver(tmp_path))
    try:
        assert net.param_count() == nets.UNET_PARAM_COUNT
        losses = _train(net, 40, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-10:].mean() < 0.8 * losses[:5].mean(), losses
    finally:
        net.deallocate()


def _two_rank_run(cos, solver):
    netz = [cos.CaffeNet(solver, "", "", 1, 2, r, True, cos.CaffeNet.SOCKET, -1, 0) for r in range(2)]
    try:
        for n in netz:
            n.set_option("grid", 8)
            n.set_option("block", 128)
            n.set_option("barrier_timeout_ms", 20000)
            n.set_option("initial_gather", 0)
            n.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        table = [n.localAddresses() for n in netz]
        with cf.ThreadPoolExecutor(2) as ex:
            assert all(ex.map(lambda r: netz[r].connect([table[p][r] if p != r else "" for p in range(2)]), range(2)))

        def run(r):
            for t in range(4):
                assert netz[r].train(0, batch_of(10 * r + t, 8)), netz[r].last_error()
            assert netz[r].synchronize(), netz[r].last_error()
            return netz[r].last_loss()

        with cf.ThreadPoolExecutor(2) as ex:
            losses = list(ex.map(run, range(2)))
        w0, w1 = to_host(netz[0].data()), to_host(netz[1].data())
        assert_bits_equal(w0, w1, "ranks hold identical weights")
        assert np.isfinite(losses).all()
        return w0
    finally:
        with cf.ThreadPoolExecutor(2) as ex:
            list(ex.map(lambda n: n.deallocate(), netz))


def test_unet_two_ranks_in_process(cos, tmp_path):
    solver = _solver(tmp_path)
    assert_bits_equal(_two_rank_run(cos, solver), _two_rank_run(cos, solver), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_unet_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, extra=f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(a, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        bias = w_a[109776:109776 + 16]
        assert_bits_equal(cos.read_caffemodel_blob(model, "upconv1", 1).ravel(), bias, "upconv1 bias")
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, 2, 7), _train(b, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
