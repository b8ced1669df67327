"""Caffe's Tile layer on the built-in engine (DESIGN.md section 14), on the GPU.

The kernels alone (layers.tile_forward / tile_backward) against tile_ref.py's fp32 restatement of Forward_cpu and
Backward_cpu, bit for bit as uint32 (every NaN taken as the GPU's canonical one), on values with NaN, both infinities,
both zeros, -FLT_MAX, FLT_MAX, a subnormal and a column of -0: shapes on both sides of the staged backward's threshold
(inner 32), the fixtures' own tiles and ImageNet-scale gates, odd sizes and top counts that are not multiples of 4,
through the 128-bit and the scalar paths.  The output is NaN-poisoned first, and two calls give the same bits.

The op in the engine through test_gpu_producer_ops.py's injector harness.  The SE-ResNet-20 and U-Net scSE fixtures:
gradients against float64 and the PyTorch fp32 mirrors, train() with every update equal to the oracle's on one rank,
two in-process ranks, and BINARYPROTO and HDF5 snapshots that resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tile_ref as R
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_bf16_producer import _task_batches
from test_gpu_crop import _harness_equal, batch_of as unet_batch
from test_gpu_native_producer import _blob_bound, _grads, _load, _params
from test_gpu_producer_ops import _engine
from test_gpu_residual import NET_BOUND as RESNET_BOUND, _StatsUpdateCheck

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
POISON = np.uint32(0x7FBADBAD)  # a signalling NaN: an element a kernel failed to write would keep it
UNET_BOUND = 1e-5  # the U-Net's bound (test_gpu_crop.py)


# --------------------------------------------------------------------------- the kernels
KERNEL_CASES = [  # (bottom, axis, tiles)
    ((32, 256, 1, 1), 2, 56),   # an ImageNet-scale SE gate along H (inner 1: staged, two tile chunks)
    ((32, 256, 56, 1), 3, 56),  # ... then along W
    ((32, 1, 56, 56), 1, 256),  # an sSE gate over 256 channels (inner 3136: direct)
    ((100, 16, 1, 1), 2, 32), ((100, 64, 8, 1), 3, 8),  # the SE-ResNet-20's
    ((8, 32, 1, 1), 2, 28), ((8, 1, 28, 28), 1, 32), ((8, 1, 52, 52), 1, 16),  # the U-Net scSE's
    ((5, 3, 1), 2, 7),          # a top of 105 elements: scalar forward
    ((3, 5, 7), 1, 3),          # inner 35, a top of 315
    ((2, 31), 1, 5), ((2, 32), 1, 5), ((3, 33), 1, 2),  # around the threshold
    ((3, 4, 4), 2, 3),          # inner 4: float4 loads and stores
    ((2, 3, 2), 1, 4),          # inner 6, a top of 48: float4 stores of single loads
    ((7, 3), 0, 1), ((1,), 0, 1000), ((1000, 7), 1, 2), ((2, 1, 3, 2, 2), -1, 3),
]


def _dev(a, misalign):
    """a on the GPU, one float past a 16-byte boundary with misalign (the scalar paths)"""
    buf = torch.empty(a.size + 4, dtype=torch.float32, device="cuda")
    t = buf[1:1 + a.size] if misalign else buf[:a.size]
    t.copy_(torch.from_numpy(np.ascontiguousarray(a).ravel()))
    return t.view(a.shape)


def _kernels(x, dy, axis, tiles, misalign=False):
    from caffeonspark_b200 import layers
    top = R.infer(x.shape, axis, tiles)
    y = _dev(np.full(top, POISON, np.uint32).view(F32), misalign)
    layers.tile_forward(_dev(x, misalign), axis, tiles, out=y)
    dx = _dev(np.full(x.shape, POISON, np.uint32).view(F32), misalign)
    layers.tile_backward(_dev(dy, misalign), x.shape, axis, tiles, out=dx)
    torch.cuda.synchronize()
    return to_host(y), to_host(dx)


@pytest.mark.parametrize("shape,axis,tiles", KERNEL_CASES)
def test_kernels_bit_for_bit(cos, shape, axis, tiles):
    rng = np.random.RandomState(int(np.prod(shape)) % 100003 + tiles)
    x = R.specials(rng, shape)
    top = R.infer(shape, axis, tiles)
    dy = R.negative_zero_column(R.specials(rng, top), shape, axis, tiles)
    want_y, want_dx = R.forward32(x, axis, tiles), R.backward32(dy, shape, axis, tiles)
    assert want_dx.reshape(-1)[-1].view(np.uint32) == 0x80000000
    runs = []
    for misalign in ([False, True] if np.prod(top) < 10 ** 6 else [False]):
        y, dx = _kernels(x, dy, axis, tiles, misalign)
        assert np.array_equal(y.view(np.uint32), want_y.view(np.uint32)), f"forward (misaligned {misalign})"
        assert np.array_equal(R.canonical_bits(dx), R.canonical_bits(want_dx)), f"backward (misaligned {misalign})"
        runs.append((y, dx))
    y2, dx2 = _kernels(x, dy, axis, tiles)
    assert_bits_equal(y2, runs[0][0], "a second forward")
    assert_bits_equal(dx2, runs[0][1], "a second backward")


def test_both_backward_kernels_are_reached():
    inners = {R.dims(s, a)[1] for s, a, _ in KERNEL_CASES}
    assert min(inners) < 32 <= max(inners) and {31, 32} <= inners


def test_bad_arguments_are_refused(cos):
    from caffeonspark_b200 import layers
    x = torch.zeros(2, 3, device="cuda")
    with pytest.raises(cos.CosError, match="Number of tiles must be positive"):
        layers.tile_forward(x, 1, 0)
    with pytest.raises(cos.CosError, match="axis 2 out of range for 2-D Blob"):
        layers.tile_forward(x, 2, 3)
    with pytest.raises(cos.CosError, match="Tile takes a bottom"):
        layers.tile_backward(torch.zeros(2, 5, device="cuda"), (2, 3), 1, 2)


# --------------------------------------------------------------------------- the op in the engine
OP_CASES = [((2, 3, 1, 1), 2, 5), ((2, 3, 4, 1), 3, 4), ((2, 1, 6, 7), 1, 3), ((3, 40), 1, 2), ((2, 3, 4), 0, 3),
            ((2, 3, 4, 5), -1, 2)]


@pytest.mark.parametrize("shape,axis,tiles", OP_CASES)
def test_op_in_the_engine(cos, tmp_path, shape, axis, tiles):
    rng = np.random.RandomState(int(np.prod(shape)) + tiles)
    x = (rng.randn(*shape) * np.exp2(rng.randint(-6, 7, shape))).astype(F32) + F32(0)  # no -0: the injectors make +0
    y = R.forward32(x, axis, tiles)
    body = f'layer {{ name: "tl" type: "Tile" bottom: "x0" top: "y" tile_param {{ axis: {axis} tiles: {tiles} }} }}\n'
    results = []
    for k in range(2):
        (tmp_path / str(k)).mkdir()
        r = _engine(cos, tmp_path / str(k), [x], body, (), y.shape, np.zeros(y.shape, F32))
        _harness_equal(r["d"], y, "y")  # B = 0: the probe returns y, the top gradient
        _harness_equal(r["dx"][0], R.backward32(y, shape, axis, tiles), "dx")
        results.append(r)
    assert_bits_equal(results[1]["d"], results[0]["d"], "two calls: y")
    assert_bits_equal(results[1]["dx"][0], results[0]["dx"][0], "two calls: dx")


# --------------------------------------------------------------------------- the fixtures
def _solver(tmp_path, name, extra=""):
    text = open(os.path.join(CONFIGS, f"{name}_solver.prototxt")).read()
    text = text.replace(f'net: "{name}_train_test.prototxt"', f'net: "{os.path.join(CONFIGS, name)}_train_test.prototxt"')
    text = text.replace(f'snapshot_prefix: "{name}"', f'snapshot_prefix: "{tmp_path}/snap"')
    path = tmp_path / f"{name}_solver.prototxt"
    path.write_text(text + extra)
    return str(path)


def _net(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


SE = "cifar10_se_resnet20"
SCSE = "unet_scse"


def _batches(name, seed, steps):
    """`steps` training batches of the fixture, as numpy arrays"""
    if name == SE:
        return [[x.numpy(), y.numpy()] for x, y in _task_batches(seed=seed, steps=steps)]
    return [unet_batch(seed + t, 8) for t in range(steps)]


def _engine_call(net, batch):
    net.diff().zero_()
    loss = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    assert net.forward_backward([torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in batch], loss.data_ptr())
    assert net.synchronize(), net.last_error()
    return float(loss.item()), to_host(net.diff())


def _se_reference(w, batch, dtype, device):
    from caffeonspark_b200 import nets
    m = nets.se_resnet20_module().to(device=device, dtype=dtype)
    _load(m, w)
    out = m(torch.from_numpy(batch[0]).to(device=device, dtype=dtype))
    loss = F.cross_entropy(out, torch.from_numpy(batch[1]).long().to(device))
    loss.backward()
    return float(loss.detach()), _grads(m), _params(m)


def test_se_resnet20_matches_float64_and_pytorch(cos, tmp_path):
    net = _net(cos, _solver(tmp_path, SE))
    try:
        w = to_host(net.data())
        b = _batches(SE, 3, 1)[0]
        l32, g = _engine_call(net, b)
        data_after = to_host(net.data())
        counts, lr_mult = net.desc.counts, net.desc.lr_mult
    finally:
        net.deallocate()
    l64, g64, p64 = _se_reference(w, b, torch.float64, "cpu")
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        lt, gt, _ = _se_reference(w, b, torch.float32, "cuda")
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    off, gated = 0, 0
    for k, c in enumerate(counts):
        sl = slice(off, off + c)
        off += c
        if lr_mult[k] == 0:  # BatchNorm statistics: no gradient, and the forward wrote them
            assert not g[sl].any(), k
            _blob_bound(data_after[sl], p64[sl], f"blob {k} statistics")
            continue
        assert np.abs(g64[sl]).max() > 0, k
        for got, what in ((g, "native"), (gt, "PyTorch fp32")):
            err, scale = np.abs(got[sl].astype(np.float64) - g64[sl]).max(), np.abs(g64[sl]).max()
            assert err <= RESNET_BOUND * scale, f"blob {k} {what}: {err:.3e} > {RESNET_BOUND} * {scale:.3e}"
        gated += 1
    assert gated == 164 - 3 * 21


def _unet_reference(w, batch, dtype, device, branches=None):
    """(loss, flat gradient, branches) of nets.unet_scse_module on the flat weights w; branches are each ReLU's mask,
    each MAX pool's argmax and each Eltwise MAX's choice, in forward order.  With `branches` (another forward's), each
    takes its branch from them."""
    from caffeonspark_b200 import nets
    m = nets.unet_scse_module().to(device=device, dtype=dtype)
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

    def vmax(a, b):
        first = (a > b).cpu() if branches is None else branches[len(taken)]
        taken.append(first)
        return torch.where(first.to(device), a, b)

    m.relu, m.pool, m.max = relu, pool, vmax
    label = m.crop_label(torch.from_numpy(batch[1]).to(device)).reshape(-1).long()
    scores = m(torch.from_numpy(batch[0]).to(device=device, dtype=dtype))
    loss = F.cross_entropy(scores.permute(0, 2, 3, 1).reshape(-1, 2), label)
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def _blob_errors(g, g64, counts):
    """Per blob, the largest error relative to the blob's largest float64 gradient, or to 1% of the net's largest"""
    floor = 1e-2 * np.abs(g64).max()
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / max(np.abs(g64[sl]).max(), floor))
    return errs


def test_unet_scse_matches_float64_and_pytorch(cos, tmp_path):
    net = _net(cos, _solver(tmp_path, SCSE))
    try:
        w = to_host(net.data())
        b = _batches(SCSE, 8, 1)[0]
        l32, g = _engine_call(net, b)
        counts = net.desc.counts
    finally:
        net.deallocate()
    # float64 takes each branch from an fp32 forward: PyTorch's on the CPU for PyTorch fp32, and PyTorch's on the GPU
    # (TF32 off) for the engine
    lt, gt, branches = _unet_reference(w, b, torch.float32, "cpu")
    _, g64t, _ = _unet_reference(w, b, torch.float64, "cpu", branches)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        branches = _unet_reference(w, b, torch.float32, "cuda")[2]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    l64, g64, _ = _unet_reference(w, b, torch.float64, "cpu", branches)
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    native, torch32 = _blob_errors(g, g64, counts), _blob_errors(gt, g64t, counts)
    report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}" for k, (a, b) in enumerate(zip(native, torch32)))
    print(f"worst native {max(native):.2e}, worst PyTorch fp32 {max(torch32):.2e}")
    assert max(native + torch32) <= UNET_BOUND, f"relative to max|g64| per blob: {report}"


def _train(net, batches, check=None):
    losses = []
    for t, b in enumerate(batches):
        if check:
            check.before()
        assert net.train(0, b), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name,param_count,steps", [(SE, 282547, 60), (SCSE, 117520, 40)])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name, param_count, steps):
    net = _net(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == param_count
        losses = _train(net, _batches(name, 1000, steps), _StatsUpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-10:].mean() < losses[:5].mean(), losses
    finally:
        net.deallocate()


def _two_rank_run(cos, name, solver):
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

        # drawn before the ranks start: a rank's first train() allocates its staging buffers, which waits for the
        # device, so a rank still drawing batches then would stall its peer's exchange
        batches = [_batches(name, 10 * (r + 1), 4) for r in range(2)]

        def run(r):
            for b in batches[r]:
                assert netz[r].train(0, b), netz[r].last_error()
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


@pytest.mark.parametrize("name", [SE, SCSE])
def test_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, name, solver), _two_rank_run(cos, name, solver), "two whole runs")


# a blob next to the Tiles in each fixture: (layer, its blob index, flat offset, count), as the plans place them
SNAPSHOT_BLOB = {SE: ("res2a_se_fc1", 0, 5235, 64), SCSE: ("scse4_c_fc1", 0, 107728, 256)}


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
@pytest.mark.parametrize("name", [SE, SCSE])
def test_snapshots_resume_bit_exact(cos, tmp_path, name, fmt):
    solver = _solver(tmp_path, name, f"snapshot_format: {fmt}\n")
    a = _net(cos, solver)
    try:
        _train(a, _batches(name, 1, 3))
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        layer, k, off, n = SNAPSHOT_BLOB[name]
        assert_bits_equal(cos.read_caffemodel_blob(model, layer, k).ravel(), w_a[off:off + n], layer)
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            more = _batches(name, 7, 2)
            la, lb = _train(a, more), _train(b, more)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
