"""Caffe's MVN layer on the built-in engine (DESIGN.md section 14) on the GPU.

The op runs through test_gpu_producer_ops.py's injector harness: x comes from an injector (so its gradient comes back
exactly), and the top meets the EuclideanLoss probe, which hands the op a known top gradient d and returns it.  y and
dx are held to mvn_ref.py's per-element bounds around float64 over every regime the kernels pick (lanes, a warp, a
block per row, split rows) and past 65,535 rows.  Through the raw cos_mvn_* entries the fp32 restatement must
reproduce y and dx bit for bit from the kernels' own row sums, two calls must agree bit for bit, and constant rows
give y = 0 and Caffe's dx = (dy - mean dy) / eps.  In place equals out of place in the engine.

Both MVN fixtures are checked against float64 and PyTorch fp32 at their own batch and an odd one, trained through
train() with every update equal to the oracle's on one rank and two, and cifar10_quick_mvn's snapshots resume
bit-exact.  Its per-sample statistics make two ranks of b/2 match one rank of b."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mvn_ref as M
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import _engine

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
QUICK, LM = "cifar10_quick_mvn", "rnn_lm_ln"
# Per-blob gradient bound relative to the blob's largest float64 gradient (blob_errors), fixed on the CPU from these
# very weights and batches: PyTorch fp32 on the CPU reached at worst 1.5e-6 (cifar10_quick_mvn, b100 and b37, with
# float64's ReLUs and MAX pools taking fp32's branches; with its own, one flipped ReLU input gives 1.1e-3) and 5.9e-7
# (rnn_lm_ln, b32 and b13), the loss 1.2e-7 relative.
NET_BOUND = 1e-4


# --------------------------------------------------------------------------- the op
def _mvn(across, variance, eps, top="y", bottom="x0"):
    return (f'layer {{ name: "m" type: "MVN" bottom: "{bottom}" top: "{top}" mvn_param {{ across_channels: '
            f'{str(across).lower()} normalize_variance: {str(variance).lower()} eps: {eps!r} }} }}\n')


# (bottom shape, across_channels): dims 1, 2, 31, 32, 33, 1023, 1024, 1025, 3.2 M over 2 rows, and > 65,535 rows
OP_SHAPES = [((4, 3), False), ((6, 2), True), ((3, 2, 31), False), ((2, 32), True), ((3, 11, 3), True),
             ((2, 3, 1023), False), ((2, 4, 16, 16), True), ((3, 1025, 1, 1), True), ((2, 1600, 2000), True),
             ((70000, 2), False), ((66000, 3, 4), True), ((3, 5, 7, 9), False)]


def _x(rng, shape):
    return (rng.randn(*shape) * 1.5 + rng.randn()).astype(F32)


@pytest.mark.parametrize("eps", [1e-9, 1e-3])
@pytest.mark.parametrize("variance", [True, False])
@pytest.mark.parametrize("shape,across", OP_SHAPES)
def test_mvn_op_within_bounds(cos, tmp_path, shape, across, variance, eps):
    rng = np.random.RandomState(sum(shape) % 1000)
    x = _x(rng, shape)
    y64, s64 = M.forward(x, variance, across, eps)
    B = (y64 - rng.randn(*y64.shape) * 0.5).astype(F32)
    out = _engine(cos, tmp_path, [x], _mvn(across, variance, eps), out_shape=y64.shape, B=B)
    rows, dim = M.rows_dim(shape, across)
    d = out["d"].astype(np.float64)
    y = (d + B).reshape(rows, dim)  # d = fl(y - B): y within u |d| of d + B
    by = M.bound_y(x.reshape(rows, dim), y64, s64)
    err = np.abs(y - y64.reshape(rows, dim)) - (by + M.U * np.abs(d.reshape(rows, dim)))
    assert err.max() <= 0, f"y: worst excess {err.max():.3e}"
    dx64 = M.backward(y64, d, s64, across)
    bd = M.bound_dx(y64.reshape(rows, dim), d.reshape(rows, dim), s64, by)
    err = np.abs(out["dx"][0].reshape(rows, dim) - dx64) - bd
    assert err.max() <= 0, f"dx: worst excess {err.max():.3e}"


def _raw(cos, x, dy, variance, eps, rows, dim, y_out=None):
    """One forward and one backward through cos_mvn_* -> (y, dx, stats) on the host."""
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    xt = torch.from_numpy(x).cuda()
    yt = xt if y_out == "in_place" else torch.empty_like(xt)
    dyt = torch.from_numpy(dy).cuda()
    dxt = torch.empty_like(xt)
    stats = torch.full((5 * rows,), float("nan"), device="cuda")
    work = torch.empty(max(1, L.cos_mvn_workspace_floats(rows, dim)), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert L.cos_mvn_forward(xt.data_ptr(), yt.data_ptr(), stats.data_ptr(), work.data_ptr(), rows, dim,
                             int(variance), eps, st), L.cos_last_error()
    assert L.cos_mvn_backward(yt.data_ptr(), dyt.data_ptr(), dxt.data_ptr(), stats.data_ptr(), work.data_ptr(), rows,
                              dim, int(variance), st), L.cos_last_error()
    torch.cuda.synchronize()
    return to_host(yt).reshape(rows, dim), to_host(dxt).reshape(rows, dim), to_host(stats).reshape(5, rows)


# (rows, dim): each regime and both sides of every threshold in mvn.hpp
RAW_CASES = [(5, 1), (70000, 1), (9, 3), (4, 16), (3, 17), (7, 512), (5, 513), (3, 1025), (1100, 16384),
             (1023, 16384), (2, 3200000), (3, 8193 * 3), (1, 16384 * 1024 + 7)]


@pytest.mark.parametrize("variance", [True, False])
@pytest.mark.parametrize("rows,dim", RAW_CASES)
def test_restatement_is_bit_exact_from_the_kernels_row_sums(cos, rows, dim, variance):
    rng = np.random.RandomState(rows + dim)
    x = (rng.randn(rows, dim) * 3 + 1).astype(F32)
    dy = rng.randn(rows, dim).astype(F32)
    y, dx, st = _raw(cos, x, dy, variance, 1e-3, rows, dim)
    y32, s32 = M.forward32(x, st[0], st[1], variance, 1e-3, M.glibc_powf_half())
    assert_bits_equal(st[2], s32, "s")
    assert_bits_equal(y, y32, "y from the kernel's row sums")
    assert_bits_equal(dx, M.backward32(y, dy, st[3], st[4], st[2], variance), "dx from the kernel's row sums")
    again = _raw(cos, x, dy, variance, 1e-3, rows, dim)
    for a, b, what in zip(again, (y, dx, st), ("y", "dx", "stats")):
        assert_bits_equal(a, b, f"{what}: two calls")
    if rows * dim <= 1 << 22:  # the row sums themselves, against float64
        assert np.abs(st[0] - x.astype(np.float64).sum(1)).max() <= (dim + 1) * M.U * np.abs(x).sum(1).max()
    yi, dxi, _ = _raw(cos, x, dy, variance, 1e-3, rows, dim, y_out="in_place")
    assert_bits_equal(yi, y, "y written over x")
    assert_bits_equal(dxi, dx, "dx after an in-place forward")


@pytest.mark.parametrize("dim", [1, 2, 32, 1024, 32768])
def test_constant_rows(cos, dim):
    rows = 3
    x = np.full((rows, dim), 0.75, F32)
    x[1] = -2.5
    dy = np.random.RandomState(dim).randn(rows, dim).astype(F32)
    y, dx, st = _raw(cos, x, dy, True, 1e-9, rows, dim)
    assert not y.any(), "a constant row normalises to 0"
    assert_bits_equal(st[2], np.full(rows, F32(1e-9)), "s = powf(0, 0.5) + eps")
    assert_bits_equal(dx, M.backward32(y, dy, np.zeros(rows, F32), st[4], st[2], True), "dx")
    want = (dy - dy.astype(np.float64).mean(1, keepdims=True)) / F32(1e-9)
    assert np.abs(dx - want).max() <= (dim + 4) * M.U * np.abs(dy).sum(1).max() / F32(1e-9)


@pytest.mark.parametrize("across", [True, False])
def test_in_place_equals_out_of_place(cos, tmp_path, across):
    rng = np.random.RandomState(3)
    x = _x(rng, (4, 5, 6, 7))
    y64, _ = M.forward(x, True, across, 1e-9)
    B = (y64 - rng.randn(*y64.shape)).astype(F32)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    body = _mvn(across, True, 1e-9, top="x0")
    a = _engine(cos, tmp_path / "a", [x], _mvn(across, True, 1e-9), out_shape=y64.shape, B=B)
    b = _engine(cos, tmp_path / "b", [x], body, out_shape=y64.shape, B=B, top="x0")
    assert_bits_equal(b["d"], a["d"], "top")
    assert_bits_equal(b["dx"][0], a["dx"][0], "dx")


# --------------------------------------------------------------------------- the fixtures
BATCH = {QUICK: 100, LM: 32}


def _solver(tmp_path, name, extra="", batch=None):
    text = open(os.path.join(CONFIGS, f"{name}_train_test.prototxt")).read()
    if batch is not None:
        text = text.replace(f"batch_size: {BATCH[name]}\n", f"batch_size: {batch}\n", 1)
    text = text.replace('mean_file: "mean.binaryproto"', "")  # the batches below are staged as they are
    net = tmp_path / f"{name}_b{batch}.prototxt"
    net.write_text(text)
    s = open(os.path.join(CONFIGS, f"{name}_solver.prototxt")).read()
    s = s.replace(f'net: "{name}_train_test.prototxt"', f'net: "{net}"')
    s = s.replace(f'snapshot_prefix: "{name}"', f'snapshot_prefix: "{tmp_path}/snap"')
    path = tmp_path / f"{name}_{batch}_solver.prototxt"
    path.write_text(s + extra)
    return str(path)


def _net_of(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


def batch_of(name, seed, n, first=False):
    """cifar10_quick_mvn: images [n, 3, 32, 32] near one of ten templates and their labels.  rnn_lm_ln: rnn_lm's
    time-major sentences (cont, tokens, targets) [20, n]."""
    rng = np.random.RandomState(seed)
    if name == QUICK:
        templates = np.random.RandomState(99).rand(10, 3, 32, 32)
        y = rng.randint(0, 10, n)
        return [(0.6 * templates[y] + 0.4 * rng.rand(n, 3, 32, 32)).astype(F32), y.astype(F32)]
    T, V = 20, 100
    tokens = np.zeros((T + 1, n), np.int64)
    tokens[0] = rng.randint(0, V, n)
    cont = np.ones((T, n), F32)
    for t in range(T):
        cont[t][rng.rand(n) < 0.15] = 0
        tokens[t + 1] = np.where(rng.rand(n) < 0.1, rng.randint(0, V, n), (tokens[t] * 7 + 3) % V)
    cont[0] = 0 if first else (rng.rand(n) < 0.33)
    return [cont, tokens[:-1].astype(F32), tokens[1:].astype(F32)]


def host_weights(name, seed):
    """Flat weights uniform in [-0.1, 0.1), each Scale's scale 1 + that, drawn on the host (the bound's CPU runs use
    them too)."""
    from caffeonspark_b200 import nets
    m = nets.cifar10_quick_mvn_module() if name == QUICK else nets.rnn_lm_ln_module()
    rng = np.random.RandomState(seed)
    parts = []
    for k, (pname, p) in enumerate(m.named_parameters()):
        v = rng.uniform(-0.1, 0.1, p.numel())
        if "weight" in pname and p.dim() == 1:  # a Scale's scale
            v = v + 1
        parts.append(v.astype(F32))
    w = np.concatenate(parts)
    assert w.size == (nets.CIFAR10_QUICK_MVN_PARAM_COUNT if name == QUICK else nets.RNN_LM_LN_PARAM_COUNT)
    return w


def reference(name, w, batch, dtype, device, argmax=None):
    """(loss, flat gradient, branches) of the PyTorch mirror on the flat weights w (rnn_lm_ln from a zero hidden
    state); branches are each ReLU's mask and each MAX pool's argmax.  With `argmax` (another forward's branches),
    every ReLU and MAX pool takes its branch from it."""
    from caffeonspark_b200 import nets
    m = (nets.cifar10_quick_mvn_module() if name == QUICK else nets.rnn_lm_ln_module()).to(device=device, dtype=dtype)
    _load(m, w)
    taken = []
    if name == QUICK:
        h = torch.from_numpy(batch[0]).to(device=device, dtype=dtype)
        for layer in m:
            if isinstance(layer, torch.nn.ReLU):  # the branch: where the input is positive
                mask = (h > 0).cpu() if argmax is None else argmax[len(taken)]
                taken.append(mask)
                h = h * mask.to(device=device, dtype=dtype)
            elif not isinstance(layer, torch.nn.MaxPool2d):
                h = layer(h)
            elif argmax is None:
                h, i = F.max_pool2d(h, layer.kernel_size, layer.stride, ceil_mode=True, return_indices=True)
                taken.append(i.cpu())
            else:
                i = argmax[len(taken)].to(device)
                taken.append(i.cpu())
                h = h.flatten(2).gather(2, i.flatten(2)).view(i.shape)
        loss = F.cross_entropy(h, torch.from_numpy(batch[1]).to(device).long())
    else:
        cont, tok, tgt = (torch.from_numpy(v).to(device) for v in batch)
        scores, _ = m(tok, cont.to(dtype), torch.zeros(tok.shape[1], 256, dtype=dtype, device=device))
        loss = F.cross_entropy(scores.reshape(-1, scores.shape[-1]), tgt.reshape(-1).long())
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def blob_errors(g, g64, counts):
    """Per blob, the largest error relative to the blob's largest float64 gradient, or to 1% of the net's largest
    where the blob's is smaller: conv2's bias has a true gradient of 0, as the per-channel MVN after it removes any
    per-channel shift."""
    floor = 1e-2 * np.abs(g64).max()
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / max(np.abs(g64[sl]).max(), floor))
    return errs


def _engine_call(net, batch):
    net.diff().zero_()
    loss = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    assert net.forward_backward([torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in batch], loss.data_ptr())
    assert net.synchronize(), net.last_error()
    return float(loss.item()), to_host(net.diff())


@pytest.mark.parametrize("batch", ["own", "odd"])
@pytest.mark.parametrize("name", [QUICK, LM])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name, batch):
    n = BATCH[name] if batch == "own" else {QUICK: 37, LM: 13}[name]
    net = _net_of(cos, _solver(tmp_path, name, batch=n), fill=False)
    try:
        w = host_weights(name, 21 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        b = batch_of(name, n, n, first=True)
        l32, g = _engine_call(net, b)
        counts = net.desc.counts
    finally:
        net.deallocate()
    # float64 takes each ReLU's and MAX pool's branch from an fp32 forward: from PyTorch's on the CPU for PyTorch fp32,
    # and from PyTorch's on the GPU (TF32 off) for the engine
    lt, gt, branches = reference(name, w, b, torch.float32, "cpu")
    _, g64t, _ = reference(name, w, b, torch.float64, "cpu", branches)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        branches = reference(name, w, b, torch.float32, "cuda")[2]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    l64, g64, _ = reference(name, w, b, torch.float64, "cpu", branches)
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    native, torch32 = blob_errors(g, g64, counts), blob_errors(gt, g64t, counts)
    report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}" for k, (a, b) in enumerate(zip(native, torch32)))
    assert max(native + torch32) <= NET_BOUND, f"relative to max|g64| per blob: {report}"


def _train(net, name, steps, seed, check=None):
    losses = []
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, batch_of(name, seed + t, BATCH[name], first=t == 0)), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", [QUICK, LM])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    from caffeonspark_b200 import nets
    net = _net_of(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == (nets.CIFAR10_QUICK_MVN_PARAM_COUNT if name == QUICK else
                                     nets.RNN_LM_LN_PARAM_COUNT)
        losses = _train(net, name, 80, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-20:].mean() < losses[:10].mean(), losses
    finally:
        net.deallocate()


def _two_rank_run(cos, solver, name):
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
                assert netz[r].train(0, batch_of(name, 10 * r + t, BATCH[name], first=t == 0)), netz[r].last_error()
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


@pytest.mark.parametrize("name", [QUICK, LM])
def test_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, solver, name), _two_rank_run(cos, solver, name), "two whole runs")


def test_two_half_batches_match_one_whole_batch(cos, tmp_path):
    """MVN's statistics are per sample, so the gradient of b images is the mean of the gradients of its two halves
    (SoftmaxWithLoss averages over the batch), to the float64 bound: the property BatchNorm's batch statistics lack."""
    n = BATCH[QUICK]
    w = host_weights(QUICK, 7)
    whole = batch_of(QUICK, 3, n)
    halves = [[v[:n // 2] for v in whole], [v[n // 2:] for v in whole]]
    got = []
    for k, (b, size) in enumerate([(whole, n), (halves[0], n // 2), (halves[1], n // 2)]):
        (tmp_path / str(k)).mkdir()
        net = _net_of(cos, _solver(tmp_path / str(k), QUICK, batch=size), fill=False)
        try:
            net.data().copy_(torch.from_numpy(w).cuda())
            got.append(_engine_call(net, b))
        finally:
            net.deallocate()
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        branches = reference(QUICK, w, whole, torch.float32, "cuda")[2]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    _, g64, _ = reference(QUICK, w, whole, torch.float64, "cpu", branches)
    from caffeonspark_b200 import nets
    counts = [p.numel() for p in nets.cifar10_quick_mvn_module().parameters()]
    split = (got[1][1].astype(np.float64) + got[2][1]) / 2
    assert max(blob_errors(got[0][1], g64, counts)) <= NET_BOUND
    assert max(blob_errors(split, g64, counts)) <= NET_BOUND


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_cifar10_quick_mvn_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, QUICK, f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(a, QUICK, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        assert_bits_equal(cos.read_caffemodel_blob(model, "scale3", 1).ravel(), w_a[79456:79456 + 64], "scale3 bias")
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, QUICK, 2, 7), _train(b, QUICK, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
