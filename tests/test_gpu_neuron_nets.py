"""The TanH LeNet and PReLU CIFAR-10-quick fixtures on the built-in engine (DESIGN.md section 14) on the GPU: gradients
at batch 64 and 100 against float64 and PyTorch fp32, training through train() alone with every update checked against
the oracle, two in-process ranks, and (PReLU net) snapshots that resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _grads, _load

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
TANH, PRELU = "lenet_tanh", "cifar10_quick_prelu"
# The per-blob gradient bound, relative to the blob's largest float64 gradient, for the engine and PyTorch fp32 alike.
# A MAX pool window whose two largest inputs lie within fp32's rounding of each other can pick another winner in fp32
# than in float64, and routes that window's gradient elsewhere: a difference of the piecewise function's branch, not
# of precision.  So the float64 reference takes each MAX pool's argmax from the fp32 forward (PyTorch fp32 on the GPU,
# TF32 off) and differentiates the branch fp32 took.  The bound was fixed on the CPU from these very weights and
# batches (_host_weights, _batch), with the branch of a CPU fp32 forward: PyTorch fp32 on the CPU reached at worst
# 8.2e-7 of a blob's largest gradient (TanH LeNet) and 5.9e-6 (PReLU CIFAR-10-quick) at b64 and b100, the loss 7.5e-8
# relative.  Against float64's own branch the same CPU fp32 gradients are off by up to 8.3e-4 and 3.3e-3, on the blobs
# before a near-tied MAX pool window.
NET_BOUND = 1e-4
STEPS = 120


def _solver(tmp_path, name, extra="", batch=None):
    net = os.path.join(CONFIGS, f"{name}_train_test.prototxt")
    text = open(net).read()
    default = 64 if name == TANH else 100
    if batch is not None:
        text = text.replace(f"batch_size: {default}\n", f"batch_size: {batch}\n", 1)
    text = text.replace('mean_file: "mean.binaryproto"', "")  # the batches below are staged as they are
    net = tmp_path / f"{name}_b{batch}.prototxt"
    net.write_text(text)
    s = open(os.path.join(CONFIGS, f"{name}_solver.prototxt")).read()
    s = s.replace(f'net: "{name}_train_test.prototxt"', f'net: "{net}"')
    s = s.replace(f'snapshot_prefix: "{"mnist_lenet_tanh" if name == TANH else name}"', f'snapshot_prefix: "{tmp_path}/snap"')
    path = tmp_path / f"{name}_{batch}_solver.prototxt"
    path.write_text(s + extra)
    return str(path)


def _net(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


def _batch(name, seed, n):
    rng = np.random.RandomState(seed)
    shape = (n, 1, 28, 28) if name == TANH else (n, 3, 32, 32)
    templates = np.random.RandomState(99).rand(10, *shape[1:])
    y = rng.randint(0, 10, n)
    x = (0.6 * templates[y] + 0.4 * rng.rand(*shape)).astype(F32)
    return x, y.astype(F32)


def _module(name):
    from caffeonspark_b200 import nets
    return nets.lenet_tanh_module() if name == TANH else nets.cifar10_quick_prelu_module()


def _reference(name, w, x, y, dtype, device, argmax=None):
    """(loss, flat gradient, each MAX pool's argmax) of the PyTorch module on the flat weights w.  With `argmax`, every
    MAX pool takes its winners from it (the branch another forward took) instead of choosing them."""
    from caffeonspark_b200 import nets
    m = _module(name).to(device=device, dtype=dtype)
    _load(m, w)
    h, taken = torch.from_numpy(x).to(device=device, dtype=dtype), []
    for layer in m:
        if not isinstance(layer, torch.nn.MaxPool2d):
            h = layer(h)
        elif argmax is None:  # Caffe's pooled size here: pad 0, ceil mode; the first maximum wins, as in Caffe
            h, i = F.max_pool2d(h, layer.kernel_size, layer.stride, ceil_mode=True, return_indices=True)
            taken.append(i.cpu())
        else:
            i = argmax[len(taken)].to(device)
            taken.append(i.cpu())
            h = h.flatten(2).gather(2, i.flatten(2)).view(i.shape)
    yt = torch.from_numpy(y).to(device)
    loss = nets.multinomial_logistic_loss(h, yt) if name == TANH else F.cross_entropy(h, yt.long())
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def _host_weights(name, seed):
    """Flat weights uniform in [-0.1, 0.1), PReLU slopes 0.25, drawn on the host so that the bound's CPU runs use them
    too."""
    from caffeonspark_b200 import nets
    counts = [p.numel() for p in _module(name).parameters()]
    w = np.random.RandomState(seed).uniform(-0.1, 0.1, sum(counts)).astype(F32)
    off = 0
    for k, c in enumerate(counts):
        if name == PRELU and k in (2, 5, 8, 11):  # the four PReLU slope blobs
            w[off:off + c] = 0.25
        off += c
    assert w.size == (nets.LENET_TANH_PARAM_COUNT if name == TANH else nets.CIFAR10_QUICK_PRELU_PARAM_COUNT)
    return w


def _weights(net, name, seed):
    w = _host_weights(name, seed)
    net.data().copy_(torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    return w


@pytest.mark.parametrize("batch", [64, 100])
@pytest.mark.parametrize("name", [TANH, PRELU])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name, batch):
    net = _net(cos, _solver(tmp_path, name, batch=batch), fill=False)
    try:
        w = _weights(net, name, 21 + batch)
        x, y = _batch(name, batch, batch)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()], loss.data_ptr())
        assert net.synchronize(), net.last_error()
        g, l32 = to_host(net.diff()), float(loss.item())
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            lt, gt, argmax = _reference(name, w, x, y, torch.float32, "cuda")
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        l64, g64, _ = _reference(name, w, x, y, torch.float64, "cpu", argmax)
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
        off, report, bad = 0, [], False
        for k, c in enumerate(net.desc.counts):
            sl = slice(off, off + c)
            off += c
            scale = np.abs(g64[sl]).max()
            assert scale > 0, k
            errs = [np.abs(got[sl].astype(np.float64) - g64[sl]).max() / scale for got in (g, gt)]
            report.append(f"blob {k}: native {errs[0]:.2e}, PyTorch fp32 {errs[1]:.2e}")
            bad = bad or max(errs) > NET_BOUND
        assert off == g.size
        assert not bad, f"relative to max|g64| per blob, bound {NET_BOUND}: " + "; ".join(report)
    finally:
        net.deallocate()


@pytest.mark.parametrize("name", [TANH, PRELU])
def test_fixture_runs_are_bitwise_identical_and_accumulate(cos, tmp_path, name):
    net = _net(cos, _solver(tmp_path, name))
    try:
        x, y = _batch(name, 4, 64 if name == TANH else 100)
        inputs = [torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()]
        loss = torch.zeros(1, device="cuda")
        runs = []
        for _ in range(3):
            if len(runs) < 2:
                net.diff().zero_()
            torch.cuda.synchronize()
            assert net.forward_backward(inputs, loss.data_ptr()) and net.synchronize(), net.last_error()
            runs.append((to_host(net.diff()), float(loss.item())))
        assert_bits_equal(runs[0][0], runs[1][0], "diff of two runs")
        assert runs[0][1] == runs[1][1]
        assert_bits_equal(runs[2][0], F32(2) * runs[0][0], "two calls accumulate 2g")
    finally:
        net.deallocate()


def _train(net, name, steps, seed, check=None):
    losses = []
    for t in range(steps):
        x, y = _batch(name, seed + t, 64 if name == TANH else 100)
        if check:
            check.before()
        assert net.train(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", [TANH, PRELU])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    from caffeonspark_b200 import nets
    net = _net(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == (nets.LENET_TANH_PARAM_COUNT if name == TANH else
                                     nets.CIFAR10_QUICK_PRELU_PARAM_COUNT)
        if name == PRELU:  # the fixture's 1e-4 conv1 filler leaves CIFAR-10-quick at ln 10 for hundreds of steps
            _weights(net, name, 5)
        losses = _train(net, name, STEPS, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        first, last = losses[:10].mean(), losses[-20:].mean()
        assert last < first, (first, last)
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
                assert netz[r].train(0, list(_batch(name, 10 * r + t, 64 if name == TANH else 100))), \
                    netz[r].last_error()
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


@pytest.mark.parametrize("name", [TANH, PRELU])
def test_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, solver, name), _two_rank_run(cos, solver, name), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_prelu_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, PRELU, f"snapshot_format: {fmt}\n")
    a = _net(cos, solver)
    try:
        _train(a, PRELU, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        for layer, off, n in (("prelu1", 2432, 32), ("prelu3", 79392, 64), ("prelu_ip1", 145056, 1)):
            assert_bits_equal(cos.read_caffemodel_blob(model, layer, 0).ravel(), w_a[off:off + n], layer)
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, PRELU, 2, 7), _train(b, PRELU, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
