"""The siamese MNIST net on the GPU (DESIGN.md section 14): shared weights, Slice and ContrastiveLoss on the built-in
engine against float64 references, determinism and accumulation, training through train() alone with every update
checked against the oracle, two in-process ranks, and snapshots that resume bit-exact."""
import concurrent.futures as cf

import numpy as np
import pytest
import torch

from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _blob_bound, _load, _grads
from test_shared_params_host import SIAMESE_COUNTS, memory_data_copy

pytestmark = pytest.mark.gpu

NAMES = ["conv1.w", "conv1.b", "conv2.w", "conv2.b", "ip1.w", "ip1.b", "ip2.w", "ip2.b", "feat.w", "feat.b"]


def _gap_margin(d):
    """A margin in the middle of the widest gap of the sorted distances d: dissimilar pairs on both sides of it, none
    close enough for float32 rounding to move a pair across."""
    s = np.sort(d)
    lo, hi = len(s) // 4, 3 * len(s) // 4
    k = lo + int(np.argmax(s[lo + 1:hi + 1] - s[lo:hi]))
    return float((s[k] + s[k + 1]) / 2)


def _solver_with_margin(tmp_path, margin, legacy=False):
    solver = memory_data_copy(tmp_path)
    net = (tmp_path / "net.prototxt").read_text()
    (tmp_path / "net.prototxt").write_text(net.replace(
        "margin: 1\n", f"margin: {margin!r}\n" + ("    legacy_version: true\n" if legacy else "")))
    return solver


def _run(net, inputs, loss):
    assert net.forward_backward(inputs, loss.data_ptr()), net.last_error()
    assert net.synchronize(), net.last_error()
    return to_host(net.diff()), float(loss.item())


def test_siamese_gradients_match_float64(cos, tmp_path):
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(3)
    w = rng.uniform(-0.1, 0.1, nets.SIAMESE_PARAM_COUNT).astype(np.float32)
    x = rng.rand(64, 2, 28, 28).astype(np.float32)
    sim = np.tile(np.float32([1, 0, 0, 1.5, 0.7, 0, 0, 1]), 8)  # int(sim): 1.5 similar, 0.7 dissimilar
    m = nets.siamese_module().double()
    _load(m, w)
    with torch.no_grad():
        a, b = m(torch.from_numpy(x).double())
    dist = (a - b).norm(dim=1).numpy()
    margin = _gap_margin(dist[sim.astype(int) == 0])
    dis = dist[sim.astype(int) == 0]
    assert (dis < margin).sum() >= 8 and (dis > margin).sum() >= 8  # dissimilar pairs inside and outside the margin
    net = cos.CaffeNet(_solver_with_margin(tmp_path, margin), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().copy_(torch.from_numpy(w).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run(net, [torch.from_numpy(x).cuda(), torch.from_numpy(sim).cuda()], loss)
        a, b = m(torch.from_numpy(x).double())
        l64 = nets.contrastive_loss(a, b, torch.from_numpy(sim).double(), margin=margin)
        l64.backward()
        g64, l64 = _grads(m), float(l64.detach())
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        off = 0
        for c, nm in zip(SIAMESE_COUNTS, NAMES):
            sl = slice(off, off + c)
            off += c
            if nm in ("ip2.b", "feat.b"):
                # no ReLU after ip2: each pair sends g into one branch and -g into the other, so these biases' two
                # uses cancel exactly, in float64 and in the engine (negation is exact, the sums run in one order)
                assert not g64[sl].any() and not g[sl].any(), nm
                continue
            assert np.abs(g64[sl]).max() > 0, nm
            _blob_bound(g[sl], g64[sl], f"siamese {nm}")
    finally:
        net.deallocate()


LOSS_NET = """name: "t"
layer {{ name: "in" type: "Input" top: "x" top: "sim" input_param {{ shape {{ dim: {n} dim: {k} }} shape {{ dim: {n} }} }} }}
layer {{ name: "ip" type: "InnerProduct" bottom: "x" top: "h" inner_product_param {{ num_output: {h} }} }}
layer {{ name: "s" type: "Slice" bottom: "h" {tops} slice_param {{ axis: 1 {points} }} }}
layer {{ name: "loss" type: "ContrastiveLoss" bottom: "t0" bottom: "t1" bottom: "sim" top: "loss"
  loss_weight: {lw} contrastive_loss_param {{ margin: {margin!r} legacy_version: {legacy} }} }}
"""


@pytest.mark.parametrize("legacy", ["false", "true"])
@pytest.mark.parametrize("n,k,c,extra", [(5, 7, 3, 0), (64, 16, 2, 3), (300, 4, 5, 1)])  # 300 pairs > one block
def test_slice_and_contrastive_loss_match_float64(cos, tmp_path, legacy, n, k, c, extra):
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(n + k)
    x = rng.randn(n, k).astype(np.float32)
    W = (0.5 * rng.randn(2 * c + extra, k)).astype(np.float32)
    bias = (0.1 * rng.randn(2 * c + extra)).astype(np.float32)
    sim = rng.randint(0, 2, n).astype(np.float32)
    lw = 0.75
    h = torch.from_numpy(x).double() @ torch.from_numpy(W).double().T + torch.from_numpy(bias).double()
    d2 = ((h[:, :c] - h[:, c:2 * c]) ** 2).sum(1).numpy()
    margin = _gap_margin((d2 if legacy == "true" else np.sqrt(d2))[sim == 0])
    # tops t0 [0, c), t1 [c, 2c) and, with extra, an unread t2 whose gradient range stays zero
    points = f"slice_point: {c}" + (f" slice_point: {2 * c}" if extra else "")
    tops = " ".join(f'top: "t{i}"' for i in range(3 if extra else 2))
    (tmp_path / "net.prototxt").write_text(LOSS_NET.format(n=n, k=k, h=2 * c + extra, tops=tops, points=points, lw=lw,
                                                           margin=margin, legacy=legacy))
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().copy_(torch.from_numpy(np.concatenate([W.ravel(), bias])).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run(net, [torch.from_numpy(x).cuda(), torch.from_numpy(sim).cuda()], loss)
        Wd = torch.from_numpy(W).double().requires_grad_()
        bd = torch.from_numpy(bias).double().requires_grad_()
        hd = torch.from_numpy(x).double() @ Wd.T + bd
        l64 = nets.contrastive_loss(hd[:, :c], hd[:, c:2 * c], torch.from_numpy(sim).double(), margin=margin,
                                    legacy=legacy == "true", loss_weight=lw)
        l64.backward()
        l64 = float(l64.detach())
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        gW, gb = Wd.grad.numpy(), bd.grad.numpy()
        _blob_bound(g[:W.size], gW.ravel(), "ip weight")
        _blob_bound(g[W.size:], gb, "ip bias")
        if extra:  # the unread top's rows of the weight gradient
            assert not g[:W.size].reshape(W.shape)[2 * c:].any()
    finally:
        net.deallocate()


def _pairs(rng, templates, n=64):
    """Synthetic pairs: a pair is similar (sim 1) when both halves come from the same class template."""
    y1 = rng.randint(0, 10, n)
    same = rng.rand(n) < 0.5
    y2 = np.where(same, y1, (y1 + rng.randint(1, 10, n)) % 10)
    x = np.stack([0.6 * templates[y1] + 0.4 * rng.rand(n, 28, 28), 0.6 * templates[y2] + 0.4 * rng.rand(n, 28, 28)], 1)
    return x.astype(np.float32), same.astype(np.float32)


def test_runs_are_bitwise_identical_and_accumulate(cos, tmp_path):
    net = cos.CaffeNet(memory_data_copy(tmp_path), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=True)
        x, sim = _pairs(np.random.RandomState(4), np.random.RandomState(99).rand(10, 28, 28))
        inputs = [torch.from_numpy(x).cuda(), torch.from_numpy(sim).cuda()]
        loss = torch.zeros(1, device="cuda")
        runs = []
        for _ in range(2):
            net.diff().zero_()
            torch.cuda.synchronize()
            runs.append(_run(net, inputs, loss))
        assert_bits_equal(runs[0][0], runs[1][0], "diff of two runs")
        assert runs[0][1] == runs[1][1]
        g2, _ = _run(net, inputs, loss)
        # no clearing: every use adds its gradient once more.  Each shared blob takes two additions per call (one per
        # branch), so the sum equals 2g up to the rounding of those additions, and is itself repeatable.
        off = 0
        for c, nm in zip(SIAMESE_COUNTS, NAMES):
            sl = slice(off, off + c)
            off += c
            g = runs[0][0][sl]
            if nm in ("ip2.b", "feat.b"):  # the two uses cancel exactly (see test_siamese_gradients_match_float64)
                assert not g.any() and not g2[sl].any(), nm
                continue
            assert np.abs(g2[sl] - 2 * g).max() <= 1e-5 * np.abs(g).max(), nm
        net.diff().zero_()
        torch.cuda.synchronize()
        _run(net, inputs, loss)
        assert_bits_equal(_run(net, inputs, loss)[0], g2, "two calls without a clear, repeated")
    finally:
        net.deallocate()


def _train(net, steps, seed, check=None):
    rng = np.random.RandomState(seed)
    templates = np.random.RandomState(99).rand(10, 28, 28)
    losses = []
    for t in range(steps):
        x, sim = _pairs(rng, templates)
        if check:
            check.before()
        assert net.train(0, [x, sim]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


def test_train_through_train_alone(cos, oracle, tmp_path):
    """The reference's siamese prototxt and nothing else (with MemoryData): xavier fillers, the inv policy.  Every
    update equals the oracle's bit for bit, and the loss falls."""
    net = cos.CaffeNet(memory_data_copy(tmp_path), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        assert net.param_count() == 431102
        net.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        w0 = to_host(net.data())
        assert np.abs(w0[:500]).max() > 0 and not w0[500:520].any()  # conv1 xavier, its bias constant 0
        losses = _train(net, 300, 1, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-50:].mean() < 0.7 * losses[:10].mean(), (losses[:10].mean(), losses[-50:].mean())
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
        templates = np.random.RandomState(99).rand(10, 28, 28)
        batches = [_pairs(np.random.RandomState(10 + r), templates) for r in range(2)]

        def run(r):
            for _ in range(6):
                assert netz[r].train(0, list(batches[r])), netz[r].last_error()
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


def test_two_ranks_in_process(cos, tmp_path):
    solver = memory_data_copy(tmp_path)
    assert_bits_equal(_two_rank_run(cos, solver), _two_rank_run(cos, solver), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshots_list_shared_layers_and_resume_bit_exact(cos, tmp_path, fmt):
    solver = memory_data_copy(tmp_path)
    text = open(solver).read().replace('snapshot_prefix: "examples/siamese/mnist_siamese"',
                                       f'snapshot_prefix: "{tmp_path}/snap"') + f"snapshot_format: {fmt}\n"
    open(solver, "w").write(text)
    a = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert a.connect(a.localAddresses())
        a.use_native_producer(fill_weights=True)
        _train(a, 3, 5)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        off = np.cumsum([0] + SIAMESE_COUNTS)
        for i, layer in enumerate(["conv1", "conv2", "ip1", "ip2", "feat"]):
            for j in range(2):
                want = w_a[off[2 * i + j]:off[2 * i + j + 1]]
                assert_bits_equal(cos.read_caffemodel_blob(model, layer, j), want, f"{layer} blob {j}")
                if fmt == "BINARYPROTO":  # Net::ToProto: the sharer holds its owner's data
                    assert_bits_equal(cos.read_caffemodel_blob(model, layer + "_p", j), want, f"{layer}_p blob {j}")
            if fmt == "HDF5":  # Net::ToHDF5 writes only blobs that own themselves
                with pytest.raises(cos.CosError):
                    cos.read_caffemodel_blob(model, layer + "_p", 0)
        _, _, _, hist = cos.read_solverstate(state)
        assert [h.size for h in hist] == SIAMESE_COUNTS  # history for owners only
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, 2, 6), _train(b, 2, 6)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
