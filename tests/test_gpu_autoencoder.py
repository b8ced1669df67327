"""Deconvolution, Flatten and SigmoidCrossEntropyLoss on the built-in engine (DESIGN.md section 14) on the GPU: each op
alone against the float64 references of autoencoder_ops_ref.py (through test_gpu_producer_ops.py's injector harness),
both autoencoder fixtures at batch 100 against float64 and PyTorch fp32, determinism and the accumulate contract,
training through train() alone with every update checked against the oracle, two in-process ranks, iter_size 2, and
snapshots that resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch

import autoencoder_ops_ref as A
import producer_ops_ref as R
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_least_squares import _near
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import FAMILIES, _check, _close, _engine, _exact_depth, _forward, _probe

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
FC = "mnist_autoencoder"
CONV = "mnist_conv_autoencoder"
# The whole nets' per-blob gradient bound (relative to the blob's largest float64 gradient), fixed before any GPU run
# from CPU runs of nets.autoencoder_module / conv_autoencoder_module in fp32 against float64, three seeds on weights of
# the fixtures' filler distributions (the FC net's sparse Gaussian included) and these images: the worst blob reached
# 7.1e-7 (FC) and 4.1e-6 (conv).  The loss keeps 1e-5 (the CPU runs: 7.5e-8).
NET_BOUND = 1e-4
STEPS = 150
# fixed before any GPU run: CPU runs of the two modules with the fixtures' solvers on these images end (mean of the
# last 20 of 150 steps) at 0.45 to 0.76 (FC) and 0.45 (conv) of the mean of the first 10, four seeds each
LOSS_RATIO = {FC: 0.9, CONV: 0.7}


def _images(seed, n=100):
    """Seeded MNIST-like batches in [0, 1]: one of ten blocky binary templates, scaled, plus noise."""
    rng = np.random.RandomState(seed)
    templates = np.kron(np.random.RandomState(99).rand(10, 7, 7) > 0.6, np.ones((4, 4)))
    y = rng.randint(0, 10, n)
    x = templates[y] * rng.uniform(0.6, 1.0, (n, 1, 1)) + 0.15 * rng.rand(n, 28, 28)
    return np.clip(x, 0, 1).astype(F32)[:, None]


def _solver(tmp_path, name, extra="", batch=None):
    """The fixture's solver, pointed at the fixture's net (a copy with another batch size when `batch` is given)."""
    net = os.path.join(CONFIGS, f"{name}_train_test.prototxt")
    if batch is not None:
        text = open(net).read().replace("batch_size: 100\n", f"batch_size: {batch}\n")
        net = str(tmp_path / f"{name}_b{batch}.prototxt")
        open(net, "w").write(text)
    text = open(os.path.join(CONFIGS, f"{name}_solver.prototxt")).read()
    text = text.replace(f'net: "{name}_train_test.prototxt"', f'net: "{net}"')
    text = text.replace(f'snapshot_prefix: "{name}"', f'snapshot_prefix: "{tmp_path}/snap"')
    path = tmp_path / f"{name}_{batch}_solver.prototxt"
    path.write_text(text + extra)
    return str(path)


def _net(cos, solver):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=True)
    torch.cuda.synchronize()
    return net


def _run(net, inputs, loss):
    assert net.forward_backward(inputs, loss.data_ptr()), net.last_error()
    assert net.synchronize(), net.last_error()
    return to_host(net.diff()), float(loss.item())


# --------------------------------------------------------------------------- Deconvolution
def _deconv_layer(cout, geo, bias):
    kh, kw, sh, sw, ph, pw = geo
    return (f'layer {{ name: "dc" type: "Deconvolution" bottom: "x0" top: "y" convolution_param {{ num_output: {cout} '
            f'kernel_h: {kh} kernel_w: {kw} stride_h: {sh} stride_w: {sw} pad_h: {ph} pad_w: {pw} '
            f'bias_term: {"true" if bias else "false"} }} }}\n')


DECONV_CASES = [  # (N, Cin, H, W, Cout, (kh, kw, sh, sw, ph, pw), bias)
    (2, 3, 5, 5, 4, (3, 3, 1, 1, 0, 0), True),
    (2, 3, 5, 5, 4, (3, 3, 1, 1, 1, 1), True),
    (2, 4, 7, 7, 3, (4, 4, 2, 2, 1, 1), True),  # the conv autoencoder's upsampling
    (2, 4, 6, 6, 3, (4, 4, 2, 2, 1, 1), False),
    (2, 3, 4, 5, 2, (3, 3, 3, 3, 0, 0), True),  # stride = kernel: no overlap
    (2, 3, 4, 4, 2, (2, 2, 3, 3, 0, 0), True),  # stride > kernel: some outputs are the bias alone
    (2, 2, 5, 4, 3, (5, 5, 2, 2, 2, 2), True),
    (2, 3, 5, 6, 4, (2, 5, 1, 2, 0, 2), True),  # non-square kernel and strides
    (2, 3, 6, 3, 2, (5, 2, 3, 1, 2, 0), False),
    (1, 5, 3, 3, 65, (2, 2, 2, 2, 0, 0), True),  # Cout across the 64-row tile edge of the forward
    (1, 65, 3, 3, 2, (1, 1, 1, 1, 0, 0), True),  # Cin across it for the data gradient
    (2, 2, 20, 20, 2, (3, 3, 1, 1, 1, 1), True),  # N H W = 800: two chunks of the weight gradient
    (1, 2, 3, 43691, 2, (1, 1, 1, 1, 0, 0), True),  # N H W = 131,073: 249 widened chunks of 528
    (256, 2, 55, 55, 2, (1, 1, 1, 1, 0, 0), True),  # N H W = 774,400: 255 chunks of 3,040
]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n,cin,h,w,cout,geo,bias", DECONV_CASES)
def test_deconvolution(cos, tmp_path, family, n, cin, h, w, cout, geo, bias):
    rng = np.random.RandomState(n * 1000 + cin * 100 + cout + h + sum(geo))
    exact = family == "dyadic"
    kh, kw = geo[:2]
    x = R.dyadic(rng, (n, cin, h, w)) if exact else R.gaussian(rng, (n, cin, h, w))
    if exact:
        wt, b = R.dyadic(rng, (cin, cout, kh, kw), bits=4), R.dyadic(rng, (cout,), bits=7)
    else:
        wt, b = R.gaussian(rng, (cin, cout, kh, kw), 1 / np.sqrt(cin * kh * kw)), R.gaussian(rng, (cout,), 0.1)
    b = b if bias else None
    y64 = A.deconv_forward(x, wt, b, geo)
    B = _probe(y64, rng, family)
    r = _engine(cos, tmp_path, [x], _deconv_layer(cout, geo, bias), [wt] + ([b] if bias else []), y64.shape, B)
    d = r["d"]
    if exact:  # x and d are dyadic in 2^-3
        adw, adb, _ = A.deconv_backward(np.abs(x), np.abs(wt), np.abs(d), geo)
        _exact_depth(adw, 2.0 ** -6, "dW")
        _exact_depth(adb, 2.0 ** -3, "db")
    by, bw, bb, bx = A.deconv_bounds(x, wt, b, d, geo)
    _forward(d, y64, B, by, "y", exact)
    dw, db, dx = A.deconv_backward(x, wt, d, geo)
    _check(r["grads"][0], dw, bw, "dW", exact)
    if bias:
        _check(r["grads"][1], db, bb, "db", exact)
    _check(r["dx"][0], dx, bx, "dx", exact)
    assert np.abs(dw).max() > 0 and np.abs(dx).max() > 0


# --------------------------------------------------------------------------- Flatten
IP = ('layer {{ name: "ip" type: "InnerProduct" bottom: "{}" top: "y" inner_product_param {{ num_output: 5 '
      'bias_term: false }} }}\n')


def test_flatten_is_no_copy_either_way(cos, tmp_path):
    """x0 -> Flatten -> InnerProduct gives every value bit for bit as InnerProduct straight on x0 (which reads its
    bottom flattened), the data gradient included: the top shares the bottom's data and diff."""
    rng = np.random.RandomState(5)
    x, wt = R.gaussian(rng, (3, 2, 4, 5)), R.gaussian(rng, (5, 40), 0.2)
    y64 = R.ip_forward(x, wt, None)
    B = _probe(y64, rng, "gaussian")
    runs = []
    for i, body in enumerate(['layer { name: "f" type: "Flatten" bottom: "x0" top: "f" }\n' + IP.format("f"),
                              IP.format("x0")]):
        (tmp_path / str(i)).mkdir()
        runs.append(_engine(cos, tmp_path / str(i), [x], body, [wt], y64.shape, B))
    assert_bits_equal(runs[0]["d"], runs[1]["d"], "d")
    assert_bits_equal(runs[0]["dx"][0], runs[1]["dx"][0], "dx")
    assert_bits_equal(runs[0]["grads"][0], runs[1]["grads"][0], "dW")
    assert runs[0]["dx"][0].shape == x.shape and np.abs(runs[0]["dx"][0]).max() > 0


# --------------------------------------------------------------------------- SigmoidCrossEntropyLoss
def _sce_inputs(rng, kind, shape):
    if kind == "large":  # |x| from 40 to 200: exp(-|x|) is tiny or underflows, sigmoid is 0 or 1 exactly
        x = (rng.choice([-1, 1], shape) * rng.uniform(40, 200, shape)).astype(F32)
        x.flat[::7] = R.gaussian(rng, x.flat[::7].shape)
    else:
        x = R.gaussian(rng, shape, 3.0)
    t = (rng.rand(*shape) < 0.4).astype(F32) if kind in ("binary", "large") else rng.rand(*shape).astype(F32)
    return x, t


@pytest.mark.parametrize("kind", ["binary", "soft", "large"])
@pytest.mark.parametrize("shape,loss_weight", [((4, 3, 5, 7), 1.0), ((3, 10), 2.5), ((100, 784), 1.0),
                                               ((3, 200000), 0.5)])  # the last: more elements than the grid's threads
def test_sigmoid_cross_entropy(cos, tmp_path, kind, shape, loss_weight):
    rng = np.random.RandomState(len(kind) * 10 + len(shape) + shape[0])
    x, t = _sce_inputs(rng, kind, shape)
    body = (f'layer {{ name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "x0" bottom: "t" top: "l" '
            f'loss_weight: {loss_weight} }}')
    r = _engine(cos, tmp_path, [x], body, staged={"t": t})
    l64, dx64 = A.sigmoid_xent(x, t, shape[0], loss_weight)
    lb, dxb = A.sigmoid_xent_bounds(x, t, shape[0], loss_weight)
    assert abs(r["loss"] - l64) <= lb, (r["loss"], l64, lb)
    _close(r["dx"][0], dx64, dxb, "dx")
    if kind == "large":
        sat = np.abs(x) >= 40
        assert_bits_equal(r["dx"][0][sat], ((x[sat] > 0).astype(F32) - t[sat]) * F32(F32(loss_weight) / F32(shape[0])),
                          "saturated sigmoid: dx = ([x > 0] - t) * loss_weight / num exactly")


def test_sigmoid_cross_entropy_passes_non_finite_inputs_to_the_loss(cos, tmp_path):
    rng = np.random.RandomState(3)
    x, t = _sce_inputs(rng, "soft", (4, 6))
    x[1, 2] = np.nan
    body = 'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "x0" bottom: "t" top: "l" }'
    r = _engine(cos, tmp_path, [x], body, staged={"t": t})  # no error from synchronize: as in Caffe
    assert np.isnan(r["loss"]) and np.isnan(r["dx"][0][1, 2]) and np.isfinite(np.delete(r["dx"][0].ravel(), 8)).all()


def test_a_flattened_target_and_a_dead_branch_change_nothing(cos, tmp_path):
    """The FC autoencoder's pattern in small: a Flatten of a staged target, and a Sigmoid + zero-weight EuclideanLoss
    hanging off a Split of the scores.  Their gradients are those of the net without them, bit for bit."""
    rng = np.random.RandomState(8)
    x, wt = R.gaussian(rng, (4, 6)), R.gaussian(rng, (12, 6), 0.5)
    t = rng.rand(4, 3, 2, 2).astype(F32)
    ip = ('layer { name: "ip" type: "InnerProduct" bottom: "x0" top: "s" inner_product_param { num_output: 12 '
          'bias_term: false } }\n')
    plain = ip + ('layer { name: "ft" type: "Flatten" bottom: "t" top: "tf" }\n'
                  'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "s" bottom: "tf" top: "l" }')
    dead = ip + ('layer { name: "sp" type: "Split" bottom: "s" top: "s0" top: "s1" }\n'
                 'layer { name: "ft" type: "Flatten" bottom: "t" top: "tf" }\n'
                 'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "s0" bottom: "tf" top: "l" }\n'
                 'layer { name: "g" type: "Sigmoid" bottom: "s1" top: "g" }\n'
                 'layer { name: "l2" type: "EuclideanLoss" bottom: "g" bottom: "tf" top: "l2" loss_weight: 0 }')
    runs = []
    for i, body in enumerate([plain, dead]):
        (tmp_path / str(i)).mkdir()
        runs.append(_engine(cos, tmp_path / str(i), [x], body, [wt], staged={"t": t}))
    assert runs[0]["loss"] == runs[1]["loss"]
    assert_bits_equal(runs[0]["grads"][0], runs[1]["grads"][0], "dW")
    assert_bits_equal(runs[0]["dx"][0], runs[1]["dx"][0], "dx")
    l64, _ = A.sigmoid_xent(x @ wt.T.astype(np.float64), t.reshape(4, -1), 4)
    assert abs(runs[0]["loss"] - l64) <= 1e-5 * abs(l64)


# --------------------------------------------------------------------------- the fixtures
def _module(name):
    from caffeonspark_b200 import nets
    return nets.autoencoder_module() if name == FC else nets.conv_autoencoder_module()


def _reference(name, w, x, dtype, device):
    from caffeonspark_b200 import nets
    m = _module(name).to(device=device, dtype=dtype)
    _load(m, w)
    xx = torch.from_numpy(x).to(device=device, dtype=dtype)
    loss = nets.sigmoid_cross_entropy_loss(m(xx), xx)
    loss.backward()
    return float(loss.detach()), _grads(m)


@pytest.mark.parametrize("name", [FC, CONV])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name):
    net = _net(cos, _solver(tmp_path, name))
    try:
        w = to_host(net.data())
        x = _images(3)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run(net, [torch.from_numpy(x).cuda()], loss)
        l64, g64 = _reference(name, w, x, torch.float64, "cpu")
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            lt, gt = _reference(name, w, x, torch.float32, "cuda")
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
        off = 0
        for k, c in enumerate(net.desc.counts):
            sl = slice(off, off + c)
            off += c
            assert np.abs(g64[sl]).max() > 0, k
            for got, what in ((g, "native"), (gt, "PyTorch fp32")):
                err, scale = np.abs(got[sl].astype(np.float64) - g64[sl]).max(), np.abs(g64[sl]).max()
                assert err <= NET_BOUND * scale, f"blob {k} {what}: {err:.3e} > {NET_BOUND} * {scale:.3e}"
        assert off == g.size
    finally:
        net.deallocate()


def test_sparse_gaussian_filler(cos, tmp_path):
    """filler.hpp's sparse: each weight of the FC autoencoder keeps its Gaussian draw with probability 15 / shape(0) and
    is 0 otherwise; the kept values are the dense filler's, bit for bit, and the biases are untouched."""
    sparse = _net(cos, _solver(tmp_path, FC))
    try:
        w = to_host(sparse.data())
        counts = sparse.desc.counts
    finally:
        sparse.deallocate()
    (tmp_path / "dense").mkdir()
    dense_net = tmp_path / "dense" / f"{FC}_train_test.prototxt"
    dense_net.write_text(open(os.path.join(CONFIGS, f"{FC}_train_test.prototxt")).read().replace("sparse: 15", ""))
    text = open(os.path.join(CONFIGS, f"{FC}_solver.prototxt")).read()
    (tmp_path / "dense" / "solver.prototxt").write_text(text.replace(f'net: "{FC}_train_test.prototxt"',
                                                                     f'net: "{dense_net}"'))
    dense = _net(cos, str(tmp_path / "dense" / "solver.prototxt"))
    try:
        d = to_host(dense.data())
    finally:
        dense.deallocate()
    widths = [784, 1000, 500, 250, 30, 250, 500, 1000, 784]
    off = 0
    for k, c in enumerate(counts):
        sl = slice(off, off + c)
        off += c
        if k % 2:  # a bias: constant 0 either way
            assert not w[sl].any() and not d[sl].any()
            continue
        kept = w[sl] != 0
        assert_bits_equal(w[sl][kept], d[sl][kept], f"blob {k}: kept values")
        p = 15 / widths[k // 2 + 1]  # shape(0) of an InnerProduct weight is its num_output
        assert abs(kept.mean() - p) <= 6 * np.sqrt(p * (1 - p) / c), (k, kept.mean(), p)


@pytest.mark.parametrize("name", [FC, CONV])
def test_fixture_runs_are_bitwise_identical_and_accumulate(cos, tmp_path, name):
    net = _net(cos, _solver(tmp_path, name))
    try:
        inputs = [torch.from_numpy(_images(4)).cuda()]
        loss = torch.zeros(1, device="cuda")
        runs = []
        for _ in range(2):
            net.diff().zero_()
            torch.cuda.synchronize()
            runs.append(_run(net, inputs, loss))
        assert_bits_equal(runs[0][0], runs[1][0], "diff of two runs")
        assert runs[0][1] == runs[1][1]
        g2, _ = _run(net, inputs, loss)  # no clearing: diff += g once more
        assert_bits_equal(g2, np.float32(2) * runs[0][0], "two calls accumulate 2g")
    finally:
        net.deallocate()


def _train(net, check=None, steps=STEPS, seed=1000):
    losses = []
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, [_images(seed + t)]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", [FC, CONV])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    from caffeonspark_b200 import nets
    net = _net(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == (nets.AUTOENCODER_PARAM_COUNT if name == FC else nets.CONV_AUTOENCODER_PARAM_COUNT)
        losses = _train(net, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        first, last = losses[:10].mean(), losses[-20:].mean()
        assert last < LOSS_RATIO[name] * first, (first, last)
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
                assert netz[r].train(0, [_images(10 * r + t)]), netz[r].last_error()
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
    solver = _solver(tmp_path, CONV)
    assert_bits_equal(_two_rank_run(cos, solver), _two_rank_run(cos, solver), "two whole runs")


def test_iter_size_two_matches_one_pass_over_both_halves(cos, tmp_path):
    """iter_size 2 over two batches of 100 against iter_size 1 over the same 200 images, from the same weights:
    SigmoidCrossEntropyLoss divides by num, so the two gradients agree up to rounding."""
    one = _net(cos, _solver(tmp_path, CONV, batch=200))
    two = _net(cos, _solver(tmp_path, CONV, "iter_size: 2\n"))
    try:
        assert two.desc.iter_size == 2
        two.data().copy_(one.data())
        torch.cuda.synchronize()
        for t in range(4):
            x = _images(50 + t, 200)
            assert one.train(0, [x]), one.last_error()
            assert two.train_accumulate(0, [[x[:100]], [x[100:]]]), two.last_error()
            assert one.synchronize() and two.synchronize()
        _near(to_host(two.data()), to_host(one.data()), "iter_size 2 against one pass over 200 images")
    finally:
        one.deallocate()
        two.deallocate()


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshots_hold_deconvolution_blobs_and_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, CONV, f"snapshot_format: {fmt}\n")
    a = _net(cos, solver)
    try:
        _train(a, steps=3)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        for layer, index, off, n in (("deconv1", 0, 4800, 8192), ("deconv1", 1, 12992, 16), ("deconv2", 0, 13008, 256)):
            assert_bits_equal(cos.read_caffemodel_blob(model, layer, index), w_a[off:off + n], f"{layer} blob {index}")
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, steps=2, seed=7), _train(b, steps=2, seed=7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
