"""Split, Eltwise and Scale on the built-in engine (DESIGN.md section 14) on the GPU: each op alone against float64,
Eltwise MAX's tie rule by equality, the ResNet-20 fixture against float64 and PyTorch fp32, determinism and the
accumulate contract, training through train() alone with every update checked against the oracle, two in-process
ranks, and snapshots that hold each Scale layer's two blobs and resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_bf16_producer import _task_batches
from test_gpu_native_producer import _UpdateCheck, _blob_bound, _grads, _load, _params

pytestmark = pytest.mark.gpu

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
NET = os.path.join(CONFIGS, "cifar10_resnet20_train_test.prototxt")
# The whole net's per-blob gradient bound, fixed before any GPU run from CPU runs of the PyTorch composition in fp32
# against float64, four seeds on weights of the fixture's filler distributions: the worst blob reached 2.3e-2 *
# max|g64| (in the 16- and 32-channel stages, where each BatchNorm backward cancels most of its input), so 1e-4 holds
# for neither fp32 arm and both take 5e-2.  The loss keeps 1e-5 (the CPU runs: 5e-8) and the BatchNorm statistics
# 1e-4 (4e-7).
NET_BOUND = 5e-2
STEPS = 150
# fixed before any GPU run: a CPU run of nets.resnet20_module with the fixture's solver, fillers of the same
# distributions and these batches falls by 0.70 and 0.68 from the mean of the first 10 steps to that of the last 50
# (two seeds)
LOSS_DROP = 0.3


def _solver(tmp_path, extra=""):
    text = open(os.path.join(CONFIGS, "cifar10_resnet20_solver.prototxt")).read()
    text = text.replace('net: "cifar10_resnet20_train_test.prototxt"', f'net: "{NET}"')
    text = text.replace('snapshot_prefix: "cifar10_resnet20"', f'snapshot_prefix: "{tmp_path}/snap"')
    (tmp_path / "solver.prototxt").write_text(text + extra)
    return str(tmp_path / "solver.prototxt")


def _run(net, inputs, loss):
    assert net.forward_backward(inputs, loss.data_ptr()), net.last_error()
    assert net.synchronize(), net.last_error()
    return to_host(net.diff()), float(loss.item())


def _op_net(cos, tmp_path, body, shapes, weights, inputs):
    """Runs a net of Input tops x (and t) of `shapes`, then `body`, once on the engine with `weights` as data_;
    -> (flat gradient, loss)."""
    dims = " ".join("shape { " + " ".join(f"dim: {d}" for d in s) + " }" for s in shapes)
    tops = " ".join(f'top: "{t}"' for t in ("x", "t")[:len(shapes)])
    (tmp_path / "net.prototxt").write_text(f'name: "t" layer {{ name: "in" type: "Input" {tops} input_param {{ {dims} '
                                           f'}} }}\n{body}\n')
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        w = np.concatenate([v.ravel() for v in weights]).astype(np.float32)
        assert net.param_count() == w.size
        net.data().copy_(torch.from_numpy(w).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        return _run(net, [torch.from_numpy(v).cuda() for v in inputs], loss)
    finally:
        net.deallocate()


def _conv(name, bottom, top, cout):
    return (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{top}" convolution_param {{ '
            f'num_output: {cout} kernel_size: 1 bias_term: false }} }}\n')


def _c1(w, x):  # 1x1 convolution
    return torch.einsum("oc,nchw->nohw", w, x)


def _d(a):
    return torch.from_numpy(a).double().requires_grad_()


def _check(g, l32, params, l64):
    """The engine's loss and each learnable blob's gradient against float64."""
    l64.backward()
    assert abs(l32 - float(l64)) <= 1e-5 * abs(float(l64)), (l32, float(l64))
    off = 0
    for i, p in enumerate(params):
        n = p.numel()
        assert np.abs(p.grad.numpy()).max() > 0, f"blob {i}"
        _blob_bound(g[off:off + n], p.grad.numpy().ravel(), f"blob {i}")
        off += n
    assert off == g.size


N, C, H, W = 4, 3, 5, 6


@pytest.mark.parametrize("ntops,unread", [(2, False), (3, True)])
def test_split_matches_float64(cos, tmp_path, ntops, unread):
    rng = np.random.RandomState(ntops)
    x = rng.randn(N, C, H, W).astype(np.float32)
    w0, wa, wb = (rng.randn(4, C) * 0.5).astype(np.float32), rng.randn(2, 4).astype(np.float32), \
        rng.randn(2, 4).astype(np.float32)
    tops = 'top: "a" top: "b"' + (' top: "u"' if unread else "")
    body = (_conv("c0", "x", "h", 4) + f'layer {{ name: "sp" type: "Split" bottom: "h" {tops} }}\n' +
            _conv("ca", "a", "pa", 2) + _conv("cb", "b", "pb", 2) +
            'layer { name: "loss" type: "EuclideanLoss" bottom: "pa" bottom: "pb" }')
    g, l32 = _op_net(cos, tmp_path, body, [(N, C, H, W)], [w0, wa, wb], [x])
    p = [_d(w0), _d(wa), _d(wb)]
    h = _c1(p[0], torch.from_numpy(x).double())
    _check(g, l32, p, ((_c1(p[1], h) - _c1(p[2], h)) ** 2).sum() / N / 2)


def _eltwise_net(k, param):
    body = f'layer {{ name: "sp" type: "Split" bottom: "x" ' + " ".join(f'top: "x{i}"' for i in range(k)) + " }\n"
    body += "".join(_conv(f"c{i}", f"x{i}", f"h{i}", 2) for i in range(k))
    body += ('layer { name: "e" type: "Eltwise" ' + " ".join(f'bottom: "h{i}"' for i in range(k)) +
             f' top: "y" eltwise_param {{ {param} }} }}\n')
    return body + 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" }'


def _eltwise_ref(op, hs, coeffs=None, stable=True):
    if op == "SUM":
        y = coeffs[0] * hs[0]
        for c, h in zip(coeffs[1:], hs[1:]):
            y = y + c * h
        return y
    if op == "PROD":
        class Prod(torch.autograd.Function):  # eltwise_layer.cpp's backward, stable or top / bottom
            @staticmethod
            def forward(ctx, *hs):
                y = hs[0]
                for h in hs[1:]:
                    y = y * h
                ctx.save_for_backward(y, *hs)
                return y

            @staticmethod
            def backward(ctx, dy):
                y, *hs = ctx.saved_tensors
                out = []
                for i in range(len(hs)):
                    if stable:
                        o = torch.ones_like(y)
                        for j, h in enumerate(hs):
                            o = o * h if j != i else o
                    else:
                        o = y / hs[i]
                    out.append(o * dy)
                return tuple(out)
        return Prod.apply(*hs)
    y, idx = torch.where(hs[0] > hs[1], hs[0], hs[1]), (hs[0] <= hs[1]).long()
    for i, h in enumerate(hs[2:], start=2):
        idx = torch.where(h > y, i, idx)
        y = torch.where(h > y, h, y)
    return y


@pytest.mark.parametrize("op,k,param,coeffs,stable", [
    ("SUM", 2, "coeff: 0.5 coeff: -2", [0.5, -2.0], True),
    ("SUM", 3, "operation: SUM coeff: 1 coeff: -1.5 coeff: 1", [1.0, -1.5, 1.0], True),
    ("PROD", 2, "operation: PROD", None, True),
    ("PROD", 3, "operation: PROD", None, True),
    ("PROD", 3, "operation: PROD stable_prod_grad: false", None, False),
    ("MAX", 2, "operation: MAX", None, True),
    ("MAX", 3, "operation: 2", None, True),
])
def test_eltwise_matches_float64(cos, tmp_path, op, k, param, coeffs, stable):
    rng = np.random.RandomState(k + len(param))
    x, t = rng.randn(N, C, H, W).astype(np.float32), rng.randn(N, 2, H, W).astype(np.float32)
    ws = [rng.randn(2, C).astype(np.float32) for _ in range(k)]
    g, l32 = _op_net(cos, tmp_path, _eltwise_net(k, param), [(N, C, H, W), (N, 2, H, W)], ws, [x, t])
    p = [_d(w) for w in ws]
    hs = [_c1(w, torch.from_numpy(x).double()) for w in p]
    y = _eltwise_ref(op, hs, coeffs, stable)
    _check(g, l32, p, ((y - torch.from_numpy(t).double()) ** 2).sum() / N / 2)


@pytest.mark.parametrize("k", [2, 3])
def test_eltwise_max_ties_go_by_caffes_rule(cos, tmp_path, k):
    """Every branch computes the same values exactly: bottom 1 beats bottom 0 on the tie, and bottom 2 needs a strict
    > to take over, so the whole gradient reaches bottom 1's branch alone."""
    rng = np.random.RandomState(9)
    x, t = rng.randn(N, C, H, W).astype(np.float32), rng.randn(N, 2, H, W).astype(np.float32)
    w = rng.randn(2, C).astype(np.float32)
    g, l32 = _op_net(cos, tmp_path, _eltwise_net(k, "operation: MAX"), [(N, C, H, W), (N, 2, H, W)], [w] * k, [x, t])
    one, _ = _op_net(cos, tmp_path, _conv("c", "x", "y", 2) +
                     'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" }',
                     [(N, C, H, W), (N, 2, H, W)], [w], [x, t])
    n = w.size
    assert not g[:n].any() and not g[2 * n:].any()
    assert_bits_equal(g[n:2 * n], one, "the winning branch's gradient is the single branch's")


SCALE_CASES = [  # (scale_param, scale blob shape, bias, in place)
    ("bias_term: true", (4,), True, True),
    ("", (4,), False, False),
    ("num_axes: 0 bias_term: true", (), True, False),
    ("num_axes: -1 bias_term: true", (4, H, W), True, True),
    ("axis: 2 num_axes: 2 bias_term: true", (H, W), True, False),
    ("axis: 2", (H,), False, False),
]


@pytest.mark.parametrize("param,shape,bias,in_place", SCALE_CASES)
def test_scale_matches_float64(cos, tmp_path, param, shape, bias, in_place):
    rng = np.random.RandomState(len(param) + len(shape))
    x, t = rng.randn(N, C, H, W).astype(np.float32), rng.randn(N, 4, H, W).astype(np.float32)
    w = rng.randn(4, C).astype(np.float32)
    s = rng.uniform(0.5, 1.5, shape).astype(np.float32)
    b = np.asarray(rng.randn(*shape), dtype=np.float32)
    top = "h" if in_place else "y"
    body = (_conv("c", "x", "h", 4) + f'layer {{ name: "sc" type: "Scale" bottom: "h" top: "{top}" '
            f'scale_param {{ {param} }} }}\n' +
            f'layer {{ name: "loss" type: "EuclideanLoss" bottom: "{top}" bottom: "t" }}')
    weights = [w, s] + ([b] if bias else [])
    g, l32 = _op_net(cos, tmp_path, body, [(N, C, H, W), (N, 4, H, W)], weights, [x, t])
    p = [_d(v) for v in weights]
    axis = 2 if "axis: 2" in param else 1
    view = (1,) * axis + shape + (1,) * (4 - axis - len(shape)) if shape else (1, 1, 1, 1)
    y = _c1(p[0], torch.from_numpy(x).double()) * p[1].reshape(view)
    if bias:
        y = y + p[2].reshape(view)
    _check(g, l32, p, ((y - torch.from_numpy(t).double()) ** 2).sum() / N / 2)


# --------------------------------------------------------------------------- the ResNet-20 fixture
def _net(cos, solver):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=True)
    torch.cuda.synchronize()
    return net


def _batch(seed):
    rng = np.random.RandomState(seed)
    return rng.rand(100, 3, 32, 32).astype(np.float32), rng.randint(0, 10, 100).astype(np.float32)


def _reference(w, x, y, dtype, device):
    from caffeonspark_b200 import nets
    m = nets.resnet20_module().to(device=device, dtype=dtype)
    _load(m, w)
    loss = F.cross_entropy(m(torch.from_numpy(x).to(device=device, dtype=dtype)), torch.from_numpy(y).long().to(device))
    loss.backward()
    return float(loss.detach()), _grads(m), _params(m)


def test_resnet20_matches_float64_and_pytorch(cos, tmp_path):
    net = _net(cos, _solver(tmp_path))
    try:
        w = to_host(net.data())
        x, y = _batch(3)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run(net, [torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()], loss)
        data_after = to_host(net.data())
        l64, g64, p64 = _reference(w, x, y, torch.float64, "cpu")
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            lt, gt, _ = _reference(w, x, y, torch.float32, "cuda")
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
        off, stats = 0, 0
        for k, c in enumerate(net.desc.counts):
            sl = slice(off, off + c)
            off += c
            if net.desc.lr_mult[k] == 0:  # BatchNorm statistics: no gradient, and the forward wrote them
                assert not g[sl].any(), k
                _blob_bound(data_after[sl], p64[sl], f"blob {k} statistics")
                stats += c
                continue
            assert np.abs(g64[sl]).max() > 0, k
            for got, what in ((g, "native"), (gt, "PyTorch fp32")):
                err, scale = np.abs(got[sl].astype(np.float64) - g64[sl]).max(), np.abs(g64[sl]).max()
                assert err <= NET_BOUND * scale, f"blob {k} {what}: {err:.3e} > {NET_BOUND} * {scale:.3e}"
        assert stats == 1589
    finally:
        net.deallocate()


def test_resnet20_runs_are_bitwise_identical_and_accumulate(cos, tmp_path):
    net = _net(cos, _solver(tmp_path))
    try:
        x, y = _batch(4)
        inputs = [torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()]
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


def _train(net, check=None, steps=STEPS):
    losses = []
    for t, (x, y) in enumerate(_task_batches(steps=steps)):
        if check:
            check.before()
        assert net.train(0, [x.numpy(), y.numpy()]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


class _StatsUpdateCheck(_UpdateCheck):
    """_UpdateCheck for a net with BatchNorm: the forward pass writes the statistics (lr_mult 0, so the update leaves
    them as written), so the oracle starts from the step's statistics and the pre-step values of everything else."""

    def __init__(self, net, oracle):
        super().__init__(net, oracle)
        d = net.desc
        self.stats = np.repeat(np.array(d.lr_mult) == 0, d.counts)

    def after(self, t):
        self.w[self.stats] = to_host(self.net.data())[self.stats]
        super().after(t)


def test_resnet20_trains_through_train_alone(cos, oracle, tmp_path):
    net = _net(cos, _solver(tmp_path))
    try:
        assert net.param_count() == 274063
        losses = _train(net, _StatsUpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-50:].mean() < losses[:10].mean() - LOSS_DROP, (losses[:10].mean(), losses[-50:].mean())
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
        batches = [_batch(10 + r) for r in range(2)]

        def run(r):
            for _ in range(4):
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
    solver = _solver(tmp_path)
    assert_bits_equal(_two_rank_run(cos, solver), _two_rank_run(cos, solver), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshots_hold_scale_blobs_and_resume_bit_exact(cos, tmp_path, fmt):
    from caffeonspark_b200 import nets
    solver = _solver(tmp_path, f"snapshot_format: {fmt}\n")
    a = _net(cos, solver)
    try:
        _train(a, steps=3)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        off, scales = 0, 0
        for (name, p), c in zip(nets.resnet20_module().named_parameters(), a.desc.counts):
            if name.endswith(("2.weight", "2.bias")):  # each unit's Scale: Sequential(conv, BatchNorm, Scale)
                layer = "scale_" + _caffe_unit(name)
                assert_bits_equal(cos.read_caffemodel_blob(model, layer, int(name.endswith("bias"))), w_a[off:off + c],
                                  f"{layer} {name}")
                scales += 1
            off += c
        assert scales == 42
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, steps=2), _train(b, steps=2)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()


def _caffe_unit(param_name):
    """'blocks.3.branch2a.2.weight' -> 'res3a_branch2a', 'conv1.2.bias' -> 'conv1' (the fixture's layer names)."""
    parts = param_name.split(".")
    if parts[0] == "conv1":
        return "conv1"
    i = int(parts[1])
    return f"res{2 + i // 3}{'abc'[i % 3]}_{parts[2]}"
