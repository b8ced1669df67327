"""The built-in gradient producer on the GPU (DESIGN.md section 14): gradients against a float64 evaluation of the same
net, determinism and the accumulate contract, training through train() alone, two in-process ranks, the fillers and
the label check."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from gpu_util import assert_bits_equal, to_host

pytestmark = pytest.mark.gpu

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
BATCH = {"lenet": 64, "cifar10_quick": 100, "cifar10_full_bn": 100}


def _load(module, w):
    off = 0
    with torch.no_grad():
        for p in module.parameters():
            n = p.numel()
            p.copy_(torch.from_numpy(w[off:off + n]).view(p.shape).to(p.dtype))
            off += n
    assert off == w.size


def _grads(module):
    return np.concatenate([(p.grad if p.grad is not None else torch.zeros_like(p)).detach().double().cpu()
                           .numpy().ravel() for p in module.parameters()])


def _params(module):
    return np.concatenate([p.detach().double().cpu().numpy().ravel() for p in module.parameters()])


def _reference(name, w, x, y, dtype, device):
    """(loss, flat gradient, flat parameters after the forward) of nets.torch_module on the same flat weights."""
    from caffeonspark_b200 import nets
    m = nets.torch_module(name).to(device=device, dtype=dtype)
    _load(m, w)
    out = m(torch.from_numpy(x).to(device=device, dtype=dtype))
    loss = F.cross_entropy(out, torch.from_numpy(y).long().to(device))
    loss.backward()
    return float(loss.detach()), _grads(m), _params(m)


def _native_net(cos, name, tmp_path, fill=False):
    from caffeonspark_b200 import nets
    net = cos.CaffeNet(nets.write_prototxts(name, str(tmp_path)), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    return net


def _run_once(net, xd, yd, loss):
    assert net.forward_backward([xd, yd], loss.data_ptr()), net.last_error()
    assert net.synchronize(), net.last_error()
    return to_host(net.diff()), float(loss.item())


def _batch(name, seed):
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(seed)
    x = rng.rand(BATCH[name], *nets.NETS[name]["input"]).astype(np.float32)
    y = rng.randint(0, 10, BATCH[name]).astype(np.float32)
    return x, y


def _blob_bound(got, want, what):
    err, scale = np.abs(got.astype(np.float64) - want).max(), np.abs(want).max()
    assert err <= 1e-4 * scale, f"{what}: max error {err:.3e} > 1e-4 * {scale:.3e}"


@pytest.mark.parametrize("name", ["lenet", "cifar10_quick", "cifar10_full_bn"])
def test_gradients_match_float64(cos, name, tmp_path):
    from caffeonspark_b200 import nets
    counts, _, _, names = nets.layout(name)
    net = _native_net(cos, name, tmp_path)
    try:
        net.fill("data", 21, 0, 0.1)
        torch.cuda.synchronize()
        w = to_host(net.data())
        x, y = _batch(name, 3)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()  # the zeroing ran on torch's stream, the producer runs on the net's
        g, l32 = _run_once(net, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), loss)
        data_after = to_host(net.data())
        l64, g64, p64 = _reference(name, w, x, y, torch.float64, "cpu")
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            lt, gt, _ = _reference(name, w, x, y, torch.float32, "cuda")
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
        off = 0
        for c, nm in zip(counts, names):
            sl = slice(off, off + c)
            off += c
            if not np.abs(g64[sl]).max():  # BatchNorm statistics: no gradient, and the forward wrote them
                assert not g[sl].any(), nm
                _blob_bound(data_after[sl], p64[sl], f"{name} {nm} statistics")
                continue
            _blob_bound(g[sl], g64[sl], f"{name} {nm} native")
            _blob_bound(gt[sl], g64[sl], f"{name} {nm} PyTorch fp32")
    finally:
        net.deallocate()


@pytest.mark.parametrize("name", ["lenet", "cifar10_quick", "cifar10_full_bn"])
def test_runs_are_bitwise_identical_and_accumulate(cos, name, tmp_path):
    net = _native_net(cos, name, tmp_path)
    try:
        net.fill("data", 5, 0, 0.1)
        x, y = _batch(name, 4)
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        loss = torch.zeros(1, device="cuda")
        runs = []
        for _ in range(2):
            net.diff().zero_()
            torch.cuda.synchronize()
            runs.append(_run_once(net, xd, yd, loss))
        assert_bits_equal(runs[0][0], runs[1][0], f"{name}: diff of two runs")
        assert runs[0][1] == runs[1][1]
        g2, _ = _run_once(net, xd, yd, loss)  # no clearing: diff += g once more
        assert_bits_equal(g2, np.float32(2) * runs[0][0], f"{name}: two calls accumulate 2g")
        # the engine rejects inputs that do not match its plan, without launching anything
        assert not net.forward_backward([xd], loss.data_ptr())
        assert not net.forward_backward([xd[:1], yd], loss.data_ptr())
    finally:
        net.deallocate()


def _task(rng, templates, noise=0.25):
    """LeNet-shaped batch: class template + noise, with a fraction `noise` of labels replaced at random."""
    y = rng.randint(0, 10, 64)
    x = (0.6 * templates[y] + 0.4 * rng.rand(64, 1, 28, 28)).astype(np.float32)
    flip = rng.rand(64) < noise
    y = np.where(flip, rng.randint(0, 10, 64), y)
    return x, y.astype(np.float32)


def _train(net, steps, seed, check=None):
    rng = np.random.RandomState(seed)
    templates = np.random.RandomState(99).rand(10, 1, 28, 28)
    losses = []
    for t in range(steps):
        x, y = _task(rng, templates)
        if check:
            check.before()
        assert net.train(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


class _UpdateCheck:
    """zero_diff = 0: the gradient stays in diff_, and the oracle's update of it must equal the net's, bit for bit."""

    def __init__(self, net, oracle):
        self.net, self.oracle, self.desc = net, oracle, net.desc
        net.set_option("zero_diff", 0)

    def before(self):
        self.w, self.h = to_host(self.net.data()), to_host(self.net.history())
        self.rate = self.net.learning_rate()
        self.net.diff().zero_()
        torch.cuda.synchronize()

    def after(self, t):
        d = self.desc
        self.oracle.apply_update(0, d.param_count, self.w, to_host(self.net.diff()), self.h, d.counts, d.lr_mult,
                                 d.decay_mult, np.float32(self.rate), np.float32(d.momentum),
                                 np.float32(d.weight_decay))
        assert_bits_equal(to_host(self.net.data()), self.w, f"weights after step {t}")
        assert_bits_equal(to_host(self.net.history()), self.h, f"history after step {t}")


def test_train_lenet_through_train_alone(cos, oracle):
    from caffeonspark_b200 import harness
    solver = os.path.join(CONFIGS, "lenet_memory_solver.prototxt")
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    ref = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses()) and ref.connect(ref.localAddresses())
        assert not net.train(0, list(_task(np.random.RandomState(0), np.zeros((10, 1, 28, 28)))))
        assert "no gradient producer registered" in net.last_error()  # nothing attached: as before
        net.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        w0 = to_host(net.data())
        assert np.abs(w0).max() > 0
        native = _train(net, 300, 1, _UpdateCheck(net, oracle))
        harness.make_producer("lenet", ref, use_graph=False)
        ref.data().copy_(torch.from_numpy(w0).cuda())
        torch.cuda.synchronize()
        torch_losses = _train(ref, 300, 1)
        first, last, last_t = native[0], native[-50:].mean(), torch_losses[-50:].mean()
        assert last < 0.5 * first, (first, last)
        assert abs(last - last_t) <= 0.1 * max(last, last_t), (last, last_t)
    finally:
        net.deallocate()
        ref.deallocate()


def test_train_lenet_with_iter_size_two(cos, tmp_path):
    text = open(os.path.join(CONFIGS, "lenet_memory_solver.prototxt")).read()
    (tmp_path / "solver.prototxt").write_text(text.replace('net: "lenet_memory_train_test.prototxt"',
                                                           f'net: "{CONFIGS}/lenet_memory_train_test.prototxt"')
                                              + "\niter_size: 2\n")
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.desc.iter_size == 2
        assert net.connect(net.localAddresses())
        net.use_native_producer()
        losses = _train(net, 60, 2)
        assert np.isfinite(losses).all() and losses[-10:].mean() < 0.7 * losses[0], losses
    finally:
        net.deallocate()


def _two_rank_run(cos):
    import concurrent.futures as cf
    solver = os.path.join(CONFIGS, "cifar10_quick_solver.prototxt")
    netz = [cos.CaffeNet(solver, "", "", 1, 2, r, True, cos.CaffeNet.SOCKET, -1, 0) for r in range(2)]
    try:
        for n in netz:
            n.set_option("grid", 8)
            n.set_option("block", 128)
            n.set_option("barrier_timeout_ms", 20000)
            n.set_option("initial_gather", 0)
            n.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        assert_bits_equal(to_host(netz[0].data()), to_host(netz[1].data()), "ranks fill identically")
        table = [n.localAddresses() for n in netz]
        with cf.ThreadPoolExecutor(2) as ex:
            assert all(ex.map(lambda r: netz[r].connect([table[p][r] if p != r else "" for p in range(2)]), range(2)))
        rng = np.random.RandomState(1)
        batches = [(rng.rand(100, 3, 32, 32).astype(np.float32), rng.randint(0, 10, 100).astype(np.float32))
                   for _ in range(2)]

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


def test_two_ranks_in_process_with_the_native_engine(cos):
    assert_bits_equal(_two_rank_run(cos), _two_rank_run(cos), "two whole runs")


FILL_NET = """name: "fill"
layer { name: "data" type: "MemoryData" top: "data" top: "label" memory_data_param { batch_size: 4 channels: 3 height: 8 width: 8 } }
layer { name: "c1" type: "Convolution" bottom: "data" top: "c1" convolution_param { num_output: 16 kernel_size: 3
  weight_filler { type: "uniform" min: -0.3 max: 0.5 } bias_filler { type: "constant" value: 0.7 } } }
layer { name: "c2" type: "Convolution" bottom: "c1" top: "c2" convolution_param { num_output: 64 kernel_size: 3
  weight_filler { type: "gaussian" mean: 0.2 std: 0.05 } bias_filler { type: "xavier" } } }
layer { name: "ip1" type: "InnerProduct" bottom: "c2" top: "ip1" inner_product_param { num_output: 32
  weight_filler { type: "xavier" variance_norm: AVERAGE } } }
layer { name: "ip2" type: "InnerProduct" bottom: "ip1" top: "ip2" inner_product_param { num_output: 10
  weight_filler { type: "msra" variance_norm: FAN_OUT } bias_filler { type: "constant" } } }
layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip2" bottom: "label" top: "loss" }
"""


def _fill_solver(tmp_path, seed="random_seed: 77\n"):
    (tmp_path / "fill_net.prototxt").write_text(FILL_NET)
    (tmp_path / "fill_solver.prototxt").write_text(
        f'net: "fill_net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n{seed}snapshot_prefix: "{tmp_path}/fill"\n')
    return str(tmp_path / "fill_solver.prototxt")


def _blobs(net):
    from itertools import accumulate
    w = to_host(net.data())
    ends = list(accumulate(net.desc.counts))
    return [w[e - c:e] for e, c in zip(ends, net.desc.counts)]


def test_fillers(cos, oracle, tmp_path):
    solver = _fill_solver(tmp_path)
    nets_ = [cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0) for _ in range(2)]
    try:
        for n in nets_:
            n.use_native_producer(fill_weights=True)
        b = _blobs(nets_[0])
        assert_bits_equal(to_host(nets_[0].data()), to_host(nets_[1].data()), "two ranks fill identically")
        f32 = np.float32
        # c1 weight (blob 0): uniform [-0.3, 0.5) = min + (max - min) * (u + 1) / 2 in float32
        u = oracle.fill_numpy(b[0].size, 77, 0, 1.0)
        want = f32(-0.3) + (f32(0.5) - f32(-0.3)) * ((u + f32(1)) * f32(0.5))
        assert_bits_equal(b[0], want.astype(np.float32), "uniform filler")
        assert_bits_equal(b[1], np.full(16, 0.7, np.float32), "constant filler")
        # c2 bias (blob 3, shape [64]): xavier, fan_in = 64 / 64 = 1
        assert_bits_equal(b[3], oracle.fill_numpy(64, 77, 3, np.sqrt(f32(3) / f32(1))), "xavier filler (1-axis)")
        # ip1 weight (blob 4, [32, 1024]): xavier AVERAGE, n = (1024 + 32) / 2
        assert_bits_equal(b[4], oracle.fill_numpy(b[4].size, 77, 4, np.sqrt(f32(3) / f32(528))), "xavier AVERAGE")
        assert not b[5].any()  # ip1 bias: no bias_filler = constant 0
        # c2 weight (blob 2): gaussian mean 0.2 std 0.05 over 9216 samples
        g = b[2].astype(np.float64)
        assert abs(g.mean() - 0.2) < 5 * 0.05 / np.sqrt(g.size) and abs(g.std() / 0.05 - 1) < 0.05
        # ip2 weight (blob 6, [10, 1024]): msra FAN_OUT, fan_out = 10240 / 1024 = 10
        m, sd = b[6].astype(np.float64), np.sqrt(2 / 10)
        assert abs(m.mean()) < 5 * sd / np.sqrt(m.size) and abs(m.std() / sd - 1) < 0.05
    finally:
        for n in nets_:
            n.deallocate()


def test_fill_weights_off_and_restored_models_leave_data_alone(cos, tmp_path):
    solver = _fill_solver(tmp_path, seed="")  # no random_seed: seed 0
    a = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        a.fill("data", 3, 0, 0.5)
        torch.cuda.synchronize()
        before = to_host(a.data())
        a.use_native_producer(fill_weights=False)
        assert_bits_equal(to_host(a.data()), before, "fill_weights=0")
        a.use_native_producer(fill_weights=True)  # seed 0, replaces the engine
        filled = to_host(a.data())
        assert not np.array_equal(filled, before)
        assert a.snapshot() == 0
        model = a.snapshotFilename(0, False)
    finally:
        a.deallocate()
    b = cos.CaffeNet(solver, model, "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        b.use_native_producer(fill_weights=True)
        assert_bits_equal(to_host(b.data()), filled, "a restored model is not refilled")
    finally:
        b.deallocate()


def test_descriptor_nets_need_a_prototxt_and_layouts_must_match(cos, tmp_path):
    from caffeonspark_b200 import nets
    net = cos.CaffeNet(nets.solver_desc("lenet"))
    try:
        with pytest.raises(cos.CosError, match="layout descriptor"):
            net.use_native_producer()
        with pytest.raises(cos.CosError, match="not the layout of this net"):
            net.use_native_producer(nets.write_prototxts("cifar10_quick", str(tmp_path)))
        net.use_native_producer(os.path.join(CONFIGS, "lenet_memory_train_test.prototxt"), fill_weights=True)
        loss = torch.zeros(1, device="cuda")
        assert not net.forward_backward([], loss.data_ptr())
    finally:
        net.deallocate()


def test_a_label_out_of_range_fails_the_next_synchronize(cos, tmp_path):
    net = _native_net(cos, "lenet", tmp_path, fill=True)
    try:
        x, y = _batch("lenet", 7)
        for bad in (10.0, -1.0, float("nan")):
            yb = y.copy()
            yb[5] = bad
            assert net.train(0, [x, yb]), net.last_error()
            assert not net.synchronize()
            assert "label outside" in net.last_error()
            assert np.isfinite(to_host(net.data())).all()
        assert net.train(0, [x, y]), net.last_error()  # the word was cleared when it was reported
        assert net.synchronize(), net.last_error()
    finally:
        net.deallocate()


def _solver_for(tmp_path, net_text, name):
    (tmp_path / f"{name}_net.prototxt").write_text(net_text)
    (tmp_path / f"{name}_solver.prototxt").write_text(f'net: "{name}_net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / f"{name}_solver.prototxt")


def test_nets_that_touch_staged_inputs_run_without_writing_them(cos, tmp_path):
    # an in-place ReLU on the data blob: its top gets storage of its own, the staged input is left as it was
    relu = _solver_for(tmp_path, 'layer { name: "data" type: "MemoryData" top: "data" top: "label" memory_data_param '
                       '{ batch_size: 2 channels: 3 height: 8 width: 8 } }\n'
                       'layer { name: "r" type: "ReLU" bottom: "data" top: "data" }\n'
                       'layer { name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param '
                       '{ num_output: 4 } }\n'
                       'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n',
                       "relu")
    # scores straight from a data layer: the loss's bottom gradient goes to a buffer of the engine's own
    scores = _solver_for(tmp_path, 'layer { name: "data" type: "Input" top: "scores" top: "label" input_param { '
                         'shape { dim: 4 dim: 5 } shape { dim: 4 } } }\n'
                         'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "scores" bottom: "label" top: "loss" }\n',
                         "scores")
    rng = np.random.RandomState(8)
    for solver, xs, classes in ((relu, (2, 3, 8, 8), 4), (scores, (4, 5), 5)):
        net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            net.use_native_producer(fill_weights=False)
            net.fill("data", 9, 0, 0.3)
            x = (rng.rand(*xs) - 0.5).astype(np.float32)
            y = rng.randint(0, classes, xs[0]).astype(np.float32)
            xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
            loss = torch.zeros(1, device="cuda")
            net.diff().zero_()
            torch.cuda.synchronize()
            g, l32 = _run_once(net, xd, yd, loss)
            assert_bits_equal(xd.cpu().numpy(), x, "the staged input is not written")
            xt = torch.from_numpy(x).double()
            if solver == relu:
                w = to_host(net.data()).astype(np.float64)
                W = torch.tensor(w[:4 * 192].reshape(4, 192), requires_grad=True)
                b = torch.tensor(w[4 * 192:], requires_grad=True)
                ref = F.cross_entropy(F.relu(xt).reshape(2, -1) @ W.t() + b, torch.from_numpy(y).long())
                ref.backward()
                _blob_bound(g[:4 * 192], W.grad.numpy().ravel(), "relu net ip weight")
                _blob_bound(g[4 * 192:], b.grad.numpy(), "relu net ip bias")
            else:
                ref = F.cross_entropy(xt, torch.from_numpy(y).long())
            ref = float(ref.detach())
            assert abs(l32 - ref) <= 1e-5 * abs(ref), (l32, ref)
            assert net.train(0, [x, y]), net.last_error()
            assert net.synchronize(), net.last_error()
        finally:
            net.deallocate()


def test_registering_another_producer_releases_the_engine(cos, tmp_path):
    net = _native_net(cos, "cifar10_quick", tmp_path, fill=True)
    try:
        torch.cuda.synchronize()
        free_attached = torch.cuda.mem_get_info()[0]
        calls = []
        assert net.set_forward_backward(lambda *a: calls.append(1))
        free_released = torch.cuda.mem_get_info()[0]
        assert free_released - free_attached > 20 << 20, (free_attached, free_released)  # activations, workspace
        x, y = _batch("cifar10_quick", 1)
        assert net.train(0, [x, y]) and net.synchronize(), net.last_error()
        assert calls == [1]
        net.use_native_producer(fill_weights=False)  # and back: the engine serves train() again
        assert net.train(0, [x, y]) and net.synchronize(), net.last_error()
        assert calls == [1] and np.isfinite(net.last_loss())
    finally:
        net.deallocate()


def test_weight_gradient_over_more_products_than_a_grid_has_chunks(cos, tmp_path):
    """A 1x1 conv over 6400 x 6400 pixels: its weight gradient sums 40,960,000 products, 80,000 chunks of 512 (more
    than the 65,535 a grid's z dimension holds), so the engine widens the chunks to keep at most 256 partials."""
    solver = _solver_for(tmp_path, 'layer { name: "data" type: "MemoryData" top: "data" top: "label" '
                         'memory_data_param { batch_size: 1 channels: 1 height: 6400 width: 6400 } }\n'
                         'layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param '
                         '{ num_output: 1 kernel_size: 1 } }\n'
                         'layer { name: "p" type: "Pooling" bottom: "c" top: "p" pooling_param '
                         '{ pool: MAX kernel_size: 64 stride: 64 } }\n'
                         'layer { name: "ip" type: "InnerProduct" bottom: "p" top: "ip" inner_product_param '
                         '{ num_output: 10 } }\n'
                         'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n',
                         "wide")
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        net.use_native_producer(fill_weights=False)
        net.fill("data", 4, 0, 0.5)
        rng = np.random.RandomState(2)
        x = rng.rand(1, 1, 6400, 6400).astype(np.float32)
        y = np.array([3], np.float32)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run_once(net, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), loss)
        w = torch.from_numpy(to_host(net.data()).astype(np.float64)).cuda()
        cw, cb = w[0:1].clone().requires_grad_(), w[1:2].clone().requires_grad_()
        iw, ib = w[2:100002].clone().requires_grad_(), w[100002:].clone().requires_grad_()
        z = F.conv2d(torch.from_numpy(x).cuda().double(), cw.view(1, 1, 1, 1), cb)
        out = F.max_pool2d(z, 64, 64, ceil_mode=True).reshape(1, -1) @ iw.view(10, -1).t() + ib
        ref = F.cross_entropy(out, torch.tensor([3], device="cuda"))
        ref.backward()
        assert abs(l32 - float(ref)) <= 1e-5 * abs(float(ref))
        for got, want, what in ((g[0:1], cw.grad, "conv weight"), (g[1:2], cb.grad, "conv bias"),
                                (g[2:100002], iw.grad, "ip weight"), (g[100002:], ib.grad, "ip bias")):
            _blob_bound(got, want.cpu().numpy().ravel(), what)
    finally:
        net.deallocate()
