"""Caffe's least-squares solver-test net on the GPU (DESIGN.md section 14): InnerProduct -> EuclideanLoss on the rows
of solver_data.h5, and its shared-weights variant with Slice and Concat, on the built-in engine.  Gradients against
float64, training through train() alone with every update checked against the oracle and the weights against the
closed form of test_gradient_based_solver.cpp (SGD and Adam), iter_size 2, 2 and 3 in-process ranks, snapshots that
resume bit-exact, and EuclideanLoss and Concat in other nets against float64."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch

from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _blob_bound
from test_hdf5_io import FIX, _read
from test_least_squares_host import D, N, write_solver

pytestmark = pytest.mark.gpu

# test_gradient_based_solver.cpp: (base_lr, weight_decay, momentum, steps K + 1 checked after every step)
SGD_CASES = {"lr1": (1.0, 0.0, 0.0, 1), "lr0.01": (0.01, 0.0, 0.0, 1), "weight_decay": (0.01, 0.5, 0.0, 5),
             "momentum": (0.01, 0.0, 0.5, 5), "everything": (0.01, 0.5, 0.5, 5)}
ADAM_CASES = {"adam": (0.01, 0.0, 0.9, 1), "adam_weight_decay": (0.01, 0.5, 0.9, 1),
              "adam_everything": (0.01, 0.5, 0.9, 5)}
CASES = {**SGD_CASES, **ADAM_CASES, "everything_accum": (0.01, 0.5, 0.9, 5)}  # the accumulation and snapshot tests'


@pytest.fixture(scope="module")
def solver_data(cos):
    """The 8 rows of solver_data.h5 (data 8x3x10x10, targets 8x1), read with the library's HDF5 reader."""
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    x, xs = _read(L, os.path.join(FIX, "solver_data.h5"), "/data")
    y, ys = _read(L, os.path.join(FIX, "solver_data.h5"), "targets")
    assert xs == [N, 3, 10, 10] and ys == [N, 1]
    return x.reshape(N, 3, 10, 10), y.reshape(N, 1)


@pytest.fixture(scope="module")
def adam(oracle):
    from oracle import adam as A
    A.build()
    A.lib()
    return A


@pytest.fixture(scope="module")
def accum(oracle):
    from oracle import accum as A
    A.build()
    A.lib()
    return A


def _solver(tmp_path, name, case, share=False, **kw):
    lr, wd, mom, _ = CASES[case]
    d = tmp_path / name
    d.mkdir()
    return write_solver(d, share, lr, wd, mom, "Adam" if case.startswith("adam") else None, **kw)


def _native(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


def _near(got, want, what):
    """CheckLeastSquaresUpdate's tolerance: max(1e-7, 1e-2 * min(|want|, |got|)) per element."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    tol = np.maximum(1e-7, 1e-2 * np.minimum(np.abs(got), np.abs(want)))
    bad = np.nonzero(np.abs(got - want) > tol)[0]
    assert bad.size == 0, f"{what}: {bad.size} elements off; first at {bad[0]}: {got[bad[0]]!r} vs {want[bad[0]]!r}"


def _closed_form(theta, hist, x, y, desc, t):
    """ComputeLeastSquaresUpdate in float64: the regularised least-squares gradient, then the SGD or Adam update of
    step t (1-based).  Returns (theta', history')."""
    Xa = np.hstack([x.reshape(len(x), -1).astype(np.float64), np.ones((len(x), 1))])
    grad = Xa.T @ (Xa @ theta - y.ravel().astype(np.float64)) / len(x) + desc.weight_decay * theta
    if desc.type == "Adam":
        b1, b2 = desc.momentum, desc.momentum2
        m = (1 - b1) * grad + b1 * hist[0]
        v = (1 - b2) * grad * grad + b2 * hist[1]
        alpha = desc.base_lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        return theta - alpha * m / (np.sqrt(v) + desc.delta), (m, v)
    upd = desc.base_lr * grad + desc.momentum * hist
    return theta - upd, upd


def _zero_history(desc):
    z = np.zeros(D + 1)
    return (z, z) if desc.type == "Adam" else z


class _StepCheck:
    """zero_diff = 0 keeps each step's device gradient in diff_: the oracle's update of it (SGD or Adam, iter_size
    passes accumulated) must equal the net's, bit for bit."""

    def __init__(self, net, oracle, adam, accum=None):
        self.net, self.oracle, self.adam, self.accum, self.desc = net, oracle, adam, accum, net.desc
        net.set_option("zero_diff", 0)

    def before(self):
        self.w, self.h = to_host(self.net.data()), to_host(self.net.history())
        self.rate, self.it = self.net.learning_rate(), self.net.iter()
        self.net.diff().zero_()
        torch.cuda.synchronize()

    def after(self, t):
        d, g = self.desc, to_host(self.net.diff())
        assert np.abs(g).max() > 0
        rate = float(np.float32(self.rate))
        if self.accum is not None:
            self.accum.step_accum([self.w], [g], [self.h], d.counts, d.lr_mult, d.decay_mult, rate, d.momentum,
                                  d.weight_decay, d.iter_size, self.it, solver_type=d.type, momentum2=d.momentum2,
                                  delta=d.delta)
        elif d.type == "Adam":
            self.adam.step_adam([self.w], [g], [self.h], d.counts, d.lr_mult, d.decay_mult, rate, d.momentum,
                                d.momentum2, d.delta, d.weight_decay, self.it)
        else:
            self.oracle.apply_update(0, d.param_count, self.w, g, self.h, d.counts, d.lr_mult, d.decay_mult,
                                     np.float32(rate), np.float32(d.momentum), np.float32(d.weight_decay))
        assert_bits_equal(to_host(self.net.data()), self.w, f"weights after step {t}")
        assert_bits_equal(to_host(self.net.history()), self.h, f"history after step {t}")


def _train_checked(net, check, solver_data, steps, passes=None):
    """steps train() (or train_accumulate() over `passes`) calls, each update checked against the oracle, and the
    weights after K + 1 = 1 .. steps steps against the float64 closed form started from the engine's filled weights."""
    x, y = solver_data
    desc = net.desc
    theta, hist = to_host(net.data()).astype(np.float64), _zero_history(desc)
    for t in range(steps):
        check.before()
        if passes:
            assert net.train_accumulate(0, passes), net.last_error()
        else:
            assert net.train(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()
        check.after(t)
        theta, hist = _closed_form(theta, hist, x, y, desc, t + 1)
        _near(to_host(net.data()), theta, f"weights after {t + 1} step(s)")
    return to_host(net.data())


def _float64_grads(w, x, y):
    """(loss, gradient of the weights, gradient of the bias) of |X w + b - y|^2 / 2n."""
    X = x.reshape(len(x), -1).astype(np.float64)
    r = X @ w[:D].astype(np.float64) + np.float64(w[D]) - y.ravel().astype(np.float64)
    return (r @ r) / len(x) / 2, X.T @ r / len(x), r.sum() / len(x)


@pytest.mark.parametrize("share", [False, True])
def test_gradients_match_float64(cos, tmp_path, solver_data, share):
    net = _native(cos, _solver(tmp_path, "s", "lr1", share))
    try:
        x, y = solver_data
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        loss = torch.zeros(1, device="cuda")
        w = to_host(net.data())
        assert w.size == D + 1 and np.abs(w).max() > 0  # gaussian std 1 from the net's fillers

        def run():
            assert net.forward_backward([xd, yd], loss.data_ptr()), net.last_error()
            assert net.synchronize(), net.last_error()
            return to_host(net.diff()), float(loss.item())

        runs = []
        for _ in range(2):
            net.diff().zero_()
            torch.cuda.synchronize()
            runs.append(run())
        (g, l32), (g2, l2) = runs
        l64, gw, gb = _float64_grads(w, x, y)
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        _blob_bound(g[:D], gw, "weights")
        _blob_bound(g[D:], np.array([gb]), "bias")
        assert_bits_equal(g, g2, "diff of two calls")
        assert l32 == l2
        if not share:  # one use per blob: the second call adds g once more, exactly
            assert_bits_equal(run()[0], np.float32(2) * g, "two calls without clearing")
    finally:
        net.deallocate()


def test_a_nan_target_reaches_the_loss_without_a_status(cos, tmp_path, solver_data):
    net = _native(cos, _solver(tmp_path, "s", "lr1"))
    try:
        x, y = solver_data
        y = y.copy()
        y[3] = np.nan
        loss = torch.zeros(1, device="cuda")
        net.diff().zero_()
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()], loss.data_ptr())
        assert net.synchronize(), net.last_error()  # as in Caffe: no error, the loss is NaN
        assert np.isnan(loss.item()) and np.isnan(to_host(net.diff())).any()
    finally:
        net.deallocate()


@pytest.mark.parametrize("case", sorted(SGD_CASES) + sorted(ADAM_CASES))
def test_train_alone_matches_oracle_and_closed_form(cos, oracle, adam, tmp_path, solver_data, case):
    """Each case of the reference's SGD and Adam least-squares tests on the plain net and on the share variant: every
    update equals the oracle's given the device gradient, the weights stay within CheckLeastSquaresUpdate's tolerance of
    the closed form, and the two nets agree to that tolerance."""
    steps = CASES[case][3]
    finals = []
    for share in (False, True):
        net = _native(cos, _solver(tmp_path, f"s{int(share)}", case, share))
        try:
            assert net.param_count() == D + 1 and net.desc.counts == [D, 1]
            finals.append((to_host(net.data()), _train_checked(net, _StepCheck(net, oracle, adam), solver_data, steps)))
        finally:
            net.deallocate()
    assert_bits_equal(finals[0][0], finals[1][0], "both nets fill the owners' blobs alike")
    _near(finals[1][1], finals[0][1], "share variant against the plain net")


@pytest.mark.parametrize("share", [False, True])
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_iter_size_two_matches_one_pass_over_all_rows(cos, oracle, adam, accum, tmp_path, solver_data, share, solver):
    """CheckAccumulation: train_accumulate on rows 0-3 and 4-7 with iter_size 2 against iter_size 1 on all 8 rows
    (the reference's accumulation cases: momentum 0.9 for SGD)."""
    x, y = solver_data
    case = "everything_accum" if solver == "SGD" else "adam_everything"
    one = _native(cos, _solver(tmp_path, "one", case, share))
    two = _native(cos, _solver(tmp_path, "two", case, share, iter_size=2))
    try:
        assert two.desc.iter_size == 2
        w_one = _train_checked(one, _StepCheck(one, oracle, adam), solver_data, 4)
        passes = [[x[:N // 2], y[:N // 2]], [x[N // 2:], y[N // 2:]]]
        w_two = _train_checked(two, _StepCheck(two, oracle, adam, accum), solver_data, 4, passes)
        _near(w_two, w_one, "iter_size 2 against iter_size 1")
    finally:
        one.deallocate()
        two.deallocate()


@pytest.mark.parametrize("ranks", [2, 3])
@pytest.mark.parametrize("case", ["everything", "adam_everything"])
def test_in_process_ranks_match_oracle_and_one_rank(cos, oracle, adam, tmp_path, solver_data, ranks, case):
    """Every rank is fed the 8 rows: the ranks hold bitwise-identical weights, each step equals the oracle's N-rank
    step given the ranks' device gradients, and the run matches the single-rank run to the closed form's tolerance."""
    from oracle.adam import AdamSimulation
    steps = 4
    single = _native(cos, _solver(tmp_path, "one", case))
    try:
        w_single = _train_checked(single, _StepCheck(single, oracle, adam), solver_data, steps)
    finally:
        single.deallocate()
    solver = _solver(tmp_path, "multi", case)
    netz = [cos.CaffeNet(solver, "", "", 1, ranks, r, True, cos.CaffeNet.SOCKET, -1, 0) for r in range(ranks)]
    try:
        for n in netz:
            n.set_option("grid", 4)
            n.set_option("block", 128)
            n.set_option("barrier_timeout_ms", 20000)
            n.set_option("initial_gather", 0)
            n.set_option("zero_diff", 0)  # keep each rank's gradient for the oracle
            n.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        table = [n.localAddresses() for n in netz]
        with cf.ThreadPoolExecutor(ranks) as ex:
            assert all(ex.map(lambda r: netz[r].connect([table[p][r] if p != r else "" for p in range(ranks)]),
                              range(ranks)))
        desc = netz[0].desc
        w0 = to_host(netz[0].data())
        for n in netz[1:]:
            assert_bits_equal(to_host(n.data()), w0, "ranks fill identically")
        kw = dict(lr_policy="fixed", base_lr=desc.base_lr, momentum=desc.momentum, weight_decay=desc.weight_decay)
        sim = (AdamSimulation(ranks, desc.counts, desc.lr_mult, desc.decay_mult, momentum2=desc.momentum2,
                              delta=desc.delta, **kw) if desc.type == "Adam"
               else oracle.Simulation(ranks, desc.counts, desc.lr_mult, desc.decay_mult, **kw))
        sim.data = [w0.copy() for _ in range(ranks)]
        x, y = solver_data

        def run(r):
            assert netz[r].train(0, [x, y]), netz[r].last_error()
            assert netz[r].synchronize(), netz[r].last_error()

        P = desc.param_count
        for t in range(steps):
            for n in netz:
                n.diff().zero_()
            torch.cuda.synchronize()
            with cf.ThreadPoolExecutor(ranks) as ex:
                list(ex.map(run, range(ranks)))
            grads = [to_host(n.diff()) for n in netz]
            for g in grads[1:]:
                assert_bits_equal(g, grads[0], f"step {t}: every rank computes the same gradient")
            sim.step(grads)
            mode = netz[0].get_option("resolved_algo")
            for r, n in enumerate(netz):
                assert_bits_equal(to_host(n.data()), sim.consistent_weights(), f"step {t} rank {r} weights")
                o, s = (0, P) if mode == 2 else cos.chunk(P, ranks, r)  # one-shot: every rank holds all history
                assert_bits_equal(to_host(n.history())[o:o + s], sim.consistent_history()[o:o + s],
                                  f"step {t} rank {r} history")
        _near(to_host(netz[0].data()), w_single, f"{ranks} ranks against one")
    finally:
        with cf.ThreadPoolExecutor(ranks) as ex:
            list(ex.map(lambda n: n.deallocate(), netz))


@pytest.mark.parametrize("share", [False, True])
@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshot_resumes_bit_exact(cos, tmp_path, solver_data, share, fmt):
    """TestSnapshot: 2k steps against k steps, a snapshot, a restore and k more; weights and history bitwise equal."""
    x, y = solver_data
    k = 4
    solver = _solver(tmp_path, "s", "everything_accum", share, extra=f"snapshot_format: {fmt}\n")

    def steps(net, n):
        for _ in range(n):
            assert net.train(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()

    full = _native(cos, solver)
    try:
        steps(full, 2 * k)
        w_full, h_full = to_host(full.data()), to_host(full.history())
    finally:
        full.deallocate()
    a = _native(cos, solver)
    try:
        steps(a, k)
        assert a.snapshot() == k, a.last_error()
        model, state = a.snapshotFilename(k, False), a.snapshotFilename(k, True)
        assert model.endswith(".h5") == (fmt == "HDF5")
    finally:
        a.deallocate()
    b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert b.connect(b.localAddresses())
        b.use_native_producer(fill_weights=True)  # a restored model is not refilled
        assert b.iter() == k
        steps(b, k)
        assert_bits_equal(to_host(b.data()), w_full, "weights after restore and k more steps")
        assert_bits_equal(to_host(b.history()), h_full, "history after restore and k more steps")
    finally:
        b.deallocate()


def _ip_params(rng, shapes):
    """Flat weights for InnerProducts of (outputs, inputs) shapes: W then b of each, in net order."""
    ws = [(0.5 * rng.randn(o, i)).astype(np.float32) for o, i in shapes]
    bs = [(0.1 * rng.randn(o)).astype(np.float32) for o, _ in shapes]
    return ws, bs, np.concatenate([a for w, b in zip(ws, bs) for a in (w.ravel(), b)])


def _run_general(cos, tmp_path, text, w, inputs):
    (tmp_path / "net.prototxt").write_text(text)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = _native(cos, str(tmp_path / "solver.prototxt"), fill=False)
    try:
        net.data().copy_(torch.from_numpy(w).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(a).cuda() for a in inputs], loss.data_ptr()), net.last_error()
        assert net.synchronize(), net.last_error()
        return to_host(net.diff()), float(loss.item())
    finally:
        net.deallocate()


def _check_general(g, l32, loss64, params):
    loss64.backward()
    l64 = float(loss64.detach())
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    off = 0
    for i, p in enumerate(params):
        n = p.numel()
        _blob_bound(g[off:off + n], p.grad.numpy().ravel(), f"param {i}")
        assert np.abs(p.grad.numpy()).max() > 0
        off += n
    assert off == g.size


def test_euclidean_loss_sends_minus_g_into_a_learnable_second_bottom(cos, tmp_path):
    rng = np.random.RandomState(5)
    n, lw = 37, 0.75
    x, z = rng.randn(n, 6).astype(np.float32), rng.randn(n, 4).astype(np.float32)
    ws, bs, w = _ip_params(rng, [(3, 6), (3, 4)])
    text = ("name: 't' layer { name: 'in' type: 'Input' top: 'x' top: 'z' input_param { "
            f"shape {{ dim: {n} dim: 6 }} shape {{ dim: {n} dim: 4 }} }} }}\n"
            "layer { name: 'ip' type: 'InnerProduct' bottom: 'x' top: 'a' inner_product_param { num_output: 3 } }\n"
            "layer { name: 'ip2' type: 'InnerProduct' bottom: 'z' top: 'b' inner_product_param { num_output: 3 } }\n"
            f"layer {{ name: 'loss' type: 'EuclideanLoss' bottom: 'a' bottom: 'b' top: 'loss' loss_weight: {lw} }}\n")
    g, l32 = _run_general(cos, tmp_path, text, w, [x, z])
    params = [torch.from_numpy(a).double().requires_grad_() for pair in zip(ws, bs) for a in pair]
    a = torch.from_numpy(x).double() @ params[0].T + params[1]
    b = torch.from_numpy(z).double() @ params[2].T + params[3]
    _check_general(g, l32, lw * ((a - b) ** 2).sum() / n / 2, params)


@pytest.mark.parametrize("axis,nbottoms", [(0, 2), (0, 3), (1, 2), (1, 3)])
def test_concat_of_learnable_and_staged_bottoms(cos, tmp_path, axis, nbottoms):
    """Bottoms: InnerProduct outputs and, second, a staged input; their concat along `axis` goes into a EuclideanLoss
    against a staged target."""
    rng = np.random.RandomState(10 * axis + nbottoms)
    # (rows, columns) of each bottom: the concat axis varies, the other matches
    sizes = [3, 2, 4][:nbottoms]
    shapes = [(s, 5) if axis == 0 else (6, s) for s in sizes]
    learn = [i for i in range(nbottoms) if i != 1]
    ws, bs, w = _ip_params(rng, [(shapes[i][1], 4) for i in learn])
    inputs, tops, dims, layers, bottoms = [], [], [], [], []
    for i, s in enumerate(shapes):
        if i == 1:
            inputs.append(rng.randn(*s).astype(np.float32))
            tops.append("s")
            dims.append(s)
            bottoms.append("s")
        else:
            inputs.append(rng.randn(s[0], 4).astype(np.float32))
            tops.append(f"x{i}")
            dims.append((s[0], 4))
            layers.append(f"layer {{ name: 'ip{i}' type: 'InnerProduct' bottom: 'x{i}' top: 'y{i}' "
                          f"inner_product_param {{ num_output: {s[1]} }} }}")
            bottoms.append(f"y{i}")
    cat = (sum(sizes), 5) if axis == 0 else (6, sum(sizes))
    target = rng.randn(*cat).astype(np.float32)
    text = ("name: 't' layer { name: 'in' type: 'Input' " + " ".join(f"top: '{t}'" for t in tops) + " top: 't' "
            "input_param { " + " ".join(f"shape {{ dim: {a} dim: {b} }}" for a, b in dims + [cat]) + " } }\n"
            + "\n".join(layers) + "\nlayer { name: 'cat' type: 'Concat' " + " ".join(f"bottom: '{b}'" for b in bottoms)
            + f" top: 'cat' concat_param {{ axis: {axis} }} }}\n"
            "layer { name: 'loss' type: 'EuclideanLoss' bottom: 'cat' bottom: 't' }\n")
    g, l32 = _run_general(cos, tmp_path, text, w, inputs + [target])
    params = [torch.from_numpy(a).double().requires_grad_() for pair in zip(ws, bs) for a in pair]
    parts, j = [], 0
    for i in range(nbottoms):
        if i == 1:
            parts.append(torch.from_numpy(inputs[1]).double())
        else:
            parts.append(torch.from_numpy(inputs[i]).double() @ params[2 * j].T + params[2 * j + 1])
            j += 1
    d = torch.cat(parts, axis) - torch.from_numpy(target).double()
    _check_general(g, l32, (d ** 2).sum() / cat[0] / 2, params)
