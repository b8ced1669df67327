"""The RNN layer on the built-in engine (DESIGN.md section 14) on the GPU.

The op runs through test_gpu_producer_ops.py's injector harness: x and x_static come from injectors (so their
gradients come back exactly) or straight from staged inputs (no gradient wanted), cont is always staged, and the top
meets the EuclideanLoss probe, which hands the op a known top gradient d and returns it exactly.  The forward top, dx,
dx_static and all six blob gradients are compared with rnn_ref.py in float64, per blob relative to max|g64|.  A second
call without clearing must add the very same gradient again, and two runs must agree bit for bit.  The hidden state
carried between calls must match the reference over consecutive calls with the gradient cut at the boundary, and
cont = 0 at t = 0 must make a call independent of the one before.

Both recurrent fixtures are checked against float64 and PyTorch fp32 (on the CPU) over two consecutive calls (streams continuing
across the boundary), at their own batch and an odd one, trained through train() with every update equal to the
oracle's on one rank and two, with iter_size 2 carrying the state from pass to pass, and rnn_lm's snapshots resume
bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import rnn_ref as R
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import _net

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
LM, CAPTION = "rnn_lm", "rnn_caption"
# The per-blob bound relative to the blob's largest float64 gradient (and the top's largest value), fixed on the CPU
# from these very cases: PyTorch fp32 (the rnn_module mirror) reached at worst 3.9e-6 over the op geometries below (H = 1,
# where a gradient is one long sum) and 1.2e-6 over the fixtures' two calls at both batches, the loss 7.7e-8 relative.
OP_BOUND = 2e-5
NET_BOUND = 2e-5


# --------------------------------------------------------------------------- the op
def _rnn_layer(bottoms, H):
    b = " ".join(f'bottom: "{x}"' for x in bottoms)
    return f'layer {{ name: "r" type: "RNN" {b} top: "y" recurrent_param {{ num_output: {H} }} }}\n'


def _cont(rng, kind, T, N):
    if kind == "ones":
        return np.ones((T, N), F32)
    if kind == "start":
        c = np.ones((T, N), F32)
        c[0] = 0
        return c
    if kind == "random":
        return (rng.rand(T, N) < 0.6).astype(F32)
    return rng.choice(np.array([0.5, 2.0, 1.0, 0.0], F32), (T, N))  # "scaled": non-binary


class _Op:
    """One net: Input -> injectors / staged inputs -> RNN -> probe + EuclideanLoss, kept open for several calls."""

    def __init__(self, cos, tmp_path, T, N, I, H, S, grad_x, grad_s, rng):
        self.T, self.N, self.I, self.H, self.S = T, N, I, H, S
        self.x = rng.randn(T, N, I).astype(F32)
        self.xs = rng.randn(N, S).astype(F32) if S else None
        self.W = {k: (rng.randn(*s) * 0.5 / np.sqrt(max(s[-1], 1))).astype(F32) for k, s in R.blob_shapes(I, H, S)}
        injected, staged, bottoms = [], {}, []
        for name, v, grad in (("x", self.x, grad_x), ("s", self.xs, grad_s)):
            if v is None:
                continue
            if grad:
                bottoms.append(f"x{len(injected)}")
                injected.append(v)
            else:
                bottoms.append(name)
                staged[name] = v
        bottoms.insert(1, "cont")
        self.injected, self.grad_x, self.grad_s = injected, grad_x, grad_s
        self.staged_names = list(staged)
        weights = [self.W[k] for k, _ in R.blob_shapes(I, H, S)]
        self.out_shape = (T, N, H)
        o64, _ = R.forward(self.W, self.x, np.ones((T, N)), np.zeros((N, H)), self.xs)
        self.B = (o64 - rng.randn(T, N, H) * 0.5).astype(F32)
        text, self.ws = _net(injected, _rnn_layer(bottoms, H), weights, self.out_shape, self.B,
                             dict(staged, cont=np.zeros((T, N), F32)))
        self.nw = sum(w.size for w in weights)
        self.staged = staged
        (tmp_path / "net.prototxt").write_text(text)
        (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
        self.net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        assert self.net.connect(self.net.localAddresses())
        self.net.use_native_producer(fill_weights=False)
        self.net.data().copy_(torch.from_numpy(np.concatenate([w.ravel() for w in self.ws])).cuda())

    def call(self, cont, clear=True):
        """-> (RNN blob gradients, dx or None, dx_static or None, d = the top gradient the op received)"""
        net = self.net
        if clear:
            net.diff().zero_()
        ins = [np.zeros(np.shape(v), F32) for v in self.injected] + [np.zeros(self.out_shape, F32)]
        ins += [self.staged[k] for k in self.staged_names] + [cont]
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in ins],
                                    loss.data_ptr()), net.last_error()
        assert net.synchronize(), net.last_error()
        g = to_host(net.diff())
        parts, off = [], 0
        for w in self.ws:
            parts.append(g[off:off + w.size].reshape(w.shape))
            off += w.size
        k = 2 * len(self.injected)
        blobs = dict(zip([n for n, _ in R.blob_shapes(self.I, self.H, self.S)], parts[k:k + 6]))
        dxs = [parts[2 * i + 1] for i in range(len(self.injected))]
        dx = dxs.pop(0) if self.grad_x else None
        dxst = dxs.pop(0) if self.grad_s else None
        return blobs, dx, dxst, -parts[-1]

    def close(self):
        self.net.deallocate()


def _rel(got, want, what, bound):
    want = np.asarray(want, np.float64)
    scale = np.abs(want).max()
    err = np.abs(np.asarray(got, np.float64) - want).max() / (scale if scale > 0 else 1.0)
    assert err <= bound, f"{what}: {err:.3e} of max|ref| = {scale:.3e}, bound {bound}"


def _compare(op, got, cont, h0, what):
    """The engine's call against the float64 reference fed the top gradient the op really received."""
    blobs, dx, dxs, d = got
    o64, _ = R.forward(op.W, op.x, cont, h0, op.xs)
    # the probe returns d = fl(y32 - B): y32 within the bound of o64
    _rel(d + op.B, o64, f"{what}: forward top", OP_BOUND)
    g64, dx64, dxs64, _ = R.backward(op.W, op.x, cont, h0, d.astype(np.float64), op.xs)
    for k, v in g64.items():
        _rel(blobs[k], v, f"{what}: {k} gradient", OP_BOUND)
    if dx is not None:
        _rel(dx, dx64, f"{what}: dx", OP_BOUND)
    if dxs is not None:
        _rel(dxs, dxs64, f"{what}: dx_static", OP_BOUND)
    return o64


# (T, N, I, H, S, cont, grad_x, grad_static)
OP_CASES = [
    (1, 1, 1, 1, 0, "ones", True, False),
    (2, 3, 5, 7, 0, "start", True, False),
    (7, 1, 3, 64, 1, "random", True, True),
    (20, 32, 128, 257, 0, "ones", True, False),
    (7, 32, 6, 64, 5, "scaled", False, True),
    (20, 3, 1, 7, 0, "random", False, False),
    (2, 32, 257, 1, 3, "ones", True, False),
    (20, 1, 7, 257, 9, "start", True, True),
    (1, 32, 64, 64, 257, "scaled", True, True),
    (7, 3, 130, 7, 1, "ones", True, False),
    (20, 32, 3, 64, 6, "random", True, False),
    (2, 1, 9, 257, 0, "scaled", False, False),
    (7, 32, 64, 1, 0, "start", True, False),
    (4, 32769, 2, 3, 0, "random", True, False),  # T N = 131,076: the weight gradients take 249 widened chunks of 528
]


@pytest.mark.parametrize("T,N,I,H,S,kind,grad_x,grad_s", OP_CASES)
def test_rnn_op_against_float64(cos, tmp_path, T, N, I, H, S, kind, grad_x, grad_s):
    rng = np.random.RandomState(T * 1000 + N * 10 + H)
    op = _Op(cos, tmp_path, T, N, I, H, S, grad_x, grad_s and S > 0, rng)
    try:
        cont = _cont(rng, kind, T, N)
        got = op.call(cont)
        _compare(op, got, cont, np.zeros((N, H)), f"T={T} N={N} I={I} H={H} S={S} {kind}")
        if not grad_x:
            assert got[1] is None
    finally:
        op.close()


def test_a_second_call_adds_the_same_gradient_and_runs_are_bitwise_equal(cos, tmp_path):
    rng = np.random.RandomState(11)
    T, N, I, H, S = 7, 5, 9, 33, 4
    cont = _cont(rng, "start", T, N)  # cont_0 = 0: every call starts from a flushed state
    runs = []
    for r in range(2):
        (tmp_path / str(r)).mkdir()
        op = _Op(cos, tmp_path / str(r), T, N, I, H, S, True, True, np.random.RandomState(11))
        try:
            first = op.call(cont)
            again = op.call(cont)
            twice = op.call(cont, clear=False)
        finally:
            op.close()
        for k in first[0]:
            assert_bits_equal(again[0][k], first[0][k], f"{k}: two calls")
            assert_bits_equal(twice[0][k], first[0][k] * 2, f"{k}: a call without clearing adds it once more")
        runs.append(first)
    for k in runs[0][0]:
        assert_bits_equal(runs[1][0][k], runs[0][0][k], f"{k}: two engines")
    assert_bits_equal(runs[1][1], runs[0][1], "dx: two engines")


def test_the_hidden_state_is_carried_between_calls(cos, tmp_path):
    rng = np.random.RandomState(12)
    T, N, I, H, S = 6, 4, 5, 19, 3
    op = _Op(cos, tmp_path, T, N, I, H, S, True, True, rng)
    try:
        conts = [_cont(rng, "ones", T, N), _cont(rng, "random", T, N), _cont(rng, "ones", T, N)]
        conts[1][0, :2] = 1  # two streams continue across the boundary
        h = np.zeros((N, H))
        for c, cont in enumerate(conts):
            got = op.call(cont)
            _compare(op, got, cont, h, f"call {c}")
            h = R.forward(op.W, op.x, cont, h, op.xs)[1][-1]
        # cont = 0 at t = 0: the next call is the one a fresh engine makes
        flush = _cont(rng, "start", T, N)
        after = op.call(flush)
    finally:
        op.close()
    (tmp_path / "fresh").mkdir()
    fresh = _Op(cos, tmp_path / "fresh", T, N, I, H, S, True, True, np.random.RandomState(12))
    try:
        first = fresh.call(flush)
    finally:
        fresh.close()
    for k in first[0]:
        assert_bits_equal(after[0][k], first[0][k], f"{k}: a flushed call after three others")
    assert_bits_equal(after[1], first[1], "dx of a flushed call")


def test_inner_product_on_axis_two(cos, tmp_path):
    rng = np.random.RandomState(13)
    x = rng.randn(5, 3, 4, 6).astype(F32)
    w, b = rng.randn(9, 24).astype(F32), rng.randn(9).astype(F32)
    y64 = x.reshape(15, 24).astype(np.float64) @ w.T.astype(np.float64) + b
    B = (y64 - rng.randn(15, 9)).astype(F32).reshape(5, 3, 9)
    body = 'layer { name: "ip" type: "InnerProduct" bottom: "x0" top: "y" inner_product_param { num_output: 9 axis: 2 } }\n'
    text, ws = _net([x], body, [w, b], (5, 3, 9), B)
    (tmp_path / "net.prototxt").write_text(text)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().copy_(torch.from_numpy(np.concatenate([v.ravel() for v in ws])).cuda())
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.zeros(x.shape, device="cuda"), torch.zeros(B.shape, device="cuda")],
                                    loss.data_ptr()), net.last_error()
        assert net.synchronize(), net.last_error()
        g = to_host(net.diff())
    finally:
        net.deallocate()
    d = -g[-B.size:].reshape(15, 9).astype(np.float64)
    _rel(d + B.reshape(15, 9), y64, "forward", 1e-6)
    off = 2 * x.size
    _rel(g[off:off + w.size].reshape(w.shape), d.T @ x.reshape(15, 24), "weight gradient", 1e-6)
    _rel(g[off + w.size:off + w.size + 9], d.sum(0), "bias gradient", 1e-6)
    _rel(g[x.size:2 * x.size].reshape(15, 24), d @ w.astype(np.float64), "dx", 1e-6)


# --------------------------------------------------------------------------- the fixtures
BATCH = {LM: 32, CAPTION: 16}
STEPS = {LM: 20, CAPTION: 12}


def _solver(tmp_path, name, extra="", batch=None):
    text = open(os.path.join(CONFIGS, f"{name}_train_test.prototxt")).read()
    if batch is not None:
        text = text.replace(f"batch_size: {BATCH[name]}\n", f"batch_size: {batch}\n", 1)
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


def _batch(name, seed, n, first=False):
    """Time-major sentences [T, n] over the first 100 words: a token's successor is a fixed function of it, and
    sentences start at random steps (cont 0).  Unless `first`, a third of the streams continue from the previous batch (cont_0 = 1).  rnn_caption
    also gets an image [n, 1, 28, 28] whose mean picks the first token."""
    rng = np.random.RandomState(seed)
    T, V = STEPS[name], 100
    tokens = np.zeros((T + 1, n), np.int64)
    tokens[0] = rng.randint(0, V, n)
    cont = np.ones((T, n), F32)
    for t in range(T):
        start = rng.rand(n) < 0.15
        cont[t][start] = 0
        nxt = (tokens[t] * 7 + 3) % V
        tokens[t + 1] = np.where(rng.rand(n) < 0.1, rng.randint(0, V, n), nxt)
    cont[0] = 0 if first else (rng.rand(n) < 0.33)
    out = [cont, tokens[:-1].astype(F32), tokens[1:].astype(F32)]
    if name == CAPTION:
        img = rng.rand(n, 1, 28, 28).astype(F32)
        out.insert(0, img)
    return out


def _module(name):
    from caffeonspark_b200 import nets
    return nets.rnn_lm_module() if name == LM else nets.rnn_caption_module()


def _host_weights(name, seed):
    from caffeonspark_b200 import nets
    total = nets.RNN_LM_PARAM_COUNT if name == LM else nets.RNN_CAPTION_PARAM_COUNT
    assert total == sum(p.numel() for p in _module(name).parameters())
    return np.random.RandomState(seed).uniform(-0.1, 0.1, total).astype(F32)


def _zero_state(name, n, dtype, device):
    z = torch.zeros(n, 256 if name == LM else 128, dtype=dtype, device=device)
    return z if name == LM else (z, z.clone())


def _detach(h):
    return h.detach() if torch.is_tensor(h) else tuple(v.detach() for v in h)


def _reference_calls(name, w, batches, dtype, device):
    """[(loss, flat gradient)] of the PyTorch mirror over consecutive calls, the state carried and detached."""
    m = _module(name).to(device=device, dtype=dtype)
    _load(m, w)
    h = _zero_state(name, batches[0][-1].shape[1], dtype, device)
    out = []
    for b in batches:
        m.zero_grad()
        t = [torch.from_numpy(v).to(device=device) for v in b]
        if name == LM:
            cont, tok, tgt = t
            scores, h = m(tok, cont.to(dtype), h)
        else:
            img, cont, tok, tgt = t
            scores, h = m(img.to(dtype), cont.to(dtype), tok, h)
        loss = F.cross_entropy(scores.reshape(-1, scores.shape[-1]), tgt.reshape(-1).long())
        loss.backward()
        out.append((float(loss.detach()), _grads(m)))
        h = _detach(h)
    return out


def _engine_calls(net, batches):
    out = []
    for b in batches:
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in b], loss.data_ptr())
        assert net.synchronize(), net.last_error()
        out.append((float(loss.item()), to_host(net.diff())))
    return out


def _blob_errors(g, g64, counts):
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        scale = np.abs(g64[sl]).max()
        assert scale > 0
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / scale)
    return errs


@pytest.mark.parametrize("batch", ["own", "odd"])
@pytest.mark.parametrize("name", [LM, CAPTION])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name, batch):
    n = BATCH[name] if batch == "own" else {LM: 13, CAPTION: 7}[name]
    net = _net_of(cos, _solver(tmp_path, name, batch=n), fill=False)
    try:
        w = _host_weights(name, 21 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        batches = [_batch(name, n, n, first=True), _batch(name, n + 1, n)]
        got = _engine_calls(net, batches)
        counts = net.desc.counts
    finally:
        net.deallocate()
    # PyTorch fp32 on the CPU, where the bound was fixed: on the GPU, cuDNN's weight-gradient algorithm for
    # rnn_caption's conv1 misses it (9e-4 of the blob's largest gradient) even without TF32
    t32 = _reference_calls(name, w, batches, torch.float32, "cpu")
    t64 = _reference_calls(name, w, batches, torch.float64, "cpu")
    for c, ((l32, g), (lt, gt), (l64, g64)) in enumerate(zip(got, t32, t64)):
        assert abs(l32 - l64) <= 1e-6 * abs(l64), (c, l32, l64)
        assert abs(lt - l64) <= 1e-6 * abs(l64), (c, lt, l64)
        native, torch32 = _blob_errors(g, g64, counts), _blob_errors(gt, g64, counts)
        report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}" for k, (a, b) in
                           enumerate(zip(native, torch32)))
        assert max(native + torch32) <= NET_BOUND, f"call {c}, relative to max|g64| per blob: {report}"


def _train(net, name, steps, seed, check=None, first=True):
    losses = []
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, _batch(name, seed + t, BATCH[name], first=first and t == 0)), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", [LM, CAPTION])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    from caffeonspark_b200 import nets
    net = _net_of(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == (nets.RNN_LM_PARAM_COUNT if name == LM else nets.RNN_CAPTION_PARAM_COUNT)
        losses = _train(net, name, 150, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        first, last = losses[:10].mean(), losses[-20:].mean()
        assert last < 0.9 * first, (first, last)
    finally:
        net.deallocate()


def test_iter_size_two_carries_the_state_from_pass_to_pass(cos, tmp_path):
    """Pass 2 continues every stream of pass 1 (cont_0 = 1): diff_ must hold the two passes' gradients of the mirror
    with the state carried, and not those of two passes that each start from zero."""
    net = _net_of(cos, _solver(tmp_path, LM, "iter_size: 2\n"), fill=False)
    try:
        net.set_option("zero_diff", 0)
        w = _host_weights(LM, 5)
        net.data().copy_(torch.from_numpy(w).cuda())
        p1, p2 = _batch(LM, 1, 32, first=True), _batch(LM, 2, 32)
        p2[0][0] = 1
        net.diff().zero_()
        torch.cuda.synchronize()
        assert net.train_accumulate(0, [p1, p2]), net.last_error()
        assert net.synchronize(), net.last_error()
        g = to_host(net.diff())
        counts = net.desc.counts
    finally:
        net.deallocate()
    carried = _reference_calls(LM, w, [p1, p2], torch.float64, "cpu")
    fresh = _reference_calls(LM, w, [p2], torch.float64, "cpu")
    want = carried[0][1] + carried[1][1]
    wrong = carried[0][1] + fresh[0][1]
    assert max(_blob_errors(g, want, counts)) <= NET_BOUND
    assert max(_blob_errors(g, wrong, counts)) > 100 * NET_BOUND


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
                assert netz[r].train(0, _batch(name, 10 * r + t, BATCH[name], first=t == 0)), netz[r].last_error()
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


@pytest.mark.parametrize("name", [LM, CAPTION])
def test_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, solver, name), _two_rank_run(cos, solver, name), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_rnn_lm_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    """The hidden state is not in the snapshot, so the first batch after it starts every stream afresh (cont_0 = 0):
    from there the resumed net and the one that kept running agree bit for bit."""
    solver = _solver(tmp_path, LM, f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(a, LM, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        assert_bits_equal(cos.read_caffemodel_blob(model, "rnn", 2), w_a[289024:289024 + 65536], "W_hh")
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, LM, 3, 7), _train(b, LM, 3, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "three more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
