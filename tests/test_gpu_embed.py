"""Embed and Reshape on the built-in engine (DESIGN.md section 14) on the GPU.

The Embed op alone runs through test_gpu_producer_ops.py's injector harness: its ids come straight from a staged input
and its top meets the EuclideanLoss probe, which returns the top gradient d exactly.  The forward is compared by value
(a table row, or one rounding of row + bias), and the weight gradient bit for bit against embed_ref.embed_backward_cpu,
Caffe's Backward_cpu order.  Two calls from a cleared diff_ must agree bit for bit, and a third without clearing must
equal the restatement over the doubled occurrence list.  Invalid ids embed as zeros, add no weight gradient and set
status 503.

Both embedding fixtures are checked against float64 and PyTorch fp32 at their own batch and an odd one, trained through
train() alone with every update checked against the oracle, on one rank and on two in-process ranks, and the n-gram
model's snapshots resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import embed_ref as E
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import _close, _net, _same

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
TEXT, LM = "text_cnn", "ngram_lm"


# --------------------------------------------------------------------------- the op
def _ids(rng, kind, shape, K):
    M = int(np.prod(shape))
    if kind == "random":
        v = rng.randint(0, K, M)
    elif kind == "skewed":  # a few ids repeat many times
        v = (rng.zipf(1.3, M) - 1) % K
    elif kind == "equal":
        v = np.full(M, rng.randint(0, K))
    elif kind == "distinct":
        v = rng.permutation(K)[:M]
    else:  # "edges": 0 and K - 1 first and last, the rest anywhere
        v = rng.randint(0, K, M)
        v[0], v[-1] = 0, K - 1
        v[M // 2] = K - 1
    return v.astype(F32).reshape(shape)


def _embed_layers(name, bottom, top, K, N, bias, param=""):
    return (f'layer {{ name: "{name}" type: "Embed" bottom: "{bottom}" top: "{top}" {param} embed_param {{ '
            f'input_dim: {K} num_output: {N} bias_term: {"true" if bias else "false"} }} }}\n')


def _run(cos, tmp_path, staged, body, weights, out_shape, B, calls=3):
    """Input -> `body` (reads the staged ids, writes "y") -> probe + EuclideanLoss.  Three calls: two from a cleared
    diff_ and one without clearing.  -> (per-call flat diff_, probe d of call 1)."""
    text, ws = _net([], body, weights, out_shape, B, staged)
    inputs = [np.zeros(out_shape, F32)] + [np.asarray(v, F32) for v in staged.values()]
    (tmp_path / "net.prototxt").write_text(text)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        flat = np.concatenate([w.ravel() for w in ws])
        assert net.param_count() == flat.size
        net.data().copy_(torch.from_numpy(flat).cuda())
        dev = [torch.from_numpy(v).cuda() for v in inputs]
        loss = torch.zeros(1, device="cuda")
        runs = []
        for c in range(calls):
            if c < 2:
                net.diff().zero_()
            torch.cuda.synchronize()
            assert net.forward_backward(dev, loss.data_ptr()), net.last_error()
            assert net.synchronize(), net.last_error()
            runs.append(to_host(net.diff()))
    finally:
        net.deallocate()
    assert_bits_equal(runs[1], runs[0], "diff_ of two calls")
    return runs, -runs[0][-B.size:].reshape(out_shape)


# (ids shape, num_output, input_dim, ids, bias)
OP_CASES = [
    ((1,), 1, 10, "random", True),
    ((7,), 3, 5, "random", False),
    ((7,), 1025, 7, "distinct", True),
    ((4096,), 64, 1000, "random", True),
    ((4096,), 300, 100, "equal", False),
    ((4096,), 64, 4096, "distinct", True),
    ((64, 64), 300, 5000, "skewed", False),
    ((8, 16, 32), 1025, 300, "random", True),
    ((65536,), 1, 50, "random", False),
    ((65536,), 3, 1, "equal", True),
    ((16, 4096), 64, 2000, "skewed", True),
    ((256, 256), 300, 50000, "skewed", False),
    ((1000,), 1, 2 ** 24, "edges", True),
    ((257,), 64, 9, "edges", False),
]


@pytest.mark.parametrize("shape,N,K,kind,bias", OP_CASES)
def test_embed_op(cos, tmp_path, shape, N, K, kind, bias):
    rng = np.random.RandomState(N + K + len(shape))
    ids = _ids(rng, kind, shape, K)
    w = rng.randn(K, N).astype(F32)
    b = rng.randn(N).astype(F32) if bias else None
    y32 = w[ids.astype(np.int64)] + (b if bias else F32(0))  # fp32 + fp32: the kernel's one rounding
    out_shape = shape + (N,)
    e = (rng.randn(*out_shape) * np.exp2(rng.randint(-6, 6, out_shape[:-1] + (1,)))).astype(F32)
    B = (y32 - e).astype(F32)
    weights = [w] + ([b] if bias else [])
    runs, d = _run(cos, tmp_path, {"ids": ids}, _embed_layers("e", "ids", "y", K, N, bias), weights, out_shape, B)
    _same(d, y32 - B, "the forward: d = fl(y - B)")
    gw = runs[0][:K * N].reshape(K, N)
    assert_bits_equal(gw, E.embed_backward_cpu(ids, d, np.zeros((K, N), F32)), "weight gradient, Caffe's order")
    twice = E.embed_backward_cpu(np.concatenate([ids.ravel()] * 2), np.concatenate([d.reshape(-1, N)] * 2),
                                 np.zeros((K, N), F32))
    assert_bits_equal(runs[2][:K * N].reshape(K, N), twice, "a call without clearing: the doubled occurrence list")
    if bias:
        gb = runs[0][K * N:K * N + N]
        ref = E.embed_bias_grad(ids, d, N)
        bound = ids.size * 2.0 ** -23 * np.abs(d.reshape(-1, N)).astype(np.float64).sum(axis=0)
        _close(gb, ref, bound, "bias gradient")


def test_two_embeds_share_one_table(cos, tmp_path):
    rng = np.random.RandomState(3)
    K, N = 40, 12
    a, b = _ids(rng, "skewed", (300,), K), _ids(rng, "skewed", (5, 41), K)
    w = rng.randn(K, N).astype(F32)
    param = 'param { name: "table" }'
    body = (_embed_layers("e1", "a", "ya", K, N, False, param) + _embed_layers("e2", "b", "yb", K, N, False, param) +
            'layer { name: "fl" type: "Reshape" bottom: "yb" top: "yb2" reshape_param { shape { dim: -1 } axis: 0 '
            'num_axes: 2 } }\n'
            'layer { name: "cat" type: "Concat" bottom: "ya" bottom: "yb2" top: "y" concat_param { axis: 0 } }\n')
    y32 = np.concatenate([w[a.astype(int)], w[b.astype(int)].reshape(-1, N)])
    e = rng.randn(*y32.shape).astype(F32)
    B = (y32 - e).astype(F32)
    runs, d = _run(cos, tmp_path, {"a": a, "b": b}, body, [w], y32.shape, B)
    _same(d, y32 - B, "the forward")
    # Caffe's backward runs the layers in reverse: e2's occurrences first, then e1's, into one diff
    want = E.embed_backward_cpu(b, d[300:], np.zeros((K, N), F32))
    want = E.embed_backward_cpu(a, d[:300], want)
    assert_bits_equal(runs[0][:K * N].reshape(K, N), want, "shared table gradient")


def test_invalid_ids_embed_zeros_add_nothing_and_set_the_status(cos, tmp_path):
    K, N = 6, 5
    rng = np.random.RandomState(4)
    ids = np.array([-1, K, 0.5, np.nan, np.inf, 2, 0, 2], F32)
    w, b = rng.randn(K, N).astype(F32), rng.randn(N).astype(F32)
    B = np.zeros((ids.size, N), F32)
    text, ws = _net([], _embed_layers("e", "ids", "y", K, N, True), [w, b], B.shape, B, {"ids": ids})
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
        assert net.forward_backward([torch.zeros(B.shape, device="cuda"), torch.from_numpy(ids).cuda()],
                                    loss.data_ptr())
        assert not net.synchronize()
        assert "Embed: an id that is not an integer in [0, input_dim)" in net.last_error(), net.last_error()
        assert "status 503" in net.last_error()
        g = to_host(net.diff())
        d = -g[-B.size:].reshape(B.shape)  # d = y - 0
        assert np.array_equal(d[:5], np.tile(b, (5, 1))), "invalid ids embed as the bias alone"
        assert np.array_equal(d[5:], w[[2, 0, 2]] + b)
        assert_bits_equal(g[:K * N].reshape(K, N), E.embed_backward_cpu(ids, d, np.zeros((K, N), F32)),
                          "only the valid ids add")
        assert not g[:K * N].reshape(K, N)[[1, 3, 4, 5]].any()
        assert net.synchronize(), "the status is reported once"
    finally:
        net.deallocate()


# --------------------------------------------------------------------------- the fixtures
# The per-blob gradient bound, relative to the blob's largest float64 gradient, for the engine and PyTorch fp32 alike.
# The float64 reference takes each MAX pool's winners from the fp32 forward (test_gpu_neuron_nets.py explains why).  The
# bound was fixed on the CPU from these very weights and batches (_host_weights, _batch) at the fixtures' batches and
# the odd ones below: PyTorch fp32 on the CPU reached at worst 9.7e-7 of a blob's largest gradient (text_cnn) and
# 4.5e-7 (ngram_lm), the loss 1.0e-7 relative.
NET_BOUND = 1e-5
STEPS = 120
BATCH = {TEXT: 50, LM: 128}


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


def _batch(name, seed, n):
    """text_cnn: uniform tokens from [20, 5000) with eight cue tokens, from [0, 10) for class 1 and [10, 20) for
    class 0.  ngram_lm: skewed (Zipf) context ids; the next token is the last one plus 1."""
    rng = np.random.RandomState(seed)
    if name == TEXT:
        y = rng.randint(0, 2, n)
        x = rng.randint(20, 5000, (n, 32))
        for i in range(n):
            x[i, rng.choice(32, 8, replace=False)] = rng.randint(0, 10, 8) + 10 * (1 - y[i])
        return x.astype(F32), y.astype(F32)
    x = (rng.zipf(1.2, (n, 4)) - 1) % 2000
    return x.astype(F32), ((x[:, 3] + 1) % 2000).astype(F32)


def _module(name):
    from caffeonspark_b200 import nets
    return nets.text_cnn_module() if name == TEXT else nets.ngram_lm_module()


def _reference(name, w, x, y, dtype, device, argmax=None):
    """(loss, flat gradient, each MAX pool's winners) of the PyTorch module on the flat weights w.  With `argmax`, every
    MAX pool takes its winners from it instead of choosing them (the first maximum wins, as in Caffe)."""
    m = _module(name).to(device=device, dtype=dtype)
    _load(m, w)
    ids, taken = torch.from_numpy(x).to(device), []
    if name == TEXT:
        h = m.embed(ids).unsqueeze(1)
        pooled = []
        for i, c in enumerate(m.convs):
            r = torch.relu(c(h)).flatten(2)
            idx = r.argmax(2, keepdim=True) if argmax is None else argmax[i].to(device)
            taken.append(idx.cpu())
            pooled.append(r.gather(2, idx).squeeze(2))
        out = m.ip(torch.cat(pooled, 1))
    else:
        out = m(ids)
    loss = F.cross_entropy(out, torch.from_numpy(y).to(device).long())
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def _host_weights(name, seed):
    """Flat weights uniform in [-0.1, 0.1), drawn on the host so that the bound's CPU runs use them too."""
    from caffeonspark_b200 import nets
    total = nets.TEXT_CNN_PARAM_COUNT if name == TEXT else nets.NGRAM_LM_PARAM_COUNT
    assert total == sum(p.numel() for p in _module(name).parameters())
    return np.random.RandomState(seed).uniform(-0.1, 0.1, total).astype(F32)


def _blob_errors(g, gt, g64, counts):
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        scale = np.abs(g64[sl]).max()
        assert scale > 0
        errs.append([np.abs(got[sl].astype(np.float64) - g64[sl]).max() / scale for got in (g, gt)])
    assert off == g64.size
    return errs


@pytest.mark.parametrize("batch", ["own", "odd"])
@pytest.mark.parametrize("name", [TEXT, LM])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name, batch):
    n = BATCH[name] if batch == "own" else {TEXT: 37, LM: 77}[name]
    net = _net_of(cos, _solver(tmp_path, name, batch=n), fill=False)
    try:
        w = _host_weights(name, 21 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        x, y = _batch(name, n, n)
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
        assert abs(l32 - l64) <= 1e-6 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-6 * abs(l64), (lt, l64)
        errs = _blob_errors(g, gt, g64, net.desc.counts)
        report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}" for k, (a, b) in enumerate(errs))
        assert max(max(e) for e in errs) <= NET_BOUND, f"relative to max|g64| per blob, bound {NET_BOUND}: {report}"
    finally:
        net.deallocate()


def _train(net, name, steps, seed, check=None):
    losses = []
    for t in range(steps):
        x, y = _batch(name, seed + t, BATCH[name])
        if check:
            check.before()
        assert net.train(0, [x, y]), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", [TEXT, LM])
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    from caffeonspark_b200 import nets
    net = _net_of(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == (nets.TEXT_CNN_PARAM_COUNT if name == TEXT else nets.NGRAM_LM_PARAM_COUNT)
        losses = _train(net, name, STEPS, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        first, last = losses[:10].mean(), losses[-20:].mean()
        assert last < first, (first, last)
    finally:
        net.deallocate()


def test_a_bad_id_reaches_train(cos, tmp_path):
    net = _net_of(cos, _solver(tmp_path, LM))
    try:
        x, y = _batch(LM, 5, BATCH[LM])
        x[3, 1] = 2000
        assert not (net.train(0, [x, y]) and net.synchronize())
        assert "Embed: an id that is not an integer" in net.last_error(), net.last_error()
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
                assert netz[r].train(0, list(_batch(name, 10 * r + t, BATCH[name]))), netz[r].last_error()
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


@pytest.mark.parametrize("name", [TEXT, LM])
def test_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, solver, name), _two_rank_run(cos, solver, name), "two whole runs")


@pytest.mark.parametrize("name", [TEXT, LM])
def test_two_fresh_runs_give_identical_weights(cos, tmp_path, name):
    runs = []
    for r in range(2):
        (tmp_path / str(r)).mkdir()
        net = _net_of(cos, _solver(tmp_path / str(r), name))
        try:
            _train(net, name, 5, 50)
            runs.append(to_host(net.data()))
        finally:
            net.deallocate()
    assert_bits_equal(runs[1], runs[0], "two fresh runs")


def _varint(b, i):
    v, s = 0, 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7F) << s
        s += 7
        if c < 0x80:
            return v, i


def _fields(b):
    """protobuf wire format -> [(field number, wire type, value or bytes)]"""
    out, i = [], 0
    while i < len(b):
        key, i = _varint(b, i)
        f, t = key >> 3, key & 7
        if t == 0:
            v, i = _varint(b, i)
        elif t == 2:
            n, i = _varint(b, i)
            v, i = b[i:i + n], i + n
        elif t == 5:
            v, i = b[i:i + 4], i + 4
        elif t == 1:
            v, i = b[i:i + 8], i + 8
        else:
            raise ValueError(f"wire type {t}")
        out.append((f, t, v))
    return out


def _caffemodel_layers(path):
    """-> {layer name: (type, [blob shapes])} of a binary .caffemodel (NetParameter.layer = 100, LayerParameter name
    = 1, type = 2, blobs = 7, BlobProto.shape = 7, BlobShape.dim = 1)"""
    layers = {}
    for f, _, v in _fields(open(path, "rb").read()):
        if f != 100:
            continue
        lf = _fields(v)
        name = next(x for g, _, x in lf if g == 1).decode()
        type_ = next(x for g, _, x in lf if g == 2).decode()
        shapes = []
        for g, _, blob in lf:
            if g != 7:
                continue
            dims = []
            for h, t, sh in _fields(blob):
                if h != 7:
                    continue
                for k, kt, d in _fields(sh):
                    if kt == 0:
                        dims.append(d)
                    else:  # packed
                        j = 0
                        while j < len(d):
                            x, j = _varint(d, j)
                            dims.append(x)
            shapes.append(tuple(dims))
        layers[name] = (type_, shapes)
    return layers


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_ngram_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, LM, f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(a, LM, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        assert_bits_equal(cos.read_caffemodel_blob(model, "embed", 0), w_a[:64000], "embed table")
        assert_bits_equal(cos.read_caffemodel_blob(model, "embed", 1), w_a[64000:64032], "embed bias")
        if fmt == "BINARYPROTO":
            assert _caffemodel_layers(model)["embed"] == ("Embed", [(2000, 32), (32,)])
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, LM, 2, 7), _train(b, LM, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
