"""Caffe's N-D Convolution and Deconvolution on the built-in engine (DESIGN.md section 14), on the GPU.

The 3-D ops run through test_gpu_producer_ops.py's injector harness with B = 0, so y is also the top gradient the op
receives: y, dW, db and dx equal gemm3d_ref.py's fp32 restatement of the 3-D gathers (Vol2col, Col2volGather) bit for
bit across conv3d_ref.py's geometry sweep, down to the widened split-K chunks, and lie within conv3d_ref's float64
bounds.  A 1-D convolution over [N, C, L] equals the 2-D op over [N, C, 1, L] bit for bit.  Two engines give the same
bits, and a second call without clearing adds exactly the same gradient again.

The V-Net and C3D clip fixtures: per-blob gradients against float64 and PyTorch fp32 (F.conv3d on the CPU) at their
own batch and an odd one; their 5-D weights filled with Caffe's fans; train() alone with every update equal to the
oracle's, on one rank and two in-process ranks; and V-Net snapshots that resume bit-exact in BINARYPROTO and HDF5,
with [Cout, Cin, KD, KH, KW] weight shapes read back from the written files."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv3d_ref as C3
import gemm3d_ref as G3
import gemm_ref as G
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_embed import _caffemodel_layers
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import _close, _engine, _same
from test_hdf5_io import MiniH5

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
NET_BOUND = 3e-5  # PyTorch fp32 on the CPU reaches 1.03e-5 (vnet3d b3, blob 25: up1's bias); the engine 1e-6


def _fields(geo3):
    kd, kh, kw, sd, sh, sw, pd, ph, pw = geo3
    return (f"kernel_size: {kd} kernel_size: {kh} kernel_size: {kw} stride: {sd} stride: {sh} stride: {sw} "
            f"pad: {pd} pad: {ph} pad: {pw}")


def _layer(kind, cout, geo3, bias, bottom="x0"):
    return (f'layer {{ name: "c" type: "{kind}" bottom: "{bottom}" top: "y" convolution_param {{ num_output: {cout} '
            f'{_fields(geo3)} bias_term: {"true" if bias else "false"} }} }}\n')


def _run(cos, tmp_path, case, deconv):
    x, w, b = C3.inputs(case, deconv)
    n, cin, d, h, wd, cout, geo3, bias = case
    dhw = (C3.deconv_out3 if deconv else C3.out3)((d, h, wd), geo3)
    shape = (n, cout) + dhw
    r = _engine(cos, tmp_path, [x], _layer("Deconvolution" if deconv else "Convolution", cout, geo3, bias),
                [w] + ([b] if bias else []), shape, np.zeros(shape, F32))
    return x, w, b, r


# --------------------------------------------------------------------------- the 3-D ops, bit for bit
@pytest.mark.parametrize("case", C3.CONV3D_CASES, ids=str)
def test_convolution3d_bit_for_bit(cos, tmp_path, case):
    x, w, b, r = _run(cos, tmp_path, case, False)
    geo3, y = case[6], r["d"]
    _same(y, G3.conv3d_forward(x, w, b, geo3), "y")
    _same(r["grads"][0], G3.conv3d_weight_grad(x, y, geo3), "dW")
    if b is not None:
        _same(r["grads"][1], G.bias_grad(y, y.shape[0], y.shape[1], int(np.prod(y.shape[2:]))), "db")
    _same(r["dx"][0], G3.conv3d_data_grad(y, w, None, x.shape, geo3), "dx")
    by, bw, bb, bx = C3.conv3d_bounds(x, w, b, y, geo3)
    _close(y, C3.conv3d64(x, w, b, geo3), by, "y against float64")
    dw, db, dx = C3.conv3d_backward64(x, w, y, geo3)
    _close(r["grads"][0], dw, bw, "dW against float64")
    if b is not None:
        _close(r["grads"][1], db, bb, "db against float64")
    _close(r["dx"][0], dx, bx, "dx against float64")


@pytest.mark.parametrize("case", C3.DECONV3D_CASES, ids=str)
def test_deconvolution3d_bit_for_bit(cos, tmp_path, case):
    x, w, b, r = _run(cos, tmp_path, case, True)
    geo3, y = case[6], r["d"]
    _same(y, G3.deconv3d_forward(x, w, b, geo3, y.shape[2:]), "y")
    _same(r["grads"][0], G3.deconv3d_weight_grad(x, y, geo3), "dW")
    if b is not None:
        _same(r["grads"][1], G.bias_grad(y, y.shape[0], y.shape[1], int(np.prod(y.shape[2:]))), "db")
    _same(r["dx"][0], G3.deconv3d_data_grad(y, w, geo3), "dx")
    by, bw, bb, bx = C3.deconv3d_bounds(x, w, b, y, geo3)
    _close(y, C3.deconv3d64(x, w, b, geo3), by, "y against float64")
    dw, db, dx = C3.deconv3d_backward64(x, w, y, geo3)
    _close(r["grads"][0], dw, bw, "dW against float64")
    if b is not None:
        _close(r["grads"][1], db, bb, "db against float64")
    _close(r["dx"][0], dx, bx, "dx against float64")


# --------------------------------------------------------------------------- 1-D: the 2-D op over [N, C, 1, L]
@pytest.mark.parametrize("kind,fields,cout", [
    ("Convolution", "kernel_size: 3 stride: 2 pad: 1", 4),
    ("Convolution", "kernel_size: 5", 65),
    ("Deconvolution", "kernel_size: 4 stride: 2 pad: 1", 3),
])
def test_one_spatial_axis_is_the_2d_op_on_a_height_of_one(cos, tmp_path, kind, fields, cout):
    rng = np.random.default_rng(cout)
    x = rng.standard_normal((3, 5, 37)).astype(F32)
    k, s, p = (int(v) for v in (fields.split()[1::2] + ["1", "0"])[:3])
    wshape = (5, cout, k) if kind == "Deconvolution" else (cout, 5, k)
    w = (rng.standard_normal(wshape) / np.sqrt(5 * k)).astype(F32)
    b = (rng.standard_normal(cout) * 0.1).astype(F32)
    L = s * (37 - 1) + k - 2 * p if kind == "Deconvolution" else (37 + 2 * p - k) // s + 1
    body = f'layer {{ name: "c" type: "{kind}" bottom: "x0" top: "y" convolution_param {{ num_output: {cout} {fields} }} }}\n'
    (tmp_path / "1d").mkdir()
    one = _engine(cos, tmp_path / "1d", [x], body, [w, b], (3, cout, L), np.zeros((3, cout, L), F32))
    body2 = (f'layer {{ name: "c" type: "{kind}" bottom: "x0" top: "y" convolution_param {{ num_output: {cout} '
             f'kernel_h: 1 kernel_w: {k} stride_h: 1 stride_w: {s} pad_h: 0 pad_w: {p} }} }}\n')
    (tmp_path / "2d").mkdir()
    two = _engine(cos, tmp_path / "2d", [x[:, :, None]], body2, [w[:, :, None], b], (3, cout, 1, L),
                  np.zeros((3, cout, 1, L), F32))
    assert_bits_equal(one["d"], two["d"][:, :, 0], "y")
    assert_bits_equal(one["grads"][0], two["grads"][0][:, :, 0], "dW")
    assert_bits_equal(one["grads"][1], two["grads"][1], "db")
    assert_bits_equal(one["dx"][0], two["dx"][0][:, :, 0], "dx")


# --------------------------------------------------------------------------- repeatability
def _twice(cos, tmp_path, case):
    """-> (diff after one call, diff after a second call without clearing) of one engine"""
    x, w, b = C3.inputs(case)
    n, cin, d, h, wd, cout, geo3, bias = case
    shape = (n, cout) + C3.out3((d, h, wd), geo3)
    body = ('layer { name: "in" type: "Input" top: "x" top: "t" input_param { ' +
            " ".join("shape { " + " ".join(f"dim: {v}" for v in s) + " }" for s in (x.shape, shape)) + " } }\n" +
            _layer("Convolution", cout, geo3, True, bottom="x") +
            'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" }\n')
    (tmp_path / "net.prototxt").write_text('name: "t"\n' + body)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = cos.CaffeNet(str(tmp_path / "solver.prototxt"), "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().copy_(torch.from_numpy(np.concatenate([w.ravel(), b.ravel()])).cuda())
        net.diff().zero_()
        t = np.random.default_rng(1).standard_normal(shape).astype(F32)
        ins = [torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()]
        loss = torch.zeros(1, device="cuda")
        out = []
        for _ in range(2):
            assert net.forward_backward(ins, loss.data_ptr()), net.last_error()
            assert net.synchronize(), net.last_error()
            out.append(to_host(net.diff()))
        return out
    finally:
        net.deallocate()


@pytest.mark.parametrize("case", [C3.CONV3D_CASES[2], C3.CONV3D_CASES[-1]], ids=str)
def test_two_engines_agree_and_a_second_call_adds_the_same_gradient(cos, tmp_path, case):
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    a1, a2 = _twice(cos, tmp_path / "a", case)
    b1, b2 = _twice(cos, tmp_path / "b", case)
    assert_bits_equal(b1, a1, "two engines")
    assert_bits_equal(b2, a2, "two engines, second call")
    assert_bits_equal(a2, a1 + a1, "the second call adds the same gradient (g + g is exact)")


# --------------------------------------------------------------------------- the fixtures
FIXTURES = {
    "vnet3d": dict(batch=2, odd=3, param_count=64362),
    "c3d_clip": dict(batch=4, odd=3, param_count=87146),
}


def _solver(tmp_path, name, extra="", batch=None):
    text = open(os.path.join(CONFIGS, f"{name}_train_test.prototxt")).read()
    if batch is not None:
        text = text.replace(f"batch_size: {FIXTURES[name]['batch']}\n", f"batch_size: {batch}\n")
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


def batch_of(name, seed, n):
    """vnet3d: n volumes [n, 32, 32, 32] of two bright balls on noise and their per-voxel labels (1 inside a ball);
    c3d_clip: n clips [n, 24, 56, 56] of a bar moving at one of 10 speeds, and the speed as the label [n, 1, 1, 1]"""
    rng = np.random.RandomState(seed)
    if name == "vnet3d":
        zz, yy, xx = np.mgrid[0:32, 0:32, 0:32]
        mask = np.zeros((n, 32, 32, 32), F32)
        for i in range(n):
            for _ in range(2):
                c, r = rng.randint(6, 26, 3), rng.randint(4, 9)
                mask[i][(zz - c[0]) ** 2 + (yy - c[1]) ** 2 + (xx - c[2]) ** 2 < r * r] = 1
        return [(0.6 * mask + 0.4 * rng.rand(n, 32, 32, 32)).astype(F32), mask]
    label = rng.randint(0, 10, n)
    clips = 0.3 * rng.rand(n, 3, 8, 56, 56)
    for i in range(n):
        for t in range(8):
            clips[i, :, t, :, (4 + t * label[i]) % 56] += 1.0
    return [clips.reshape(n, 24, 56, 56).astype(F32), label.reshape(n, 1, 1, 1).astype(F32)]


def host_weights(name, seed):
    """Flat weights drawn on the host: each weight Gaussian with Caffe's msra deviation sqrt(2 / fan_in), each PReLU
    slope uniform in [0.1, 0.4), each bias uniform in [-0.05, 0.05)"""
    from caffeonspark_b200 import nets
    rng = np.random.RandomState(seed)
    parts = []
    for nm, p in _module(name).named_parameters():
        if p.dim() > 1:
            parts.append((rng.randn(p.numel()) * np.sqrt(2.0 / (p.numel() // p.shape[0]))).astype(F32))
        elif "prelu" in nm:
            parts.append(rng.uniform(0.1, 0.4, p.numel()).astype(F32))
        else:
            parts.append(rng.uniform(-0.05, 0.05, p.numel()).astype(F32))
    w = np.concatenate(parts)
    assert w.size == getattr(nets, name.upper() + "_PARAM_COUNT")
    return w


def _module(name):
    from caffeonspark_b200 import nets
    return nets.vnet3d_module() if name == "vnet3d" else nets.c3d_clip_module()


def reference(name, w, batch, dtype):
    """(loss, flat gradient) of the fixture's PyTorch mirror on the CPU on the flat weights w"""
    m = _module(name).to(dtype=dtype)
    _load(m, w)
    n = batch[0].shape[0]
    if name == "vnet3d":
        scores = m(torch.from_numpy(batch[0]).to(dtype).view(n, 1, 32, 32, 32))
        loss = F.cross_entropy(scores.permute(0, 2, 3, 4, 1).reshape(-1, 2), torch.from_numpy(batch[1]).long().view(-1))
    else:
        scores = m(torch.from_numpy(batch[0]).to(dtype).view(n, 3, 8, 56, 56))
        loss = F.cross_entropy(scores, torch.from_numpy(batch[1]).long().view(-1))
    loss.backward()
    return float(loss.detach()), _grads(m)


def blob_errors(g, g64, counts):
    """Per blob, the largest error relative to the blob's largest float64 gradient, or to 1% of the net's largest
    where the blob's is smaller"""
    floor = 1e-2 * np.abs(g64).max()
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / max(np.abs(g64[sl]).max(), floor))
    return errs


@pytest.mark.parametrize("name,which", [(n, w) for n in FIXTURES for w in ("batch", "odd")])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, name, which):
    n = FIXTURES[name][which]
    net = _net_of(cos, _solver(tmp_path, name, batch=n), fill=False)
    try:
        w = host_weights(name, 31 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        b = batch_of(name, n, n)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        assert net.forward_backward([torch.from_numpy(v).cuda() for v in b], loss.data_ptr())
        assert net.synchronize(), net.last_error()
        l32, g, counts = float(loss.item()), to_host(net.diff()), net.desc.counts
    finally:
        net.deallocate()
    tf32 = torch.backends.cudnn.allow_tf32
    lt, gt = reference(name, w, b, torch.float32)
    l64, g64 = reference(name, w, b, torch.float64)
    assert torch.backends.cudnn.allow_tf32 == tf32
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    native, torch32 = blob_errors(g, g64, counts), blob_errors(gt, g64, counts)
    report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {c:.2e}" for k, (a, c) in enumerate(zip(native, torch32)))
    print(f"{name} b{n}: worst native {max(native):.2e}, worst PyTorch fp32 {max(torch32):.2e}")
    assert max(native + torch32) <= NET_BOUND, f"relative to max|g64| per blob: {report}"


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_fillers_use_caffes_fans(cos, tmp_path, name):
    """msra (and c3d's xavier fc4) over 5-D weights: std sqrt(2 / fan_in) (sqrt(1 / fan_in) for xavier's uniform
    variance), fan_in = count / shape(0)"""
    net = _net_of(cos, _solver(tmp_path, name), fill=True)
    try:
        w, d = to_host(net.data()), net.desc
    finally:
        net.deallocate()
    text = cos.native_producer_plan(_solver(tmp_path, name))
    fillers = [line.split()[4] for line in text.splitlines() if line.startswith("blob ")]
    off = 0
    for k, (c, shape) in enumerate(zip(d.counts, [tuple(int(v) for v in line.split()[3].split("x"))
                                                   for line in text.splitlines() if line.startswith("blob ")])):
        v = w[off:off + c].astype(np.float64)
        off += c
        if fillers[k] == "msra":
            want = np.sqrt(2.0 / (c // shape[0]))
        elif fillers[k] == "xavier":
            want = np.sqrt(3.0 / (c // shape[0])) / np.sqrt(3.0)  # uniform in +-sqrt(3 / fan_in)
        else:
            continue
        assert len(shape) in (2, 5)
        assert abs(v.std() / want - 1) < 0.1 + 3 / np.sqrt(c), (k, shape, v.std(), want)


def _train(name, net, steps, seed, check=None):
    losses = []
    n = FIXTURES[name]["batch"]
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, batch_of(name, seed + t, n)), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_trains_through_train_alone(cos, oracle, tmp_path, name):
    net = _net_of(cos, _solver(tmp_path, name))
    try:
        assert net.param_count() == FIXTURES[name]["param_count"]
        losses = _train(name, net, 12, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-4:].mean() < losses[:2].mean(), losses
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

        def run(r):
            for t in range(3):
                assert netz[r].train(0, batch_of(name, 10 * r + t, FIXTURES[name]["batch"])), netz[r].last_error()
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


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_two_ranks_in_process(cos, tmp_path, name):
    solver = _solver(tmp_path, name)
    assert_bits_equal(_two_rank_run(cos, name, solver), _two_rank_run(cos, name, solver), "two whole runs")


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_vnet3d_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    name = "vnet3d"
    solver = _solver(tmp_path, name, extra=f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(name, a, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        # conv4's weight [16, 32, 3, 3, 3] at 45976, up1's (a Deconvolution's [Cin, Cout, KD, KH, KW]) at 59832
        for layer, off, shape in (("conv4", 45976, (16, 32, 3, 3, 3)), ("up1", 59832, (16, 8, 2, 2, 2))):
            assert_bits_equal(cos.read_caffemodel_blob(model, layer, 0), w_a[off:off + int(np.prod(shape))], layer)
            if fmt == "BINARYPROTO":
                assert _caffemodel_layers(model)[layer][1][0] == shape
            else:
                assert tuple(MiniH5(model).objects[f"/data/{layer}/0"]["shape"]) == shape
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(name, a, 2, 7), _train(name, b, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
