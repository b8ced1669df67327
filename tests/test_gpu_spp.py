"""Caffe's SPP layer on the built-in engine (DESIGN.md section 14), on the GPU.

The kernels alone (layers.spp_forward / spp_backward) against spp_ref.py's fp32 restatement of Caffe's expansion, bit
for bit as uint32 (every NaN taken as the GPU's canonical one), MAX and AVE, on values with NaN, both infinities, both
zeros, -FLT_MAX, ties and a plane with no value > -FLT_MAX: Caffe's test geometries, the fixture's, an SPP-net head
and maps padded in both dimensions.  dx is NaN-poisoned first, and two calls give the same bits.

The op in the engine through test_gpu_producer_ops.py's injector harness.  The SPP CIFAR-10-quick fixture, and its AVE
variant, against the same net with SPP written out as Caffe's expansion (an explicit Split, one Pooling and one
Flatten per level and a Concat) on the engine: the loss, every gradient and every train() update equal bit for bit.
The fixture's gradients against float64 and the PyTorch fp32 mirror; train() with every update equal to the oracle's
on one rank and two in-process ranks; BINARYPROTO and HDF5 snapshots that resume bit-exact."""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import spp_ref as R
from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_crop import _harness_equal
from test_gpu_native_producer import _UpdateCheck, _grads, _load
from test_gpu_producer_ops import _engine

pytestmark = pytest.mark.gpu

F32 = np.float32
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
NAME = "cifar10_quick_spp"
BATCH = 100
NET_BOUND = 1e-5  # PyTorch fp32 on the CPU reaches 6.5e-7 on b100 (weights host_weights(121))
POISON = np.uint32(0x7FBADBAD)


# --------------------------------------------------------------------------- the kernels
KERNEL_CASES = [  # (bottom, pyramid height)
    ((2, 3, 9, 8), 3), ((10, 3, 7, 7), 3), ((4, 3, 1024, 765), 5),  # Caffe's test_spp_layer.cpp
    ((100, 64, 6, 6), 3),    # the fixture
    ((64, 256, 13, 13), 3),  # an SPP-net head over conv5
    ((3, 4, 6, 10), 3),      # padded in both dimensions
    ((2, 5, 11, 9), 2), ((2, 3, 9, 8), 1), ((1, 2, 16, 16), 4),
]


def _kernels(x, h, pool, dy):
    from caffeonspark_b200 import layers
    xt = torch.from_numpy(x).cuda()
    y, arg = layers.spp_forward(xt, h, pool)
    dx = torch.from_numpy(np.full(x.shape, POISON, np.uint32).view(F32)).cuda()
    layers.spp_backward(torch.from_numpy(dy).cuda(), arg, x.shape, h, pool, out=dx)
    torch.cuda.synchronize()
    return to_host(y), (to_host(arg) if arg is not None else None), to_host(dx)


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("shape,h", KERNEL_CASES)
def test_kernels_bit_for_bit(cos, shape, h, pool):
    rng = np.random.RandomState(sum(shape) + h)
    x = R.specials(rng, shape)
    want_y, want_arg = R.expansion32(x, h, pool)
    dy = R.specials(rng, want_y.shape, ties=False)
    want_dx = R.expansion32_backward(dy, want_arg, shape, h, pool)
    y, arg, dx = _kernels(x, h, pool, dy)
    assert y.shape == want_y.shape
    assert np.array_equal(R.canonical_bits(y), R.canonical_bits(want_y)), "forward"
    if pool == "MAX":
        assert np.array_equal(arg, want_arg), "argmax"
    assert np.array_equal(R.canonical_bits(dx), R.canonical_bits(want_dx)), "backward"
    y2, arg2, dx2 = _kernels(x, h, pool, dy)
    assert_bits_equal(y2, y, "a second forward")
    assert_bits_equal(dx2, dx, "a second backward")
    if pool == "MAX":
        assert np.array_equal(arg2, arg)


def test_a_level_padded_past_its_kernel_is_refused(cos):
    from caffeonspark_b200 import layers
    with pytest.raises(cos.CosError, match="cos_spp_forward"):
        layers.spp_forward(torch.zeros(2, 3, 13, 13, device="cuda"), 4)


# --------------------------------------------------------------------------- the op in the engine
OP_CASES = [((2, 3, 9, 8), 3), ((3, 4, 6, 10), 3), ((2, 2, 7, 7), 1), ((2, 3, 16, 16), 4)]


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
@pytest.mark.parametrize("shape,h", OP_CASES)
def test_op_in_the_engine(cos, tmp_path, shape, h, pool):
    rng = np.random.RandomState(sum(shape))
    x = (np.round(rng.randn(*shape) * 2) / 2).astype(F32) + F32(0)  # ties; no -0, which the injectors make +0
    y, arg = R.expansion32(x, h, pool)
    body = f'layer {{ name: "s" type: "SPP" bottom: "x0" top: "y" spp_param {{ pyramid_height: {h} pool: {pool} }} }}\n'
    results = []
    for k in range(2):
        (tmp_path / str(k)).mkdir()
        r = _engine(cos, tmp_path / str(k), [x], body, (), y.shape, np.zeros(y.shape, F32))
        _harness_equal(r["d"], y, "y")  # B = 0: the probe returns y, the top gradient
        _harness_equal(r["dx"][0], R.expansion32_backward(y, arg, shape, h, pool), "dx")
        results.append(r)
    assert_bits_equal(results[1]["d"], results[0]["d"], "two calls: y")
    assert_bits_equal(results[1]["dx"][0], results[0]["dx"][0], "two calls: dx")


# --------------------------------------------------------------------------- the fixture
SPP_LAYER = """layer {
  name: "spp"
  type: "SPP"
  bottom: "conv3"
  top: "spp"
  spp_param {
    pyramid_height: 3
    pool: MAX
  }
}"""


def expansion(pool):
    """Caffe's SPP written out: Split, one Pooling and Flatten per level (spp_level's geometry on the 6 x 6 map) and
    a Concat"""
    layers = ['layer { name: "spp_split" type: "Split" bottom: "conv3" top: "s0" top: "s1" top: "s2" }']
    for lv in range(3):
        _, k, _, pad, _ = R.level(6, 6, lv)
        layers.append(f'layer {{ name: "spp_pool{lv}" type: "Pooling" bottom: "s{lv}" top: "p{lv}" pooling_param {{ '
                      f'pool: {pool} kernel_size: {k} stride: {k} pad: {pad} }} }}')
        layers.append(f'layer {{ name: "spp_flat{lv}" type: "Flatten" bottom: "p{lv}" top: "f{lv}" }}')
    layers.append('layer { name: "spp_concat" type: "Concat" bottom: "f0" bottom: "f1" bottom: "f2" top: "spp" }')
    return "\n".join(layers)


def _solver(tmp_path, extra="", batch=None, pool="MAX", expanded=False):
    text = open(os.path.join(CONFIGS, f"{NAME}_train_test.prototxt")).read()
    assert SPP_LAYER in text
    text = text.replace(SPP_LAYER, expansion(pool) if expanded else SPP_LAYER.replace("pool: MAX", f"pool: {pool}"))
    if batch is not None:
        text = text.replace(f"batch_size: {BATCH}\n", f"batch_size: {batch}\n", 1)
    text = text.replace('mean_file: "mean.binaryproto"', "")  # the batches below are staged as they are
    tag = f"{pool}_{'x' if expanded else 's'}_{batch}"
    net = tmp_path / f"{NAME}_{tag}.prototxt"
    net.write_text(text)
    s = open(os.path.join(CONFIGS, f"{NAME}_solver.prototxt")).read()
    s = s.replace(f'net: "{NAME}_train_test.prototxt"', f'net: "{net}"')
    s = s.replace(f'snapshot_prefix: "{NAME}"', f'snapshot_prefix: "{tmp_path}/snap_{tag}"')
    path = tmp_path / f"{NAME}_{tag}_solver.prototxt"
    path.write_text(s + extra)
    return str(path)


def _net_of(cos, solver, fill=True):
    net = cos.CaffeNet(solver, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=fill)
    torch.cuda.synchronize()
    return net


def batch_of(seed, n):
    """images [n, 3, 32, 32] near one of ten templates, and their labels"""
    rng = np.random.RandomState(seed)
    templates = np.random.RandomState(99).rand(10, 3, 32, 32)
    y = rng.randint(0, 10, n)
    return [(0.6 * templates[y] + 0.4 * rng.rand(n, 3, 32, 32)).astype(F32), y.astype(F32)]


def host_weights(seed):
    """Flat weights uniform in [-0.1, 0.1), drawn on the host"""
    from caffeonspark_b200 import nets
    w = np.random.RandomState(seed).uniform(-0.1, 0.1, nets.CIFAR10_QUICK_SPP_PARAM_COUNT).astype(F32)
    return w


def _engine_call(net, batch):
    net.diff().zero_()
    loss = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    assert net.forward_backward([torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in batch], loss.data_ptr())
    assert net.synchronize(), net.last_error()
    return float(loss.item()), to_host(net.diff())


@pytest.mark.parametrize("pool", ["MAX", "AVE"])
def test_fused_op_equals_the_expansion_bit_for_bit(cos, tmp_path, pool):
    w, b = host_weights(5), batch_of(5, BATCH)
    got = []
    for expanded in (False, True):
        net = _net_of(cos, _solver(tmp_path, pool=pool, expanded=expanded), fill=False)
        try:
            net.data().copy_(torch.from_numpy(w).cuda())
            got.append(_engine_call(net, b))
        finally:
            net.deallocate()
    assert np.float32(got[0][0]).view(np.uint32) == np.float32(got[1][0]).view(np.uint32), "loss"
    assert_bits_equal(got[0][1], got[1][1], "every gradient")
    # train(): the two nets filled from the same seed, every update equal
    nets_ = [_net_of(cos, _solver(tmp_path, pool=pool, expanded=e)) for e in (False, True)]
    try:
        assert_bits_equal(to_host(nets_[0].data()), to_host(nets_[1].data()), "filled weights")
        for t in range(6):
            for net in nets_:
                assert net.train(0, batch_of(300 + t, BATCH)), net.last_error()
                assert net.synchronize(), net.last_error()
            assert_bits_equal(to_host(nets_[0].data()), to_host(nets_[1].data()), f"weights after step {t + 1}")
            assert nets_[0].last_loss() == nets_[1].last_loss()
    finally:
        for net in nets_:
            net.deallocate()


def reference(w, batch, dtype, device, branches=None):
    """(loss, flat gradient, branches) of nets.cifar10_quick_spp_module on the flat weights w; branches are each
    ReLU's mask and each MAX pool's argmax (the SPP's per level, on its padded map).  With `branches` (another
    forward's), every ReLU and MAX pool takes its branch from them."""
    from caffeonspark_b200 import nets
    m = nets.cifar10_quick_spp_module().to(device=device, dtype=dtype)
    _load(m, w)
    taken = []

    def max_pool(h, k, s):
        if branches is None:
            out, i = F.max_pool2d(h, k, s, ceil_mode=True, return_indices=True)
            taken.append(i.cpu())
            return out
        i = branches[len(taken)].to(device)
        taken.append(i.cpu())
        return h.flatten(2).gather(2, i.flatten(2)).view(i.shape)

    h = torch.from_numpy(batch[0]).to(device=device, dtype=dtype)
    for layer in m:
        if isinstance(layer, torch.nn.ReLU):
            mask = (h > 0).cpu() if branches is None else branches[len(taken)]
            taken.append(mask)
            h = h * mask.to(device=device, dtype=dtype)
        elif isinstance(layer, torch.nn.MaxPool2d):
            h = max_pool(h, layer.kernel_size, layer.stride)
        elif type(layer).__name__ == "SPP":
            parts = []
            for lv in range(nets.CIFAR10_QUICK_SPP["pyramid_height"]):
                _, k, _, pad, _ = nets.spp_level(h.shape[2], h.shape[3], lv)
                parts.append(max_pool(F.pad(h, (pad, pad, pad, pad), value=float("-inf")), k, k).flatten(1))
            h = torch.cat(parts, 1)
        else:
            h = layer(h)
    loss = F.cross_entropy(h, torch.from_numpy(batch[1]).to(device).long())
    loss.backward()
    return float(loss.detach()), _grads(m), taken


def blob_errors(g, g64, counts):
    """Per blob, the largest error relative to the blob's largest float64 gradient, or to 1% of the net's largest"""
    floor = 1e-2 * np.abs(g64).max()
    off, errs = 0, []
    for c in counts:
        sl = slice(off, off + c)
        off += c
        errs.append(np.abs(g[sl].astype(np.float64) - g64[sl]).max() / max(np.abs(g64[sl]).max(), floor))
    return errs


@pytest.mark.parametrize("n", [BATCH, 37])
def test_fixture_matches_float64_and_pytorch(cos, tmp_path, n):
    net = _net_of(cos, _solver(tmp_path, batch=n), fill=False)
    try:
        w = host_weights(21 + n)
        net.data().copy_(torch.from_numpy(w).cuda())
        b = batch_of(n, n)
        l32, g = _engine_call(net, b)
        counts = net.desc.counts
    finally:
        net.deallocate()
    lt, gt, branches = reference(w, b, torch.float32, "cpu")
    _, g64t, _ = reference(w, b, torch.float64, "cpu", branches)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        branches = reference(w, b, torch.float32, "cuda")[2]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    l64, g64, _ = reference(w, b, torch.float64, "cpu", branches)
    assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
    assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
    native, torch32 = blob_errors(g, g64, counts), blob_errors(gt, g64t, counts)
    report = "; ".join(f"blob {k}: native {a:.2e}, PyTorch fp32 {b:.2e}"
                       for k, (a, b) in enumerate(zip(native, torch32)))
    print(f"b{n}: worst native {max(native):.2e}, worst PyTorch fp32 {max(torch32):.2e}")
    assert max(native + torch32) <= NET_BOUND, f"relative to max|g64| per blob: {report}"


def _train(net, steps, seed, check=None):
    losses = []
    for t in range(steps):
        if check:
            check.before()
        assert net.train(0, batch_of(seed + t, BATCH)), net.last_error()
        assert net.synchronize(), net.last_error()
        losses.append(net.last_loss())
        if check:
            check.after(t)
    return np.array(losses)


def test_fixture_trains_through_train_alone(cos, oracle, tmp_path):
    from caffeonspark_b200 import nets
    net = _net_of(cos, _solver(tmp_path))
    try:
        assert net.param_count() == nets.CIFAR10_QUICK_SPP_PARAM_COUNT
        losses = _train(net, 80, 1000, _UpdateCheck(net, oracle))
        assert np.isfinite(losses).all()
        assert losses[-20:].mean() < losses[:10].mean(), losses
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
                assert netz[r].train(0, batch_of(10 * r + t, BATCH)), netz[r].last_error()
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
def test_snapshots_resume_bit_exact(cos, tmp_path, fmt):
    solver = _solver(tmp_path, f"snapshot_format: {fmt}\n")
    a = _net_of(cos, solver)
    try:
        _train(a, 3, 1)
        assert a.snapshot() == 3, a.last_error()
        model, state = a.snapshotFilename(3, False), a.snapshotFilename(3, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        assert_bits_equal(cos.read_caffemodel_blob(model, "ip1", 1).ravel(), w_a[165344:165344 + 64], "ip1 bias")
        b = cos.CaffeNet(solver, model, state, 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
        try:
            assert b.connect(b.localAddresses())
            b.use_native_producer(fill_weights=True)  # a restored model is not refilled
            assert b.iter() == 3
            assert_bits_equal(to_host(b.data()), w_a, "resumed data")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            la, lb = _train(a, 2, 7), _train(b, 2, 7)
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "two more steps after resume")
            assert np.array_equal(la, lb)
        finally:
            b.deallocate()
    finally:
        a.deallocate()
