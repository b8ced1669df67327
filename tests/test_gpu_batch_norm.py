"""-m gpu: the native BatchNorm kernels against a restatement of batch_norm_layer.cpp, and BatchNorm nets through the
sync library: statistics that follow their shard owner, snapshots, and train() with the fp32 and bf16 producers."""
import ctypes
import ctypes.util

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import Ranks, assert_bits_equal, to_host
from test_batch_norm_host import numpy_bn_backward, numpy_bn_forward
from test_caffe_proto_io import pb  # noqa: F401  (fixture: caffe.proto subset on the real protobuf runtime)
from test_hdf5_io import MiniH5

pytestmark = pytest.mark.gpu

EPS, FRAC = 1e-5, 0.999
# the example net's three BN inputs at batch 100, then ragged ones
SHAPES = [(100, 32, 16, 16), (100, 32, 16, 16), (100, 64, 8, 8), (1, 5, 3, 3), (7, 1, 9, 11), (3, 6, 1, 1),
          (5, 3, 7, 7), (2, 3, 37, 41), (1, 1, 1, 1)]
SHAPES = list(dict.fromkeys(SHAPES))

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype = ctypes.c_float
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]


def c_powf_half(v):
    return np.array([_libm.powf(float(a), 0.5) for a in np.asarray(v, np.float32)], np.float32)


def f32(v):
    return np.asarray(v, np.float32)


def restate_forward(x, mean, var, blobs, global_stats):
    """Caffe's fp32 operation order from the saved statistics: y and the updated blobs, each operation rounded
    once (numpy float32 scalar-vector operations round like the kernel's __f*_rn)."""
    c = x.shape[1]
    sd = c_powf_half(f32(var) + f32(EPS))
    y = (f32(x).reshape(x.shape[0], c, -1) - f32(mean)[None, :, None]) / sd[None, :, None]
    if global_stats:
        return y.reshape(x.shape), blobs
    mb, vb, s = (f32(b) for b in blobs)
    m = x.size // c
    corr = np.float32(m) / np.float32(m - 1) if m > 1 else np.float32(1)
    f = np.float32(FRAC)
    return y.reshape(x.shape), (f32(mean) + f * mb, corr * f32(var) + f * vb, s * f + np.float32(1))


def restate_backward(x, dy, mean, var, global_stats):
    n, c = x.shape[0], x.shape[1]
    sd = c_powf_half(f32(var) + f32(EPS))[None, :, None]
    g = f32(dy).reshape(n, c, -1)
    if global_stats:
        return (g / sd).reshape(x.shape)
    xh = (f32(x).reshape(n, c, -1) - f32(mean)[None, :, None]) / sd
    s1 = g.astype(np.float64).sum((0, 2)).astype(np.float32)[None, :, None]
    s2 = (xh * g).astype(np.float64).sum((0, 2)).astype(np.float32)[None, :, None]
    k = np.float32(-1.0 / (x.size // c))
    return ((g + k * (s1 + xh * s2)) / sd).reshape(x.shape), s1, s2


def run_native(x, blobs, global_stats, dy=None, dtype=torch.float32):
    """-> (y, save, blobs', dx) from the C entry points through layers.BatchNormFunction"""
    from caffeonspark_b200 import layers
    c = x.shape[1]
    mean, var, s = (torch.from_numpy(f32(b).reshape(-1).copy()).cuda() for b in blobs)
    xt = torch.from_numpy(x).cuda().to(dtype).requires_grad_(True)
    y = layers.BatchNormFunction.apply(xt, mean, var, s, global_stats, FRAC, EPS)
    save = y.grad_fn.saved_tensors[1].clone()
    dx = None
    if dy is not None:
        y.backward(torch.from_numpy(dy).cuda().to(dtype))
        dx = xt.grad
    torch.cuda.synchronize()
    return y, save, (mean.cpu().numpy(), var.cpu().numpy(), s.cpu().numpy()), dx


def _inputs(shape, seed):
    rng = np.random.RandomState(seed)
    x = (rng.randn(*shape) * 1.5 + 2.0).astype(np.float32)  # an offset keeps the mean away from 0
    dy = rng.randn(*shape).astype(np.float32)
    c = shape[1]
    blobs = (rng.rand(c).astype(np.float32) * 10, rng.rand(c).astype(np.float32) * 10 + 1, np.float32([7.25]))
    return x, dy, blobs


@pytest.mark.parametrize("shape", SHAPES)
def test_training_forward_backward_match_the_restatement(cos, shape):
    x, dy, blobs = _inputs(shape, sum(shape))
    y, save, nb, dx = run_native(x, blobs, False, dy)
    save = save.cpu().numpy()
    c = shape[1]
    mean, var = save[:c], save[c:]
    _, wmean, wvar, _ = numpy_bn_forward(x, blobs[0].astype(np.float64), blobs[1].astype(np.float64),
                                         float(blobs[2][0]))
    np.testing.assert_allclose(mean, wmean, rtol=1e-6)
    np.testing.assert_allclose(var, wvar, rtol=1e-6, atol=1e-12)
    wy, wblobs = restate_forward(x, mean, var, blobs, False)
    assert_bits_equal(y.detach().cpu().numpy(), wy, f"{shape}: y")
    for k, what in enumerate(("mean blob", "variance blob", "scale factor")):
        assert_bits_equal(nb[k], wblobs[k], f"{shape}: {what}")
    wdx64 = numpy_bn_backward(x, dy, mean.astype(np.float64), var.astype(np.float64))
    # dx: the two channel sums are fp32 partial sums; relative to the scale of dy / std
    scale = np.abs(wdx64).max() + 1e-30
    np.testing.assert_allclose(dx.cpu().numpy(), wdx64, rtol=0, atol=2e-5 * scale)
    wdx, _, _ = restate_backward(x, dy, mean, var, False)
    np.testing.assert_allclose(dx.cpu().numpy(), wdx, rtol=0, atol=2e-6 * scale)


@pytest.mark.parametrize("shape", SHAPES[:4])
def test_global_stats_forward_backward_and_untouched_blobs(cos, shape):
    x, dy, blobs = _inputs(shape, 3 + sum(shape))
    for s in (blobs[2], np.float32([0.0])):
        b = (blobs[0], blobs[1], s)
        y, save, nb, dx = run_native(x, b, True, dy)
        for k in range(3):
            assert_bits_equal(nb[k], b[k], f"{shape}: blob {k} untouched")
        sf = np.float32(0) if s[0] == 0 else np.float32(1) / s[0]
        mean, var = sf * f32(b[0]), sf * f32(b[1])
        c = shape[1]
        assert_bits_equal(save.cpu().numpy(), np.concatenate([mean, var]), f"{shape}: global statistics")
        wy, _ = restate_forward(x, mean, var, b, True)
        assert_bits_equal(y.detach().cpu().numpy(), wy, f"{shape}: y (global)")
        assert_bits_equal(dx.cpu().numpy(), restate_backward(x, dy, mean, var, True), f"{shape}: dx (global)")
        assert c == save.numel() // 2


@pytest.mark.parametrize("global_stats", [False, True])
@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[2], (5, 3, 7, 7), (3, 6, 1, 1)])
def test_bf16_is_the_fp32_kernel_on_upcast_inputs_rounded_once(cos, shape, global_stats):
    x, dy, blobs = _inputs(shape, 11 + sum(shape))
    xb = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    dyb = torch.from_numpy(dy).to(torch.bfloat16).float().numpy()
    y32, s32, b32, dx32 = run_native(xb, blobs, global_stats, dyb)
    y16, s16, b16, dx16 = run_native(xb, blobs, global_stats, dyb, dtype=torch.bfloat16)
    assert y16.dtype == torch.bfloat16 and dx16.dtype == torch.bfloat16
    assert torch.equal(y16.detach().view(torch.int16), y32.detach().to(torch.bfloat16).view(torch.int16))
    assert torch.equal(dx16.view(torch.int16), dx32.to(torch.bfloat16).view(torch.int16))
    assert_bits_equal(s16.cpu().numpy(), s32.cpu().numpy(), "save")
    for k in range(3):
        assert_bits_equal(b16[k], b32[k], f"blob {k}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(64, 32, 33, 31), (16, 8, 48, 48)], ids=["warp_per_plane", "block_per_plane"])
def test_run_to_run_and_graph_replay_are_bitwise_identical(cos, shape, dtype):
    """Forward and backward, eagerly three times and replayed from one captured graph twice: y, dx and the
    blobs are bitwise identical.  H*W = 1023 takes the warp-per-plane reduction, 2304 the block-per-plane one."""
    from caffeonspark_b200 import layers
    x, dy, blobs = _inputs(shape, 5)
    xt = torch.from_numpy(x).cuda().to(dtype).requires_grad_(True)
    dyt = torch.from_numpy(dy).cuda().to(dtype)
    stats = [torch.from_numpy(f32(b).reshape(-1).copy()).cuda() for b in blobs]

    def reset():
        for t, b in zip(stats, blobs):
            t.copy_(torch.from_numpy(f32(b).reshape(-1)))

    def step(xin):
        y = layers.BatchNormFunction.apply(xin, *stats, False, FRAC, EPS)
        (dx,) = torch.autograd.grad(y, xin, dyt)  # no AccumulateGrad node: capturable on any stream
        return y, dx

    bits = lambda t: t.detach().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).clone()  # noqa
    reset()
    y, dx = step(xt)
    ref = (bits(y), bits(dx), [t.clone() for t in stats])
    for _ in range(3):
        reset()
        y, dx = step(xt)
        assert torch.equal(bits(y), ref[0]) and torch.equal(bits(dx), ref[1])
        assert all(torch.equal(a, b) for a, b in zip(stats, ref[2]))
    del y, dx
    xg = xt.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        reset()
        step(xg)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y, dx = step(xg)
    for _ in range(2):
        reset()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(y), ref[0]), "y under replay"
        assert torch.equal(bits(dx), ref[1]), "dx under replay"
        assert all(torch.equal(a, b) for a, b in zip(stats, ref[2])), "blobs under replay"


@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[2], (5, 3, 7, 7)])
def test_against_pytorch_batch_norm(cos, shape):
    x, dy, blobs = _inputs(shape, 17 + sum(shape))
    y, _, _, dx = run_native(x, blobs, False, dy)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    ry = F.batch_norm(xt, None, None, training=True, eps=EPS)
    ry.backward(torch.from_numpy(dy).cuda())
    torch.testing.assert_close(y.detach(), ry.detach(), rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(dx, xt.grad, rtol=1e-4, atol=2e-5)


# ------------------------------------------------------------------ statistics follow their shard owner

def _bn_slots(counts, lr_mult):
    """flat indices of the blobs with lr_mult 0 (the BN statistics)"""
    off, out = 0, []
    for n, lm in zip(counts, lr_mult):
        if lm == 0.0:
            out.append(np.arange(off, off + n))
        off += n
    return np.concatenate(out)


@pytest.mark.parametrize("N", [2, 3])
@pytest.mark.parametrize("wire", ["fp32", "bf16"])
def test_statistics_follow_their_shard_owner(cos, oracle, N, wire):
    from caffeonspark_b200 import nets
    desc = nets.solver_desc("cifar10_full_bn", grad_dtype=wire)
    slots = _bn_slots(desc.counts, desc.lr_mult)
    sim = oracle.Simulation(N, desc.counts, desc.lr_mult, desc.decay_mult, seed=9, bf16=wire == "bf16",
                            **desc.hyper())
    R = Ranks(cos, desc, N)
    try:
        R.set_weights(sim.data)
        R.connect()
        # each rank's forward pass wrote its own batch statistics into data_
        rng = np.random.RandomState(N)
        post_forward = []
        for r in range(N):
            w = sim.data[r]
            w[slots] = rng.rand(slots.size).astype(np.float32) + r
            post_forward.append(w.copy())
        R.set_weights(post_forward)
        grads = []
        for r in range(N):
            g = sim.gradient(r, 0)
            g[slots] = 0.0  # Caffe's BN diff stays zero
            grads.append(g)
        sim.step(grads)
        R.step(grads)
        want = sim.consistent_weights()
        P = sim.P
        owner = np.empty(P, np.int64)
        for q in range(N):
            o, s = oracle.chunk(P, N, q)
            owner[o:o + s] = q
        for r in range(N):
            w = R.weights(r)
            assert_bits_equal(w, want, f"rank {r} weights")
            o, s = oracle.chunk(P, N, r)
            assert_bits_equal(R.history(r)[o:o + s], sim.own(r)[1], f"rank {r} own history")
            assert_bits_equal(w[slots], np.array([post_forward[owner[i]][i] for i in slots], np.float32),
                              f"rank {r}: BN statistics = owner's post-forward values")
        assert len(set(owner[slots])) >= 2  # the statistics lie in more than one rank's shard
    finally:
        R.close()


@pytest.fixture(scope="module")
def solver_oracles(oracle):
    from oracle import accum, adam
    for m in (accum, adam):
        m.build()
        m.lib()
    return accum, adam


# (N, solver, iter_size, gradient wire)
PRODUCER_CASES = [(2, "SGD", 2, "fp32"), (3, "SGD", 2, "bf16"), (2, "Adam", 1, "fp32"), (3, "Adam", 1, "bf16")]


@pytest.mark.parametrize("N,solver,k,wire", PRODUCER_CASES,
                         ids=[f"N{n}-{sv}-iter_size{k}-{w}" for n, sv, k, w in PRODUCER_CASES])
def test_native_forward_statistics_follow_their_owner_through_a_step(cos, oracle, solver_oracles, N, solver, k,
                                                                      wire):
    """Every rank runs the real producer (native BatchNorm forward, backward) on its own batches, k passes, then
    one fused step.  The forward passes have written the statistics into data_ before the sync launch, and the step
    leaves every rank holding, in each BN slot, its owner's post-forward value; with lr_mult 0 neither SGD nor
    Adam changes them.  Conv/ip weights and the history (m, and v for Adam) equal the oracle fed the ranks' data_
    and diff_."""
    from caffeonspark_b200 import harness, layers, nets
    accum, adam = solver_oracles
    desc = nets.solver_desc("cifar10_full_bn", grad_dtype=wire, iter_size=k, type=solver)
    slots = _bn_slots(desc.counts, desc.lr_mult)
    counts = desc.counts
    off = np.cumsum([0] + counts)
    R = Ranks(cos, desc, N)
    try:
        prods = [harness.TorchProducer(net, nets.torch_module("cifar10_full_bn"), seed=1234, use_graph=False)
                 for net in R.nets]
        R.connect()
        seen = [[] for _ in range(N)]  # bn1's input, per rank and pass
        for r, p in enumerate(prods):
            bn1 = p.module[2]
            assert isinstance(bn1, layers.BatchNorm)
            bn1.register_forward_hook(lambda m, inp, out, r=r: seen[r].append(inp[0].detach().double().cpu()))
        g = torch.Generator().manual_seed(100 + N)
        for q in range(k):
            for r, p in enumerate(prods):  # a different batch on every rank and pass
                x = (torch.rand(100, 3, 32, 32, generator=g) * (1 + r)).cuda()
                y = torch.randint(0, 10, (100,), generator=g).cuda()
                p.forward_backward(x, y)
        torch.cuda.synchronize()
        post = [R.weights(r) for r in range(N)]
        grads = [R.diff(r) for r in range(N)]
        assert all(not g_[slots].any() for g_ in grads)  # no gradient reaches the statistics
        # the statistics on each rank are its own forward passes' (Caffe's moving average over k passes)
        s = np.float32(0)
        for _ in range(k):
            s = np.float32(np.float32(s * np.float32(FRAC)) + np.float32(1))
        for r in range(N):
            for b in (3, 7, 11):  # bn1..bn3 scale factors
                assert_bits_equal(post[r][off[b]:off[b + 1]], [s], f"rank {r}: scale factor after {k} passes")
            want = np.zeros(32)
            for xin in seen[r]:
                want = xin.mean((0, 2, 3)).numpy() + FRAC * want
            np.testing.assert_allclose(post[r][off[1]:off[2]], want, rtol=1e-5, atol=1e-6)
        assert not np.array_equal(post[0][slots], post[1][slots])
        # the oracle: each rank's post-forward data_ and its diff_ (bf16-rounded where the wire is bf16)
        wire_grads = [oracle.round_bf16(g_) for g_ in grads] if wire == "bf16" else grads
        hp = desc.hyper()
        if solver == "Adam":
            sim = adam.AdamSimulation(N, counts, desc.lr_mult, desc.decay_mult, seed=1, **hp)
            sim.data = [w.copy() for w in post]
            sim.step(wire_grads)
        else:
            sim = accum.AccumSimulation(N, counts, desc.lr_mult, desc.decay_mult, seed=1, **hp)
            sim.data = [w.copy() for w in post]
            sim.step_accumulated(wire_grads)
        for net in R.nets:
            assert net.sync_step(0), net.last_error()
        for net in R.nets:
            assert net.synchronize(), net.last_error()
        P = sim.P
        owner = np.empty(P, np.int64)
        for q in range(N):
            o, sz = oracle.chunk(P, N, q)
            owner[o:o + sz] = q
        want_stats = np.array([post[owner[i]][i] for i in slots], np.float32)
        for r in range(N):
            w = R.weights(r)
            assert_bits_equal(w, sim.consistent_weights(), f"rank {r} weights")
            assert_bits_equal(w[slots], want_stats, f"rank {r}: BN statistics = owner's post-forward values")
            o, sz = oracle.chunk(P, N, r)
            h = R.history(r)
            assert_bits_equal(h[o:o + sz], sim.hist[r][o:o + sz], f"rank {r} own history (m)")
            if solver == "Adam":
                assert_bits_equal(h[P + o:P + o + sz], sim.hist[r][P + o:P + o + sz], f"rank {r} own v")
            assert not R.diff(r).any()
    finally:
        R.close()


# ------------------------------------------------------------------ snapshot / resume with a real bn1 layer

@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshot_writes_bn_layers_and_resumes_bit_exact(cos, pb, tmp_path, fmt):  # noqa: F811
    from caffeonspark_b200 import harness, nets
    solver = nets.write_prototxts("cifar10_full_bn", str(tmp_path))
    text = open(solver).read().replace('snapshot_prefix: "cifar10_full_sigmoid_bn"',
                                       f'snapshot_prefix: "{tmp_path}/snap"') + f"snapshot_format: {fmt}\n"
    open(solver, "w").write(text)
    rng = np.random.RandomState(2)
    x = torch.from_numpy(rng.rand(100, 3, 32, 32).astype(np.float32)).pin_memory()
    y = torch.from_numpy(rng.randint(0, 10, (100,)).astype(np.float32)).pin_memory()
    a = cos.CaffeNet(solver)
    try:
        assert a.connect(a.localAddresses())
        harness.make_producer("cifar10_full_bn", a, seed=4, use_graph=False)
        for _ in range(2):
            assert a.train(0, [x, y]), a.last_error()
        assert a.synchronize()
        assert a.snapshot() == 2, a.last_error()
        model, state = a.snapshotFilename(2, False), a.snapshotFilename(2, True)
        w_a, h_a = to_host(a.data()), to_host(a.history())
        counts, _, _, _ = nets.layout("cifar10_full_bn")
        off = np.cumsum([0] + counts)
        assert w_a[off[1]:off[4]].any() and w_a[off[3]] == pytest.approx(1 + FRAC)  # bn1 written by 2 forwards
        if fmt == "BINARYPROTO":  # parsed by the real protobuf runtime
            net = pb["NetParameter"]()
            net.ParseFromString(open(model, "rb").read())
            got = {l.name: l for l in net.layer}
            for name, c in (("bn1", 32), ("bn2", 32), ("bn3", 64)):
                assert got[name].type == "BatchNorm" and len(got[name].blobs) == 3
                assert [list(b.shape.dim) for b in got[name].blobs] == [[c], [c], [1]]
            blobs = [np.asarray(b.data, np.float32) for b in got["bn1"].blobs]
        else:  # parsed by the independent HDF5 reader of test_hdf5_io
            mini = MiniH5(model)
            # an HDF5 group lists its links in name order
            assert mini.objects["/data"]["links"] == sorted(["conv1", "bn1", "conv2", "bn2", "conv3", "bn3", "ip1"])
            for name, c in (("bn1", 32), ("bn2", 32), ("bn3", 64)):
                assert [mini.objects[f"/data/{name}/{j}"]["shape"] for j in range(3)] == [[c], [c], [1]]
                assert f"/data/{name}/3" not in mini.objects
            blobs = [np.frombuffer(mini.objects[f"/data/bn1/{j}"]["data"], np.float32) for j in range(3)]
        for j in range(3):
            assert_bits_equal(blobs[j], w_a[off[1 + j]:off[2 + j]], f"bn1 blob {j} in the snapshot")
        b = cos.CaffeNet(solver, model, state)
        try:
            assert b.connect(b.localAddresses())
            assert b.iter() == 2
            assert_bits_equal(to_host(b.data()), w_a, "resumed data (statistics included)")
            assert_bits_equal(to_host(b.history()), h_a, "resumed history")
            g = np.random.RandomState(3).randn(w_a.size).astype(np.float32) * 1e-2
            for n in (a, b):
                n.diff().copy_(torch.from_numpy(g).cuda())
                torch.cuda.synchronize()
                assert n.sync_step(0), n.last_error()
                assert n.synchronize()
            assert_bits_equal(to_host(b.data()), to_host(a.data()), "one more step after resume")
        finally:
            b.deallocate()
    finally:
        a.deallocate()


# ------------------------------------------------------------------ train() end to end

# The final 50-step window loss on the synthetic task of test_bf16_producer_converges_like_fp32.  With the reference
# solver (base_lr 0.001, no weight decay) and sigmoid activations the net learns slowly: a measured run on one H100
# went from 2.436 at the first step to 2.017 (fp32) and 2.017 (bf16) in the final window (DESIGN.md section 13).
# The threshold sits below chance (ln 10 = 2.303) with room for the run-to-run spread of cuDNN's algorithms.
BN_STEPS, BN_WINDOW = 300, 50
BN_MAX_LOSS = 2.15


def _train_bn(cos, precision):
    from caffeonspark_b200 import harness, nets
    from test_gpu_bf16_producer import _task_batches
    net = cos.CaffeNet(nets.solver_desc("cifar10_full_bn"))
    try:
        assert net.connect(net.localAddresses())
        prod = harness.make_producer("cifar10_full_bn", net, seed=1234, precision=precision)
        xh, yh = torch.empty(100, 3, 32, 32).pin_memory(), torch.empty(100).pin_memory()
        losses = []
        for x, y in _task_batches(steps=BN_STEPS):
            xh.copy_(x)
            yh.copy_(y)
            assert net.train(0, [xh, yh]), net.last_error()
            assert net.synchronize(), net.last_error()
            losses.append(net.last_loss())
        assert prod.use_graph and any(st["graph"] is not None for st in prod._graphs.values())
        assert not to_host(net.diff()).any()
        bn = prod.module[2]
        assert float(bn.scale_factor) == pytest.approx((1 - FRAC ** BN_STEPS) / (1 - FRAC), rel=1e-4)
        return np.array(losses)
    finally:
        net.deallocate()


def test_cifar10_full_bn_trains_through_train_fp32_and_bf16(cos):
    fp32, bf16 = _train_bn(cos, "fp32"), _train_bn(cos, "bf16")
    assert np.isfinite(fp32).all() and np.isfinite(bf16).all()
    f, b = fp32[-BN_WINDOW:].mean(), bf16[-BN_WINDOW:].mean()
    print(f"cifar10_full_bn final-window loss over the last {BN_WINDOW} of {BN_STEPS} steps: fp32 {f:.4f}, "
          f"bf16 {b:.4f}; first step {fp32[0]:.4f} / {bf16[0]:.4f}")
    assert f < BN_MAX_LOSS and b < BN_MAX_LOSS, (f, b)
    assert fp32[0] - f > 0.2 and bf16[0] - b > 0.2
