"""-m gpu: iter_size > 1 (gradient accumulation), bit-exact against the oracle's step (oracle/accum_oracle.c:
passes add up in diff_, scale + reduce-scatter, Normalize g = (1/iter_size) * g, then the SGD or Adam update)."""
import numpy as np
import pytest
import torch

from gpu_util import Ranks, assert_bits_equal, to_dev, to_host

pytestmark = pytest.mark.gpu

SGD = dict(lr_policy="inv", base_lr=0.01, gamma=0.0001, power=0.75, momentum=0.9, weight_decay=0.0005)
ADAM = dict(lr_policy="fixed", base_lr=0.001, momentum=0.9, weight_decay=0.0005, type="Adam", momentum2=0.999,
            delta=1e-8)
LAYOUTS = {
    "lenet": ([500, 20, 25000, 50, 400000, 500, 5000, 10], [1, 2] * 4, [1, 0] * 4),
    "ragged_tiny_blobs": ([3, 1, 2, 5, 1, 1, 7, 1021, 2, 1], [1, 2, 1, 2, 1, 2, 1, 0, 1, 2],
                          [1, 0, 1, 0, 1, 0, 1, 1, 0, 1]),
    "not_multiple_of_4": ([4099], [1], [1]),
}
MULTI = ([5000, 20, 2500, 50, 7, 1021], [1, 2, 1, 2, 0, 2], [1, 0, 1, 0, 1, 1])


@pytest.fixture(scope="module")
def accum(oracle):
    from oracle import accum as A
    A.build()
    A.lib()
    return A


def _sim(accum, N, counts, lm, dm, hp, k, seed, reg="L2"):
    kw = {key: v for key, v in hp.items() if key != "type"}
    return accum.AccumSimulation(N, counts, lm, dm, iter_size=k, solver_type=hp.get("type", "SGD"), seed=seed,
                                 regularization_type=reg, **kw)


def _step(accum, oracle, sim, R, t, bf16):
    """Pass gradients of step t on every rank: the device gets their fp32 sum in diff_ (what k producer calls
    leave there), the oracle the same sum (bf16-rounded where the kernel reads a bf16 wire)."""
    per_pass = [[sim.pass_gradient(r, t, q) for r in range(sim.N)] for q in range(sim.iter_size)]
    acc = accum.accumulate(per_pass)
    sim.step_accumulated([oracle.round_bf16(a) for a in acc] if bf16 else acc)
    R.step(acc)


def _check(cos, oracle, accum, N, counts, lm, dm, hp, k, steps=3, bf16=False, reg="L2", seed=7, **opts):
    desc = cos.SolverDesc(counts, lm, dm, grad_dtype="bf16" if bf16 else "fp32", iter_size=k,
                          regularization_type=reg, **hp)
    sim = _sim(accum, N, counts, lm, dm, hp, k, seed, reg)
    R = Ranks(cos, desc, N, **opts)
    try:
        R.set_weights(sim.data)
        R.connect()
        rk = R.nets[0].get_option("resolved_kernel")
        mode = R.nets[0].get_option("resolved_algo")
        P = sim.P
        adam = hp.get("type") == "Adam"
        for t in range(steps):
            _step(accum, oracle, sim, R, t, bf16)
            for r in range(N):
                assert R.nets[r].iter() == t + 1
                assert_bits_equal(R.weights(r), sim.consistent_weights() if N > 1 else sim.data[0],
                                  f"N={N} k={k} weights step {t} rank {r}")
                o, s = (0, P) if N == 1 or mode == 2 else cos.chunk(P, N, r)  # one-shot: every rank holds all
                h = R.history(r)
                ref = sim.hist[0] if N == 1 else None
                cm = sim.consistent_history()[:P] if ref is None else ref[:P]
                assert_bits_equal(h[o:o + s], cm[o:o + s], f"N={N} k={k} history step {t} rank {r}")
                if adam:
                    cv = sim.consistent_v() if ref is None else ref[P:]
                    assert_bits_equal(h[P + o:P + o + s], cv[o:o + s], f"N={N} k={k} v step {t} rank {r}")
                assert not R.diff(r).any()
        return rk
    finally:
        R.close()


@pytest.mark.parametrize("name", sorted(LAYOUTS))
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
@pytest.mark.parametrize("bf16", [False, True])
def test_local_ldg_bit_exact(cos, oracle, accum, name, solver, bf16):
    counts, lm, dm = LAYOUTS[name]
    for k in (2, 3):
        assert _check(cos, oracle, accum, 1, counts, lm, dm, SGD if solver == "SGD" else ADAM, k, bf16=bf16,
                      kernel=0) == 0


@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_full_size_caffenet(cos, oracle, accum, solver):
    from caffeonspark_b200 import nets
    d = nets.solver_desc("caffenet")
    hp = dict(lr_policy=d.lr_policy, base_lr=d.base_lr, gamma=d.gamma, stepsize=d.stepsize, momentum=d.momentum,
              weight_decay=d.weight_decay)
    if solver == "Adam":
        hp.update(type="Adam", momentum2=0.999, delta=1e-8)
    _check(cos, oracle, accum, 1, d.counts, d.lr_mult, d.decay_mult, hp, 4, steps=2)


def test_local_tma_sgd_bit_exact(cos, oracle, accum):
    counts, lm, dm = LAYOUTS["lenet"]
    for k in (2, 5):
        assert _check(cos, oracle, accum, 1, counts, lm, dm, SGD, k, kernel=1) == 1


@pytest.mark.parametrize("N", [2, 3, 4])
@pytest.mark.parametrize("kernel", [-1, 0, 1, 2, 4], ids=["auto", "ldg", "tma", "push", "ll"])
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_multi_rank_two_shot_bit_exact(cos, oracle, accum, N, kernel, solver):
    if solver == "Adam" and kernel == 1:
        pytest.skip("the TMA kernel implements SGD only (forcing it on an Adam net is refused)")
    counts, lm, dm = MULTI
    rk = _check(cos, oracle, accum, N, counts, lm, dm, SGD if solver == "SGD" else ADAM, 3, algo=1, kernel=kernel)
    if kernel >= 0:
        assert rk == kernel


@pytest.mark.parametrize("solver", ["SGD", "Adam"])
@pytest.mark.parametrize("kernel", [0, 2, 4], ids=["ldg", "push", "ll"])
def test_multi_rank_bf16_wire_and_l1(cos, oracle, accum, solver, kernel):
    counts, lm, dm = MULTI
    hp = SGD if solver == "SGD" else ADAM
    _check(cos, oracle, accum, 2, counts, lm, dm, hp, 2, bf16=True, algo=1, kernel=kernel)
    _check(cos, oracle, accum, 3, counts, lm, dm, hp, 7, reg="L1", algo=1, kernel=kernel)


@pytest.mark.parametrize("N", [2, 3])
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_multi_rank_one_shot_bit_exact(cos, oracle, accum, N, solver):
    counts, lm, dm = MULTI
    _check(cos, oracle, accum, N, counts, lm, dm, SGD if solver == "SGD" else ADAM, 3, algo=2, kernel=0)
    if solver == "SGD":
        _check(cos, oracle, accum, N, counts, lm, dm, SGD, 3, algo=2, kernel=1)


def test_kernel_choice_does_not_depend_on_iter_size(cos):
    """AUTO resolves the same kernel for k = 1 and k > 1 (64 MB: TMA for SGD; 4 KB: LL)."""
    for counts, opts in (([16 << 20], dict(push_max_bytes=1 << 20)), ([1000], {})):
        for solver in ("SGD", "Adam"):
            got = []
            for k in (1, 3):
                hp = dict(SGD if solver == "SGD" else ADAM)
                R = Ranks(cos, cos.SolverDesc(counts, iter_size=k, **hp), 2, **opts)
                try:
                    got.append([(R.nets[0].set_option("algo", a), R.nets[0].get_option("resolved_kernel"))[1]
                                for a in (0, 1, 2)])
                finally:
                    R.close()
            assert got[0] == got[1], (counts, solver, got)


def test_nvls_to_tolerance(cos, oracle, accum):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("NVLS needs a multicast team over at least two GPUs")
    N = 2
    counts, lm, dm = MULTI
    desc = cos.SolverDesc(counts, lm, dm, iter_size=3, **SGD)
    sim = _sim(accum, N, counts, lm, dm, SGD, 3, 5)
    R = Ranks(cos, desc, N, devices=list(range(N)), algo=1, nvls=1, kernel=3)
    try:
        R.set_weights(sim.data)
        R.connect()
        if R.nets[0].get_option("nvls_active") != 1:
            pytest.skip("no multicast team on this system")
        assert R.nets[0].get_option("resolved_kernel") == 3
        for t in range(3):
            _step(accum, oracle, sim, R, t, False)
            for r in range(N):  # the switch chooses the summation order: 1e-5, not bit equality
                np.testing.assert_allclose(R.weights(r), sim.consistent_weights(), rtol=1e-5, atol=1e-8)
                assert not R.diff(r).any()
    finally:
        R.close()


def test_zeroed_descriptor_field_is_iter_size_one(cos, oracle):
    """A descriptor whose iter_size is 0 (built before the field existed) runs the iter_size 1 step."""
    counts, lm, dm = LAYOUTS["lenet"]
    desc = cos.SolverDesc(counts, lm, dm, **SGD)
    d, keep = desc.to_c()
    d.iter_size = 0
    sim = oracle.Simulation(1, counts, lm, dm, seed=3, **SGD)
    import ctypes
    from caffeonspark_b200 import _lib
    h = ctypes.c_void_p()
    L = _lib.lib()
    assert L.cos_net_allocate_desc(ctypes.byref(d), 1, 1, 0, 1, 0, -1, ctypes.byref(h)) == 1
    net = cos.CaffeNet.__new__(cos.CaffeNet)
    net._L, net._h, net._fb_keep, net.desc = L, h, None, desc
    net.cluster_size, net.node_rank, net.num_local_devices = 1, 0, 1
    try:
        assert net.connect(net.localAddresses())
        to_dev(net.data(), sim.data[0])
        for t in range(2):
            g = sim.gradient(0, t)
            sim.step([g])
            to_dev(net.diff(), g)
            torch.cuda.synchronize()
            assert net.sync_step(0) and net.synchronize(), net.last_error()
        assert_bits_equal(to_host(net.data()), sim.data[0], "weights")
    finally:
        net.deallocate()


# ------------------------------------------------------------ train() / train_accumulate() with a producer

class _SyntheticProducer:
    """Adds a known gradient per pass into diff_ and writes a known loss; records what each call saw."""

    def __init__(self, net, P, seed=9, local=1):
        from oracle import oracle as O
        self.net, self.P, self.seed, self.O = net, P, seed, O
        self.calls = []
        self.step = 0
        self.dev = [torch.device(f"cuda:{net.deviceID(i)}") for i in range(local)]
        net.set_forward_backward(self)

    def grad(self, t, q, rank=0):
        return self.O.fill(self.P, self.seed, (t + 1) * 4096 + 256 * q + rank, 0.01)

    def loss(self, t, q):
        return np.float32(1.0 + 0.37 * q + 0.001 * t + 1.0 / 3.0 * ((q * 7 + t) % 5))

    def __call__(self, solver_index, blobs, loss_dev, stream):
        from caffeonspark_b200.caffenet import _DevArray
        t, i = self.step, solver_index
        q = sum(1 for c in self.calls if c[0] == t and c[4] == i)
        self.calls.append((t, q, blobs[0][0], loss_dev, i))
        dev = self.dev[i]
        ext = torch.cuda.ExternalStream(stream, device=dev)
        with torch.cuda.device(dev), torch.cuda.stream(ext):
            diff = self.net.diff(i)
            diff.add_(torch.from_numpy(self.grad(t, q, self.net.global_rank(i))).to(dev, non_blocking=False))
            torch.as_tensor(_DevArray(loss_dev, 1), device=dev).fill_(float(self.loss(t, q)))
        return 0


def _batch(v, n=4):
    return [np.full((n, 1, 2, 2), v, np.float32), np.zeros(n, np.float32)]


@pytest.mark.parametrize("pipeline", [1, 0])
def test_train_calls_producer_k_times_on_the_same_batch(cos, oracle, accum, pipeline):
    counts, lm, dm = LAYOUTS["ragged_tiny_blobs"]
    k = 3
    net = cos.CaffeNet(cos.SolverDesc(counts, lm, dm, iter_size=k, **SGD))
    try:
        assert net.connect(net.localAddresses())
        net.set_option("train_pipeline", pipeline)
        sim = _sim(accum, 1, counts, lm, dm, SGD, k, 1)
        to_dev(net.data(), sim.data[0])
        prod = _SyntheticProducer(net, sim.P)
        for t in range(4):
            prod.step = t
            assert net.train(0, _batch(float(t))), net.last_error()
            sim.step([[prod.grad(t, q)] for q in range(k)])
        assert net.synchronize(), net.last_error()
        assert net.iter() == 4                                          # one ++iter_ per step
        assert_bits_equal(to_host(net.data()), sim.data[0], "weights after 4 steps")
        assert_bits_equal(to_host(net.history()), sim.hist[0], "history after 4 steps")
        assert not to_host(net.diff()).any()
        assert [c[:2] for c in prod.calls] == [(t, q) for t in range(4) for q in range(k)]
        for t in range(4):
            calls = [c for c in prod.calls if c[0] == t]
            assert len({c[2] for c in calls}) == 1                      # every pass read the one staged batch
            assert len({c[3] for c in calls}) == k                      # each pass has its own loss slot
        want = accum.loss_mean([prod.loss(3, q) for q in range(k)])
        assert np.float32(net.last_loss()).view(np.uint32) == np.float32(want).view(np.uint32)
    finally:
        net.deallocate()


@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_train_accumulate_micro_batches_pipelined_equals_synchronous(cos, oracle, accum, solver):
    counts, lm, dm = LAYOUTS["lenet"]
    k = 4
    hp = SGD if solver == "SGD" else ADAM
    results = []
    for pipeline in (1, 0):
        net = cos.CaffeNet(cos.SolverDesc(counts, lm, dm, iter_size=k, **hp))
        try:
            assert net.connect(net.localAddresses())
            net.set_option("train_pipeline", pipeline)
            sim = _sim(accum, 1, counts, lm, dm, hp, k, 1)
            to_dev(net.data(), sim.data[0])
            prod = _SyntheticProducer(net, sim.P)
            losses = []
            for t in range(5):
                prod.step = t
                assert net.train_accumulate(0, [_batch(10.0 * t + q) for q in range(k)]), net.last_error()
                sim.step([[prod.grad(t, q)] for q in range(k)])
                if not pipeline:
                    losses.append(net.last_loss())
            assert net.synchronize(), net.last_error()
            assert net.iter() == 5
            for t in range(5):
                calls = [c for c in prod.calls if c[0] == t]
                assert len(calls) == k and len({c[2] for c in calls}) == k  # k distinct staged micro-batches
            if not pipeline:
                for t in range(5):
                    want = accum.loss_mean([prod.loss(t, q) for q in range(k)])
                    assert np.float32(losses[t]).view(np.uint32) == np.float32(want).view(np.uint32)
            assert_bits_equal(to_host(net.data()), sim.data[0], f"weights pipeline={pipeline}")
            assert_bits_equal(to_host(net.history()), sim.hist[0], f"history pipeline={pipeline}")
            assert not to_host(net.diff()).any()
            results.append((to_host(net.data()), to_host(net.history())))
        finally:
            net.deallocate()
    assert_bits_equal(results[0][0], results[1][0], "pipelined == synchronous")


def test_train_accumulate_argument_checks(cos):
    net = cos.CaffeNet(cos.SolverDesc([100], iter_size=2, **SGD))
    try:
        assert net.connect(net.localAddresses())
        assert not net.train_accumulate(0, [_batch(1.0)])              # 1 micro-batch, iter_size 2
        assert "must equal the solver's iter_size" in net.last_error()
        assert not net.train_accumulate(0, [_batch(1.0), _batch(2.0)])  # no producer registered
        assert "no gradient producer" in net.last_error()
        with pytest.raises(cos.CosError):
            net.train_accumulate(0, None)
        with pytest.raises(cos.CosError, match="same number of blobs"):
            net.train_accumulate(0, [_batch(1.0), _batch(2.0)[:1]])
        assert not net.train_accumulate(3, [_batch(1.0), _batch(2.0)])
        assert net.iter() == 0
    finally:
        net.deallocate()


def test_multi_device_net_accumulates_per_rank(cos, oracle, accum, monkeypatch):
    """-devices 2 in one executor: train() on every local rank runs its k passes, then the one collective step.
    With one GPU the two local solvers share it (COS_ALLOW_SHARED_DEVICE, tests only)."""
    monkeypatch.setenv("COS_ALLOW_SHARED_DEVICE", "1")
    counts, lm, dm = MULTI
    k = 3
    desc = cos.SolverDesc(counts, lm, dm, iter_size=k, **SGD)
    net = cos.CaffeNet(desc, "", "", 2, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        for opt, v in (("grid", 4), ("block", 128), ("barrier_timeout_ms", 8000), ("initial_gather", 0)):
            net.set_option(opt, v)
        sim = _sim(accum, 2, counts, lm, dm, SGD, k, 1)
        for i in range(2):
            to_dev(net.data(i), sim.data[i])
        torch.cuda.synchronize()
        assert net.connect(net.localAddresses()), net.last_error()
        for i in range(2):
            assert net.all_gather_weights(i), net.last_error()
        assert net.synchronize(), net.last_error()
        prod = _SyntheticProducer(net, sim.P, local=2)
        for t in range(3):
            prod.step = t
            for i in range(2):  # train() of rank 0 returns after its launch, before rank 1's passes ran
                assert net.train(i, _batch(float(t))), net.last_error()
            sim.step([[prod.grad(t, q, r) for r in range(2)] for q in range(k)])
        assert net.synchronize(), net.last_error()
        for i in range(2):
            assert [c[:2] for c in prod.calls if c[4] == i] == [(t, q) for t in range(3) for q in range(k)]
            assert_bits_equal(to_host(net.data(i)), sim.consistent_weights(), f"local rank {i}")
            assert not to_host(net.diff(i)).any()
    finally:
        net.deallocate()


@pytest.mark.parametrize("fmt", ["BINARYPROTO", "HDF5"])
def test_snapshot_and_resume_mid_run(cos, oracle, accum, tmp_path, fmt):
    from caffeonspark_b200 import nets
    (tmp_path / "net.prototxt").write_text(nets.net_prototxt("cifar10_quick"))
    prefix = str(tmp_path / "ckpt")
    solver = tmp_path / "solver.prototxt"
    solver.write_text(f'net: "net.prototxt"\nbase_lr: 0.001\nmomentum: 0.9\nweight_decay: 0.004\nlr_policy: "fixed"\n'
                      f'max_iter: 100\niter_size: 2\nsnapshot_prefix: "{prefix}"\nsnapshot_format: {fmt}\n')
    P = nets.EXPECTED_PARAM_COUNT["cifar10_quick"]
    grads = [oracle.fill(P, 21, 4096 * (t + 1), 0.01) for t in range(4)]

    def run_steps(net, ts):
        for t in ts:
            to_dev(net.diff(), grads[t])
            torch.cuda.synchronize()
            assert net.sync_step(0) and net.synchronize(), net.last_error()

    a = cos.CaffeNet(str(solver))
    try:
        assert a.desc.iter_size == 2
        assert a.connect(a.localAddresses())
        to_dev(a.data(), oracle.fill(P, 21, 0, 0.05))
        run_steps(a, [0, 1])
        assert a.snapshot() == 2, a.last_error()                        # iter counts steps, not passes
        model, state = a.snapshotFilename(2, False), a.snapshotFilename(2, True)
        h2 = to_host(a.history())
        run_steps(a, [2, 3])
        w_ref, h_ref = to_host(a.data()), to_host(a.history())
    finally:
        a.deallocate()
    b = cos.CaffeNet(str(solver), model, state)
    try:
        assert b.connect(b.localAddresses())
        assert b.iter() == 2
        assert_bits_equal(to_host(b.history()), h2, "restored history")
        run_steps(b, [2, 3])
        assert_bits_equal(to_host(b.data()), w_ref, "weights after resume")
        assert_bits_equal(to_host(b.history()), h_ref, "history after resume")
    finally:
        b.deallocate()
    # a different iter_size may resume the same state (Caffe allows it): the step then normalises by 1/4
    other = tmp_path / "solver4.prototxt"
    other.write_text(solver.read_text().replace("iter_size: 2", "iter_size: 4"))
    c = cos.CaffeNet(str(other), model, state)
    try:
        assert c.connect(c.localAddresses()) and c.iter() == 2
        assert_bits_equal(to_host(c.history()), h2, "restored under iter_size 4")
    finally:
        c.deallocate()


# ------------------------------------------------------------------------------------------ functional

# Four micro-batches of 16 with iter_size 4 against one batch of 64 with iter_size 1: the mean losses differ only in
# rounding (sum of 4 means of 16, times 1/4, against one mean of 64), so after one step the weights agree to a few
# fp32 ulps of the update.  Tolerance: 1e-6 absolute on weights of magnitude ~0.1 after a step of lr 0.01.
LENET_ATOL = 1e-6


def test_lenet_micro_batches_match_one_large_batch(cos):
    from caffeonspark_b200 import harness, nets
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    rng = np.random.RandomState(5)
    x = rng.rand(64, *nets.NETS["lenet"]["input"]).astype(np.float32)
    y = rng.randint(0, 10, (64,)).astype(np.float32)
    out = []
    for k in (1, 4):
        net = cos.CaffeNet(nets.solver_desc("lenet", iter_size=k))
        try:
            assert net.connect(net.localAddresses())
            harness.make_producer("lenet", net, seed=3, use_graph=False)
            w0 = to_host(net.data())
            if k == 1:
                assert net.train(0, [x, y]), net.last_error()
            else:
                assert net.train_accumulate(0, [[x[16 * q:16 * (q + 1)], y[16 * q:16 * (q + 1)]]
                                                for q in range(4)]), net.last_error()
            assert net.synchronize(), net.last_error()
            out.append((w0, to_host(net.data()), net.last_loss()))
        finally:
            net.deallocate()
    assert_bits_equal(out[0][0], out[1][0], "same initial weights")
    delta = np.abs(out[0][1] - out[0][0]).max()
    assert delta > 1e-4                                                  # the step moved the weights
    np.testing.assert_allclose(out[1][1], out[0][1], rtol=0, atol=LENET_ATOL)
    assert abs(out[1][2] - out[0][2]) < 1e-5 * abs(out[0][2])


def test_cifar10_quick_iter_size_2_converges(cos):
    from caffeonspark_b200 import harness, nets
    import test_gpu_bf16_producer as B
    net = cos.CaffeNet(nets.solver_desc("cifar10_quick", iter_size=2))
    try:
        assert net.connect(net.localAddresses())
        harness.make_producer("cifar10_quick", net, seed=1234)
        xh = [torch.empty(50, 3, 32, 32).pin_memory() for _ in range(2)]
        yh = [torch.empty(50).pin_memory() for _ in range(2)]
        losses = []
        for x, y in B._task_batches():
            for q in range(2):
                xh[q].copy_(x[50 * q:50 * (q + 1)])
                yh[q].copy_(y[50 * q:50 * (q + 1)])
            assert net.train_accumulate(0, [[xh[0], yh[0]], [xh[1], yh[1]]]), net.last_error()
            assert net.synchronize(), net.last_error()
            losses.append(net.last_loss())
        assert net.iter() == B.CONV_STEPS
    finally:
        net.deallocate()
    losses = np.array(losses)
    f = losses[-B.CONV_WINDOW:].mean()
    print(f"iter_size 2 CIFAR-10-quick: first step {losses[0]:.4f}, final {B.CONV_WINDOW}-step window {f:.4f}")
    assert np.isfinite(losses).all()
    assert f < B.CONV_MAX_LOSS, f
