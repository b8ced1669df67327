"""-m gpu: the fused sync kernels on the named layouts of tests/sync_layouts.py (segment tables on both sides of the
shared-memory limits, rounding multipliers, zero-count blobs, a ResNet-152-like BN net, Adam with P odd), bit for bit
against oracle.Simulation / AdamSimulation / AccumSimulation over three steps: the weights on every rank, the owned
history shard (m and v for Adam), and diff_ zero afterwards."""
import os
import sys

import numpy as np
import pytest

import sync_layouts as S
from conftest import ROOT, gpu_count
from gpu_util import Ranks, assert_bits_equal

pytestmark = pytest.mark.gpu

SGD_HP = dict(lr_policy="inv", base_lr=0.01, gamma=0.0001, power=0.75, momentum=0.9, weight_decay=0.0005)
ADAM_HP = dict(lr_policy="fixed", base_lr=0.001, momentum=0.9, weight_decay=0.0005, type="Adam", momentum2=0.999,
               delta=1e-8)
STEPS = 3
MULTI_LAYOUTS = ["seg_513", "seg_1025", "empty_blobs", "resnet152_bn_like"]
KERNELS = {"ldg": 0, "tma": 1, "push": 2, "ll": 4}


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


def _simulation(oracle, adam, accum, N, counts, lm, dm, solver, reg, bf16, iter_size, seed):
    if iter_size > 1:
        hp = {k: v for k, v in (SGD_HP if solver == "SGD" else ADAM_HP).items() if k != "type"}
        # bf16 stays off here: the wire rounds the accumulated gradient, which check() rounds itself
        return accum.AccumSimulation(N, counts, lm, dm, iter_size=iter_size, solver_type=solver, seed=seed,
                                     regularization_type=reg, **hp)
    if solver == "Adam":
        hp = {k: v for k, v in ADAM_HP.items() if k != "type"}
        return adam.AdamSimulation(N, counts, lm, dm, seed=seed, bf16=bf16, regularization_type=reg, **hp)
    return oracle.Simulation(N, counts, lm, dm, seed=seed, bf16=bf16, regularization_type=reg, **SGD_HP)


def check(cos, oracle, adam, accum, N, counts, lm, dm, solver="SGD", reg="L2", bf16=False, iter_size=1, seed=7,
          desc=None, **opts):
    """STEPS steps of N in-process ranks against the oracle; returns the resolved kernel."""
    if desc is None:
        hp = SGD_HP if solver == "SGD" else ADAM_HP
        desc = cos.SolverDesc(counts, lm, dm, grad_dtype="bf16" if bf16 else "fp32", regularization_type=reg,
                              iter_size=iter_size, **hp)
    sim = _simulation(oracle, adam, accum, N, counts, lm, dm, solver, reg, bf16, iter_size, seed)
    R = Ranks(cos, desc, N, **opts)
    try:
        R.set_weights(sim.data)
        R.connect()
        kernel = R.nets[0].get_option("resolved_kernel")
        mode = R.nets[0].get_option("resolved_algo")
        P = sim.P
        for t in range(STEPS):
            if iter_size > 1:
                per_pass = [[sim.pass_gradient(r, t, k) for r in range(N)] for k in range(iter_size)]
                acc = accum.accumulate(per_pass)   # what iter_size producer calls leave in diff_
                sim.step_accumulated([oracle.round_bf16(a) for a in acc] if bf16 else acc)
                R.step(acc)
            else:
                grads = [oracle.fill(P, seed, (t + 1) * 4096 + r, 0.01) for r in range(N)]  # bf16: rounded in-kernel
                sim.step()
                R.step(grads)
            w_ref = sim.data[0] if N == 1 else sim.consistent_weights()
            m_ref = sim.hist[0][:P] if N == 1 else sim.consistent_history()[:P]
            v_ref = None
            if solver == "Adam":
                v_ref = sim.hist[0][P:] if N == 1 else sim.consistent_v()
            for r in range(N):
                what = f"N={N} step {t} rank {r}"
                assert R.nets[r].iter() == sim.iter
                assert_bits_equal(R.weights(r), w_ref, f"weights {what}")
                o, s = (0, P) if N == 1 or mode == 2 else cos.chunk(P, N, r)
                h = R.history(r)
                assert_bits_equal(h[o:o + s], m_ref[o:o + s], f"history {what}")
                if v_ref is not None:
                    assert_bits_equal(h[P + o:P + o + s], v_ref[o:o + s], f"v {what}")
                assert not R.diff(r).any(), f"diff_ not zero, {what}"
        return kernel
    finally:
        R.close()


def _layout_check(cos, oracle, adam, accum, name, N, kernel, **kw):
    counts, lm, dm = S.layout(name)
    rk = check(cos, oracle, adam, accum, N, counts, lm, dm, kernel=kernel, **kw)
    assert rk == kernel, (name, kernel, rk)


# ------------------------------------------------------------------ N = 1

@pytest.mark.parametrize("name", S.NAMES)
@pytest.mark.parametrize("variant", ["sgd_l2", "sgd_l1", "bf16"])
@pytest.mark.parametrize("kernel", [0, 1], ids=["ldg", "tma"])
def test_local_sgd(cos, oracle, adam, accum, name, variant, kernel):
    _layout_check(cos, oracle, adam, accum, name, 1, kernel, reg="L1" if variant == "sgd_l1" else "L2",
                  bf16=variant == "bf16")


@pytest.mark.parametrize("name", S.NAMES)
@pytest.mark.parametrize("variant", ["adam", "iter_size_3"])
def test_local_ldg_adam_and_iter_size(cos, oracle, adam, accum, name, variant):
    if variant == "adam":
        _layout_check(cos, oracle, adam, accum, name, 1, 0, solver="Adam")
    else:
        _layout_check(cos, oracle, adam, accum, name, 1, 0, iter_size=3)


# ------------------------------------------------------- N = 2, 3, 4 in process

@pytest.mark.parametrize("name", MULTI_LAYOUTS)
@pytest.mark.parametrize("N", [2, 3, 4])
@pytest.mark.parametrize("kernel", sorted(KERNELS.values()), ids=sorted(KERNELS, key=KERNELS.get))
def test_two_shot(cos, oracle, adam, accum, name, N, kernel):
    _layout_check(cos, oracle, adam, accum, name, N, kernel, algo=1)


@pytest.mark.parametrize("name", ["seg_513", "seg_1025"])
@pytest.mark.parametrize("N", [2, 3, 4])
@pytest.mark.parametrize("kernel", [0, 1], ids=["ldg", "tma"])
def test_one_shot(cos, oracle, adam, accum, name, N, kernel):
    _layout_check(cos, oracle, adam, accum, name, N, kernel, algo=2)


@pytest.mark.parametrize("variant", ["bf16_wire", "l1", "adam", "iter_size_3"])
@pytest.mark.parametrize("N", [2, 4])
@pytest.mark.parametrize("kernel", sorted(KERNELS.values()), ids=sorted(KERNELS, key=KERNELS.get))
def test_two_shot_variants_on_seg_1025(cos, oracle, adam, accum, variant, N, kernel):
    if variant == "adam" and kernel == 1:
        pytest.skip("the TMA kernel implements SGD only (forcing it on an Adam net is refused)")
    kw = dict(bf16_wire=dict(bf16=True), l1=dict(reg="L1"), adam=dict(solver="Adam"),
              iter_size_3=dict(iter_size=3))[variant]
    _layout_check(cos, oracle, adam, accum, "seg_1025", N, kernel, algo=1, **kw)


@pytest.mark.parametrize("name", ["empty_blobs", "resnet152_bn_like"])
@pytest.mark.parametrize("kernel", [0, 2, 4], ids=["ldg", "push", "ll"])
def test_adam_multi_rank(cos, oracle, adam, accum, name, kernel):
    _layout_check(cos, oracle, adam, accum, name, 3, kernel, algo=1, solver="Adam")


@pytest.mark.parametrize("name", S.ADAM_ODD_P)
@pytest.mark.parametrize("N", [2, 3])
@pytest.mark.parametrize("kernel", [0, 2, 4], ids=["ldg", "push", "ll"])
def test_adam_odd_p(cos, oracle, adam, accum, name, N, kernel):
    """hist + P misaligned by 4, 8 or 12 bytes: load_v / store_v take the scalar or float2 path at N >= 2."""
    _layout_check(cos, oracle, adam, accum, name, N, kernel, algo=1, solver="Adam")


@pytest.mark.parametrize("kernel", [0, 4], ids=["ldg", "ll"])
def test_parsed_fractional_multipliers_reach_the_device(cos, oracle, adam, accum, tmp_path, kernel):
    """The prototxt of test_sync_layouts_host (multipliers 10, 0.1, 0.7, 20, 3, ...) through cos.parse_solver, then a
    two-rank net built from the parsed descriptor, against the oracle fed the protobuf-rounded multipliers."""
    import test_sync_layouts_host as H
    desc = cos.parse_solver(H.fractional_prototxt(tmp_path / "s.prototxt"))
    lm, dm = H.expected_multipliers()
    assert desc.counts == H.FRACTIONAL_COUNTS and desc.lr_mult == lm and desc.decay_mult == dm
    assert desc.hyper()["lr_policy"] == SGD_HP["lr_policy"]
    rk = check(cos, oracle, adam, accum, 2, desc.counts, lm, dm, desc=desc, algo=1, kernel=kernel)
    assert rk == kernel


# --------------------------------------------------- one process per GPU (>= 2)

def _worker(rank, world, port, name, solver, kernel, nvls, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch
    import torch.distributed as dist
    import caffeonspark_b200 as C
    import sync_layouts as L
    from caffeonspark_b200.harness import Cluster
    from gpu_util import to_dev, to_host
    from oracle import adam as A
    from oracle import oracle as O
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        counts, lm, dm = L.layout(name)
        hp = SGD_HP if solver == "SGD" else ADAM_HP
        desc = C.SolverDesc(counts, lm, dm, **hp)
        sim_hp = {k: v for k, v in hp.items() if k != "type"}
        sim = (O.Simulation(world, counts, lm, dm, seed=77, **sim_hp) if solver == "SGD" else
               A.AdamSimulation(world, counts, lm, dm, seed=77, **sim_hp))
        P = sim.P
        cl = Cluster(desc, rank=rank, world=world, device=rank)
        net = cl.net
        net.set_option("algo", 1)
        net.set_option("kernel", kernel)
        net.set_option("nvls", int(nvls))
        net.set_option("barrier_timeout_ms", 15000)
        to_dev(net.data(), sim.data[rank])
        torch.cuda.synchronize()
        cl.start()
        ok = True
        for t in range(STEPS):
            g = O.fill(P, 77, (t + 1) * 4096 + rank, 0.01)
            sim.step()
            to_dev(net.diff(), g)
            torch.cuda.synchronize()
            assert net.sync_step(0), net.last_error()
            assert net.synchronize(), net.last_error()
            o, s = net.shard()
            hist = to_host(net.history())
            got = [to_host(net.data()), hist[o:o + s]]
            want = [sim.consistent_weights(), sim.consistent_history()[:P][o:o + s]]
            if solver == "Adam":
                got.append(hist[P + o:P + o + s])
                want.append(sim.consistent_v()[o:o + s])
            for k, (a, b) in enumerate(zip(got, want)):
                if nvls and net.get_option("nvls_active") == 1:  # the switch chooses the summation order
                    ok = ok and np.allclose(a, b, rtol=1e-5, atol=1e-8 if k == 0 else 1e-9)
                else:
                    ok = ok and np.array_equal(a.view(np.uint32), b.view(np.uint32))
            ok = ok and not bool(net.diff().any())
        q.put((rank, bool(ok), int(net.get_option("nvls_active")), int(net.get_option("resolved_kernel"))))
        assert net.sync()
        net.deallocate()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(gpu_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("name,solver,kernel,nvls", [("seg_1025", "SGD", 0, False), ("seg_1025", "SGD", 2, False),
                                                     ("seg_1025", "SGD", 3, True), ("seg_513", "SGD", 1, False),
                                                     ("seg_1025", "Adam", 2, False)])
def test_one_process_per_gpu(cos, oracle, name, solver, kernel, nvls):
    """Default grid sizes, real NVLink.  NVLS (kernel 3) is held to 1e-5 while multicast is active and is bit-exact
    when the library keeps the P2P path."""
    import torch.multiprocessing as mp
    from test_gpu_multiproc import _free_port
    world = min(gpu_count(), 8)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, solver, kernel, nvls, q)) for r in range(world)]
    [p.start() for p in procs]
    [p.join(300) for p in procs]
    for p in procs:
        if p.is_alive():
            p.kill()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = sorted(q.get(timeout=5) for _ in range(world))
    assert all(ok for _, ok, _, _ in res), res
    assert len({a for _, _, a, _ in res}) == 1, "ranks disagree on whether NVLS is active"
    if not nvls:
        assert all(k == kernel for _, _, _, k in res), res
    print(name, solver, "kernel", kernel, "NVLS active:", res[0][2])
