"""iter_size > 1 (gradient accumulation) on the host: parser, C ABI descriptor, the new entry point's argument
checks, and the C oracle against the independent numpy restatement.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

from conftest import gpu_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENET_NET = os.path.join(ROOT, "tests", "golden", "configs", "lenet_memory_train_test.prototxt")


@pytest.fixture(scope="module")
def accum(oracle):
    from oracle import accum
    accum.build()
    accum.lib()
    return accum


def _solver(tmp_path, extra):
    p = tmp_path / "s.prototxt"
    p.write_text(f'net: "{LENET_NET}"\nbase_lr: 0.01\nmomentum: 0.9\nlr_policy: "fixed"\n{extra}')
    return str(p)


def test_iter_size_parses(cos, tmp_path):
    assert cos.parse_solver(_solver(tmp_path, "iter_size: 3\n")).iter_size == 3
    assert cos.parse_solver(_solver(tmp_path, "")).iter_size == 1               # caffe.proto default
    assert cos.parse_solver(_solver(tmp_path, 'iter_size: 2\ntype: "Adam"\n')).iter_size == 2


@pytest.mark.parametrize("k", [0, -1])
def test_iter_size_below_one_is_rejected(cos, tmp_path, k):
    with pytest.raises(cos.CosError, match="iter_size must be >= 1"):
        cos.parse_solver(_solver(tmp_path, f"iter_size: {k}\n"))


def test_clip_gradients_stays_rejected_with_iter_size(cos, tmp_path):
    with pytest.raises(cos.CosError, match="clip_gradients"):
        cos.parse_solver(_solver(tmp_path, "iter_size: 2\nclip_gradients: 10\n"))


def test_desc_round_trips_and_zero_reads_as_one(cos, tmp_path):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    d = _lib.cos_solver_desc()
    cap = 64
    c, lm, dm = (ctypes.c_int64 * cap)(), (ctypes.c_float * cap)(), (ctypes.c_float * cap)()
    n = L.cos_parse_solver(_solver(tmp_path, "iter_size: 5\n").encode(), ctypes.byref(d), c, lm, dm, cap, None,
                           None, 0, None, 0, None)
    assert n > 0 and d.iter_size == 5
    # the field is the last one of the struct: a descriptor built before it existed reads it as 0
    assert _lib.cos_solver_desc._fields_[-1] == ("iter_size", ctypes.c_int)
    assert _lib.cos_solver_desc.iter_size.offset > _lib.cos_solver_desc.delta.offset
    desc = cos.SolverDesc([100], iter_size=4)
    cd, keep = desc.to_c()
    assert cd.iter_size == 4 and desc.hyper()["iter_size"] == 4
    assert "iter_size" not in cos.SolverDesc([100]).hyper()     # iter_size 1: the existing oracle's arguments
    with pytest.raises(ValueError, match="iter_size"):
        cos.SolverDesc([100], iter_size=0)
    from caffeonspark_b200 import nets
    assert nets.solver_desc("lenet", iter_size=2).iter_size == 2


def test_desc_iter_size_checked_before_any_device(cos):
    """A negative iter_size is refused by the descriptor check; 0 passes it (read as 1) and only then meets the
    device, which on a GPU-less host is the "no CPU path" failure."""
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    d, keep = cos.SolverDesc([100]).to_c()
    out = ctypes.c_void_p()
    d.iter_size = -2
    assert L.cos_net_allocate_desc(ctypes.byref(d), 1, 1, 0, 1, 0, -1, ctypes.byref(out)) == 0
    assert b"iter_size must be >= 1" in L.cos_last_error()
    if gpu_count() == 0:
        d.iter_size = 0
        assert L.cos_net_allocate_desc(ctypes.byref(d), 1, 1, 0, 1, 0, -1, ctypes.byref(out)) == 0
        assert b"no CPU path" in L.cos_last_error()


def test_train_accumulate_survives_null_arguments(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert L.cos_net_train_accumulate(None, 0, None, 0, 0) == 0
    assert b"net is NULL" in L.cos_last_error()
    assert L.cos_net_train_accumulate(None, -1, None, 1, 2) == 0
    blobs = (_lib.cos_blob * 2)()
    assert L.cos_net_train_accumulate(None, 0, blobs, 1, 2) == 0


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
def test_iter_size_net_fails_loudly_without_a_gpu(cos):
    with pytest.raises(cos.CosError, match="no CPU path"):
        cos.CaffeNet(cos.SolverDesc([100], lr_policy="fixed", base_lr=0.1, iter_size=2))


def test_accum_norm_and_loss_mean(accum):
    from oracle import numpy_accum as NA
    for k in (1, 2, 3, 5, 7):
        assert np.float32(accum.accum_norm(k)) == np.float32(1.0) / np.float32(k)
    rng = np.random.RandomState(3)
    for k in (2, 3, 5, 7):
        losses = rng.rand(k).astype(np.float32) * 5
        assert np.float32(accum.loss_mean(losses)).view(np.uint32) == NA.loss_mean(losses).view(np.uint32)


def _case(N, k, rng, adam):
    counts = [int(x) for x in rng.randint(1, 300, size=rng.randint(1, 6))]
    lm = [float(x) for x in rng.choice([0.0, 1.0, 2.0], len(counts))]
    dm = [float(x) for x in rng.choice([0.0, 1.0], len(counts))]
    P = sum(counts)
    data = [(rng.randn(P) * 0.05).astype(np.float32)] * N
    hist = [(rng.randn(P * (2 if adam else 1)) * 0.01).astype(np.float32) for _ in range(N)]
    if adam:
        for h in hist:
            h[P:] = np.abs(h[P:])  # v >= 0
    grads = [[(rng.randn(P) * 0.01).astype(np.float32) for _ in range(N)] for _ in range(k)]
    return counts, lm, dm, data, hist, grads


@pytest.mark.parametrize("solver", ["SGD", "Adam"])
@pytest.mark.parametrize("reg", ["L2", "L1"])
def test_c_oracle_matches_numpy_bitwise(accum, solver, reg):
    from oracle import numpy_accum as NA
    rng = np.random.RandomState(17 if solver == "SGD" else 19)
    for k in (2, 3, 5, 7):
        for N in (1, 2, 3, 4):
            counts, lm, dm, data, hist, grads = _case(N, k, rng, solver == "Adam")
            it = int(rng.randint(0, 50))
            hp = dict(rate=0.01, momentum=0.9, weight_decay=0.0005, iter_size=k, it=it, regularization_type=reg,
                      solver_type=solver, momentum2=0.999, delta=1e-8)
            diff_c = accum.accumulate(grads)
            diff_n = NA.accumulate(grads)
            for a, b in zip(diff_c, diff_n):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
            d_c = [x.copy() for x in data]
            h_c = [x.copy() for x in hist]
            accum.step_accum(d_c, [x.copy() for x in diff_c], h_c, counts, lm, dm, **hp)
            d_n, h_n = NA.step_accum(data, diff_n, hist, counts, lm, dm, **hp)
            for r in range(N):
                o, s = accum.O.chunk(sum(counts), N, r)
                P = sum(counts)
                assert np.array_equal(d_c[r][o:o + s].view(np.uint32), d_n[r][o:o + s].view(np.uint32)), (k, N, r)
                assert np.array_equal(h_c[r][o:o + s].view(np.uint32), h_n[r][o:o + s].view(np.uint32)), (k, N, r)
                if solver == "Adam":
                    assert np.array_equal(h_c[r][P + o:P + o + s].view(np.uint32),
                                          h_n[r][P + o:P + o + s].view(np.uint32)), (k, N, r)


@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_two_identical_passes_equal_one_pass(accum, oracle, solver):
    """g + g and 0.5 * (g + g) are exact: iter_size 2 with the same gradient twice is the iter_size 1 step."""
    rng = np.random.RandomState(5)
    for N in (1, 2, 3):
        counts, lm, dm, data, hist, grads = _case(N, 1, rng, solver == "Adam")
        hp = dict(rate=0.01, momentum=0.9, weight_decay=0.0005, it=3, solver_type=solver)
        d1, h1 = [x.copy() for x in data], [x.copy() for x in hist]
        accum.step_accum(d1, accum.accumulate(grads), h1, counts, lm, dm, iter_size=1, **hp)
        d2, h2 = [x.copy() for x in data], [x.copy() for x in hist]
        accum.step_accum(d2, accum.accumulate(grads * 2), h2, counts, lm, dm, iter_size=2, **hp)
        for r in range(N):
            assert np.array_equal(d1[r].view(np.uint32), d2[r].view(np.uint32))
            assert np.array_equal(h1[r].view(np.uint32), h2[r].view(np.uint32))
        if solver == "SGD":  # iter_size 1 is the existing oracle's step
            d0, h0 = [x.copy() for x in data], [x.copy() for x in hist]
            oracle.step(d0, [g.copy() for g in grads[0]], h0, counts, lm, dm, 0.01, 0.9, 0.0005)
            for r in range(N):
                assert np.array_equal(d0[r].view(np.uint32), d1[r].view(np.uint32))
