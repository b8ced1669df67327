"""Adam solver (type: "Adam") on the host: parser, C ABI descriptor, oracles, powf restatement.  No GPU needed."""
import concurrent.futures as cf
import ctypes
import os

import numpy as np
import pytest

from conftest import gpu_count


@pytest.fixture(scope="module")
def adam_oracle(oracle):
    from oracle import adam
    adam.build()
    adam.lib()
    return adam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENET_NET = os.path.join(ROOT, "tests", "golden", "configs", "lenet_memory_train_test.prototxt")

# examples/mnist/lenet_solver_adam.prototxt's values
ADAM_SOLVER = (f'net: "{LENET_NET}"\ntest_iter: 100\ntest_interval: 500\nbase_lr: 0.001\nmomentum: 0.9\n'
               'momentum2: 0.999\nlr_policy: "fixed"\ndisplay: 100\nmax_iter: 10000\nsnapshot: 5000\n'
               'snapshot_prefix: "examples/mnist/lenet"\ntype: "Adam"\nsolver_mode: GPU\n')


def test_adam_prototxt_parses(cos, tmp_path):
    p = tmp_path / "lenet_solver_adam.prototxt"
    p.write_text(ADAM_SOLVER)
    d = cos.parse_solver(str(p))
    assert d.type == "Adam"
    assert d.base_lr == pytest.approx(0.001) and d.momentum == pytest.approx(0.9)
    assert np.float32(d.momentum2) == np.float32(0.999) and np.float32(d.delta) == np.float32(1e-8)
    assert d.lr_policy == "fixed" and d.max_iter == 10000
    sgd = cos.parse_solver(os.path.join(ROOT, "tests", "golden", "configs", "lenet_memory_solver.prototxt"))
    assert d.counts == sgd.counts and d.lr_mult == sgd.lr_mult  # same net, same layout
    assert sgd.type == "SGD"
    assert d.history_count == 2 * d.param_count and sgd.history_count == sgd.param_count


def test_adam_defaults_and_deprecated_enum(cos, tmp_path):
    p = tmp_path / "s.prototxt"
    p.write_text(f'net: "{LENET_NET}"\nbase_lr: 0.01\nmomentum: 0.8\nmomentum2: 0.99\ndelta: 1e-6\ntype: "Adam"\n')
    d = cos.parse_solver(str(p))
    assert np.float32(d.momentum2) == np.float32(0.99) and np.float32(d.delta) == np.float32(1e-6)
    p.write_text(f'net: "{LENET_NET}"\nbase_lr: 0.01\nsolver_type: ADAM\n')  # caffe.proto SolverType
    d = cos.parse_solver(str(p))
    assert d.type == "Adam"
    assert np.float32(d.momentum2) == np.float32(0.999) and np.float32(d.delta) == np.float32(1e-8)


@pytest.mark.parametrize("kind", ['type: "Nesterov"', 'type: "AdaGrad"', 'type: "RMSProp"', 'type: "AdaDelta"',
                                  "solver_type: NESTEROV", "solver_type: ADAGRAD"])
def test_other_solver_types_still_rejected(cos, tmp_path, kind):
    p = tmp_path / "s.prototxt"
    p.write_text(f'net: "{LENET_NET}"\nbase_lr: 0.01\n{kind}\n')
    with pytest.raises(cos.CosError, match="not on the accelerated path"):
        cos.parse_solver(str(p))


def test_adam_needs_learnable_parameters(cos, tmp_path):
    """A net without learnable parameters has no history blobs, so its Adam and SGD states could not be told apart
    on restore: Adam is refused for it, from a prototxt and from a descriptor (before any device is touched)."""
    p = tmp_path / "s.prototxt"
    p.write_text('type: "Adam"\nbase_lr: 0.1\nlr_policy: "fixed"\nnet_param { }\n')
    with pytest.raises(cos.CosError, match="needs learnable parameters"):
        cos.parse_solver(str(p))
    p.write_text('base_lr: 0.1\nlr_policy: "fixed"\nnet_param { }\n')
    assert cos.parse_solver(str(p)).counts == []
    with pytest.raises(cos.CosError, match="needs learnable parameters"):
        cos.CaffeNet(cos.SolverDesc([], type="Adam"))


def test_desc_round_trips_through_cos_parse_solver(cos, tmp_path):
    from caffeonspark_b200 import _lib
    p = tmp_path / "s.prototxt"
    p.write_text(f'net: "{LENET_NET}"\nbase_lr: 0.002\nmomentum: 0.85\nmomentum2: 0.995\ndelta: 3e-7\n'
                 'type: "Adam"\nweight_decay: 0.0005\nregularization_type: "L1"\n')
    L = _lib.lib()
    d = _lib.cos_solver_desc()
    cap = 64
    c, lm, dm = (ctypes.c_int64 * cap)(), (ctypes.c_float * cap)(), (ctypes.c_float * cap)()
    pol, pre = ctypes.create_string_buffer(64), ctypes.create_string_buffer(64)
    sv, bs = (ctypes.c_int * 4)(), ctypes.c_int()
    n = L.cos_parse_solver(str(p).encode(), ctypes.byref(d), c, lm, dm, cap, pol, pre, 64, sv, 4, ctypes.byref(bs))
    assert n > 0
    assert d.solver_type == 1 and d.regularization_l1 == 1
    assert d.momentum2 == np.float32(0.995) and d.delta == np.float32(3e-7) and d.momentum == np.float32(0.85)
    # Python mirror -> C struct -> same fields
    desc = cos.parse_solver(str(p))
    c2, keep = desc.to_c()
    assert (c2.solver_type, c2.momentum2, c2.delta, c2.regularization_l1) == (1, d.momentum2, d.delta, 1)
    del keep
    # an SGD desc leaves the new fields at zero: existing callers that zero the struct stay SGD
    c3, keep = cos.SolverDesc([10]).to_c()
    assert c3.solver_type == 0
    with pytest.raises(ValueError):
        cos.SolverDesc([10], type="Nesterov")


def test_nets_solver_desc_passes_adam_through():
    from caffeonspark_b200 import nets
    d = nets.solver_desc("lenet", type="Adam", momentum2=0.99, delta=1e-7)
    assert d.type == "Adam" and d.momentum2 == 0.99 and d.delta == 1e-7
    h = d.hyper()
    assert h["solver_type"] == "Adam" and h["momentum2"] == 0.99 and h["delta"] == 1e-7
    assert "solver_type" not in nets.solver_desc("lenet").hyper()


@pytest.mark.parametrize("beta1,beta2", [(0.9, 0.999), (0.8, 0.99), (0.5, 0.5)])
def test_host_correction_matches_double_rounded_to_float(adam_oracle, beta1, beta2):
    import math
    for it in (0, 1, 2, 9, 99, 999, 12345, 10 ** 6):
        t = it + 1
        b1, b2 = float(np.float32(beta1)), float(np.float32(beta2))
        want = np.float32(math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))
        assert np.float32(adam_oracle.adam_correction(beta1, beta2, it)) == want
        from oracle import numpy_adam as NO
        assert NO.adam_correction(np.float32(beta1), np.float32(beta2), it) == want


def _random_case(rng):
    nb = int(rng.integers(1, 6))
    counts = [int(x) for x in rng.integers(1, 300, nb)]
    lm = [float(x) for x in rng.choice([0.0, 1.0, 2.0, 0.5], nb)]
    dm = [float(x) for x in rng.choice([0.0, 1.0], nb)]
    return counts, lm, dm


@pytest.mark.parametrize("case", range(12))
def test_c_oracle_matches_numpy_oracle_bitwise(oracle, adam_oracle, case):
    from oracle import numpy_adam as NO
    rng = np.random.default_rng(100 + case)
    counts, lm, dm = _random_case(rng)
    N = int(rng.integers(1, 5))
    reg = "L1" if case % 3 == 0 else "L2"
    P = sum(counts)
    b1, b2, delta, wd, rate = 0.9, 0.999, 1e-8, float(rng.choice([0.0, 5e-4])), 0.001
    it0 = int(rng.choice([0, 7, 5000]))
    data = [oracle.fill(P, case, 0, 0.05) for _ in range(N)]
    hist = [np.zeros(2 * P, np.float32) for _ in range(N)]
    nd, nh = [d.copy() for d in data], [h.copy() for h in hist]
    for t in range(int(rng.integers(1, 21))):
        grads = [oracle.fill(P, case, 1000 * t + r + 1, 0.01) for r in range(N)]
        adam_oracle.step_adam(data, [g.copy() for g in grads], hist, counts, lm, dm, rate, b1, b2, delta, wd, it0 + t,
                         reg)
        nd, nh = NO.step_adam(nd, grads, nh, counts, lm, dm, rate, b1, b2, delta, wd, it0 + t, reg)
        for r in range(N):
            assert np.array_equal(data[r].view(np.uint32), nd[r].view(np.uint32)), (t, r)
            assert np.array_equal(hist[r].view(np.uint32), nh[r].view(np.uint32)), (t, r)


def test_adam_matches_analytic_least_squares_update(adam_oracle):
    """Caffe's GradientBasedSolverTest checks Adam against a closed form for a least-squares problem; restated:
    m = (1-b1) g + b1 m0, v = (1-b2) g^2 + b2 v0, alpha_t = lr sqrt(1 - b2^t) / (1 - b1^t),
    update = alpha_t m / (sqrt(v) + delta), w' = w - update (t = number of iterations run, here iter + 1)."""
    rng = np.random.default_rng(7)
    n, d = 8, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = rng.standard_normal(n).astype(np.float32)
    w = (0.1 * rng.standard_normal(d)).astype(np.float32)
    b = np.float32(0.3)
    lr, b1, b2, delta = 0.01, 0.9, 0.999, 1e-8
    m0 = (0.01 * rng.standard_normal(d + 1)).astype(np.float32)
    v0 = (0.001 * rng.random(d + 1)).astype(np.float32)
    for it in (0, 3, 50):
        resid = X.astype(np.float64) @ w + b - y
        grad = np.concatenate([X.T.astype(np.float64) @ resid / n, [resid.mean()]])  # d/dw, d/db of |r|^2 / 2n
        data = np.concatenate([w, [b]]).astype(np.float32)
        hist = np.concatenate([m0, v0]).astype(np.float32)
        g = grad.astype(np.float32)
        adam_oracle.step_adam([data], [g.copy()], [hist], [d, 1], [1.0, 1.0], [1.0, 1.0], lr, b1, b2, delta, 0.0, it)
        t = it + 1
        m = (1 - b1) * g + b1 * m0.astype(np.float64)
        v = (1 - b2) * g.astype(np.float64) ** 2 + b2 * v0.astype(np.float64)
        alpha = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        want = np.concatenate([w, [b]]) - alpha * m / (np.sqrt(v) + delta)
        np.testing.assert_allclose(data, want, rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(hist[:d + 1], m, rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(hist[d + 1:], v, rtol=1e-5, atol=1e-12)


def test_powf_half_exhaustive(adam_oracle):
    """Every non-negative float bit pattern: the kernels' double-precision restatement of glibc's powf(x, 0.5f)
    (csrc/powf_half.h) is bit-identical to powf, which is not sqrtf."""
    chunks = 16
    step = (1 << 31) // chunks
    with cf.ThreadPoolExecutor(min(chunks, os.cpu_count() or 1)) as ex:  # ctypes releases the GIL
        res = list(ex.map(lambda k: adam_oracle.powf_half_check(k * step, (k + 1) * step), range(chunks)))
    vs_sqrt = sum(r[0] for r in res)
    vs_device = sum(r[1] for r in res)
    # glibc's powf rounds a double approximation and sqrtf is correctly rounded: with glibc 2.39 they differ by
    # one ulp on 1,361,091 inputs, so __fsqrt_rn would not reproduce the reference's update
    print(f"powf(x, 0.5f) != sqrtf(x) on {vs_sqrt} inputs; kernel restatement != powf on {vs_device}")
    assert vs_device == 0


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
def test_adam_net_fails_loudly_without_a_gpu(cos):
    d = cos.SolverDesc([100], lr_policy="fixed", base_lr=0.1, momentum=0.9, type="Adam")
    with pytest.raises(cos.CosError, match="no CPU path"):
        cos.CaffeNet(d)
