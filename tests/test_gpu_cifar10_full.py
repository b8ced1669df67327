"""cifar10_full on the GPU (DESIGN.md section 14): the built-in engine's gradients against a float64 evaluation of the
same net, its determinism and accumulate contract, training through train() alone from the reference's own prototxt
with every update checked against the oracle, and the PyTorch producer in bf16."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from gpu_util import assert_bits_equal, to_host
from test_gpu_bf16_producer import _task_batches
from test_gpu_native_producer import _UpdateCheck, _blob_bound, _native_net, _reference, _run_once

pytestmark = pytest.mark.gpu

NAME = "cifar10_full"
SOLVER = os.path.join(ROOT, "tests", "golden", "configs", "cifar10_full_solver.prototxt")


def _batch(seed, scale=1.0):
    rng = np.random.RandomState(seed)
    x = (scale * rng.rand(100, 3, 32, 32)).astype(np.float32)
    return x, rng.randint(0, 10, 100).astype(np.float32)


@pytest.mark.parametrize("scale", [1.0, 60.0])  # 60: pixel-scale inputs, where alpha s is not negligible in the LRNs
def test_gradients_match_float64(cos, tmp_path, scale):
    from caffeonspark_b200 import nets
    counts, _, _, names = nets.layout(NAME)
    net = _native_net(cos, NAME, tmp_path)
    try:
        net.fill("data", 21, 0, 0.1)
        torch.cuda.synchronize()
        w = to_host(net.data())
        x, y = _batch(3, scale)
        net.diff().zero_()
        loss = torch.zeros(1, device="cuda")
        torch.cuda.synchronize()
        g, l32 = _run_once(net, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), loss)
        l64, g64, _ = _reference(NAME, w, x, y, torch.float64, "cpu")
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            lt, gt, _ = _reference(NAME, w, x, y, torch.float32, "cuda")
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        assert abs(l32 - l64) <= 1e-5 * abs(l64), (l32, l64)
        assert abs(lt - l64) <= 1e-5 * abs(l64), (lt, l64)
        off = 0
        for c, nm in zip(counts, names):
            sl = slice(off, off + c)
            off += c
            assert np.abs(g64[sl]).max() > 0, nm
            _blob_bound(g[sl], g64[sl], f"{NAME} {nm} native")
            _blob_bound(gt[sl], g64[sl], f"{NAME} {nm} PyTorch fp32")
    finally:
        net.deallocate()


def test_runs_are_bitwise_identical_and_accumulate(cos, tmp_path):
    net = _native_net(cos, NAME, tmp_path)
    try:
        net.fill("data", 5, 0, 0.1)
        x, y = _batch(4, 60.0)
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        loss = torch.zeros(1, device="cuda")
        runs = []
        for _ in range(2):
            net.diff().zero_()
            torch.cuda.synchronize()
            runs.append(_run_once(net, xd, yd, loss))
        assert_bits_equal(runs[0][0], runs[1][0], "diff of two runs")
        assert runs[0][1] == runs[1][1]
        g2, _ = _run_once(net, xd, yd, loss)  # no clearing: diff += g once more
        assert_bits_equal(g2, np.float32(2) * runs[0][0], "two calls accumulate 2g")
    finally:
        net.deallocate()


def test_train_through_train_alone(cos, oracle):
    """The reference's cifar10_full prototxt and nothing else: its fillers (conv1 std 1e-4), its solver (fixed lr
    0.001, momentum 0.9, weight decay 0.004, ip1 decay_mult 250).  Every update equals the oracle's, bit for bit."""
    net = cos.CaffeNet(SOLVER, "", "", 1, 1, 0, True, cos.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        assert net.param_count() == 89578
        net.use_native_producer(fill_weights=True)
        torch.cuda.synchronize()
        w0 = to_host(net.data())
        assert 0 < np.abs(w0[:2400]).max() < 1e-3  # conv1: gaussian std 1e-4
        check = _UpdateCheck(net, oracle)
        losses = []
        for t, (x, y) in enumerate(_task_batches()):
            check.before()
            assert net.train(0, [x.numpy(), y.numpy()]), net.last_error()
            assert net.synchronize(), net.last_error()
            losses.append(net.last_loss())
            check.after(t)
        losses = np.array(losses)
        assert np.isfinite(losses).all()
        # fixed before the first GPU run: a CPU run of the PyTorch composition with the same solver, fillers of the
        # same distributions and these batches falls from 2.302 (first 10 steps) to 2.05-2.16 (last 50), two seeds
        assert losses[-50:].mean() < losses[:10].mean() - 0.02, (losses[:10].mean(), losses[-50:].mean())
    finally:
        net.deallocate()


def test_bf16_pytorch_producer_trains(cos):
    from caffeonspark_b200 import harness, nets
    net = cos.CaffeNet(nets.solver_desc(NAME))
    try:
        assert net.connect(net.localAddresses())
        prod = harness.make_producer(NAME, net, seed=3, precision="bf16")
        x, y = _batch(5, 60.0)
        xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
        w0 = to_host(net.data()).copy()
        losses = []
        for _ in range(8):
            assert net.train(0, [xh, yh]), net.last_error()
            assert net.synchronize(), net.last_error()
            losses.append(net.last_loss())
        assert np.isfinite(losses).all(), losses
        w = to_host(net.data())
        assert np.isfinite(w).all() and not np.array_equal(w, w0)
        lrn = [m for m in prod.module if type(m).__name__ == "LRN"]
        assert [m.region for m in lrn] == ["WITHIN_CHANNEL"] * 2
    finally:
        net.deallocate()
