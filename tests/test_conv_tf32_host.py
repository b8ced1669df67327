"""CPU tests of the native TF32 convolutions (csrc/conv_tf32.cu, DESIGN.md section 10.2): the entry points' argument
checks and their loud failure without a GPU; a float64 numpy restatement of the kernels' three implicit-GEMM gathers
(forward, the strided data gradient with its divisibility test, the weight gradient, all per group) against
torch.nn.functional.conv2d and torch.nn.grad; and the rule that picks F.conv2d for CPU tensors, bf16 or autocast,
TF32 off and the geometries where cuDNN is faster."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import gpu_count

GEOM = (2, 6, 9, 11, 8, 3, 2, 2, 1, 1, 0, 2)  # n, c, h, w, k, r, s, stride_h, stride_w, pad_h, pad_w, groups


# --------------------------------------------------------------------------- the C entry points
def _calls(L, geom, x=1, w=1, y=1, ws=1):
    s = None
    return (lambda: L.cos_conv_forward(x, w, None, y, *geom, s),
            lambda: L.cos_conv_backward_data(y, w, x, *geom, s),
            lambda: L.cos_conv_backward_filter(x, y, w, ws, *geom, s))


@pytest.mark.parametrize("bad, msg", [
    ((0,) + GEOM[1:], "bad shape"),
    (GEOM[:7] + (0,) + GEOM[8:], "bad stride or pad"),
    (GEOM[:9] + (-1,) + GEOM[10:], "bad stride or pad"),
    (GEOM[:11] + (4,), "groups must divide"),
    (GEOM[:1] + (3,) + GEOM[2:11] + (2,), "groups must divide"),
    (GEOM[:5] + (12,) + GEOM[6:9] + (0,) + GEOM[10:], "larger than the padded input"),
    ((1 << 16, 1 << 10, 64, 64) + GEOM[4:], "2^31"),
])
def test_entry_points_refuse_bad_geometry(cos, bad, msg):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert L.cos_conv_workspace_floats(*bad) == 0
    for call in _calls(L, bad):
        assert call() == 0
        assert msg in L.cos_last_error().decode()


def test_entry_points_refuse_null_tensors(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for call in _calls(L, GEOM, x=None) + _calls(L, GEOM, w=None) + _calls(L, GEOM, y=None):
        assert call() == 0
        assert "NULL tensor" in L.cos_last_error().decode()
    big = (256, 3, 227, 227, 96, 11, 11, 4, 4, 0, 0, 1)  # CaffeNet conv1 splits its weight gradient
    assert L.cos_conv_workspace_floats(*big) > 0
    assert _calls(L, big, ws=None)[2]() == 0
    assert "NULL workspace" in L.cos_last_error().decode()


@pytest.mark.skipif(gpu_count() > 0, reason="only meaningful on a GPU-less box")
def test_entry_points_fail_loudly_without_a_gpu(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    for call in _calls(L, GEOM):
        assert call() == 0
        assert "no CPU path" in L.cos_last_error().decode()


# --------------------------------------------------------------------------- the gathers, restated
def _out(h, r, stride, pad):
    return (h + 2 * pad - r) // stride + 1


def gather_forward(x, w, stride, pad, g):
    """y[img, g·Kg + n, p, q] = sum over k = (c, r, s) of A[m, k] B[k, n], A the zero-padded window of x."""
    n, c, h, wd = x.shape
    k, cg, r, s = w.shape
    kg, P, Q = k // g, _out(h, r, stride[0], pad[0]), _out(wd, s, stride[1], pad[1])
    y = np.zeros((n, k, P, Q))
    for grp in range(g):
        A = np.zeros((n * P * Q, cg * r * s))
        for m in range(n * P * Q):
            img, p, q = m // (P * Q), m % (P * Q) // Q, m % Q
            for kk in range(cg * r * s):
                ch, rr, ss = kk // (r * s), kk % (r * s) // s, kk % s
                ih, iw = p * stride[0] - pad[0] + rr, q * stride[1] - pad[1] + ss
                if 0 <= ih < h and 0 <= iw < wd:
                    A[m, kk] = x[img, grp * cg + ch, ih, iw]
        B = w[grp * kg:(grp + 1) * kg].reshape(kg, -1).T
        y[:, grp * kg:(grp + 1) * kg] = (A @ B).reshape(n, P, Q, kg).transpose(0, 3, 1, 2)
    return y


def gather_data(dy, w, xshape, stride, pad, g):
    """dx[img, g·Cg + n, h, w] = sum over k = (f, r, s) of dy[img, g·Kg + f, (h + ph - r) / sh, (w + pw - s) / sw],
    kept only where both divisions are exact and land in the output plane."""
    n, c, h, wd = xshape
    k, cg, r, s = w.shape
    kg, P, Q = k // g, dy.shape[2], dy.shape[3]
    dx = np.zeros(xshape)
    for grp in range(g):
        A = np.zeros((n * h * wd, kg * r * s))
        for m in range(n * h * wd):
            img, hh, ww = m // (h * wd), m % (h * wd) // wd, m % wd
            for kk in range(kg * r * s):
                f, rr, ss = kk // (r * s), kk % (r * s) // s, kk % s
                ph, pw = hh + pad[0] - rr, ww + pad[1] - ss
                if ph < 0 or pw < 0 or ph % stride[0] or pw % stride[1]:
                    continue
                p, q = ph // stride[0], pw // stride[1]
                if p < P and q < Q:
                    A[m, kk] = dy[img, grp * kg + f, p, q]
        B = w[grp * kg:(grp + 1) * kg].transpose(0, 2, 3, 1).reshape(kg * r * s, cg)
        dx[:, grp * cg:(grp + 1) * cg] = (A @ B).reshape(n, h, wd, cg).transpose(0, 3, 1, 2)
    return dx


def gather_filter(x, dy, wshape, stride, pad, g, chunks=3):
    """dw[g·Kg + m, n] = sum over chunks, in order, of the chunk's sum over k = (img, p, q) of dy[img, g·Kg + m, p, q]
    times the window of x at tap n = (c, r, s)."""
    n, c, h, wd = x.shape
    k, cg, r, s = wshape
    kg, P, Q = k // g, dy.shape[2], dy.shape[3]
    dw = np.zeros(wshape)
    K = n * P * Q
    bounds = np.linspace(0, K, chunks + 1).astype(int)
    for grp in range(g):
        A = dy[:, grp * kg:(grp + 1) * kg].transpose(1, 0, 2, 3).reshape(kg, K)
        B = np.zeros((K, cg * r * s))
        for kk in range(K):
            img, p, q = kk // (P * Q), kk % (P * Q) // Q, kk % Q
            for t in range(cg * r * s):
                ch, rr, ss = t // (r * s), t % (r * s) // s, t % s
                ih, iw = p * stride[0] - pad[0] + rr, q * stride[1] - pad[1] + ss
                if 0 <= ih < h and 0 <= iw < wd:
                    B[kk, t] = x[img, grp * cg + ch, ih, iw]
        acc = np.zeros((kg, cg * r * s))
        for a, b in zip(bounds[:-1], bounds[1:]):
            acc = acc + A[:, a:b] @ B[a:b]
        dw[grp * kg:(grp + 1) * kg] = acc.reshape(kg, cg, r, s)
    return dw


@pytest.mark.parametrize("geom", [
    (2, 6, 9, 11, 8, (3, 2), (2, 1), (1, 0), 2),
    (1, 4, 10, 7, 6, (2, 4), (3, 4), (2, 3), 1),
    (3, 3, 13, 13, 4, (5, 5), (4, 4), (0, 0), 1),
    (2, 8, 6, 6, 12, (3, 3), (1, 1), (1, 1), 4),
])
def test_gathers_match_torch_in_float64(geom):
    n, c, h, w, k, kern, stride, pad, g = geom
    rng = np.random.RandomState(0)
    x = rng.randn(n, c, h, w)
    wt = rng.randn(k, c // g, *kern)
    P, Q = _out(h, kern[0], stride[0], pad[0]), _out(w, kern[1], stride[1], pad[1])
    dy = rng.randn(n, k, P, Q)
    tx, tw, tdy = (torch.from_numpy(a) for a in (x, wt, dy))
    np.testing.assert_allclose(gather_forward(x, wt, stride, pad, g),
                               F.conv2d(tx, tw, None, stride, pad, 1, g).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gather_data(dy, wt, x.shape, stride, pad, g),
                               torch.nn.grad.conv2d_input(x.shape, tw, tdy, stride, pad, 1, g).numpy(),
                               rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gather_filter(x, dy, wt.shape, stride, pad, g),
                               torch.nn.grad.conv2d_weight(tx, wt.shape, tdy, stride, pad, 1, g).numpy(),
                               rtol=1e-12, atol=1e-12)


# --------------------------------------------------------------------------- the selection rule
class _Fake:
    """Stands in for a tensor in native_conv (which reads only these attributes)."""

    def __init__(self, shape, dtype=torch.float32, cuda=True):
        self.shape, self.dtype, self.is_cuda = shape, dtype, cuda

    def dim(self):
        return len(self.shape)


CONV1_X, CONV1_W = (256, 3, 227, 227), (96, 3, 11, 11)


def test_native_route_only_where_cudnn_would_run_tf32_and_is_slower(monkeypatch):
    from caffeonspark_b200 import layers
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
    assert layers.native_conv(_Fake(CONV1_X), _Fake(CONV1_W))
    assert not layers.native_conv(_Fake(CONV1_X, cuda=False), _Fake(CONV1_W, cuda=False))
    assert not layers.native_conv(_Fake(CONV1_X, torch.bfloat16), _Fake(CONV1_W))
    assert not layers.native_conv(_Fake(CONV1_X, torch.float64), _Fake(CONV1_W, torch.float64))
    # CaffeNet conv2..conv5, CIFAR-10-quick conv1 (75 taps) and LeNet conv1 (25 taps): cuDNN
    for w in ((256, 48, 5, 5), (384, 256, 3, 3), (384, 192, 3, 3), (32, 3, 5, 5), (20, 1, 5, 5)):
        assert not layers.native_conv(_Fake((8, w[1], 32, 32)), _Fake(w))
    with monkeypatch.context() as m:  # autocast itself cannot be entered on a GPU-less host
        m.setattr(torch, "is_autocast_enabled", lambda *a: True)
        assert not layers.native_conv(_Fake(CONV1_X), _Fake(CONV1_W))
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    assert not layers.native_conv(_Fake(CONV1_X), _Fake(CONV1_W))


def test_cpu_modules_evaluate_f_conv2d():
    from caffeonspark_b200 import layers, nets
    torch.manual_seed(0)
    conv = layers.Conv2d(3, 8, 5, stride=2, padding=1, groups=1)
    ref = torch.nn.Conv2d(3, 8, 5, stride=2, padding=1)
    ref.load_state_dict(conv.state_dict())
    x = torch.randn(2, 3, 17, 17)
    assert torch.equal(conv(x), ref(x))
    assert type(conv).__name__ == "Conv2d" and isinstance(conv, torch.nn.Conv2d)
    kinds = [type(m).__name__ for m in nets.torch_module("caffenet")]
    assert kinds[4] == "Conv2d" and isinstance(nets.torch_module("caffenet")[4], layers.Conv2d)
