"""What the N-D convolution tests share (DESIGN.md section 14): the geometry sweep of the 3-D Convolution and
Deconvolution, their inputs, and float64 references (PyTorch's conv3d in double on the CPU) with per-element bounds.

A case is (N, Cin, D, H, W, Cout, geo3, bias) with geo3 = (kd, kh, kw, sd, sh, sw, pd, ph, pw).  The bound on an fp32
result of a chain of K products is (K + 2) u sum |a b| (u = 2^-24), the sum of magnitudes computed by the same
reference on |a| and |b|; gemm3d_ref's split-K adds at most 256 partials, inside that K."""
import numpy as np

F32 = np.float32
U = 2.0 ** -24

CONV3D_CASES = [
    (2, 3, 5, 6, 7, 4, (1, 1, 1, 1, 1, 1, 0, 0, 0), True),     # 1x1x1
    (2, 3, 6, 6, 6, 4, (2, 2, 2, 2, 2, 2, 0, 0, 0), True),     # 2x2x2 stride 2: V-Net's way down
    (2, 3, 5, 6, 7, 4, (3, 3, 3, 1, 1, 1, 1, 1, 1), True),     # 3x3x3 pad 1
    (1, 2, 7, 9, 11, 3, (3, 3, 3, 2, 2, 2, 0, 0, 0), True),    # stride 2 over odd sizes
    (2, 3, 4, 9, 9, 5, (1, 3, 3, 1, 2, 2, 0, 1, 1), True),     # (1, 3, 3), stride (1, 2, 2), pad (0, 1, 1)
    (2, 1, 5, 5, 5, 3, (3, 3, 3, 1, 1, 1, 1, 0, 0), False),    # Cin = 1; pad on the depth axis only
    (2, 4, 5, 5, 5, 1, (3, 3, 3, 1, 1, 1, 0, 1, 1), True),     # Cout = 1
    (1, 3, 8, 9, 10, 2, (3, 3, 3, 1, 2, 2, 1, 1, 1), True),    # C3D's conv1 geometry
    (2, 17, 4, 4, 4, 65, (2, 2, 2, 1, 1, 1, 0, 0, 0), True),   # K = 136 across the 16-deep step, Cout across 64
    (1, 2, 3, 4, 5, 3, (2, 2, 2, 3, 3, 3, 0, 0, 0), True),     # stride > kernel
    (1, 2, 4, 4, 4, 2, (2, 2, 2, 1, 1, 1, 2, 2, 2), True),     # pad >= kernel
    (2, 2, 48, 48, 48, 3, (1, 1, 1, 1, 1, 1, 0, 0, 0), True),  # N OD OH OW = 221,184: 256 widened chunks of 864
]
DECONV3D_CASES = [
    (2, 4, 3, 4, 5, 2, (2, 2, 2, 2, 2, 2, 0, 0, 0), True),     # V-Net's way up
    (2, 3, 3, 3, 3, 2, (3, 3, 3, 1, 1, 1, 1, 1, 1), True),
    (1, 3, 3, 4, 4, 2, (1, 3, 3, 1, 2, 2, 0, 1, 1), True),
    (1, 1, 4, 5, 3, 1, (2, 3, 2, 3, 2, 1, 0, 0, 1), False),    # Cin = Cout = 1; stride > kernel on the depth axis
    (2, 2, 24, 24, 24, 2, (2, 2, 2, 2, 2, 2, 0, 0, 0), True),  # N D H W of the bottom = 27,648: 54 chunks
]


def out3(dhw, geo3):
    return tuple((dhw[a] + 2 * geo3[6 + a] - geo3[a]) // geo3[3 + a] + 1 for a in range(3))


def deconv_out3(dhw, geo3):
    return tuple(geo3[3 + a] * (dhw[a] - 1) + geo3[a] - 2 * geo3[6 + a] for a in range(3))


def inputs(case, deconv=False):
    """-> (x, w, b or None): x Gaussian, w Gaussian / sqrt(fan-in), b Gaussian / 10"""
    n, cin, d, h, w, cout, geo3, bias = case
    rng = np.random.default_rng(n * 7919 + cin * 613 + cout * 31 + d * 7 + h * 3 + w + sum(geo3) + (5 if deconv else 0))
    x = rng.standard_normal((n, cin, d, h, w)).astype(F32)
    wshape = (cin, cout) + geo3[:3] if deconv else (cout, cin) + geo3[:3]
    wt = (rng.standard_normal(wshape) / np.sqrt(cin * np.prod(geo3[:3]))).astype(F32)
    b = (rng.standard_normal(cout) * 0.1).astype(F32)
    return x, wt, (b if bias else None)


def _t(a):
    import torch
    return None if a is None else torch.from_numpy(np.asarray(a, np.float64))


def conv3d64(x, w, b, geo3):
    import torch.nn.functional as F
    return F.conv3d(_t(x), _t(w), _t(b), stride=geo3[3:6], padding=geo3[6:9]).numpy()


def conv3d_backward64(x, w, dy, geo3):
    """-> (dW, db, dx) of the convolution for the top gradient dy, in float64"""
    import torch
    import torch.nn.functional as F
    xt, wt = _t(x).requires_grad_(), _t(w).requires_grad_()
    F.conv3d(xt, wt, None, stride=geo3[3:6], padding=geo3[6:9]).backward(_t(dy))
    return wt.grad.numpy(), np.asarray(dy, np.float64).sum(axis=(0, 2, 3, 4)), xt.grad.numpy()


def conv3d_bounds(x, w, b, dy, geo3):
    """-> per-element bounds on the fp32 y, dW, db and dx"""
    ax, aw, ady = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(w, np.float64)), np.abs(np.asarray(dy, np.float64))
    k = w.shape[1] * int(np.prod(geo3[:3]))
    y = (k + 2) * U * (conv3d64(ax, aw, None, geo3) + (0 if b is None else np.abs(b)[None, :, None, None, None]))
    gw, gb, gx = conv3d_backward64(ax, aw, ady, geo3)
    depth = dy.shape[0] * int(np.prod(dy.shape[2:]))
    return y, (depth + 258) * U * gw, (depth + 2) * U * gb, (w.shape[0] * int(np.prod(geo3[:3])) + 2) * U * gx


def deconv3d64(x, w, b, geo3):
    import torch.nn.functional as F
    return F.conv_transpose3d(_t(x), _t(w), _t(b), stride=geo3[3:6], padding=geo3[6:9]).numpy()


def deconv3d_backward64(x, w, dy, geo3):
    import torch
    import torch.nn.functional as F
    xt, wt = _t(x).requires_grad_(), _t(w).requires_grad_()
    F.conv_transpose3d(xt, wt, None, stride=geo3[3:6], padding=geo3[6:9]).backward(_t(dy))
    return wt.grad.numpy(), np.asarray(dy, np.float64).sum(axis=(0, 2, 3, 4)), xt.grad.numpy()


def deconv3d_bounds(x, w, b, dy, geo3):
    """the deconvolution is the convolution from its top to its bottom: y a chain over Cin KD KH KW, dW over the
    bottom's N D H W, dx over Cout KD KH KW"""
    ax, aw, ady = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(w, np.float64)), np.abs(np.asarray(dy, np.float64))
    kk = int(np.prod(geo3[:3]))
    y = (w.shape[0] * kk + 2) * U * (deconv3d64(ax, aw, None, geo3) +
                                    (0 if b is None else np.abs(b)[None, :, None, None, None]))
    gw, gb, gx = deconv3d_backward64(ax, aw, ady, geo3)
    depth = x.shape[0] * int(np.prod(x.shape[2:]))
    dyd = dy.shape[0] * int(np.prod(dy.shape[2:]))
    return y, (depth + 258) * U * gw, (dyd + 2) * U * gb, (w.shape[1] * kk + 2) * U * gx
