"""The native TF32 convolutions (csrc/conv_tf32.cu, DESIGN.md section 10.2) on the GPU.

Every element of y, dx and dw is held against float64 to

    |err| <= C_TF32 * (2^-10 + K * 2^-23) * sum |a * b|

where K is the pass's reduction length and sum |a * b| the same convolution of the operands' magnitudes: rounding
both operands to TF32 costs at most 2^-10 of each product (2 * 2^-11 plus their product), and K fp32 additions at most
K * 2^-24 of the magnitude sum each, doubled for slack.  C_TF32 = 2 was fixed before the first GPU run.  The same bound
holds for cuDNN's TF32 result on the same inputs (test_cudnn_tf32_meets_the_same_bound).  That bound grows with the
full reduction length, so for the weight gradient it accepts dw = 0 at CIFAR-10-quick conv1 b100.  So each output is
also held to a bound that follows the kernels' order: against float64 on the operands rounded as cvt.rna rounds them
(conv_tf32_ref.tf32_rna), to C_TF32 * (depth + 8) * 2^-23 * sum |a * b|, where depth is K for y and dx and, for dw,
one chunk's k-tiles of 16 products plus the number of chunks (conv_tf32_ref.filter_split).  The shapes are every
convolution of CaffeNet, LeNet and CIFAR-10-quick at their own batch and at batch 1 to 4, and ragged ones: M, N and K
off the tile sizes, groups 1 to 4, strides 1 to 4, pads 0 to 3 and non-square kernels.  Two calls give identical bits,
a captured graph's replay equals the eager call, NaN and Inf propagate, and a small-batch CaffeNet's gradients stay
within twice the error of the same net on cuDNN TF32."""
import pytest
import torch
import torch.nn.functional as F

import conv_tf32_ref as R
from caffeonspark_b200 import layers, nets

pytestmark = pytest.mark.gpu

NET_SHAPES = [pytest.param(shape, id=cid) for cid, shape in R.NET_SHAPES]
RAGGED = R.RAGGED
RAGGED_SHAPES = [pytest.param(shape, id=f"ragged{i}") for i, shape in enumerate(RAGGED)]


@pytest.fixture(autouse=True, scope="module")
def _release_cached_memory():
    """The float64 references of the batch-256 cases take gigabytes of PyTorch's caching allocator.  Hand them back to
    the driver when the module ends, so that later tests in the same process find the device as free as before."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _inputs(shape, seed):
    n, c, k, kern, stride, pad, g, h, w = shape
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((n, c, h, w), device="cuda", generator=gen)
    wt = torch.randn((k, c // g, *kern), device="cuda", generator=gen) / (c // g * kern[0] * kern[1]) ** 0.5
    p = (h + 2 * pad[0] - kern[0]) // stride[0] + 1
    q = (w + 2 * pad[1] - kern[1]) // stride[1] + 1
    dy = torch.randn((n, k, p, q), device="cuda", generator=gen)
    return x, wt, dy


_bound = R.tf32_bound


def _tf32(t):
    """cvt.rna.tf32.f32 of every element (conv_tf32_ref.tf32_rna), as float64."""
    return torch.from_numpy(R.tf32_rna(t.cpu().numpy())).to(t.device).double()


def _check(name, got, ref, bound):
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), (f"{name}: {int(bad.sum())} elements out of bound, worst {float((err / bound).max()):.3f} "
                           f"of the bound")


def _references(x, wt, dy, stride, pad, g):
    xd, wd, dyd = x.double(), wt.double(), dy.double()
    y = F.conv2d(xd, wd, None, stride, pad, 1, g)
    ym = F.conv2d(xd.abs(), wd.abs(), None, stride, pad, 1, g)
    dx = torch.nn.grad.conv2d_input(x.shape, wd, dyd, stride, pad, 1, g)
    dxm = torch.nn.grad.conv2d_input(x.shape, wd.abs(), dyd.abs(), stride, pad, 1, g)
    dw = torch.nn.grad.conv2d_weight(xd, wt.shape, dyd, stride, pad, 1, g)
    dwm = torch.nn.grad.conv2d_weight(xd.abs(), wt.shape, dyd.abs(), stride, pad, 1, g)
    return (y, ym), (dx, dxm), (dw, dwm)


def _native(x, wt, dy, stride, pad, g, bias=None):
    xr = x.clone().requires_grad_(True)
    wr = wt.clone().requires_grad_(True)
    br = None if bias is None else bias.clone().requires_grad_(True)
    y = layers.ConvFunction.apply(xr, wr, br, stride, pad, g)
    y.backward(dy)
    return y.detach(), xr.grad, wr.grad, (None if br is None else br.grad)


def _run_bounds(shape, seed=0):
    n, c, k, kern, stride, pad, g, h, w = shape
    x, wt, dy = _inputs(shape, seed)
    y, dx, dw, _ = _native(x, wt, dy, stride, pad, g)
    (yr, ym), (dxr, dxm), (dwr, dwm) = _references(x, wt, dy, stride, pad, g)
    _check("y", y, yr, _bound(c // g * kern[0] * kern[1], ym))
    _check("dx", dx, dxr, _bound(k // g * kern[0] * kern[1], dxm))
    _check("dw", dw, dwr, _bound(n * dy.shape[2] * dy.shape[3], dwm))
    del yr, ym, dxr, dxm, dwr, dwm
    # the same outputs against float64 on the TF32-rounded operands, to the bound of the kernels' addition order
    depth = R.depths(shape)
    (yr, ym), (dxr, dxm), (dwr, dwm) = _references(_tf32(x), _tf32(wt), _tf32(dy), stride, pad, g)
    _check("y (order)", y, yr, R.order_bound(depth["fwd"], ym))
    _check("dx (order)", dx, dxr, R.order_bound(depth["data"], dxm))
    _check("dw (order)", dw, dwr, R.order_bound(depth["filter"], dwm))


@pytest.mark.parametrize("shape", NET_SHAPES)
def test_net_convolutions_within_the_tf32_bound(shape):
    b, cin, cout, kern, stride, pad, g, h, w = shape
    _run_bounds((b, cin, cout, kern, stride, pad, g, h, w))


@pytest.mark.parametrize("shape", RAGGED_SHAPES)
def test_ragged_convolutions_within_the_tf32_bound(shape):
    _run_bounds(shape, seed=1)


def test_fused_bias_and_its_gradient():
    shape = (3, 16, 24, (3, 3), (1, 1), (1, 1), 2, 13, 13)
    n, c, k, kern, stride, pad, g, h, w = shape
    x, wt, dy = _inputs(shape, 2)
    bias = torch.randn(k, device="cuda")
    y, _, _, db = _native(x, wt, dy, stride, pad, g, bias)
    (yr, ym), _, _ = _references(x, wt, dy, stride, pad, g)
    _check("y + bias", y, yr + bias.double().view(1, -1, 1, 1), _bound(c // g * 9, ym + bias.double().abs().view(
        1, -1, 1, 1)))
    torch.testing.assert_close(db.double(), dy.double().sum((0, 2, 3)), rtol=1e-5, atol=1e-5)


def test_cudnn_tf32_meets_the_same_bound():
    """The bound is not looser than what cuDNN's own TF32 convolutions reach on the same inputs."""
    was = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        for shape in [(8, 96, 256, (5, 5), (1, 1), (2, 2), 2, 27, 27), (8, 256, 384, (3, 3), (1, 1), (1, 1), 1, 13, 13)]:
            n, c, k, kern, stride, pad, g, h, w = shape
            x, wt, dy = _inputs(shape, 3)
            (yr, ym), _, _ = _references(x, wt, dy, stride, pad, g)
            _check("cuDNN y", F.conv2d(x, wt, None, stride, pad, 1, g), yr, _bound(c // g * kern[0] * kern[1], ym))
    finally:
        torch.backends.cudnn.allow_tf32 = was


@pytest.mark.parametrize("shape", [RAGGED[1], (16, 96, 256, (5, 5), (1, 1), (2, 2), 2, 27, 27),
                                   (16, 3, 96, (11, 11), (4, 4), (0, 0), 1, 227, 227)])
def test_repeatable_and_graph_replay_equals_eager(shape):
    n, c, k, kern, stride, pad, g, h, w = shape
    x, wt, dy = _inputs(shape, 4)
    a = _native(x, wt, dy, stride, pad, g)
    b = _native(x, wt, dy, stride, pad, g)
    for u, v in zip(a[:3], b[:3]):
        assert torch.equal(u, v)
    xs, ws, dys = x.clone(), wt.clone().requires_grad_(True), dy.clone()
    xs.requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        layers.ConvFunction.apply(xs, ws, None, stride, pad, g).backward(dys)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    xs.grad = ws.grad = None
    with torch.cuda.graph(graph):
        out = layers.ConvFunction.apply(xs, ws, None, stride, pad, g)
        out.backward(dys)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a[0]) and torch.equal(xs.grad, a[1]) and torch.equal(ws.grad, a[2])


def test_nan_and_inf_propagate():
    shape = (2, 8, 16, (3, 3), (1, 1), (1, 1), 1, 9, 9)
    n, c, k, kern, stride, pad, g, h, w = shape
    x, wt, dy = _inputs(shape, 5)
    x[0, 1, 4, 4] = float("nan")
    x[1, 2, 0, 0] = float("inf")
    dy[0, 3, 2, 2] = float("-inf")
    y, dx, dw, _ = _native(x, wt, dy, stride, pad, g)
    (yr, _), (dxr, _), (dwr, _) = _references(x, wt, dy, stride, pad, g)
    for name, got, ref in (("y", y, yr), ("dx", dx, dxr), ("dw", dw, dwr)):
        assert torch.equal(torch.isnan(got), torch.isnan(ref)), name
        fin = torch.isinf(ref)
        assert torch.equal(got[fin], ref[fin].float()), name


def _grads(mod, x, label):
    for p in mod.parameters():
        p.grad = None
    torch.nn.functional.cross_entropy(mod(x), label).backward()
    return [p.grad.detach().double().cpu() for p in mod.parameters()]


def test_caffenet_gradients_within_twice_cudnn_tf32(monkeypatch):
    torch.manual_seed(7)
    mod = nets.torch_module("caffenet")
    for m in mod.modules():
        if hasattr(m, "reset_parameters"):
            m.reset_parameters()
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    x = torch.rand((4,) + tuple(nets.NETS["caffenet"]["input"]))
    label = torch.randint(0, nets.NETS["caffenet"]["classes"], (4,))
    ref = _grads(mod.double(), x.double(), label)
    mod = mod.float().cuda()
    xc, lc = x.cuda(), label.cuda()
    was = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        native = _grads(mod, xc, lc)
        monkeypatch.setattr(layers, "native_conv", lambda *a: False)
        cudnn = _grads(mod, xc, lc)
    finally:
        torch.backends.cudnn.allow_tf32 = was
    for i, (r, a, b) in enumerate(zip(ref, native, cudnn)):
        scale = r.abs().max().item() + 1e-30
        ea, eb = (a - r).abs().max().item() / scale, (b - r).abs().max().item() / scale
        assert ea <= 2 * eb + 1e-6, f"blob {i}: native error {ea:.3g} against cuDNN TF32 {eb:.3g}"
