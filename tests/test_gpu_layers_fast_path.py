"""GPU tests of the staged bias+ReLU+max-pool kernels (the fast path of csrc/caffe_layers.cu) against the per-element
reference kernels, forced with cos_layers_set_reference_kernels(1): y, index, dx, dbias and the bias gradient's
per-plane partials must be bit-identical, in fp32 and bf16, at CaffeNet b256's and CIFAR-10-quick's exact shapes and at
ragged ones, on inputs with ties, NaN, +-Inf, -0.0 and subnormals.  A fast-path forward/backward is also captured
into a CUDA graph and replayed."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from caffeonspark_b200 import _lib  # noqa: E402

# (N, C, H, W) of the bias-free conv output, pool kernel, stride
CASES = {
    "caffenet_conv1_b256": ((256, 96, 55, 55), 3, 2),
    "caffenet_conv2_b256": ((256, 256, 27, 27), 3, 2),
    "caffenet_conv5_b256": ((256, 256, 13, 13), 3, 2),
    "cifar10_quick_conv1_b100": ((100, 32, 32, 32), 3, 2),  # 32 -> 16: the last window is clipped
    "lenet_pool_k2s2": ((64, 20, 24, 24), 2, 2),
    "ragged_17x23": ((3, 5, 17, 23), 3, 2),  # odd planes, both last windows clipped, tail block of planes
    "ragged_hw33": ((7, 3, 3, 11), 3, 2),  # backward block 64 with two passes per thread, 3 planes per block
    "ragged_hw257": ((3, 3, 257, 3), 3, 2),  # backward block 256, a partial second pass
    "planes_tail": ((1, 37, 13, 13), 3, 2),  # 37 planes: the last block of both kernels is partly empty
    "batch_300_c33": ((300, 33, 13, 13), 3, 2),  # the bias gradient: 3 row passes, a ragged channel block
    "k2s1": ((2, 3, 9, 7), 2, 1),
    "k3s1": ((2, 3, 9, 10), 3, 1),
    "k4s3": ((2, 3, 10, 11), 4, 3),
    "k5s3_clipped": ((2, 3, 13, 12), 5, 3),
    "k2s3_gaps": ((2, 3, 9, 8), 2, 3),
    "k3s3": ((2, 3, 14, 9), 3, 3),
    "plane_near_smem_limit": ((2, 2, 90, 100), 3, 2),  # one plane per block in both directions
}
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    ne = (_bits(a) != _bits(b)).nonzero()
    assert ne.numel() == 0, f"{what}: {ne.shape[0]} elements differ, first at {ne[0].tolist()}"


def _specials(t, g, frac=0.01):
    """NaN, +-Inf, -0.0, +0.0 and +-subnormals at random positions of t (in place)"""
    vals = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 0.0, 1e-40, -1e-40, 3e-45],
                        device="cuda")
    m = torch.rand(t.shape, device="cuda", generator=g) < frac
    pick = torch.randint(0, vals.numel(), t.shape, device="cuda", generator=g)
    t[m] = vals[pick][m]
    return t


def _inputs(shape, k, s, seed, kind):
    n, c, h, w = shape
    ph, pw = (h - k + s - 1) // s + 1, (w - k + s - 1) // s + 1
    ph -= (ph - 1) * s >= h
    pw -= (pw - 1) * s >= w
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    dy = torch.randn((n, c, ph, pw), device="cuda", generator=g)
    b = 0.3 * torch.randn(c, device="cuda", generator=g)
    if kind == "ties":  # equal values and exact zeros: first maximum wins, the <= 0 cut, dy sums that tie
        x, dy, b = torch.round(x * 2), torch.round(dy * 2), torch.zeros_like(b)
    elif kind == "specials":
        x, dy = _specials(x, g), _specials(dy, g)
        b[::3] = 0.0  # subnormal x + 0 stays subnormal
    return x, b, dy, (ph, pw)


def _run(L, dtype, x, b, dy, index_in, shape, k, s, ph, pw, reference):
    """forward and backward on one path; the backward reads index_in (the same for both paths) when given"""
    n, c, h, w = shape
    sfx = "" if dtype == torch.float32 else "_bf16"
    stream = torch.cuda.current_stream().cuda_stream
    L.cos_layers_set_reference_kernels(1 if reference else 0)
    try:
        assert L.cos_layers_reference_kernels() == (1 if reference else 0)
        xt, dyt = x.to(dtype), dy.to(dtype)
        y = torch.full((n, c, ph, pw), 7, device="cuda", dtype=dtype)
        index = torch.full((n, c, ph, pw), 77, device="cuda", dtype=torch.uint8)
        dx = torch.full(shape, 7, device="cuda", dtype=dtype)
        partials = torch.full((n * c,), 7.0, device="cuda")
        dbias = torch.full((c,), 7.0, device="cuda")
        assert getattr(L, "cos_bias_relu_maxpool_forward" + sfx)(
            xt.data_ptr(), b.data_ptr(), y.data_ptr(), index.data_ptr(), n, c, h, w, k, s, ph, pw, stream), \
            L.cos_last_error()
        idx = index if index_in is None else index_in
        assert getattr(L, "cos_bias_relu_maxpool_backward" + sfx)(
            dyt.data_ptr(), idx.data_ptr(), dx.data_ptr(), partials.data_ptr(), dbias.data_ptr(), n, c, h, w, k, s,
            ph, pw, stream), L.cos_last_error()
        torch.cuda.synchronize()
    finally:
        L.cos_layers_set_reference_kernels(0)
    return dict(y=y, index=index, dx=dx, partials=partials, dbias=dbias)


# every case, input kind and dtype, except the full-batch CaffeNet shapes, which run every kind in fp32 and random
# inputs in bf16 (each of those moves several hundred MB per call)
PARAMS = [(case, kind, dtype) for case in CASES for kind in ("random", "ties", "specials") for dtype in DTYPES
          if CASES[case][0][0] != 256 or dtype == "fp32" or kind == "random"]


@pytest.mark.parametrize("case,kind,dtype", PARAMS)
def test_staged_pool_is_bit_identical_to_reference(cos, case, kind, dtype):
    L = _lib.lib()
    shape, k, s = CASES[case]
    assert L.cos_pool_fast_path(*shape, k, s) == 1, "this case must exercise the staged kernels"
    x, b, dy, (ph, pw) = _inputs(shape, k, s, seed=sum(map(ord, case + kind)), kind=kind)
    dt = DTYPES[dtype]
    ref = _run(L, dt, x, b, dy, None, shape, k, s, ph, pw, reference=True)
    fast = _run(L, dt, x, b, dy, None, shape, k, s, ph, pw, reference=False)
    for name in ("y", "index", "dx", "partials", "dbias"):
        _same(fast[name], ref[name], f"{case} {kind} {dtype}: {name}")
    # the backward alone on an index that points anywhere in (or past) its window, or nowhere
    g = torch.Generator(device="cuda").manual_seed(11)
    rnd = torch.randint(0, k * k + 1, ref["index"].shape, device="cuda", generator=g).to(torch.uint8)
    rnd[rnd == k * k] = 255
    ref = _run(L, dt, x, b, dy, rnd, shape, k, s, ph, pw, reference=True)
    fast = _run(L, dt, x, b, dy, rnd, shape, k, s, ph, pw, reference=False)
    for name in ("dx", "partials", "dbias"):
        _same(fast[name], ref[name], f"{case} {kind} {dtype} random index: {name}")


# geometries the staged pool kernels do not take: the switch still selects the bias gradient's second pass
FALLBACK = {"k1s1": ((2, 3, 5, 6), 1, 1), "k7s2": ((3, 5, 15, 16), 7, 2), "large_plane": ((2, 3, 130, 140), 3, 2),
            "batch_131_k4s1": ((131, 40, 9, 9), 4, 1)}


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("case", list(FALLBACK))
def test_fallback_geometries_are_bit_identical(cos, case, dtype):
    L = _lib.lib()
    shape, k, s = FALLBACK[case]
    assert L.cos_pool_fast_path(*shape, k, s) == 0
    x, b, dy, (ph, pw) = _inputs(shape, k, s, seed=sum(map(ord, case)), kind="specials")
    ref = _run(L, DTYPES[dtype], x, b, dy, None, shape, k, s, ph, pw, reference=True)
    fast = _run(L, DTYPES[dtype], x, b, dy, None, shape, k, s, ph, pw, reference=False)
    for name in ("y", "index", "dx", "partials", "dbias"):
        _same(fast[name], ref[name], f"{case} {dtype}: {name}")


def test_reference_switch_round_trips(cos):
    L = _lib.lib()
    was = L.cos_layers_reference_kernels()
    try:
        L.cos_layers_set_reference_kernels(1)
        assert L.cos_layers_reference_kernels() == 1
        L.cos_layers_set_reference_kernels(0)
        assert L.cos_layers_reference_kernels() == 0
    finally:
        L.cos_layers_set_reference_kernels(was)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_staged_pool_is_graph_capturable(cos, dtype):
    L = _lib.lib()
    shape, k, s = CASES["caffenet_conv2_b256"]
    n, c, h, w = shape
    x, b, dy, (ph, pw) = _inputs(shape, k, s, seed=5, kind="random")
    dt = DTYPES[dtype]
    ref = _run(L, dt, x, b, dy, None, shape, k, s, ph, pw, reference=True)
    sfx = "" if dt == torch.float32 else "_bf16"
    xt, dyt = x.to(dt), dy.to(dt)
    y = torch.empty((n, c, ph, pw), device="cuda", dtype=dt)
    index = torch.empty((n, c, ph, pw), device="cuda", dtype=torch.uint8)
    dx, partials, dbias = torch.empty(shape, device="cuda", dtype=dt), torch.empty(n * c, device="cuda"), \
        torch.empty(c, device="cuda")
    assert L.cos_layers_reference_kernels() == 0
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        st = torch.cuda.current_stream().cuda_stream
        assert getattr(L, "cos_bias_relu_maxpool_forward" + sfx)(
            xt.data_ptr(), b.data_ptr(), y.data_ptr(), index.data_ptr(), n, c, h, w, k, s, ph, pw, st)
        assert getattr(L, "cos_bias_relu_maxpool_backward" + sfx)(
            dyt.data_ptr(), index.data_ptr(), dx.data_ptr(), partials.data_ptr(), dbias.data_ptr(), n, c, h, w, k,
            s, ph, pw, st)
    for _ in range(2):
        for t in (y, dx, partials, dbias):
            t.fill_(3)
        index.fill_(3)
        graph.replay()
        torch.cuda.synchronize()
        got = dict(y=y, index=index, dx=dx, partials=partials, dbias=dbias)
        for name in got:
            _same(got[name], ref[name], f"graph replay {dtype}: {name}")
