"""-m gpu: the BatchNorm kernels (csrc/batch_norm.cu) against the float64 references, bounds and fp32 restatement of
bn_ref.py, across the geometries they accept: every thread-group size PlaneGrid picks from H*W, channel counts past
the 128-channel blocks of the per-channel kernels, batches up to 256 and ResNet planes; the hyperparameters; NaN and
infinity containment; writes outside or missing from every buffer; bf16; and the device copy of powf_half.h on every
float."""
import numpy as np
import pytest
import torch

import bn_ref as B
import test_gpu_batch_norm as BN
import test_gpu_producer_graph_ops as G
from gpu_util import assert_bits_equal

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS, FRAC = BN.EPS, BN.FRAC
FILL32, FILL16 = 0x7fa5a5a5, 0x7fa5  # NaN payloads the kernels never produce
GUARD = 256  # elements on each side of every buffer

# H*W -> threads per plane: 1 -> 1, 2 -> 2, 3 and 4 -> 4, 5 and 8 -> 8, 9 and 16 -> 16, 17 ... 1024 -> 32,
# above 1024 the whole 256-thread block
SWEEP = [
    (2, 257, 1, 1), (256, 129, 1, 1), (7, 128, 1, 2), (32, 3, 3, 1), (2, 2048, 2, 2), (7, 255, 1, 5),
    (1, 256, 2, 4), (32, 127, 3, 3), (2, 1, 4, 4), (7, 129, 4, 4), (2, 257, 1, 17), (32, 3, 1, 31),
    (7, 256, 4, 8), (1, 129, 3, 11), (2, 255, 33, 31), (2, 3, 32, 32), (7, 129, 1, 1025), (1, 257, 56, 56),
    (2, 128, 112, 112), (256, 1, 112, 112), (256, 3, 4, 4), (1, 3, 1, 1), (1, 1, 1, 1),
    # ResNet-50's five BatchNorm planes at batch 32
    (32, 64, 112, 112), (32, 256, 56, 56), (32, 512, 28, 28), (32, 1024, 14, 14), (32, 2048, 7, 7),
    # resnet20 at batch 128, cifar10_full_bn at 100, the engine's 2-D bottom after an InnerProduct
    (128, 16, 32, 32), (128, 32, 16, 16), (128, 64, 8, 8), (100, 32, 16, 16), (100, 64, 8, 8), (256, 4096),
]


def _ids(shapes):
    return ["x".join(map(str, s)) for s in shapes]


def _hw(shape):
    return int(np.prod(shape[2:], dtype=np.int64)) if len(shape) > 2 else 1


def _geom(shape):
    n, c = shape[0], shape[1] if len(shape) > 1 else 1
    return n, c, _hw(shape), 1


def _blobs(rng, c):
    return (rng.standard_normal(c).astype(F32), (rng.random(c) * 10 + 1).astype(F32), F32([7.25]))


class Guarded:
    """A device buffer of n elements with GUARD elements on both sides, every element set to the fill pattern
    (or the interior to `init`)."""

    def __init__(self, n, dtype=torch.float32, init=None):
        self.int_dtype, self.fill = (torch.int32, FILL32) if dtype == torch.float32 else (torch.int16, FILL16)
        self.raw = torch.full((n + 2 * GUARD,), self.fill, dtype=self.int_dtype, device="cuda")
        self.t = self.raw[GUARD:GUARD + n].view(dtype)
        if init is not None:
            self.t.copy_(torch.as_tensor(np.ascontiguousarray(init).reshape(-1)).to(dtype))

    def ptr(self):
        return self.t.data_ptr()

    def guards_intact(self):
        return bool((self.raw[:GUARD] == self.fill).all()) and bool((self.raw[-GUARD:] == self.fill).all())

    def unwritten(self):
        return int((self.raw[GUARD:-GUARD] == self.fill).sum())

    def host(self):
        return self.t.float().cpu().numpy()


def run_raw(x, dy, blobs, global_stats=False, f=FRAC, eps=EPS, dtype=torch.float32):
    """Forward then backward through the raw cos_batch_norm_* entries on guarded buffers -> dict of numpy results
    (fp32; bf16 y and dx upcast) and the Guarded buffers themselves under "buf"."""
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    sfx = "" if dtype == torch.float32 else "_bf16"
    shape = x.shape
    n, c, h, w = _geom(shape)
    size = x.size
    bx, bdy = Guarded(size, dtype, x), Guarded(size, dtype, dy)
    by, bdx = Guarded(size, dtype), Guarded(size, dtype)
    bm, bv, bs = (Guarded(b.size, torch.float32, b) for b in blobs)
    save = Guarded(2 * c)
    wf, wb = Guarded(2 * (n + 1) * c), Guarded(2 * (n + 1) * c)
    st = torch.cuda.current_stream().cuda_stream
    assert getattr(L, "cos_batch_norm_forward" + sfx)(bx.ptr(), by.ptr(), bm.ptr(), bv.ptr(), bs.ptr(), save.ptr(),
                                                      wf.ptr(), n, c, h, w, int(global_stats), f, eps, st), \
        L.cos_last_error()
    assert getattr(L, "cos_batch_norm_backward" + sfx)(bx.ptr(), bdy.ptr(), bdx.ptr(), save.ptr(), wb.ptr(), n, c, h,
                                                       w, int(global_stats), eps, st), L.cos_last_error()
    torch.cuda.synchronize()
    sums = wb.host()[2 * n * c:]
    return dict(y=by.host().reshape(shape), dx=bdx.host().reshape(shape), save=save.host(),
                mean=save.host()[:c], var=save.host()[c:], s1=sums[:c], s2=sums[c:],
                blobs=tuple(b.host() for b in (bm, bv, bs)),
                buf=dict(x=bx, dy=bdy, y=by, dx=bdx, mean_blob=bm, var_blob=bv, scale=bs, save=save, work_fwd=wf,
                         work_bwd=wb))


def _check_within(x, dy, mean, var, y, dx, eps, what):
    """mean, var, y against the float64 forward and dx against the float64 backward from the saved statistics,
    each within bn_ref's bounds"""
    y64, mean64, var64 = B.reference(x, eps)
    dm = B.mean_bound(x)
    dv = B.var_bound(x, var64, dm)
    for name, got, want, bound in (("mean", mean, mean64, dm), ("var", var, var64, dv),
                                   ("y", y, y64, B.y_bound(y64, var64, eps, dm, dv)),
                                   ("dx", dx, B.reference_backward(x, dy, mean, var, eps),
                                    B.dx_bound(x, dy, mean, var, eps))):
        bad = B.outside(got, want, bound)
        if bad.any():
            i = np.unravel_index(np.argmax(bad), bad.shape)
            raise AssertionError(f"{what}: {name} outside the bound on {int(bad.sum())} of {bad.size}; first at {i}: "
                                 f"{got[i]!r} vs {want[i]!r} +- {np.broadcast_to(bound, bad.shape)[i]!r}")


def _check_exact_given_stats(x, blobs, mean, var, y, nb, eps, f, what):
    """y from the saved statistics (libm powf) and the three blob updates from them, bit for bit"""
    wy, _, _, _ = B.restate_forward(x, blobs, f=f, eps=eps, stats=(mean, var))
    assert_bits_equal(y, wy, f"{what}: y from the saved statistics")
    m = x.size // B.planes(x).shape[1]
    corr = F32(m) / F32(m - 1) if m > 1 else F32(1)
    ff = F32(f)
    want = (mean + ff * blobs[0], corr * var + ff * blobs[1], blobs[2] * ff + F32(1))
    for k, name in enumerate(("mean blob", "variance blob", "scale factor")):
        assert_bits_equal(nb[k], want[k], f"{what}: {name}")


# ------------------------------------------------------------------ 1. geometry sweep, two input families

@pytest.mark.parametrize("family", ["dyadic", "gaussian"])
@pytest.mark.parametrize("shape", SWEEP, ids=_ids(SWEEP))
def test_geometry_sweep(cos, shape, family):
    rng = np.random.default_rng(sum(shape) + (family == "gaussian"))
    x, dy = B.dyadic(rng, shape) if family == "dyadic" else B.gaussian(rng, shape)
    c = shape[1] if len(shape) > 1 else 1
    blobs = _blobs(rng, c)
    y, save, nb, dx = BN.run_native(x, blobs, False, dy)
    y, dx, save = y.detach().cpu().numpy(), dx.cpu().numpy(), save.cpu().numpy()
    mean, var = save[:c], save[c:]
    what = f"{shape} {family}"
    _check_exact_given_stats(x, blobs, mean, var, y, nb, EPS, FRAC, what)
    if family == "dyadic":  # every sum exact: the statistics, the blobs and S1 equal the restatement
        _, wmean, wvar, wblobs = B.restate_forward(x, blobs)
        assert_bits_equal(mean, wmean, f"{what}: mean")
        assert_bits_equal(var, wvar, f"{what}: var")
        for k in range(3):
            assert_bits_equal(nb[k], wblobs[k], f"{what}: blob {k}")
        r = run_raw(x, dy, blobs)
        _, ws1, _ = B.restate_backward(x, dy, mean, var)
        assert_bits_equal(r["s1"], ws1, f"{what}: S1")
        assert_bits_equal(r["dx"], dx, f"{what}: dx of the raw entry = dx through BatchNormFunction")
    _check_within(x, dy, mean, var, y, dx, EPS, what)


# ------------------------------------------------------------------ 2. hyperparameters

HYPER_SHAPES = [(7, 129, 3, 3), (2, 257, 33, 33)]


@pytest.mark.parametrize("f", [0.0, 0.999, 1.0])
@pytest.mark.parametrize("eps", [0.0, 1e-5, 1e-3])
@pytest.mark.parametrize("shape", HYPER_SHAPES, ids=_ids(HYPER_SHAPES))
def test_eps_and_moving_average_fraction(cos, shape, eps, f):
    rng = np.random.default_rng(sum(shape))
    x, dy = B.gaussian(rng, shape, constant=eps > 0)  # eps = 0 needs var > 0
    blobs = _blobs(rng, shape[1])
    r = run_raw(x, dy, blobs, f=f, eps=eps)
    what = f"{shape} eps {eps} f {f}"
    _check_exact_given_stats(x, blobs, r["mean"], r["var"], r["y"], r["blobs"], eps, f, what)
    _check_within(x, dy, r["mean"], r["var"], r["y"], r["dx"], eps, what)


GLOBAL_SHAPES = [(3, 129, 1, 1), (3, 129, 1, 2), (3, 129, 3, 1), (3, 129, 2, 4), (3, 129, 3, 3), (3, 129, 4, 4),
                 (3, 129, 1, 17), (3, 257, 33, 31), (2, 257, 1, 1025), (2, 2048, 7, 7), (4, 300)]


@pytest.mark.parametrize("s", [7.25, 0.0], ids=["s7.25", "s0"])
@pytest.mark.parametrize("shape", GLOBAL_SHAPES, ids=_ids(GLOBAL_SHAPES))
def test_global_stats_bit_exact(cos, shape, s):
    rng = np.random.default_rng(sum(shape))
    x, dy = B.gaussian(rng, shape)
    mb, vb, _ = _blobs(rng, shape[1])
    blobs = (mb, vb, F32([s]))
    r = run_raw(x, dy, blobs, global_stats=True)
    what = f"{shape} global s={s}"
    for k in range(3):
        assert_bits_equal(r["blobs"][k], blobs[k], f"{what}: blob {k} untouched")
    sf = F32(0) if s == 0 else F32(1) / F32(s)
    mean, var = sf * mb, sf * vb
    assert_bits_equal(r["save"], np.concatenate([mean, var]), f"{what}: saved statistics")
    wy, _, _, _ = B.restate_forward(x, blobs, global_stats=True)
    assert_bits_equal(r["y"], wy, f"{what}: y")
    wdx, _, _ = B.restate_backward(x, dy, mean, var, global_stats=True)
    assert_bits_equal(r["dx"], wdx, f"{what}: dx")


# ------------------------------------------------------------------ 3. NaN / Inf containment

POISON_HW = [(1, 1), (1, 2), (3, 1), (2, 2), (1, 5), (2, 4), (3, 3), (4, 4), (32, 64)]  # groups 1 ... 16 and 256
POISON = [("x", (np.nan,)), ("x", (np.inf,)), ("x", (-np.inf, np.inf)), ("dy", (np.nan,)), ("dy", (np.inf,)),
          ("dy", (-np.inf, np.nan))]


def _classes(a):
    a = np.asarray(a, np.float64)
    return np.select([np.isnan(a), np.isposinf(a), np.isneginf(a)], [1, 2, 3], 0)


@pytest.mark.parametrize("where,values", POISON, ids=[f"{w}-{'_'.join(map(str, v))}" for w, v in POISON])
@pytest.mark.parametrize("hw", POISON_HW, ids=[f"{h}x{w}" for h, w in POISON_HW])
def test_non_finite_values_stay_in_their_channel(cos, hw, where, values):
    """Channel 3 of 7 gets the non-finite values; with H*W <= 16 several of its planes share a warp with other
    channels' planes.  Channel 3's y, dx and blobs have the float64 reference's classes (NaN, +inf, -inf, finite);
    every other channel is bit-identical to a run without them."""
    shape = (3, 7) + hw
    rng = np.random.default_rng(sum(shape) + len(values))
    x, dy = B.gaussian(rng, shape)
    blobs = _blobs(rng, 7)
    clean = run_raw(x, dy, blobs)
    px, pdy = x.copy(), dy.copy()
    target = px if where == "x" else pdy
    pos = rng.choice(3 * _hw(shape), size=len(values), replace=False)
    for p, v in zip(pos, values):
        target[p // _hw(shape), 3].reshape(-1)[p % _hw(shape)] = v
    r = run_raw(px, pdy, blobs)
    others = [ch for ch in range(7) if ch != 3]
    for name in ("y", "dx"):
        assert_bits_equal(r[name][:, others], clean[name][:, others], f"{name} of the other channels")
    for k in range(2):
        assert_bits_equal(r["blobs"][k][others], clean["blobs"][k][others], f"blob {k} of the other channels")
    assert_bits_equal(r["blobs"][2], clean["blobs"][2], "scale factor")
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        y64, mean64, var64, nb64 = B.numpy_bn_forward(px, blobs[0].astype(np.float64), blobs[1].astype(np.float64),
                                                      float(blobs[2][0]))
        dx64 = B.numpy_bn_backward(px, pdy, mean64, var64)
    assert np.array_equal(_classes(r["y"][:, 3]), _classes(y64[:, 3])), "y classes of the poisoned channel"
    assert np.array_equal(_classes(r["dx"][:, 3]), _classes(dx64[:, 3])), "dx classes of the poisoned channel"
    for k in range(2):
        assert _classes(r["blobs"][k][3]) == _classes(nb64[k][3]), f"blob {k} class of the poisoned channel"
    if where == "x":
        assert not np.isfinite(r["y"][:, 3]).any()


# ------------------------------------------------------------------ 4. nothing written out of bounds or left unwritten

GUARD_SHAPES = [(3, 129, 1, 1), (2, 257, 3, 3), (2, 5, 33, 31), (1, 3, 1, 1025), (7, 130, 4, 4), (5, 33)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("global_stats", [False, True], ids=["batch", "global"])
@pytest.mark.parametrize("shape", GUARD_SHAPES, ids=_ids(GUARD_SHAPES))
def test_guards_untouched_and_outputs_fully_written(cos, shape, global_stats, dtype):
    rng = np.random.default_rng(sum(shape))
    x, dy = B.gaussian(rng, shape)
    blobs = _blobs(rng, shape[1])
    r = run_raw(x, dy, blobs, global_stats=global_stats, dtype=dtype)
    for name, b in r["buf"].items():
        assert b.guards_intact(), f"{name}: a guard element was written"
    for name in ("y", "dx", "save"):
        assert r["buf"][name].unwritten() == 0, f"{name}: elements still hold the fill value"
    if global_stats:
        for k in range(3):
            assert_bits_equal(r["blobs"][k], blobs[k], f"blob {k} unchanged")
    else:
        for k in range(3):
            assert np.isfinite(r["blobs"][k]).all(), f"blob {k} written"


# ------------------------------------------------------------------ 5. bf16

BF16_SHAPES = [(4, 129, 1, 1), (4, 129, 1, 2), (4, 129, 1, 3), (4, 129, 2, 4), (4, 129, 3, 3), (4, 129, 4, 4),
               (4, 129, 5, 5), (2, 129, 33, 31), (2, 129, 48, 48), (8, 2048, 7, 7), (2, 2048, 1, 1)]


@pytest.mark.parametrize("global_stats", [False, True], ids=["batch", "global"])
@pytest.mark.parametrize("shape", BF16_SHAPES, ids=_ids(BF16_SHAPES))
def test_bf16_is_the_fp32_kernel_on_upcast_inputs(cos, shape, global_stats):
    rng = np.random.default_rng(sum(shape))
    x, dy = B.gaussian(rng, shape)
    xb = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    dyb = torch.from_numpy(dy).to(torch.bfloat16).float().numpy()
    blobs = _blobs(rng, shape[1])
    r32 = run_raw(xb, dyb, blobs, global_stats)
    r16 = run_raw(xb, dyb, blobs, global_stats, dtype=torch.bfloat16)
    for name in ("y", "dx"):
        got = r16["buf"][name].t.view(torch.int16).cpu()
        want = r32["buf"][name].t.to(torch.bfloat16).view(torch.int16).cpu()
        assert torch.equal(got, want), f"bf16 {name} != fp32 {name} rounded once"
    assert_bits_equal(r16["save"], r32["save"], "saved statistics")
    for k in range(3):
        assert_bits_equal(r16["blobs"][k], r32["blobs"][k], f"blob {k}")


# ------------------------------------------------------------------ 6. the device powf_half on every float

POWF_CHUNK = 1 << 24
LAST_FINITE = 0x7f7fffff


def _powf_launch(L, x, var, scale, save, work, y, dx, c):
    st = torch.cuda.current_stream().cuda_stream
    mean = torch.zeros(c, dtype=torch.float32, device="cuda")
    assert L.cos_batch_norm_forward(x.data_ptr(), y.data_ptr(), mean.data_ptr(), var.data_ptr(), scale.data_ptr(),
                                    save.data_ptr(), work.data_ptr(), 1, c, 1, 1, 1, 1.0, 0.0, st), L.cos_last_error()
    assert L.cos_batch_norm_backward(x.data_ptr(), x.data_ptr(), dx.data_ptr(), save.data_ptr(), work.data_ptr(), 1,
                                     c, 1, 1, 1, 0.0, st), L.cos_last_error()


def test_device_powf_half_matches_glibc_on_every_float(cos):
    """One channel per float bit pattern v: N = H = W = 1, global statistics with scale factor 1, mean blob 0,
    eps 0, var blob v and x = glibc powf(v, 0.5f).  y = x / sd is exactly 1.0 iff the kernel's cos_powf_half(v)
    equals glibc's (two adjacent floats never divide to 1.0); the global backward with dy = x checks the second
    inlined copy the same way.  128 launches of 2^24 channels cover 0x00000001 ... 0x7f7fffff; +0, -0, +inf, NaN
    and a negative value are checked by class."""
    from caffeonspark_b200 import _lib
    from oracle import adam
    adam.build()
    L = _lib.lib()
    c = POWF_CHUNK
    scale = torch.ones(1, dtype=torch.float32, device="cuda")
    save = torch.empty(2 * c, dtype=torch.float32, device="cuda")
    work = torch.empty(4 * c, dtype=torch.float32, device="cuda")
    y, dx = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    host = torch.empty(c, dtype=torch.float32).pin_memory()
    xd = torch.empty(c, dtype=torch.float32, device="cuda")
    bad_y = bad_dx = checked = 0
    first = []
    for lo in range(0, 1 << 31, c):
        adam.powf_half_fill(lo, lo + c, host.numpy())
        xd.copy_(host, non_blocking=True)
        bits = torch.arange(lo, lo + c, dtype=torch.int64, device="cuda")
        var = bits.to(torch.int32).view(torch.float32)
        _powf_launch(L, xd, var, scale, save, work, y, dx, c)
        valid = (bits >= 1) & (bits <= LAST_FINITE)
        wy, wdx = valid & (y != 1.0), valid & (dx != 1.0)
        bad_y += int(wy.sum())
        bad_dx += int(wdx.sum())
        checked += int(valid.sum())
        if len(first) < 8 and bool((wy | wdx).any()):
            first += [hex(int(b)) for b in bits[wy | wdx][:8].cpu()]
    print(f"device cos_powf_half vs glibc powf(v, 0.5f): {bad_y} mismatches in the forward's copy, {bad_dx} in the "
          f"global backward's, over {checked} patterns 0x00000001 ... 0x7f7fffff")
    assert checked == LAST_FINITE
    assert bad_y == 0 and bad_dx == 0, first
    # the special classes: v = +0 and -0 give sd = +0 (1 / sd = +inf), +inf gives sd = +inf (3e38 / sd = 0), NaN and
    # negative v give NaN
    v = np.array([0.0, -0.0, np.inf, np.nan, -1.0], F32)
    xs = np.array([1.0, 1.0, 3e38, 1.0, 1.0], F32)
    k = v.size
    out = [torch.empty(k, device="cuda") for _ in range(2)]
    _powf_launch(L, torch.from_numpy(xs).cuda(), torch.from_numpy(v).cuda(), scale,
                 torch.empty(2 * k, device="cuda"), torch.empty(4 * k, device="cuda"), out[0], out[1], k)
    for o in out:
        o = o.cpu().numpy()
        assert o[0] == np.inf and o[1] == np.inf and o[2] == 0 and np.isnan(o[3]) and np.isnan(o[4]), o


# ------------------------------------------------------------------ 7. the built-in engine past one channel block

@pytest.mark.parametrize("global_stats", [False, True], ids=["batch", "global"])
def test_engine_batch_norm_257_channels_batch_33(cos, tmp_path, global_stats):
    G.test_batch_norm(cos, tmp_path, (33, 257, 3, 3), global_stats, False)
