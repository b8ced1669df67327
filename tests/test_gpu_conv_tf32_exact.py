"""The native TF32 convolutions (csrc/conv_tf32.cu, DESIGN.md section 10.2) held to exact answers on the GPU.

On dyadic operands whose magnitude sums stay under 2^22 product units (tests/conv_tf32_ref.py says why), every
partial sum is exact in fp32 whatever the kernel's order, so y, y + bias, dx and dw must equal the float64 answer
element for element.  The cases are every convolution of CaffeNet, LeNet and CIFAR-10-quick (own batch and 1 to 4),
the ragged shapes and the edges of conv_tf32_ref.EDGES: one, two and three tap-table segments, both tile variants
of every pass with M and N one off the tile, weight-gradient splits of one chunk, of nkt / 8 chunks with a short last
chunk and CaffeNet conv1 b256's 341, stride over kernel, pad over kernel, groups 1 to 4 with odd group sizes and a
1 x 1 image.  Each case runs two operand families ('small' integers everywhere, and one tensor odd 11-bit against
ternary ones) through layers.ConvFunction and through the raw entry points; the raw calls write into NaN-poisoned
outputs and workspace with guard words on both sides, so a missed element or a stray write fails the case, and the
inputs are checked unchanged.

Two assumptions are tested rather than taken: the K = 1 probes pin each operand's rounding to cvt.rna.tf32.f32
(conv_tf32_ref.tf32_rna) bit for bit on every pass, and cuDNN's TF32 forward on two strided dyadic cases is exact
too (if it were not, the exactness precondition would be wrong, not the kernels)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_tf32_ref as R
from caffeonspark_b200 import _lib, layers

pytestmark = pytest.mark.gpu

CASES = [pytest.param(i, shape, id=cid) for i, (cid, shape) in enumerate(R.EXACT_CASES)]
CASE_INDEX = {cid: i for i, (cid, _) in enumerate(R.EXACT_CASES)}

GUARD = 4096  # guard words on each side of an output
GUARD_BITS = 0x5A5A5A5A  # a finite float no result here takes
POISON_BITS = 0x7FC0DEAD  # a quiet NaN: no finite operands produce it


class _Arena:
    """`count` fp32 words poisoned with NaN, between two guards of GUARD_BITS, in one allocation."""

    def __init__(self, count):
        self.count = count
        self.bits = torch.full((count + 2 * GUARD,), GUARD_BITS, dtype=torch.int32, device="cuda")
        self.bits[GUARD:GUARD + count] = POISON_BITS
        self.body = self.bits[GUARD:GUARD + count].view(torch.float32)

    def ptr(self):
        return self.bits.data_ptr() + 4 * GUARD

    def check(self, name):
        for side, g in (("before", self.bits[:GUARD]), ("after", self.bits[GUARD + self.count:])):
            changed = int((g != GUARD_BITS).sum())
            assert changed == 0, f"{name}: {changed} guard words {side} the output were written"
        left = int(torch.isnan(self.body).sum())
        assert left == 0, f"{name}: {left} of {self.count} elements never written (or NaN)"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc):
    assert rc, _lib.lib().cos_last_error().decode()


def _raw(shape, x, w, dy, bias=None, passes=("y", "dx", "dw")):
    """{pass: output} from the raw entry points, each output and the weight-gradient workspace in its own _Arena,
    checked for coverage and containment; the inputs must come back unchanged."""
    L = _lib.lib()
    geom = R.geom12(shape)
    ins = {"x": x, "w": w, "dy": dy, "bias": bias}
    kept = {name: t.clone() for name, t in ins.items() if t is not None}
    out = {}
    if "y" in passes:
        out["y"] = _Arena(dy.numel())
        _ok(L.cos_conv_forward(x.data_ptr(), w.data_ptr(), None if bias is None else bias.data_ptr(),
                               out["y"].ptr(), *geom, _stream()))
    if "dx" in passes:
        out["dx"] = _Arena(x.numel())
        _ok(L.cos_conv_backward_data(dy.data_ptr(), w.data_ptr(), out["dx"].ptr(), *geom, _stream()))
    if "dw" in passes:
        out["dw"], out["workspace"] = _Arena(w.numel()), _Arena(L.cos_conv_workspace_floats(*geom))
        _ok(L.cos_conv_backward_filter(x.data_ptr(), dy.data_ptr(), out["dw"].ptr(), out["workspace"].ptr(), *geom,
                                       _stream()))
    torch.cuda.synchronize()
    for name, a in out.items():
        a.check(name)
    for name, k in kept.items():
        assert torch.equal(ins[name].view(torch.int32), k.view(torch.int32)), f"{name} was modified"
    like = {"y": dy, "dx": x, "dw": w}
    return {p: out[p].body.view(like[p].shape) for p in passes}


@pytest.fixture(autouse=True, scope="module")
def _release_cached_memory():
    """The float64 references of the batch-256 cases take gigabytes of PyTorch's caching allocator.  Hand them back to
    the driver when the module ends, so that later tests in the same process find the device as free as before (the
    in-process two-rank runs allocate device memory while a peer's kernel spins waiting for them)."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _exact(shape, ints, exps):
    """The float64 answers (exact on these operands), after checking the precondition exactly: the magnitude sums,
    the same convolutions of the integers' absolute values, stay under the ceiling."""
    n, c, k, kern, stride, pad, g, h, w = shape
    A = {t: v.abs().cuda() for t, v in ints.items()}
    mags = {"fwd": float(F.conv2d(A["x"], A["w"], None, stride, pad, 1, g).max() + A["bias"].max()),
            "data": float(torch.nn.grad.conv2d_input(A["x"].shape, A["w"], A["dy"], stride, pad, 1, g).max()),
            "filter": float(torch.nn.grad.conv2d_weight(A["x"], A["w"].shape, A["dy"], stride, pad, 1, g).max())}
    del A
    for ps, m in mags.items():
        assert m <= R.CEILING, f"{ps}: magnitude sum {m:.0f} units is above the exact ceiling"
    V = {t: v.cuda() * 2.0 ** exps[t] for t, v in ints.items()}
    y = F.conv2d(V["x"], V["w"], None, stride, pad, 1, g)
    dx = torch.nn.grad.conv2d_input(V["x"].shape, V["w"], V["dy"], stride, pad, 1, g)
    dw = torch.nn.grad.conv2d_weight(V["x"], V["w"].shape, V["dy"], stride, pad, 1, g)
    return y, y + V["bias"].view(1, -1, 1, 1), dx, dw


def _equal(name, got, ref):
    bad = got.double() != ref
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ from the exact answer, "
                             f"first at {i}: {float(got[i])!r} against {float(ref[i])!r}")


@pytest.mark.parametrize("family", R.FAMILIES)
@pytest.mark.parametrize("index, shape", CASES)
def test_exact_on_dyadic_operands(index, shape, family):
    n, c, k, kern, stride, pad, g, h, w = shape
    print(R.describe(shape))
    ints, exps = R.operands(shape, family, index)
    ref_y, ref_yb, ref_dx, ref_dw = _exact(shape, ints, exps)
    v = {t: a.cuda() for t, a in R.as_values(ints, exps).items()}

    got = _raw(shape, v["x"], v["w"], v["dy"])
    _equal("raw y", got["y"], ref_y)
    _equal("raw dx", got["dx"], ref_dx)
    _equal("raw dw", got["dw"], ref_dw)
    got = _raw(shape, v["x"], v["w"], v["dy"], v["bias"], passes=("y",))
    _equal("raw y + bias", got["y"], ref_yb)
    del got

    xr, wr, br = (v[t].clone().requires_grad_(True) for t in ("x", "w", "bias"))
    out = layers.ConvFunction.apply(xr, wr, br, stride, pad, g)
    out.backward(v["dy"])
    _equal("ConvFunction y + bias", out.detach(), ref_yb)
    _equal("ConvFunction dx", xr.grad, ref_dx)
    _equal("ConvFunction dw", wr.grad, ref_dw)


# --------------------------------------------------------------------------- operand rounding, K = 1
def _normal_bits(rng, count):
    """Random normal fp32 bit patterns, a quarter of them ties (the 13 dropped bits exactly 0x1000) and a quarter
    one ulp either side of a tie, without those whose rounding carries past the largest finite float."""
    bits = (rng.integers(0, 2, count, dtype=np.uint32) << np.uint32(31)) | \
        (rng.integers(1, 255, count, dtype=np.uint32) << np.uint32(23)) | \
        rng.integers(0, 1 << 23, count, dtype=np.uint32)
    q = count // 4
    low = np.uint32(0x1FFF)
    bits[:q] = (bits[:q] & ~low) | np.uint32(0x1000)
    bits[q:2 * q] = (bits[q:2 * q] & ~low) | np.where(np.arange(q) % 2, np.uint32(0x0FFF), np.uint32(0x1001))
    bits[:64] |= np.uint32(0x007FE000)  # ties that carry into the exponent
    return bits[(bits & np.uint32(0x7FFFFFFF)) < np.uint32(0x7F7FF000)]


def _run(shape, x, w, dy, which):
    """One pass of a 1 x 1 convolution through the raw entry points (coverage and containment checked)."""
    return _raw(shape, x, w, dy, passes=(which,))[which]


def _cuda(a, shape):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).reshape(shape).cuda()


def _probes(count):
    """(name, shape, the tensor holding the probed values, the output): the other tensors are all ones."""
    return [
        ("y = tf32(x)", (1, 1, 1, (1, 1), (1, 1), (0, 0), 1, 1, count), "x", "y"),
        ("y = tf32(w)", (1, 1, count, (1, 1), (1, 1), (0, 0), 1, 1, 1), "w", "y"),
        ("dx = tf32(dy)", (1, 1, 1, (1, 1), (1, 1), (0, 0), 1, 1, count), "dy", "dx"),
        ("dx = tf32(w)", (1, count, 1, (1, 1), (1, 1), (0, 0), 1, 1, 1), "w", "dx"),
        ("dw = tf32(x) tf32(dy=1)", (1, count, 1, (1, 1), (1, 1), (0, 0), 1, 1, 1), "x", "dw"),
        ("dw = tf32(dy) tf32(x=1)", (1, 1, count, (1, 1), (1, 1), (0, 0), 1, 1, 1), "dy", "dw"),
    ]


def _tensor_shapes(shape):
    n, c, k, (r, s), _, _, g, h, w = shape
    p, q = R.out_plane(shape)
    return {"x": (n, c, h, w), "w": (k, c // g, r, s), "dy": (n, k, p, q)}


@pytest.mark.parametrize("probe", range(6))
def test_k1_probes_round_every_operand_with_cvt_rna(probe):
    rng = np.random.default_rng(100 + probe)
    vals = _normal_bits(rng, 1 << 16).view(np.float32)
    name, shape, probed, out = _probes(vals.size)[probe]
    shapes = _tensor_shapes(shape)
    t = {name_: torch.ones(sh, device="cuda") for name_, sh in shapes.items()}
    t[probed] = _cuda(vals, shapes[probed])
    got = _run(shape, t["x"], t["w"], t["dy"], out).reshape(-1).cpu().numpy()
    want = R.tf32_rna(vals)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {vals.size} differ, first {vals[bad][0].view(np.uint32):#010x}"
                           f" -> {got[bad][0].view(np.uint32):#010x}, cvt.rna gives {want[bad][0].view(np.uint32):#010x}")


def test_k1_probes_take_exact_tf32_products():
    """dw = tf32(x) tf32(dy) with N·P·Q = 1 over an outer product of tie-heavy operands (exponents kept within
    +-50, so every 22-bit product is a normal float), and the same for y = tf32(x) tf32(w) and dx = tf32(dy) tf32(w)."""
    rng = np.random.default_rng(7)

    def vals(count):
        b = _normal_bits(rng, 4 * count)
        e = (b >> np.uint32(23)) & np.uint32(0xFF)
        return b[(e >= 77) & (e <= 177)][:count].view(np.float32)

    a, b = vals(300), vals(200)
    prod = (R.tf32_rna(a).astype(np.float64)[None, :] * R.tf32_rna(b).astype(np.float64)[:, None]).astype(np.float32)
    # dw[k, c] = x[c] dy[k]
    dw = _run((1, 300, 200, (1, 1), (1, 1), (0, 0), 1, 1, 1), _cuda(a, (1, 300, 1, 1)),
              torch.ones((200, 300, 1, 1), device="cuda"), _cuda(b, (1, 200, 1, 1)), "dw")
    # y[0, k, 0, q] = x[q] w[k]
    y = _run((1, 1, 200, (1, 1), (1, 1), (0, 0), 1, 1, 300), _cuda(a, (1, 1, 1, 300)), _cuda(b, (200, 1, 1, 1)),
             torch.ones((1, 200, 1, 300), device="cuda"), "y")
    # dx[0, c, 0, q] = dy[q] w[c]
    dx = _run((1, 200, 1, (1, 1), (1, 1), (0, 0), 1, 1, 300), torch.ones((1, 200, 1, 300), device="cuda"),
              _cuda(b, (1, 200, 1, 1)), _cuda(a, (1, 1, 1, 300)), "dx")
    for name, got in (("dw", dw), ("y", y), ("dx", dx)):
        g = got.reshape(200, 300).cpu().numpy()
        assert np.array_equal(g.view(np.uint32), prod.view(np.uint32)), f"{name}: a product differs from tf32 x tf32"


def test_k1_probe_records_rounding_past_the_largest_float():
    """cvt.rna of a finite value whose rounding carries past FLT_MAX is not pinned by PTX; record what the forward
    gives (+-inf, or the largest finite TF32 value of the same sign)."""
    mags = np.arange(0x7F7FF000, 0x7F800000, 0x101, dtype=np.uint32)
    vals = np.concatenate([mags, mags | np.uint32(0x80000000)]).view(np.float32)
    shape = (1, 1, 1, (1, 1), (1, 1), (0, 0), 1, 1, vals.size)
    y = _run(shape, _cuda(vals, (1, 1, 1, vals.size)), torch.ones((1, 1, 1, 1), device="cuda"),
             torch.ones((1, 1, 1, vals.size), device="cuda"), "y").reshape(-1).cpu().numpy()
    kinds = {f"{v:#010x}" for v in np.unique(y.view(np.uint32))}
    print("forward of values rounding past FLT_MAX gives", sorted(kinds))
    assert kinds <= {"0x7f800000", "0xff800000", "0x7f7fe000", "0xff7fe000"}, kinds
    assert np.array_equal(np.signbit(y), np.signbit(vals))


# --------------------------------------------------------------------------- the cuDNN control
@pytest.mark.parametrize("cid", ["caffenet-conv1-b4", "ragged2"])
@pytest.mark.parametrize("family", R.FAMILIES)
def test_cudnn_tf32_is_exact_on_the_same_operands(cid, family):
    """Strided cases, so cuDNN runs an implicit GEMM (no Winograd or FFT, which are not exact by construction)."""
    index = CASE_INDEX[cid]
    shape = dict(R.EXACT_CASES)[cid]
    n, c, k, kern, stride, pad, g, h, w = shape
    ints, exps = R.operands(shape, family, index)
    ref_y = _exact(shape, ints, exps)[0]
    v = {t: a.cuda() for t, a in R.as_values(ints, exps).items()}
    was = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        _equal("cuDNN TF32 y", F.conv2d(v["x"], v["w"], None, stride, pad, 1, g), ref_y)
    finally:
        torch.backends.cudnn.allow_tf32 = was
