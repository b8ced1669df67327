"""CPU checks of what the exact TF32 convolution tests stand on (tests/conv_tf32_ref.py, DESIGN.md section 10.2):
filter_split agrees with the library's weight-gradient workspace, the case list reaches every edge it is meant to,
the exactness precondition holds for every case's operands, every plausible wrong kernel differs from the exact answer
on them, the bound that follows the kernels' order rejects a zero weight gradient that the K-length bound accepts,
and tf32_rna gives cvt.rna's known answers."""
import numpy as np
import pytest
import torch

import conv_tf32_ref as R

CASES = [pytest.param(i, shape, id=cid) for i, (cid, shape) in enumerate(R.EXACT_CASES)]


# --------------------------------------------------------------------------- the weight-gradient split
def _sweep():
    shapes = [s for _, s in R.EXACT_CASES]
    for n in (1, 2, 7, 16, 64, 255, 256, 257):
        for c, k, kern, stride, pad, g, h in ((3, 96, (11, 11), (4, 4), (0, 0), 1, 227), (96, 256, (5, 5), (1, 1),
                                              (2, 2), 2, 27), (3, 32, (5, 5), (1, 1), (2, 2), 1, 32),
                                              (384, 256, (3, 3), (1, 1), (1, 1), 2, 13), (1, 20, (5, 5), (1, 1),
                                              (0, 0), 1, 28)):
            shapes.append((n, c, k, kern, stride, pad, g, h, h))
    return shapes


def test_filter_split_agrees_with_the_library_workspace(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    assert R.split_of(R.CAFFENET_CONV1_B256) == (341, 142)
    for shape in _sweep():
        n, c, k, (r, s), _, _, g, _, _ = shape
        chunks, chunk_ktiles = R.split_of(shape)
        nkt = R.geometry(shape)["filter"]["nkt"]
        assert (chunks - 1) * chunk_ktiles < nkt <= chunks * chunk_ktiles, shape
        want = chunks * k * (c // g) * r * s if chunks > 1 else 0
        assert L.cos_conv_workspace_floats(*R.geom12(shape)) == want, shape


# --------------------------------------------------------------------------- what the case list reaches
def _reached(pred):
    return [cid for cid, shape in R.EXACT_CASES if pred(shape, R.geometry(shape))]


def test_the_exact_cases_reach_every_edge():
    assert _reached(lambda s, d: d["fwd"]["segments"] == 3)
    assert _reached(lambda s, d: d["fwd"]["segments"] == 2)
    assert _reached(lambda s, d: d["data"]["segments"] == 3)
    for ps in ("fwd", "data", "filter"):
        for bn in (64, 128):
            on = lambda s, d, ps=ps, bn=bn: d[ps]["BN"] == bn  # noqa: E731
            assert _reached(lambda s, d: on(s, d) and d[ps]["M"] % 128 == 1), (ps, bn, "M = tile + 1")
            assert _reached(lambda s, d: on(s, d) and d[ps]["M"] % 128 == 127), (ps, bn, "M = tile - 1")
            assert _reached(lambda s, d: on(s, d) and d[ps]["N"] % bn == bn - 1), (ps, bn, "N = tile - 1")
            # a 128-wide tile is never picked for N = 128 j + 1 (64 columns waste less), so it is checked at 128 j
            assert _reached(lambda s, d: on(s, d) and d[ps]["N"] % bn == (1 if bn == 64 else 0)), (ps, bn)
    f = lambda s, d: d["filter"]  # noqa: E731
    assert _reached(lambda s, d: f(s, d)["chunks"] == 1)
    assert _reached(lambda s, d: f(s, d)["chunks"] == f(s, d)["nkt"] // R.FILTER_MIN_KTILES > 1)
    assert _reached(lambda s, d: f(s, d)["nkt"] % f(s, d)["chunk_ktiles"] != 0 and f(s, d)["chunks"] > 1)
    assert _reached(lambda s, d: f(s, d)["chunks"] == 341)
    assert _reached(lambda s, d: s[4][0] > s[3][0] and s[4][1] > s[3][1])
    assert _reached(lambda s, d: s[5][0] >= s[3][0] and s[5][1] >= s[3][1])
    for g in (1, 2, 3, 4):
        assert _reached(lambda s, d, g=g: s[6] == g and (s[1] // g) % 8 and (s[2] // g) % 8)
    assert _reached(lambda s, d: s[0] == 1 and s[7] == s[8] == 1)


def test_every_tap_of_a_segmented_table_reads_the_image():
    for cid, shape in R.EXACT_CASES:
        d = R.geometry(shape)
        if d["fwd"]["segments"] == 1 and d["data"]["segments"] == 1:
            continue
        n, c, k, kern, stride, pad, g, h, w = shape
        p, q = R.out_plane(shape)
        live = torch.nn.grad.conv2d_weight(torch.ones((n, c, h, w), dtype=torch.float64), (k, c // g) + kern,
                                           torch.ones((n, k, p, q), dtype=torch.float64), stride, pad, 1, g)
        assert (live > 0).all(), f"{cid}: a tap that only ever reads padding"


@pytest.mark.parametrize("cid", ["stride-over-kernel", "stride-over-kernel-padded"])
def test_stride_over_kernel_leaves_dx_pixels_no_window_reaches(cid):
    n, c, k, kern, stride, pad, g, h, w = shape = dict(R.EXACT_CASES)[cid]
    p, q = R.out_plane(shape)
    reach = torch.nn.grad.conv2d_input((n, c, h, w), torch.ones((k, c // g) + kern, dtype=torch.float64),
                                       torch.ones((n, k, p, q), dtype=torch.float64), stride, pad, 1, g)
    assert (reach == 0).any() and (reach > 0).any()


def test_pad_over_kernel_has_outputs_that_see_only_padding():
    n, c, k, kern, stride, pad, g, h, w = shape = dict(R.EXACT_CASES)["pad-over-kernel"]
    seen = torch.nn.functional.conv2d(torch.ones((n, c, h, w), dtype=torch.float64),
                                      torch.ones((k, c // g) + kern, dtype=torch.float64), None, stride, pad, 1, g)
    assert (seen == 0).any() and (seen > 0).any()


# --------------------------------------------------------------------------- the exactness precondition
@pytest.mark.parametrize("family", R.FAMILIES)
@pytest.mark.parametrize("index, shape", CASES)
def test_precondition_holds(index, shape, family):
    ints, exps = R.operands(shape, family, index)
    R.check_precondition(shape, ints)
    for t, v in R.as_values(ints, exps).items():  # every value a normal TF32 value (or zero)
        a = v.numpy()
        assert np.array_equal(R.tf32_rna(a), a), t
        nz = np.abs(a[a != 0])
        assert nz.size == 0 or nz.min() >= np.finfo(np.float32).tiny, t


def test_magnitude_bounds_cover_the_exact_magnitude_sums():
    for index, (cid, shape) in enumerate(R.EXACT_CASES):
        if cid.startswith(("caffenet", "lenet-conv2-b64", "cifar10_quick")) or cid.startswith("taps"):
            continue  # the exact sums are costly on a CPU; the bound's argument does not depend on the size
        n, c, k, kern, stride, pad, g, h, w = shape
        for family in R.FAMILIES:
            ints, _ = R.operands(shape, family, index)
            a = {t: v.abs() for t, v in ints.items()}
            exact = {"fwd": float(torch.nn.functional.conv2d(a["x"], a["w"], None, stride, pad, 1, g).max() +
                                  a["bias"].max()),
                     "data": float(torch.nn.grad.conv2d_input(a["x"].shape, a["w"], a["dy"], stride, pad, 1,
                                                              g).max()),
                     "filter": float(torch.nn.grad.conv2d_weight(a["x"], a["w"].shape, a["dy"], stride, pad, 1,
                                                                 g).max())}
            bound = R.magnitude_bounds(shape, ints)
            for ps in exact:
                assert exact[ps] <= bound[ps], (cid, family, ps)


# --------------------------------------------------------------------------- mutants
MUTANT_SHAPES = [
    (2, 4, 6, (3, 3), (1, 1), (1, 1), 2, 7, 6),
    (4, 2, 4, (3, 3), (2, 1), (1, 1), 2, 17, 9),  # a weight gradient in 2 chunks
    (3, 6, 9, (2, 3), (1, 2), (0, 1), 3, 8, 9),
]


@pytest.mark.parametrize("shape", MUTANT_SHAPES, ids=[f"mutant-shape{i}" for i in range(len(MUTANT_SHAPES))])
def test_every_mutant_differs_from_the_exact_answer(shape):
    n, c, k, kern, stride, pad, g, h, w = shape
    ints, exps = R.operands(shape, "small", 3)
    v = {t: a.numpy() for t, a in R.as_values(ints, exps).items()}
    x, wt, dy = (v[t].astype(np.float64) for t in ("x", "w", "dy"))
    tx, tw, tdy = (torch.from_numpy(a) for a in (x, wt, dy))
    y = R.forward(x, wt, stride, pad, g)
    dw = R.weight_grad(x, dy, wt.shape, stride, pad, g)
    assert np.array_equal(y, torch.nn.functional.conv2d(tx, tw, None, stride, pad, 1, g).numpy())
    assert np.array_equal(dw, torch.nn.grad.conv2d_weight(tx, wt.shape, tdy, stride, pad, 1, g).numpy())
    table = []
    for m in R.MUTANTS:
        got = R.weight_grad(x, dy, wt.shape, stride, pad, g, m) if m in ("drop_image", "drop_chunk") else \
            R.forward(x, wt, stride, pad, g, m)
        ref = dw if m in ("drop_image", "drop_chunk") else y
        differ = int((got != ref).sum())
        table.append(f"{m}: {differ} of {ref.size} elements differ")
        assert differ > 0, m
    print("\n".join(table))


def test_old_bound_accepts_a_zero_weight_gradient_the_order_bound_rejects():
    """At CIFAR-10-quick conv1 b100, on Gaussian operands built as test_gpu_conv_tf32.py builds them, dw = 0 is within
    the K-length bound everywhere and far outside the bound that follows the kernel's split."""
    n, c, k, kern, stride, pad, g, h, w = shape = dict(R.NET_SHAPES)["cifar10_quick-conv1-b100"]
    p, q = R.out_plane(shape)
    gen = torch.Generator().manual_seed(0)
    x = torch.randn((n, c, h, w), generator=gen)
    wt = torch.randn((k, c // g, *kern), generator=gen) / (c // g * kern[0] * kern[1]) ** 0.5
    dy = torch.randn((n, k, p, q), generator=gen)
    dw = torch.nn.grad.conv2d_weight(x.double(), wt.shape, dy.double(), stride, pad, 1, g)
    xr, dyr = (torch.from_numpy(R.tf32_rna(t.numpy())).double() for t in (x, dy))
    dwm = torch.nn.grad.conv2d_weight(xr.abs(), wt.shape, dyr.abs(), stride, pad, 1, g)
    old = R.tf32_bound(n * p * q, dwm)
    new = R.order_bound(R.depths(shape)["filter"], dwm)
    assert (dw.abs() <= old).all()
    worst = float((dw.abs() / new).max())
    print(f"dw = 0: within the K-length bound; {worst:.1f} times the order bound")
    assert worst > 4


# --------------------------------------------------------------------------- cvt.rna known answers
def _f(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


@pytest.mark.parametrize("src, want", [
    (0x3F800000, 0x3F800000),  # 1.0 is a TF32 value
    (0x3F801000, 0x3F802000),  # 1 + 2^-11, a tie: away from zero (to nearest even would give 1.0)
    (0x3F803000, 0x3F804000),  # a tie above an odd last bit
    (0xBF801000, 0xBF802000),  # negative tie: away from zero
    (0x3F800FFF, 0x3F800000),  # below a tie
    (0x3F801001, 0x3F802000),  # above a tie
    (0xBF800FFF, 0xBF800000),
    (0x3FFFF000, 0x40000000),  # a tie that carries into the exponent
    (0x7F7FE000, 0x7F7FE000),  # the largest finite TF32 value
    (0x7F7FEFFF, 0x7F7FE000),  # below the carry past it
    (0x00001000, 0x00002000),  # subnormal tie
    (0x00000FFF, 0x00000000),
    (0x007FF000, 0x00800000),  # the largest subnormal tie rounds to the smallest normal
    (0x00000000, 0x00000000),
    (0x80000000, 0x80000000),
    (0x7F800000, 0x7F800000),
    (0xFF800000, 0xFF800000),
    (0x7FC00001, 0x7FC00001),  # NaN left alone, payload and all
    (0xFF801234, 0xFF801234),
])
def test_tf32_rna_known_answers(src, want):
    assert R.tf32_rna(_f([src])).view(np.uint32)[0] == want


def test_tf32_rna_is_a_function_of_the_value_and_keeps_10_bits():
    rng = np.random.default_rng(0)
    bits = rng.integers(0x00800000, 0x7F7FF000, 1 << 16, dtype=np.uint32)  # positive normals
    out = R.tf32_rna(bits.view(np.float32)).view(np.uint32)
    assert not (out & np.uint32(0x1FFF)).any()
    assert np.array_equal(R.tf32_rna((bits | np.uint32(1 << 31)).view(np.float32)).view(np.uint32),
                          out | np.uint32(1 << 31))
    err = np.abs(out.view(np.float32).astype(np.float64) - bits.view(np.float32).astype(np.float64))
    assert (err <= 2.0 ** -11 * np.abs(bits.view(np.float32).astype(np.float64))).all()
