"""Host-side restatements for the native TF32 convolutions (csrc/conv_tf32.cu, DESIGN.md section 10.2): the case lists
both GPU test files run, the kernels' operand rounding and weight-gradient split, exact (dyadic) operands with the
precondition that makes every partial sum exact in fp32, and a float64 implicit GEMM with the plausible wrong versions
of it that exact comparison has to catch.  CPU only: nothing here touches a GPU.

Why equality is the right check on dyadic operands.  Let every element of one operand be i * 2^ea and every element
of the other j * 2^eb, i and j integers of at most 11 significant bits.  Every such value is a TF32 value (so the
kernels' cvt.rna changes nothing), every product is i*j units of 2^(ea + eb) and exact in fp32, and every partial sum
of an output, in any order, tile split or chunk split, is an integer number of units no larger in magnitude than the
magnitude sum  sum |i| |j|  over that output's terms.  When that sum is at most 2^22 units, every partial sum has at
most 23 significant bits and is exact in fp32, so the float64 answer is the only answer a correct kernel can give.
This assumes that mma.sync's TF32 path adds exactly below that ceiling; the GPU file's K = 1 probes and its cuDNN
control test that assumption."""
import numpy as np
import torch
import torch.nn.functional as F

CEILING = 2 ** 22  # largest magnitude sum, in product units, of any exact case
BK = 16  # k-tile depth
TAP_SEG = 3584  # taps per shared-memory table segment
FILTER_TARGET_BLOCKS, FILTER_MIN_KTILES = 1024, 8


# --------------------------------------------------------------------------- the case lists
def _net_convs(name):
    """(in_channels, out_channels, kernel, stride, pad, groups, h, w) of every convolution of a net, in order."""
    from caffeonspark_b200 import layers, nets
    mod = nets.torch_module(name)
    found = []

    def hook(m, inp, _):
        found.append((m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding, m.groups,
                      inp[0].shape[2], inp[0].shape[3]))

    for m in mod.modules():
        if isinstance(m, layers.ConvReluMaxPool):  # the block calls its conv's weights, not the module
            m.register_forward_hook(lambda blk, inp, out: hook(blk.conv, inp, out))
        elif isinstance(m, torch.nn.Conv2d) and not any(getattr(b, "conv", None) is m for b in mod.modules()):
            m.register_forward_hook(hook)
    with torch.no_grad():
        mod(torch.zeros((1,) + tuple(nets.NETS[name]["input"])))
    return found


def _net_shapes():
    from caffeonspark_b200 import nets
    out = []
    for name in ("caffenet", "lenet", "cifar10_quick"):
        for i, cv in enumerate(_net_convs(name)):
            for b in sorted({nets.NETS[name]["batch"], 1, 2, 3, 4}):
                out.append((f"{name}-conv{i + 1}-b{b}", (b,) + cv))
    return out


# (id, shape): every convolution of CaffeNet, LeNet and CIFAR-10-quick at its own batch and at batch 1 to 4.
# A shape is (n, c, k, kernel, stride, pad, groups, h, w).
NET_SHAPES = _net_shapes()

# M, N and K off the tile sizes, groups 1 to 4, strides 1 to 4, pads 0 to 3, non-square kernels
RAGGED = [
    (3, 5, 7, (3, 3), (1, 1), (1, 1), 1, 9, 11),
    (2, 12, 20, (5, 3), (2, 1), (2, 0), 4, 17, 13),
    (5, 6, 9, (2, 4), (3, 4), (0, 3), 3, 19, 23),
    (1, 8, 130, (1, 1), (1, 1), (0, 0), 2, 7, 7),
    (7, 3, 1, (11, 11), (4, 4), (3, 3), 1, 31, 29),
    (2, 64, 66, (3, 3), (2, 2), (1, 1), 2, 15, 15),
    (4, 130, 40, (3, 2), (1, 3), (2, 1), 1, 6, 10),
    (1, 1, 1, (1, 1), (1, 1), (0, 0), 1, 1, 1),
]

# The edges the exact tests add to the two lists above (which tile, segment and split each reaches is asserted by
# tests/test_conv_tf32_exact_host.py, from geometry()).
EDGES = [
    # forward tap tables of one, two (3,585 and 3,600 taps) and three segments; the last also has a 3-segment dx.
    # Every tap reads image pixels for some output, so a wrong table entry at a segment's end cannot hide in padding.
    ("taps3584", (1, 224, 8, (4, 4), (1, 1), (0, 0), 1, 6, 6)),
    ("taps3585", (1, 717, 8, (1, 5), (1, 1), (0, 2), 1, 3, 4)),
    ("taps3600", (2, 16, 9, (15, 15), (1, 1), (7, 7), 1, 17, 17)),
    ("taps7200-g2", (1, 64, 6, (15, 15), (1, 1), (7, 7), 2, 16, 16)),
    ("taps7200-dx7425", (1, 32, 33, (15, 15), (2, 2), (7, 7), 1, 9, 9)),
    # M and N one off the tile edges, on both tile variants of every pass
    ("tile-fwd-n127-m129", (1, 2, 127, (3, 3), (1, 1), (1, 1), 1, 3, 43)),
    ("tile-fwd-n128-m127", (1, 2, 128, (1, 3), (1, 1), (0, 1), 1, 1, 127)),
    ("tile-fwd-n63-m129", (3, 2, 63, (3, 3), (1, 1), (1, 1), 1, 1, 43)),
    ("tile-fwd-n129-m127", (1, 3, 129, (1, 1), (1, 1), (0, 0), 1, 1, 127)),
    ("tile-data-n127-m129", (1, 127, 5, (3, 3), (1, 1), (1, 1), 1, 3, 43)),
    ("tile-data-n128-m127-g2", (1, 256, 6, (1, 3), (1, 1), (0, 1), 2, 1, 127)),
    ("tile-data-n63-m129", (3, 63, 4, (3, 3), (2, 2), (1, 1), 1, 1, 43)),
    ("tile-data-n129-m127", (1, 129, 3, (1, 1), (1, 1), (0, 0), 1, 1, 127)),
    ("tile-filter-n127-m127", (2, 127, 127, (1, 1), (1, 1), (0, 0), 1, 5, 7)),
    ("tile-filter-n128-m129", (2, 8, 129, (4, 4), (1, 1), (1, 1), 1, 9, 9)),
    ("tile-filter-n63-m129", (2, 7, 129, (3, 3), (2, 2), (1, 1), 1, 11, 11)),
    ("tile-filter-n129-m127", (2, 43, 127, (1, 3), (1, 1), (0, 1), 1, 6, 6)),
    # weight-gradient splits: one chunk (no workspace), nkt / 8 the limit with a one-k-tile last chunk
    ("split-one-chunk", (2, 3, 5, (3, 3), (1, 1), (1, 1), 1, 9, 9)),
    ("split-nkt-limit-short-last", (4, 3, 8, (3, 3), (1, 1), (1, 1), 1, 20, 20)),
    # stride > kernel (dx pixels no window reaches), pad >= kernel (outputs that see only padding)
    ("stride-over-kernel", (2, 3, 4, (2, 2), (3, 3), (0, 0), 1, 8, 8)),
    ("stride-over-kernel-padded", (2, 4, 6, (1, 2), (3, 4), (1, 1), 2, 10, 13)),
    ("pad-over-kernel", (2, 3, 5, (2, 3), (1, 1), (2, 3), 1, 4, 5)),
    # groups 1 to 4 with channels and filters per group not multiples of 8
    ("groups1-c5-k7", (2, 5, 7, (3, 3), (1, 1), (1, 1), 1, 7, 6)),
    ("groups2-cg7-kg9", (2, 14, 18, (3, 3), (1, 1), (1, 1), 2, 7, 6)),
    ("groups3-cg3-kg5", (2, 9, 15, (3, 2), (2, 1), (1, 0), 3, 8, 7)),
    ("groups4-cg5-kg7", (2, 20, 28, (3, 3), (1, 1), (1, 1), 4, 7, 6)),
    # a 1 x 1 image at batch 1, bare and padded
    ("image1x1-b1", (1, 5, 7, (1, 1), (1, 1), (0, 0), 1, 1, 1)),
    ("image1x1-b1-padded", (1, 3, 4, (3, 3), (1, 1), (1, 1), 1, 1, 1)),
]

# every case the exact tests run: (id, shape)
EXACT_CASES = NET_SHAPES + [(f"ragged{i}", s) for i, s in enumerate(RAGGED)] + EDGES

CAFFENET_CONV1_B256 = (256, 3, 96, (11, 11), (4, 4), (0, 0), 1, 227, 227)


def out_plane(shape):
    n, c, k, (r, s), (sh, sw), (ph, pw), g, h, w = shape
    return (h + 2 * ph - r) // sh + 1, (w + 2 * pw - s) // sw + 1


def geom12(shape):
    """The 12 ints the cos_conv_* entry points take: n, c, h, w, k, r, s, stride_h, stride_w, pad_h, pad_w, groups."""
    n, c, k, (r, s), (sh, sw), (ph, pw), g, h, w = shape
    return (n, c, h, w, k, r, s, sh, sw, ph, pw, g)


# --------------------------------------------------------------------------- the kernels' host-side decisions
def _ceil_div(a, b):
    return (a + b - 1) // b


def narrow(cols):
    """conv_tf32.cu's narrow(): 64 columns when that wastes fewer of them than 128."""
    return _ceil_div(cols, 64) * 64 - cols < _ceil_div(cols, 128) * 128 - cols


def filter_split(n, c, h, w, k, r, s, stride, pad, groups):
    """conv_tf32.cu's filter_split(): (chunks, chunk_ktiles) of the weight gradient's N·P·Q reduction.  stride and
    pad are (h, w) pairs."""
    p = (h + 2 * pad[0] - r) // stride[0] + 1
    q = (w + 2 * pad[1] - s) // stride[1] + 1
    ng, kg = c // groups * r * s, k // groups
    tiles = _ceil_div(kg, 128) * _ceil_div(ng, 64 if narrow(ng) else 128) * groups
    nkt = _ceil_div(n * p * q, BK)
    want = max(1, _ceil_div(FILTER_TARGET_BLOCKS, tiles))
    want = max(1, min(want, nkt // FILTER_MIN_KTILES))
    chunk_ktiles = _ceil_div(nkt, want)
    return _ceil_div(nkt, chunk_ktiles), chunk_ktiles


def split_of(shape):
    n, c, k, (r, s), stride, pad, g, h, w = shape
    return filter_split(n, c, h, w, k, r, s, stride, pad, g)


def geometry(shape):
    """What each pass of a case reaches: per pass (M, N, K, tile columns BN, table segments or weight-gradient
    chunks), keyed 'fwd', 'data', 'filter'."""
    n, c, k, (r, s), stride, pad, g, h, w = shape
    p, q = out_plane(shape)
    cg, kg = c // g, k // g
    chunks, chunk_ktiles = split_of(shape)
    fwd_k, data_k = cg * r * s, kg * r * s
    return {
        "fwd": dict(M=n * p * q, N=kg, K=fwd_k, BN=64 if narrow(kg) else 128, segments=_ceil_div(fwd_k, TAP_SEG)),
        "data": dict(M=n * h * w, N=cg, K=data_k, BN=64 if narrow(cg) else 128,
                     segments=_ceil_div(data_k, TAP_SEG)),
        "filter": dict(M=kg, N=cg * r * s, K=n * p * q, BN=64 if narrow(cg * r * s) else 128, chunks=chunks,
                       chunk_ktiles=chunk_ktiles, nkt=_ceil_div(n * p * q, BK)),
    }


def describe(shape):
    d = geometry(shape)
    f, a, b = d["fwd"], d["data"], d["filter"]
    return (f"fwd 128x{f['BN']} M={f['M']} N={f['N']} segs={f['segments']} | "
            f"data 128x{a['BN']} M={a['M']} N={a['N']} segs={a['segments']} | "
            f"filter 128x{b['BN']} M={b['M']} N={b['N']} chunks={b['chunks']}x{b['chunk_ktiles']} of {b['nkt']}")


# --------------------------------------------------------------------------- error bounds on Gaussian operands
C_TF32 = 2.0  # slack of both bounds, fixed before their first GPU run


def tf32_bound(reduce_len, mag):
    """Against float64 on the unrounded operands: TF32 rounding of both operands costs at most 2^-10 of each product
    and reduce_len fp32 additions at most reduce_len * 2^-24 of the magnitude sum mag each; doubled, and doubled
    again for the slack."""
    return C_TF32 * (2.0 ** -10 + reduce_len * 2.0 ** -23) * mag + 1e-30


def order_bound(depth, mag):
    """Against float64 on the TF32-rounded operands (tf32_rna), where only fp32 accumulation is left: depth additions
    in the longest chain of the kernel's order, plus one m16n8k8 step's 8 products, each off by at most an ulp
    (2^-23) of the magnitude sum mag of those rounded operands, doubled."""
    return C_TF32 * (depth + 8) * 2.0 ** -23 * mag + 1e-30


def depths(shape):
    """The longest addition chain of one output: the whole reduction for the forward and the data gradient, and for
    the weight gradient one chunk's k-tiles of BK products plus the chunk-order sum of the partials."""
    d = geometry(shape)
    return {"fwd": d["fwd"]["K"], "data": d["data"]["K"],
            "filter": d["filter"]["chunk_ktiles"] * BK + d["filter"]["chunks"]}


# --------------------------------------------------------------------------- cvt.rna.tf32.f32
def tf32_rna(a):
    """cvt.rna.tf32.f32 on an fp32 array: keep 10 mantissa bits, rounding to nearest with ties away from zero (add
    half of the 13 dropped bits to the magnitude, then clear them); +-0, +-inf and NaN are left alone.  A finite
    value whose rounding carries past the largest finite float comes out as inf here; PTX does not pin that case."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    bits = a.view(np.uint32)
    mag = bits & np.uint32(0x7FFFFFFF)
    rounded = ((mag + np.uint32(0x1000)) & np.uint32(0xFFFFE000)) | (bits & np.uint32(0x80000000))
    return np.where(mag >= np.uint32(0x7F800000), bits, rounded).astype(np.uint32).view(np.float32)


# --------------------------------------------------------------------------- dyadic operands
EXPONENTS = (-12, 0, 9)
FAMILIES = ("small", "wide")
WIDE = ("x", "w", "dy")  # which tensor the wide family makes 11-bit, by case index
MEAN_NONZERO = {"small": 8.0, "wide": 1024.0, "ternary": 1.0}  # mean |i| of a nonzero entry
MAX_INT = {"small": 15, "wide": 2047, "ternary": 1}


def _ints(gen, shape, kind, density):
    """Integers: 'small' uniform in [-15, 15], 'ternary' in {-1, 0, 1}, 'wide' odd in [-2047, 2047] (all 11 bits
    significant), each kept with probability `density` and zero otherwise."""
    if kind == "wide":
        v = torch.randint(-1024, 1024, shape, generator=gen, dtype=torch.int32) * 2 + 1
    else:
        v = torch.randint(-MAX_INT[kind], MAX_INT[kind] + 1, shape, generator=gen, dtype=torch.int32)
    if density < 1:
        v = v * (torch.rand(shape, generator=gen) < density)
    return v.to(torch.float64)


def operands(shape, family, index, seed=0):
    """Dyadic x, w, dy and bias of a case as float64 integer arrays plus their exponents: the values are
    ints * 2^exp, with exp from EXPONENTS varied per case.  family 'small': every tensor in [-15, 15];
    'wide': one tensor (WIDE[index % 3]) odd 11-bit, the others in {-1, 0, 1}.  Each pass thins one operand (the
    forward w, both gradients dy) so that (max |other|) * (expected sum of |thinned| over an output's terms) is about
    2^20, a quarter of the ceiling; check_precondition() then proves the ceiling for these exact values."""
    n, c, k, (r, s), _, _, g, h, w = shape
    p, q = out_plane(shape)
    kind = {t: family for t in ("x", "w", "dy")} if family == "small" else \
        {t: ("wide" if t == WIDE[index % 3] else "ternary") for t in ("x", "w", "dy")}
    lens = {"fwd": c // g * r * s, "data": k // g * r * s, "filter": n * p * q}

    def density(t, passes):  # passes: (pass, the other operand)
        d = 1.0
        for ps, other in passes:
            d = min(d, 2.0 ** 20 / (MAX_INT[kind[other]] * MEAN_NONZERO[kind[t]] * lens[ps]))
        return d

    gen = torch.Generator().manual_seed(seed * 1000003 + index * 7 + FAMILIES.index(family))
    ints = {
        "x": _ints(gen, (n, c, h, w), kind["x"], 1.0),
        "w": _ints(gen, (k, c // g, r, s), kind["w"], density("w", [("fwd", "x")])),
        "dy": _ints(gen, (n, k, p, q), kind["dy"], density("dy", [("data", "w"), ("filter", "x")])),
        "bias": _ints(gen, (k,), "wide", 1.0),
    }
    ex, ew, ed = (EXPONENTS[(index + i + FAMILIES.index(family)) % 3] for i in range(3))
    exps = {"x": ex, "w": ew, "dy": ed, "bias": ex + ew}
    return ints, exps


def as_values(ints, exps):
    """float32 tensors i * 2^e (exact)."""
    return {t: (v * 2.0 ** exps[t]).to(torch.float32) for t, v in ints.items()}


def _conv(x, w, stride, pad, g):
    return F.conv2d(x, w, None, stride, pad, 1, g)


def _conv_input(xshape, w, dy, stride, pad, g):
    return torch.nn.grad.conv2d_input(xshape, w, dy, stride, pad, 1, g)


def _conv_weight(x, wshape, dy, stride, pad, g):
    return torch.nn.grad.conv2d_weight(x, wshape, dy, stride, pad, 1, g)


def magnitude_bounds(shape, ints):
    """For each pass, an upper bound on the largest magnitude sum sum |i| |j| over one output's terms, in product
    units.  Each is the smaller of two bounds that hold element by element: (max |a|) * (sum of |b| over the terms)
    and the same with a and b swapped, where the sum of one operand over an output's terms is the same convolution
    with the other operand replaced by ones (no element is a term of one output twice).  The ones-convolutions have
    one filter per group, so this is cheap where the exact magnitude sums are not."""
    n, c, k, kern, stride, pad, g, h, w = shape
    ax, aw, ady = (ints[t].abs() for t in ("x", "w", "dy"))
    mx, mw, mdy = (float(t.max()) if t.numel() else 0.0 for t in (ax, aw, ady))
    cg, kg = c // g, k // g
    ones_w = torch.ones((g, cg) + tuple(kern), dtype=torch.float64)  # one filter per group
    per_grp = lambda t: t.repeat_interleave(kg, 1)  # noqa: E731  one value per group -> one per filter
    # forward: sum_{c,r,s} |x| |w|
    y_x = per_grp(_conv(ax, ones_w, stride, pad, g))  # window sums of |x| per group
    y_w = aw.sum((1, 2, 3)).view(1, k, 1, 1)
    fwd = torch.minimum(mw * y_x, mx * y_w).max()
    # data gradient: sum_{f,r,s} |dy| |w|
    dx_dy = _conv_input((n, g, h, w), torch.ones((g, 1) + tuple(kern), dtype=torch.float64),
                        ady.view(n, g, kg, *ady.shape[2:]).sum(2), stride, pad, g).repeat_interleave(cg, 1)
    dx_w = aw.view(g, kg, cg, -1).sum((1, 3)).reshape(1, c, 1, 1)
    data = torch.minimum(mw * dx_dy, mdy * dx_w).max()
    # weight gradient: sum_{img,p,q} |dy| |x|
    dw_dy = ady.sum((0, 2, 3)).view(k, 1, 1, 1)
    dw_x = _conv_weight(ax, (g, cg) + tuple(kern), torch.ones((n, g) + ady.shape[2:], dtype=torch.float64),
                        stride, pad, g).repeat_interleave(kg, 0)
    filt = torch.minimum(mx * dw_dy, mdy * dw_x).max()
    fwd_bias = fwd + float(ints["bias"].abs().max())
    return {"fwd": float(fwd_bias), "data": float(data), "filter": float(filt)}


def check_precondition(shape, ints):
    bounds = magnitude_bounds(shape, ints)
    for ps, b in bounds.items():
        assert b <= CEILING, f"{ps}: magnitude sum up to {b:.0f} product units, above the exact ceiling 2^22"
    return bounds


# --------------------------------------------------------------------------- float64 implicit GEMM and its mutants
MUTANTS = ("drop_tap", "swap_channels", "drop_last_ktile", "drop_image", "drop_chunk", "pad_off_by_one",
           "group_offset")


def _windows(x, kern, stride, pad, g, chan_shift=0, pad_shift=0):
    """A[grp, m, k]: the zero-padded window of x at output pixel m = (img, p, q) and tap k = (c, r, s) of group grp,
    reading channel grp·Cg + c + chan_shift (zero outside the tensor) with the pad taken as pad + pad_shift."""
    n, c, h, w = x.shape
    r, s = kern
    ph, pw = pad[0] + pad_shift, pad[1] + pad_shift
    p = (h + 2 * pad[0] - r) // stride[0] + 1
    q = (w + 2 * pad[1] - s) // stride[1] + 1
    cg = c // g
    xp = np.zeros((n, c + abs(chan_shift) * 2, h + 2 * max(ph, 0) + 2 * r, w + 2 * max(pw, 0) + 2 * s))
    oc, oh, ow = abs(chan_shift), max(ph, 0) + r, max(pw, 0) + s
    xp[:, oc:oc + c, oh:oh + h, ow:ow + w] = x
    A = np.zeros((g, n, p, q, cg, r, s))
    for grp in range(g):
        for rr in range(r):
            for ss in range(s):
                hs = oh - ph + rr
                ws = ow - pw + ss
                c0 = oc + grp * cg + chan_shift
                A[grp, :, :, :, :, rr, ss] = xp[:, c0:c0 + cg, hs:hs + stride[0] * p:stride[0],
                                                ws:ws + stride[1] * q:stride[1]].transpose(0, 2, 3, 1)
    return A.reshape(g, n * p * q, cg * r * s), p, q


def forward(x, w, stride, pad, g, mutation=None):
    """y = the implicit GEMM A @ B per group in float64; `mutation` names a plausible wrong kernel."""
    n = x.shape[0]
    k, cg, r, s = w.shape
    kg = k // g
    if mutation == "swap_channels" and x.shape[1] > 1:  # neighbouring channels 0 and 1 read swapped
        x = x.copy()
        x[:, [0, 1]] = x[:, [1, 0]]
    A, p, q = _windows(x, (r, s), stride, pad, g, chan_shift=1 if mutation == "group_offset" else 0,
                       pad_shift=1 if mutation == "pad_off_by_one" else 0)
    B = w.reshape(g, kg, cg * r * s).transpose(0, 2, 1)
    if mutation == "drop_tap":  # the window's last tap never loaded
        A = A.copy()
        A[:, :, -1] = 0
    if mutation == "drop_last_ktile":
        kt = cg * r * s
        A = A.copy()
        A[:, :, (kt - 1) // BK * BK:] = 0
    y = A @ B  # (g, n·p·q, kg)
    return y.reshape(g, n, p, q, kg).transpose(1, 0, 4, 2, 3).reshape(n, k, p, q)


def weight_grad(x, dy, wshape, stride, pad, g, mutation=None):
    """dw = sum over the filter_split chunks, in order, of each chunk's A @ B in float64."""
    k, cg, r, s = wshape
    n, c, h, wd = x.shape
    kg = k // g
    A, p, q = _windows(x, (r, s), stride, pad, g)  # (g, n·p·q, cg·r·s): the weight gradient's B
    D = dy.reshape(n, g, kg, p * q).transpose(1, 2, 0, 3).reshape(g, kg, n * p * q)
    if mutation == "drop_image":
        D = D.copy()
        D[:, :, (n - 1) * p * q:] = 0
    chunks, chunk_ktiles = filter_split(n, c, h, wd, k, r, s, stride, pad, g)
    bounds = [min(i * chunk_ktiles * BK, n * p * q) for i in range(chunks + 1)]
    if mutation == "drop_chunk":
        bounds = bounds[:-1]
    dw = np.zeros((g, kg, cg * r * s))
    for a, b in zip(bounds[:-1], bounds[1:]):
        dw = dw + D[:, :, a:b] @ A[:, a:b]
    return dw.reshape(k, cg, r, s)
