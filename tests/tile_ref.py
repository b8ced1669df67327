"""Caffe's Tile layer (tile_layer.cpp) restated in numpy, twice: in float64, and in fp32 in Forward_cpu's and
Backward_cpu's order (the form the engine's kernels compute bit for bit).  With outer = count(0, axis) and inner =
count(axis) of the bottom, the top is [outer, tiles, inner] in memory.  The backward copies tile 0's gradient and adds
tiles 1 .. tiles - 1 in order, each add rounded once in fp32 (caffe_copy, then caffe_axpy with alpha 1), so a column of
-0 stays -0.  infer() restates Reshape's shape rule and CHECKs for the parser's tests.

dims(), tile_order() and start() are the three choices a restatement could get wrong; the host tests replace each
with a plausible mistake and show that a check fails."""
import numpy as np

F32 = np.float32
FLT_MAX = np.finfo(F32).max


def infer(bottom, axis, tiles):
    """The top shape, or ValueError with Caffe's wording (Blob::CanonicalAxisIndex's as the parser words it)"""
    n = len(bottom)
    a = axis + n if axis < 0 else axis
    if not 0 <= a < n:
        raise ValueError(f"axis {axis} out of range for {n}-D Blob")
    if tiles is None:
        raise ValueError("Number of tiles must be specified")
    if tiles <= 0:
        raise ValueError("Number of tiles must be positive.")
    top = list(bottom)
    top[a] *= tiles
    return tuple(top)


def dims(bottom_shape, axis):
    """(outer, inner): count(0, axis) and count(axis) of the bottom"""
    a = axis + len(bottom_shape) if axis < 0 else axis
    return int(np.prod(bottom_shape[:a], dtype=np.int64)), int(np.prod(bottom_shape[a:], dtype=np.int64))


def tile_order(tiles):
    """(the tile copied first, the tiles added after it in order)"""
    return 0, range(1, tiles)


def start(column):
    """the first tile's gradient as the sum's start: caffe_copy"""
    return column.copy()


def forward64(x, axis, tiles):
    outer, inner = dims(x.shape, axis)
    y = np.broadcast_to(np.asarray(x, np.float64).reshape(outer, 1, inner), (outer, tiles, inner))
    return y.reshape(infer(x.shape, axis, tiles))


def backward64(dy, bottom_shape, axis, tiles):
    outer, inner = dims(bottom_shape, axis)
    return np.asarray(dy, np.float64).reshape(outer, tiles, inner).sum(1).reshape(bottom_shape)


def forward32(x, axis, tiles):
    """Forward_cpu: for each outer row, `tiles` copies of its inner elements"""
    outer, inner = dims(x.shape, axis)
    rows = np.asarray(x, F32).reshape(outer, inner)
    y = np.empty((outer, tiles, inner), F32)
    for t in range(tiles):
        y[:, t] = rows
    return y.reshape(infer(x.shape, axis, tiles))


def backward32(dy, bottom_shape, axis, tiles):
    """Backward_cpu: dx = dy[:, first], then dy[:, t] added for each later t, each add rounded once in fp32"""
    outer, inner = dims(bottom_shape, axis)
    d = np.asarray(dy, F32).reshape(outer, tiles, inner)
    first, rest = tile_order(tiles)
    with np.errstate(invalid="ignore", over="ignore"):
        dx = start(d[:, first])
        for t in rest:
            dx = (dx + d[:, t]).astype(F32)
    return dx.reshape(bottom_shape)


SPECIALS = np.array([0x7FC00000, 0xFFC00001, 0x7F800000, 0xFF800000, 0x00000000, 0x80000000, 0xFF7FFFFF, 0x7F7FFFFF,
                     0x00000001], np.uint32).view(F32)  # NaNs, +-inf, +-0, -+FLT_MAX, the smallest subnormal


def specials(rng, shape, count=None):
    """Gaussian fp32 values of several magnitudes (so that the order of a sum shows in its bits) with each special
    value placed once at random (or at `count` places): NaN of two payloads, both infinities, both zeros, -FLT_MAX,
    FLT_MAX and the smallest subnormal"""
    x = (rng.randn(*shape) * np.exp2(rng.randint(-8, 9, shape))).astype(F32)
    flat = x.reshape(-1)
    n = min(flat.size, SPECIALS.size if count is None else count)
    flat[rng.choice(flat.size, size=n, replace=False)] = np.resize(SPECIALS, n)
    return x


def negative_zero_column(dy, bottom_shape, axis, tiles, column=-1):
    """dy with every tile of one dx element (the last, by default) set to -0"""
    outer, inner = dims(bottom_shape, axis)
    d = np.array(dy, F32).reshape(outer, tiles, inner)
    o, i = divmod(column % (outer * inner), inner)
    d[o, :, i] = F32(-0.0)
    return d.reshape(dy.shape)


def canonical_bits(a):
    """a's bits with every NaN as 0x7FFFFFFF, the GPU's canonical NaN (numpy carries an input's payload through an add,
    the GPU does not)"""
    b = np.ascontiguousarray(a, F32).view(np.uint32).copy()
    b[np.isnan(np.asarray(a, F32))] = 0x7FFFFFFF
    return b
