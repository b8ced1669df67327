"""Caffe's Crop layer (crop_layer.cpp) restated in numpy, twice: from Python slices, and as an index map from each
output element to its source (the form the engine's kernels compute).  Both are copies, so either direction is exact
and compared bit for bit.  infer() restates LayerSetUp and Reshape's shape rule and CHECKs for the parser's tests."""
import numpy as np


def window(offsets, size):
    return tuple(slice(o, o + n) for o, n in zip(offsets, size))


def forward(x, top_shape, offsets):
    """x[o_0:o_0 + t_0, ..] for one offset per axis"""
    return x[window(offsets, top_shape)].copy()


def backward(dy, bottom_shape, offsets):
    """dx: dy inside the window, +0 outside it"""
    dx = np.zeros(bottom_shape, dy.dtype)
    dx[window(offsets, dy.shape)] = dy
    return dx


def forward_index_map(x, top_shape, offsets):
    """every top element's bottom index from its coordinates plus the offsets"""
    coords = np.indices(top_shape).reshape(len(top_shape), -1) + np.asarray(offsets).reshape(-1, 1)
    return x.ravel()[np.ravel_multi_index(tuple(coords), x.shape)].reshape(top_shape)


def backward_index_map(dy, bottom_shape, offsets):
    """every bottom element's top coordinates (its own minus the offsets): dy there when all lie inside, else +0"""
    coords = np.indices(bottom_shape).reshape(len(bottom_shape), -1) - np.asarray(offsets).reshape(-1, 1)
    inside = np.all((coords >= 0) & (coords < np.asarray(dy.shape).reshape(-1, 1)), axis=0)
    flat = np.zeros(int(np.prod(bottom_shape)), dy.dtype)
    flat[inside] = dy.ravel()[np.ravel_multi_index(tuple(coords[:, inside]), dy.shape)]
    return flat.reshape(bottom_shape)


def infer(bottom, ref, axis=2, offsets=()):
    """-> (canonical axis, top shape, one offset per axis of bottom); ValueError with Caffe's CHECK wording"""
    n = len(bottom)
    a = axis + n if axis < 0 else axis
    if not 0 <= a < n:
        raise ValueError(f"axis {axis} out of range for {n}-D Blob")
    if len(offsets) > 1 and a + len(offsets) != n:
        raise ValueError("number of offset values specified must be equal to the number of dimensions following axis.")
    top, offs = list(bottom), [0] * n
    for i in range(a, n):
        if i >= len(ref):  # Blob::shape(i) of the reference
            raise ValueError(f"axis {i} out of range for {len(ref)}-D Blob")
        o = 0 if not offsets else offsets[0] if len(offsets) == 1 else offsets[i - a]
        if bottom[i] - o < ref[i]:
            raise ValueError(f"the crop for dimension {i} is out-of-bounds with size {ref[i]} and offset {o}")
        top[i], offs[i] = ref[i], o
    return a, tuple(top), tuple(offs)


def specials(rng, shape):
    """Gaussian fp32 values with NaNs of several payloads (quiet and signalling, both signs), infinities, subnormals
    and both zeros spread through them"""
    x = rng.randn(*shape).astype(np.float32).ravel()
    bits = np.array([0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FA5A5A5, 0xFF812345, 0x7F800000, 0xFF800000, 0x00000001,
                     0x807FFFFF, 0x00000000, 0x80000000, 0x7F7FFFFF], np.uint32)
    k = rng.choice(x.size, size=min(x.size, bits.size), replace=False)
    x[k] = bits[:k.size].view(np.float32)
    return x.reshape(shape)
