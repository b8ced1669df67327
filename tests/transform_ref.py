"""numpy restatement of Caffe's TRAIN-phase DataTransformer (data_transformer.cpp) as the library runs it on the device,
and of its draws (DESIGN.md, "Input transform on the device").  float32 arithmetic, one operation at a time:
(x - mean) * scale, or x * scale without a mean.

Two input formats, as the JVM hands them to the transformer:
  u8:  N x H x W x C uint8 images, Transform(cv::Mat) per image -- one mirror / crop draw per image n
  f32: N x C x H x W float32 blob, Transform(Blob*, Blob*) -- one draw per batch (n = 0)
"""
import numpy as np

PHI = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def mix64(z):
    """splitmix64 finaliser on a Python int (mod 2^64)."""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key(seed, rank, input_index, it, pass_index):
    """mix64(mix64(mix64(mix64(seed * phi + rank) + input) + iter) + pass); a negative seed counts as 0."""
    s = max(int(seed), 0)
    k = mix64(s * PHI + rank)
    k = mix64(k + input_index)
    k = mix64(k + it)
    return mix64(k + pass_index)


def draw(k, n, j, rng):
    """uint32(mix64(key + (n * 4 + j) * phi) >> 32) % range; j: 0 mirror (range 2), 1 h_off, 2 w_off."""
    return ((mix64(k + (n * 4 + j) * PHI) >> 32) & 0xFFFFFFFF) % rng


def draws(k, n, height, width, crop, mirror):
    """-> (do_mirror, h_off, w_off) of image n (Caffe: mirror && Rand(2); Rand(H - crop + 1); Rand(W - crop + 1))."""
    m = bool(mirror) and draw(k, n, 0, 2) == 1
    h_off = draw(k, n, 1, height - crop + 1) if crop else 0
    w_off = draw(k, n, 2, width - crop + 1) if crop else 0
    return m, h_off, w_off


def _one(x_chw, mean, mean_values, scale, h_off, w_off, ho, wo, do_mirror):
    """x_chw: C x H x W float32 of one image; returns C x ho x wo float32."""
    C = x_chw.shape[0]
    x = x_chw[:, h_off:h_off + ho, w_off:w_off + wo]
    s = np.float32(scale)
    if mean is not None:
        m = np.asarray(mean, np.float32).reshape(C, x_chw.shape[1], x_chw.shape[2])
        m = m[:, h_off:h_off + ho, w_off:w_off + wo]
        v = np.subtract(x, m, dtype=np.float32)
        v = np.multiply(v, s, dtype=np.float32)
    elif mean_values is not None and len(mean_values):
        mv = np.asarray(mean_values, np.float32)
        mv = np.repeat(mv, C) if mv.size == 1 else mv  # one value is replicated over the channels
        v = np.subtract(x, mv[:, None, None], dtype=np.float32)
        v = np.multiply(v, s, dtype=np.float32)
    else:
        v = np.multiply(x, s, dtype=np.float32)
    # mirrored: output column w holds input column wo-1-w, and so its (unmirrored) mean
    return np.ascontiguousarray(v[:, :, ::-1] if do_mirror else v)


def transform(x, fmt, crop=0, mirror=False, mean=None, mean_values=None, scale=1.0, k=0):
    """x: uint8 N x H x W x C (fmt "u8") or float32 N x C x H x W (fmt "f32") -> float32 N x C x ho x wo."""
    if fmt == "u8":
        N, H, W, C = x.shape
        chw = lambda n: np.ascontiguousarray(x[n].transpose(2, 0, 1)).astype(np.float32)  # noqa: E731
    else:
        N, C, H, W = x.shape
        chw = lambda n: np.asarray(x[n], np.float32)  # noqa: E731
    ho, wo = (crop, crop) if crop else (H, W)
    out = np.empty((N, C, ho, wo), np.float32)
    for n in range(N):
        m, h_off, w_off = draws(k, n if fmt == "u8" else 0, H, W, crop, mirror)
        out[n] = _one(chw(n), mean, mean_values, scale, h_off, w_off, ho, wo, m)
    return out


def blobproto(data, shape=None, legacy=None):
    """A Caffe BlobProto as bytes: `shape` (field 7, packed dims) or legacy num/channels/height/width (fields 1-4),
    and packed float data (field 5)."""
    def varint(v):
        out = bytearray()
        while True:
            b = v & 0x7F
            v >>= 7
            if v:
                out.append(b | 0x80)
            else:
                out.append(b)
                return bytes(out)

    def field(num, wire, payload):
        return varint((num << 3) | wire) + payload

    msg = b""
    if legacy is not None:
        for i, d in enumerate(legacy):
            msg += field(i + 1, 0, varint(int(d)))
    if shape is not None:
        dims = b"".join(varint(int(d)) for d in shape)
        inner = field(1, 2, varint(len(dims)) + dims)
        msg += field(7, 2, varint(len(inner)) + inner)
    raw = np.ascontiguousarray(data, np.float32).tobytes()
    msg += field(5, 2, varint(len(raw)) + raw)
    return msg


def same_bits(a, b):
    """bitwise equality of two float32 arrays, every NaN equal to every NaN."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape:
        return False
    nan = np.isnan(a)
    return bool(np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan]))
