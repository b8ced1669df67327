"""An fp32 restatement of the built-in engine's 3-D convolution GEMMs (native_producer.cu, DESIGN.md section 14), bit
for bit: the Vol2col and Col2volGather gathers over three spatial axes, fed to gemm_ref.py's restatement of the GEMM
core (the fmaf chain over k in increasing order, the fixed-chunk split-K and its partials added in chunk order).
ChanMajor, WeightT, StoreNCHW and bias_grad_kernel serve the 3-D case as they are, over D H W in place of H W.

`mutation` names a plausible wrong version: gemm_ref's chain and reduction mutations, or one of GATHER_MUTATIONS, a
wrong index in Vol2col, for the tests that show the checks would catch it."""
import numpy as np

from gemm_ref import F32, chan_major, gemm, gemm_split
from producer_ops_ref import out_size


# geo3 = (kd, kh, kw, sd, sh, sw, pd, ph, pw)
def out_size3(dhw, geo3):
    return tuple(out_size(dhw[a], geo3[a], geo3[3 + a], geo3[6 + a]) for a in range(3))


def vol2col(x, geo3, mutation=None):
    """Vol2col's B[k, j]: k = ((ci * KD + kd) * KH + kh) * KW + kw, j = ((n * OD + od) * OH + oh) * OW + ow, zero
    outside the input.  The mutations read the input with a plausible wrong index (the output's size stays the
    geometry's): "depth_height_swapped" reads x[n, c, h, d, w]; "pad_rotated" applies the depth's pad to the height and
    the height's to the depth; "stride_reversed" applies (sd, sh, sw) as (sw, sh, sd)."""
    x = np.asarray(x, F32)
    k, s, p = list(geo3[0:3]), list(geo3[3:6]), list(geo3[6:9])
    n, c = x.shape[:2]
    outs = out_size3(x.shape[2:], geo3)
    if mutation == "depth_height_swapped":
        x = x.swapaxes(2, 3)
    if mutation == "pad_rotated":
        p = [p[1], p[0], p[2]]
    if mutation == "stride_reversed":
        s = s[::-1]
    idx, ok = [], []
    for a in range(3):  # per axis, the input position of tap t at output o, and whether it lies inside
        i = np.arange(outs[a])[None, :] * s[a] - p[a] + np.arange(k[a])[:, None]
        ok.append((i >= 0) & (i < x.shape[2 + a]))
        idx.append(np.clip(i, 0, x.shape[2 + a] - 1))
    g = np.take(x, idx[0], axis=2)             # n, c, kd, od, H, W
    g = np.take(g, idx[1], axis=4)             # n, c, kd, od, kh, oh, W
    g = np.take(g, idx[2], axis=6)             # n, c, kd, od, kh, oh, kw, ow
    inside = ok[0][:, :, None, None, None, None] & ok[1][None, None, :, :, None, None] & ok[2][None, None, None, None]
    g = np.where(inside, g, F32(0))
    return np.ascontiguousarray(g.transpose(1, 2, 4, 6, 0, 3, 5, 7)).reshape(c * k[0] * k[1] * k[2], -1)


def weight_t3(w):
    """WeightT's A[ci, k2] = W[co, ci, kd, kh, kw], k2 = ((co * KD + kd) * KH + kh) * KW + kw."""
    w = np.asarray(w, F32)
    return w.transpose(1, 0, 2, 3, 4).reshape(w.shape[1], -1)


def col2vol_gather(dy, x_shape, geo3):
    """Col2volGather's B[k2, j]: dy[n, co, od, oh, ow] at the output whose window puts tap (kd, kh, kw) on input voxel
    j = ((n * D + d) * H + h) * W + w, i.e. d + PD - kd = od * SD (and so for h and w); zero where there is none."""
    dy = np.asarray(dy, F32)
    n, _, d, h, w = x_shape
    cout, od, oh, ow = dy.shape[1:]
    out = np.zeros((cout, geo3[0], geo3[1], geo3[2], n, d, h, w), F32)
    dyt = dy.transpose(1, 0, 2, 3, 4)
    # per axis and tap: the input positions with an output there, and that output's index
    hit = []
    for ax, (size, osize) in enumerate(((d, od), (h, oh), (w, ow))):
        k, s, p = geo3[ax], geo3[3 + ax], geo3[6 + ax]
        taps = []
        for t in range(k):
            q = np.arange(size) + p - t
            ok = np.flatnonzero((q >= 0) & (q % s == 0) & (q // s < osize))
            taps.append((ok, q[ok] // s))
        hit.append(taps)
    for a, (da, oda) in enumerate(hit[0]):
        for i, (hi, ohi) in enumerate(hit[1]):
            for j, (wj, owj) in enumerate(hit[2]):
                out[:, a, i, j][np.ix_(range(cout), range(n), da, hi, wj)] = dyt[np.ix_(range(cout), range(n), oda, ohi,
                                                                                          owj)]
    return out.reshape(cout * geo3[0] * geo3[1] * geo3[2], n * d * h * w)


def _ncdhw(c, n, dhw):
    """C[m = channel, j = (n, voxel)] -> [N, C, D, H, W] (StoreNCHW over D H W)"""
    return np.ascontiguousarray(c.reshape(c.shape[0], n, *dhw).transpose(1, 0, 2, 3, 4))


def _gathers(mutation):
    """(the gather's mutation, the GEMM's): vol2col's own go to it, the rest to the chain or the split-K reduction"""
    return (mutation, None) if mutation in GATHER_MUTATIONS else (None, mutation)


GATHER_MUTATIONS = ("depth_height_swapped", "pad_rotated", "stride_reversed")


def conv3d_forward(x, w, b, geo3, mutation=None):
    """y = W * vol2col(x) (+ bias): A = W [Cout, Cin KD KH KW], B = Vol2col."""
    x, w = np.asarray(x, F32), np.asarray(w, F32)
    gm, mm = _gathers(mutation)
    c = gemm(w.reshape(w.shape[0], -1), vol2col(x, geo3, gm), b, mm)
    return _ncdhw(c, x.shape[0], out_size3(x.shape[2:], geo3))


def conv3d_weight_grad(x, dy, geo3, mutation=None):
    """dW [Cout, Cin, KD, KH, KW] = dy * vol2col(x)^T over N OD OH OW, split-K: A = ChanMajor(dy), B = Vol2col
    transposed.  dy may hold a subset of the output channels; dW then holds theirs."""
    gm, mm = _gathers(mutation)
    g = gemm_split(chan_major(dy), vol2col(x, geo3, gm).T, mm)
    return g.reshape(np.shape(dy)[1], np.shape(x)[1], *geo3[:3])


def conv3d_data_grad(dy, w, b, x_shape, geo3, mutation=None):
    """dx = W^T * dy gathered back to the input (+ bias): A = WeightT, B = Col2volGather."""
    c = gemm(weight_t3(w), col2vol_gather(dy, x_shape, geo3), b, mutation)
    return _ncdhw(c, x_shape[0], x_shape[2:])


def deconv3d_forward(x, w, b, geo3, out_dhw, mutation=None):
    """the 3-D convolution's data gradient of x, with the bias: w is [Cin, Cout, KD, KH, KW], the convolution's
    [Cout, Cin]"""
    return conv3d_data_grad(x, w, b, (np.shape(x)[0], np.shape(w)[1]) + tuple(out_dhw), geo3, mutation)


def deconv3d_weight_grad(x, dy, geo3, mutation=None):
    """the 3-D convolution's weight gradient with the top's gradient dy as its input and the bottom x as its dy"""
    return conv3d_weight_grad(dy, x, geo3, mutation)


def deconv3d_data_grad(dy, w, geo3, mutation=None):
    """the 3-D convolution's forward of dy, without the bias"""
    return conv3d_forward(dy, w, None, geo3, mutation)
