"""Named, seeded blob layouts for the fused sync kernels' parity tests (no GPU needed).

A layout is (counts, lr_mult, decay_mult), one entry per learnable blob, built deterministically.  The existing sync
tests use at most ten blobs and multipliers in {0, 0.25, 0.5, 1, 2}; these layouts reach what real Caffe nets reach:

- seg_511 ... seg_3000: that many blobs, on both sides of the kernels' shared-memory segment-table limits (512 for the
  TMA kernel, 1024 for the others).  Counts come from {1, 2, 3, 5, 7, 64, 333} plus two or three blobs of 10^4..10^5
  elements, so shards cut through blobs and float4 vectors straddle up to four blob ends; multipliers come from
  LR_MULTS / DECAY_MULTS, which round when multiplied.
- empty_blobs: zero-count blobs first, last, two in a row, and one between two blobs that share a float4.
- resnet152_bn_like: the learnable blobs of a Caffe ResNet-152 (conv without bias, BatchNorm's 3 blobs, Scale's 2,
  fc weight and bias: 932 blobs) at a small width, with fine-tuning multipliers: BatchNorm 0, conv1 and res2 0.1,
  res5 3, the new classifier 10 / 20.
- adam_odd_p_1 / _2 / _3: small layouts with P = 1, 2, 3 (mod 4), so Adam's second-moment half (hist + P) is 4-, 8-
  or 16-byte misaligned.
"""
import numpy as np

SMALL_COUNTS = (1, 2, 3, 5, 7, 64, 333)
LR_MULTS = (0.0, 0.1, 0.7, 1.0, 3.0, 10.0, 20.0)
DECAY_MULTS = (0.0, 0.1, 0.3, 1.0, 3.0)

SEG_SIZES = (511, 512, 513, 1023, 1024, 1025, 3000)

# Caffe ResNet-152: bottleneck blocks per stage and the stage's middle width (in units of the base width)
_RESNET152_STAGES = ((3, 1), (8, 2), (36, 4), (3, 8))
RESNET152_BLOBS = 932       # 155 convolutions x (conv + BatchNorm 3 + Scale 2) + fc weight and bias


def _seg_layout(nseg):
    rng = np.random.RandomState(1000 + nseg)
    counts = rng.choice(SMALL_COUNTS, nseg).astype(np.int64)
    nbig = 2 + nseg % 2
    for k in rng.choice(nseg, nbig, replace=False):
        counts[k] = rng.randint(10 ** 4, 10 ** 5)
    # one run of three 1-element blobs whose ends are 1, 2 and 3 (mod 4): a float4 that straddles three blob ends
    m = nseg // 2
    e = int(counts[:m - 1].sum()) % 4
    counts[m - 1] = {0: 1, 1: 64, 2: 3, 3: 2}[e]
    counts[m:m + 3] = 1
    lr = rng.choice(LR_MULTS, nseg)
    dm = rng.choice(DECAY_MULTS, nseg)
    return [int(c) for c in counts], [float(x) for x in lr], [float(x) for x in dm]


def _empty_blobs():
    # first; 5 | 0 | 3 share the float4 [4, 8); two in a row after 333 and after 2; last
    counts = [0, 5, 0, 3, 7, 333, 0, 0, 1, 1, 1, 64, 12345, 2, 0, 0, 3, 7, 20011, 64, 5, 0, 2, 0]
    rng = np.random.RandomState(77)
    lr = [float(x) for x in rng.choice(LR_MULTS[1:], len(counts))]
    dm = [float(x) for x in rng.choice(DECAY_MULTS[1:], len(counts))]
    return counts, lr, dm


def _resnet152_bn_like(width=8, classes=1000):
    """Blob sequence of Caffe's ResNet-152 (conv1, res2a..res5c with projection shortcuts on the first block of each
    stage, fc1000) at base width `width` (64 in the real net)."""
    counts, lr, dm = [], [], []

    def conv(cin, cout, k, lr_mult):
        counts.append(cout * cin * k * k)   # bias_term: false
        lr.append(lr_mult)
        dm.append(1.0)
        counts.extend([cout, cout, 1])      # BatchNorm: mean, variance, moving-average factor
        lr.extend([0.0, 0.0, 0.0])
        dm.extend([0.0, 0.0, 0.0])
        counts.extend([cout, cout])         # Scale: gamma, beta
        lr.extend([lr_mult, lr_mult])
        dm.extend([0.0, 0.0])

    conv(3, width, 7, 0.1)                  # early layers barely move when fine-tuning
    cin = width
    for stage, (blocks, mid_units) in enumerate(_RESNET152_STAGES):
        mid, out = mid_units * width, 4 * mid_units * width
        lr_mult = (0.1, 1.0, 1.0, 3.0)[stage]  # res2 nearly frozen, res5 adapts faster
        for b in range(blocks):
            if b == 0:
                conv(cin, out, 1, lr_mult)  # branch1 projection
            conv(cin, mid, 1, lr_mult)      # branch2a
            conv(mid, mid, 3, lr_mult)      # branch2b
            conv(mid, out, 1, lr_mult)      # branch2c
            cin = out
    counts.extend([classes * cin, classes])  # the new classifier: lr_mult 10 / 20, decay 1 / 0
    lr.extend([10.0, 20.0])
    dm.extend([1.0, 0.0])
    return counts, lr, dm


def _adam_odd_p(residue):
    counts = [4096, 7, 333, 5, 64, 2, 10240 + residue, 3, 1]
    counts[-1] += (residue - sum(counts)) % 4
    lr = [0.1, 0.7, 3.0, 10.0, 20.0, 0.7, 1.0, 3.0, 0.1]
    dm = [1.0, 0.1, 0.3, 3.0, 0.0, 1.0, 0.1, 0.3, 3.0]
    return counts, lr, dm


def _build():
    out = {f"seg_{n}": _seg_layout(n) for n in SEG_SIZES}
    out["empty_blobs"] = _empty_blobs()
    out["resnet152_bn_like"] = _resnet152_bn_like()
    for r in (1, 2, 3):
        out[f"adam_odd_p_{r}"] = _adam_odd_p(r)
    return out


LAYOUTS = _build()
NAMES = sorted(LAYOUTS)
SEG_NAMES = [f"seg_{n}" for n in SEG_SIZES]
ADAM_ODD_P = ["adam_odd_p_1", "adam_odd_p_2", "adam_odd_p_3"]


def layout(name):
    """(counts, lr_mult, decay_mult) of a named layout, as fresh lists."""
    c, lm, dm = LAYOUTS[name]
    return list(c), list(lm), list(dm)


def ends(counts):
    return np.cumsum(np.asarray(counts, np.int64))


def blob_of_element(counts):
    """Index of the blob every element belongs to (zero-count blobs own no element)."""
    return np.repeat(np.arange(len(counts)), counts)


def max_ends_in_a_float4(counts, lo=0, hi=None):
    """Most blob ends strictly inside one 4-aligned float4 [4v, 4v+4) fully inside [lo, hi); repeated ends (a
    zero-count blob) count once per blob."""
    e = ends(counts)
    hi = int(e[-1]) if hi is None else hi
    inner = e[(e % 4 != 0) & (e > lo) & (e < hi)]
    inner = inner[(inner // 4 * 4 >= lo) & (inner // 4 * 4 + 4 <= hi)]
    if inner.size == 0:
        return 0
    return int(np.bincount(inner // 4).max())


def shard_cuts_inside_a_blob(counts, N, chunk):
    """True when some boundary between two of the N shards (chunk(P, N, r) -> (offset, size)) falls strictly inside
    a blob."""
    e = set(int(x) for x in ends(counts)) | {0}
    P = int(sum(counts))
    return any(chunk(P, N, r)[0] not in e for r in range(1, N))
