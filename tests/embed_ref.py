"""References for the built-in engine's Embed and Reshape (DESIGN.md section 14).

- embed_forward: Caffe's Embed forward in float64.  A valid id (an integer in [0, input_dim)) selects its table row;
  any other id (negative, too large, fractional, NaN, infinite) embeds as the zero vector.  The bias is added to every
  row.
- embed_backward_cpu: embed_layer.cpp Backward_cpu restated in fp32.  Each occurrence's dy row is added into its table
  row one at a time, in bottom order, starting from the value already in diff.  Invalid ids add nothing.
- reshape_shape: ReshapeLayer::LayerSetUp and Reshape's shape inference, with their CHECK wording.
"""
import numpy as np

F32 = np.float32


def valid_rows(ids, input_dim):
    """-> int64 array of the table row of each id, -1 where the id is not an integer in [0, input_dim)"""
    f = np.asarray(ids, F32).ravel().astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok = (f >= 0) & (f < input_dim) & (f == np.floor(f))
    return np.where(ok, np.nan_to_num(f), -1).astype(np.int64)


def embed_forward(ids, w, b=None):
    """float64 y = w[id] (+ b), shape ids.shape + (num_output,); zero rows (+ b) for invalid ids"""
    w = np.asarray(w, np.float64)
    rows = valid_rows(ids, w.shape[0])
    y = np.where((rows >= 0)[:, None], w[np.maximum(rows, 0)], 0.0)
    if b is not None:
        y = y + np.asarray(b, np.float64)
    return y.reshape(np.shape(ids) + (w.shape[1],))


def embed_backward_cpu(ids, dy, diff):
    """fp32 Backward_cpu: for n in bottom order, diff[id_n] += dy[n] (one rounding per element per occurrence).
    Returns a new array."""
    out = np.array(diff, F32, copy=True)
    rows = valid_rows(ids, out.shape[0])
    dy = np.asarray(dy, F32).reshape(rows.size, out.shape[1])
    for n, k in enumerate(rows):
        if k >= 0:
            out[k] = out[k] + dy[n]  # float32 + float32: one rounding per element
    return out


def embed_backward_summed_first(ids, dy, diff):
    """A plausible wrong order: each id's rows summed (in bottom order, from 0) before one add into diff"""
    out = np.array(diff, F32, copy=True)
    rows = valid_rows(ids, out.shape[0])
    dy = np.asarray(dy, F32).reshape(rows.size, out.shape[1])
    sums = {}
    for n, k in enumerate(rows):
        if k >= 0:
            sums[k] = sums.get(k, np.zeros(out.shape[1], F32)) + dy[n]
    for k, s in sums.items():
        out[k] = out[k] + s
    return out


def embed_bias_grad(ids, dy, num_output):
    """float64 sum of every dy row (invalid ids included, as Caffe's gemv does)"""
    return np.asarray(dy, np.float64).reshape(-1, num_output).sum(axis=0)


class ReshapeError(ValueError):
    pass


def reshape_shape(bottom, dims, axis=0, num_axes=-1, start_of=None):
    """ReshapeLayer's top shape of a bottom of shape `bottom` for reshape_param {shape {dim: dims} axis num_axes}, or
    ReshapeError with its CHECK wording.  `start_of` replaces the start-axis rule (for mutation tests)."""
    dims = list(dims)
    inferred, copies, constant = -1, [], 1
    for i, d in enumerate(dims):
        if d == 0:
            copies.append(i)
        elif d == -1:
            if inferred != -1:
                raise ReshapeError("new shape contains multiple -1 dims; at most a single (1) value of -1 may be "
                                   "specified")
            inferred = i
        else:
            constant *= d
    n = len(bottom)
    start = start_of(axis, n) if start_of else (axis if axis >= 0 else n + axis + 1)
    if start < 0:
        raise ReshapeError(f"axis {axis} out of range")
    if start > n:
        raise ReshapeError(f"axis {axis} out of range for {n}-D input blob")
    if num_axes < -1:
        raise ReshapeError("num_axes must be >= 0, or -1 for all")
    end = n if num_axes == -1 else start + num_axes
    if end > n:
        raise ReshapeError("end_axis = axis + num_axes is out of range")
    top = list(bottom[:start]) + dims + list(bottom[end:])
    for c in copies:
        if n <= start + c:
            raise ReshapeError("new shape contains a 0, but there was no corresponding bottom axis to copy")
        top[start + c] = bottom[start + c]
    count = int(np.prod(bottom, dtype=np.int64))
    if inferred >= 0:
        explicit = constant * int(np.prod(bottom[:start], dtype=np.int64)) * int(np.prod(bottom[end:], dtype=np.int64))
        for c in copies:
            explicit *= top[start + c]
        if explicit == 0 or count % explicit:
            raise ReshapeError(f"bottom count ({count}) must be divisible by the product of the specified dimensions "
                               f"({explicit})")
        top[start + inferred] = count // explicit
    if int(np.prod(top, dtype=np.int64)) != count:
        raise ReshapeError("output count must match input count")
    return tuple(int(v) for v in top)
