"""A float64 numpy restatement of Caffe's RNN layer (rnn_layer.cpp's unrolled net, recurrent_layer.cpp without
expose_hidden): the forward, backpropagation through time and the hidden state carried from call to call.

    hc_{t-1} = cont_t * h_{t-1}                          (Scale h_conted_{t-1})
    h_t      = tanh(W_hh hc_{t-1} + (W_xh x_t + b_h) + W_xh_static x_static)   (Eltwise SUM, TanH)
    o_t      = tanh(W_ho h_t + b_o)

h_{-1} is the state the previous call left (zero at first).  The gradient stops at h_{-1}: nothing crosses into the
previous call.  Blobs are a dict with the keys of BLOBS; `mutation` names a plausible wrong version, for the tests that
show the checks catch it."""
import numpy as np

BLOBS = ["w_xh", "b_h", "w_xh_static", "w_hh", "w_ho", "b_o"]
MUTATIONS = ["cont_on_h_t", "w_hh_transposed", "state_not_carried", "grad_across_calls", "static_dropped",
             "no_output_tanh", "blob_order_swapped"]


def blob_shapes(I, H, S=0):
    """The blobs' shapes in the layer's blob order (W_xh_static only with S)."""
    shapes = {"w_xh": (H, I), "b_h": (H,), "w_xh_static": (H, S), "w_hh": (H, H), "w_ho": (H, H), "b_o": (H,)}
    return [(k, shapes[k]) for k in BLOBS if S or k != "w_xh_static"]


def unpack(flat, I, H, S=0, mutation=None):
    """Flat learnable blobs in the layer's order -> dict."""
    order = blob_shapes(I, H, S)
    if mutation == "blob_order_swapped":
        names = [k for k, _ in order]
        a, b = names.index("w_hh"), names.index("w_ho")
        order[a], order[b] = order[b], order[a]
    out, off = {}, 0
    for k, s in order:
        n = int(np.prod(s))
        out[k] = np.asarray(flat[off:off + n], np.float64).reshape(s)
        off += n
    return out


def pack(blobs):
    return np.concatenate([np.ravel(blobs[k]) for k in BLOBS if k in blobs])


def forward(W, x, cont, h0, x_static=None, mutation=None):
    """-> (o [T, N, H], h [T + 1, N, H] with h[0] = h_{-1}).  x is [T, N, ...], cont [T, N], h0 [N, H]."""
    T, N = cont.shape
    x = np.asarray(x, np.float64).reshape(T, N, -1)
    cont = np.asarray(cont, np.float64)
    whh = W["w_hh"].T if mutation == "w_hh_transposed" else W["w_hh"]
    g = x @ W["w_xh"].T + W["b_h"]
    z = 0.0
    if x_static is not None and mutation != "static_dropped":
        z = np.asarray(x_static, np.float64).reshape(N, -1) @ W["w_xh_static"].T
    h = [np.asarray(h0, np.float64)]
    for t in range(T):
        if mutation == "cont_on_h_t":  # the flush applied after the step instead of before
            h.append(cont[t][:, None] * np.tanh(h[-1] @ whh.T + g[t] + z))
        else:
            h.append(np.tanh((cont[t][:, None] * h[-1]) @ whh.T + g[t] + z))
    h = np.stack(h)
    a = h[1:] @ W["w_ho"].T + W["b_o"]
    return (a if mutation == "no_output_tanh" else np.tanh(a)), h


def backward(W, x, cont, h0, dtop, x_static=None, mutation=None, dh_last=None):
    """-> (grads dict of the blobs, dx, dx_static or None, dh_{-1}).  dtop is the top's gradient [T, N, H]; dh_last is
    a gradient reaching h_{T-1} from outside the call (only the grad_across_calls mutation uses it)."""
    T, N = cont.shape
    xs = np.asarray(x, np.float64).reshape(T, N, -1)
    cont = np.asarray(cont, np.float64)
    whh = W["w_hh"].T if mutation == "w_hh_transposed" else W["w_hh"]
    o, h = forward(W, x, cont, h0, x_static, mutation)
    dz_o = dtop * (1.0 if mutation == "no_output_tanh" else 1 - o ** 2)
    g = {"w_ho": np.einsum("tnj,tnk->jk", dz_o, h[1:]), "b_o": dz_o.sum(axis=(0, 1))}
    dh_o = dz_o @ W["w_ho"]
    dpre = np.zeros_like(dh_o)
    dh = np.zeros((N, dh_o.shape[2])) if dh_last is None else dh_last
    for t in range(T - 1, -1, -1):
        dpre[t] = (dh_o[t] + dh) * (1 - h[t + 1] ** 2)
        dh = cont[t][:, None] * (dpre[t] @ whh)
    hc = cont[:, :, None] * h[:-1]
    gw = np.einsum("tnj,tnk->jk", dpre, hc)
    g["w_hh"] = gw.T if mutation == "w_hh_transposed" else gw
    g["w_xh"] = np.einsum("tnj,tnk->jk", dpre, xs)
    g["b_h"] = dpre.sum(axis=(0, 1))
    dx = (dpre @ W["w_xh"]).reshape(np.shape(x))
    dxs = None
    if x_static is not None:
        dz = dpre.sum(axis=0) if mutation != "static_dropped" else np.zeros_like(dpre[0])
        xst = np.asarray(x_static, np.float64).reshape(N, -1)
        g["w_xh_static"] = dz.T @ xst
        dxs = (dz @ W["w_xh_static"]).reshape(np.shape(x_static))
    return g, dx, dxs, dh


def run_calls(W, calls, h0=None, mutation=None):
    """Consecutive calls [(x, cont, dtop, x_static)] of one layer.  Each starts from the state the previous left (zero
    at first) and backpropagates inside itself alone.  -> [(o, grads, dx, dx_static)] and the final state."""
    H = W["w_hh"].shape[0]
    N = calls[0][1].shape[1]
    state = np.zeros((N, H)) if h0 is None else np.asarray(h0, np.float64)
    out = []
    for x, cont, dtop, xs in calls:
        start = np.zeros((N, H)) if mutation == "state_not_carried" else state
        o, h = forward(W, x, cont, start, xs, mutation)
        out.append([o, *backward(W, x, cont, start, dtop, xs, mutation)[:3]])
        state = h[-1]
    if mutation == "grad_across_calls":  # each call's dh_{-1} sent back into the previous one's last step
        state = np.zeros((N, H)) if h0 is None else np.asarray(h0, np.float64)
        starts = []
        for x, cont, dtop, xs in calls:
            starts.append(state)
            state = forward(W, x, cont, state, xs)[1][-1]
        dh = None
        for i in range(len(calls) - 1, -1, -1):
            x, cont, dtop, xs = calls[i]
            g, dx, dxs, dh = backward(W, x, cont, starts[i], dtop, xs, dh_last=dh)
            out[i][1:] = [g, dx, dxs]
    return out, state
