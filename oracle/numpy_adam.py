"""Independent restatement of the Adam step in vectorised float32 numpy (TEST INFRASTRUCTURE).

oracle/adam_oracle.c is the oracle the GPU tests use; this file restates the same iteration with numpy, written
separately from the C code, so the two can be cross-checked on random cases (tests/test_adam_host.py).  The
scale / reduce-scatter / on_start part is numpy_oracle.step's.
"""
import numpy as np

from .numpy_oracle import F, shard, step


def _libm_powf():
    import ctypes
    import ctypes.util
    f = ctypes.CDLL(ctypes.util.find_library("m")).powf
    f.argtypes, f.restype = [ctypes.c_float, ctypes.c_float], ctypes.c_float
    return np.vectorize(lambda x: f(x, 0.5), otypes=[F])


_powf_half_impl = None


def _powf_half(v):
    """libm's powf(v, 0.5f) element by element.  numpy's own float32 power is not libm's powf (and x**0.5 is
    sqrt): the two differ in the last bit on some inputs."""
    global _powf_half_impl
    if _powf_half_impl is None:
        _powf_half_impl = _libm_powf()
    return _powf_half_impl(v).astype(F)


def adam_correction(beta1, beta2, it):
    """adam_solver.cpp:39-41 for float32 betas: double throughout, rounded once to float."""
    t = it + 1
    return F(np.sqrt(1.0 - float(F(beta2)) ** t) / (1.0 - float(F(beta1)) ** t))


def step_adam(data, grads, hist, counts, lr_mult, decay_mult, rate, beta1, beta2, delta, weight_decay, it,
              regularization_type="L2"):
    """One Solver::Step of AdamSolver; hist[r] = concat(m, v) (2P).  Returns new (data, hist) lists."""
    N, P = len(data), data[0].size
    zero = [np.zeros(P, F) for _ in range(N)]
    # the scale / reduce / on_start part does not depend on the solver: reuse step() with a zero update
    data, _ = step(data, grads, zero, counts, lr_mult, decay_mult, 0.0, 0.0, 0.0)
    g = _reduced_grads(grads)
    corr = adam_correction(F(beta1), F(beta2), it)
    lrc = np.repeat((F(rate) * np.asarray(lr_mult, F)).astype(F) * corr, counts).astype(F)
    ld = np.repeat((F(weight_decay) * np.asarray(decay_mult, F)).astype(F), counts)
    b1, b2 = F(beta1), F(beta2)
    out_d, out_h = [], []
    for r in range(N):
        w = data[r]
        m, v = hist[r][:P].astype(F), hist[r][P:].astype(F)
        x = w if regularization_type == "L2" else np.sign(w).astype(F)
        gr = np.where(ld != 0, ld * x + g[r], g[r]).astype(F)
        m = ((F(1) - b1) * gr + (b1 * m).astype(F)).astype(F)
        v = ((F(1) - b2) * (gr * gr).astype(F) + (b2 * v).astype(F)).astype(F)
        t = _powf_half(v)                                # caffe_powx = vsPowx = libm powf
        t = ((m / (t + F(delta)).astype(F)).astype(F))
        upd = (lrc * t).astype(F)
        out_d.append((F(-1.0) * upd + w).astype(F))
        out_h.append(np.concatenate([m, v]))
    return out_d, out_h


def _reduced_grads(grads):
    """Per-rank gradient after scale + reduce-scatter (only the own shard is reduced; N == 1: unscaled)."""
    N, P = len(grads), grads[0].size
    g = [x.astype(F).copy() for x in grads]
    if N == 1:
        return g
    inv = F(1.0 / N)
    g = [inv * x for x in g]
    red = [x.copy() for x in g]
    for r in range(N):
        lo, hi = shard(P, N, r)
        s = g[r][lo:hi].copy()
        for j in range(1, N):
            s = g[(r + j) % N][lo:hi] + s
        red[r][lo:hi] = s
    return red
