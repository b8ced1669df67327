"""Independent restatement of an iter_size > 1 step in vectorised float32 numpy (TEST INFRASTRUCTURE).

oracle/accum_oracle.c is the oracle the GPU tests use; this file restates the same step with numpy, written
separately from the C code, so the two can be cross-checked on random cases (tests/test_iter_size_host.py).
Order: the passes add up in diff_, on_start + scale + reduce-scatter, then per rank Normalize (g = (1/k) * g,
sgd_solver.cpp:118-142), Regularize and the SGD or Adam update.
"""
import numpy as np

from .numpy_adam import _powf_half, _reduced_grads, adam_correction
from .numpy_oracle import F, step

__all__ = ["accumulate", "step_accum", "loss_mean"]


def accumulate(grads_per_pass):
    """diff_ of every rank after the passes, from a zeroed diff_."""
    out = [np.zeros_like(np.asarray(g, F)) for g in grads_per_pass[0]]
    for grads in grads_per_pass:
        out = [(np.asarray(g, F) + d).astype(F) for g, d in zip(grads, out)]
    return out


def loss_mean(losses):
    s = F(0)
    for x in losses:
        s = F(s + F(x))
    return F(s / F(len(losses)))


def step_accum(data, diff, hist, counts, lr_mult, decay_mult, rate, momentum, weight_decay, iter_size, it=0,
               regularization_type="L2", solver_type="SGD", momentum2=0.999, delta=1e-8):
    """Returns new (data, hist) lists for one step of len(data) ranks; diff[r] is rank r's accumulated gradient."""
    N, P = len(data), data[0].size
    zero = [np.zeros(P, F) for _ in range(N)]
    data, _ = step(data, diff, zero, counts, lr_mult, decay_mult, 0.0, 0.0, 0.0)  # on_start only (zero update)
    g = _reduced_grads(diff)
    if iter_size != 1:
        a = F(F(1.0) / F(iter_size))
        g = [(a * x).astype(F) for x in g]
    ld = np.repeat((F(weight_decay) * np.asarray(decay_mult, F)).astype(F), counts)
    out_d, out_h = [], []
    for r in range(N):
        w = data[r]
        x = w if regularization_type == "L2" else np.sign(w).astype(F)
        gr = np.where(ld != 0, ld * x + g[r], g[r]).astype(F)
        if solver_type == "Adam":
            lrc = np.repeat((F(rate) * np.asarray(lr_mult, F)).astype(F) * adam_correction(F(momentum), F(momentum2),
                                                                                            it), counts).astype(F)
            b1, b2 = F(momentum), F(momentum2)
            m, v = hist[r][:P].astype(F), hist[r][P:].astype(F)
            m = ((F(1) - b1) * gr + (b1 * m).astype(F)).astype(F)
            v = ((F(1) - b2) * (gr * gr).astype(F) + (b2 * v).astype(F)).astype(F)
            t = ((m / (_powf_half(v) + F(delta)).astype(F)).astype(F))
            out_d.append((F(-1.0) * (lrc * t).astype(F) + w).astype(F))
            out_h.append(np.concatenate([m, v]))
        else:
            lr = np.repeat((F(rate) * np.asarray(lr_mult, F)).astype(F), counts)
            h = (F(momentum) * hist[r]).astype(F)
            h = (lr * gr + h).astype(F)
            out_d.append((F(-1.0) * h + w).astype(F))
            out_h.append(h)
    return out_d, out_h
