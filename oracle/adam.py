"""ctypes binding of the Adam CPU ORACLE (oracle/adam_oracle.c) -- TEST INFRASTRUCTURE.

Only tests/ and __graft_entry__ may import this module; the product package never does.  adam_oracle.c is linked
with sync_oracle.c (on_start, scale, reduce-scatter) into _build/libadam_oracle.so with the flags of
oracle/Makefile, so every fp32 operation is rounded once.
"""
import concurrent.futures as cf
import ctypes
import os
import subprocess

import numpy as np

from . import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_build", "libadam_oracle.so")
SOURCES = [os.path.join(HERE, "adam_oracle.c"), os.path.join(HERE, "sync_oracle.c")]
DEPS = SOURCES + [os.path.join(HERE, "sync_oracle.h"),
                  os.path.join(HERE, "..", "caffeonspark_b200", "csrc", "powf_half.h")]

_lib = None


def build():
    """Compile libadam_oracle.so when it is missing or older than its sources."""
    if os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in DEPS):
        return
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                    "-shared", "-o", LIB_PATH] + SOURCES + ["-lm"], check=True)


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(LIB_PATH)
        u64, i32, f32 = ctypes.c_uint64, ctypes.c_int, ctypes.c_float
        pf = ctypes.POINTER(ctypes.c_float)
        ppf = ctypes.POINTER(pf)
        pi64 = ctypes.POINTER(ctypes.c_int64)
        L.cos_oracle_adam_correction.argtypes = [f32, f32, i32]
        L.cos_oracle_adam_correction.restype = f32
        L.cos_oracle_apply_update_adam.argtypes = [u64, u64, u64, pf, pf, pf, i32, pi64, pf, pf, f32, f32, f32, f32,
                                                   f32, i32, i32]
        L.cos_oracle_step_adam.argtypes = [i32, u64, ppf, ppf, ppf, i32, pi64, pf, pf, f32, f32, f32, f32, f32, i32,
                                           i32]
        L.cos_oracle_powf_half_check.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(u64)]
        L.cos_oracle_powf_half_fill.argtypes = [ctypes.c_uint32, ctypes.c_uint32, pf]
        _lib = L
    return _lib


def adam_correction(beta1, beta2, it):
    """sqrt(1 - beta2^t) / (1 - beta1^t), t = it + 1, as adam_solver.cpp:39-41 rounds it."""
    return float(np.float32(lib().cos_oracle_adam_correction(beta1, beta2, int(it))))


def step_adam(data, diff, hist, counts, lr_mult, decay_mult, rate, beta1, beta2, delta, weight_decay, it,
              regularization_type="L2"):
    """One Solver::Step of an Adam solver on len(data) simulated ranks (in place); hist[r] holds 2P floats
    (m, then v) and `it` is the iteration before the step."""
    c, lm, dm = O._layout(counts, lr_mult, decay_mult)
    N, P = len(data), data[0].size
    assert all(h.size == 2 * P for h in hist)
    lib().cos_oracle_step_adam(N, P, O._ppf(data), O._ppf(diff), O._ppf(hist), len(c),
                               c.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), O._pf(lm), O._pf(dm), rate, beta1,
                               beta2, delta, weight_decay, int(regularization_type == "L1"), int(it))


def powf_half_check(lo, hi):
    """(inputs where powf(x, 0.5f) != sqrtf(x), inputs where powf differs from the kernels' restatement) over
    the float bit patterns [lo, hi)."""
    out = (ctypes.c_uint64 * 2)()
    lib().cos_oracle_powf_half_check(lo, hi, out)
    return out[0], out[1]


def powf_half_fill(lo, hi, out=None, threads=None):
    """libm's powf(x, 0.5f) for the float bit patterns [lo, hi), as a float32 array (into `out` when given), filled
    by `threads` threads (default: one per CPU); ctypes releases the GIL during each chunk."""
    n = hi - lo
    out = np.empty(n, np.float32) if out is None else out
    assert out.dtype == np.float32 and out.size == n and out.flags.c_contiguous
    k = max(1, min(threads or os.cpu_count() or 1, n))
    cuts = [lo + n * i // k for i in range(k + 1)]
    L = lib()
    with cf.ThreadPoolExecutor(k) as ex:
        list(ex.map(lambda i: L.cos_oracle_powf_half_fill(cuts[i], cuts[i + 1], O._pf(out[cuts[i] - lo:])),
                    range(k)))
    return out


class AdamSimulation(O.Simulation):
    """oracle.Simulation with an Adam solver: hist[r] holds 2P floats, m of every blob then v of every blob.
    momentum is beta1."""

    def __init__(self, N, counts, lr_mult=None, decay_mult=None, momentum2=0.999, delta=1e-8, solver_type="Adam",
                 **kw):
        assert solver_type == "Adam", solver_type
        super().__init__(N, counts, lr_mult, decay_mult, **kw)
        self.momentum2, self.delta = momentum2, delta
        self.hist = [np.zeros(2 * self.P, np.float32) for _ in range(N)]

    def step(self, grads=None):
        diff = grads if grads is not None else [self.gradient(r, self.iter) for r in range(self.N)]
        diff = [np.ascontiguousarray(g, dtype=np.float32).copy() for g in diff]
        rate = self.rate()
        step_adam(self.data, diff, self.hist, self.counts, self.lr_mult, self.decay_mult, rate, self.hp["momentum"],
                  self.momentum2, self.delta, self.hp["weight_decay"], self.iter, self.regularization_type)
        self.iter += 1
        return rate

    def consistent_v(self):
        """The owners' second moments (hist[P:]), concatenated."""
        out = np.empty(self.P, np.float32)
        for r in range(self.N):
            o, s = O.chunk(self.P, self.N, r)
            out[o:o + s] = self.hist[r][self.P + o:self.P + o + s]
        return out
