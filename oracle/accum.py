"""ctypes binding of the iter_size CPU ORACLE (oracle/accum_oracle.c) -- TEST INFRASTRUCTURE.

Only tests/ and __graft_entry__ may import this module; the product package never does.  accum_oracle.c is linked
with sync_oracle.c and adam_oracle.c into _build/libaccum_oracle.so with the flags of oracle/Makefile, so every fp32
operation is rounded once.
"""
import ctypes
import os
import subprocess

import numpy as np

from . import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_build", "libaccum_oracle.so")
SOURCES = [os.path.join(HERE, n) for n in ("accum_oracle.c", "adam_oracle.c", "sync_oracle.c")]
DEPS = SOURCES + [os.path.join(HERE, "sync_oracle.h"),
                  os.path.join(HERE, "..", "caffeonspark_b200", "csrc", "powf_half.h")]

_lib = None


def build():
    """Compile libaccum_oracle.so when it is missing or older than its sources."""
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
        L.cos_oracle_accum_norm.argtypes = [i32]
        L.cos_oracle_accum_norm.restype = f32
        L.cos_oracle_accumulate.argtypes = [u64, pf, pf]
        L.cos_oracle_normalize.argtypes = [u64, pf, f32]
        L.cos_oracle_loss_mean.argtypes = [i32, pf]
        L.cos_oracle_loss_mean.restype = f32
        L.cos_oracle_step_accum.argtypes = [i32, u64, ppf, ppf, ppf, i32, pi64, pf, pf, f32, f32, f32, i32, f32, i32,
                                            f32, f32, i32]
        _lib = L
    return _lib


def accum_norm(iter_size):
    """Dtype(1.) / iter_size (sgd_solver.cpp:118-142)."""
    return float(np.float32(lib().cos_oracle_accum_norm(int(iter_size))))


def loss_mean(losses):
    """Solver::Step's loss over the passes (solver.cpp:221-224), in float."""
    a = np.ascontiguousarray(losses, dtype=np.float32)
    return float(np.float32(lib().cos_oracle_loss_mean(a.size, O._pf(a))))


def accumulate(grads_per_pass):
    """diff_ after the passes, starting from the zeroed diff_: [pass][rank] -> [rank]."""
    N, P = len(grads_per_pass[0]), grads_per_pass[0][0].size
    diff = [np.zeros(P, np.float32) for _ in range(N)]
    for grads in grads_per_pass:
        for r in range(N):
            lib().cos_oracle_accumulate(P, O._pf(diff[r]), O._pf(np.ascontiguousarray(grads[r], np.float32)))
    return diff


def step_accum(data, diff, hist, counts, lr_mult, decay_mult, rate, momentum, weight_decay, iter_size, it=0,
               regularization_type="L2", solver_type="SGD", momentum2=0.999, delta=1e-8):
    """The update half of one Solver::Step on len(data) simulated ranks (in place): diff[r] holds rank r's
    accumulated gradient; hist[r] holds P floats (SGD) or 2P (Adam: m, then v)."""
    c, lm, dm = O._layout(counts, lr_mult, decay_mult)
    N, P = len(data), data[0].size
    lib().cos_oracle_step_accum(N, P, O._ppf(data), O._ppf(diff), O._ppf(hist), len(c),
                                c.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), O._pf(lm), O._pf(dm), rate,
                                momentum, weight_decay, int(regularization_type == "L1"), accum_norm(iter_size),
                                int(solver_type == "Adam"), momentum2, delta, int(it))


class AccumSimulation(O.Simulation):
    """oracle.Simulation with iter_size passes per step, SGD or Adam.  step() takes the per-pass gradients
    [pass][rank] (or one list [rank] of already accumulated gradients via step_accumulated)."""

    def __init__(self, N, counts, lr_mult=None, decay_mult=None, iter_size=1, solver_type="SGD", momentum2=0.999,
                 delta=1e-8, **kw):
        super().__init__(N, counts, lr_mult, decay_mult, **kw)
        self.iter_size, self.solver_type, self.momentum2, self.delta = iter_size, solver_type, momentum2, delta
        if solver_type == "Adam":
            self.hist = [np.zeros(2 * self.P, np.float32) for _ in range(N)]

    def pass_gradient(self, rank, it, k):
        """Seeded synthetic gradient of pass k of step it on rank r."""
        g = O.fill(self.P, self.seed, (it + 1) * 4096 + 256 * k + rank, self.g_amp)
        return O.round_bf16(g) if self.bf16 else g

    def step(self, grads_per_pass=None):
        if grads_per_pass is None:
            grads_per_pass = [[self.pass_gradient(r, self.iter, k) for r in range(self.N)]
                              for k in range(self.iter_size)]
        assert len(grads_per_pass) == self.iter_size
        return self.step_accumulated(accumulate(grads_per_pass))

    def step_accumulated(self, diff):
        diff = [np.ascontiguousarray(g, dtype=np.float32).copy() for g in diff]
        rate = self.rate()
        step_accum(self.data, diff, self.hist, self.counts, self.lr_mult, self.decay_mult, rate, self.hp["momentum"],
                   self.hp["weight_decay"], self.iter_size, self.iter, self.regularization_type, self.solver_type,
                   self.momentum2, self.delta)
        self.iter += 1
        return rate

    def consistent_v(self):
        out = np.empty(self.P, np.float32)
        for r in range(self.N):
            o, s = O.chunk(self.P, self.N, r)
            out[o:o + s] = self.hist[r][self.P + o:self.P + o + s]
        return out
