"""Time per call and achieved bandwidth of the native bias+ReLU+max-pool and cross-channel LRN calls at CaffeNet b256's
shapes and CIFAR-10-quick's conv1 block.  The pool calls are timed with the staged kernels (the fast path) and with the
reference kernels forced (`cos_layers_set_reference_kernels`), alternated round by round in one process; the switch
does not select an LRN kernel, so the LRN calls are timed once, as path "unaffected" (DESIGN.md section 10).

For each case, dtype (fp32, bf16), direction and arm, CUDA events time `--iters` back-to-back calls on one stream,
`--rounds` times after `--warmup` untimed calls.  The pool backward call includes its bias-gradient pass.  The
bandwidth is the minimum traffic over the median time, each tensor read or written once: pool forward reads x and
writes y and the 1-byte index, pool backward reads dy and index and writes dx (the same bytes); LRN forward reads x
and writes y, LRN backward reads x and dy and writes dx.  Prints one JSON line per case, direction and dtype with the
card's name, power limit and SM clock.  Needs a GPU (no CPU path).
"""
import argparse
import json
import subprocess

import torch

from caffeonspark_b200 import _lib

# name, (N, C, H, W) of the bias-free conv output, pool kernel, stride
POOL_CASES = [("caffenet conv1 pool block b256", (256, 96, 55, 55), 3, 2),
              ("caffenet conv2 pool block b256", (256, 256, 27, 27), 3, 2),
              ("caffenet conv5 pool block b256", (256, 256, 13, 13), 3, 2),
              ("cifar10_quick conv1 pool block b100", (100, 32, 32, 32), 3, 2)]
# name, (N, C, H, W), local_size
LRN_CASES = [("caffenet norm1 b256", (256, 96, 27, 27), 5), ("caffenet norm2 b256", (256, 256, 13, 13), 5)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    fields = (q.stdout.strip().splitlines() or [", , "])[0].split(", ")
    return (fields + ["", "", ""])[:3]


def time_arms(fn, lib, iters, warmup, rounds):
    """median, min, max ms per call of fn with the fast path ("fast") and the reference kernels ("reference"),
    alternated within every round"""
    samples = {"fast": [], "reference": []}
    for ref in (0, 1):
        lib.cos_layers_set_reference_kernels(ref)
        for _ in range(warmup):
            fn()
    for _ in range(rounds):
        for arm, ref in (("fast", 0), ("reference", 1)):
            lib.cos_layers_set_reference_kernels(ref)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            samples[arm].append(a.elapsed_time(b) / iters)
    lib.cos_layers_set_reference_kernels(0)
    out = {}
    for arm, s in samples.items():
        s.sort()
        out[arm] = (s[len(s) // 2], s[0], s[-1])
    return out


def time_one(fn, iters, warmup, rounds):
    """median, min, max ms per call of fn with the switch off (for calls the switch does not affect)"""
    for _ in range(warmup):
        fn()
    s = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        s.append(a.elapsed_time(b) / iters)
    s.sort()
    return s[len(s) // 2], s[0], s[-1]


def report(what, shape, dtype, direction, arms, nbytes, gpu, extra):
    for arm, (med, lo, hi) in arms.items():
        print(json.dumps(dict(case=what, shape=list(shape), dtype=str(dtype).split(".")[1], direction=direction,
                              path=arm, us_median=round(med * 1e3, 2), us_min=round(lo * 1e3, 2),
                              us_max=round(hi * 1e3, 2), min_bytes=nbytes, gb_per_s=round(nbytes / med / 1e6, 1),
                              gpu=gpu[0], power_limit=gpu[1], sm_clock=gpu[2], **extra)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_layers.py needs a GPU (there is no CPU path)"
    lib = _lib.lib()
    gpu = card()
    stream = torch.cuda.current_stream().cuda_stream
    for dtype in (torch.float32, torch.bfloat16):
        sfx = "" if dtype == torch.float32 else "_bf16"
        for what, shape, k, s in POOL_CASES:
            n, c, h, w = shape
            ph, pw = (h - k + s - 1) // s + 1, (w - k + s - 1) // s + 1
            g = torch.Generator(device="cuda").manual_seed(1)
            x = torch.randn(shape, device="cuda", generator=g).to(dtype)
            bias = 0.1 * torch.randn(c, device="cuda", generator=g)
            y = torch.empty((n, c, ph, pw), device="cuda", dtype=dtype)
            index = torch.empty((n, c, ph, pw), device="cuda", dtype=torch.uint8)
            dy = torch.randn((n, c, ph, pw), device="cuda", generator=g).to(dtype)
            dx = torch.empty_like(x)
            partials = torch.empty(n * c, device="cuda")
            dbias = torch.empty(c, device="cuda")
            fwd_fn = getattr(lib, "cos_bias_relu_maxpool_forward" + sfx)
            bwd_fn = getattr(lib, "cos_bias_relu_maxpool_backward" + sfx)

            def fwd():
                assert fwd_fn(x.data_ptr(), bias.data_ptr(), y.data_ptr(), index.data_ptr(), *shape, k, s, ph, pw,
                              stream)

            def bwd():
                assert bwd_fn(dy.data_ptr(), index.data_ptr(), dx.data_ptr(), partials.data_ptr(), dbias.data_ptr(),
                              *shape, k, s, ph, pw, stream)

            fwd()
            nbytes = x.numel() * x.element_size() + y.numel() * y.element_size() + index.numel()
            extra = dict(kernel=k, stride=s, fast_path=bool(lib.cos_pool_fast_path(n, c, h, w, k, s)))
            for direction, fn in (("forward", fwd), ("backward", bwd)):
                report(what, shape, dtype, direction, time_arms(fn, lib, args.iters, args.warmup, args.rounds),
                       nbytes, gpu, extra)
        for what, shape, size in LRN_CASES:
            g = torch.Generator(device="cuda").manual_seed(1)
            x = (40 * torch.randn(shape, device="cuda", generator=g)).to(dtype)
            dy = torch.randn(shape, device="cuda", generator=g).to(dtype)
            y, dx = torch.empty_like(x), torch.empty_like(x)
            fwd_fn, bwd_fn = getattr(lib, "cos_lrn_forward" + sfx), getattr(lib, "cos_lrn_backward" + sfx)

            def lfwd():
                assert fwd_fn(x.data_ptr(), y.data_ptr(), *shape, size, 1e-4, 0.75, 1.0, stream)

            def lbwd():
                assert bwd_fn(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), *shape, size, 1e-4, 0.75, 1.0, stream)

            nb = x.numel() * x.element_size()
            for direction, fn, tensors in (("forward", lfwd, 2), ("backward", lbwd, 3)):
                # the switch does not select an LRN kernel: one arm, labelled as such
                report(what, shape, dtype, direction,
                       {"unaffected": time_one(fn, args.iters, args.warmup, args.rounds)}, tensors * nb, gpu,
                       dict(local_size=size))


if __name__ == "__main__":
    main()
