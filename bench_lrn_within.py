"""Time per call and achieved bandwidth of the within-channel LRN kernels (DESIGN.md section 10).

Shapes: cifar10_full's norm1 (100x32x16x16) and norm2 (100x32x8x8) at b100, n = 3, and a larger plane
(32x64x128x128) with n = 3 and n = 9.  For each shape and dtype (fp32, bf16), CUDA events time `--iters` back-to-back
forward calls and, separately, backward calls on one stream after `--warmup` untimed ones, `--rounds` times.  The
bandwidth is the minimum traffic over the median time: forward reads x and writes y (2 tensors), backward reads x
and dy and writes dx (3 tensors); halo re-reads are not counted.  Prints one JSON line per case with the card's name
and power limit.  Needs a GPU (no CPU path).
"""
import argparse
import json
import subprocess

import torch

from caffeonspark_b200 import layers

CASES = [("cifar10_full norm1 b100", (100, 32, 16, 16), 3), ("cifar10_full norm2 b100", (100, 32, 8, 8), 3),
         ("large plane", (32, 64, 128, 128), 3), ("large plane", (32, 64, 128, 128), 9)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines() or [", "])[0].split(", ")[:2]
    return name, power


def time_ms(fn, iters, warmup, rounds):
    for _ in range(warmup):
        fn()
    samples = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        samples.append(a.elapsed_time(b) / iters)
    samples.sort()
    return samples[len(samples) // 2], samples[0], samples[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lrn_within.py needs a GPU (there is no CPU path)"
    name, power = card()
    lib = layers._lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    for what, shape, n in CASES:
        for dtype in (torch.float32, torch.bfloat16):
            g = torch.Generator(device="cuda").manual_seed(1)
            x = (40 * torch.randn(shape, device="cuda", generator=g)).to(dtype)
            dy = torch.randn(shape, device="cuda", generator=g).to(dtype)
            y, dx = torch.empty_like(x), torch.empty_like(x)
            sfx = "" if dtype == torch.float32 else "_bf16"
            fwd_fn, bwd_fn = getattr(lib, "cos_lrn_within_forward" + sfx), getattr(lib, "cos_lrn_within_backward" + sfx)

            def fwd():
                assert fwd_fn(x.data_ptr(), y.data_ptr(), *shape, n, 5e-05, 0.75, stream)

            def bwd():
                assert bwd_fn(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), *shape, n, 5e-05, 0.75, stream)

            nbytes = x.numel() * x.element_size()
            for direction, fn, tensors in (("forward", fwd, 2), ("backward", bwd, 3)):
                med, lo, hi = time_ms(fn, args.iters, args.warmup, args.rounds)
                print(json.dumps(dict(case=what, shape=list(shape), local_size=n, dtype=str(dtype).split(".")[1],
                                      direction=direction, ms_median=round(med, 5), ms_min=round(lo, 5),
                                      ms_max=round(hi, 5), min_bytes=tensors * nbytes,
                                      gb_per_s=round(tensors * nbytes / med / 1e6, 1), gpu=name, power_limit=power)),
                      flush=True)


if __name__ == "__main__":
    main()
