#!/usr/bin/env python
"""bench_mvn.py -- Caffe's MVN layer on the native kernels (csrc/mvn.cu, DESIGN.md section 14), one GPU.

  python bench_mvn.py [--iters 50] [--warmup 10]

For each shape, one forward and one backward through cos_mvn_forward / cos_mvn_backward, against eager PyTorch
running the same formulas (layers._mvn_formula_forward / _mvn_formula_backward) on the same device.  The shapes are
ones users run, with at least one on each side of every regime threshold of mvn.hpp: lanes (dim <= 16), a warp
(dim <= 512), a block per row, and split rows (dim >= 16384 with fewer than 1024 rows).  Kernel time is the sum of the
CUDA kernels' device time per call in a torch.profiler run; achieved bytes/s count the least traffic from the shape
(forward: read x, write y, 8 B per element; backward: read y and dy, write dx, 12 B), and bound_us is that traffic
at the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line per shape with the card's name and power limit read in
the same run; writes nothing in the tree.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PEAK_BPS = 3.35e12
# (name, bottom shape, across_channels, normalize_variance)
SHAPES = [("resnet_plane", (64, 64, 56, 56), False, True),         # rows 4096, dim 3136: a block per row
          ("cifar_plane", (256, 32, 32, 32), False, True),          # rows 8192, dim 1024: a block per row
          ("layer_norm", (20, 32, 1024), False, True),              # rows 640, dim 1024: a block per row
          ("layer_norm_512", (20, 32, 512), False, True),           # rows 640, dim 512: a warp per row
          ("layer_norm_mean_only", (20, 32, 1024), False, False),
          ("across_28", (32, 256, 28, 28), True, True),             # rows 32, dim 200,704: split rows
          ("across_224", (2, 64, 224, 224), True, True),            # rows 2, dim 3,211,264: split rows
          ("across_224_mean_only", (2, 64, 224, 224), True, False),
          ("across_16k_1024_rows", (1024, 16, 32, 32), True, True), # rows 1024, dim 16,384: a block per row
          ("across_16k_1023_rows", (1023, 16, 32, 32), True, True), # rows 1023, dim 16,384: split rows
          ("tiny_channels", (262144, 8, 1, 1), False, True),        # rows 2,097,152, dim 1: lanes
          ("tiny_rows", (262144, 8, 1, 1), True, True),             # rows 262,144, dim 8: lanes
          ("rows_of_17", (262144, 17), True, True)]                 # rows 262,144, dim 17: a warp per row


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from caffeonspark_b200 import _lib, layers

    if not torch.cuda.is_available():
        raise SystemExit("bench_mvn.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    L = _lib.lib()
    for name, shape, across, variance in SHAPES:
        n, c = layers.legacy_shape(shape)[:2]
        rows = n * (1 if across else c)
        count = 1
        for d in shape:
            count *= d
        dim = count // rows
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(count, device="cuda", generator=g) * 2 + 0.5
        dy = torch.randn(count, device="cuda", generator=g)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        stats = torch.empty(5 * rows, device="cuda")
        work = torch.empty(max(1, L.cos_mvn_workspace_floats(rows, dim)), device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def forward():
            assert L.cos_mvn_forward(x.data_ptr(), y.data_ptr(), stats.data_ptr(), work.data_ptr(), rows, dim,
                                     int(variance), 1e-9, stream), L.cos_last_error()

        def backward():
            assert L.cos_mvn_backward(y.data_ptr(), dy.data_ptr(), dx.data_ptr(), stats.data_ptr(), work.data_ptr(),
                                      rows, dim, int(variance), stream), L.cos_last_error()

        x2, dy2 = x.view(rows, dim), dy.view(rows, dim)
        saved = {}

        def torch_forward():
            saved["y"], saved["s"] = layers._mvn_formula_forward(x2, rows, dim, variance, 1e-9)

        def torch_backward():
            layers._mvn_formula_backward(saved["y"], dy2, saved["s"], dim)

        res = {"bench": "mvn", "case": name, "shape": list(shape), "across_channels": across,
               "normalize_variance": variance, "rows": rows, "dim": dim, "gpu": gpu, "iters": args.iters}
        for label, fn, nbytes in (("native_forward", forward, 8 * count), ("native_backward", backward, 12 * count),
                                  ("torch_forward", torch_forward, 8 * count),
                                  ("torch_backward", torch_backward, 12 * count)):
            if label == "native_backward":
                forward()
            if label == "torch_backward":
                torch_forward()
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    fn()
                torch.cuda.synchronize()
            ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
                  and "Memset" not in e.name]
            us = sum(e.device_time for e in ks) / args.iters
            res[label] = {"kernel_us": round(us, 2), "launches": len(ks) // args.iters,
                          "achieved_TBps": round(nbytes / us / 1e6, 3) if us > 0 else "not measured",
                          "bound_us": round(nbytes / PEAK_BPS * 1e6, 2),
                          "share_of_bound": round(nbytes / PEAK_BPS * 1e6 / us, 3) if us > 0 else "not measured"}
        print(json.dumps(res), flush=True)
        del x, dy, y, dx, stats, work, saved
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
