#!/usr/bin/env python
"""bench_tile.py -- Caffe's Tile layer on the built-in engine's kernels (DESIGN.md section 14) and the SE-ResNet-20
fixture's training step, one GPU.

  python bench_tile.py [--iters 50] [--steps 30] [--warmup 10]

Workloads, on both sides of the staged backward's threshold (inner 32): the fixtures' own tiles (SE-ResNet-20 at b100,
its 16- and 64-channel stages; U-Net scSE at b8, its channel gate along H and W and its spatial gate over the
channels), an ImageNet-scale SE gate (b32, [32, 256, 1, 1] tiled to 56 x 56, along H and then W) and an sSE gate
([32, 1, 56, 56] tiled over 256 channels).  The gates are tiled along an axis of size 1, so eager PyTorch's
expand().contiguous() forward and sum(axis) backward compute the same values; they are timed beside the kernels for
comparison only (their sums are not Caffe's order).

Kernel times are medians over calls of the device time in a torch.profiler run.  The least traffic is computed from
the shapes: each direction reads one of bottom and top and writes the other; bound_us is it at the H100 SXM data
sheet's 3.35 TB/s.  The fixture (tests/golden/configs/cifar10_se_resnet20_solver.prototxt, b100): one train() step
(forward, backward and the fused SGD update; host clock around a synchronised window) against the eager PyTorch fp32
mirror (nets.se_resnet20_module, TF32 off) doing the same forward, backward and SGD momentum update.  Prints one JSON
line per measurement with the card's name, power limit and maximum SM clock read in the same run; writes nothing in
the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PEAK_BPS = 3.35e12
# (name, bottom, axis, tiles)
WORKLOADS = [
    ("se_resnet20_res2_h", (100, 16, 1, 1), 2, 32), ("se_resnet20_res2_w", (100, 16, 32, 1), 3, 32),
    ("se_resnet20_res4_h", (100, 64, 1, 1), 2, 8), ("se_resnet20_res4_w", (100, 64, 8, 1), 3, 8),
    ("unet_scse4_c_h", (8, 32, 1, 1), 2, 28), ("unet_scse4_c_w", (8, 32, 28, 1), 3, 28),
    ("unet_scse4_s", (8, 1, 28, 28), 1, 32), ("unet_scse5_s", (8, 1, 52, 52), 1, 16),
    ("imagenet_se_h", (32, 256, 1, 1), 2, 56), ("imagenet_se_w", (32, 256, 56, 1), 3, 56),
    ("imagenet_sse", (32, 1, 56, 56), 1, 256),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def count(shape):
    n = 1
    for d in shape:
        n *= d
    return n


def device_us(torch, profile, ProfilerActivity, fn, iters, warmup):
    """median over calls of the summed device time of the kernels one call launches"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
            torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name]
    per = len(ks) // iters
    return statistics.median(sum(e.device_time for e in ks[i * per:(i + 1) * per]) for i in range(iters))


def bench_kernels(torch, profile, ProfilerActivity, gpu, iters, warmup):
    from caffeonspark_b200 import layers
    for name, bottom, axis, tiles in WORKLOADS:
        top = layers.tile_top_shape(bottom, axis, tiles)
        x = torch.randn(bottom, device="cuda")
        y = torch.empty(top, device="cuda")
        dy = torch.randn(top, device="cuda")
        dx = torch.empty(bottom, device="cuda")
        outer = count(bottom[:axis])
        inner = count(bottom) // outer
        bound = 4 * (count(bottom) + count(top)) / PEAK_BPS * 1e6
        fwd = device_us(torch, profile, ProfilerActivity, lambda: layers.tile_forward(x, axis, tiles, out=y), iters,
                        warmup)
        bwd = device_us(torch, profile, ProfilerActivity,
                        lambda: layers.tile_backward(dy, bottom, axis, tiles, out=dx), iters, warmup)
        expand = [tiles if k == axis else -1 for k in range(len(bottom))]
        tf = device_us(torch, profile, ProfilerActivity, lambda: x.expand(*expand).contiguous(), iters, warmup)
        tb = device_us(torch, profile, ProfilerActivity, lambda: dy.sum(axis, keepdim=True), iters, warmup)
        print(json.dumps({"bench": "tile", "workload": name, "gpu": gpu, "bottom": list(bottom), "axis": axis,
                          "tiles": tiles, "inner": inner, "backward": "staged" if inner < 32 else "direct",
                          "bound_us": round(bound, 2), "forward_us": round(fwd, 2), "backward_us": round(bwd, 2),
                          "forward_pct_of_bound": round(100 * bound / fwd, 1),
                          "backward_pct_of_bound": round(100 * bound / bwd, 1),
                          "pytorch_expand_contiguous_us": round(tf, 2), "pytorch_sum_us": round(tb, 2)}), flush=True)
        del x, y, dy, dx
        torch.cuda.empty_cache()


def bench_fixture(C, np, torch, gpu, steps, warmup):
    from caffeonspark_b200 import nets
    cfg = os.path.join(ROOT, "tests", "golden", "configs")
    n = nets.RESNET20["batch"]
    rng = np.random.RandomState(0)
    host = [[rng.rand(n, 3, 32, 32).astype(np.float32), rng.randint(0, 10, n).astype(np.float32)] for _ in range(8)]
    net = C.CaffeNet(os.path.join(cfg, "cifar10_se_resnet20_solver.prototxt"), "", "", 1, 1, 0, True,
                     C.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=True)
        for i in range(warmup):
            assert net.train(0, host[i % 8]), net.last_error()
        assert net.synchronize(), net.last_error()
        t0 = time.perf_counter()
        for i in range(steps):
            assert net.train(0, host[i % 8]), net.last_error()
        assert net.synchronize(), net.last_error()
        train_ms = (time.perf_counter() - t0) * 1e3 / steps
    finally:
        net.deallocate()

    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    m = nets.se_resnet20_module().cuda()
    opt = torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    dev = [[torch.from_numpy(v).cuda() for v in b] for b in host]

    def step(i):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(m(dev[i % 8][0]), dev[i % 8][1].long()).backward()
        opt.step()

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(i)
    torch.cuda.synchronize()
    torch_ms = (time.perf_counter() - t0) * 1e3 / steps
    print(json.dumps({"bench": "cifar10_se_resnet20", "gpu": gpu, "batch": n, "steps": steps,
                      "native_train_ms": round(train_ms, 4), "pytorch_fp32_eager_step_ms": round(torch_ms, 4)}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import caffeonspark_b200 as C

    if not torch.cuda.is_available():
        raise SystemExit("bench_tile.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    bench_kernels(torch, profile, ProfilerActivity, gpu, args.iters, args.warmup)
    bench_fixture(C, np, torch, gpu, args.steps, args.warmup)


if __name__ == "__main__":
    main()
