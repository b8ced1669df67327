#!/usr/bin/env python
"""bench_unet.py -- Caffe's Crop on the built-in engine's kernels and the U-Net fixture's training step (DESIGN.md
section 14), one GPU.

  python bench_unet.py [--iters 50] [--steps 50] [--warmup 10]

Crop alone: forward and backward through layers.crop_forward / crop_backward at the U-Net fixture's three crops (skip
40 -> 32 and 88 -> 56 at 32 and 16 channels, the label 92 -> 52) and one large map, [8, 64, 392, 392] -> 200 x 200,
against eager PyTorch (a strided copy of the window; a zero fill and a strided copy into it).  Kernel times are the
medians of the calls' device time in a torch.profiler run.  The least traffic is computed from the shape: the forward
reads and writes the top (8 B per top element), the backward reads dy and writes all of dx (4 B per top element and 4
B per bottom element); bound_us is that traffic at the H100 SXM data sheet's 3.35 TB/s.

U-Net (tests/golden/configs/unet_solver.prototxt, b8): one forward + backward on the engine (CUDA events) and one
train() step (forward, backward and the fused SGD update; host clock around a synchronised window), against the eager
PyTorch fp32 mirror (nets.unet_module, TF32 off) doing the same forward, backward and SGD momentum update.  A
torch.profiler run of the engine's forward + backward then says where its time goes: each kernel's share, and the
single-block softmax_loss_kernel over the 21,632 pixel rows in particular.  Prints one JSON line per measurement with
the card's name and power limit read in the same run; writes nothing in the tree.
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
# (name, bottom, top, offsets)
CROPS = [("unet_crop2", (8, 32, 40, 40), (8, 32, 32, 32), (0, 0, 4, 4)),
         ("unet_crop1", (8, 16, 88, 88), (8, 16, 56, 56), (0, 0, 16, 16)),
         ("unet_label", (8, 1, 92, 92), (8, 1, 52, 52), (0, 0, 20, 20)),
         ("large_map", (8, 64, 392, 392), (8, 64, 200, 200), (0, 0, 96, 96))]


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


def kernel_median_us(torch, profile, ProfilerActivity, fn, iters, warmup):
    """median over calls of the device time of the kernels (and memsets) one call launches"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name]
    per = len(ks) // iters
    return statistics.median(sum(e.device_time for e in ks[i * per:(i + 1) * per]) for i in range(iters)), per


def bench_crop(torch, profile, ProfilerActivity, gpu, iters, warmup):
    from caffeonspark_b200 import layers
    for name, bottom, top, offs in CROPS:
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(bottom, device="cuda", generator=g)
        dy = torch.randn(top, device="cuda", generator=g)
        y, dx = torch.empty(top, device="cuda"), torch.empty(bottom, device="cuda")
        window = tuple(slice(o, o + t) for o, t in zip(offs, top))

        def torch_backward():
            dx.zero_()
            dx[window].copy_(dy)

        res = {"bench": "crop", "case": name, "bottom": list(bottom), "top": list(top), "offsets": list(offs),
               "gpu": gpu, "iters": iters}
        nt, nb = count(top), count(bottom)
        for label, fn, nbytes in (("native_forward", lambda: layers.crop_forward(x, top, offs, out=y), 8 * nt),
                                  ("native_backward", lambda: layers.crop_backward(dy, bottom, offs, out=dx),
                                   4 * (nt + nb)),
                                  ("torch_forward", lambda: y.copy_(x[window]), 8 * nt),
                                  ("torch_backward", torch_backward, 4 * (nt + nb))):
            us, launches = kernel_median_us(torch, profile, ProfilerActivity, fn, iters, warmup)
            res[label] = {"kernel_us_median": round(us, 2), "launches": launches,
                          "achieved_TBps": round(nbytes / us / 1e6, 3) if us > 0 else "not measured",
                          "bound_us": round(nbytes / PEAK_BPS * 1e6, 2),
                          "share_of_bound": round(nbytes / PEAK_BPS * 1e6 / us, 3) if us > 0 else "not measured"}
        print(json.dumps(res), flush=True)
        del x, dy, y, dx
        torch.cuda.empty_cache()


def batches(np, n, count_):
    """images of three bright disks on noise and their per-pixel labels, as the tests draw them"""
    rng = np.random.RandomState(0)
    yy, xx = np.mgrid[0:92, 0:92]
    out = []
    for _ in range(count_):
        mask = np.zeros((n, 1, 92, 92), np.float32)
        for i in range(n):
            for _ in range(3):
                cy, cx, r = rng.randint(10, 82), rng.randint(10, 82), rng.randint(8, 20)
                mask[i, 0][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 1
        out.append([(0.7 * mask + 0.3 * rng.rand(n, 1, 92, 92)).astype(np.float32), mask])
    return out


def bench_unet(C, np, torch, profile, ProfilerActivity, gpu, iters, steps, warmup):
    from caffeonspark_b200 import nets
    solver = os.path.join(ROOT, "tests", "golden", "configs", "unet_solver.prototxt")
    n = nets.UNET["batch"]
    host = batches(np, n, 8)
    dev = [[torch.from_numpy(v).cuda() for v in b] for b in host]
    net = C.CaffeNet(solver, "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=True)
    loss = torch.zeros(1, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    torch.cuda.set_stream(stream)

    def call(i):
        assert net.forward_backward(dev[i % 8], loss.data_ptr(), stream=stream.cuda_stream), net.last_error()

    for i in range(warmup):
        call(i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        call(i)
    b.record()
    b.synchronize()
    fb_ms = a.elapsed_time(b) / iters
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(iters):
            call(i)
        torch.cuda.synchronize()
    torch.cuda.set_stream(torch.cuda.default_stream())
    by_name = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            by_name[e.name] = by_name.get(e.name, 0.0) + e.device_time / 1e3 / iters
    kernels_ms = sum(by_name.values())
    top = sorted(by_name.items(), key=lambda kv: -kv[1])[:8]
    softmax = sum(v for k, v in by_name.items() if "softmax_loss_kernel" in k)
    crop = sum(v for k, v in by_name.items() if "crop_" in k)

    for i in range(warmup):
        assert net.train(0, host[i % 8]), net.last_error()
    assert net.synchronize(), net.last_error()
    t0 = time.perf_counter()
    for i in range(steps):
        assert net.train(0, host[i % 8]), net.last_error()
    assert net.synchronize(), net.last_error()
    train_ms = (time.perf_counter() - t0) * 1e3 / steps
    net.deallocate()

    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    m = nets.unet_module().cuda()
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=0.0005)
    labels = [m.crop_label(bt[1]).reshape(-1).long() for bt in dev]

    def torch_fb(i):
        scores = m(dev[i % 8][0])
        torch.nn.functional.cross_entropy(scores.permute(0, 2, 3, 1).reshape(-1, 2), labels[i % 8]).backward()

    def torch_step(i):
        opt.zero_grad()
        torch_fb(i)
        opt.step()

    timings = {}
    for label, fn in (("fb", torch_fb), ("step", torch_step)):
        for i in range(warmup):
            fn(i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(steps):
            fn(i)
        torch.cuda.synchronize()
        timings[label] = (time.perf_counter() - t0) * 1e3 / steps
    print(json.dumps({"bench": "unet", "gpu": gpu, "batch": n, "iters": iters, "steps": steps,
                      "native_forward_backward_ms": round(fb_ms, 4),
                      "native_train_ms": round(train_ms, 4),
                      "pytorch_fp32_eager_forward_backward_ms": round(timings["fb"], 4),
                      "pytorch_fp32_eager_step_ms": round(timings["step"], 4),
                      "native_kernels_ms_per_call": round(kernels_ms, 4),
                      "softmax_loss_kernel_ms": round(softmax, 4),
                      "softmax_loss_share_of_kernels": round(softmax / kernels_ms, 3) if kernels_ms else "not measured",
                      "crop_kernels_ms": round(crop, 4),
                      "top_kernels_ms": [[k[:90], round(v, 4)] for k, v in top]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import caffeonspark_b200 as C

    if not torch.cuda.is_available():
        raise SystemExit("bench_unet.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    bench_crop(torch, profile, ProfilerActivity, gpu, args.iters, args.warmup)
    bench_unet(C, np, torch, profile, ProfilerActivity, gpu, args.iters, args.steps, args.warmup)


if __name__ == "__main__":
    main()
