#!/usr/bin/env python
"""bench_iter_size.py -- gradient accumulation (iter_size k) on CaffeNet b256, one GPU.

  python bench_iter_size.py [--runs 3] [--steps 30] [--warmup 10] [--sizes 1,2,4] [--out FILE]

For every k in --sizes, --runs runs, alternated (k = 1, 2, 4, 1, 2, 4, ...).  A run builds a CaffeNet net with
`iter_size: k` and the PyTorch producer (fp32, forward/backward captured in CUDA graphs), and trains with
train_accumulate(): k distinct host micro-batches of 256 images per step, staged and pipelined like train().
Reported per k (median and [min, max] over runs):
  * images/s and ms per step: host wall clock around --steps train_accumulate() calls and the final synchronize();
    a step processes k x 256 images;
  * forward/backward per pass: CUDA events around the producer's forward/backward on device-resident inputs;
  * the fused sync + update kernel in the step: the library's CUDA events around its launch during full steps.
The card name, power limit and maximum SM clock are read in the same process.  Prints one JSON line; writes
nothing in the tree (--out names the file to write, if any).
"""
import argparse
import gc
import json
import sys
import time

import bench  # emit; its import sends everything but the JSON line to stderr
from bench_producer_precision import card, stats

WORKLOAD = "caffenet"


def run_one(torch, cos, harness, nets, k, args):
    batch = nets.NETS[WORKLOAD]["batch"]
    c, h, w = nets.NETS[WORKLOAD]["input"]
    net = cos.CaffeNet(nets.solver_desc(WORKLOAD, iter_size=k))
    try:
        assert net.connect(net.localAddresses()), net.last_error()
        prod = harness.make_producer(WORKLOAD, net)
        g = torch.Generator().manual_seed(1)
        xs = [torch.rand((batch, c, h, w), generator=g).pin_memory() for _ in range(k)]
        ys = [torch.randint(0, nets.NETS[WORKLOAD]["classes"], (batch,), generator=g).float().pin_memory()
              for _ in range(k)]
        micro = [[xs[q], ys[q]] for q in range(k)]
        for _ in range(args.warmup):  # every (staging set, pass) reaches its CUDA-graph replay
            assert net.train_accumulate(0, micro), net.last_error()
        assert net.synchronize(), net.last_error()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            if not net.train_accumulate(0, micro):
                raise RuntimeError(net.last_error())
        if not net.synchronize():
            raise RuntimeError(net.last_error())
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        # the fused kernel inside full steps (library-side events around the launch)
        net.set_option("timing", 1)
        kms = []
        for _ in range(10):
            assert net.train_accumulate(0, micro), net.last_error()
            kms.append(net.last_kernel_ms())
        net.set_option("timing", 0)
        assert net.synchronize(), net.last_error()
        # forward/backward of one pass, device-resident inputs, eager (same kernels as the graph replays)
        x_dev, y_dev = xs[0].cuda(), ys[0].cuda().long()
        fb = []
        for _ in range(10):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            prod.forward_backward(x_dev, y_dev)
            b.record()
            fb.append((a, b))
        torch.cuda.synchronize()
        net.diff().zero_()
        torch.cuda.synchronize()
        return {"images_per_s": k * batch * args.steps / s, "ms_per_step": 1e3 * s / args.steps,
                "fb_ms_per_pass": sorted(a.elapsed_time(b) for a, b in fb)[5],
                "sync_kernel_in_step_ms": sorted(kms)[len(kms) // 2], "last_loss": net.last_loss()}
    finally:
        net.deallocate()
        del net
        gc.collect()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--sizes", default="1,2,4")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_iter_size.py needs a CUDA device (there is no CPU path)")
    import caffeonspark_b200 as cos
    from caffeonspark_b200 import harness, nets
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    sizes = [int(x) for x in args.sizes.split(",")]
    keys = ("images_per_s", "ms_per_step", "fb_ms_per_pass", "sync_kernel_in_step_ms")
    res = {k: {key: [] for key in keys} for k in sizes}
    for r in range(args.runs):
        for k in sizes:
            out = run_one(torch, cos, harness, nets, k, args)
            for key in keys:
                res[k][key].append(out[key])
            print(f"[iter_size] k={k} run {r}: {out['images_per_s']:.0f} images/s, {out['ms_per_step']:.3f} ms/step, "
                  f"fb {out['fb_ms_per_pass']:.3f} ms/pass, sync kernel {out['sync_kernel_in_step_ms'] * 1e3:.1f} us, "
                  f"loss {out['last_loss']:.4f}", file=sys.stderr, flush=True)
    summary = {str(k): {key: stats(v) for key, v in res[k].items()} for k in sizes}
    out = {"card": card(), "workload": f"{WORKLOAD} b256 per pass, N=1, fp32 producer (CUDA graphs)",
           "P": nets.solver_desc(WORKLOAD).param_count, "runs": args.runs, "steps": args.steps,
           "warmup": args.warmup, "iter_size": summary}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    bench.emit(out)


if __name__ == "__main__":
    main()
