#!/usr/bin/env python
"""bench_batchnorm.py -- the native BatchNorm kernels (csrc/batch_norm.cu, DESIGN.md section 13), one GPU.

  python bench_batchnorm.py [--iters 50] [--runs 3] [--steps 50] [--warmup 10] [--out FILE]

Per kernel: training-mode forward and backward, fp32 and bf16, at the cifar10_full_bn shapes (batch 100) and at
ResNet-50-like shapes (batch 64), timed with CUDA events over --iters launches after a warm-up.  Next to the native
kernels: the PyTorch composite of the same formulas (layers.batch_norm_composite) and cuDNN's F.batch_norm.  Bytes
come from the byte model below; TB/s is over the H100 SXM data-sheet 3.35 TB/s.

Step: cifar10_full_bn b100 at N = 1 with the fp32 and the bf16 producer, native BatchNorm against the composite,
--runs alternated runs each of bench.py's measure_workload; images/s as median [min, max].

Prints one JSON line with the card name, power limit and maximum SM clock read in the same process; writes nothing
in the tree (--out names the file to write, if any).
"""
import argparse
import functools
import json
import os
import tempfile
import types

import bench  # measure_workload, emit; its import sends everything but the JSON line to stderr
from bench_producer_precision import card, stats

PEAK_TBS = 3.35
SHAPES = {"cifar10_full_bn/bn1": (100, 32, 16, 16), "cifar10_full_bn/bn3": (100, 64, 8, 8),
          "resnet50/conv1": (64, 64, 112, 112), "resnet50/res2": (64, 256, 56, 56),
          "resnet50/res5": (64, 2048, 7, 7)}


def byte_model(numel, esize):
    """minimum traffic, and what the native design moves: the forward reads x three times (mean, variance,
    normalise) and writes y; the backward reads x and dy twice (channel sums, dx) and writes dx"""
    return {"forward": {"minimum": 2 * numel * esize, "native": 4 * numel * esize},
            "backward": {"minimum": 3 * numel * esize, "native": 5 * numel * esize}}


def _time(torch, fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us


def kernels(args):
    import torch
    import torch.nn.functional as F
    from caffeonspark_b200 import layers
    out = {}
    for name, shape in SHAPES.items():
        for dt in (torch.float32, torch.bfloat16):
            g = torch.Generator(device="cuda").manual_seed(1)
            x = (torch.randn(shape, device="cuda", generator=g) + 1).to(dt)
            dy = torch.randn(shape, device="cuda", generator=g).to(dt)
            c = shape[1]
            stats_ = [torch.zeros(c, device="cuda"), torch.zeros(c, device="cuda"), torch.zeros(1, device="cuda")]
            xr = x.detach().requires_grad_(True)
            # forward alone, then forward + backward (backward = the difference), for all three implementations
            impl = {
                "native": lambda: layers.BatchNormFunction.apply(xr, *stats_, False, 0.999, 1e-5),
                "composite": lambda: layers.batch_norm_composite(xr, *stats_),
                "cudnn": lambda: F.batch_norm(xr, None, None, training=True, eps=1e-5),
            }
            esize = x.element_size()
            bm = byte_model(x.numel(), esize)
            row = {"bytes": bm}
            for k, f in impl.items():
                with torch.no_grad():
                    fwd = _time(torch, f, args.iters)

                def fb(f=f):
                    xr.grad = None
                    f().backward(dy)
                fwdbwd = _time(torch, fb, args.iters)
                bwd = max(fwdbwd - fwd, 1e-9)
                row[k] = {"forward_us": fwd, "backward_us": bwd,
                          "forward_TBs_min_bytes": bm["forward"]["minimum"] / fwd / 1e6,
                          "backward_TBs_min_bytes": bm["backward"]["minimum"] / bwd / 1e6}
                if k == "native":
                    row[k]["forward_TBs_moved"] = bm["forward"]["native"] / fwd / 1e6
                    row[k]["backward_TBs_moved"] = bm["backward"]["native"] / bwd / 1e6
                    row[k]["forward_share_of_3.35"] = row[k]["forward_TBs_moved"] / PEAK_TBS
                    row[k]["backward_share_of_3.35"] = row[k]["backward_TBs_moved"] / PEAK_TBS
            key = f"{name} {tuple(shape)} {str(dt).split('.')[-1]}"
            out[key] = row
            n = row["native"]
            print(f"[bn] {key}: native fwd {n['forward_us']:.1f} us ({n['forward_TBs_moved']:.2f} TB/s moved), "
                  f"bwd {n['backward_us']:.1f} us ({n['backward_TBs_moved']:.2f} TB/s moved); composite "
                  f"{row['composite']['forward_us']:.1f}/{row['composite']['backward_us']:.1f}; cudnn "
                  f"{row['cudnn']['forward_us']:.1f}/{row['cudnn']['backward_us']:.1f}", flush=True)
    return out


def composite_producer(harness, name, net, precision, **kw):
    """make_producer with every BatchNorm module evaluated by the PyTorch composite instead of the native kernels"""
    from caffeonspark_b200 import layers, nets
    mod = nets.torch_module(name)
    for m in mod.modules():
        if isinstance(m, layers.BatchNorm):
            m.forward = functools.partial(lambda m, x: layers.batch_norm_composite(
                x, m.mean, m.variance, m.scale_factor, m.use_global_stats, m.moving_average_fraction, m.eps), m)
    return harness.TorchProducer(net, mod, precision=precision, **kw)


def steps(args):
    import numpy as np
    import torch
    import torch.distributed as dist
    import caffeonspark_b200 as C
    from caffeonspark_b200 import harness, nets
    torch.backends.cudnn.benchmark = True
    bargs = argparse.Namespace(algo=0, kernel=-1, nvls=-1, no_graph=False, steps=args.steps, warmup=args.warmup,
                               dump_outputs="", no_cpu_baseline=True)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.runs):
            for p in ("fp32", "bf16"):
                for impl in ("native", "composite"):
                    if impl == "native":
                        mk = functools.partial(harness.make_producer, precision=p)
                    else:
                        mk = lambda name, net, p=p, **kw: composite_producer(harness, name, net, p, **kw)  # noqa
                    shim = types.SimpleNamespace(Cluster=harness.Cluster, make_producer=mk)
                    bargs.dump_outputs = os.path.join(tmp, f"{p}_{impl}_{r}")
                    o, _ = bench.measure_workload(torch, dist, C, shim, nets, bargs, "cifar10_full_bn", "fp32", 0, 1,
                                                  0, primary=True)
                    d = res.setdefault(p, {}).setdefault(impl, {"images_per_s": [], "loss": []})
                    d["images_per_s"].append(o["value"])
                    d["loss"].append(float(np.load(os.path.join(bargs.dump_outputs, "loss.npy"))[0]))
                    print(f"[bn] step {p} {impl} run {r}: {o['value']:.0f} images/s", flush=True)
    return {p: {i: {"images_per_s": stats(d["images_per_s"]), "loss": d["loss"]} for i, d in v.items()}
            for p, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_batchnorm.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    res = {"card": card(), "kernels": kernels(args), "steps": steps(args), "card_after": card()}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    bench.emit(res)


if __name__ == "__main__":
    main()
