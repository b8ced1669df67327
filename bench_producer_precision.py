#!/usr/bin/env python
"""bench_producer_precision.py -- the fp32 and the bf16 (autocast) gradient producer side by side, one GPU.

  python bench_producer_precision.py [--runs 3] [--steps 50] [--warmup 10] [--out FILE]
  python bench_producer_precision.py --profile [--out FILE]

Timing mode: for CaffeNet b256, LeNet b64 and CIFAR-10-quick b100, --runs runs of each precision, alternated,
each one bench.py's measure_workload (the same device-timed steps, L2 flush and forward/backward split as bench.py,
so the numbers compare with DESIGN.md section 5) with make_producer(..., precision=p).  Reports the median and
[min, max] of images/s, ms per step and forward/backward ms, the loss after the timed steps (same seeds for both
precisions), and the card name, power limit and maximum SM clock read in the same process.

Profile mode (a run of its own: tracing slows the host): torch.profiler over 10 graph-replayed CaffeNet b256
forward/backwards per precision, kernel time per category, and each native layer kernel's time and achieved
bandwidth on the minimum-traffic byte table of its activation dtype (DESIGN.md section 10).

Prints one JSON line; writes nothing in the tree (--out names the file to write, if any).
"""
import argparse
import functools
import json
import os
import re
import subprocess
import sys
import tempfile
import types

import bench  # measure_workload, emit; its import sends everything but the JSON line to stderr

WORKLOADS = ("caffenet", "lenet", "cifar10_quick")
PRECISIONS = ("fp32", "bf16")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (c.strip() for c in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # the numbers are still reported, marked as not attributed to a card
        return {"error": f"nvidia-smi: {e}"}


def stats(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1], "all": v}


def timing(args):
    import numpy as np
    import torch
    import torch.distributed as dist
    import caffeonspark_b200 as C
    from caffeonspark_b200 import harness, nets
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    res = {w: {p: {"images_per_s": [], "ms_per_step": [], "forward_backward_ms": [], "loss": []} for p in PRECISIONS}
           for w in WORKLOADS}
    bargs = argparse.Namespace(algo=0, kernel=-1, nvls=-1, no_graph=False, steps=args.steps, warmup=args.warmup,
                               dump_outputs="", no_cpu_baseline=True)
    clocks = {}
    with tempfile.TemporaryDirectory() as tmp:
        for w in WORKLOADS:
            for r in range(args.runs):
                for p in PRECISIONS:
                    shim = types.SimpleNamespace(Cluster=harness.Cluster,
                                                 make_producer=functools.partial(harness.make_producer, precision=p))
                    bargs.dump_outputs = os.path.join(tmp, f"{w}_{p}_{r}")
                    out, _ = bench.measure_workload(torch, dist, C, shim, nets, bargs, w, "fp32", 0, 1, 0,
                                                    primary=True)
                    d = res[w][p]
                    d["images_per_s"].append(out["value"])
                    d["ms_per_step"].append(out["ms_per_step"])
                    d["forward_backward_ms"].append(out["split_ms"]["forward_backward"])
                    d["loss"].append(float(np.load(os.path.join(bargs.dump_outputs, "loss.npy"))[0]))
                    clocks.setdefault(w, {}).setdefault(p, []).append(out.get("clocks"))
                    print(f"[precision] {w} {p} run {r}: {out['value']:.0f} images/s, {out['ms_per_step']:.3f} "
                          f"ms/step, fb {out['split_ms']['forward_backward']:.3f} ms, loss {d['loss'][-1]:.6f}",
                          flush=True)
    summary = {}
    for w in WORKLOADS:
        summary[w] = {}
        for p in PRECISIONS:
            d = res[w][p]
            summary[w][p] = {k: stats(v) for k, v in d.items() if k != "loss"}
            summary[w][p]["loss_after_timed_steps"] = d["loss"]
            summary[w][p]["clocks"] = clocks[w][p]
        lf, lb = res[w]["fp32"]["loss"][0], res[w]["bf16"]["loss"][0]
        summary[w]["loss_gap"] = {"abs": abs(lb - lf), "rel": abs(lb - lf) / abs(lf) if lf else None}
    return {"mode": "timing", "runs": args.runs, "steps": args.steps, "warmup": args.warmup, "workloads": summary}


# CaffeNet b256 native layers: (tensor elements in, out) of each block, from the net's shapes
def byte_table(act_bytes):
    n = 256
    t = {}
    for name, (c, h, ph) in {"pool1": (96, 55, 27), "pool2": (256, 27, 13), "pool5": (256, 13, 6)}.items():
        x, y = n * c * h * h, n * c * ph * ph
        t[name] = {"forward": act_bytes * (x + y) + y, "backward": act_bytes * (y + x) + y}
    for name, (c, h) in {"norm1": (96, 27), "norm2": (256, 13)}.items():
        x = n * c * h * h
        t[name] = {"forward": 2 * act_bytes * x, "backward": 3 * act_bytes * x}
    return t


CATEGORIES = [  # first match wins; native kernels are matched before anything else
    ("native layers", r"lrn_forward_kernel|lrn_backward_kernel|pool_forward_kernel|pool_backward_kernel|"
                      r"bias_grad_kernel"),
    ("cuDNN NCHW<->NHWC transposes", r"nchwToNhwc|nhwcToNchw"),
    ("conv GEMMs (cuDNN / CUTLASS)", r"fprop|dgrad|wgrad|conv|implicit|cudnn"),
    ("FC GEMMs (cuBLAS)", r"gemm|nvjet|cublas|cutlass"),
    ("dtype casts and copies", r"copy_kernel|CopyKernel|_to_copy"),
    ("ReLU fwd + threshold_backward", r"threshold|relu|clamp"),
    ("reductions (bias grads, loss)", r"reduce_kernel|reduction"),
]


def profile(args):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import caffeonspark_b200 as C
    from caffeonspark_b200 import harness, nets
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    reps = 10
    out = {"mode": "profile", "forward_backwards": reps, "precisions": {}}
    for p in PRECISIONS:
        net = C.CaffeNet(nets.solver_desc("caffenet"))
        try:
            assert net.connect(net.localAddresses()), net.last_error()
            prod = harness.make_producer("caffenet", net, precision=p)
            g = torch.Generator().manual_seed(1)
            x = torch.rand((256, 3, 227, 227), generator=g).cuda()
            y = torch.randint(0, 1000, (256,), generator=g).cuda()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(3):
                    prod.forward_backward(x, y)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                prod.forward_backward(x, y)
            for _ in range(3):
                graph.replay()
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            for _ in range(reps):
                graph.replay()
            ev[1].record()
            torch.cuda.synchronize()
            event_ms = ev[0].elapsed_time(ev[1]) / reps
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    graph.replay()
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    k = kernels.setdefault(e.name, [0.0, 0])
                    k[0] += e.time_range.elapsed_us()  # a kernel event's interval is its device time
                    k[1] += 1
            cats = {}
            for name, (us, cnt) in kernels.items():
                cat = next((c for c, rx in CATEGORIES if re.search(rx, name, re.I)), "other (elementwise, dropout, "
                                                                                     "loss, memsets)")
                cats[cat] = cats.get(cat, 0.0) + us / reps
            native = {}
            for name, (us, cnt) in kernels.items():
                m = re.search(r"(lrn_forward_kernel|lrn_backward_kernel|pool_forward_kernel|pool_backward_kernel|"
                              r"bias_grad_kernel)<([^>]*)>|(bias_grad_kernel)", name)
                if m:
                    key = m.group(1) or m.group(3)
                    native[key] = {"us": native.get(key, {}).get("us", 0.0) + us / reps,
                                   "launches": native.get(key, {}).get("launches", 0) + cnt // reps,
                                   "instantiation": m.group(2)}
            tab = byte_table(2 if p == "bf16" else 4)
            fwd_pool = sum(tab[k]["forward"] for k in ("pool1", "pool2", "pool5"))
            bwd_pool = sum(tab[k]["backward"] for k in ("pool1", "pool2", "pool5"))
            fwd_lrn = sum(tab[k]["forward"] for k in ("norm1", "norm2"))
            bwd_lrn = sum(tab[k]["backward"] for k in ("norm1", "norm2"))
            bw = {}
            for key, nbytes in (("pool_forward_kernel", fwd_pool), ("lrn_forward_kernel", fwd_lrn),
                                ("lrn_backward_kernel", bwd_lrn)):
                if key in native:
                    bw[key] = {"us": native[key]["us"], "bytes": nbytes,
                               "TB_per_s": nbytes / (native[key]["us"] * 1e-6) / 1e12}
            if "pool_backward_kernel" in native:
                us = native["pool_backward_kernel"]["us"] + native.get("bias_grad_kernel", {}).get("us", 0.0)
                bw["pool_backward_kernel + bias_grad_kernel"] = {"us": us, "bytes": bwd_pool,
                                                                 "TB_per_s": bwd_pool / (us * 1e-6) / 1e12}
            out["precisions"][p] = {"forward_backward_ms_events": event_ms, "categories_us": cats,
                                    "native_kernels": native, "native_bandwidth": bw, "byte_table": tab,
                                    "top_kernels_us": sorted(((n[:120], v[0] / reps) for n, v in kernels.items()),
                                                             key=lambda t: -t[1])[:25]}
            del graph, prod
        finally:
            net.deallocate()
        torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_producer_precision.py needs a CUDA device (the producers have no CPU path)")
    res = profile(args) if args.profile else timing(args)
    res["card"] = card()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    bench.emit(res)


if __name__ == "__main__":
    sys.exit(main())
