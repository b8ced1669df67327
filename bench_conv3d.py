#!/usr/bin/env python
"""bench_conv3d.py -- Caffe's N-D Convolution and Deconvolution on the built-in engine (DESIGN.md section 14), one GPU.

  python bench_conv3d.py [--iters 20] [--steps 20] [--warmup 5] [--rounds 3]

Nets: the V-Net fixture (tests/golden/configs/vnet3d_solver.prototxt) at its own size (b2, 32^3) and at a size a user
would train (b2, 96^3: the same net with the volume and label tops at 96 x 96 x 96), and the C3D clip fixture (b4,
3 x 8 x 56 x 56).  For each:

- the engine's forward + backward under torch.profiler, with the device time per call of the three 3-D GEMM
  instantiations by their stable kernel names: gemm_kernel<DenseRM, Vol2col, StoreNCHW> (a Convolution's forward, a
  Deconvolution's data gradient), gemm_kernel<WeightT, Col2volGather, StoreNCHW> (a Convolution's data gradient, a
  Deconvolution's forward) and gemm_kernel<ChanMajor, Transposed<Vol2col>, StorePartial> (both weight gradients,
  before reduce_partials_kernel).  Their FLOPs come from the plan's shapes (2 M N K per GEMM; a bottom that wants no
  gradient runs no data-gradient GEMM), and the achieved rate is given as a share of the H100 SXM's FP32 data-sheet
  rate, 67 TFLOP/s.
- one train() step (forward, backward and the fused SGD update; host clock around a synchronised window) against the
  eager PyTorch fp32 mirror (nets.vnet3d_module / c3d_clip_module; cuDNN, TF32 off) doing the same forward, backward
  and SGD momentum update, in alternated runs: engine, PyTorch, engine, ... for --rounds rounds; the medians.

Prints one JSON line per net with the card's name and power limit read in the same run; writes nothing in the tree
(the 96^3 prototxts go to a temporary directory).
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
FP32_PEAK = 67e12
GEMMS = ("forward", "data_grad", "weight_grad")


def gemm_of(kernel):
    """which 3-D GEMM instantiation a kernel name (mangled or not) is, or None"""
    if "gemm_kernel" not in kernel:
        return None
    if "Col2volGather" in kernel:
        return "data_grad"
    if "Vol2col" in kernel:
        return "weight_grad" if "Transposed" in kernel else "forward"
    return None


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def solver_for(name, side, tmp):
    """the fixture's solver, or (vnet3d at another side) a copy whose volume and label tops are side^3"""
    solver = os.path.join(CONFIGS, f"{name}_solver.prototxt")
    if name != "vnet3d" or side == 32:
        return solver
    net = open(os.path.join(CONFIGS, "vnet3d_train_test.prototxt")).read()
    net = re.sub(r"(channels|height|width): 32\n", lambda m: f"{m.group(1)}: {side}\n", net)
    net = net.replace("      dim: 32\n", f"      dim: {side}\n")
    open(os.path.join(tmp, "vnet3d_train_test.prototxt"), "w").write(net)
    path = os.path.join(tmp, "vnet3d_solver.prototxt")
    open(path, "w").write(open(solver).read())
    return path


def gemm_flops(plan):
    """FLOPs per call of each 3-D GEMM instantiation, from the plan's 3-D Convolution and Deconvolution lines"""
    flops = dict.fromkeys(GEMMS, 0.0)
    for line in plan.splitlines():
        m = re.match(r"op \d+ (Convolution|Deconvolution) \S+ (\S+) -> (\S+) k(\d+)x(\d+)x(\d+) ", line)
        if not m:
            continue
        bottom, top = [[int(v) for v in s.split("x")] for s in m.groups()[1:3]]
        kk = int(m.group(4)) * int(m.group(5)) * int(m.group(6))
        # the convolution from its bottom to its top; a Deconvolution is the one from its top to its bottom
        x, y = (bottom, top) if m.group(1) == "Convolution" else (top, bottom)
        cin, cout, vox_x, vox_y = x[1], y[1], x[0] * x[2] * x[3] * x[4], y[0] * y[2] * y[3] * y[4]
        conv_fwd, conv_dgrad = 2.0 * cout * vox_y * cin * kk, 2.0 * cin * vox_x * cout * kk
        wants_dx = "staged-bottom" not in line and "no-bottom-grad" not in line
        if m.group(1) == "Convolution":
            flops["forward"] += conv_fwd
            flops["data_grad"] += conv_dgrad if wants_dx else 0.0
        else:
            flops["data_grad"] += conv_dgrad  # the Deconvolution's forward
            flops["forward"] += conv_fwd if wants_dx else 0.0
        flops["weight_grad"] += 2.0 * cout * cin * kk * vox_y
    return flops


def batches(np, name, side, n, count):
    rng = np.random.RandomState(0)
    if name == "vnet3d":
        return [[rng.rand(n, side, side, side).astype(np.float32),
                 (rng.rand(n, side, side, side) > 0.5).astype(np.float32)] for _ in range(count)]
    return [[rng.rand(n, 24, 56, 56).astype(np.float32), rng.randint(0, 10, (n, 1, 1, 1)).astype(np.float32)]
            for _ in range(count)]


def bench(C, np, torch, profile, ProfilerActivity, gpu, name, side, args, tmp):
    from caffeonspark_b200 import nets
    solver = solver_for(name, side, tmp)
    plan = C.native_producer_plan(solver)
    n = C.parse_solver(solver).batch_size
    host = batches(np, name, side, n, 4)
    dev = [[torch.from_numpy(v).cuda() for v in b] for b in host]
    net = C.CaffeNet(solver, "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=True)
    loss = torch.zeros(1, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()

    def call(i):
        assert net.forward_backward(dev[i % 4], loss.data_ptr(), stream=stream.cuda_stream), net.last_error()

    for i in range(args.warmup):
        call(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.iters):
            call(i)
        torch.cuda.synchronize()
    us = dict.fromkeys(GEMMS, 0.0)
    total = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        total += e.device_time / args.iters
        if gemm_of(e.name):
            us[gemm_of(e.name)] += e.device_time / args.iters
    flops = gemm_flops(plan)
    gemms = {k: {"kernel_us_per_call": round(us[k], 1), "gflop": round(flops[k] / 1e9, 3),
                 "tflops": round(flops[k] / us[k] / 1e6, 3) if us[k] > 0 else "not measured",
                 "share_of_fp32_peak": round(flops[k] / us[k] / 1e6 / (FP32_PEAK / 1e12), 3) if us[k] > 0
                 else "not measured"} for k in GEMMS}

    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    m = (nets.vnet3d_module() if name == "vnet3d" else nets.c3d_clip_module()).cuda()
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=0.0005)
    shape = (n, 1, side, side, side) if name == "vnet3d" else (n, 3, 8, 56, 56)
    xs = [b[0].view(shape) for b in dev]
    labels = [b[1].reshape(-1).long() for b in dev]

    def torch_step(i):
        opt.zero_grad()
        scores = m(xs[i % 4])
        if name == "vnet3d":
            scores = scores.permute(0, 2, 3, 4, 1).reshape(-1, 2)
        torch.nn.functional.cross_entropy(scores, labels[i % 4]).backward()
        opt.step()

    def native_block():
        t0 = time.perf_counter()
        for i in range(args.steps):
            assert net.train(0, host[i % 4]), net.last_error()
        assert net.synchronize(), net.last_error()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    def torch_block():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(args.steps):
            torch_step(i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    for i in range(args.warmup):
        assert net.train(0, host[i % 4]), net.last_error()
        torch_step(i)
    assert net.synchronize(), net.last_error()
    native, eager = [], []
    for _ in range(args.rounds):
        native.append(native_block())
        eager.append(torch_block())
    net.deallocate()
    print(json.dumps({"bench": "conv3d", "net": name, "gpu": gpu, "batch": n,
                      "input": list(shape[1:]), "iters": args.iters, "steps": args.steps, "rounds": args.rounds,
                      "native_kernels_us_per_forward_backward": round(total, 1), "gemms_3d": gemms,
                      "native_train_ms_median": round(statistics.median(native), 3),
                      "pytorch_fp32_eager_step_ms_median": round(statistics.median(eager), 3),
                      "native_train_ms": [round(v, 3) for v in native],
                      "pytorch_fp32_eager_step_ms": [round(v, 3) for v in eager]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import caffeonspark_b200 as C

    if not torch.cuda.is_available():
        raise SystemExit("bench_conv3d.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    with tempfile.TemporaryDirectory() as tmp:
        for name, side in (("vnet3d", 32), ("vnet3d", 96), ("c3d_clip", 0)):
            bench(C, np, torch, profile, ProfilerActivity, gpu, name, side, args, tmp)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
