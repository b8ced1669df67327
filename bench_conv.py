"""Time per call and achieved TF32 rate of the convolutions of CaffeNet b256, LeNet b64 and CIFAR-10-quick b100, per
layer and pass: the native implicit-GEMM kernels (csrc/conv_tf32.cu) against cuDNN on the same NCHW fp32 tensors with
TF32 allowed and its autotuner on, so cuDNN's times include its NCHW<->NHWC transposes (DESIGN.md section 10.2).

For each layer, pass and arm, CUDA events time `--iters` back-to-back calls on one stream, `--rounds` times after
`--warmup` untimed calls, the two arms alternated within every round.  The rate is the pass's 2·M·N·K FLOP over the
median time, and its share is against the data sheet's 495 TFLOP/s dense TF32 (H100 SXM).  With --profile, each
cuDNN call also runs 10 times under torch.profiler and its kernel time is split into layout transposes and the rest.
Prints one JSON line per layer and pass with the card's name, power limit and SM clock.  Needs a GPU (no CPU path).
"""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

from caffeonspark_b200 import layers

PEAK_TF32 = 495e12
# name, (N, C, H, W), K, kernel, stride, pad, groups, data gradient timed
CASES = [("conv1", (256, 3, 227, 227), 96, 11, 4, 0, 1, False),
         ("conv2", (256, 96, 27, 27), 256, 5, 1, 2, 2, True),
         ("conv3", (256, 256, 13, 13), 384, 3, 1, 1, 1, True),
         ("conv4", (256, 384, 13, 13), 384, 3, 1, 1, 2, True),
         ("conv5", (256, 384, 13, 13), 256, 3, 1, 1, 2, True),
         ("lenet conv1", (64, 1, 28, 28), 20, 5, 1, 0, 1, False),
         ("lenet conv2", (64, 20, 12, 12), 50, 5, 1, 0, 1, True),
         ("cifar10_quick conv1", (100, 3, 32, 32), 32, 5, 1, 2, 1, False),
         ("cifar10_quick conv2", (100, 32, 16, 16), 32, 5, 1, 2, 1, True)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    fields = (q.stdout.strip().splitlines() or [", , "])[0].split(", ")
    return (fields + ["", "", ""])[:3]


def calls(x, w, dy, stride, pad, groups):
    """{pass: (native call, cuDNN call)}"""
    geom = layers._conv_geometry(x, w, (stride, stride), (pad, pad), groups)
    L = layers._lib.lib()
    s = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    y, dx, dw = torch.empty_like(dy), torch.empty_like(x), torch.empty_like(w)
    work = torch.empty(max(1, L.cos_conv_workspace_floats(*geom)), device="cuda")
    st, pd, dl = [stride] * 2, [pad] * 2, [1, 1]

    def cudnn_bwd(mask):
        return lambda: torch.ops.aten.convolution_backward(dy, x, w, None, st, pd, dl, False, [0, 0], groups, mask)

    return {"forward": (lambda: L.cos_conv_forward(x.data_ptr(), w.data_ptr(), None, y.data_ptr(), *geom, s()),
                        lambda: F.conv2d(x, w, None, stride, pad, 1, groups)),
            "data": (lambda: L.cos_conv_backward_data(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), *geom, s()),
                     cudnn_bwd([True, False, False])),
            "filter": (lambda: L.cos_conv_backward_filter(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), work.data_ptr(),
                                                          *geom, s()),
                       cudnn_bwd([False, True, False]))}


def time_arms(fns, iters, warmup, rounds):
    for fn in fns:
        for _ in range(warmup):
            fn()
    samples = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            samples[i].append(a.elapsed_time(b) * 1e3 / iters)
    return [sorted(s)[len(s) // 2] for s in samples], [(min(s), max(s)) for s in samples]


def profile_split(fn):
    """µs of cuDNN's transposes and of its other kernels per call (10 calls under torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
    tr = other = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.lower()
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "nchwtonhwc" in name or "nhwctonchw" in name or "transpose" in name:
            tr += us
        else:
            other += us
    return tr / 10, other / 10


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv.py needs a GPU (there is no CPU path)")
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = True
    name_, power, clock = card()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, (n, c, h, w), k, r, stride, pad, groups, has_data in CASES:
        x = torch.randn((n, c, h, w), device="cuda", generator=gen)
        wt = torch.randn((k, c // groups, r, r), device="cuda", generator=gen) * 0.05
        p = (h + 2 * pad - r) // stride + 1
        dy = torch.randn((n, k, p, p), device="cuda", generator=gen)
        gemm = {"forward": (n * p * p, k // groups, c // groups * r * r),
                "data": (n * h * w, c // groups, k // groups * r * r),
                "filter": (k // groups, c // groups * r * r, n * p * p)}
        for pas, (native, cudnn) in calls(x, wt, dy, stride, pad, groups).items():
            if pas == "data" and not has_data:
                continue
            (tn, tc), (rn, rc) = time_arms([native, cudnn], args.iters, args.warmup, args.rounds)
            M, N, K = gemm[pas]
            flop = 2.0 * M * N * K * groups
            row = {"layer": name, "pass": pas, "gemm_mnk_per_group": [M, N, K], "groups": groups,
                   "native_us": round(tn, 1), "native_range_us": [round(v, 1) for v in rn],
                   "cudnn_us": round(tc, 1), "cudnn_range_us": [round(v, 1) for v in rc],
                   "native_tflops": round(flop / tn / 1e6, 1), "cudnn_tflops": round(flop / tc / 1e6, 1),
                   "native_share_of_495": round(flop / tn / 1e-6 / PEAK_TF32, 3),
                   "card": name_, "power_limit": power, "sm_clock": clock}
            if args.profile:
                tr, other = profile_split(cudnn)
                row.update({"cudnn_transpose_us": round(tr, 1), "cudnn_gemm_us": round(other, 1)})
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
