"""Time of the built-in engine's Embed op alone (DESIGN.md section 14): the forward gather and the weight gradient,
which groups the ids by row with integer passes and adds each row's dy rows in Caffe's bottom order.

The net is Input (ids, target) -> Embed (no bias) -> EuclideanLoss, at a size a text model runs: M = 8,192 ids
(e.g. 256 sentences of 32 tokens), num_output 300 and input_dim 50,000.  Ids are drawn uniformly and from a Zipf
distribution, where a few words fill much of every batch.  One torch.profiler run per distribution gives each Embed
kernel's device time per call (median over --iters calls); CUDA events around --iters back-to-back calls give the whole
call.  Achieved bytes/s come from shapes: the forward reads the ids and M table rows and writes M top rows; the weight
gradient reads the ids (three times), the top gradient once, and reads and writes each distinct id's table row, plus the
grouping's integer traffic.  Prints one JSON line per distribution with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FORWARD = ("embed_forward_kernel",)
GRADIENT = ("embed_count_kernel", "exclusive_scan_kernel", "embed_place_kernel", "embed_weight_grad_kernel")


def card():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--num-output", type=int, default=300)
    ap.add_argument("--input-dim", type=int, default=50000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import caffeonspark_b200 as C

    if not torch.cuda.is_available():
        raise SystemExit("bench_embed.py needs a CUDA device (there is no CPU path)")
    M, N, K = args.tokens, args.num_output, args.input_dim
    gpu = card()
    tmp = tempfile.mkdtemp(prefix="bench_embed_")
    with open(os.path.join(tmp, "net.prototxt"), "w") as f:
        f.write(f'name: "embed" layer {{ name: "in" type: "Input" top: "ids" top: "t" input_param {{ '
                f'shape {{ dim: {M} }} shape {{ dim: {M} dim: {N} }} }} }}\n'
                f'layer {{ name: "embed" type: "Embed" bottom: "ids" top: "y" embed_param {{ input_dim: {K} '
                f'num_output: {N} bias_term: false weight_filler {{ type: "uniform" min: -0.1 max: 0.1 }} }} }}\n'
                'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n')
    with open(os.path.join(tmp, "solver.prototxt"), "w") as f:
        f.write('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = C.CaffeNet(os.path.join(tmp, "solver.prototxt"), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    net.use_native_producer(fill_weights=True)
    rng = np.random.RandomState(0)
    t = torch.from_numpy(rng.randn(M, N).astype(np.float32)).cuda()
    loss = torch.zeros(1, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    torch.cuda.set_stream(stream)
    for dist in ("uniform", "zipf"):
        ids_np = rng.randint(0, K, M) if dist == "uniform" else (rng.zipf(1.2, M) - 1) % K
        ids = torch.from_numpy(ids_np.astype(np.float32)).cuda()
        distinct = int(np.unique(ids_np).size)

        def call():
            assert net.forward_backward([ids, t], loss.data_ptr(), stream=stream.cuda_stream), net.last_error()

        for _ in range(args.warmup):
            call()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            call()
        b.record()
        b.synchronize()
        call_ms = a.elapsed_time(b) / args.iters
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                call()
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            for k in FORWARD + GRADIENT:
                if k in e.name:
                    per.setdefault(k, []).append(e.device_time / 1e3)
        ms = {k: statistics.median(v) for k, v in per.items()}
        fwd_ms = sum(ms.get(k, 0.0) for k in FORWARD)
        grad_ms = sum(ms.get(k, 0.0) for k in GRADIENT)
        fwd_bytes = 4 * (M + 2 * M * N)
        grad_bytes = 4 * (3 * M + M * N + 2 * distinct * N) + 4 * (2 * (K + 1) + 2 * M + 2 * M)
        res = {"bench": "embed", "dist": dist, "tokens": M, "num_output": N, "input_dim": K, "distinct_ids": distinct,
               "gpu": gpu, "iters": args.iters, "call_ms": round(call_ms, 4),
               "kernel_ms": {k: round(v, 4) for k, v in ms.items()},
               "forward_ms": round(fwd_ms, 4), "weight_grad_ms": round(grad_ms, 4),
               "forward_GBps": round(fwd_bytes / fwd_ms / 1e6, 1) if fwd_ms else "not measured",
               "weight_grad_GBps": round(grad_bytes / grad_ms / 1e6, 1) if grad_ms else "not measured"}
        print(json.dumps(res), flush=True)
    torch.cuda.synchronize()
    torch.cuda.set_stream(torch.cuda.default_stream())
    net.deallocate()


if __name__ == "__main__":
    main()
