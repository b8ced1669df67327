"""Input transform on the device (DESIGN.md, "Input transform on the device"): three reports.

  1. cos_data_transform kernel time (CUDA events over many launches) and achieved bytes/s as a share of the H100 SXM
     data-sheet HBM3 bandwidth (3.35 TB/s).  Bytes come from shapes (transform_bytes below): the crop region read
     once, the fp32 output written once, and a mean file read once.
  2. CaffeNet b256 step time with the PyTorch producer: train_raw(uint8 256x256x3 images) against train(fp32 batches
     already transformed), in alternated rounds, both from pinned host memory.
  3. For context only: the host time of the numpy restatement (tests/transform_ref.py) per CaffeNet batch -- a CPU
     number, one core, not Caffe's transformer.

  python bench_input_transform.py [--rounds R] [--steps K] [--iters I]

Prints one human-readable block and one JSON line.  Writes nothing into the tree (temporary prototxts go to a
temporary directory).  Needs a GPU; there is no CPU fallback.
"""
import argparse
import ctypes
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
MEAN_VALUES = [104.0, 117.0, 123.0]


def transform_bytes(fmt, N, C, H, W, crop, mean_file):
    """Minimum traffic of one transform: the crop region of the input read once, the fp32 output written once, and
    the mean file (C x H x W fp32) read once."""
    ho, wo = (crop, crop) if crop else (H, W)
    elem = 1 if fmt == "u8" else 4
    return N * C * ho * wo * elem + N * C * ho * wo * 4 + (C * H * W * 4 if mean_file else 0)


CASES = [  # name, format, N, C, H, W, crop, mirror, mean ("values" / "file")
    ("caffenet_b256_u8", "u8", 256, 3, 256, 256, 227, True, "values"),
    ("caffenet_b256_f32", "f32", 256, 3, 256, 256, 227, True, "values"),
    ("cifar10_b100_u8_mean_file", "u8", 100, 3, 32, 32, 0, False, "file"),
    ("cifar10_b100_f32_mean_file", "f32", 100, 3, 32, 32, 0, False, "file"),
]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def kernel_report(torch, L, iters):
    out = []
    for name, fmt, N, C, H, W, crop, mirror, mean in CASES:
        g = torch.Generator(device="cuda").manual_seed(1)
        if fmt == "u8":
            x = torch.randint(0, 256, (N, H, W, C), dtype=torch.uint8, device="cuda", generator=g)
        else:
            x = torch.rand((N, C, H, W), device="cuda", generator=g) * 255
        ho, wo = (crop, crop) if crop else (H, W)
        y = torch.empty((N, C, ho, wo), device="cuda")
        m = torch.rand(C * H * W, device="cuda", generator=g) * 255 if mean == "file" else None
        mv = (ctypes.c_float * 3)(*MEAN_VALUES)
        mptr = ctypes.cast(m.data_ptr(), ctypes.POINTER(ctypes.c_float)) if m is not None else None

        def launch(k):
            s = torch.cuda.current_stream().cuda_stream
            rc = L.cos_data_transform(x.data_ptr(), 1 if fmt == "u8" else 0, N, C, H, W, y.data_ptr(), crop,
                                      int(mirror), mptr, mv if mean == "values" else None,
                                      3 if mean == "values" else 0, 1.0, k, s)
            assert rc == 1, L.cos_last_error()

        for k in range(20):
            launch(k)
        torch.cuda.synchronize()
        # the launches are captured in a CUDA graph, so that the host's ctypes call rate does not bound small cases
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for k in range(iters):
                launch(k)
        graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for rep in range(5):
            e0.record()
            graph.replay()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / iters)
        us = statistics.median(times)
        b = transform_bytes(fmt, N, C, H, W, crop, mean == "file")
        out.append(dict(case=name, us=round(us, 2), bytes=b, tb_per_s=round(b / us / 1e6, 3),
                        share_of_3_35=round(b / us / 1e6 / 3.35, 3), floor_us=round(b / HBM_BYTES_PER_S * 1e6, 1)))
    return out


def caffenet_solver(d, batch):
    text = open(os.path.join(ROOT, "tests", "golden", "configs", "bvlc_reference_net.prototxt")).read()
    text = re.sub(r"batch_size:\s*2\b", f"batch_size: {batch}", text, count=1)
    with open(os.path.join(d, "net.prototxt"), "w") as f:
        f.write(text)
    s = os.path.join(d, "solver.prototxt")
    with open(s, "w") as f:
        f.write('net: "net.prototxt"\nbase_lr: 0.0001\nlr_policy: "fixed"\nmomentum: 0.9\nmax_iter: 100000\n')
    return s


def step_report(torch, C, harness, rounds, steps):
    import transform_ref as T
    batch = 256
    with tempfile.TemporaryDirectory() as d:
        net = C.CaffeNet(caffenet_solver(d, batch), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
        try:
            assert net.connect(net.localAddresses())
            harness.make_producer("caffenet", net)
            g = torch.Generator().manual_seed(3)
            raw = torch.randint(0, 256, (batch, 256, 256, 3), dtype=torch.uint8, generator=g).pin_memory()
            label = torch.randint(0, 1000, (batch,), generator=g).float().pin_memory()
            x32 = torch.from_numpy(T.transform(raw.numpy()[:8], "u8", 227, True, None, MEAN_VALUES, 1.0, 5))
            fp32 = torch.empty((batch, 3, 227, 227)).pin_memory()
            fp32.copy_(x32.repeat(batch // 8, 1, 1, 1))
            raw_np, label_np = raw.numpy(), label.numpy()

            def run(kind):
                t0 = time.perf_counter()
                for _ in range(steps):
                    ok = net.train_raw(0, [raw_np, label_np]) if kind == "raw" else net.train(0, [fp32, label])
                    assert ok, net.last_error()
                assert net.synchronize(), net.last_error()
                return (time.perf_counter() - t0) * 1e3 / steps

            run("raw"), run("fp32")  # warm-up: graphs, algorithms, staging buffers
            res = {"raw": [], "fp32": []}
            for r in range(rounds):
                for kind in (("raw", "fp32") if r % 2 == 0 else ("fp32", "raw")):
                    res[kind].append(run(kind))
            t0 = time.perf_counter()
            T.transform(raw_np, "u8", 227, True, None, MEAN_VALUES, 1.0, 1)
            host_ms = (time.perf_counter() - t0) * 1e3
        finally:
            net.deallocate()
    return dict(train_raw_u8_ms=round(statistics.median(res["raw"]), 3),
                train_fp32_ms=round(statistics.median(res["fp32"]), 3),
                train_raw_u8_rounds=[round(v, 3) for v in res["raw"]],
                train_fp32_rounds=[round(v, 3) for v in res["fp32"]],
                h2d_bytes_raw=batch * 256 * 256 * 3 + batch * 4, h2d_bytes_fp32=batch * 3 * 227 * 227 * 4 + batch * 4,
                cpu_numpy_restatement_ms_per_batch=round(host_ms, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    import torch
    import caffeonspark_b200 as C
    from caffeonspark_b200 import _lib, harness
    if not torch.cuda.is_available():
        raise SystemExit("bench_input_transform.py needs a CUDA device (no CPU fallback)")
    L = _lib.lib()
    gpu = card()
    kern = kernel_report(torch, L, args.iters)
    step = step_report(torch, C, harness, args.rounds, args.steps)
    print(f"card: {gpu}  (name, power limit, max SM clock)")
    print("1. cos_data_transform kernel (CUDA events, median of 5 graph replays of %d launches)" % args.iters)
    for k in kern:
        print(f"   {k['case']:28s} {k['us']:9.2f} us  {k['bytes'] / 1e6:8.1f} MB  {k['tb_per_s']:.3f} TB/s "
              f"= {100 * k['share_of_3_35']:.1f} % of 3.35 TB/s (floor {k['floor_us']} us)")
    print("2. CaffeNet b256 step, PyTorch producer, pinned host memory, medians of %d alternated rounds x %d steps"
          % (args.rounds, args.steps))
    print(f"   train_raw(u8 256x256x3): {step['train_raw_u8_ms']:.3f} ms/step  "
          f"({step['h2d_bytes_raw'] / 1e6:.1f} MB H2D)")
    print(f"   train(fp32 227x227):     {step['train_fp32_ms']:.3f} ms/step  "
          f"({step['h2d_bytes_fp32'] / 1e6:.1f} MB H2D)")
    print(f"3. CPU, for context only: numpy restatement {step['cpu_numpy_restatement_ms_per_batch']} ms per CaffeNet "
          "b256 batch (one host core)")
    print(json.dumps(dict(card=gpu, kernel=kern, step=step)))


if __name__ == "__main__":
    main()
