"""Ragged images resized and transformed on the device (DESIGN.md, "Images of any size"): three reports.

  1. cos_image_transform kernel time (CUDA events over many launches, captured in a CUDA graph) on a seeded list of
     256 ImageNet-like sizes (500x375, 375x500, 500x333, 640x480, ...), mirror and three mean values, for two targets:
     resize to 227x227 (crop 227), and resize to 256x256 then crop 227.  Bytes come from shapes: the source taps the
     crop window needs (distinct rows x distinct columns x channels per image), plus the fp32 output.  Reported as a
     share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), with the card read in the same run.
  2. CaffeNet b256 step time with the PyTorch producer, in alternated rounds: train_raw(list of images,
     resize=(256, 256)), train_raw of an already-resized uint8 256x256 block, and train(fp32 227x227), all from
     pinned host memory.
  3. For context only: one host core's cv2.resize of the same 256 images to 256x256 (a CPU number), when cv2 is
     installed.

  python bench_image_transform.py [--rounds R] [--steps K] [--iters I]

Prints one human-readable block and one JSON line.  Writes nothing into the tree.  Needs a GPU; there is no CPU
fallback.
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench_input_transform as B  # noqa: E402

MEAN_VALUES = B.MEAN_VALUES
SIZES = [(500, 375), (375, 500), (500, 333), (333, 500), (640, 480), (480, 640), (500, 500), (400, 500), (500, 400),
         (375, 500), (500, 375), (427, 640), (640, 427), (300, 400)]
TARGETS = [("resize_227_crop_227", (227, 227)), ("resize_256_crop_227", (256, 256))]
CROP = 227


def imagenet_sizes(n=256, seed=0):
    rng = np.random.RandomState(seed)
    return [SIZES[i] for i in rng.randint(0, len(SIZES), n)]


def tap_bytes(sizes, target, crop, mirror, key, C=3):
    """Source bytes the crop window reads: per image, the distinct source rows times the distinct source columns of
    its 2x2 taps (resize_ref's rule and transform_ref's draws), times channels."""
    import resize_ref as R
    import transform_ref as T
    total = 0
    for n, (H, W) in enumerate(sizes):
        _, h_off, w_off = T.draws(key, n, target[0], target[1], crop, mirror)
        iy, _ = R.taps(H, target[0])
        ix, _ = R.taps(W, target[1])
        iy, ix = iy[h_off:h_off + crop], ix[w_off:w_off + crop]
        rows = np.union1d(np.clip(iy, 0, H - 1), np.clip(iy + 1, 0, H - 1))
        cx = np.clip(ix, 0, W - 1)
        cols = np.union1d(cx, np.minimum(cx + 1, W - 1))
        total += rows.size * cols.size * C
    return total


def kernel_report(torch, L, iters):
    from caffeonspark_b200 import _lib
    sizes = imagenet_sizes()
    N, C = len(sizes), 3
    rng = np.random.RandomState(1)
    geom = (_lib.cos_image_geometry * N)()
    off = 0
    for n, (h, w) in enumerate(sizes):
        geom[n].offset, geom[n].height, geom[n].width = off, h, w
        off += h * w * C
    arena = torch.from_numpy(rng.randint(0, 256, off).astype(np.uint8)).cuda()
    gd = torch.frombuffer(bytearray(bytes(geom)), dtype=torch.uint8).cuda()
    gptr = ctypes.cast(gd.data_ptr(), ctypes.POINTER(_lib.cos_image_geometry))
    out = torch.empty((N, C, CROP, CROP), device="cuda")
    mv = (ctypes.c_float * 3)(*MEAN_VALUES)
    key = 1  # one key for every launch, so that the bytes below are the bytes each launch moves
    res = []
    for name, (th, tw) in TARGETS:
        def launch():
            rc = L.cos_image_transform(arena.data_ptr(), gptr, N, C, th, tw, out.data_ptr(), CROP, CROP, CROP, 1,
                                       None, 0, 0, mv, 3, 1.0, key, torch.cuda.current_stream().cuda_stream)
            assert rc == 1, L.cos_last_error()

        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(iters):
                launch()
        graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(5):
            e0.record()
            graph.replay()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / iters)
        us = statistics.median(times)
        src = tap_bytes(sizes, (th, tw), CROP, True, key)
        b = src + N * C * CROP * CROP * 4
        res.append(dict(case=name, us=round(us, 2), source_bytes=src, output_bytes=N * C * CROP * CROP * 4, bytes=b,
                        tb_per_s=round(b / us / 1e6, 3), share_of_3_35=round(b / us / 1e6 / 3.35, 3),
                        floor_us=round(b / B.HBM_BYTES_PER_S * 1e6, 1), spread_us=[round(t, 2) for t in times]))
    return res


def step_report(torch, C, harness, rounds, steps):
    import transform_ref as T
    batch = 256
    sizes = imagenet_sizes(batch, seed=2)
    with tempfile.TemporaryDirectory() as d:
        net = C.CaffeNet(B.caffenet_solver(d, batch), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
        try:
            assert net.connect(net.localAddresses())
            harness.make_producer("caffenet", net)
            g = torch.Generator().manual_seed(3)
            total = sum(h * w * 3 for h, w in sizes)
            arena = torch.randint(0, 256, (total,), dtype=torch.uint8, generator=g).pin_memory().numpy()
            images, off = [], 0
            for h, w in sizes:  # each image its own (pinned) array, as a decoder hands them over
                images.append(arena[off:off + h * w * 3].reshape(h, w, 3))
                off += h * w * 3
            block = torch.randint(0, 256, (batch, 256, 256, 3), dtype=torch.uint8, generator=g).pin_memory()
            label = torch.randint(0, 1000, (batch,), generator=g).float().pin_memory()
            x32 = torch.from_numpy(T.transform(block.numpy()[:8], "u8", 227, True, None, MEAN_VALUES, 1.0, 5))
            fp32 = torch.empty((batch, 3, 227, 227)).pin_memory()
            fp32.copy_(x32.repeat(batch // 8, 1, 1, 1))
            block_np, label_np = block.numpy(), label.numpy()
            # every kind on its own net would double the producer's memory; the net keeps one target, so the images
            # path is compared on this net and the block and fp32 paths on a second one
            net2 = C.CaffeNet(B.caffenet_solver(d, batch), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
            try:
                assert net2.connect(net2.localAddresses())
                harness.make_producer("caffenet", net2)

                def run(kind):
                    t0 = time.perf_counter()
                    for _ in range(steps):
                        if kind == "images":
                            ok, n = net.train_raw(0, [images, label_np], resize=(256, 256)), net
                        elif kind == "block":
                            ok, n = net2.train_raw(0, [block_np, label_np]), net2
                        else:
                            ok, n = net2.train(0, [fp32, label]), net2
                        assert ok, n.last_error()
                    assert net.synchronize() and net2.synchronize()
                    return (time.perf_counter() - t0) * 1e3 / steps

                kinds = ("images", "block", "fp32")
                for k in kinds:
                    run(k)  # warm-up: graphs, algorithms, staging buffers
                res = {k: [] for k in kinds}
                for r in range(rounds):
                    order = kinds if r % 2 == 0 else kinds[::-1]
                    for k in order:
                        res[k].append(run(k))
            finally:
                net2.deallocate()
        finally:
            net.deallocate()
    med = {k: round(statistics.median(v), 3) for k, v in res.items()}
    return dict(train_raw_images_ms=med["images"], train_raw_u8_block_ms=med["block"], train_fp32_ms=med["fp32"],
                rounds={k: [round(x, 3) for x in v] for k, v in res.items()},
                h2d_bytes_images=total + batch * 4, h2d_bytes_block=batch * 256 * 256 * 3 + batch * 4,
                h2d_bytes_fp32=batch * 3 * 227 * 227 * 4 + batch * 4), sizes


def cpu_report(sizes):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    rng = np.random.RandomState(4)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        for img in images:
            cv2.resize(img, (256, 256), interpolation=cv2.INTER_LINEAR)
        times.append((time.perf_counter() - t0) * 1e3)
    return dict(opencv=cv2.__version__, cv2_resize_ms_per_batch_one_core=round(statistics.median(times), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=100)
    args = ap.parse_args()
    import torch
    import caffeonspark_b200 as C
    from caffeonspark_b200 import _lib, harness
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_transform.py needs a CUDA device (no CPU fallback)")
    L = _lib.lib()
    gpu = B.card()
    kern = kernel_report(torch, L, args.iters)
    step, sizes = step_report(torch, C, harness, args.rounds, args.steps)
    cpu = cpu_report(sizes)
    print(f"card: {gpu}  (name, power limit, max SM clock)")
    print("1. cos_image_transform, 256 ImageNet-like images, crop 227, mirror, 3 mean values "
          "(CUDA events, median of 5 graph replays of %d launches)" % args.iters)
    for k in kern:
        print(f"   {k['case']:22s} {k['us']:9.2f} us  {k['bytes'] / 1e6:7.1f} MB ({k['source_bytes'] / 1e6:.1f} MB taps "
              f"+ {k['output_bytes'] / 1e6:.1f} MB fp32)  {k['tb_per_s']:.3f} TB/s = {100 * k['share_of_3_35']:.1f} % "
              f"of 3.35 TB/s (floor {k['floor_us']} us)")
    print("2. CaffeNet b256 step, PyTorch producer, pinned host memory, medians of %d alternated rounds x %d steps"
          % (args.rounds, args.steps))
    print(f"   train_raw(256 images, resize 256x256): {step['train_raw_images_ms']:.3f} ms/step  "
          f"({step['h2d_bytes_images'] / 1e6:.1f} MB H2D)")
    print(f"   train_raw(u8 256x256x3 block):         {step['train_raw_u8_block_ms']:.3f} ms/step  "
          f"({step['h2d_bytes_block'] / 1e6:.1f} MB H2D)")
    print(f"   train(fp32 227x227):                   {step['train_fp32_ms']:.3f} ms/step  "
          f"({step['h2d_bytes_fp32'] / 1e6:.1f} MB H2D)")
    if cpu:
        print(f"3. CPU, for context only: cv2.resize of the same 256 images to 256x256 on one host core: "
              f"{cpu['cv2_resize_ms_per_batch_one_core']} ms per batch (OpenCV {cpu['opencv']})")
    else:
        print("3. CPU: cv2 is not installed; no host resize time")
    print(json.dumps(dict(card=gpu, kernel=kern, step=step, cpu=cpu)))


if __name__ == "__main__":
    main()
