#!/usr/bin/env python
"""bench_spp.py -- Caffe's SPP layer on the built-in engine's fused kernels against its hand-written expansion, and the
SPP CIFAR-10-quick fixture's training step (DESIGN.md section 14), one GPU.

  python bench_spp.py [--iters 50] [--steps 50] [--warmup 10]

Workloads: the fixture's SPP (b100, 64 x 6 x 6, 3 levels, MAX), an SPP-net head over conv5 (b64, 256 x 13 x 13, 3
levels, MAX) and Caffe's own test geometry (4 x 3 x 1024 x 765, 5 levels) with MAX and with AVE, whose level 0 sums
the whole 783,360-value plane in one thread, as Caffe's AVE pooling does.

For each: the fused kernels alone (layers.spp_forward / spp_backward), and one forward + backward on the engine of
Input -> Scale (so that the bottom wants a gradient) -> SPP -> EuclideanLoss against the same net with SPP written out
as an explicit Split, one Pooling and one Flatten per level and a Concat, counting the device time of the SPP part's
kernels only (spp_*, *pool*, Concat's slice_copy and Split's add / accumulate).  Kernel times are medians over calls in
a torch.profiler run.  The least traffic is computed from the shapes: the forward reads x and writes y (and MAX's int32
argmax), the backward reads dy (and the argmax) and writes dx; bound_us is it at the H100 SXM data sheet's 3.35 TB/s.

The fixture (tests/golden/configs/cifar10_quick_spp_solver.prototxt, b100): one train() step (forward, backward and
the fused SGD update; host clock around a synchronised window) against the eager PyTorch fp32 mirror
(nets.cifar10_quick_spp_module, TF32 off) doing the same forward, backward and SGD momentum update.  Prints one JSON
line per measurement with the card's name and power limit read in the same run; writes nothing in the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PEAK_BPS = 3.35e12
# (name, bottom, pyramid height, pool)
WORKLOADS = [("fixture", (100, 64, 6, 6), 3, "MAX"), ("sppnet_head", (64, 256, 13, 13), 3, "MAX"),
             ("caffe_test_max", (4, 3, 1024, 765), 5, "MAX"), ("caffe_test_ave", (4, 3, 1024, 765), 5, "AVE")]
EXPANSION_KERNELS = ("pool", "slice_copy", "add_kernel", "accumulate_kernel")


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


def device_us(torch, profile, ProfilerActivity, fn, iters, warmup, keep=lambda name: "Memcpy" not in name):
    """median over calls of the device time of the kernels one call launches that `keep` selects"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
            torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type.name == "CUDA"]
    per = len(ks) // iters
    calls = [ks[i * per:(i + 1) * per] for i in range(iters)]
    kept = [[e for e in c if keep(e.name)] for c in calls]
    return statistics.median(sum(e.device_time for e in c) for c in kept), len(kept[0])


def net_text(bottom, h, pool, expanded):
    """Input -> Scale -> SPP (or its expansion) -> EuclideanLoss"""
    from caffeonspark_b200 import nets
    n, c, hh, ww = bottom
    top = (n, c * (4 ** h - 1) // 3) if h > 1 else (n, c, 1, 1)
    dims = lambda s: " ".join(f"dim: {d}" for d in s)  # noqa: E731
    text = (f'name: "b" layer {{ name: "in" type: "Input" top: "x" top: "t" input_param {{ shape {{ {dims(bottom)} }} '
            f'shape {{ {dims(top)} }} }} }}\n'
            'layer { name: "sc" type: "Scale" bottom: "x" top: "a" scale_param { axis: 0 } }\n')
    if not expanded:
        text += (f'layer {{ name: "spp" type: "SPP" bottom: "a" top: "y" spp_param {{ pyramid_height: {h} '
                 f'pool: {pool} }} }}\n')
    else:
        tops = " ".join(f'top: "s{lv}"' for lv in range(h))
        text += f'layer {{ name: "split" type: "Split" bottom: "a" {tops} }}\n'
        for lv in range(h):
            _, kh, kw, ph, pw = nets.spp_level(hh, ww, lv)
            text += (f'layer {{ name: "pool{lv}" type: "Pooling" bottom: "s{lv}" top: "p{lv}" pooling_param {{ '
                     f'pool: {pool} kernel_h: {kh} kernel_w: {kw} stride_h: {kh} stride_w: {kw} pad_h: {ph} '
                     f'pad_w: {pw} }} }}\n')
            text += f'layer {{ name: "flat{lv}" type: "Flatten" bottom: "p{lv}" top: "f{lv}" }}\n'
        bottoms = " ".join(f'bottom: "f{lv}"' for lv in range(h))
        text += f'layer {{ name: "cat" type: "Concat" {bottoms} top: "y" }}\n'
    return text + 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n', top


def engine_us(C, torch, profile, ProfilerActivity, bottom, h, pool, expanded, iters, warmup, tmp):
    text, top = net_text(bottom, h, pool, expanded)
    d = os.path.join(tmp, f"{'x' if expanded else 'f'}_{'_'.join(map(str, bottom))}_{h}_{pool}")
    os.makedirs(d)
    with open(os.path.join(d, "net.prototxt"), "w") as f:
        f.write(text)
    with open(os.path.join(d, "solver.prototxt"), "w") as f:
        f.write('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = C.CaffeNet(os.path.join(d, "solver.prototxt"), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    try:
        assert net.connect(net.localAddresses())
        net.use_native_producer(fill_weights=False)
        net.data().fill_(1.0)
        g = torch.Generator(device="cuda").manual_seed(0)
        inputs = [torch.randn(bottom, device="cuda", generator=g), torch.randn(top, device="cuda", generator=g)]
        loss = torch.zeros(1, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def call():
            assert net.forward_backward(inputs, loss.data_ptr(), stream=stream), net.last_error()

        keep = (lambda n: "spp_" in n) if not expanded else (lambda n: any(k in n for k in EXPANSION_KERNELS))
        return device_us(torch, profile, ProfilerActivity, call, iters, warmup, keep)
    finally:
        net.deallocate()


def bench_op(C, torch, profile, ProfilerActivity, gpu, iters, warmup):
    from caffeonspark_b200 import layers
    tmp = tempfile.mkdtemp(prefix="bench_spp_")
    for name, bottom, h, pool in WORKLOADS:
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(bottom, device="cuda", generator=g)
        y, arg = layers.spp_forward(x, h, pool)
        dy = torch.randn(y.shape, device="cuda", generator=g)
        dx = torch.empty_like(x)
        nb, nt = count(bottom), y.numel()
        arg_bytes = 4 * nt if pool == "MAX" else 0
        res = {"bench": "spp", "case": name, "bottom": list(bottom), "pyramid_height": h, "pool": pool, "gpu": gpu,
               "iters": iters}
        for label, fn, nbytes in (("fused_forward", lambda: layers.spp_forward(x, h, pool, out=y, argmax=arg),
                                   4 * nb + 4 * nt + arg_bytes),
                                  ("fused_backward", lambda: layers.spp_backward(dy, arg, bottom, h, pool, out=dx),
                                   4 * nt + arg_bytes + 4 * nb)):
            us, launches = device_us(torch, profile, ProfilerActivity, fn, iters, warmup)
            res[label] = {"kernel_us_median": round(us, 2), "launches": launches,
                          "bound_us": round(nbytes / PEAK_BPS * 1e6, 2),
                          "share_of_bound": round(nbytes / PEAK_BPS * 1e6 / us, 3) if us > 0 else "not measured"}
        for label, expanded in (("engine_fused_fb", False), ("engine_expansion_fb", True)):
            us, launches = engine_us(C, torch, profile, ProfilerActivity, bottom, h, pool, expanded, iters, warmup,
                                     tmp)
            res[label] = {"kernel_us_median": round(us, 2), "launches": launches}
        fused, expansion = res["engine_fused_fb"]["kernel_us_median"], res["engine_expansion_fb"]["kernel_us_median"]
        res["expansion_over_fused"] = round(expansion / fused, 3) if fused > 0 else "not measured"
        print(json.dumps(res), flush=True)
        del x, y, arg, dy, dx
        torch.cuda.empty_cache()


def bench_fixture(C, np, torch, gpu, steps, warmup):
    from caffeonspark_b200 import nets
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    tmp = tempfile.mkdtemp(prefix="bench_spp_fixture_")
    cfg = os.path.join(ROOT, "tests", "golden", "configs")
    text = open(os.path.join(cfg, "cifar10_quick_spp_train_test.prototxt")).read()
    with open(os.path.join(tmp, "net.prototxt"), "w") as f:
        f.write(text.replace('mean_file: "mean.binaryproto"', ""))
    solver = open(os.path.join(cfg, "cifar10_quick_spp_solver.prototxt")).read()
    with open(os.path.join(tmp, "solver.prototxt"), "w") as f:
        f.write(solver.replace('net: "cifar10_quick_spp_train_test.prototxt"', 'net: "net.prototxt"'))
    n = nets.CIFAR10_QUICK_SPP["batch"]
    rng = np.random.RandomState(0)
    host = [[rng.rand(n, 3, 32, 32).astype(np.float32), rng.randint(0, 10, n).astype(np.float32)] for _ in range(8)]
    net = C.CaffeNet(os.path.join(tmp, "solver.prototxt"), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
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
    m = nets.cifar10_quick_spp_module().cuda()
    opt = torch.optim.SGD(m.parameters(), lr=0.001, momentum=0.9, weight_decay=0.004)
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
    print(json.dumps({"bench": "cifar10_quick_spp", "gpu": gpu, "batch": n, "steps": steps,
                      "native_train_ms": round(train_ms, 4), "pytorch_fp32_eager_step_ms": round(torch_ms, 4)}),
          flush=True)


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
        raise SystemExit("bench_spp.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    bench_op(C, torch, profile, ProfilerActivity, gpu, args.iters, args.warmup)
    bench_fixture(C, np, torch, gpu, args.steps, args.warmup)


if __name__ == "__main__":
    main()
