"""Time of the built-in engine's RNN op and of the rnn_lm fixture's training step (DESIGN.md section 14).

The op alone runs in Input (x, cont, target) -> RNN -> EuclideanLoss at three sizes: the two recurrent fixtures' RNN
layers (rnn_lm: T 20, N 32, I 128, H 256; rnn_caption's rnn1: T 12, N 16, I 64, H 128 with a 256-wide x_static) and
LRCN's (T 20, N 16, I = H = 1000).  CUDA events around --iters back-to-back forward + backward calls give the whole
call; one torch.profiler run splits it into the per-step recurrent launches (2T - 1 of them) and the rest.  The CTAs per
recurrent step are ceil(H / 64) * ceil(N / 64), the GEMM tile's grid.

The rnn_lm step is one train() call (forward, backward and the fused SGD update), timed over --steps steps after
--warmup, against an eager PyTorch fp32 mirror (nets.rnn_lm_module) doing the same forward, backward and SGD momentum
update on the same batch.  Prints one JSON line per measurement with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

STEP_KERNELS = ("RnnStep", "RnnBackStep")


def card():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def bench_op(C, np, torch, profile, ProfilerActivity, gpu, name, T, N, I, H, S, iters, warmup):
    tmp = tempfile.mkdtemp(prefix="bench_rnn_")
    shapes = [(T, N, I), (T, N), (T, N, H)] + ([(N, S)] if S else [])
    tops = ["x", "cont", "t"] + (["xs"] if S else [])
    with open(os.path.join(tmp, "net.prototxt"), "w") as f:
        f.write('name: "rnn" layer { name: "in" type: "Input" ' + " ".join(f'top: "{t}"' for t in tops) +
                " input_param { " + " ".join("shape { " + " ".join(f"dim: {d}" for d in s) + " }" for s in shapes) +
                " } }\n"
                'layer { name: "r" type: "RNN" bottom: "x" bottom: "cont" ' + ('bottom: "xs" ' if S else "") +
                f'top: "y" recurrent_param {{ num_output: {H} weight_filler {{ type: "uniform" min: -0.08 max: 0.08 }} '
                '} }\nlayer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" top: "l" }\n')
    with open(os.path.join(tmp, "solver.prototxt"), "w") as f:
        f.write('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    net = C.CaffeNet(os.path.join(tmp, "solver.prototxt"), "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    net.use_native_producer(fill_weights=True)
    rng = np.random.RandomState(0)
    cont = np.ones((T, N), np.float32)
    cont[0] = 0
    ins = [torch.from_numpy(v).cuda() for v in (rng.randn(T, N, I).astype(np.float32), cont,
                                               rng.randn(T, N, H).astype(np.float32) * 0.5)]
    if S:
        ins.append(torch.from_numpy(rng.randn(N, S).astype(np.float32)).cuda())
    loss = torch.zeros(1, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    torch.cuda.set_stream(stream)

    def call():
        assert net.forward_backward(ins, loss.data_ptr(), stream=stream.cuda_stream), net.last_error()

    for _ in range(warmup):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    b.synchronize()
    call_ms = a.elapsed_time(b) / iters
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    steps, other = [], []
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        (steps if any(k in e.name for k in STEP_KERNELS) else other).append(e.device_time / 1e3)
    torch.cuda.set_stream(torch.cuda.default_stream())
    net.deallocate()
    launches = 2 * T - 1
    res = {"bench": "rnn_op", "case": name, "T": T, "N": N, "I": I, "H": H, "S": S, "gpu": gpu, "iters": iters,
           "call_ms": round(call_ms, 4),
           "recurrent_launches_per_call": launches,
           "ctas_per_recurrent_step": -(-H // 64) * -(-N // 64),
           "recurrent_step_us_median": round(statistics.median(steps) * 1e3, 2) if steps else "not measured",
           "recurrent_steps_ms_per_call": round(sum(steps) / iters, 4) if steps else "not measured",
           "other_kernels_ms_per_call": round(sum(other) / iters, 4) if other else "not measured"}
    print(json.dumps(res), flush=True)


def bench_lm_step(C, np, torch, gpu, steps, warmup):
    from caffeonspark_b200 import nets
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    solver = os.path.join(ROOT, "tests", "golden", "configs", "rnn_lm_solver.prototxt")
    s = nets.RNN_LM
    T, N, V = s["steps"], s["batch"], s["vocab"]
    rng = np.random.RandomState(0)
    batches = []
    for _ in range(8):
        cont = (rng.rand(T, N) > 0.1).astype(np.float32)
        tok = rng.randint(0, V, (T + 1, N))
        batches.append([cont, tok[:-1].astype(np.float32), tok[1:].astype(np.float32)])
    net = C.CaffeNet(solver, "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
    assert net.connect(net.localAddresses())
    net.use_native_producer(fill_weights=True)
    torch.cuda.synchronize()
    for i in range(warmup):
        assert net.train(0, batches[i % 8]), net.last_error()
    assert net.synchronize(), net.last_error()
    t0 = time.perf_counter()
    for i in range(steps):
        assert net.train(0, batches[i % 8]), net.last_error()
    assert net.synchronize(), net.last_error()
    native_ms = (time.perf_counter() - t0) * 1e3 / steps
    net.deallocate()

    torch.backends.cuda.matmul.allow_tf32 = False
    m = nets.rnn_lm_module().cuda()
    for p in m.parameters():
        torch.nn.init.uniform_(p, -0.08, 0.08)
    opt = torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9, weight_decay=0.0005)
    dev = [[torch.from_numpy(v).cuda() for v in b] for b in batches]
    h = torch.zeros(N, s["hidden"], device="cuda")

    def step(b, h):
        cont, tok, tgt = b
        opt.zero_grad()
        scores, h = m(tok, cont, h)
        torch.nn.functional.cross_entropy(scores.reshape(-1, V), tgt.reshape(-1).long()).backward()
        opt.step()
        return h.detach()

    for i in range(warmup):
        h = step(dev[i % 8], h)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        h = step(dev[i % 8], h)
    torch.cuda.synchronize()
    torch_ms = (time.perf_counter() - t0) * 1e3 / steps
    print(json.dumps({"bench": "rnn_lm_step", "gpu": gpu, "steps": steps, "native_train_ms": round(native_ms, 4),
                      "pytorch_fp32_eager_ms": round(torch_ms, 4)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import caffeonspark_b200 as C

    if not torch.cuda.is_available():
        raise SystemExit("bench_rnn.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    for case in (("rnn_lm", 20, 32, 128, 256, 0), ("rnn_caption.rnn1", 12, 16, 64, 128, 256),
                 ("lrcn", 20, 16, 1000, 1000, 0)):
        bench_op(C, np, torch, profile, ProfilerActivity, gpu, *case, args.iters, args.warmup)
    bench_lm_step(C, np, torch, gpu, args.steps, args.warmup)


if __name__ == "__main__":
    main()
