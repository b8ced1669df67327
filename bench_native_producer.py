"""Forward/backward time of the built-in producer against the PyTorch fp32 producer (DESIGN.md section 14).

Workloads: the eight nets the engine runs, at their reference batch sizes (LeNet b64, CIFAR-10-quick b100,
cifar10_full_bn b100, cifar10_full b100, the siamese MNIST example b64 of 2x28x28 pairs: its two LeNet trunks share
their weights and end in a ContrastiveLoss, timed against the PyTorch module that runs one trunk twice; and the
ResNet-20 fixture b100, timed against nets.resnet20_module, whose BatchNorms run the same native kernels; the two
autoencoder fixtures b100 of 1x28x28, Caffe's MNIST autoencoder and the convolutional one with Deconvolutions, each
scoring its reconstruction against its input with SigmoidCrossEntropyLoss, timed against nets.autoencoder_module and
nets.conv_autoencoder_module; the TanH LeNet fixture b64, whose head is Softmax + MultinomialLogisticLoss, and the
PReLU CIFAR-10-quick fixture b100, timed against nets.lenet_tanh_module and nets.cifar10_quick_prelu_module; the two
embedding fixtures, whose staged inputs are token ids: the sentence classifier text_cnn b50 of 32 ids and the n-gram
language model ngram_lm b128 of 4 ids, timed against nets.text_cnn_module and nets.ngram_lm_module; and the two MVN
fixtures: cifar10_quick_mvn b100 and the layer-normalised RNN language model rnn_lm_ln of 20 steps x 32 streams, timed
against nets.cifar10_quick_mvn_module and nets.rnn_lm_ln_module, whose MVNs run the same native kernels).  For each, one process times the native engine, the PyTorch module with TF32 off and with
TF32 on (cuDNN's default, here applied to matmuls too), alternating the three in every round; each sample is CUDA events around `--iters`
back-to-back forward/backward calls on one stream after `--warmup` untimed ones.  Prints one JSON line per
workload with median / min / max ms per call and images/s, and the card's name and power limit.

--profile adds a torch.profiler run of the native engine: per-kernel device time per call, and the achieved FLOP/s of
each net's largest GEMM (2*M*N*K from the plan's shapes over that launch's kernel time) against the H100 SXM data
sheet's 67 TFLOP/s FP32.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = ("lenet", "cifar10_quick", "cifar10_full_bn", "cifar10_full", "mnist_siamese", "cifar10_resnet20",
             "mnist_autoencoder", "mnist_conv_autoencoder", "lenet_tanh", "cifar10_quick_prelu", "text_cnn", "ngram_lm",
             "cifar10_quick_mvn", "rnn_lm_ln")
FIXTURES = ("cifar10_resnet20", "mnist_autoencoder", "mnist_conv_autoencoder", "lenet_tanh",
            "cifar10_quick_prelu", "text_cnn", "ngram_lm", "cifar10_quick_mvn", "rnn_lm_ln")  # nets kept under tests/golden/configs
FP32_PEAK = 67e12  # H100 SXM data sheet, dense FP32, at up to 700 W


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def siamese_solver(directory):
    """The reference's siamese example with its TRAIN Data layer swapped for MemoryData (batch 64, 2x28x28)."""
    configs = os.path.join(ROOT, "tests", "golden", "configs")
    net = open(os.path.join(configs, "mnist_siamese_train_test.prototxt")).read()
    start, end = net.index("layer {"), net.index('layer {\n  name: "slice_pair"')
    data = ('layer { name: "pair_data" type: "MemoryData" top: "pair_data" top: "sim" include { phase: TRAIN } '
            'memory_data_param { batch_size: 64 channels: 2 height: 28 width: 28 } }\n')
    with open(os.path.join(directory, "mnist_siamese_net.prototxt"), "w") as f:
        f.write(net[:start] + data + net[end:])
    solver = open(os.path.join(configs, "mnist_siamese_solver.prototxt")).read()
    path = os.path.join(directory, "mnist_siamese_solver.prototxt")
    with open(path, "w") as f:
        f.write(solver.replace("examples/siamese/mnist_siamese_train_test.prototxt", "mnist_siamese_net.prototxt"))
    return path


def fixture_solver(directory, name):
    """A fixture's solver and net, the net without a mean_file (the timed batches are staged as they are)."""
    configs = os.path.join(ROOT, "tests", "golden", "configs")
    net = open(os.path.join(configs, f"{name}_train_test.prototxt")).read()
    with open(os.path.join(directory, f"{name}_train_test.prototxt"), "w") as f:
        f.write(net.replace('mean_file: "mean.binaryproto"', ""))
    solver = open(os.path.join(configs, f"{name}_solver.prototxt")).read()
    path = os.path.join(directory, f"{name}_solver.prototxt")
    with open(path, "w") as f:
        f.write(solver)
    return path


def plan_gemms(text):
    """(label, flops) of every GEMM one forward/backward launches, in launch order (native_producer.cu)."""
    fwd, bwd = [], []
    for line in text.splitlines():
        if not line.startswith("op "):
            continue
        f = line.split()
        kind, name = f[2], f[3]
        ins = [int(v) for v in f[4].split("x")]
        w = int(re.search(r" w=\d+:(\d+)", line).group(1)) if " w=" in line else 0
        # the plan's rule: no data gradient into a staged input, nor into a blob with no learnable blob before it
        need_dx = " staged-bottom" not in line and " no-bottom-grad" not in line
        if kind == "Deconvolution":  # the transpose of the convolution from its top to its bottom
            kh, kw = (int(v) for v in re.search(r" k(\d+)x(\d+)", line).groups())
            n, cin, h, wd = ins
            cout, oh, ow = (int(v) for v in f[6].split("x")[1:])
            fwd.append((f"{name} forward", 2 * cout * n * oh * ow * cin * kh * kw))
            back = [(f"{name} weight gradient", 2 * cin * cout * kh * kw * n * h * wd)]
            if need_dx:
                back.append((f"{name} data gradient", 2 * cin * n * h * wd * cout * kh * kw))
            bwd.append(back if " no-backward" not in line else [])
        elif kind in ("Convolution", "ConvBiasReLUMaxPool"):
            kh, kw = (int(v) for v in re.search(r" k(\d+)x(\d+)", line).groups())
            sh, sw = (int(v) for v in re.search(r" s(\d+)x(\d+)", line).groups())
            ph, pw = (int(v) for v in re.search(r" p(\d+)x(\d+)", line).groups())
            n, cin, h, wd = ins
            cout = w // (cin * kh * kw)
            oh, ow = (h + 2 * ph - kh) // sh + 1, (wd + 2 * pw - kw) // sw + 1
            k, cols = cin * kh * kw, n * oh * ow
            fwd.append((f"{name} forward", 2 * cout * cols * k))
            back = [(f"{name} weight gradient", 2 * cout * k * cols)]
            if need_dx:
                back.append((f"{name} data gradient", 2 * cin * n * h * wd * cout * kh * kw))
            bwd.append(back if " no-backward" not in line else [])
        elif kind == "InnerProduct":
            b = ins[0]
            k = 1
            for d in ins[1:]:
                k *= d
            nout = w // k
            fwd.append((f"{name} forward", 2 * b * nout * k))
            back = [(f"{name} weight gradient", 2 * nout * k * b)]
            if need_dx:
                back.append((f"{name} data gradient", 2 * b * k * nout))
            bwd.append(back if " no-backward" not in line else [])
    return fwd + [g for back in reversed(bwd) for g in back]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    import caffeonspark_b200 as C
    from caffeonspark_b200 import nets

    if not torch.cuda.is_available():
        raise SystemExit("bench_native_producer.py needs a CUDA device (there is no CPU path)")
    gpu = card()
    tmp = tempfile.mkdtemp(prefix="bench_native_producer_")
    for name in args.workloads.split(","):
        siamese, resnet = name == "mnist_siamese", name == "cifar10_resnet20"
        autoencoder = name in ("mnist_autoencoder", "mnist_conv_autoencoder")
        solver = (siamese_solver(tmp) if siamese else fixture_solver(tmp, name) if name in FIXTURES
                  else nets.write_prototxts(name, tmp))
        net = C.CaffeNet(solver, "", "", 1, 1, 0, True, C.CaffeNet.NONE, -1, 0)
        net.use_native_producer(fill_weights=False)
        net.fill("data", 1, 0, 0.05)
        torch.cuda.synchronize()
        text, lm = name in ("text_cnn", "ngram_lm"), name == "rnn_lm_ln"
        spec = (nets.RESNET20 if resnet else None if siamese else nets.AUTOENCODER if name == "mnist_autoencoder"
                else nets.CONV_AUTOENCODER if autoencoder else nets.LENET_TANH if name == "lenet_tanh"
                else nets.CIFAR10_QUICK_PRELU if name == "cifar10_quick_prelu" else nets.TEXT_CNN if name == "text_cnn"
                else nets.NGRAM_LM if name == "ngram_lm" else nets.CIFAR10_QUICK_MVN if name == "cifar10_quick_mvn"
                else nets.RNN_LM if lm else nets.NETS[name])
        batch = 64 if siamese else spec["batch"]
        rng = np.random.RandomState(0)
        if lm:  # time-major sentences [steps, batch]: cont (0 where a sentence starts), tokens and next tokens
            ids = (rng.zipf(1.2, (spec["steps"] + 1, batch)) - 1) % spec["vocab"]
            cont = torch.from_numpy((rng.rand(spec["steps"], batch) > 0.15).astype(np.float32)).cuda()
            x = torch.from_numpy(ids[:-1].astype(np.float32)).cuda()
            y = torch.from_numpy(ids[1:].astype(np.float32)).cuda()
        elif text:  # token ids (Zipf-skewed, as words are) and a class or next-token label
            ids = (rng.zipf(1.2, (batch, spec["tokens"])) - 1) % spec["vocab"]
            x = torch.from_numpy(ids.astype(np.float32)).cuda()
            y = torch.from_numpy(rng.randint(0, spec.get("classes", spec["vocab"]), batch).astype(np.float32)).cuda()
        else:
            shape = (2, 28, 28) if siamese else spec["input"]
            x = torch.from_numpy(rng.rand(batch, *shape).astype(np.float32)).cuda()
            y = torch.from_numpy(rng.randint(0, 2 if siamese else 10, batch).astype(np.float32)).cuda()
        loss = torch.zeros(1, device="cuda")
        # a stream of its own: the legacy default stream's handle is 0, which would send the engine to the net's
        # stream, outside the events
        stream = torch.cuda.Stream()
        torch.cuda.synchronize()
        torch.cuda.set_stream(stream)

        # an autoencoder's one staged input is its target too
        inputs = [x] if autoencoder else [cont, x, y] if lm else [x, y]

        def native():
            assert net.forward_backward(inputs, loss.data_ptr(), stream=stream.cuda_stream), net.last_error()

        module = (nets.siamese_module() if siamese else nets.resnet20_module() if resnet
                  else nets.autoencoder_module() if name == "mnist_autoencoder"
                  else nets.conv_autoencoder_module() if autoencoder else nets.lenet_tanh_module() if name == "lenet_tanh"
                  else nets.cifar10_quick_prelu_module() if name == "cifar10_quick_prelu"
                  else nets.text_cnn_module() if name == "text_cnn" else nets.ngram_lm_module() if name == "ngram_lm"
                  else nets.cifar10_quick_mvn_module() if name == "cifar10_quick_mvn"
                  else nets.rnn_lm_ln_module() if lm
                  else nets.torch_module(name)).cuda()
        with torch.no_grad():
            w, off = net.data().clone(), 0
            for p in module.parameters():
                p.copy_(w[off:off + p.numel()].view(p.shape))
                off += p.numel()
        ylong = y.long()

        def torch_fb():
            if siamese:
                a, b = module(x)
                nets.contrastive_loss(a, b, y).backward()
                return
            if autoencoder:
                nets.sigmoid_cross_entropy_loss(module(x), x).backward()
                return
            if lm:  # each call from a zero hidden state, as the engine's first call
                h0 = torch.zeros(batch, spec["hidden"], device="cuda")
                scores, _ = module(x.long(), cont, h0)
                F.cross_entropy(scores.reshape(-1, spec["vocab"]), ylong.reshape(-1)).backward()
                return
            out = module(x)
            if name == "lenet_tanh":
                nets.multinomial_logistic_loss(out, y).backward()
                return
            F.cross_entropy(out, ylong).backward()

        default_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)

        def with_tf32(on, fn):
            def run():
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
                fn()
            return run

        impls = {"native": native, "torch_fp32": with_tf32(False, torch_fb),
                 "torch_tf32": with_tf32(True, torch_fb)}
        samples = {k: [] for k in impls}
        for fn in impls.values():  # every shape warmed before the first timed round
            for _ in range(args.warmup):
                fn()
        for _ in range(args.rounds):
            for k, fn in impls.items():
                for _ in range(args.warmup):
                    fn()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    fn()
                b.record()
                b.synchronize()
                samples[k].append(a.elapsed_time(b) / args.iters)
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = default_tf32
        res = {"workload": name, "batch": batch, "gpu": gpu, "rounds": args.rounds, "iters": args.iters}
        for k, v in samples.items():
            med = statistics.median(v)
            res[k] = {"ms_median": round(med, 4), "ms_min": round(min(v), 4), "ms_max": round(max(v), 4),
                      "images_per_s": round(batch / med * 1e3, 1)}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            calls = 10
            native()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    native()
                torch.cuda.synchronize()
            kernels = [e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
                       and "Memset" not in e.name]
            res["profile_kernel_ms_per_call_total"] = round(sum(e.device_time for e in kernels) / 1e3 / calls, 4)
            per = {}
            for e in kernels:
                short = re.sub(r"\(anonymous namespace\)::|cosb::", "", e.name)[:90]
                per[short] = per.get(short, 0.0) + e.device_time / 1e3 / calls
            res["profile_ms_per_call"] = {k: round(v, 4) for k, v in sorted(per.items(), key=lambda t: -t[1])}
            gemms = plan_gemms(C.native_producer_plan(solver))
            times = [e.device_time / 1e3 for e in kernels if "gemm_kernel" in e.name]
            if len(times) == len(gemms) * calls:
                big = max(range(len(gemms)), key=lambda i: gemms[i][1])
                t = statistics.median(times[big::len(gemms)])
                res["largest_gemm"] = {"gemm": gemms[big][0], "gflop": round(gemms[big][1] / 1e9, 3),
                                       "ms": round(t, 4), "tflops": round(gemms[big][1] / t / 1e9, 2),
                                       "share_of_67_tflops": round(gemms[big][1] / t / 1e-3 / FP32_PEAK, 3)}
            else:
                res["largest_gemm"] = f"not measured ({len(times)} GEMM launches, expected {len(gemms) * calls})"
        print(json.dumps(res), flush=True)
        torch.cuda.synchronize()
        torch.cuda.set_stream(torch.cuda.default_stream())
        net.deallocate()


if __name__ == "__main__":
    main()
