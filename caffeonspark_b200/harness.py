"""Executor-side harness: what CaffeProcessor.doTrain + Caffe's Net do around
the sync library in the reference (caffe-grid .../CaffeProcessor.scala:413-471,
caffe-public solver.cpp:221-223), reduced to what the benchmark needs.

* ``TorchProducer`` is the gradient producer (Net::ForwardBackward): a PyTorch
  module whose parameters and gradients ALIAS the library's flat Params buffers
  (data_/diff_, parallel.cpp:27-57 does the same re-pointing for Caffe blobs),
  registered as the C callback cos_net_train() invokes.
* ``Cluster`` plays the Spark driver's 3-phase address exchange
  (CaffeOnSpark.scala:105-154) over torch.distributed: gather every rank's
  localAddresses(), hand rank r the column addressed to it, connect().

PyTorch here is plumbing (device tensors, streams, process group); the sync
path itself is entirely inside libcaffedistri_b200.so.
"""
import os

import torch

from .caffenet import CaffeNet, CosError, _DevArray
from . import nets


PRECISIONS = ("fp32", "bf16")


class TorchProducer:
    """precision="bf16" runs forward/backward under torch.autocast(bfloat16): convolutions, FC layers and the
    native layers take bf16 activations, while parameters, their gradients (diff_) and the solver state stay
    fp32.  An opt-in trade of bitwise parity for speed; "fp32" (the default) is the full-precision producer."""

    def __init__(self, net: CaffeNet, module: torch.nn.Module, seed=1234, use_graph=True, precision="fp32"):
        if precision not in PRECISIONS:
            raise CosError(f"unknown producer precision {precision!r} (expected one of {', '.join(PRECISIONS)})")
        self.precision = precision
        self.net = net
        self.device = torch.device(f"cuda:{net.deviceID(0)}")
        self.module = module.to(self.device)
        flat_w, flat_g = net.data(), net.diff()
        torch.manual_seed(seed)  # identical initial weights on every rank
        for m in self.module.modules():
            if hasattr(m, "reset_parameters"):
                m.reset_parameters()
        off = 0
        with torch.no_grad():
            for p in self.module.parameters():  # learnable_params() order: layer by layer, weight then bias
                n = p.numel()
                w = flat_w[off:off + n].view(p.shape)
                w.copy_(p.data)
                p.data = w
                p.grad = flat_g[off:off + n].view(p.shape)
                off += n
        if off != net.param_count():
            raise CosError(f"module has {off} parameters, the net layout has {net.param_count()}")
        self.loss_fn = torch.nn.CrossEntropyLoss()  # SoftmaxWithLoss, normalised by batch
        self._streams = {}
        self._graphs = {}
        self.use_graph = use_graph
        self._capture_stream = torch.cuda.Stream(device=self.device)
        net.set_forward_backward(self._callback)

    def forward_backward(self, x, label):
        """Accumulates d(loss)/d(w) into diff_ (the kernel zeroes it after use)."""
        if self.precision == "bf16":
            # cache_enabled=False: autocast's weight-cast cache must not outlive a CUDA-graph capture; the casts
            # are recomputed every call, so a replay always reads the current fp32 weights
            with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
                loss = self.loss_fn(self.module(x), label)
        else:
            logits = self.module(x)
            loss = self.loss_fn(logits, label)
        loss.backward()
        return loss.detach()

    # called from C (cos_net_train) with device pointers of the staged blobs
    def _callback(self, solver_index, blobs, loss_dev, stream):
        ext = self._streams.get(stream)
        if ext is None:
            ext = torch.cuda.ExternalStream(stream, device=self.device) if stream else torch.cuda.current_stream()
            self._streams[stream] = ext
        (xp, xs), (lp, ls) = blobs[0], blobs[1]
        key = (xp, lp, xs, loss_dev)
        st = self._graphs.get(key)
        if st is None:
            nx = xs[0] * xs[1] * xs[2] * xs[3]
            st = self._graphs[key] = {
                "x": torch.as_tensor(_DevArray(xp, nx), device=self.device).view(xs),
                "lab": torch.as_tensor(_DevArray(lp, ls[0]), device=self.device),
                "loss": torch.as_tensor(_DevArray(loss_dev, 1), device=self.device),
                "calls": 0, "graph": None}
        with torch.cuda.stream(ext):
            if st["graph"] is not None:
                st["graph"].replay()
                return 0
            st["calls"] += 1
            if self.use_graph and st["calls"] == 4:
                # the staged-input addresses are stable across train() calls: capture forward/backward once
                # (after cuDNN autotuning ran eagerly) and replay it from then on
                try:
                    ext.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=self._capture_stream, capture_error_mode="thread_local"):
                        loss = self.forward_backward(st["x"], st["lab"].long())
                        st["loss"].copy_(loss.reshape(1))
                    # the capture itself did not execute anything: run this step through the graph
                    g.replay()
                    st["graph"] = g
                    return 0
                except Exception as e:  # the producer (not the product path) falls back to eager
                    print(f"[harness] CUDA-graph capture of forward/backward failed ({e}); staying eager")
                    self.use_graph = False
            loss = self.forward_backward(st["x"], st["lab"].long())
            st["loss"].copy_(loss.reshape(1))
        return 0


class Cluster:
    """The Spark driver's role: rank assignment + address exchange + connect."""

    def __init__(self, desc, rank=None, world=None, device=None, connection=CaffeNet.SOCKET):
        self.rank = int(os.environ.get("RANK", 0)) if rank is None else rank
        self.world = int(os.environ.get("WORLD_SIZE", 1)) if world is None else world
        local = int(os.environ.get("LOCAL_RANK", self.rank)) if device is None else device
        # one executor per GPU: start_device_id = local - 1 makes FindDevice pick `local`
        self.net = CaffeNet(desc, "", "", 1, self.world, self.rank, True,
                            connection if self.world > 1 else CaffeNet.NONE, local - 1, 0)

    def start(self):
        """CaffeOnSpark.setupTraining phases 1-3 (CaffeOnSpark.scala:113-154)."""
        net = self.net
        if self.world == 1:
            if not net.connect(net.localAddresses()):
                raise CosError(net.last_error())
            return net
        import torch.distributed as dist
        mine = net.localAddresses()                      # phase 1: collect
        table = [None] * self.world
        dist.all_gather_object(table, mine)              # phase 2: "broadcast"
        addrs = [table[p][self.rank] if p != self.rank else "" for p in range(self.world)]
        if not net.connect(addrs):                       # phase 3: processor.start
            raise CosError(net.last_error())
        if not net.sync():
            raise CosError(net.last_error())
        return net


def make_producer(name, net, seed=1234, use_graph=True, precision="fp32"):
    return TorchProducer(net, nets.torch_module(name), seed=seed, use_graph=use_graph, precision=precision)
