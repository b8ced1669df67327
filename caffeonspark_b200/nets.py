"""The three BASELINE nets and the reference's CIFAR-10-full examples (plain and BatchNorm) as layer lists -> (a) Caffe prototxt text for the C
library's layout parser, (b) the learnable-blob layout, (c) a PyTorch module
used ONLY as the gradient producer (Net::ForwardBackward is out of scope of
the sync library; SURVEY.md section 8 row f1).

Architectures follow the reference's configuration files
  data/lenet_memory_train_test.prototxt, data/lenet_memory_solver.prototxt
  data/cifar10_quick_train_test.prototxt, data/cifar10_quick_solver.prototxt
  data/bvlc_reference_net.prototxt, data/bvlc_reference_solver.prototxt
  caffe-public/examples/cifar10/cifar10_full_sigmoid_train_test_bn.prototxt (+ _solver_bn)
  caffe-public/examples/cifar10/cifar10_full_train_test.prototxt, cifar10_full_solver.prototxt
(batch 256/device for CaffeNet per
 caffe-public/models/bvlc_reference_caffenet/train_val.prototxt:25).
"""
from .caffenet import SolverDesc

# layer tuples:
#   ("conv", name, cout, k, stride, pad, group, (lr_w, dm_w), (lr_b, dm_b) or None for bias_term: false)
#   ("ip",   name, nout, (lr_w, dm_w), (lr_b, dm_b))
#   ("pool", name, "MAX"|"AVE", k, stride)   ("relu", name)
#   ("lrn",  name, size, alpha, beta[, "ACROSS_CHANNELS"|"WITHIN_CHANNEL"]): norm_region, ACROSS_CHANNELS if absent
#   ("drop", name, ratio)   ("sigmoid", name)
#   ("bn",   name): Caffe BatchNorm, blobs mean [C], variance [C], scale factor [1], each lr_mult 0 decay_mult 1
_W, _B = (1.0, 1.0), (2.0, 1.0)
_B0 = (2.0, 0.0)  # CaffeNet biases: lr_mult 2, decay_mult 0
_BN = (0.0, 1.0)  # BatchNorm statistics: written by the forward pass, never by the solver

NETS = {
    "lenet": dict(
        input=(1, 28, 28), batch=64, classes=10,
        layers=[("conv", "conv1", 20, 5, 1, 0, 1, _W, _B), ("pool", "pool1", "MAX", 2, 2),
                ("conv", "conv2", 50, 5, 1, 0, 1, _W, _B), ("pool", "pool2", "MAX", 2, 2),
                ("ip", "ip1", 500, _W, _B), ("relu", "relu1"), ("ip", "ip2", 10, _W, _B)],
        solver=dict(lr_policy="inv", base_lr=0.01, gamma=0.0001, power=0.75, momentum=0.9, weight_decay=0.0005,
                    max_iter=2000, test_iter=10, test_interval=100, snapshot_prefix="mnist_lenet")),
    "cifar10_quick": dict(
        input=(3, 32, 32), batch=100, classes=10,
        layers=[("conv", "conv1", 32, 5, 1, 2, 1, _W, _B), ("pool", "pool1", "MAX", 3, 2), ("relu", "relu1"),
                ("conv", "conv2", 32, 5, 1, 2, 1, _W, _B), ("relu", "relu2"), ("pool", "pool2", "AVE", 3, 2),
                ("conv", "conv3", 64, 5, 1, 2, 1, _W, _B), ("relu", "relu3"), ("pool", "pool3", "AVE", 3, 2),
                ("ip", "ip1", 64, _W, _B), ("ip", "ip2", 10, _W, _B)],
        solver=dict(lr_policy="fixed", base_lr=0.001, momentum=0.9, weight_decay=0.004, max_iter=4000,
                    test_iter=100, test_interval=100, snapshot_prefix="cifar10_quick")),
    "caffenet": dict(
        input=(3, 227, 227), batch=256, classes=1000,
        layers=[("conv", "conv1", 96, 11, 4, 0, 1, _W, _B0), ("relu", "relu1"), ("pool", "pool1", "MAX", 3, 2),
                ("lrn", "norm1", 5, 0.0001, 0.75),
                ("conv", "conv2", 256, 5, 1, 2, 2, _W, _B0), ("relu", "relu2"), ("pool", "pool2", "MAX", 3, 2),
                ("lrn", "norm2", 5, 0.0001, 0.75),
                ("conv", "conv3", 384, 3, 1, 1, 1, _W, _B0), ("relu", "relu3"),
                ("conv", "conv4", 384, 3, 1, 1, 2, _W, _B0), ("relu", "relu4"),
                ("conv", "conv5", 256, 3, 1, 1, 2, _W, _B0), ("relu", "relu5"), ("pool", "pool5", "MAX", 3, 2),
                ("ip", "fc6", 4096, _W, _B0), ("relu", "relu6"), ("drop", "drop6", 0.5),
                ("ip", "fc7", 4096, _W, _B0), ("relu", "relu7"), ("drop", "drop7", 0.5),
                ("ip", "fc8", 1000, _W, _B0)],
        solver=dict(lr_policy="step", base_lr=0.01, gamma=0.1, stepsize=100000, momentum=0.9, weight_decay=0.0005,
                    max_iter=450000, test_iter=0, test_interval=0, snapshot_prefix="bvlc_reference_caffenet")),
    # caffe-public/examples/cifar10/cifar10_full_sigmoid_{train_test,solver}_bn.prototxt
    "cifar10_full_bn": dict(
        input=(3, 32, 32), batch=100, classes=10,
        layers=[("conv", "conv1", 32, 5, 1, 2, 1, _W, None), ("pool", "pool1", "MAX", 3, 2), ("bn", "bn1"),
                ("sigmoid", "Sigmoid1"),
                ("conv", "conv2", 32, 5, 1, 2, 1, _W, None), ("bn", "bn2"), ("sigmoid", "Sigmoid2"),
                ("pool", "pool2", "AVE", 3, 2),
                ("conv", "conv3", 64, 5, 1, 2, 1, _W, None), ("bn", "bn3"), ("sigmoid", "Sigmoid3"),
                ("pool", "pool3", "AVE", 3, 2),
                ("ip", "ip1", 10, _W, (1.0, 0.0))],
        solver=dict(lr_policy="step", base_lr=0.001, gamma=1, stepsize=5000, momentum=0.9, max_iter=60000,
                    test_iter=10, test_interval=1000, snapshot_prefix="cifar10_full_sigmoid_bn")),
    # caffe-public/examples/cifar10/cifar10_full_{train_test,solver}.prototxt: conv3 has no param specs (lr_mult 1 for
    # its bias too); ip1's weight decays 250x.  fillers: gaussian std of each weight (biases constant 0).
    "cifar10_full": dict(
        input=(3, 32, 32), batch=100, classes=10,
        layers=[("conv", "conv1", 32, 5, 1, 2, 1, _W, _B), ("pool", "pool1", "MAX", 3, 2), ("relu", "relu1"),
                ("lrn", "norm1", 3, 5e-05, 0.75, "WITHIN_CHANNEL"),
                ("conv", "conv2", 32, 5, 1, 2, 1, _W, _B), ("relu", "relu2"), ("pool", "pool2", "AVE", 3, 2),
                ("lrn", "norm2", 3, 5e-05, 0.75, "WITHIN_CHANNEL"),
                ("conv", "conv3", 64, 5, 1, 2, 1, _W, _W), ("relu", "relu3"), ("pool", "pool3", "AVE", 3, 2),
                ("ip", "ip1", 10, (1.0, 250.0), (2.0, 0.0))],
        fillers={"conv1": 0.0001, "conv2": 0.01, "conv3": 0.01, "ip1": 0.01},
        solver=dict(lr_policy="fixed", base_lr=0.001, momentum=0.9, weight_decay=0.004, max_iter=60000,
                    test_iter=100, test_interval=1000, snapshot_prefix="cifar10_full")),
}

# SURVEY.md App. D: expected flat sizes (checked by tests); cifar10_full: conv1 2432, conv2 25632, conv3 51264,
# ip1 10250
EXPECTED_PARAM_COUNT = {"lenet": 431080, "cifar10_quick": 145578, "caffenet": 60965224, "cifar10_full": 89578}
# Nets with BatchNorm statistics among their learnable blobs: the forward pass writes those, and no backward
# gives them a gradient.  3x32x32 -> conv1 2400, bn1 65, conv2 25600, bn2 65, conv3 51200, bn3 129, ip1 10240 + 10
STATS_NET_PARAM_COUNT = {"cifar10_full_bn": 89709}


def _pool_out(h, k, s):
    import math
    return int(math.ceil((h - k) / s)) + 1  # pooling_layer.cpp (pad 0)


def layout(name):
    """-> (counts, lr_mult, decay_mult, blob_names) in learnable_params() order."""
    net = NETS[name]
    c, h, w = net["input"]
    counts, lr, dm, names = [], [], [], []
    flat = None
    for L in net["layers"]:
        kind = L[0]
        if kind == "conv":
            _, nm, cout, k, s, p, g, pw, pb = L
            counts.append(cout * (c // g) * k * k)
            lr.append(pw[0])
            dm.append(pw[1])
            names.append(nm + ".w")
            if pb is not None:
                counts.append(cout)
                lr.append(pb[0])
                dm.append(pb[1])
                names.append(nm + ".b")
            h, w, c = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1, cout
        elif kind == "pool":
            _, nm, _mode, k, s = L
            h, w = _pool_out(h, k, s), _pool_out(w, k, s)
        elif kind == "ip":
            _, nm, nout, pw, pb = L
            fan_in = flat if flat is not None else c * h * w
            counts += [nout * fan_in, nout]
            lr += [pw[0], pb[0]]
            dm += [pw[1], pb[1]]
            names += [nm + ".w", nm + ".b"]
            flat = nout
        elif kind == "bn":
            nm = L[1]
            counts += [c, c, 1]
            lr += [_BN[0]] * 3
            dm += [_BN[1]] * 3
            names += [nm + ".mean", nm + ".variance", nm + ".scale"]
    return counts, lr, dm, names


def solver_desc(name, grad_dtype="fp32", **overrides):
    counts, lr, dm, _ = layout(name)
    kw = dict(NETS[name]["solver"])
    kw.update(overrides)
    return SolverDesc(counts, lr, dm, grad_dtype=grad_dtype, batch_size=NETS[name]["batch"], **kw)


def net_prototxt(name):
    """Caffe text-format net definition (TRAIN + TEST MemoryData, like the reference's files)."""
    net = NETS[name]
    c, h, w = net["input"]
    out = [f'name: "{name}"']
    for phase in ("TRAIN", "TEST"):
        out.append(f'layer {{ name: "data" type: "MemoryData" top: "data" top: "label" include {{ phase: {phase} }}\n'
                   f'  memory_data_param {{ batch_size: {net["batch"]} channels: {c} height: {h} width: {w} '
                   f'share_in_parallel: false }} }}')
    bottom = "data"
    fillers = net.get("fillers", {})

    def filler(nm):  # gaussian weights, constant-0 biases; nothing for a net without fillers
        return (f' weight_filler {{ type: "gaussian" std: {fillers[nm]:g} }} bias_filler {{ type: "constant" }}'
                if nm in fillers else "")

    for L in net["layers"]:
        kind, nm = L[0], L[1]
        if kind == "conv":
            _, _, cout, k, s, p, g, pw, pb = L
            grp = f" group: {g}" if g != 1 else ""
            pad = f" pad: {p}" if p else ""
            bias = (f' param {{ lr_mult: {pb[0]:g} decay_mult: {pb[1]:g} }}' if pb is not None else "")
            out.append(f'layer {{ name: "{nm}" type: "Convolution" bottom: "{bottom}" top: "{nm}"\n'
                       f'  param {{ lr_mult: {pw[0]:g} decay_mult: {pw[1]:g} }}{bias}\n'
                       f'  convolution_param {{ num_output: {cout} kernel_size: {k} stride: {s}{pad}{grp}'
                       f'{"" if pb is not None else " bias_term: false"}{filler(nm)} }} }}')
            bottom = nm
        elif kind == "pool":
            _, _, mode, k, s = L
            out.append(f'layer {{ name: "{nm}" type: "Pooling" bottom: "{bottom}" top: "{nm}" '
                       f'pooling_param {{ pool: {mode} kernel_size: {k} stride: {s} }} }}')
            bottom = nm
        elif kind == "ip":
            _, _, nout, pw, pb = L
            out.append(f'layer {{ name: "{nm}" type: "InnerProduct" bottom: "{bottom}" top: "{nm}"\n'
                       f'  param {{ lr_mult: {pw[0]:g} decay_mult: {pw[1]:g} }} param {{ lr_mult: {pb[0]:g} '
                       f'decay_mult: {pb[1]:g} }}\n'
                       f'  inner_product_param {{ num_output: {nout}{filler(nm)} }} }}')
            bottom = nm
        elif kind == "relu":
            out.append(f'layer {{ name: "{nm}" type: "ReLU" bottom: "{bottom}" top: "{bottom}" }}')
        elif kind == "lrn":
            size, alpha, beta = L[2:5]
            region = f" norm_region: {L[5]}" if len(L) > 5 else ""
            out.append(f'layer {{ name: "{nm}" type: "LRN" bottom: "{bottom}" top: "{nm}" '
                       f'lrn_param {{ local_size: {size} alpha: {alpha:g} beta: {beta:g}{region} }} }}')
            bottom = nm
        elif kind == "drop":
            out.append(f'layer {{ name: "{nm}" type: "Dropout" bottom: "{bottom}" top: "{bottom}" '
                       f'dropout_param {{ dropout_ratio: {L[2]:g} }} }}')
        elif kind == "bn":
            out.append(f'layer {{ name: "{nm}" type: "BatchNorm" bottom: "{bottom}" top: "{nm}"\n'
                       + "".join(f'  param {{ lr_mult: {_BN[0]:g} decay_mult: {_BN[1]:g} }}' for _ in range(3))
                       + ' }')
            bottom = nm
        elif kind == "sigmoid":
            out.append(f'layer {{ name: "{nm}" type: "Sigmoid" bottom: "{bottom}" top: "{nm}" }}')
            bottom = nm
    out.append(f'layer {{ name: "accuracy" type: "Accuracy" bottom: "{bottom}" bottom: "label" top: "accuracy" '
               f'include {{ phase: TEST }} }}')
    out.append(f'layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "{bottom}" bottom: "label" top: "loss" }}')
    return "\n".join(out) + "\n"


def solver_prototxt(name, net_file):
    s = NETS[name]["solver"]
    lines = [f'net: "{net_file}"']
    for k in ("test_iter", "test_interval", "base_lr", "momentum", "weight_decay", "gamma", "power", "stepsize",
              "max_iter"):
        if k in s:
            lines.append(f"{k}: {s[k]}")
    lines.append(f'lr_policy: "{s["lr_policy"]}"')
    lines.append(f'snapshot_prefix: "{s["snapshot_prefix"]}"')
    lines.append("solver_mode: GPU")
    return "\n".join(lines) + "\n"


def write_prototxts(name, directory):
    """Writes <name>_net.prototxt + <name>_solver.prototxt; returns the solver path."""
    import os
    net_file = os.path.join(directory, f"{name}_net.prototxt")
    solver_file = os.path.join(directory, f"{name}_solver.prototxt")
    with open(net_file, "w") as f:
        f.write(net_prototxt(name))
    with open(solver_file, "w") as f:
        f.write(solver_prototxt(name, os.path.basename(net_file)))
    return solver_file


def _relu_maxpool_after(layers, i):
    """The MAX pool tuple when layers[i+1:i+3] is relu + MAX pool in either order, else None."""
    nxt = layers[i + 1:i + 3]
    kinds = sorted(L[0] for L in nxt)
    if kinds != ["pool", "relu"]:
        return None
    pool = next(L for L in nxt if L[0] == "pool")
    return pool if pool[2] == "MAX" else None


def torch_module(name):
    """PyTorch gradient producer with parameters in learnable_params() order.  LRN and BatchNorm layers and every
    conv with a bias followed by ReLU + MAX pool (either order) run on the library's native kernels (layers.py); the
    rest is PyTorch."""
    return _sequential(NETS[name])


def _sequential(net):
    import torch.nn as nn
    from .layers import LRN, BatchNorm, ConvReluMaxPool
    c, h, w = net["input"]
    layers = net["layers"]
    mods, flat, skip = [], None, 0
    for i, L in enumerate(layers):
        if skip:
            skip -= 1
            continue
        kind = L[0]
        if kind == "conv":
            _, _, cout, k, s, p, g, _, pb = L
            conv = nn.Conv2d(c, cout, k, stride=s, padding=p, groups=g, bias=pb is not None)
            h, w, c = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1, cout
            pool = _relu_maxpool_after(layers, i) if pb is not None else None
            if pool is None:
                mods.append(conv)
            else:
                _, _, _, pk, ps = pool
                mods.append(ConvReluMaxPool(conv, pk, ps))
                h, w = _pool_out(h, pk, ps), _pool_out(w, pk, ps)
                skip = 2
        elif kind == "pool":
            _, _, mode, k, s = L
            mods.append((nn.MaxPool2d if mode == "MAX" else nn.AvgPool2d)(k, s, ceil_mode=True))
            h, w = _pool_out(h, k, s), _pool_out(w, k, s)
        elif kind == "ip":
            if flat is None:
                mods.append(nn.Flatten())
                flat = c * h * w
            mods.append(nn.Linear(flat, L[2]))
            flat = L[2]
        elif kind == "relu":
            mods.append(nn.ReLU(inplace=True))
        elif kind == "lrn":
            mods.append(LRN(L[2], alpha=L[3], beta=L[4], k=1.0, region=L[5] if len(L) > 5 else "ACROSS_CHANNELS"))
        elif kind == "drop":
            mods.append(nn.Dropout(L[2]))
        elif kind == "bn":
            mods.append(BatchNorm(c))
        elif kind == "sigmoid":
            mods.append(nn.Sigmoid())
    return nn.Sequential(*mods)


# caffe-public/examples/siamese/mnist_siamese_train_test.prototxt: a 2x28x28 pair sliced into two LeNet trunks with an
# extra 2-output InnerProduct `feat`; every param of the second trunk (the `_p` layers) is named after the first's, so
# the net has LeNet's blobs plus feat's: 431,102 parameters in 10 blobs.
SIAMESE = dict(input=(1, 28, 28), layers=NETS["lenet"]["layers"] + [("ip", "feat", 2, _W, _B)])
SIAMESE_PARAM_COUNT = 431102


def siamese_module():
    """The siamese net as one PyTorch module: both halves of a pair go through the same trunk, whose parameters are in
    learnable_params() order.  forward(pair [N, 2, 28, 28]) -> (feat, feat_p)."""
    import torch.nn as nn

    class Siamese(nn.Module):
        def __init__(self):
            super().__init__()
            self.trunk = _sequential(SIAMESE)

        def forward(self, pair):
            return self.trunk(pair[:, :1]), self.trunk(pair[:, 1:])

    return Siamese()


def contrastive_loss(a, b, sim, margin=1.0, legacy=False, loss_weight=1.0):
    """Caffe's ContrastiveLoss (contrastive_loss_layer.cpp) with its backward: a similar pair (int(sim) != 0) costs
    d^2, a dissimilar one max(margin - d^2, 0) (legacy) or max(margin - d, 0)^2, summed over N pairs / (2N).  The
    gradient of a dissimilar pair divides by d + 1e-4 as Caffe does, so it is not autograd's derivative of the loss."""
    import torch

    class _Loss(torch.autograd.Function):
        @staticmethod
        def forward(ctx, a, b):
            d = a.reshape(a.shape[0], -1) - b.reshape(b.shape[0], -1)
            dist_sq = (d * d).sum(1)
            similar = sim.to(torch.int64) != 0
            if legacy:
                mdist = margin - dist_sq
                dissimilar = mdist.clamp(min=0)
                beta = torch.full_like(dist_sq, -1.0)
            else:
                dist = dist_sq.sqrt()
                mdist = margin - dist
                dissimilar = mdist.clamp(min=0) ** 2
                beta = -mdist / (dist + 1e-4)
            per = torch.where(similar, dist_sq, dissimilar)
            n = a.shape[0]
            scale = torch.where(similar, torch.ones_like(beta), torch.where(mdist > 0, beta, torch.zeros_like(beta)))
            # caffe_set: an exact 0 where a dissimilar pair has !(mdist > 0), not 0 * d (a NaN d stays out of it)
            on = (similar | (mdist > 0))[:, None]
            ctx.save_for_backward(torch.where(on, scale[:, None] * d, torch.zeros_like(d)))
            ctx.shapes = (a.shape, b.shape)
            return loss_weight * (per.sum() / n / 2)

        @staticmethod
        def backward(ctx, grad):
            (g,) = ctx.saved_tensors
            g = g * (grad * loss_weight / g.shape[0])
            return g.reshape(ctx.shapes[0]), (-g).reshape(ctx.shapes[1])

    return _Loss.apply(a, b)


# He et al.'s CIFAR-10 ResNet-20 (tests/golden/configs/cifar10_resnet20_train_test.prototxt): conv1 and three stages of
# three basic blocks, every convolution bias-free and followed by BatchNorm + Scale (with bias), explicit Splits,
# Eltwise SUM shortcuts with a 1x1 stride-2 projection where the shape changes, global AVE pooling and a 10-way
# InnerProduct.  Batch 100 of 3x32x32.
RESNET20 = dict(input=(3, 32, 32), batch=100, classes=10, stages=(16, 32, 64), blocks=3)


def resnet20_module():
    """ResNet-20 as one PyTorch module with its parameters in learnable_params() order: per convolution its weight, the
    BatchNorm's three statistics and the Scale's scale and bias; per block branch2a, branch2b, then the projection
    (branch1) where there is one; the InnerProduct last.  forward(x [N, 3, 32, 32]) -> scores [N, 10]."""
    import torch
    import torch.nn as nn
    from .layers import BatchNorm

    class Scale(nn.Module):
        """Caffe's Scale with bias_term over axis 1: y = x * s[c] + b[c] (scale_layer.cpp), s filled with 1, b with 0."""

        def __init__(self, channels):
            super().__init__()
            self.weight = nn.Parameter(torch.ones(channels))
            self.bias = nn.Parameter(torch.zeros(channels))

        def forward(self, x):
            shape = (1, -1) + (1,) * (x.dim() - 2)
            return x * self.weight.view(shape) + self.bias.view(shape)

    def unit(cin, cout, k, stride):  # conv (no bias) + BatchNorm + Scale
        return nn.Sequential(nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False), BatchNorm(cout),
                             Scale(cout))

    class Block(nn.Module):
        def __init__(self, cin, cout):
            super().__init__()
            stride = 1 if cin == cout else 2
            self.branch2a = unit(cin, cout, 3, stride)
            self.branch2b = unit(cout, cout, 3, 1)
            self.branch1 = unit(cin, cout, 1, 2) if cin != cout else None

        def forward(self, x):
            y = self.branch2b(self.branch2a(x).relu())
            return (y + (self.branch1(x) if self.branch1 is not None else x)).relu()

    class ResNet20(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = unit(3, 16, 3, 1)
            blocks, cin = [], 16
            for cout in RESNET20["stages"]:
                for _ in range(RESNET20["blocks"]):
                    blocks.append(Block(cin, cout))
                    cin = cout
            self.blocks = nn.Sequential(*blocks)
            self.fc10 = nn.Linear(cin, RESNET20["classes"])

        def forward(self, x):
            y = self.blocks(self.conv1(x).relu())
            return self.fc10(y.mean(dim=(2, 3)))

    return ResNet20()
