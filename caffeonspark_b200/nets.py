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
    from .layers import LRN, BatchNorm, Conv2d, ConvReluMaxPool
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
            conv = Conv2d(c, cout, k, stride=s, padding=p, groups=g, bias=pb is not None)
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


# caffe-public/examples/mnist/mnist_autoencoder.prototxt (tests/golden/configs/mnist_autoencoder_train_test.prototxt):
# InnerProducts 784-1000-500-250-30-250-500-1000-784 with a Sigmoid after each but the code layer (encode4) and the
# output, whose logits go to SigmoidCrossEntropyLoss against the flattened input.  2,837,314 parameters in 16 blobs.
AUTOENCODER = dict(input=(1, 28, 28), batch=100, widths=(784, 1000, 500, 250, 30, 250, 500, 1000, 784))
AUTOENCODER_PARAM_COUNT = 2837314
# tests/golden/configs/mnist_conv_autoencoder_train_test.prototxt: 13,264 parameters in 7 blobs
CONV_AUTOENCODER = dict(input=(1, 28, 28), batch=100)
CONV_AUTOENCODER_PARAM_COUNT = 13264


def autoencoder_module():
    """The MNIST autoencoder as one PyTorch module, parameters in learnable_params() order.  forward(x [N, 1, 28, 28])
    -> logits [N, 784]."""
    import torch.nn as nn
    w = AUTOENCODER["widths"]
    code, mods = w.index(min(w)), [nn.Flatten()]
    for i in range(1, len(w)):
        mods.append(nn.Linear(w[i - 1], w[i]))
        if i not in (code, len(w) - 1):  # no Sigmoid on the code layer (encode4) nor on the logits (decode1)
            mods.append(nn.Sigmoid())
    return nn.Sequential(*mods)


def conv_autoencoder_module():
    """The convolutional autoencoder fixture as one PyTorch module (nn.ConvTranspose2d's weight is [Cin, Cout, KH, KW],
    Caffe's Deconvolution layout).  forward(x [N, 1, 28, 28]) -> logits [N, 1, 28, 28]."""
    import torch.nn as nn
    return nn.Sequential(nn.Conv2d(1, 16, 3, stride=2, padding=1), nn.ReLU(),
                         nn.Conv2d(16, 32, 3, stride=2, padding=1), nn.ReLU(),
                         nn.ConvTranspose2d(32, 16, 4, stride=2, padding=1), nn.ReLU(),
                         nn.ConvTranspose2d(16, 1, 4, stride=2, padding=1, bias=False))


def sigmoid_cross_entropy_loss(logits, target, loss_weight=1.0):
    """Caffe's SigmoidCrossEntropyLoss: the summed cross-entropy of sigmoid(logits) against target, over num =
    logits.shape[0]; its gradient is (sigmoid(logits) - target) * loss_weight / num."""
    import torch.nn.functional as F
    t = target.reshape(logits.shape)
    return loss_weight * F.binary_cross_entropy_with_logits(logits, t, reduction="sum") / logits.shape[0]


# tests/golden/configs/lenet_tanh_train_test.prototxt: the reference's LeNet with a TanH after pool1 and after pool2,
# TanH in place of relu1, and ip2 -> Softmax -> MultinomialLogisticLoss as its head.  LeNet's 431,080 parameters.
LENET_TANH = dict(input=(1, 28, 28), batch=64, classes=10)
LENET_TANH_PARAM_COUNT = 431080
# tests/golden/configs/cifar10_quick_prelu_train_test.prototxt: CIFAR-10-quick with a per-channel PReLU for each ReLU
# and a channel_shared PReLU after ip1: 145,578 + 32 + 32 + 64 + 1 = 145,707 parameters in 14 blobs.
CIFAR10_QUICK_PRELU = dict(input=(3, 32, 32), batch=100, classes=10)
CIFAR10_QUICK_PRELU_PARAM_COUNT = 145707
# tests/golden/configs/cifar10_quick_mvn_train_test.prototxt: CIFAR-10-quick with MVN on the staged input, after conv2
# (then a Scale with a bias), after pool2 (mean-only), after pool3 (eps 0.001, then a Scale with a bias) and across
# ip1's channels: 145,578 + 64 + 128 = 145,770 parameters in 14 blobs.
CIFAR10_QUICK_MVN = dict(input=(3, 32, 32), batch=100, classes=10)
CIFAR10_QUICK_MVN_PARAM_COUNT = 145770


def scale_module(dim, axis=1):
    """Caffe's one-bottom Scale with bias_term over `dim` elements of axis `axis`: y = x * s + b (scale_layer.cpp),
    s filled with 1 and b with 0."""
    import torch
    import torch.nn as nn

    class Scale(nn.Module):
        def __init__(self):
            super().__init__()
            self.weight = nn.Parameter(torch.ones(dim))
            self.bias = nn.Parameter(torch.zeros(dim))

        def forward(self, x):
            shape = (dim,) + (1,) * (x.dim() - axis - 1)
            return x * self.weight.view(shape) + self.bias.view(shape)

    return Scale()


def mvn_module(normalize_variance=True, across_channels=False, eps=1e-9):
    """Caffe's MVN (layers.MVN) as a module: its top has the bottom's legacy 4-D shape."""
    import torch.nn as nn
    from .layers import MVN

    class _MVN(nn.Module):
        def forward(self, x):
            return MVN.apply(x, normalize_variance, across_channels, eps)

    return _MVN()


def cifar10_quick_mvn_module():
    """The MVN CIFAR-10-quick fixture as one PyTorch module, parameters in learnable_params() order.
    forward(x [N, 3, 32, 32]) -> scores [N, 10]."""
    import torch.nn as nn
    return nn.Sequential(mvn_module(), nn.Conv2d(3, 32, 5, padding=2), nn.MaxPool2d(3, 2, ceil_mode=True), nn.ReLU(),
                         nn.Conv2d(32, 32, 5, padding=2), mvn_module(), scale_module(32), nn.ReLU(),
                         nn.AvgPool2d(3, 2, ceil_mode=True), mvn_module(normalize_variance=False),
                         nn.Conv2d(32, 64, 5, padding=2), nn.ReLU(), nn.AvgPool2d(3, 2, ceil_mode=True),
                         mvn_module(eps=1e-3), scale_module(64), nn.Flatten(), nn.Linear(1024, 64),
                         mvn_module(across_channels=True), nn.Flatten(), nn.Linear(64, 10))


def lenet_tanh_module():
    """The TanH LeNet fixture as one PyTorch module, parameters in learnable_params() order.  forward(x [N, 1, 28, 28])
    -> class probabilities [N, 10] (the Softmax's top)."""
    import torch.nn as nn
    return nn.Sequential(nn.Conv2d(1, 20, 5), nn.MaxPool2d(2, 2, ceil_mode=True), nn.Tanh(),
                         nn.Conv2d(20, 50, 5), nn.MaxPool2d(2, 2, ceil_mode=True), nn.Tanh(),
                         nn.Flatten(), nn.Linear(800, 500), nn.Tanh(), nn.Linear(500, 10), nn.Softmax(dim=1))


def cifar10_quick_prelu_module():
    """The PReLU CIFAR-10-quick fixture as one PyTorch module, parameters in learnable_params() order (each PReLU's
    slopes after the layer before it; the shared slope is one value, Caffe's 0-axis blob).  forward(x [N, 3, 32, 32])
    -> scores [N, 10]."""
    import torch.nn as nn
    return nn.Sequential(nn.Conv2d(3, 32, 5, padding=2), nn.MaxPool2d(3, 2, ceil_mode=True), nn.PReLU(32),
                         nn.Conv2d(32, 32, 5, padding=2), nn.PReLU(32), nn.AvgPool2d(3, 2, ceil_mode=True),
                         nn.Conv2d(32, 64, 5, padding=2), nn.PReLU(64), nn.AvgPool2d(3, 2, ceil_mode=True),
                         nn.Flatten(), nn.Linear(1024, 64), nn.PReLU(1), nn.Linear(64, 10))


def multinomial_logistic_loss(prob, label, loss_weight=1.0):
    """Caffe's MultinomialLogisticLoss (multinomial_logistic_loss_layer.cpp): -loss_weight * sum over the num rows of
    log(max(prob[label], 1e-20)) / num.  Its gradient is -loss_weight / num / max(prob[label], 1e-20) at the label (the
    clamp does not stop it, unlike autograd's) and 0 elsewhere."""
    import torch

    class _Loss(torch.autograd.Function):
        @staticmethod
        def forward(ctx, p):
            p2 = p.reshape(p.shape[0], -1)
            idx = label.reshape(-1).long()[:, None]
            picked = torch.gather(p2, 1, idx).clamp(min=1e-20)
            g = torch.zeros_like(p2).scatter_(1, idx, -loss_weight / p2.shape[0] / picked)
            ctx.save_for_backward(g.reshape(p.shape))
            return -loss_weight * torch.log(picked).sum() / p2.shape[0]

        @staticmethod
        def backward(ctx, grad):
            (g,) = ctx.saved_tensors
            return g * grad

    return _Loss.apply(prob)


def hinge_loss(scores, label, norm="L1", loss_weight=1.0):
    """Caffe's HingeLoss (hinge_loss_layer.cpp): h = max(0, 1 + x) off the label and max(0, 1 - x) at it, summed (L1)
    or summed squared (L2) over num = scores.shape[0].  Its gradient is sign(g) * loss_weight / num (L1, sign(0) = 0) or
    g * 2 * loss_weight / num (L2), with g = h off the label and -h at it."""
    import torch

    class _Loss(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x):
            x2 = x.reshape(x.shape[0], -1)
            num = x2.shape[0]
            at = torch.zeros_like(x2, dtype=torch.bool).scatter_(1, label.reshape(-1).long()[:, None], True)
            h = torch.clamp(1 + torch.where(at, -x2, x2), min=0)
            g = torch.where(at, -h, h)
            g = torch.sign(g) * (loss_weight / num) if norm == "L1" else g * (loss_weight * 2 / num)
            ctx.save_for_backward(g.reshape(x.shape))
            return loss_weight * (h.sum() if norm == "L1" else (h * h).sum()) / num

        @staticmethod
        def backward(ctx, grad):
            (g,) = ctx.saved_tensors
            return g * grad

    return _Loss.apply(scores)


# tests/golden/configs/text_cnn_train_test.prototxt: Embed 5000 x 64 (no bias) of 32 tokens, Reshape to N x 1 x 32 x 64,
# three Convolutions of 32 filters spanning 3, 4 and 5 tokens and the whole embedding, ReLU, MAX pool over time, Concat,
# InnerProduct 96 -> 2.  320,000 + 6,176 + 8,224 + 10,272 + 194 = 344,866 parameters in 9 blobs.
TEXT_CNN = dict(tokens=32, batch=50, vocab=5000, dim=64, widths=(3, 4, 5), filters=32, classes=2)
TEXT_CNN_PARAM_COUNT = 344866
# tests/golden/configs/ngram_lm_train_test.prototxt: Embed 2000 x 32 (with its bias) of 4 context tokens, InnerProduct
# 128 -> 128, TanH, InnerProduct 128 -> 2000.  64,032 + 16,512 + 258,000 = 338,544 parameters in 6 blobs.
NGRAM_LM = dict(tokens=4, batch=128, vocab=2000, dim=32, hidden=128)
NGRAM_LM_PARAM_COUNT = 338544


def embed_module(input_dim, num_output, bias=True):
    """Caffe's Embed as a PyTorch module: weight [input_dim, num_output] (then bias [num_output]), forward(ids of any
    shape, float or integer) -> ids.shape + (num_output,), the table's rows (plus the bias)."""
    import torch
    import torch.nn as nn

    class Embed(nn.Module):
        def __init__(self):
            super().__init__()
            self.weight = nn.Parameter(torch.zeros(input_dim, num_output))
            self.bias = nn.Parameter(torch.zeros(num_output)) if bias else None

        def forward(self, ids):
            y = self.weight[ids.long()]
            return y + self.bias if self.bias is not None else y

    return Embed()


def text_cnn_module():
    """The sentence classifier fixture as one PyTorch module, parameters in learnable_params() order.
    forward(tokens [N, 32]) -> scores [N, 2]; its `convs` are the three Convolutions, each followed by ReLU and a MAX
    pool over all its positions."""
    import torch
    import torch.nn as nn
    s = TEXT_CNN

    class TextCNN(nn.Module):
        def __init__(self):
            super().__init__()
            self.embed = embed_module(s["vocab"], s["dim"], bias=False)
            self.convs = nn.ModuleList(nn.Conv2d(1, s["filters"], (k, s["dim"])) for k in s["widths"])
            self.ip = nn.Linear(s["filters"] * len(s["widths"]), s["classes"])

        def forward(self, tokens):
            x = self.embed(tokens).unsqueeze(1)  # Reshape: N x 1 x tokens x dim
            pooled = [torch.relu(c(x)).amax(dim=(2, 3)) for c in self.convs]
            return self.ip(torch.cat(pooled, 1))

    return TextCNN()


def ngram_lm_module():
    """The n-gram language model fixture as one PyTorch module, parameters in learnable_params() order.
    forward(context [N, 4]) -> next-token scores [N, 2000]."""
    import torch.nn as nn
    s = NGRAM_LM
    return nn.Sequential(embed_module(s["vocab"], s["dim"]), nn.Flatten(), nn.Linear(s["tokens"] * s["dim"], s["hidden"]),
                         nn.Tanh(), nn.Linear(s["hidden"], s["vocab"]))


# tests/golden/configs/rnn_lm_train_test.prototxt: time-major sentences of 20 tokens in 32 streams, Embed 2000 x 128 (no
# bias), RNN of 256 units, InnerProduct 256 -> 2000 on axis 2.  256,000 + (32,768 + 256 + 65,536 + 65,536 + 256) +
# (512,000 + 2,000) = 934,352 parameters in 8 blobs.
RNN_LM = dict(steps=20, batch=32, vocab=2000, dim=128, hidden=256)
RNN_LM_PARAM_COUNT = 934352
# tests/golden/configs/rnn_caption_train_test.prototxt: a 1x28x28 image through LeNet's conv/pool stack and ip1 (256) +
# ReLU into x_static of rnn1 (128 units, over Embed 1000 x 64 of the caption), rnn2 (128) over rnn1, both reading one
# cont, InnerProduct 128 -> 1000 on axis 2; 12 timesteps of 16 streams.  547,018 parameters in 20 blobs.
RNN_CAPTION = dict(steps=12, batch=16, vocab=1000, dim=64, hidden=128, image=256)
RNN_CAPTION_PARAM_COUNT = 547018
# tests/golden/configs/rnn_lm_ln_train_test.prototxt: rnn_lm with an MVN over each timestep's 256 hidden outputs and a
# Scale with a bias on axis 2 before the scores: 934,352 + 512 = 934,864 parameters in 10 blobs.
RNN_LM_LN_PARAM_COUNT = 934864


def rnn_module(input_dim, num_output, static_dim=0):
    """Caffe's RNN layer (rnn_layer.cpp's unrolled net, without expose_hidden) as a PyTorch module, parameters in its
    blobs' order: W_xh [H, I], b_h [H], W_xh_static [H, S] (with static_dim), W_hh [H, H], W_ho [H, H], b_o [H].
    forward(x [T, N, ...], cont [T, N], h0 [N, H], x_static [N, ...] or None) -> (o [T, N, H], h_{T-1} [N, H]), with
    h_t = tanh(W_hh (cont_t h_{t-1}) + W_xh x_t + b_h (+ W_xh_static x_static)) and o_t = tanh(W_ho h_t + b_o).  The
    caller carries h_{T-1} into the next call's h0, detached: no gradient crosses calls."""
    import torch
    import torch.nn as nn

    class RNN(nn.Module):
        def __init__(self):
            super().__init__()
            H = num_output
            self.w_xh = nn.Parameter(torch.zeros(H, input_dim))
            self.b_h = nn.Parameter(torch.zeros(H))
            self.w_xh_static = nn.Parameter(torch.zeros(H, static_dim)) if static_dim else None
            self.w_hh = nn.Parameter(torch.zeros(H, H))
            self.w_ho = nn.Parameter(torch.zeros(H, H))
            self.b_o = nn.Parameter(torch.zeros(H))

        def forward(self, x, cont, h0, x_static=None):
            g = x.flatten(2) @ self.w_xh.t() + self.b_h
            z = x_static.flatten(1) @ self.w_xh_static.t() if self.w_xh_static is not None else None
            h, hs = h0, []
            for t in range(x.shape[0]):
                a = (cont[t].unsqueeze(1) * h) @ self.w_hh.t() + g[t]
                h = torch.tanh(a + z if z is not None else a)
                hs.append(h)
            hs = torch.stack(hs)
            return torch.tanh(hs @ self.w_ho.t() + self.b_o), h

    return RNN()


def rnn_lm_module():
    """The RNN language model fixture as one PyTorch module, parameters in learnable_params() order.
    forward(tokens [T, N], cont [T, N], h0 [N, 256]) -> (scores [T, N, 2000], h_{T-1})."""
    import torch.nn as nn
    s = RNN_LM

    class RNNLM(nn.Module):
        def __init__(self):
            super().__init__()
            self.embed = embed_module(s["vocab"], s["dim"], bias=False)
            self.rnn = rnn_module(s["dim"], s["hidden"])
            self.predict = nn.Linear(s["hidden"], s["vocab"])

        def forward(self, tokens, cont, h0):
            o, h = self.rnn(self.embed(tokens), cont, h0)
            return self.predict(o), h

    return RNNLM()


def rnn_caption_module():
    """The miniature LRCN fixture as one PyTorch module, parameters in learnable_params() order.
    forward(image [N, 1, 28, 28], cont [T, N], tokens [T, N], (h1, h2) [N, 128] each) -> (scores [T, N, 1000],
    (h1_{T-1}, h2_{T-1}))."""
    import torch
    import torch.nn as nn
    s = RNN_CAPTION

    class RNNCaption(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = nn.Conv2d(1, 20, 5)
            self.conv2 = nn.Conv2d(20, 50, 5)
            self.ip1 = nn.Linear(800, s["image"])
            self.embed = embed_module(s["vocab"], s["dim"], bias=False)
            self.rnn1 = rnn_module(s["dim"], s["hidden"], s["image"])
            self.rnn2 = rnn_module(s["hidden"], s["hidden"])
            self.predict = nn.Linear(s["hidden"], s["vocab"])

        def forward(self, image, cont, tokens, h0):
            f = nn.functional.max_pool2d(self.conv1(image), 2, 2)
            f = nn.functional.max_pool2d(self.conv2(f), 2, 2)
            f = torch.relu(self.ip1(f.flatten(1)))
            o1, h1 = self.rnn1(self.embed(tokens), cont, h0[0], f)
            o2, h2 = self.rnn2(o1, cont, h0[1])
            return self.predict(o2), (h1, h2)

    return RNNCaption()


def rnn_lm_ln_module():
    """The layer-normalised RNN language model fixture as one PyTorch module, parameters in learnable_params() order.
    forward(tokens [T, N], cont [T, N], h0 [N, 256]) -> (scores [T, N, 2000], h_{T-1})."""
    import torch.nn as nn
    s = RNN_LM

    class RNNLMLN(nn.Module):
        def __init__(self):
            super().__init__()
            self.embed = embed_module(s["vocab"], s["dim"], bias=False)
            self.rnn = rnn_module(s["dim"], s["hidden"])
            self.ln = mvn_module()
            self.scale = scale_module(s["hidden"], axis=2)
            self.predict = nn.Linear(s["hidden"], s["vocab"])

        def forward(self, tokens, cont, h0):
            o, h = self.rnn(self.embed(tokens), cont, h0)
            return self.predict(self.scale(self.ln(o)).flatten(2)), h

    return RNNLMLN()


# tests/golden/configs/unet_train_test.prototxt: a three-level U-Net over 1 x 92 x 92 images and their per-pixel labels
# (batch 8): unpadded 3x3 convolutions at 16, 32 and 64 channels, each followed by ReLU, 2/2 MAX pools, 2x2 stride-2
# up-convolutions (Deconvolution) with ReLU, skips cropped to the up-convolutions' size and concatenated before them,
# and a 1x1 score convolution to 2 classes at 52 x 52.  116,770 parameters in 26 blobs.
UNET = dict(input=(1, 92, 92), batch=8, classes=2, score=52)
UNET_PARAM_COUNT = 116770


def crop(x, size, offsets):
    """Caffe's Crop from axis 2 by slicing: x[:, :, o_h:o_h + h, o_w:o_w + w] for size (h, w), offsets (o_h, o_w)."""
    return x[:, :, offsets[0]:offsets[0] + size[0], offsets[1]:offsets[1] + size[1]]


def unet_module():
    """The U-Net fixture as one PyTorch module, parameters in learnable_params() order.  forward(images [N, 1, 92, 92])
    -> scores [N, 2, 52, 52]; crop_label(labels [N, 1, 92, 92]) -> the labels of the scored pixels.  Every ReLU and
    MAX pool goes through relu() and pool(), so that a caller can fix their branches."""
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    class UNet(nn.Module):
        def __init__(self):
            super().__init__()
            conv = lambda cin, cout: nn.Conv2d(cin, cout, 3)  # noqa: E731
            self.conv1a, self.conv1b = conv(1, 16), conv(16, 16)
            self.conv2a, self.conv2b = conv(16, 32), conv(32, 32)
            self.conv3a, self.conv3b = conv(32, 64), conv(64, 64)
            self.upconv2 = nn.ConvTranspose2d(64, 32, 2, stride=2)
            self.conv4a, self.conv4b = conv(64, 32), conv(32, 32)
            self.upconv1 = nn.ConvTranspose2d(32, 16, 2, stride=2)
            self.conv5a, self.conv5b = conv(32, 16), conv(16, 16)
            self.score = nn.Conv2d(16, 2, 1)

        def relu(self, x):
            return torch.relu(x)

        def pool(self, x):
            return F.max_pool2d(x, 2, 2, ceil_mode=True)

        def forward(self, x):
            r = self.relu
            d1 = r(self.conv1b(r(self.conv1a(x))))
            d2 = r(self.conv2b(r(self.conv2a(self.pool(d1)))))
            d3 = r(self.conv3b(r(self.conv3a(self.pool(d2)))))
            u2 = r(self.upconv2(d3))
            h = torch.cat([crop(d2, u2.shape[2:], (4, 4)), u2], 1)
            u1 = r(self.upconv1(r(self.conv4b(r(self.conv4a(h))))))
            h = torch.cat([crop(d1, u1.shape[2:], (16, 16)), u1], 1)
            return self.score(r(self.conv5b(r(self.conv5a(h)))))

        @staticmethod
        def crop_label(label):
            return crop(label, (UNET["score"], UNET["score"]), (20, 20))

    return UNet()
