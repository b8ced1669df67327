"""The three BASELINE nets as layer lists -> (a) Caffe prototxt text for the C
library's layout parser, (b) the learnable-blob layout, (c) a PyTorch module
used ONLY as the gradient producer (Net::ForwardBackward is out of scope of
the sync library; SURVEY.md section 8 row f1).

Architectures follow the reference's configuration files
  data/lenet_memory_train_test.prototxt, data/lenet_memory_solver.prototxt
  data/cifar10_quick_train_test.prototxt, data/cifar10_quick_solver.prototxt
  data/bvlc_reference_net.prototxt, data/bvlc_reference_solver.prototxt
(batch 256/device for CaffeNet per
 caffe-public/models/bvlc_reference_caffenet/train_val.prototxt:25).
"""
from .caffenet import SolverDesc

# layer tuples:
#   ("conv", name, cout, k, stride, pad, group, (lr_w, dm_w), (lr_b, dm_b))
#   ("ip",   name, nout, (lr_w, dm_w), (lr_b, dm_b))
#   ("pool", name, "MAX"|"AVE", k, stride)   ("relu", name)  ("lrn", name, size, alpha, beta)
#   ("drop", name, ratio)
_W, _B = (1.0, 1.0), (2.0, 1.0)
_B0 = (2.0, 0.0)  # CaffeNet biases: lr_mult 2, decay_mult 0

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
}

# SURVEY.md App. D: expected flat sizes (checked by tests)
EXPECTED_PARAM_COUNT = {"lenet": 431080, "cifar10_quick": 145578, "caffenet": 60965224}


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
            counts += [cout * (c // g) * k * k, cout]
            lr += [pw[0], pb[0]]
            dm += [pw[1], pb[1]]
            names += [nm + ".w", nm + ".b"]
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
    for L in net["layers"]:
        kind, nm = L[0], L[1]
        if kind == "conv":
            _, _, cout, k, s, p, g, pw, pb = L
            grp = f" group: {g}" if g != 1 else ""
            pad = f" pad: {p}" if p else ""
            out.append(f'layer {{ name: "{nm}" type: "Convolution" bottom: "{bottom}" top: "{nm}"\n'
                       f'  param {{ lr_mult: {pw[0]:g} decay_mult: {pw[1]:g} }} param {{ lr_mult: {pb[0]:g} '
                       f'decay_mult: {pb[1]:g} }}\n'
                       f'  convolution_param {{ num_output: {cout} kernel_size: {k} stride: {s}{pad}{grp} }} }}')
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
                       f'  inner_product_param {{ num_output: {nout} }} }}')
            bottom = nm
        elif kind == "relu":
            out.append(f'layer {{ name: "{nm}" type: "ReLU" bottom: "{bottom}" top: "{bottom}" }}')
        elif kind == "lrn":
            _, _, size, alpha, beta = L
            out.append(f'layer {{ name: "{nm}" type: "LRN" bottom: "{bottom}" top: "{nm}" '
                       f'lrn_param {{ local_size: {size} alpha: {alpha:g} beta: {beta:g} }} }}')
            bottom = nm
        elif kind == "drop":
            out.append(f'layer {{ name: "{nm}" type: "Dropout" bottom: "{bottom}" top: "{bottom}" '
                       f'dropout_param {{ dropout_ratio: {L[2]:g} }} }}')
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
    """PyTorch gradient producer with parameters in learnable_params() order.  LRN layers and every conv followed
    by ReLU + MAX pool (either order) run on the library's native kernels (layers.py); the rest is PyTorch."""
    import torch.nn as nn
    from .layers import LRN, ConvReluMaxPool
    net = NETS[name]
    c, h, w = net["input"]
    layers = net["layers"]
    mods, flat, skip = [], None, 0
    for i, L in enumerate(layers):
        if skip:
            skip -= 1
            continue
        kind = L[0]
        if kind == "conv":
            _, _, cout, k, s, p, g, _, _ = L
            conv = nn.Conv2d(c, cout, k, stride=s, padding=p, groups=g)
            h, w, c = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1, cout
            pool = _relu_maxpool_after(layers, i)
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
            mods.append(LRN(L[2], alpha=L[3], beta=L[4], k=1.0))
        elif kind == "drop":
            mods.append(nn.Dropout(L[2]))
    return nn.Sequential(*mods)
