"""Native producer layers: autograd Functions and modules over the library's LRN (across and within channels) and fused
conv-bias + ReLU + MAX-pool entry points (csrc/caffe_layers.cu, DESIGN.md section 10), its
BatchNorm entry points (csrc/batch_norm.cu, DESIGN.md section 13), its MVN entry points (csrc/mvn.cu, DESIGN.md
section 14), its Crop, SPP and Tile kernels (csrc/native_producer.cu, DESIGN.md section 14) and its TF32 convolutions
(csrc/conv_tf32.cu, DESIGN.md section 10.2).

Activations may be fp32 or bf16 (the mixed-precision producer runs these layers under
torch.autocast, where the convolutions hand them bf16).  bf16 tensors take the bf16 entry points,
which compute in fp32 and round each output once; the conv bias and its gradient stay fp32.

Every call enqueues on torch.cuda.current_stream() and takes its buffers from torch.empty, so
forward/backward can be captured with torch.cuda.graph.  CUDA tensors always take the native
kernels: a missing library or a failed launch raises.  The modules evaluate CPU tensors with the
PyTorch composition that defines the layer, so a producer module can still be checked on a
GPU-less host; the autograd Functions themselves take CUDA tensors only.
"""
import ctypes
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .caffenet import CosError


def _call(fn, *args):
    if not fn(*args):
        raise CosError(_lib.lib().cos_last_error().decode())


_ENTRY = {torch.float32: "", torch.bfloat16: "_bf16"}  # activation dtype -> suffix of the C entry point


def _check(t):
    if not t.is_cuda or t.dtype not in _ENTRY or t.dim() != 4:
        raise CosError(f"native producer layers take 4-d fp32 or bf16 CUDA tensors (no CPU path), got {t.dtype} "
                       f"{tuple(t.shape)} on {t.device}")
    return t.contiguous()


def _entry(name, dtype):
    return getattr(_lib.lib(), name + _ENTRY[dtype])


def _grad(dy, dtype):
    if dy.dtype != dtype:
        raise CosError(f"gradient dtype {dy.dtype} does not match the activation dtype {dtype}")
    return dy.contiguous()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def pooled_size(n, k, s):
    """Ceil-mode pooling with pad 0, the last window starting inside the input (PyTorch's and Caffe's rule)."""
    out = (n - k + s - 1) // s + 1
    return out - 1 if (out - 1) * s >= n else out


class LRNFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, size, alpha, beta, k):
        x = _check(x)
        y = torch.empty_like(x)
        _call(_entry("cos_lrn_forward", x.dtype), x.data_ptr(), y.data_ptr(), *x.shape, size, alpha, beta, k,
              _stream())
        ctx.save_for_backward(x)
        ctx.hyper = (size, alpha, beta, k)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dy = _grad(dy, x.dtype)
        dx = torch.empty_like(x)
        _call(_entry("cos_lrn_backward", x.dtype), x.data_ptr(), dy.data_ptr(), dx.data_ptr(), *x.shape, *ctx.hyper,
              _stream())
        return dx, None, None, None, None


class LRNWithinFunction(torch.autograd.Function):
    """Caffe's WITHIN_CHANNEL LRN on the native stencil kernels (no k: Caffe does not use it for this region)."""

    @staticmethod
    def forward(ctx, x, size, alpha, beta):
        x = _check(x)
        y = torch.empty_like(x)
        _call(_entry("cos_lrn_within_forward", x.dtype), x.data_ptr(), y.data_ptr(), *x.shape, size, alpha, beta,
              _stream())
        ctx.save_for_backward(x)
        ctx.hyper = (size, alpha, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dy = _grad(dy, x.dtype)
        dx = torch.empty_like(x)
        _call(_entry("cos_lrn_within_backward", x.dtype), x.data_ptr(), dy.data_ptr(), dx.data_ptr(), *x.shape,
              *ctx.hyper, _stream())
        return dx, None, None, None


def lrn_within_composite(x, size, alpha, beta):
    """Caffe's WITHIN_CHANNEL LRN as its own layer composition (lrn_layer.cpp): square, AVE pool size x size with pad
    size // 2 and stride 1 (the divisor counts the pad cells), power (1 + alpha * a)^-beta, product with x."""
    a = F.avg_pool2d(x * x, size, stride=1, padding=size // 2, count_include_pad=True)
    return x * torch.pow(1 + alpha * a, -beta)


class BiasReluMaxPoolFunction(torch.autograd.Function):
    """y = max_pool2d(relu(x + bias), kernel, stride, ceil_mode=True) for a bias-free conv output x (fp32 or bf16)
    and an fp32 bias; y and dx have x's dtype, the bias gradient is fp32."""

    @staticmethod
    def forward(ctx, x, bias, kernel, stride):
        x = _check(x)
        if not bias.is_cuda or bias.dtype != torch.float32 or bias.shape != (x.shape[1],):
            raise CosError(f"the pool block's bias must be an fp32 CUDA tensor of {x.shape[1]} elements, got "
                           f"{bias.dtype} {tuple(bias.shape)} on {bias.device}")
        n, c, h, w = x.shape
        ph, pw = pooled_size(h, kernel, stride), pooled_size(w, kernel, stride)
        y = torch.empty((n, c, ph, pw), dtype=x.dtype, device=x.device)
        index = torch.empty((n, c, ph, pw), dtype=torch.uint8, device=x.device)
        _call(_entry("cos_bias_relu_maxpool_forward", x.dtype), x.data_ptr(), bias.contiguous().data_ptr(),
              y.data_ptr(), index.data_ptr(), n, c, h, w, kernel, stride, ph, pw, _stream())
        ctx.save_for_backward(index)
        ctx.dtype = x.dtype
        ctx.geom = (n, c, h, w, kernel, stride, ph, pw)
        ctx.mark_non_differentiable(index)
        return y

    @staticmethod
    def backward(ctx, dy):
        (index,) = ctx.saved_tensors
        n, c, h, w, kernel, stride, ph, pw = ctx.geom
        dy = _grad(dy, ctx.dtype)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device)
        partials = torch.empty((n, c), dtype=torch.float32, device=dy.device)
        db = torch.empty((c,), dtype=torch.float32, device=dy.device)
        _call(_entry("cos_bias_relu_maxpool_backward", ctx.dtype), dy.data_ptr(), index.data_ptr(), dx.data_ptr(),
              partials.data_ptr(), db.data_ptr(), *ctx.geom, _stream())
        return dx, db, None, None


def _bn_geometry(x):
    """(num, channels, height, width) of Caffe's BatchNorm view of x: channels = shape(1) (1 for a 1-axis bottom),
    the remaining axes flattened into height."""
    n = x.shape[0]
    c = x.shape[1] if x.dim() > 1 else 1
    return n, c, x[0].numel() // c if n else 0, 1


def _bn_blob(t, c):
    if not t.is_cuda or t.dtype != torch.float32 or t.numel() != c or not t.is_contiguous():
        raise CosError(f"BatchNorm statistics must be contiguous fp32 CUDA tensors of {c} elements, got {t.dtype} "
                       f"{tuple(t.shape)} on {t.device}")
    return t


class BatchNormFunction(torch.autograd.Function):
    """Caffe's BatchNorm on fp32 or bf16 activations.  The forward updates mean/variance/scale (fp32, usually
    views of data_) in place unless use_global_stats; the backward returns dx only."""

    @staticmethod
    def forward(ctx, x, mean, variance, scale, use_global_stats, moving_average_fraction, eps):
        if not x.is_cuda or x.dtype not in _ENTRY or x.dim() < 1 or x.numel() == 0:
            raise CosError(f"BatchNorm takes non-empty fp32 or bf16 CUDA tensors (no CPU path), got {x.dtype} "
                           f"{tuple(x.shape)} on {x.device}")
        x = x.contiguous()
        geom = _bn_geometry(x)
        n, c = geom[0], geom[1]
        for t, k in ((mean, c), (variance, c), (scale, 1)):
            _bn_blob(t, k)
        y = torch.empty_like(x)
        save = torch.empty(2 * c, dtype=torch.float32, device=x.device)
        work = torch.empty(2 * (n + 1) * c, dtype=torch.float32, device=x.device)
        _call(_entry("cos_batch_norm_forward", x.dtype), x.data_ptr(), y.data_ptr(), mean.data_ptr(),
              variance.data_ptr(), scale.data_ptr(), save.data_ptr(), work.data_ptr(), *geom, int(use_global_stats),
              moving_average_fraction, eps, _stream())
        ctx.save_for_backward(x, save)
        ctx.hyper = (geom, int(use_global_stats), eps)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, save = ctx.saved_tensors
        geom, use_global_stats, eps = ctx.hyper
        dy = _grad(dy, x.dtype)
        dx = torch.empty_like(x)
        work = torch.empty(2 * (geom[0] + 1) * geom[1], dtype=torch.float32, device=x.device)
        _call(_entry("cos_batch_norm_backward", x.dtype), x.data_ptr(), dy.data_ptr(), dx.data_ptr(), save.data_ptr(),
              work.data_ptr(), *geom, use_global_stats, eps, _stream())
        return dx, None, None, None, None, None, None


def batch_norm_composite(x, mean, variance, scale, use_global_stats=False, moving_average_fraction=0.999, eps=1e-5):
    """Caffe's BatchNorm as a PyTorch composition of the same formulas (any device, autograd through x).  Updates
    the three statistics tensors in place unless use_global_stats, as the native forward does."""
    n, c = x.shape[0], (x.shape[1] if x.dim() > 1 else 1)
    xf = x.float().reshape(n, c, -1)
    if use_global_stats:
        s = scale.detach()[0]
        sf = torch.where(s == 0, torch.zeros_like(s), 1 / s)
        mu, var = sf * mean.detach(), sf * variance.detach()
    else:
        # batch statistics as functions of x: autograd then gives Caffe's (dy - mean(dy) - x^ mean(dy x^)) / std
        m = xf.shape[0] * xf.shape[2]
        mu = xf.mean((0, 2))
        var = ((xf - mu.view(1, c, 1)) ** 2).mean((0, 2))
        f = moving_average_fraction
        corr = float(torch.tensor(m, dtype=torch.float32) / torch.tensor(m - 1, dtype=torch.float32)) if m > 1 else 1.0
        with torch.no_grad():
            scale.mul_(f).add_(1)
            mean.copy_(mu + f * mean)
            variance.copy_(corr * var + f * variance)
    sd = torch.pow(var + eps, 0.5)
    y = (xf - mu.view(1, c, 1)) / sd.view(1, c, 1)
    return y.reshape(x.shape).to(x.dtype)


def legacy_shape(shape):
    """Blob::LegacyShape's (num, channels, height, width) of a shape of at most 4 axes: the missing axes are 1."""
    if len(shape) > 4:
        raise CosError("Cannot use legacy accessors on Blobs with > 4 axes.")
    return tuple(shape) + (1,) * (4 - len(shape))


def _mvn_formula_forward(x, rows, dim, normalize_variance, eps):
    """mvn_layer.cu Forward_gpu in x's dtype: -> (y, s) with y [rows, dim] and s [rows, 1] (None mean-only)."""
    alpha = torch.tensor(1.0 / dim, dtype=x.dtype)
    xr = x.reshape(rows, dim)
    y = xr - xr.sum(1, keepdim=True) * alpha
    if not normalize_variance:
        return y, None
    s = torch.pow((y * y).sum(1, keepdim=True) * alpha, 0.5) + torch.tensor(eps, dtype=x.dtype)
    return y / s, s


def _mvn_formula_backward(y, dy, s, dim):
    """mvn_layer.cu Backward_gpu's formula (the exact derivative only where s >> eps) in y's dtype."""
    if s is None:
        return dy - dy.sum(1, keepdim=True) * torch.tensor(1.0 / dim, dtype=y.dtype)
    a, b = (y * dy).sum(1, keepdim=True), dy.sum(1, keepdim=True)
    return (dy + torch.tensor(-1.0 / dim, dtype=y.dtype) * (y * a + b)) / s


class MVN(torch.autograd.Function):
    """Caffe's MVN layer: MVN.apply(x, normalize_variance=True, across_channels=False, eps=1e-9) -> the normalised x
    in the bottom's legacy 4-D shape (num, channels, height, width), as mvn_layer.cpp reshapes its top.  Each of the
    num * channels rows (num with across_channels) of count / rows elements is centred on its mean and, with
    normalize_variance, divided by s = sqrt(mean of squared deviations) + eps.  The backward is Caffe's formula
    dx = (dy - (y * sum(y dy) + sum(dy)) / dim) / s (dy - mean(dy) mean-only), which is the exact derivative only
    where s >> eps.  fp32 CUDA tensors take the native kernels; CPU tensors, of any float dtype, the same formulas
    in PyTorch."""

    @staticmethod
    def forward(ctx, x, normalize_variance=True, across_channels=False, eps=1e-9):
        shape = legacy_shape(x.shape)
        if x.numel() == 0:
            raise CosError(f"MVN needs a bottom with no zero dimension, got {tuple(x.shape)}")
        rows = shape[0] * (1 if across_channels else shape[1])
        dim = x.numel() // rows
        ctx.geom, ctx.in_shape = (rows, dim, bool(normalize_variance)), x.shape
        if not x.is_cuda:
            y, s = _mvn_formula_forward(x, rows, dim, normalize_variance, eps)
            ctx.save_for_backward(y, s)
            return y.reshape(shape)
        if x.dtype != torch.float32:
            raise CosError(f"MVN takes fp32 CUDA tensors (or CPU tensors), got {x.dtype} on {x.device}")
        x = x.contiguous()
        y = torch.empty(shape, dtype=torch.float32, device=x.device)
        stats = torch.empty(5 * rows, dtype=torch.float32, device=x.device)
        work = torch.empty(max(1, _lib.lib().cos_mvn_workspace_floats(rows, dim)), dtype=torch.float32,
                           device=x.device)
        _call(_lib.lib().cos_mvn_forward, x.data_ptr(), y.data_ptr(), stats.data_ptr(), work.data_ptr(), rows, dim,
              int(bool(normalize_variance)), float(eps), _stream())
        ctx.save_for_backward(y, stats)
        return y

    @staticmethod
    def backward(ctx, dy):
        rows, dim, normalize_variance = ctx.geom
        y, saved = ctx.saved_tensors
        if not y.is_cuda:
            return _mvn_formula_backward(y, dy.reshape(rows, dim), saved, dim).reshape(ctx.in_shape), None, None, None
        dy = dy.contiguous().float()
        dx = torch.empty(ctx.in_shape, dtype=torch.float32, device=y.device)
        work = torch.empty(max(1, _lib.lib().cos_mvn_workspace_floats(rows, dim)), dtype=torch.float32,
                           device=y.device)
        stats = saved.clone()  # the backward writes its row sums A and B into stats; the saved tensor stays as it was
        _call(_lib.lib().cos_mvn_backward, y.data_ptr(), dy.data_ptr(), dx.data_ptr(), stats.data_ptr(),
              work.data_ptr(), rows, dim, int(normalize_variance), _stream())
        return dx, None, None, None


class LRN(nn.Module):
    """Caffe's LRN on the native kernels.  region ACROSS_CHANNELS (the default) is nn.LocalResponseNorm's function;
    WITHIN_CHANNEL normalises over a size x size window of each plane and ignores k, as Caffe does.  CPU tensors take
    the PyTorch composition that defines the region."""

    REGIONS = ("ACROSS_CHANNELS", "WITHIN_CHANNEL")

    def __init__(self, size, alpha=1e-4, beta=0.75, k=1.0, region="ACROSS_CHANNELS"):
        super().__init__()
        if size < 1 or size % 2 == 0:
            raise ValueError("LRN only supports odd values for local_size")
        if region not in self.REGIONS:
            raise ValueError(f"LRN region must be one of {self.REGIONS}, got {region!r}")
        self.size, self.alpha, self.beta, self.k, self.region = size, alpha, beta, k, region

    def forward(self, x):
        if self.region == "WITHIN_CHANNEL":
            if not x.is_cuda:
                return lrn_within_composite(x, self.size, self.alpha, self.beta)
            return LRNWithinFunction.apply(x, self.size, self.alpha, self.beta)
        if not x.is_cuda:
            return F.local_response_norm(x, self.size, self.alpha, self.beta, self.k)
        return LRNFunction.apply(x, self.size, self.alpha, self.beta, self.k)


class BatchNorm(nn.Module):
    """Caffe's BatchNorm layer.  Its three blobs (mean sum, variance sum, scale factor) are parameters, in that
    order, so a producer aliases them into data_ like any weight; the forward pass writes them (training mode) and
    they never receive a gradient.  CUDA tensors take the native kernels; CPU tensors batch_norm_composite."""

    def __init__(self, channels, use_global_stats=False, moving_average_fraction=0.999, eps=1e-5):
        super().__init__()
        self.mean = nn.Parameter(torch.zeros(channels), requires_grad=False)
        self.variance = nn.Parameter(torch.zeros(channels), requires_grad=False)
        self.scale_factor = nn.Parameter(torch.zeros(1), requires_grad=False)
        self.use_global_stats = use_global_stats
        self.moving_average_fraction, self.eps = moving_average_fraction, eps

    def reset_parameters(self):
        with torch.no_grad():  # batch_norm_layer.cpp LayerSetUp: caffe_set(0)
            for p in (self.mean, self.variance, self.scale_factor):
                p.zero_()

    def forward(self, x):
        hyper = (self.use_global_stats, self.moving_average_fraction, self.eps)
        if not x.is_cuda:
            return batch_norm_composite(x, self.mean, self.variance, self.scale_factor, *hyper)
        return BatchNormFunction.apply(x, self.mean, self.variance, self.scale_factor, *hyper)


def _conv_geometry(x, weight, stride, padding, groups):
    n, c, h, w = x.shape
    k, _, r, s = weight.shape
    return (n, c, h, w, k, r, s, stride[0], stride[1], padding[0], padding[1], groups)


class ConvFunction(torch.autograd.Function):
    """A convolution on the native TF32 implicit-GEMM kernels (csrc/conv_tf32.cu): fp32 CUDA tensors, NCHW in and
    out.  The data gradient is skipped when x needs none (a net's first layer)."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, groups):
        x, weight = x.contiguous(), weight.contiguous()
        geom = _conv_geometry(x, weight, stride, padding, groups)
        n, _, h, w, k, r, s, sh, sw, ph, pw, _ = geom
        y = torch.empty((n, k, (h + 2 * ph - r) // sh + 1, (w + 2 * pw - s) // sw + 1), dtype=x.dtype, device=x.device)
        _call(_lib.lib().cos_conv_forward, x.data_ptr(), weight.data_ptr(),
              None if bias is None else bias.contiguous().data_ptr(), y.data_ptr(), *geom, _stream())
        ctx.save_for_backward(x, weight)
        ctx.geom, ctx.has_bias = geom, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy, geom = dy.contiguous(), ctx.geom
        dx = dw = db = None
        L = _lib.lib()
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _call(L.cos_conv_backward_data, dy.data_ptr(), weight.data_ptr(), dx.data_ptr(), *geom, _stream())
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(weight)
            work = torch.empty(max(1, L.cos_conv_workspace_floats(*geom)), dtype=torch.float32, device=x.device)
            _call(L.cos_conv_backward_filter, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), work.data_ptr(), *geom,
                  _stream())
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum((0, 2, 3))
        return dx, dw, db, None, None, None


# The geometry where the native kernels beat cuDNN (DESIGN.md section 10.2): few input channels per group, where
# cuDNN's channels-last kernels are poorly filled, and a reduction long enough to fill the k-tiles.  At CaffeNet
# conv1 (3 channels, 363 taps) the native calls take half of cuDNN's forward time and three quarters of its
# weight-gradient time.  From 48 channels up (CaffeNet conv2 to conv5) cuDNN is 1.4 to 5 times faster than this
# mma.sync mainloop, and CIFAR-10-quick (conv1: 3 channels, 75 taps) trained 9 % slower with its conv1 native.
NATIVE_CONV_MAX_GROUP_CHANNELS = 4
NATIVE_CONV_MIN_TAPS = 128


def native_conv(x, weight):
    """Whether conv2d runs on the native TF32 kernels: where cuDNN would run TF32 anyway (fp32 CUDA tensors, autocast
    off, torch.backends.cudnn.allow_tf32 set) and the geometry is one where they are faster (few input channels per
    group, many taps)."""
    return (x.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32 and x.dim() == 4 and
            not torch.is_autocast_enabled("cuda") and torch.backends.cudnn.allow_tf32 and
            weight.dim() == 4 and weight.shape[1] <= NATIVE_CONV_MAX_GROUP_CHANNELS and
            weight.shape[1] * weight.shape[2] * weight.shape[3] >= NATIVE_CONV_MIN_TAPS)


def conv2d(x, weight, bias=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1), groups=1):
    """F.conv2d with int pairs for stride, padding and dilation, on the native kernels where native_conv() holds
    (and the dilation is 1)."""
    if native_conv(x, weight) and tuple(dilation) == (1, 1):
        return ConvFunction.apply(x, weight, bias, tuple(stride), tuple(padding), groups)
    return F.conv2d(x, weight, bias, stride, padding, dilation, groups)


class Conv2d(nn.Conv2d):
    """nn.Conv2d (same parameters, initialisation and type name) whose zero-padded convolution runs through
    conv2d() above."""

    def forward(self, x):
        if self.padding_mode != "zeros" or isinstance(self.padding, str):
            return super().forward(x)
        return conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)


class ConvReluMaxPool(nn.Module):
    """conv -> ReLU -> MAX pool (or conv -> MAX pool -> ReLU, the same function).  `conv` holds the weight and the
    bias; the convolution runs without bias and the native block adds it."""

    def __init__(self, conv: nn.Conv2d, kernel, stride):
        super().__init__()
        self.conv = conv
        self.kernel, self.stride = kernel, stride

    def forward(self, x):
        c = self.conv
        z = conv2d(x, c.weight, None, c.stride, c.padding, c.dilation, c.groups)
        if not z.is_cuda:
            return F.max_pool2d(F.relu(z + c.bias.view(1, -1, 1, 1)), self.kernel, self.stride, ceil_mode=True)
        return BiasReluMaxPoolFunction.apply(z, c.bias, self.kernel, self.stride)


def _crop_call(fn, src, dst, bottom_shape, top_shape, offsets):
    n = len(bottom_shape)
    if not (src.is_cuda and dst.is_cuda and src.dtype == dst.dtype == torch.float32 and src.is_contiguous() and
            dst.is_contiguous()) or len(top_shape) != n or len(offsets) != n:
        raise CosError("Crop takes contiguous fp32 CUDA tensors and one top dim and offset per bottom axis")
    arr = ctypes.c_longlong * n
    _call(fn, src.data_ptr(), dst.data_ptr(), n, arr(*bottom_shape), arr(*top_shape), arr(*offsets), _stream())
    return dst


def crop_forward(x, top_shape, offsets, out=None):
    """Caffe's Crop forward on the native kernel: x[o_0:o_0 + t_0, .., o_n:o_n + t_n] for top_shape t and one offset o
    per axis of x, copied bit for bit into `out` (a new tensor when None)."""
    out = torch.empty(tuple(top_shape), dtype=torch.float32, device=x.device) if out is None else out
    return _crop_call(_lib.lib().cos_crop_forward, x, out, tuple(x.shape), tuple(top_shape), offsets)


def crop_backward(dy, bottom_shape, offsets, out=None):
    """Crop's data gradient on the native kernel: dx of bottom_shape, dy's bits inside the window at `offsets` and +0
    outside it; every element of `out` (a new tensor when None) is written."""
    out = torch.empty(tuple(bottom_shape), dtype=torch.float32, device=dy.device) if out is None else out
    return _crop_call(_lib.lib().cos_crop_backward, dy, out, tuple(bottom_shape), tuple(dy.shape), offsets)


def spp_top_shape(bottom_shape, pyramid_height):
    """Caffe's SPP top for a [N, C, H, W] bottom: Pooling's [N, C, 1, 1] for one level, else the Concat of every level's
    Flatten, [N, C * (4^h - 1) / 3]."""
    n, c = bottom_shape[0], bottom_shape[1]
    return (n, c, 1, 1) if pyramid_height == 1 else (n, c * (4 ** pyramid_height - 1) // 3)


def _spp_check(tensors, pool):
    if pool not in ("MAX", "AVE"):
        raise CosError(f"SPP pool method {pool} is not supported (MAX and AVE are)")
    for t, dtype in tensors:
        if t is not None and not (t.is_cuda and t.dtype == dtype and t.is_contiguous()):
            raise CosError("SPP takes contiguous CUDA tensors: fp32 data and gradients, int32 argmax")


def spp_forward(x, pyramid_height, pool="MAX", out=None, argmax=None):
    """Caffe's SPP forward on the native kernel (one launch): x [N, C, H, W] -> (y of spp_top_shape, argmax), with
    argmax the int32 index in its plane of each MAX window's first maximum (-1 when no value is > -FLT_MAX), None for
    AVE.  `out` and `argmax` are written when given, else new tensors."""
    shape = spp_top_shape(tuple(x.shape), pyramid_height)
    out = torch.empty(shape, dtype=torch.float32, device=x.device) if out is None else out
    if argmax is None and pool == "MAX":
        argmax = torch.empty(shape, dtype=torch.int32, device=x.device)
    _spp_check([(x, torch.float32), (out, torch.float32), (argmax, torch.int32)], pool)
    if x.dim() != 4 or out.numel() != math.prod(shape) or (argmax is not None and argmax.numel() != out.numel()):
        raise CosError(f"SPP takes a 4-d bottom and a top of {shape}")
    _call(_lib.lib().cos_spp_forward, x.data_ptr(), out.data_ptr(), argmax.data_ptr() if argmax is not None else None,
          *x.shape, pyramid_height, int(pool == "MAX"), _stream())
    return out, argmax


def spp_backward(dy, argmax, bottom_shape, pyramid_height, pool="MAX", out=None):
    """SPP's data gradient on the native kernel (one launch): dx of bottom_shape, each level's Pooling gradient added
    in level order; every element of `out` (a new tensor when None) is written.  argmax is the forward's (MAX only)."""
    out = torch.empty(tuple(bottom_shape), dtype=torch.float32, device=dy.device) if out is None else out
    _spp_check([(dy, torch.float32), (out, torch.float32), (argmax if pool == "MAX" else None, torch.int32)], pool)
    shape = spp_top_shape(tuple(bottom_shape), pyramid_height)
    if (len(bottom_shape) != 4 or tuple(out.shape) != tuple(bottom_shape) or dy.numel() != math.prod(shape) or
            (pool == "MAX" and (argmax is None or argmax.numel() != dy.numel()))):
        raise CosError(f"SPP's backward takes a top gradient (and MAX argmax) of {shape} and a dx of {bottom_shape}")
    _call(_lib.lib().cos_spp_backward, dy.data_ptr(), argmax.data_ptr() if pool == "MAX" else None, out.data_ptr(),
          *bottom_shape, pyramid_height, int(pool == "MAX"), _stream())
    return out


def tile_top_shape(bottom_shape, axis, tiles):
    """Caffe's Tile top: the bottom's shape with shape[axis] (negative counted from the end) multiplied by tiles."""
    if not -len(bottom_shape) <= axis < len(bottom_shape):
        raise CosError(f"axis {axis} out of range for {len(bottom_shape)}-D Blob")
    shape = list(bottom_shape)
    shape[axis] *= tiles
    return tuple(shape)


def _tile_call(forward, x, y, bottom_shape, axis, tiles):
    """The forward (x to y) or the backward (y to x) over the bottom-sized x and the top-sized y"""
    n = len(bottom_shape)
    if tiles < 1:
        raise CosError("Number of tiles must be positive.")
    if not all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in (x, y)):
        raise CosError("Tile takes contiguous fp32 CUDA tensors")
    top = tile_top_shape(bottom_shape, axis, tiles)
    axis = axis + n if axis < 0 else axis
    if x.numel() != math.prod(bottom_shape) or y.numel() != math.prod(top):
        raise CosError(f"Tile takes a bottom of {tuple(bottom_shape)} and a top of {top} (axis {axis}, tiles {tiles})")
    fn, src, dst = (_lib.lib().cos_tile_forward, x, y) if forward else (_lib.lib().cos_tile_backward, y, x)
    _call(fn, src.data_ptr(), dst.data_ptr(), n, (ctypes.c_longlong * n)(*bottom_shape), axis, tiles, _stream())


def tile_forward(x, axis, tiles, out=None):
    """Caffe's Tile forward on the native kernel (one launch): x repeated `tiles` times along `axis`, every bit copied
    into `out` (a new tensor of tile_top_shape when None)."""
    shape = tile_top_shape(tuple(x.shape), axis, tiles)
    out = torch.empty(shape, dtype=torch.float32, device=x.device) if out is None else out
    _tile_call(True, x, out, tuple(x.shape), axis, tiles)
    return out


def tile_backward(dy, bottom_shape, axis, tiles, out=None):
    """Tile's data gradient on the native kernel (one launch): dx of bottom_shape, each element the first tile's
    gradient with the later tiles' added in tile order, each add rounded once (Caffe's Backward_cpu bit for bit); every
    element of `out` (a new tensor when None) is written."""
    out = torch.empty(tuple(bottom_shape), dtype=torch.float32, device=dy.device) if out is None else out
    _tile_call(False, out, dy, tuple(bottom_shape), axis, tiles)
    return out
