"""Native producer layers: autograd Functions and modules over the library's LRN and fused
conv-bias + ReLU + MAX-pool entry points (csrc/caffe_layers.cu, DESIGN.md section 10).

Activations may be fp32 or bf16 (the mixed-precision producer runs these layers under
torch.autocast, where the convolutions hand them bf16).  bf16 tensors take the bf16 entry points,
which compute in fp32 and round each output once; the conv bias and its gradient stay fp32.

Every call enqueues on torch.cuda.current_stream() and takes its buffers from torch.empty, so
forward/backward can be captured with torch.cuda.graph.  CUDA tensors always take the native
kernels: a missing library or a failed launch raises.  The modules evaluate CPU tensors with the
PyTorch composition that defines the layer, so a producer module can still be checked on a
GPU-less host; the autograd Functions themselves take CUDA tensors only.
"""
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


class LRN(nn.Module):
    """Caffe's cross-channel LRN (nn.LocalResponseNorm's function) on the native kernels."""

    def __init__(self, size, alpha=1e-4, beta=0.75, k=1.0):
        super().__init__()
        if size < 1 or size % 2 == 0:
            raise ValueError("LRN only supports odd values for local_size")
        self.size, self.alpha, self.beta, self.k = size, alpha, beta, k

    def forward(self, x):
        if not x.is_cuda:
            return F.local_response_norm(x, self.size, self.alpha, self.beta, self.k)
        return LRNFunction.apply(x, self.size, self.alpha, self.beta, self.k)


class ConvReluMaxPool(nn.Module):
    """conv -> ReLU -> MAX pool (or conv -> MAX pool -> ReLU, the same function).  `conv` holds the weight and the
    bias; the convolution runs without bias and the native block adds it."""

    def __init__(self, conv: nn.Conv2d, kernel, stride):
        super().__init__()
        self.conv = conv
        self.kernel, self.stride = kernel, stride

    def forward(self, x):
        c = self.conv
        z = F.conv2d(x, c.weight, None, c.stride, c.padding, c.dilation, c.groups)
        if not z.is_cuda:
            return F.max_pool2d(F.relu(z + c.bias.view(1, -1, 1, 1)), self.kernel, self.stride, ceil_mode=True)
        return BiasReluMaxPoolFunction.apply(z, c.bias, self.kernel, self.stride)
