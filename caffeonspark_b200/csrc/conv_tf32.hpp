// conv_tf32.hpp -- the gradient producer's convolutions on sm_90a TF32 tensor cores (conv_tf32.cu, DESIGN.md
// section 10.2).
//
// x [N, C, H, W], w [K, C/G, R, S], y [N, K, P, Q] are contiguous fp32 NCHW tensors on the device, with
// P = (H + 2 pad_h - R) / stride_h + 1 and Q likewise.  Each group g runs one implicit GEMM whose tile loaders
// gather their operands straight from the NCHW tensors (no column buffer, no layout transpose):
//   forward          y[n, k, p, q]   M = N·P·Q  pixels,  N = K/G  filters,   K = C/G·R·S taps
//   backward_data    dx[n, c, h, w]  M = N·H·W  pixels,  N = C/G  channels,  K = K/G·R·S taps (the strided gather
//                                    keeps the dy elements with (h + pad - r) divisible by the stride)
//   backward_filter  dw[k, c, r, s]  M = K/G    filters, N = C/G·R·S taps,   K = N·P·Q  pixels
// Every operand is rounded to TF32 with cvt.rna (round to nearest, ties away) before it enters the tensor core, and
// the products are accumulated in fp32 by mma.sync.m16n8k8.  The summation order depends on the shape alone:
// backward_filter splits its reduction into conv_filter_chunks() chunks, writes each chunk's partial sums to the
// workspace and adds them in chunk order, so repeated calls give the same bits.  The launchers only enqueue on
// `stream` (no allocation, synchronisation or device query).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace cosb {

struct ConvGeom {
  int n, c, h, w;        // input
  int k, r, s;           // filters and their window
  int stride_h, stride_w, pad_h, pad_w, groups;
  int p, q;              // output plane, from the above
};

// fills g.p and g.q and returns an error message, or nullptr when the shape is one the kernels take
const char* conv_geometry(ConvGeom* g);
// the number of chunks backward_filter splits its N·P·Q reduction into (a function of the shape alone)
int conv_filter_chunks(const ConvGeom& g);
// floats of workspace backward_filter needs (0 when it runs in one chunk)
size_t conv_workspace_floats(const ConvGeom& g);

cudaError_t conv_forward(const float* x, const float* w, const float* bias, float* y, const ConvGeom& g,
                         cudaStream_t stream);
cudaError_t conv_backward_data(const float* dy, const float* w, float* dx, const ConvGeom& g, cudaStream_t stream);
cudaError_t conv_backward_filter(const float* x, const float* dy, float* dw, float* workspace, const ConvGeom& g,
                                 cudaStream_t stream);

}  // namespace cosb
