// batch_norm.hpp -- Caffe's BatchNorm layer (batch_norm_layer.cpp) for the gradient producer (batch_norm.cu,
// DESIGN.md section 13).
//
// x, y, dy, dx are contiguous NCHW on the device (a 2-axis N x C bottom is passed with height = width = 1), fp32 or
// bf16 in the overloads that take __nv_bfloat16; those compute in fp32 exactly as the fp32 ones and round each
// output element once.  The statistics are fp32 in both:
//   mean_blob, var_blob [C], scale_blob [1]  the layer's three learnable blobs (pointers into data_)
//   save [2C]       the mean and variance the forward normalised with (batch statistics, or the global ones)
//   workspace       bn_workspace_floats(N, C) floats of scratch
// The launchers only enqueue on `stream`: no allocation, no synchronisation, no device query, so they can be
// captured into a CUDA graph.  They return the launch's cudaError_t.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>

namespace cosb {

inline size_t bn_workspace_floats(int num, int channels) { return 2 * ((size_t)num + 1) * (size_t)channels; }

// Training (use_global_stats 0): normalise with the batch statistics and fold them into the three blobs with
// Caffe's moving average.  use_global_stats 1: normalise with mean_blob / s and var_blob / s; the blobs are only read.
cudaError_t batch_norm_forward(const float* x, float* y, float* mean_blob, float* var_blob, float* scale_blob,
                               float* save, float* workspace, int num, int channels, int height, int width,
                               bool use_global_stats, float moving_average_fraction, float eps, cudaStream_t stream);
cudaError_t batch_norm_forward(const __nv_bfloat16* x, __nv_bfloat16* y, float* mean_blob, float* var_blob,
                               float* scale_blob, float* save, float* workspace, int num, int channels, int height,
                               int width, bool use_global_stats, float moving_average_fraction, float eps,
                               cudaStream_t stream);
// dx from dy, the forward's input x and its save buffer.  No parameter gradient exists.
cudaError_t batch_norm_backward(const float* x, const float* dy, float* dx, const float* save, float* workspace,
                                int num, int channels, int height, int width, bool use_global_stats, float eps,
                                cudaStream_t stream);
cudaError_t batch_norm_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx,
                                const float* save, float* workspace, int num, int channels, int height, int width,
                                bool use_global_stats, float eps, cudaStream_t stream);

}  // namespace cosb
