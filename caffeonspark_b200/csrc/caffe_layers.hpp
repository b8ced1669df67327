// caffe_layers.hpp -- native layers of the CaffeNet / CIFAR-10-quick gradient producer (caffe_layers.cu).
//
// All tensors are contiguous NCHW on the device.  Activations (x, y, dy, dx) are fp32, or bf16 in the overloads
// that take __nv_bfloat16: those compute in fp32 exactly as the fp32 ones and round each output element once to
// bf16.  Bias, its gradient and the partials are fp32 in both.  The launchers only enqueue on `stream`: no allocation,
// no synchronisation, no device query, so they can be captured into a CUDA graph.  They return the launch's
// cudaError_t (cudaSuccess when nothing was launched because the tensor is empty).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cosb {

// LRN across channels needs local_size odd and <= kLrnMaxLocalSize.
constexpr int kLrnMaxLocalSize = 15;

cudaError_t lrn_forward(const float* x, float* y, int num, int channels, int height, int width, int local_size,
                        float alpha, float beta, float k, cudaStream_t stream);
cudaError_t lrn_backward(const float* x, const float* dy, float* dx, int num, int channels, int height, int width,
                         int local_size, float alpha, float beta, float k, cudaStream_t stream);
cudaError_t lrn_forward(const __nv_bfloat16* x, __nv_bfloat16* y, int num, int channels, int height, int width,
                        int local_size, float alpha, float beta, float k, cudaStream_t stream);
cudaError_t lrn_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx, int num, int channels,
                         int height, int width, int local_size, float alpha, float beta, float k,
                         cudaStream_t stream);

// LRN within the channel (Caffe's WITHIN_CHANNEL), local_size odd and <= kLrnMaxLocalSize:
// s = 1 + alpha/local_size^2 * sum of x^2 over the local_size x local_size window centred on the pixel, clipped to the
// plane; y = x * s^-beta.  Caffe ignores k for this region, so there is none.  Not in place (x != y, dx != x, dy).
cudaError_t lrn_within_forward(const float* x, float* y, int num, int channels, int height, int width, int local_size,
                               float alpha, float beta, cudaStream_t stream);
cudaError_t lrn_within_backward(const float* x, const float* dy, float* dx, int num, int channels, int height,
                                int width, int local_size, float alpha, float beta, cudaStream_t stream);
cudaError_t lrn_within_forward(const __nv_bfloat16* x, __nv_bfloat16* y, int num, int channels, int height, int width,
                               int local_size, float alpha, float beta, cudaStream_t stream);
cudaError_t lrn_within_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx, int num,
                                int channels, int height, int width, int local_size, float alpha, float beta,
                                cudaStream_t stream);

// Window clipping of ceil-mode pooling with pad 0: the pooled size, or -1 when the shape is invalid.
int pooled_size(int in, int kernel, int stride);

// index == kPoolNoGrad: the window's maximum was <= 0, nothing flows back through it.
constexpr uint8_t kPoolNoGrad = 0xFF;
cudaError_t bias_relu_maxpool_forward(const float* x, const float* bias, float* y, uint8_t* index, int num,
                                      int channels, int height, int width, int kernel, int stride, int pooled_h,
                                      int pooled_w, cudaStream_t stream);
// dbias_partials holds num * channels floats of scratch.
cudaError_t bias_relu_maxpool_backward(const float* dy, const uint8_t* index, float* dx, float* dbias_partials,
                                       float* dbias, int num, int channels, int height, int width, int kernel,
                                       int stride, int pooled_h, int pooled_w, cudaStream_t stream);
cudaError_t bias_relu_maxpool_forward(const __nv_bfloat16* x, const float* bias, __nv_bfloat16* y, uint8_t* index,
                                      int num, int channels, int height, int width, int kernel, int stride,
                                      int pooled_h, int pooled_w, cudaStream_t stream);
cudaError_t bias_relu_maxpool_backward(const __nv_bfloat16* dy, const uint8_t* index, __nv_bfloat16* dx,
                                       float* dbias_partials, float* dbias, int num, int channels, int height,
                                       int width, int kernel, int stride, int pooled_h, int pooled_w,
                                       cudaStream_t stream);

// The bias+ReLU+max-pool launchers run shared-memory staged kernels where pool_fast_path() holds and the per-element
// kernels (the reference path) elsewhere; both give the same bits.  set_reference_kernels(true) forces the reference
// path everywhere, for tests and benchmarks.  Its initial value is COS_LAYERS_REFERENCE_KERNELS (set and not "0":
// on), read once when the library loads.  It is host state read at launch, so the launchers stay graph capturable.
void set_reference_kernels(bool on);
bool reference_kernels();
// true when the staged pool kernels take this geometry (forward and backward alike); a pure host function
bool pool_fast_path(int num, int channels, int height, int width, int kernel, int stride);

}  // namespace cosb
