// batch_norm.cu -- Caffe's BatchNorm layer (batch_norm_layer.cpp, CPU branch) as launch-only kernels
// (DESIGN.md section 13).
//
// Training forward, per channel c over M = N*H*W elements:
//   mean = sum(x) / M,  var = sum(fl(x - mean)^2) / M            (two passes: E((x-mean)^2), not E[x^2]-mean^2)
//   y    = fl(fl(x - mean) / std),  std = powf(fl(var + eps), 0.5)  (caffe_powx is libm powf: powf_half.h)
//   s = fl(fl(s*f) + 1),  mean_blob = fl(mean + fl(f*mean_blob)),
//   var_blob = fl(fl(corr*var) + fl(f*var_blob)),  corr = (float)M / (float)(M-1)   (axpby = scal, then axpy)
// Backward (x^ recomputed from x and the saved statistics):
//   dx = fl(fl(dy + fl(k * fl(S1 + fl(x^ * S2)))) / std),  S1 = sum(dy), S2 = sum(fl(x^ * dy)), k = (float)(-1/M)
// Global statistics: mean = fl(mean_blob * sf), var = fl(var_blob * sf), sf = s == 0 ? 0 : 1/s; dx = fl(dy / std).
//
// Every element operation is one explicitly rounded fp32 operation (__f*_rn: nothing is contracted into an FMA).
// The reductions are deterministic: each plane (n, c) is summed by one thread group in a fixed order (strided
// per-thread sums, an xor tree within the warp, then the warps in order; double accumulators), its sum is stored
// as an fp32 partial, and a one-thread-per-channel kernel adds the partials over n in order.  The grouping depends
// on the shape only, so results are bit-identical run to run and under CUDA-graph replay.
#include <math.h>

#include "batch_norm.hpp"
#include "powf_half.h"

namespace cosb {
namespace {

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

constexpr int kBnBlock = 256;
constexpr int kBnBlockPlane = 1024;  // planes of more elements take a whole block, smaller ones a (sub-)warp

// Threads per plane: the block for large planes, else the smallest power of two >= H*W, at most a warp.
struct PlaneGrid {
  long long planes, blocks;
  int hw, group;
  PlaneGrid(int num, int channels, int height, int width)
      : planes((long long)num * channels), blocks(0), hw(height * width), group(1) {
    if (hw > kBnBlockPlane) group = kBnBlock;
    else
      while (group < hw && group < 32) group <<= 1;
    blocks = (planes * group + kBnBlock - 1) / kBnBlock;
  }
  bool fits() const { return blocks < (1ll << 31); }
};

__device__ __forceinline__ float bn_std(float var, float eps) { return cos_powf_half(__fadd_rn(var, eps)); }
__device__ __forceinline__ float bn_xhat(float x, float mean, float sd) { return __fdiv_rn(__fsub_rn(x, mean), sd); }

// The sum of v over one plane's group of threads, in a fixed order; every thread of the group gets it.
__device__ __forceinline__ double group_sum(double v, int group, double* warp_sums) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    if (o < group) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (group <= 32) return v;
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < kBnBlock / 32; ++i) s += warp_sums[i];
  return s;
}

enum { kSumX = 0, kSumSqDev = 1, kSumDy = 2 };

// part[plane] = sum over the plane of x (kSumX), of fl(x - mean)^2 (kSumSqDev), or of dy (kSumDy, which also
// stores sum(fl(x^ * dy)) at part[planes + plane]).
template <typename T, int MODE>
__global__ void __launch_bounds__(kBnBlock) bn_plane_sums_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                                 const float* __restrict__ save,
                                                                 float* __restrict__ part, long long planes, int C,
                                                                 int hw, int group, float eps) {
  __shared__ double warp_sums[2][kBnBlock / 32];
  const long long t = (long long)blockIdx.x * kBnBlock + threadIdx.x;
  const long long plane = t / group;
  const int lane = (int)(t - plane * group);
  const bool valid = plane < planes;  // no early return: the whole warp takes part in the shuffles
  double s0 = 0.0, s1 = 0.0;
  if (valid) {
    const int c = (int)(plane % C);
    const float mean = MODE == kSumX ? 0.f : save[c];
    const float sd = MODE == kSumDy ? bn_std(save[C + c], eps) : 1.f;
    const T* xp = x + (size_t)plane * hw;
    const T* dp = dy + (size_t)plane * hw;
#pragma unroll 4
    for (int e = lane; e < hw; e += group) {
      const float v = to_f32(xp[e]);
      if (MODE == kSumX) {
        s0 += v;
      } else if (MODE == kSumSqDev) {
        const float d = __fsub_rn(v, mean);
        s0 += __fmul_rn(d, d);
      } else {
        const float g = to_f32(dp[e]);
        s0 += g;
        s1 += __fmul_rn(bn_xhat(v, mean, sd), g);
      }
    }
  }
  s0 = group_sum(s0, group, warp_sums[0]);
  if (MODE == kSumDy) s1 = group_sum(s1, group, warp_sums[1]);
  if (valid && lane == 0) {
    part[plane] = (float)s0;
    if (MODE == kSumDy) part[planes + plane] = (float)s1;
  }
}

// save[c] = mean = (sum over n, in order, of the plane sums) / M
__global__ void bn_mean_kernel(const float* __restrict__ part, float* __restrict__ save, int N, int C, double m) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
#pragma unroll 16  // the loads issue ahead; the additions keep their order
  for (int n = 0; n < N; ++n) s += part[(size_t)n * C + c];
  save[c] = (float)(s / m);
}

// save[C + c] = var, then Caffe's moving average into the three blobs
__global__ void bn_var_update_kernel(const float* __restrict__ part, float* __restrict__ save,
                                     float* __restrict__ mean_blob, float* __restrict__ var_blob,
                                     float* __restrict__ scale_blob, int N, int C, double m, float f, float corr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
#pragma unroll 16  // the loads issue ahead; the additions keep their order
  for (int n = 0; n < N; ++n) s += part[(size_t)n * C + c];
  const float var = (float)(s / m);
  save[C + c] = var;
  mean_blob[c] = __fadd_rn(save[c], __fmul_rn(f, mean_blob[c]));
  var_blob[c] = __fadd_rn(__fmul_rn(corr, var), __fmul_rn(f, var_blob[c]));
  if (c == 0) scale_blob[0] = __fadd_rn(__fmul_rn(scale_blob[0], f), 1.f);
}

// use_global_stats: save = the blobs scaled by 1 / s (0 when s == 0)
__global__ void bn_global_stats_kernel(const float* __restrict__ mean_blob, const float* __restrict__ var_blob,
                                       const float* __restrict__ scale_blob, float* __restrict__ save, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s = scale_blob[0];
  const float sf = s == 0.f ? 0.f : __fdiv_rn(1.f, s);
  save[c] = __fmul_rn(sf, mean_blob[c]);
  save[C + c] = __fmul_rn(sf, var_blob[c]);
}

// sums[c] = S1, sums[C + c] = S2: the backward's plane sums added over n, in order
__global__ void bn_channel_sums_kernel(const float* __restrict__ part, float* __restrict__ sums, long long planes,
                                       int N, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
#pragma unroll 16
  for (int n = 0; n < N; ++n) {
    s1 += part[(size_t)n * C + c];
    s2 += part[planes + (size_t)n * C + c];
  }
  sums[c] = (float)s1;
  sums[C + c] = (float)s2;
}

template <typename T>
__global__ void __launch_bounds__(kBnBlock) bn_normalize_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                                const float* __restrict__ save, long long planes,
                                                                int C, int hw, int group, float eps) {
  const long long t = (long long)blockIdx.x * kBnBlock + threadIdx.x;
  const long long plane = t / group;
  if (plane >= planes) return;
  const int lane = (int)(t - plane * group);
  const int c = (int)(plane % C);
  const float mean = save[c], sd = bn_std(save[C + c], eps);
  const T* xp = x + (size_t)plane * hw;
  T* yp = y + (size_t)plane * hw;
#pragma unroll 4
  for (int e = lane; e < hw; e += group) yp[e] = from_f32<T>(bn_xhat(to_f32(xp[e]), mean, sd));
}

template <typename T, bool GLOBAL>
__global__ void __launch_bounds__(kBnBlock) bn_backward_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                               T* __restrict__ dx, const float* __restrict__ save,
                                                               const float* __restrict__ sums, long long planes,
                                                               int C, int hw, int group, float eps, float k) {
  const long long t = (long long)blockIdx.x * kBnBlock + threadIdx.x;
  const long long plane = t / group;
  if (plane >= planes) return;
  const int lane = (int)(t - plane * group);
  const int c = (int)(plane % C);
  const float mean = save[c], sd = bn_std(save[C + c], eps);
  const float S1 = GLOBAL ? 0.f : sums[c], S2 = GLOBAL ? 0.f : sums[C + c];
  const T* xp = x + (size_t)plane * hw;
  const T* dp = dy + (size_t)plane * hw;
  T* dxp = dx + (size_t)plane * hw;
#pragma unroll 4
  for (int e = lane; e < hw; e += group) {
    const float g = to_f32(dp[e]);
    float r;
    if (GLOBAL) {
      r = __fdiv_rn(g, sd);
    } else {
      const float xh = bn_xhat(to_f32(xp[e]), mean, sd);
      r = __fdiv_rn(__fadd_rn(g, __fmul_rn(k, __fadd_rn(S1, __fmul_rn(xh, S2)))), sd);
    }
    dxp[e] = from_f32<T>(r);
  }
}

constexpr int kChanBlock = 128;

template <typename T>
cudaError_t forward_t(const T* x, T* y, float* mean_blob, float* var_blob, float* scale_blob, float* save,
                      float* part, int num, int channels, int height, int width, bool global, float f, float eps,
                      cudaStream_t st) {
  const PlaneGrid g(num, channels, height, width);
  if (!g.fits()) return cudaErrorInvalidValue;
  const unsigned cb = (unsigned)((channels + kChanBlock - 1) / kChanBlock);
  const unsigned blocks = (unsigned)g.blocks;
  if (global) {
    bn_global_stats_kernel<<<cb, kChanBlock, 0, st>>>(mean_blob, var_blob, scale_blob, save, channels);
  } else {
    const long long m = (long long)num * g.hw;
    const float corr = m > 1 ? (float)m / (float)(m - 1) : 1.f;  // batch_norm_layer.cpp: Dtype(m) / (m - 1)
    bn_plane_sums_kernel<T, kSumX><<<blocks, kBnBlock, 0, st>>>(x, x, save, part, g.planes, channels, g.hw, g.group,
                                                                eps);
    bn_mean_kernel<<<cb, kChanBlock, 0, st>>>(part, save, num, channels, (double)m);
    bn_plane_sums_kernel<T, kSumSqDev><<<blocks, kBnBlock, 0, st>>>(x, x, save, part, g.planes, channels, g.hw,
                                                                    g.group, eps);
    bn_var_update_kernel<<<cb, kChanBlock, 0, st>>>(part, save, mean_blob, var_blob, scale_blob, num, channels,
                                                    (double)m, f, corr);
  }
  bn_normalize_kernel<T><<<blocks, kBnBlock, 0, st>>>(x, y, save, g.planes, channels, g.hw, g.group, eps);
  return cudaGetLastError();
}

template <typename T>
cudaError_t backward_t(const T* x, const T* dy, T* dx, const float* save, float* part, int num, int channels,
                       int height, int width, bool global, float eps, cudaStream_t st) {
  const PlaneGrid g(num, channels, height, width);
  if (!g.fits()) return cudaErrorInvalidValue;
  const unsigned blocks = (unsigned)g.blocks;
  if (global) {
    bn_backward_kernel<T, true><<<blocks, kBnBlock, 0, st>>>(x, dy, dx, save, nullptr, g.planes, channels, g.hw,
                                                             g.group, eps, 0.f);
    return cudaGetLastError();
  }
  const long long m = (long long)num * g.hw;
  const float k = (float)(-1.0 / (double)m);  // Dtype(-1. / (num * spatial_dim))
  float* sums = part + 2 * g.planes;
  bn_plane_sums_kernel<T, kSumDy><<<blocks, kBnBlock, 0, st>>>(x, dy, save, part, g.planes, channels, g.hw, g.group,
                                                               eps);
  bn_channel_sums_kernel<<<(unsigned)((channels + kChanBlock - 1) / kChanBlock), kChanBlock, 0, st>>>(
      part, sums, g.planes, num, channels);
  bn_backward_kernel<T, false><<<blocks, kBnBlock, 0, st>>>(x, dy, dx, save, sums, g.planes, channels, g.hw, g.group,
                                                            eps, k);
  return cudaGetLastError();
}

}  // namespace

cudaError_t batch_norm_forward(const float* x, float* y, float* mean_blob, float* var_blob, float* scale_blob,
                               float* save, float* workspace, int num, int channels, int height, int width,
                               bool use_global_stats, float moving_average_fraction, float eps, cudaStream_t stream) {
  return forward_t(x, y, mean_blob, var_blob, scale_blob, save, workspace, num, channels, height, width,
                   use_global_stats, moving_average_fraction, eps, stream);
}
cudaError_t batch_norm_forward(const __nv_bfloat16* x, __nv_bfloat16* y, float* mean_blob, float* var_blob,
                               float* scale_blob, float* save, float* workspace, int num, int channels, int height,
                               int width, bool use_global_stats, float moving_average_fraction, float eps,
                               cudaStream_t stream) {
  return forward_t(x, y, mean_blob, var_blob, scale_blob, save, workspace, num, channels, height, width,
                   use_global_stats, moving_average_fraction, eps, stream);
}

cudaError_t batch_norm_backward(const float* x, const float* dy, float* dx, const float* save, float* workspace,
                                int num, int channels, int height, int width, bool use_global_stats, float eps,
                                cudaStream_t stream) {
  return backward_t(x, dy, dx, save, workspace, num, channels, height, width, use_global_stats, eps, stream);
}
cudaError_t batch_norm_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx,
                                const float* save, float* workspace, int num, int channels, int height, int width,
                                bool use_global_stats, float eps, cudaStream_t stream) {
  return backward_t(x, dy, dx, save, workspace, num, channels, height, width, use_global_stats, eps, stream);
}

}  // namespace cosb
