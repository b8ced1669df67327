// caffe_layers.cu -- the memory-bound layers of the CaffeNet / CIFAR-10-quick gradient producer as single
// passes over their tensors (DESIGN.md section 10):
//
//  * cross-channel LRN, forward and backward.  The scale s is never stored: the backward recomputes it from x.
//    One thread walks CH consecutive channels of one pixel with the window (and the backward's second window)
//    in registers; pixels are the fast thread index, so every load and store is coalesced along w.
//  * conv bias + ReLU + MAX pool, forward and backward.  The forward adds the bias to the bias-free conv
//    output, takes the first maximum of each window and stores a 1-byte window position (kPoolNoGrad when the
//    maximum is <= 0).  The backward gathers dy per conv-output element in PyTorch's max_pool_backward_nchw
//    order, so dx is bit-identical to threshold_backward(max_pool2d_backward(...)), and reduces the bias
//    gradient with per-plane partials and a fixed-order second pass (no float atomics: deterministic).
//
// Every kernel is a template on the activation storage type T (x, y, dy, dx): fp32, or bf16 for the mixed-precision
// producer.  Arithmetic is fp32 for both, in the same expressions, so a bf16 kernel's output is the fp32 kernel's
// output on the upcast inputs rounded once to bf16 (round to nearest even).  The bias, its gradient and the
// gradient's partials are fp32 for both.
#include <math.h>

#include "caffe_layers.hpp"

namespace cosb {
namespace {

// n / d for 0 <= n < 2^31 with a multiply-high and a shift instead of an integer division (a division per
// element costs more issue slots than the element's memory traffic takes time)
struct FastDiv {
  unsigned d, m, s;
  explicit FastDiv(unsigned div) : d(div), m(0), s(0) {
    while (s < 31 && (1u << s) < d) ++s;
    m = (unsigned)((((1ull << 32) * ((1ull << s) - d)) / d) + 1);
  }
  __device__ __forceinline__ unsigned div(unsigned n) const { return (__umulhi(n, m) + n) >> s; }
};

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

constexpr int kLrnChunk = 16;   // channels per thread; the halo costs 2*HALF (fwd) / 4*HALF (bwd) extra loads
constexpr int kLrnBlock = 128;

// blockIdx.x = pixel_block * nchunks + chunk: the chunks of one pixel range run side by side, so the halo
// loads of neighbouring chunks hit L2.
template <typename T, int HALF>
__global__ void __launch_bounds__(kLrnBlock) lrn_forward_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                                int C, FastDiv fd_hw, unsigned npix, int nchunks,
                                                                float alpha_over_n, float beta, float k) {
  const int chunk = blockIdx.x % nchunks;
  const unsigned p = (blockIdx.x / nchunks) * kLrnBlock + threadIdx.x;
  if (p >= npix) return;
  const unsigned HW = fd_hw.d, n = fd_hw.div(p);
  const size_t base = (size_t)n * C * HW + (p - n * HW);
  const int c0 = chunk * kLrnChunk;
  float xv[kLrnChunk + 2 * HALF];
#pragma unroll
  for (int i = 0; i < kLrnChunk + 2 * HALF; ++i) {
    const int c = c0 - HALF + i;
    xv[i] = (c >= 0 && c < C) ? to_f32(x[base + (size_t)c * HW]) : 0.f;
  }
#pragma unroll
  for (int t = 0; t < kLrnChunk; ++t) {
    const int c = c0 + t;
    if (c < C) {
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j <= 2 * HALF; ++j) ss += xv[t + j] * xv[t + j];
      const float s = k + alpha_over_n * ss;
      y[base + (size_t)c * HW] = from_f32<T>(xv[t + HALF] * powf(s, -beta));
    }
  }
}

// dx_c = dy_c s_c^-beta - (2 alpha beta / n) x_c sum_{c' in window(c)} r_c',  r_c' = dy_c' x_c' s_c'^(-beta-1)
template <typename T, int HALF>
__global__ void __launch_bounds__(kLrnBlock) lrn_backward_kernel(const T* __restrict__ x,
                                                                 const T* __restrict__ dy, T* __restrict__ dx,
                                                                 int C, FastDiv fd_hw, unsigned npix, int nchunks,
                                                                 float alpha_over_n, float beta, float k, float coef) {
  const int chunk = blockIdx.x % nchunks;
  const unsigned p = (blockIdx.x / nchunks) * kLrnBlock + threadIdx.x;
  if (p >= npix) return;
  const unsigned HW = fd_hw.d, n = fd_hw.div(p);
  const size_t base = (size_t)n * C * HW + (p - n * HW);
  const int c0 = chunk * kLrnChunk;
  constexpr int NR = kLrnChunk + 2 * HALF;  // channels c0-HALF .. c0+CH+HALF-1: where r and s are needed
  float xv[NR + 2 * HALF];                  // channels c0-2*HALF ..
  float dv[NR];
#pragma unroll
  for (int i = 0; i < NR + 2 * HALF; ++i) {
    const int c = c0 - 2 * HALF + i;
    xv[i] = (c >= 0 && c < C) ? to_f32(x[base + (size_t)c * HW]) : 0.f;
  }
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    const int c = c0 - HALF + i;
    dv[i] = (c >= 0 && c < C) ? to_f32(dy[base + (size_t)c * HW]) : 0.f;
  }
  float r[NR], sb[NR];  // sb = s^-beta
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    const int c = c0 - HALF + i;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j <= 2 * HALF; ++j) ss += xv[i + j] * xv[i + j];
    const float s = k + alpha_over_n * ss;
    sb[i] = powf(s, -beta);
    r[i] = (c >= 0 && c < C) ? dv[i] * xv[i + HALF] * sb[i] / s : 0.f;
  }
#pragma unroll
  for (int t = 0; t < kLrnChunk; ++t) {
    const int c = c0 + t;
    if (c < C) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j <= 2 * HALF; ++j) acc += r[t + j];
      dx[base + (size_t)c * HW] = from_f32<T>(dv[t + HALF] * sb[t + HALF] - coef * xv[t + 2 * HALF] * acc);
    }
  }
}

template <template <int> class Launch, typename... A>
cudaError_t lrn_dispatch(int half, A... args) {
  switch (half) {
    case 0: return Launch<0>::run(args...);
    case 1: return Launch<1>::run(args...);
    case 2: return Launch<2>::run(args...);
    case 3: return Launch<3>::run(args...);
    case 4: return Launch<4>::run(args...);
    case 5: return Launch<5>::run(args...);
    case 6: return Launch<6>::run(args...);
    case 7: return Launch<7>::run(args...);
  }
  return cudaErrorInvalidValue;
}

struct LrnGrid {
  long long npix;
  int nchunks;
  long long blocks;
  FastDiv fd_hw;
  LrnGrid(int num, int channels, int hw)
      : npix((long long)num * hw), nchunks((channels + kLrnChunk - 1) / kLrnChunk),
        blocks(((npix + kLrnBlock - 1) / kLrnBlock) * nchunks), fd_hw(hw) {}
  // pixel indices and the block count must fit the kernels' 32-bit index arithmetic
  bool fits() const { return npix < (1ll << 31) && blocks < (1ll << 31); }
};

template <int HALF>
struct LrnFwd {
  template <typename T>
  static cudaError_t run(const T* x, T* y, int C, const LrnGrid& g, float aon, float beta, float k,
                         cudaStream_t st) {
    lrn_forward_kernel<T, HALF><<<(unsigned)g.blocks, kLrnBlock, 0, st>>>(x, y, C, g.fd_hw, (unsigned)g.npix,
                                                                        g.nchunks, aon, beta, k);
    return cudaGetLastError();
  }
};

template <int HALF>
struct LrnBwd {
  template <typename T>
  static cudaError_t run(const T* x, const T* dy, T* dx, int C, const LrnGrid& g, float aon, float beta,
                         float k, float coef, cudaStream_t st) {
    lrn_backward_kernel<T, HALF><<<(unsigned)g.blocks, kLrnBlock, 0, st>>>(x, dy, dx, C, g.fd_hw, (unsigned)g.npix,
                                                                         g.nchunks, aon, beta, k, coef);
    return cudaGetLastError();
  }
};

// ---------------------------------------------------------------- bias + ReLU + MAX pool

// KERNEL/STRIDE > 0: compile-time pooling geometry (CaffeNet and CIFAR-10-quick: 3/2); 0: the runtime values
template <typename T, int KERNEL, int STRIDE>
__global__ void pool_forward_kernel(const T* __restrict__ x, const float* __restrict__ bias,
                                    T* __restrict__ y, uint8_t* __restrict__ index, unsigned total, FastDiv fd_pp,
                                    FastDiv fd_pw, FastDiv fd_c, int H, int W, int kernel_rt, int stride_rt) {
  const int kernel = KERNEL ? KERNEL : kernel_rt, stride = STRIDE ? STRIDE : stride_rt;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const unsigned plane = fd_pp.div(i);
  const unsigned e = i - plane * fd_pp.d;
  const int ph = (int)fd_pw.div(e);
  const int pw = (int)(e - ph * fd_pw.d);
  const float b = bias[plane - fd_c.div(plane) * fd_c.d];
  const T* xp = x + (size_t)plane * H * W;
  const int hs = ph * stride, ws = pw * stride;
  float vmax = -INFINITY;
  int pos = 0;
#pragma unroll
  for (int dh = 0; dh < (KERNEL ? KERNEL : 15); ++dh) {
    if (dh >= kernel || hs + dh >= H) break;
#pragma unroll
    for (int dw = 0; dw < (KERNEL ? KERNEL : 15); ++dw) {
      if (dw >= kernel || ws + dw >= W) break;
      const float v = to_f32(xp[(hs + dh) * W + ws + dw]) + b;
      if (v > vmax || isnan(v)) {  // first maximum wins; NaN propagates (max_pool_forward_nchw)
        vmax = v;
        pos = dh * kernel + dw;
      }
    }
  }
  const bool pass = vmax > 0.f || isnan(vmax);
  y[i] = from_f32<T>(pass ? vmax : 0.f);
  index[i] = pass ? (uint8_t)pos : kPoolNoGrad;
}

// One block per (n, c) plane: dx of every conv-output element is the sum, over ph then pw, of the dy of the
// windows whose stored position is this element; the plane's sum of dx (= its share of dbias) is reduced in a
// fixed order into partials[plane].
template <typename T, int KERNEL, int STRIDE>
__global__ void pool_backward_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ index,
                                     T* __restrict__ dx, float* __restrict__ partials, FastDiv fd_w, int H,
                                     int kernel_rt, int stride_rt, int PH, int PW) {
  const int kernel = KERNEL ? KERNEL : kernel_rt, stride = STRIDE ? STRIDE : stride_rt;
  const int W = (int)fd_w.d;
  const long long plane = blockIdx.x;
  const T* dyp = dy + (size_t)plane * PH * PW;
  const uint8_t* ip = index + (size_t)plane * PH * PW;
  T* dxp = dx + (size_t)plane * H * W;
  float part = 0.f;
  for (int e = threadIdx.x; e < H * W; e += blockDim.x) {
    const int h = (int)fd_w.div(e), w = e - h * W;
    const int phs = h < kernel ? 0 : (h - kernel) / stride + 1, phe = min(h / stride + 1, PH);
    const int pws = w < kernel ? 0 : (w - kernel) / stride + 1, pwe = min(w / stride + 1, PW);
    float g = 0.f;
    if (KERNEL) {
      // at most NW x NW windows cover an element: issue all their loads first, then sum in (ph, pw) order
      // (adding +0.f for a window that does not point here leaves g's bits unchanged: g is never -0.f)
      constexpr int NW = KERNEL ? (KERNEL + STRIDE - 1) / STRIDE : 1;
      unsigned id[NW][NW];
      float v[NW][NW];
#pragma unroll
      for (int a = 0; a < NW; ++a) {
#pragma unroll
        for (int b = 0; b < NW; ++b) {
          const bool ok = phs + a < phe && pws + b < pwe;
          const int o = ok ? (phs + a) * PW + pws + b : 0;
          id[a][b] = ok ? ip[o] : kPoolNoGrad;
          v[a][b] = ok ? to_f32(dyp[o]) : 0.f;
        }
      }
#pragma unroll
      for (int a = 0; a < NW; ++a) {
#pragma unroll
        for (int b = 0; b < NW; ++b)
          g += id[a][b] == (unsigned)((h - (phs + a) * stride) * kernel + (w - (pws + b) * stride)) ? v[a][b] : 0.f;
      }
    } else {
      for (int ph = phs; ph < phe; ++ph) {
        for (int pw = pws; pw < pwe; ++pw) {
          if (ip[ph * PW + pw] == (h - ph * stride) * kernel + (w - pw * stride)) g += to_f32(dyp[ph * PW + pw]);
        }
      }
    }
    dxp[e] = from_f32<T>(g);
    part += g;  // the unrounded g: dbias does not depend on the storage type
  }
  __shared__ float warp_sums[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += warp_sums[i];
    partials[plane] = s;
  }
}

// dbias[c] = sum over n, in order, of partials[n * C + c]
__global__ void bias_grad_kernel(const float* __restrict__ partials, float* __restrict__ dbias, int N, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int n = 0; n < N; ++n) s += partials[(size_t)n * C + c];
  dbias[c] = s;
}

template <typename T>
cudaError_t lrn_forward_t(const T* x, T* y, int num, int channels, int height, int width, int local_size, float alpha,
                          float beta, float k, cudaStream_t stream) {
  const LrnGrid g(num, channels, height * width);
  if (g.blocks == 0) return cudaSuccess;
  if (!g.fits()) return cudaErrorInvalidValue;
  return lrn_dispatch<LrnFwd>(local_size / 2, x, y, channels, g, alpha / local_size, beta, k, stream);
}

template <typename T>
cudaError_t lrn_backward_t(const T* x, const T* dy, T* dx, int num, int channels, int height, int width,
                           int local_size, float alpha, float beta, float k, cudaStream_t stream) {
  const LrnGrid g(num, channels, height * width);
  if (g.blocks == 0) return cudaSuccess;
  if (!g.fits()) return cudaErrorInvalidValue;
  return lrn_dispatch<LrnBwd>(local_size / 2, x, dy, dx, channels, g, alpha / local_size, beta, k,
                              2.f * alpha * beta / local_size, stream);
}

template <typename T>
cudaError_t pool_forward_t(const T* x, const float* bias, T* y, uint8_t* index, int num, int channels, int height,
                           int width, int kernel, int stride, int pooled_h, int pooled_w, cudaStream_t stream) {
  const long long total = (long long)num * channels * pooled_h * pooled_w;
  if (total == 0) return cudaSuccess;
  if (total >= (1ll << 31) || (long long)height * width >= (1ll << 31)) return cudaErrorInvalidValue;
  const int block = 256;
  const unsigned grid = (unsigned)((total + block - 1) / block);
  const FastDiv fpp(pooled_h * pooled_w), fpw(pooled_w), fc(channels);
  if (kernel == 3 && stride == 2)
    pool_forward_kernel<T, 3, 2><<<grid, block, 0, stream>>>(x, bias, y, index, (unsigned)total, fpp, fpw, fc,
                                                             height, width, kernel, stride);
  else
    pool_forward_kernel<T, 0, 0><<<grid, block, 0, stream>>>(x, bias, y, index, (unsigned)total, fpp, fpw, fc,
                                                             height, width, kernel, stride);
  return cudaGetLastError();
}

template <typename T>
cudaError_t pool_backward_t(const T* dy, const uint8_t* index, T* dx, float* dbias_partials, float* dbias, int num,
                            int channels, int height, int width, int kernel, int stride, int pooled_h, int pooled_w,
                            cudaStream_t stream) {
  const long long planes = (long long)num * channels;
  if (channels == 0) return cudaSuccess;
  if (planes > 0) {
    if (planes >= (1ll << 31) || (long long)height * width >= (1ll << 31)) return cudaErrorInvalidValue;
    // the block size depends on the shape only, so the partials' summation order is fixed
    const int hw = height * width;
    const int block = hw >= 256 ? 256 : ((hw + 31) / 32) * 32;
    const FastDiv fw(width);
    if (kernel == 3 && stride == 2)
      pool_backward_kernel<T, 3, 2><<<(unsigned)planes, block, 0, stream>>>(dy, index, dx, dbias_partials, fw,
                                                                            height, kernel, stride, pooled_h,
                                                                            pooled_w);
    else
      pool_backward_kernel<T, 0, 0><<<(unsigned)planes, block, 0, stream>>>(dy, index, dx, dbias_partials, fw,
                                                                            height, kernel, stride, pooled_h,
                                                                            pooled_w);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  bias_grad_kernel<<<(channels + 127) / 128, 128, 0, stream>>>(dbias_partials, dbias, num, channels);
  return cudaGetLastError();
}

}  // namespace

cudaError_t lrn_forward(const float* x, float* y, int num, int channels, int height, int width, int local_size,
                        float alpha, float beta, float k, cudaStream_t stream) {
  return lrn_forward_t(x, y, num, channels, height, width, local_size, alpha, beta, k, stream);
}
cudaError_t lrn_forward(const __nv_bfloat16* x, __nv_bfloat16* y, int num, int channels, int height, int width,
                        int local_size, float alpha, float beta, float k, cudaStream_t stream) {
  return lrn_forward_t(x, y, num, channels, height, width, local_size, alpha, beta, k, stream);
}

cudaError_t lrn_backward(const float* x, const float* dy, float* dx, int num, int channels, int height, int width,
                         int local_size, float alpha, float beta, float k, cudaStream_t stream) {
  return lrn_backward_t(x, dy, dx, num, channels, height, width, local_size, alpha, beta, k, stream);
}
cudaError_t lrn_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx, int num, int channels,
                         int height, int width, int local_size, float alpha, float beta, float k,
                         cudaStream_t stream) {
  return lrn_backward_t(x, dy, dx, num, channels, height, width, local_size, alpha, beta, k, stream);
}

int pooled_size(int in, int kernel, int stride) {
  // ceil mode, pad 0; the last window must start inside the input (pooling_output_shape)
  if (kernel < 1 || stride < 1 || in < kernel) return -1;
  int out = (in - kernel + stride - 1) / stride + 1;
  if ((out - 1) * stride >= in) --out;
  return out;
}

cudaError_t bias_relu_maxpool_forward(const float* x, const float* bias, float* y, uint8_t* index, int num,
                                      int channels, int height, int width, int kernel, int stride, int pooled_h,
                                      int pooled_w, cudaStream_t stream) {
  return pool_forward_t(x, bias, y, index, num, channels, height, width, kernel, stride, pooled_h, pooled_w, stream);
}
cudaError_t bias_relu_maxpool_forward(const __nv_bfloat16* x, const float* bias, __nv_bfloat16* y, uint8_t* index,
                                      int num, int channels, int height, int width, int kernel, int stride,
                                      int pooled_h, int pooled_w, cudaStream_t stream) {
  return pool_forward_t(x, bias, y, index, num, channels, height, width, kernel, stride, pooled_h, pooled_w, stream);
}

cudaError_t bias_relu_maxpool_backward(const float* dy, const uint8_t* index, float* dx, float* dbias_partials,
                                       float* dbias, int num, int channels, int height, int width, int kernel,
                                       int stride, int pooled_h, int pooled_w, cudaStream_t stream) {
  return pool_backward_t(dy, index, dx, dbias_partials, dbias, num, channels, height, width, kernel, stride, pooled_h,
                         pooled_w, stream);
}
cudaError_t bias_relu_maxpool_backward(const __nv_bfloat16* dy, const uint8_t* index, __nv_bfloat16* dx,
                                       float* dbias_partials, float* dbias, int num, int channels, int height,
                                       int width, int kernel, int stride, int pooled_h, int pooled_w,
                                       cudaStream_t stream) {
  return pool_backward_t(dy, index, dx, dbias_partials, dbias, num, channels, height, width, kernel, stride, pooled_h,
                         pooled_w, stream);
}

}  // namespace cosb
