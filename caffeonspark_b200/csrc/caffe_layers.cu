// caffe_layers.cu -- the memory-bound layers of the CaffeNet / CIFAR-10-quick gradient producer as single
// passes over their tensors (DESIGN.md section 10):
//
//  * cross-channel LRN, forward and backward.  The scale s is never stored: the backward recomputes it from x.
//    One thread walks CH consecutive channels of one pixel with the window (and the backward's second window)
//    in registers; pixels are the fast thread index, so every load and store is coalesced along w.
//  * within-channel LRN (cifar10_full), forward and backward: a 2-D stencil over each plane from a shared-memory
//    tile with a halo; the backward recomputes s as well.
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
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>

#include "caffe_layers.hpp"
#include "fast_div.cuh"

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

// ---------------------------------------------------------------- within-channel LRN
//
// One block per kLrwTileH x kLrwTileW tile of one (n, c) plane, one output per thread.  The block stages x over the
// tile plus a halo (HALF = n/2 for the forward, 2*HALF for the backward: s is needed on the tile plus HALF) in shared
// memory, zero outside the plane, so every global load is a row segment (coalesced along w) and the window sums are
// separable: each window row's n terms are added from 0.f in increasing w, then the n row sums from 0.f in increasing
// h.  A zero cell adds +0.f to a sum of squares, which leaves it unchanged, so this equals the clipped window's sum.
constexpr int kLrwTileW = 32, kLrwTileH = 8, kLrwThreads = kLrwTileW * kLrwTileH;

__device__ __forceinline__ float sq(float v) { return __fmul_rn(v, v); }  // never contracted into an FMA

// s = 1 + alpha * S / n^2 (Caffe's AVE pool divisor counts the pad cells: always n^2 here)
__device__ __forceinline__ float lrw_scale(float S, float nn, float alpha) { return fmaf(alpha, S / nn, 1.f); }

template <typename T, int HALF>
__global__ void __launch_bounds__(kLrwThreads) lrn_within_forward_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                                         int H, int W, int tiles_w, int tiles,
                                                                         float nn, float alpha, float beta) {
  constexpr int N = 2 * HALF + 1, RH = kLrwTileH + 2 * HALF, RW = kLrwTileW + 2 * HALF;
  __shared__ float xs[RH][RW];        // x on the tile + HALF
  __shared__ float hs[RH][kLrwTileW];  // window-row sums of x^2
  const unsigned plane = blockIdx.x / tiles;
  const int t = blockIdx.x - plane * tiles;
  const int h0 = (t / tiles_w) * kLrwTileH, w0 = (t % tiles_w) * kLrwTileW;
  const size_t base = (size_t)plane * H * W;
  const int tid = threadIdx.y * kLrwTileW + threadIdx.x;
  for (int i = tid; i < RH * RW; i += kLrwThreads) {
    const int r = i / RW, c = i - r * RW, h = h0 - HALF + r, w = w0 - HALF + c;
    xs[r][c] = (h >= 0 && h < H && w >= 0 && w < W) ? to_f32(x[base + (size_t)h * W + w]) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < RH * kLrwTileW; i += kLrwThreads) {
    const int r = i / kLrwTileW, c = i - r * kLrwTileW;
    float a = 0.f;
#pragma unroll
    for (int b = 0; b < N; ++b) a += sq(xs[r][c + b]);
    hs[r][c] = a;
  }
  __syncthreads();
  const int ty = threadIdx.y, tx = threadIdx.x, h = h0 + ty, w = w0 + tx;
  if (h >= H || w >= W) return;
  float S = 0.f;
#pragma unroll
  for (int a = 0; a < N; ++a) S += hs[ty + a][tx];
  y[base + (size_t)h * W + w] = from_f32<T>(xs[ty + HALF][tx + HALF] * powf(lrw_scale(S, nn, alpha), -beta));
}

// dx_i = dy_i s_i^-beta - (2 alpha beta / n^2) x_i sum_{j in window(i)} r_j,  r_j = dy_j x_j s_j^-beta / s_j
template <typename T, int HALF>
__global__ void __launch_bounds__(kLrwThreads) lrn_within_backward_kernel(const T* __restrict__ x,
                                                                          const T* __restrict__ dy,
                                                                          T* __restrict__ dx, int H, int W,
                                                                          int tiles_w, int tiles, float nn,
                                                                          float alpha, float beta, float coef) {
  constexpr int N = 2 * HALF + 1;
  constexpr int XH = kLrwTileH + 4 * HALF, XW = kLrwTileW + 4 * HALF;  // x: the tile + 2*HALF
  constexpr int MH = kLrwTileH + 2 * HALF, MW = kLrwTileW + 2 * HALF;  // r: the tile + HALF
  __shared__ float xs[XH][XW];
  __shared__ float hs[XH][MW];  // window-row sums of x^2 over r's columns
  __shared__ float rs[MH][MW];  // r, 0 outside the plane
  __shared__ float hr[MH][kLrwTileW];  // window-row sums of r
  __shared__ float dyc[kLrwTileH][kLrwTileW], sbc[kLrwTileH][kLrwTileW];  // dy and s^-beta on the tile
  const unsigned plane = blockIdx.x / tiles;
  const int t = blockIdx.x - plane * tiles;
  const int h0 = (t / tiles_w) * kLrwTileH, w0 = (t % tiles_w) * kLrwTileW;
  const size_t base = (size_t)plane * H * W;
  const int tid = threadIdx.y * kLrwTileW + threadIdx.x;
  for (int i = tid; i < XH * XW; i += kLrwThreads) {
    const int r = i / XW, c = i - r * XW, h = h0 - 2 * HALF + r, w = w0 - 2 * HALF + c;
    xs[r][c] = (h >= 0 && h < H && w >= 0 && w < W) ? to_f32(x[base + (size_t)h * W + w]) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < XH * MW; i += kLrwThreads) {
    const int r = i / MW, c = i - r * MW;
    float a = 0.f;
#pragma unroll
    for (int b = 0; b < N; ++b) a += sq(xs[r][c + b]);
    hs[r][c] = a;
  }
  __syncthreads();
  for (int i = tid; i < MH * MW; i += kLrwThreads) {
    const int r = i / MW, c = i - r * MW, h = h0 - HALF + r, w = w0 - HALF + c;
    float rv = 0.f;
    if (h >= 0 && h < H && w >= 0 && w < W) {
      float S = 0.f;
#pragma unroll
      for (int a = 0; a < N; ++a) S += hs[r + a][c];
      const float s = lrw_scale(S, nn, alpha), sb = powf(s, -beta);
      const float d = to_f32(dy[base + (size_t)h * W + w]);
      rv = d * xs[r + HALF][c + HALF] * sb / s;
      const int cr = r - HALF, cc = c - HALF;
      if (cr >= 0 && cr < kLrwTileH && cc >= 0 && cc < kLrwTileW) {
        dyc[cr][cc] = d;
        sbc[cr][cc] = sb;
      }
    }
    rs[r][c] = rv;
  }
  __syncthreads();
  for (int i = tid; i < MH * kLrwTileW; i += kLrwThreads) {
    const int r = i / kLrwTileW, c = i - r * kLrwTileW;
    float a = 0.f;
#pragma unroll
    for (int b = 0; b < N; ++b) a += rs[r][c + b];
    hr[r][c] = a;
  }
  __syncthreads();
  const int ty = threadIdx.y, tx = threadIdx.x, h = h0 + ty, w = w0 + tx;
  if (h >= H || w >= W) return;
  float acc = 0.f;
#pragma unroll
  for (int a = 0; a < N; ++a) acc += hr[ty + a][tx];
  const float xv = xs[ty + 2 * HALF][tx + 2 * HALF];
  dx[base + (size_t)h * W + w] = from_f32<T>(fmaf(-(coef * xv), acc, dyc[ty][tx] * sbc[ty][tx]));
}

struct LrwGrid {
  int tiles_w, tiles;
  long long blocks;
  LrwGrid(int num, int channels, int height, int width)
      : tiles_w((width + kLrwTileW - 1) / kLrwTileW), tiles(tiles_w * ((height + kLrwTileH - 1) / kLrwTileH)),
        blocks((long long)num * channels * tiles) {}
  // plane offsets are size_t; in-plane offsets and the block count must fit the kernels' 32-bit arithmetic
  static bool fits(long long blocks, int height, int width) {
    return blocks < (1ll << 31) && (long long)height * width < (1ll << 31);
  }
};

template <int HALF>
struct LrwFwd {
  template <typename T>
  static cudaError_t run(const T* x, T* y, int H, int W, const LrwGrid& g, float nn, float alpha, float beta,
                         cudaStream_t st) {
    lrn_within_forward_kernel<T, HALF><<<(unsigned)g.blocks, dim3(kLrwTileW, kLrwTileH), 0, st>>>(
        x, y, H, W, g.tiles_w, g.tiles, nn, alpha, beta);
    return cudaGetLastError();
  }
};

template <int HALF>
struct LrwBwd {
  template <typename T>
  static cudaError_t run(const T* x, const T* dy, T* dx, int H, int W, const LrwGrid& g, float nn, float alpha,
                         float beta, float coef, cudaStream_t st) {
    lrn_within_backward_kernel<T, HALF><<<(unsigned)g.blocks, dim3(kLrwTileW, kLrwTileH), 0, st>>>(
        x, dy, dx, H, W, g.tiles_w, g.tiles, nn, alpha, beta, coef);
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

// ---------------------------------------------------------------- staged bias + ReLU + MAX pool (the fast path)
//
// The kernels above gather straight from global memory, one element per thread: 9 x loads per pooled output, and up
// to 4 index and 4 dy loads plus ~80 instructions of window arithmetic per dx element, which makes the backward
// issue-bound.  The bias gradient's second pass walks N partials per channel with one thread each, so it waits on N
// loads in turn.  The staged kernels give the same bits with less work:
//
//  * a block copies whole planes into shared memory first (x for the forward; dy and the 1-byte index for the
//    backward) with 16-byte loads over the planes' aligned body and scalar loads for the head and tail;
//  * the forward computes each output from shared memory with pool_forward_kernel's expressions;
//  * the backward (compile-time geometry) computes dx per S x S cell of conv-output elements: the cell's at most
//    ceil(K/S)^2 windows are read once, and each element adds the dy of the windows that point at it in (ph, pw)
//    order from +0.f.  The reference adds +0.f for every other window of the element; g is never -0.f, so that leaves
//    g's bits unchanged and skipping it gives the same g.  g goes to shared memory; then dx is stored coalesced while
//    each warp re-runs the reduction of one warp of pool_backward_kernel's B-thread block (B depends on H * W only):
//    the same elements per lane in the same order, the same butterfly, the plane's warp sums in the same order, so
//    the partials keep their bits;
//  * the bias gradient stages a 32-channel column of partials per block and sums each channel over n in order.
//
// Small planes share a block, so every block has enough elements for its threads.  Both paths' outputs are compared
// bit for bit by tests/test_gpu_layers_fast_path.py.
constexpr int kPoolSmemMax = 48 * 1024;  // dynamic + static shared memory a block may take without an opt-in attribute
constexpr int kPoolFwdThreads = 256;
constexpr int kPoolFwdSmem = 32 * 1024;  // the forward's target per block
constexpr int kPoolFwdMaxPlanes = 16;
constexpr int kPoolBwdThreads = 256;
constexpr int kPoolBwdSmem = 32 * 1024;  // the backward's target per block
constexpr int kPoolBwdMaxWarps = 256;    // the reference kernel's warps a staged backward block stands in for
constexpr int kPoolBwdStatic = (int)sizeof(float) * kPoolBwdMaxWarps;  // warp_sums
constexpr int kStageSlack = 16;  // elements before a staged region's aligned body (< 16 / sizeof(element))

__device__ __forceinline__ float to_staged(float v) { return v; }
__device__ __forceinline__ float to_staged(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ uint8_t to_staged(uint8_t v) { return v; }

// 16 bytes of S, converted, to 16-byte aligned shared memory
__device__ __forceinline__ void put16(uint4 u, float* d, const float*) { *reinterpret_cast<uint4*>(d) = u; }
__device__ __forceinline__ void put16(uint4 u, uint8_t* d, const uint8_t*) { *reinterpret_cast<uint4*>(d) = u; }
__device__ __forceinline__ void put16(uint4 u, float* d, const __nv_bfloat16*) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
  float4 a, b;
  a.x = __low2float(h[0]), a.y = __high2float(h[0]), a.z = __low2float(h[1]), a.w = __high2float(h[1]);
  b.x = __low2float(h[2]), b.y = __high2float(h[2]), b.z = __low2float(h[3]), b.w = __high2float(h[3]);
  reinterpret_cast<float4*>(d)[0] = a;
  reinterpret_cast<float4*>(d)[1] = b;
}

// dst[off + i] = src[i] for i < n, by the whole block, off = the number of S elements src lies past a 16-byte
// boundary: the 16-byte aligned body of src lands on 16-byte aligned dst + off + head (dst must be 16-byte aligned and
// hold n + kStageSlack elements).  Every global load is coalesced; the body's are 16 bytes wide.  Returns off.
template <typename S, typename D>
__device__ __forceinline__ int stage(const S* __restrict__ src, D* __restrict__ dst, int n) {
  constexpr int V = 16 / (int)sizeof(S);
  const int off = (int)((reinterpret_cast<uintptr_t>(src) / sizeof(S)) % V);
  const int head = min(n, (V - off) % V), nv = (n - head) / V, nt = (int)blockDim.x;
  for (int i = threadIdx.x; i < head; i += nt) dst[off + i] = to_staged(src[i]);
  const uint4* sv = reinterpret_cast<const uint4*>(src + head);
  D* dv = dst + off + head;
  int i = threadIdx.x;
  for (; i + nt < nv; i += 2 * nt) {  // two 16-byte loads in flight per thread
    const uint4 a = sv[i], b = sv[i + nt];
    put16(a, dv + i * V, src);
    put16(b, dv + (i + nt) * V, src);
  }
  if (i < nv) put16(sv[i], dv + i * V, src);
  for (int j = head + nv * V + threadIdx.x; j < n; j += nt) dst[off + j] = to_staged(src[j]);
  return off;
}

__host__ __device__ constexpr int round4(int n) { return (n + 3) & ~3; }
// shared memory of a staged forward block of G planes, and of a staged backward block (g, then dy, then index)
int pool_fwd_smem(int G, int hw) { return (int)sizeof(float) * (G * hw + kStageSlack); }
int pool_bwd_smem(int G, int hw, int phw) {
  return (int)sizeof(float) * (round4(G * hw) + round4(G * phw + kStageSlack)) + G * phw + kStageSlack;
}

// One block per G consecutive (n, c) planes: x of the G planes in shared memory, then the G * PH * PW outputs, one
// per thread in turn, stored coalesced.
template <typename T, int KERNEL, int STRIDE>
__global__ void __launch_bounds__(kPoolFwdThreads) pool_forward_staged_kernel(
    const T* __restrict__ x, const float* __restrict__ bias, T* __restrict__ y, uint8_t* __restrict__ index,
    unsigned planes, int G, FastDiv fd_pp, FastDiv fd_pw, FastDiv fd_c, int H, int W, int kernel_rt, int stride_rt) {
  extern __shared__ __align__(16) float smem[];
  const int kernel = KERNEL ? KERNEL : kernel_rt, stride = STRIDE ? STRIDE : stride_rt;
  const unsigned plane0 = blockIdx.x * (unsigned)G;
  const int np = (int)min((unsigned)G, planes - plane0);
  const int HW = H * W, PHW = (int)fd_pp.d;
  const float* xs = smem + stage(x + (size_t)plane0 * HW, smem, np * HW);
  __syncthreads();
  T* yb = y + (size_t)plane0 * PHW;
  uint8_t* ib = index + (size_t)plane0 * PHW;
  for (int o = threadIdx.x; o < np * PHW; o += blockDim.x) {
    const int gp = (int)fd_pp.div(o), e = o - gp * PHW;
    const int ph = (int)fd_pw.div(e), pw = e - ph * (int)fd_pw.d;
    const unsigned plane = plane0 + gp;
    const float b = bias[plane - fd_c.div(plane) * fd_c.d];
    const float* xp = xs + gp * HW;
    const int hs = ph * stride, ws = pw * stride;
    float vmax = -INFINITY;
    int pos = 0;
#pragma unroll
    for (int dh = 0; dh < (KERNEL ? KERNEL : 15); ++dh) {
      if (dh >= kernel || hs + dh >= H) break;
#pragma unroll
      for (int dw = 0; dw < (KERNEL ? KERNEL : 15); ++dw) {
        if (dw >= kernel || ws + dw >= W) break;
        const float v = xp[(hs + dh) * W + ws + dw] + b;
        if (v > vmax || isnan(v)) {  // as pool_forward_kernel
          vmax = v;
          pos = dh * kernel + dw;
        }
      }
    }
    const bool pass = vmax > 0.f || isnan(vmax);
    yb[o] = from_f32<T>(pass ? vmax : 0.f);
    ib[o] = pass ? (uint8_t)pos : kPoolNoGrad;
  }
}

// One block per G consecutive planes (see above).  In the second phase each warp stands in for warps of
// pool_backward_kernel's B-thread blocks in turn: lane l of reference warp vw of a plane sums the elements
// vw * 32 + l + k * B, then the butterfly, then the plane's warp sums in order.  KERNEL/STRIDE 0: the runtime
// geometry, whose first phase gathers per element as pool_backward_kernel does.
template <typename T, int KERNEL, int STRIDE>
__global__ void __launch_bounds__(kPoolBwdThreads) pool_backward_staged_kernel(
    const T* __restrict__ dy, const uint8_t* __restrict__ index, T* __restrict__ dx, float* __restrict__ partials,
    unsigned planes, int G, int B, FastDiv fd_w, FastDiv fd_cells, FastDiv fd_cw, int H, int kernel_rt,
    int stride_rt, int PH, int PW) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float warp_sums[kPoolBwdMaxWarps];
  const int kernel = KERNEL ? KERNEL : kernel_rt, stride = STRIDE ? STRIDE : stride_rt;
  const int W = (int)fd_w.d, HW = H * W, PHW = PH * PW;
  float* gs = smem;                                  // g of the G planes
  float* dys = gs + round4(G * HW);                  // dy of the G planes
  uint8_t* ids = reinterpret_cast<uint8_t*>(dys + round4(G * PHW + kStageSlack));  // index of the G planes
  const unsigned plane0 = blockIdx.x * (unsigned)G;
  const int np = (int)min((unsigned)G, planes - plane0);
  const float* dyb = dys + stage(dy + (size_t)plane0 * PHW, dys, np * PHW);
  const uint8_t* ib = ids + stage(index + (size_t)plane0 * PHW, ids, np * PHW);
  __syncthreads();
  if (KERNEL) {
    constexpr int S = STRIDE ? STRIDE : 1, K = KERNEL ? KERNEL : 1;
    constexpr int NA = (K - 1) / S;  // windows that start before a cell's row (column) and still cover part of it
    const int cells = (int)fd_cells.d, CW = (int)fd_cw.d;
    for (int q = threadIdx.x; q < np * cells; q += blockDim.x) {
      const int gp = (int)fd_cells.div(q), cq = q - gp * cells;
      const int ci = (int)fd_cw.div(cq), cj = cq - ci * CW;
      const float* dyp = dyb + gp * PHW;
      const uint8_t* ip = ib + gp * PHW;
      // the windows (ci - da, cj - db): index (kPoolNoGrad, which matches no position, outside the pooled plane), dy
      unsigned id[NA + 1][NA + 1];
      float v[NA + 1][NA + 1];
#pragma unroll
      for (int da = 0; da <= NA; ++da) {
#pragma unroll
        for (int db = 0; db <= NA; ++db) {
          const int ph = ci - da, pw = cj - db;
          const bool ok = ph >= 0 && pw >= 0 && ph < PH && pw < PW;
          const int o = ok ? ph * PW + pw : 0;
          id[da][db] = ok ? ip[o] : kPoolNoGrad;
          v[da][db] = ok ? dyp[o] : 0.f;
        }
      }
      float* gp_s = gs + gp * HW;
#pragma unroll
      for (int r = 0; r < S; ++r) {
        const int h = ci * S + r;
        if (h >= H) break;
#pragma unroll
        for (int c = 0; c < S; ++c) {
          const int w = cj * S + c;
          if (w >= W) break;
          float g = 0.f;
#pragma unroll
          for (int da = NA; da >= 0; --da) {  // ph = ci - da ascending
#pragma unroll
            for (int db = NA; db >= 0; --db) {
              if (r + da * S < K && c + db * S < K) {  // the window covers (h, w): compile-time
                if (id[da][db] == (unsigned)((r + da * S) * K + c + db * S)) g += v[da][db];
              }
            }
          }
          gp_s[h * W + w] = g;
        }
      }
    }
  } else {
    for (int q = threadIdx.x; q < np * HW; q += blockDim.x) {
      const int gp = q / HW, e = q - gp * HW;
      const float* dyp = dyb + gp * PHW;
      const uint8_t* ip = ib + gp * PHW;
      const int h = (int)fd_w.div(e), w = e - h * W;
      const int phs = h < kernel ? 0 : (h - kernel) / stride + 1, phe = min(h / stride + 1, PH);
      const int pws = w < kernel ? 0 : (w - kernel) / stride + 1, pwe = min(w / stride + 1, PW);
      float g = 0.f;
      for (int ph = phs; ph < phe; ++ph) {
        for (int pw = pws; pw < pwe; ++pw) {
          if (ip[ph * PW + pw] == (h - ph * stride) * kernel + (w - pw * stride)) g += dyp[ph * PW + pw];
        }
      }
      gs[q] = g;
    }
  }
  __syncthreads();
  const int VW = B >> 5, lane = (int)threadIdx.x & 31;
  for (int item = (int)threadIdx.x >> 5; item < np * VW; item += (int)blockDim.x >> 5) {
    const int gp = item / VW, t = (item - gp * VW) * 32 + lane;
    const float* g = gs + gp * HW;
    T* dxp = dx + (size_t)(plane0 + gp) * HW;
    float part = 0.f;
    for (int e = t; e < HW; e += B) {
      dxp[e] = from_f32<T>(g[e]);
      part += g[e];  // the unrounded g: dbias does not depend on the storage type
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) warp_sums[item] = part;
  }
  __syncthreads();
  for (int gp = threadIdx.x; gp < np; gp += blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < VW; ++i) s += warp_sums[gp * VW + i];
    partials[plane0 + gp] = s;
  }
}

// dbias[c] = sum over n, in order, of partials[n * C + c], as bias_grad_kernel: each block stages kBiasRows x 32
// partials at a time (all loads in flight at once) and its first warp adds them, one channel per thread.
constexpr int kBiasThreads = 256, kBiasRows = 128;
__global__ void __launch_bounds__(kBiasThreads) bias_grad_staged_kernel(const float* __restrict__ partials,
                                                                        float* __restrict__ dbias, int N, int C) {
  __shared__ float ps[kBiasRows][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), row = threadIdx.x >> 5;
  float s = 0.f;
  for (int n0 = 0; n0 < N; n0 += kBiasRows) {
    const int rows = min(kBiasRows, N - n0);
#pragma unroll 4
    for (int r = row; r < rows; r += kBiasThreads / 32)
      ps[r][threadIdx.x & 31] = c < C ? partials[(size_t)(n0 + r) * C + c] : 0.f;
    __syncthreads();
    if (threadIdx.x < 32)
      for (int r = 0; r < rows; ++r) s += ps[r][threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.x < 32 && c < C) dbias[c] = s;
}

// the backward's threads per plane (the reference kernel's block size): it depends on the shape only, so the
// partials' summation order is fixed
int pool_backward_block(int hw) { return hw >= 256 ? 256 : ((hw + 31) / 32) * 32; }

struct PoolStaged {
  int fwd_planes, fwd_smem, bwd_planes, bwd_smem;
  PoolStaged(long long planes, int hw, int phw) {
    fwd_planes = (int)std::max(1ll, std::min({(long long)kPoolFwdMaxPlanes, planes, kPoolFwdSmem / (hw * 4ll)}));
    fwd_smem = pool_fwd_smem(fwd_planes, hw);
    bwd_planes = (int)std::max(1ll, std::min((long long)(kPoolBwdMaxWarps / (pool_backward_block(hw) / 32)), planes));
    while (bwd_planes > 1 && pool_bwd_smem(bwd_planes, hw, phw) > kPoolBwdSmem) --bwd_planes;
    bwd_smem = pool_bwd_smem(bwd_planes, hw, phw);
  }
};

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
cudaError_t lrn_within_forward_t(const T* x, T* y, int num, int channels, int height, int width, int local_size,
                                 float alpha, float beta, cudaStream_t stream) {
  const LrwGrid g(num, channels, height, width);
  if (g.blocks == 0) return cudaSuccess;
  if (!LrwGrid::fits(g.blocks, height, width)) return cudaErrorInvalidValue;
  return lrn_dispatch<LrwFwd>(local_size / 2, x, y, height, width, g, (float)(local_size * local_size), alpha, beta,
                              stream);
}

template <typename T>
cudaError_t lrn_within_backward_t(const T* x, const T* dy, T* dx, int num, int channels, int height, int width,
                                  int local_size, float alpha, float beta, cudaStream_t stream) {
  const LrwGrid g(num, channels, height, width);
  if (g.blocks == 0) return cudaSuccess;
  if (!LrwGrid::fits(g.blocks, height, width)) return cudaErrorInvalidValue;
  const float nn = (float)(local_size * local_size);
  return lrn_dispatch<LrwBwd>(local_size / 2, x, dy, dx, height, width, g, nn, alpha, beta,
                              2.f * alpha * beta / nn, stream);
}

template <typename T>
cudaError_t pool_forward_t(const T* x, const float* bias, T* y, uint8_t* index, int num, int channels, int height,
                           int width, int kernel, int stride, int pooled_h, int pooled_w, cudaStream_t stream) {
  const long long total = (long long)num * channels * pooled_h * pooled_w;
  if (total == 0) return cudaSuccess;
  if (total >= (1ll << 31) || (long long)height * width >= (1ll << 31)) return cudaErrorInvalidValue;
  const FastDiv fpp(pooled_h * pooled_w), fpw(pooled_w), fc(channels);
  if (!reference_kernels() && pool_fast_path(num, channels, height, width, kernel, stride)) {
    const long long planes = (long long)num * channels;
    const PoolStaged p(planes, height * width, pooled_h * pooled_w);
    const unsigned grid = (unsigned)((planes + p.fwd_planes - 1) / p.fwd_planes);
    if (kernel == 3 && stride == 2)
      pool_forward_staged_kernel<T, 3, 2><<<grid, kPoolFwdThreads, p.fwd_smem, stream>>>(
          x, bias, y, index, (unsigned)planes, p.fwd_planes, fpp, fpw, fc, height, width, kernel, stride);
    else
      pool_forward_staged_kernel<T, 0, 0><<<grid, kPoolFwdThreads, p.fwd_smem, stream>>>(
          x, bias, y, index, (unsigned)planes, p.fwd_planes, fpp, fpw, fc, height, width, kernel, stride);
    return cudaGetLastError();
  }
  const int block = 256;
  const unsigned grid = (unsigned)((total + block - 1) / block);
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
    const int hw = height * width;
    const int block = pool_backward_block(hw);
    const FastDiv fw(width);
    if (!reference_kernels() && pool_fast_path(num, channels, height, width, kernel, stride)) {
      const PoolStaged p(planes, hw, pooled_h * pooled_w);
      const unsigned grid = (unsigned)((planes + p.bwd_planes - 1) / p.bwd_planes);
      // S x S cells of conv-output elements (compile-time geometry)
      const int cw = (width + stride - 1) / stride, cells = cw * ((height + stride - 1) / stride);
      const FastDiv fcells(cells), fcw(cw);
      if (kernel == 3 && stride == 2)
        pool_backward_staged_kernel<T, 3, 2><<<grid, kPoolBwdThreads, p.bwd_smem, stream>>>(
            dy, index, dx, dbias_partials, (unsigned)planes, p.bwd_planes, block, fw, fcells, fcw, height, kernel, stride, pooled_h,
            pooled_w);
      else
        pool_backward_staged_kernel<T, 0, 0><<<grid, kPoolBwdThreads, p.bwd_smem, stream>>>(
            dy, index, dx, dbias_partials, (unsigned)planes, p.bwd_planes, block, fw, fcells, fcw, height, kernel, stride, pooled_h,
            pooled_w);
    } else if (kernel == 3 && stride == 2)
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
  if (!reference_kernels()) {
    bias_grad_staged_kernel<<<(channels + 31) / 32, kBiasThreads, 0, stream>>>(dbias_partials, dbias, num, channels);
    return cudaGetLastError();
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

cudaError_t lrn_within_forward(const float* x, float* y, int num, int channels, int height, int width, int local_size,
                               float alpha, float beta, cudaStream_t stream) {
  return lrn_within_forward_t(x, y, num, channels, height, width, local_size, alpha, beta, stream);
}
cudaError_t lrn_within_forward(const __nv_bfloat16* x, __nv_bfloat16* y, int num, int channels, int height, int width,
                               int local_size, float alpha, float beta, cudaStream_t stream) {
  return lrn_within_forward_t(x, y, num, channels, height, width, local_size, alpha, beta, stream);
}

cudaError_t lrn_within_backward(const float* x, const float* dy, float* dx, int num, int channels, int height,
                                int width, int local_size, float alpha, float beta, cudaStream_t stream) {
  return lrn_within_backward_t(x, dy, dx, num, channels, height, width, local_size, alpha, beta, stream);
}
cudaError_t lrn_within_backward(const __nv_bfloat16* x, const __nv_bfloat16* dy, __nv_bfloat16* dx, int num,
                                int channels, int height, int width, int local_size, float alpha, float beta,
                                cudaStream_t stream) {
  return lrn_within_backward_t(x, dy, dx, num, channels, height, width, local_size, alpha, beta, stream);
}

int pooled_size(int in, int kernel, int stride) {
  // ceil mode, pad 0; the last window must start inside the input (pooling_output_shape)
  if (kernel < 1 || stride < 1 || in < kernel) return -1;
  int out = (in - kernel + stride - 1) / stride + 1;
  if ((out - 1) * stride >= in) --out;
  return out;
}

namespace {
bool reference_from_env() {
  const char* v = getenv("COS_LAYERS_REFERENCE_KERNELS");
  return v && *v && strcmp(v, "0") != 0;
}
std::atomic<bool> g_reference_kernels{reference_from_env()};
}  // namespace

void set_reference_kernels(bool on) { g_reference_kernels.store(on, std::memory_order_relaxed); }
bool reference_kernels() { return g_reference_kernels.load(std::memory_order_relaxed); }

bool pool_fast_path(int num, int channels, int height, int width, int kernel, int stride) {
  // A 1-wide window shares nothing with its neighbours, so staging buys nothing.  Windows that overlap by more than
  // two rows (k > s + 2) stay on the per-element kernels: no net here uses them and each element's gather grows as
  // (k/s)^2.
  if (num < 1 || channels < 1 || kernel < 2 || stride < 1 || kernel > stride + 2) return false;
  const int ph = pooled_size(height, kernel, stride), pw = pooled_size(width, kernel, stride);
  if (ph < 1 || pw < 1) return false;
  const long long hw = (long long)height * width, phw = (long long)ph * pw, planes = (long long)num * channels;
  // one plane of x (forward), and of dy and index (backward), must fit a block's shared memory
  if (hw > kPoolSmemMax || pool_fwd_smem(1, (int)hw) > kPoolSmemMax ||
      pool_bwd_smem(1, (int)hw, (int)phw) + kPoolBwdStatic > kPoolSmemMax)
    return false;
  // plane and output indices are 32-bit
  return planes * phw < (1ll << 31);
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
