// native_producer.cu -- kernels and device side of the built-in gradient producer (DESIGN.md section 14).
//
// One fp32 GEMM core serves every convolution and inner product, forward and both backwards: a 64x64x16 shared-memory
// tile with FFMA and fp32 accumulation, templated on how it gathers its A and B operands and how it stores C.
// Convolutions are implicit GEMMs (the tile loader gathers im2col, or the transposed-convolution window for the data
// gradient, on the fly; no column buffer exists).  A Deconvolution runs as the convolution from its top to its bottom,
// on the same three instantiations.  No TF32, no atomics: every output element is one thread's sum over
// k in increasing order, and weight gradients reduce over N*OH*OW in fixed chunks (split_chunk) whose partials a
// second kernel adds in chunk order.  Bias gradients are fixed-shape block reductions.  So a forward/backward is bitwise
// reproducible run to run.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <type_traits>

#include "batch_norm.hpp"
#include "caffe_layers.hpp"
#include "fast_div.cuh"
#include "fused_sync_sgd.hpp"
#include "mvn.hpp"
#include "native_producer.hpp"

namespace cosb {
namespace {

constexpr int kBM = 64, kBN = 64, kBK = 16, kGemmThreads = 256;
constexpr int kSplitK = 512;    // weight gradients: smallest k-chunk of one partial (a multiple of kBK)
constexpr int kMaxSplits = 256;  // at most this many partials (gridDim.z, and the workspace is splits * weights)
constexpr int kThreads = 256;

// ------------------------------------------------------------------ operand gathers: value at (row, col)
struct DenseRM {  // p[r * ld + c]
  const float* p;
  int ld;
  __device__ float operator()(int r, int c) const { return __ldg(p + (size_t)r * ld + c); }
};
struct DenseCM {  // p[c * ld + r]
  const float* p;
  int ld;
  __device__ float operator()(int r, int c) const { return __ldg(p + (size_t)c * ld + r); }
};
struct ConvGeom {
  int C, H, W, KH, KW, SH, SW, PH, PW, OH, OW;
};
// B[k, j] of the forward: k = (ci * KH + kh) * KW + kw, j = (n * OH + oh) * OW + ow; zero padding
struct Im2col {
  const float* x;
  ConvGeom g;
  __device__ float operator()(int k, int j) const {
    const int kw = k % g.KW, t = k / g.KW, kh = t % g.KH, ci = t / g.KH;
    const int ow = j % g.OW, t2 = j / g.OW, oh = t2 % g.OH, n = t2 / g.OH;
    const int h = oh * g.SH - g.PH + kh, w = ow * g.SW - g.PW + kw;
    if (h < 0 || h >= g.H || w < 0 || w >= g.W) return 0.f;
    return __ldg(x + ((size_t)(n * g.C + ci) * g.H + h) * g.W + w);
  }
};
template <class G>
struct Transposed {
  G g;
  __device__ float operator()(int r, int c) const { return g(c, r); }
};
// A[c, j] = dy[n, c, p] with j = n * HW + p
struct ChanMajor {
  const float* p;
  int C, HW;
  __device__ float operator()(int c, int j) const { return __ldg(p + ((size_t)(j / HW) * C + c) * HW + j % HW); }
};
// A[ci, k2] = W[co, ci, kh, kw] with k2 = (co * KH + kh) * KW + kw
struct WeightT {
  const float* w;
  int Cin, KK;
  __device__ float operator()(int ci, int k2) const { return __ldg(w + ((size_t)(k2 / KK) * Cin + ci) * KK + k2 % KK); }
};
// B[k2, j] of the data gradient: dy at the output position whose window puts tap (kh, kw) on input pixel j
struct Col2imGather {
  const float* dy;
  int Cout, H, W, KH, KW, SH, SW, PH, PW, OH, OW;
  __device__ float operator()(int k2, int j) const {
    const int kw = k2 % KW, t = k2 / KW, kh = t % KH, co = t / KH;
    const int w = j % W, t2 = j / W, h = t2 % H, n = t2 / H;
    const int th = h + PH - kh, tw = w + PW - kw;
    if (th < 0 || tw < 0 || th % SH || tw % SW) return 0.f;
    const int oh = th / SH, ow = tw / SW;
    if (oh >= OH || ow >= OW) return 0.f;
    return __ldg(dy + ((size_t)(n * Cout + co) * OH + oh) * OW + ow);
  }
};
// The same two gathers over three spatial axes (a Convolution or Deconvolution over [N, C, D, H, W]).  ChanMajor and
// WeightT serve the 3-D weight and data gradients as they are, with HW = OD OH OW and KK = KD KH KW.
struct ConvGeom3 {
  int C, D, H, W, KD, KH, KW, SD, SH, SW, PD, PH, PW, OD, OH, OW;
};
// B[k, j] of the forward: k = ((ci * KD + kd) * KH + kh) * KW + kw, j = ((n * OD + od) * OH + oh) * OW + ow; zero
// padding
struct Vol2col {
  const float* x;
  ConvGeom3 g;
  __device__ float operator()(int k, int j) const {
    const int kw = k % g.KW, t = k / g.KW, kh = t % g.KH, t1 = t / g.KH, kd = t1 % g.KD, ci = t1 / g.KD;
    const int ow = j % g.OW, t2 = j / g.OW, oh = t2 % g.OH, t3 = t2 / g.OH, od = t3 % g.OD, n = t3 / g.OD;
    const int d = od * g.SD - g.PD + kd, h = oh * g.SH - g.PH + kh, w = ow * g.SW - g.PW + kw;
    if (d < 0 || d >= g.D || h < 0 || h >= g.H || w < 0 || w >= g.W) return 0.f;
    return __ldg(x + (((size_t)(n * g.C + ci) * g.D + d) * g.H + h) * g.W + w);
  }
};
// B[k2, j] of the data gradient: dy at the output position whose window puts tap (kd, kh, kw) on input voxel j =
// ((n * D + d) * H + h) * W + w, k2 = ((co * KD + kd) * KH + kh) * KW + kw; g.C is Cout, dy's channels
struct Col2volGather {
  const float* dy;
  ConvGeom3 g;
  __device__ float operator()(int k2, int j) const {
    const int kw = k2 % g.KW, t = k2 / g.KW, kh = t % g.KH, t1 = t / g.KH, kd = t1 % g.KD, co = t1 / g.KD;
    const int w = j % g.W, t2 = j / g.W, h = t2 % g.H, t3 = t2 / g.H, d = t3 % g.D, n = t3 / g.D;
    const int td = d + g.PD - kd, th = h + g.PH - kh, tw = w + g.PW - kw;
    if (td < 0 || th < 0 || tw < 0 || td % g.SD || th % g.SH || tw % g.SW) return 0.f;
    const int od = td / g.SD, oh = th / g.SH, ow = tw / g.SW;
    if (od >= g.OD || oh >= g.OH || ow >= g.OW) return 0.f;
    return __ldg(dy + (((size_t)(n * g.C + co) * g.OD + od) * g.OH + oh) * g.OW + ow);
  }
};

// ------------------------------------------------------------------ epilogues
struct StoreNCHW {  // C[m = channel, n = (img, pixel)] -> out[img, m, pixel] (+ bias[m])
  float* out;
  const float* bias;
  int C, HW;
  __device__ void operator()(int m, int n, int, float v) const {
    out[((size_t)(n / HW) * C + m) * HW + n % HW] = bias ? __fadd_rn(v, __ldg(bias + m)) : v;
  }
};
struct StoreRM {  // out[m * ld + n] (+ bias[n])
  float* out;
  const float* bias;
  int ld;
  __device__ void operator()(int m, int n, int, float v) const {
    out[(size_t)m * ld + n] = bias ? __fadd_rn(v, __ldg(bias + n)) : v;
  }
};
struct StorePartial {  // split-K partial z of C[M, N]
  float* ws;
  int M, N;
  __device__ void operator()(int m, int n, int z, float v) const { ws[((size_t)z * M + m) * N + n] = v; }
};

// ------------------------------------------------------------------ the RNN's gathers and epilogues (rnn_layer.cpp's
// unrolled net: each Caffe layer's operation rounded once, in its order)
// hc[r, c] = cont[r] * h[r, c]: the Scale layer h_conted_{t-1} = cont_t * h_{t-1}, over one step's rows or all T N
struct ContGather {
  const float* h;
  const float* cont;
  int ld;
  __device__ float operator()(int r, int c) const { return __fmul_rn(__ldg(cont + r), __ldg(h + (size_t)r * ld + c)); }
};
// h_t = tanh(fl(fl(W_hh hc_{t-1} + g_t) + z)): the Eltwise SUM in bottom order (z only with x_static), then TanH
struct RnnStep {
  const float* g;
  const float* z;
  float* h;
  int ld;
  __device__ void operator()(int m, int n, int, float v) const {
    const size_t i = (size_t)m * ld + n;
    float a = __fadd_rn(v, __ldg(g + i));
    if (z) a = __fadd_rn(a, __ldg(z + i));
    h[i] = tanhf(a);
  }
};
struct StoreTanhRM {  // out[m * ld + n] = tanh(fl(v + bias[n])): W_ho_h_t then o_neuron_t
  float* out;
  const float* bias;
  int ld;
  __device__ void operator()(int m, int n, int, float v) const {
    out[(size_t)m * ld + n] = tanhf(__fadd_rn(v, __ldg(bias + n)));
  }
};
// dho = dzo W_ho, the gradient W_ho_h_t sends to h_t.  h_{T-1} has that one reader, so on the last step's rows
// (m >= last) it is already the hidden TanH's: dpre = dho * (1 - h^2).
struct RnnOutGrad {
  float* dho;
  float* dpre;
  const float* h;
  int ld, last;
  __device__ void operator()(int m, int n, int, float v) const {
    const size_t i = (size_t)m * ld + n;
    dho[i] = v;
    if (m >= last) {
      const float t = __ldg(h + i);
      dpre[i] = __fmul_rn(v, __fsub_rn(1.f, __fmul_rn(t, t)));
    }
  }
};
// One step of backpropagation through time, v = (dpre_t W_hh)[m, n]: the Scale's backward cont_t * v, the implicit
// Split of h_{t-1} (its W_ho reader first), then h_neuron_{t-1}'s TanH: dpre_{t-1} = fl(dho_{t-1} + cont_t v) (1 - h^2)
struct RnnBackStep {
  const float* cont;  // cont_t
  const float* dho;   // these three at step t - 1
  const float* h;
  float* dpre;
  int ld;
  __device__ void operator()(int m, int n, int, float v) const {
    const size_t i = (size_t)m * ld + n;
    const float d = __fadd_rn(__ldg(dho + i), __fmul_rn(__ldg(cont + m), v));
    const float t = __ldg(h + i);
    dpre[i] = __fmul_rn(d, __fsub_rn(1.f, __fmul_rn(t, t)));
  }
};

// C = A[M, K] * B[K, N]; blockIdx.z covers k in [z * kchunk, min(K, (z + 1) * kchunk)).
template <class GA, class GB, class EPI>
__global__ void __launch_bounds__(kGemmThreads) gemm_kernel(GA ga, GB gb, EPI epi, int M, int N, int K, int kchunk) {
  __shared__ float As[kBK][kBM + 4];
  __shared__ float Bs[kBK][kBN + 4];
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const int kb = blockIdx.z * kchunk, ke = min(K, kb + kchunk);
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kb; k0 < ke; k0 += kBK) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int e = threadIdx.x + r * kGemmThreads;
      const int am = e / kBK, ak = e % kBK;
      As[ak][am] = (m0 + am < M && k0 + ak < ke) ? ga(m0 + am, k0 + ak) : 0.f;
      const int bk = e / kBN, bn = e % kBN;
      Bs[bk][bn] = (n0 + bn < N && k0 + bk < ke) ? gb(k0 + bk, n0 + bn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
      if (m < M && n < N) epi(m, n, blockIdx.z, acc[i][j]);
    }
}

template <class GA, class GB, class EPI>
cudaError_t gemm(GA ga, GB gb, EPI epi, int M, int N, int K, int kchunk, cudaStream_t s) {
  const int splits = static_cast<int>((static_cast<int64_t>(K) + kchunk - 1) / kchunk);
  dim3 grid((N + kBN - 1) / kBN, (M + kBM - 1) / kBM, splits > 0 ? splits : 1);
  gemm_kernel<<<grid, kGemmThreads, 0, s>>>(ga, gb, epi, M, N, K, kchunk);
  return cudaGetLastError();
}

// k-chunk of a weight gradient over K products: kSplitK, or larger (a multiple of kBK) when that would give more than
// kMaxSplits partials.  Fixed by the shape alone, so the reduction order never changes between calls.
int split_chunk(int K) {
  const int64_t need = (static_cast<int64_t>(K) + kMaxSplits - 1) / kMaxSplits;
  const int64_t chunk = (need + kBK - 1) / kBK * kBK;
  return static_cast<int>(std::max<int64_t>(kSplitK, chunk));
}
int splits_of(int K) { return static_cast<int>((static_cast<int64_t>(K) + split_chunk(K) - 1) / split_chunk(K)); }

// dst[i] += ws[0][i] + ws[1][i] + ... (partials added in chunk order, then once into dst)
__global__ void reduce_partials_kernel(const float* ws, int splits, int n, float* dst) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < splits; ++z) s = __fadd_rn(s, ws[(size_t)z * n + i]);
    dst[i] = __fadd_rn(dst[i], s);
  }
}

__device__ float block_sum(float v, float* sh) {  // fixed tree over kThreads threads
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + w]);
    __syncthreads();
  }
  return sh[0];
}

// dst[c] += sum over (n, p) of dy[n, c, p]: one block per channel
__global__ void __launch_bounds__(kThreads) bias_grad_kernel(const float* dy, int N, int C, int HW, float* dst) {
  __shared__ float sh[kThreads];
  const int c = blockIdx.x;
  float s = 0.f;
  for (int i = threadIdx.x; i < N * HW; i += kThreads) s = __fadd_rn(s, dy[((size_t)(i / HW) * C + c) * HW + i % HW]);
  s = block_sum(s, sh);
  if (threadIdx.x == 0) dst[c] = __fadd_rn(dst[c], s);
}

// out[i] = d[0][i] + d[1][i] + ... in step order: the implicit Split of x_static's transform, read by every step
__global__ void sum_steps_kernel(const float* d, int steps, int n, float* out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float a = d[i];
    for (int t = 1; t < steps; ++t) a = __fadd_rn(a, d[(size_t)t * n + i]);
    out[i] = a;
  }
}

__global__ void accumulate_kernel(float* dst, const float* src, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dst[i] = __fadd_rn(dst[i], src[i]);
}

// ------------------------------------------------------------------ pooling (pooling_layer.cu semantics)
struct PoolGeom {
  int N, C, H, W, PH, PW, KH, KW, SH, SW, PADH, PADW;
};

// Output (ph, pw)'s window: rows [*hs, *he) and columns [*ws, *we) of the plane, the padding clipped off
__device__ __forceinline__ void pool_window(int ph, int pw, const PoolGeom& g, int* hs, int* he, int* ws, int* we) {
  *hs = ph * g.SH - g.PADH, *ws = pw * g.SW - g.PADW;
  *he = min(*hs + g.KH, g.H), *we = min(*ws + g.KW, g.W);
  *hs = max(*hs, 0), *ws = max(*ws, 0);
}

// MAX over a window in (h, w) order from -FLT_MAX: the first value > the running maximum wins, so NaN never does, and
// *mi is -1 when no value is > -FLT_MAX
__device__ __forceinline__ float window_max(const float* plane, int W, int hs, int he, int ws, int we, int* mi) {
  float m = -FLT_MAX;
  *mi = -1;
  for (int h = hs; h < he; ++h)
    for (int w = ws; w < we; ++w)
      if (plane[h * W + w] > m) {  // the first maximum wins
        *mi = h * W + w;
        m = plane[*mi];
      }
  return m;
}

// AVE's sum over a window: row-major, one rounding per add, from +0
__device__ __forceinline__ float window_sum(const float* plane, int W, int hs, int he, int ws, int we) {
  float s = 0.f;
  for (int h = hs; h < he; ++h)
    for (int w = ws; w < we; ++w) s = __fadd_rn(s, plane[h * W + w]);
  return s;
}

__global__ void max_pool_forward_kernel(const float* x, float* y, int* idx, PoolGeom g) {
  const int total = g.N * g.C * g.PH * g.PW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int pw = i % g.PW, ph = (i / g.PW) % g.PH, nc = i / (g.PW * g.PH);
    int hs, he, ws, we;
    pool_window(ph, pw, g, &hs, &he, &ws, &we);
    int mi;
    y[i] = window_max(x + (size_t)nc * g.H * g.W, g.W, hs, he, ws, we, &mi);
    idx[i] = mi;
  }
}

// gather: every input pixel sums dy over the windows whose argmax it is, in (ph, pw) order
__global__ void max_pool_backward_kernel(const float* dy, const int* idx, float* dx, PoolGeom g) {
  const int total = g.N * g.C * g.H * g.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int w = i % g.W, h = (i / g.W) % g.H, nc = i / (g.W * g.H);
    const int phs = (h + g.PADH < g.KH) ? 0 : (h + g.PADH - g.KH) / g.SH + 1;
    const int phe = min((h + g.PADH) / g.SH + 1, g.PH);
    const int pws = (w + g.PADW < g.KW) ? 0 : (w + g.PADW - g.KW) / g.SW + 1;
    const int pwe = min((w + g.PADW) / g.SW + 1, g.PW);
    const size_t o = (size_t)nc * g.PH * g.PW;
    float s = 0.f;
    for (int ph = phs; ph < phe; ++ph)
      for (int pw = pws; pw < pwe; ++pw)
        if (idx[o + ph * g.PW + pw] == h * g.W + w) s = __fadd_rn(s, dy[o + ph * g.PW + pw]);
    dx[i] = s;
  }
}

// AVE divides by the window clipped to H + pad before it is clipped to H (pooling_layer.cpp)
__device__ __forceinline__ int ave_pool_size(int ph, int pw, const PoolGeom& g) {
  const int hs = ph * g.SH - g.PADH, ws = pw * g.SW - g.PADW;
  const int he = min(hs + g.KH, g.H + g.PADH), we = min(ws + g.KW, g.W + g.PADW);
  return (he - hs) * (we - ws);
}

__global__ void ave_pool_forward_kernel(const float* x, float* y, PoolGeom g) {
  const int total = g.N * g.C * g.PH * g.PW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int pw = i % g.PW, ph = (i / g.PW) % g.PH, nc = i / (g.PW * g.PH);
    int hs, he, ws, we;
    pool_window(ph, pw, g, &hs, &he, &ws, &we);
    y[i] = __fdiv_rn(window_sum(x + (size_t)nc * g.H * g.W, g.W, hs, he, ws, we),
                     static_cast<float>(ave_pool_size(ph, pw, g)));
  }
}

__global__ void ave_pool_backward_kernel(const float* dy, float* dx, PoolGeom g) {
  const int total = g.N * g.C * g.H * g.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int w = i % g.W + g.PADW, h = (i / g.W) % g.H + g.PADH, nc = i / (g.W * g.H);
    const int phs = (h < g.KH) ? 0 : (h - g.KH) / g.SH + 1, phe = min(h / g.SH + 1, g.PH);
    const int pws = (w < g.KW) ? 0 : (w - g.KW) / g.SW + 1, pwe = min(w / g.SW + 1, g.PW);
    const size_t o = (size_t)nc * g.PH * g.PW;
    float s = 0.f;
    for (int ph = phs; ph < phe; ++ph)
      for (int pw = pws; pw < pwe; ++pw)
        s = __fadd_rn(s, __fdiv_rn(dy[o + ph * g.PW + pw], static_cast<float>(ave_pool_size(ph, pw, g))));
    dx[i] = s;
  }
}

// ------------------------------------------------------------------ SPP (spp_layer.cpp)
// The pyramid over one [N, C, H, W] bottom: level l pools bins = 2^l windows per side with kernel kh[l] x kw[l], stride
// equal to the kernel and pad padh[l] x padw[l] (spp_level); the top holds per_sample = C * sum of 4^l values per
// sample, level l's from C * (4^l - 1) / 3 on, ordered (c, ph, pw): the Concat of each level's Flatten.
struct SppGeom {
  int N, C, H, W, levels, per_sample;
  int kh[kSppMaxLevels], kw[kSppMaxLevels], padh[kSppMaxLevels], padw[kSppMaxLevels];
};

// Level l as the Pooling layer Caffe's SPP builds for it
__device__ __forceinline__ PoolGeom spp_pool_geom(const SppGeom& g, int l) {
  return PoolGeom{g.N, g.C, g.H, g.W, 1 << l, 1 << l, g.kh[l], g.kw[l], g.kh[l], g.kw[l], g.padh[l], g.padw[l]};
}

// Forward: one thread per top element over every level, written straight to its place in the top (no Split, per-level
// buffer or Concat copy), with the pooling kernels' window arithmetic: MAX's first maximum and argmax, or AVE's
// row-major sum over the clipped window divided by ave_pool_size.
__global__ void spp_forward_kernel(const float* __restrict__ x, float* __restrict__ y, int* __restrict__ idx,
                                   SppGeom g, bool max_pool) {
  const int total = g.N * g.per_sample;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int n = i / g.per_sample;
    int r = i - n * g.per_sample, l = 0;
    while (r >= (g.C << (2 * l))) r -= g.C << (2 * l), ++l;  // level l holds C * 4^l values
    const int bins = 1 << l, pw = r % bins, ph = (r / bins) % bins, c = r / (bins * bins);
    const PoolGeom pg = spp_pool_geom(g, l);
    int hs, he, ws, we;
    pool_window(ph, pw, pg, &hs, &he, &ws, &we);
    const float* plane = x + ((size_t)n * g.C + c) * g.H * g.W;
    if (max_pool) {
      int mi;
      y[i] = window_max(plane, g.W, hs, he, ws, we, &mi);
      idx[i] = mi;
    } else {
      y[i] = __fdiv_rn(window_sum(plane, g.W, hs, he, ws, we), static_cast<float>(ave_pool_size(ph, pw, pg)));
    }
  }
}

// Backward: one thread per bottom element, each written once.  Stride equals kernel, so the element lies in one window
// per level; that level's term is what its Pooling backward writes there (0 + dy for MAX's argmax, else +0; 0 + dy /
// size for AVE), and the terms are added in level order, ((g0 + g1) + g2) + .., as Split's backward sums its tops.
__global__ void spp_backward_kernel(const float* __restrict__ dy, const int* __restrict__ idx, float* __restrict__ dx,
                                    SppGeom g, bool max_pool) {
  const int total = g.N * g.C * g.H * g.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int w = i % g.W, h = (i / g.W) % g.H, nc = i / (g.W * g.H), n = nc / g.C, c = nc - n * g.C;
    size_t level = (size_t)n * g.per_sample;  // where level l starts in the top
    float s = 0.f;
    for (int l = 0; l < g.levels; ++l) {
      const PoolGeom pg = spp_pool_geom(g, l);
      const int ph = (h + pg.PADH) / pg.KH, pw = (w + pg.PADW) / pg.KW;
      const size_t o = level + ((size_t)c * pg.PH + ph) * pg.PW + pw;
      float t = 0.f;
      if (!max_pool) t = __fadd_rn(0.f, __fdiv_rn(dy[o], static_cast<float>(ave_pool_size(ph, pw, pg))));
      else if (idx[o] == h * g.W + w) t = __fadd_rn(0.f, dy[o]);
      s = l == 0 ? t : __fadd_rn(s, t);
      level += (size_t)g.C << (2 * l);
    }
    dx[i] = s;
  }
}

// ------------------------------------------------------------------ elementwise
__global__ void relu_forward_kernel(const float* x, float* y, int n, float slope) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i];
    y[i] = v > 0.f ? v : __fmul_rn(v, slope);
  }
}
// x is the bottom's memory: the input, or the output itself for an in-place layer (as in relu_layer.cu)
__global__ void relu_backward_kernel(const float* x, const float* dy, float* dx, int n, float slope) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dx[i] = x[i] > 0.f ? dy[i] : __fmul_rn(dy[i], slope);
}
__device__ __forceinline__ float sigmoid(float x) {  // sigmoid_layer.cu
  return __fadd_rn(__fmul_rn(0.5f, tanhf(__fmul_rn(0.5f, x))), 0.5f);
}
__global__ void sigmoid_forward_kernel(const float* x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = sigmoid(x[i]);
}
__global__ void sigmoid_backward_kernel(const float* y, const float* dy, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float s = y[i];
    dx[i] = __fmul_rn(__fmul_rn(dy[i], s), __fsub_rn(1.f, s));
  }
}

// ------------------------------------------------------------------ SoftmaxWithLoss
// One block.  Row r = (o, s) of the scores x[o, c, s] (outer o, class c along the softmax axis, inner s): p = softmax
// over c, loss_r = -log(max(p[label], FLT_MIN)), dx = (p - onehot) * loss_weight / count.  Rows are summed per thread in order, then by a fixed tree, so the loss is
// reproducible; *loss = loss_weight * (sum / count).  A label outside [0, C) (or NaN) sets *status and contributes
// neither loss nor gradient; nothing outside the row is read.
__global__ void __launch_bounds__(kThreads) softmax_loss_kernel(const float* x, const float* label, float* dx,
                                                                float* loss, int rows, int C, int inner,
                                                                float loss_weight, int* status) {
  __shared__ float sh[kThreads];
  const float count = static_cast<float>(rows);
  const float scale = __fdiv_rn(loss_weight, count);
  float part = 0.f;
  for (int r = threadIdx.x; r < rows; r += kThreads) {
    const size_t base = (size_t)(r / inner) * C * inner + r % inner;
    float m = -INFINITY;
    for (int c = 0; c < C; ++c) m = fmaxf(m, x[base + (size_t)c * inner]);
    float sum = 0.f;
    for (int c = 0; c < C; ++c) sum = __fadd_rn(sum, expf(__fsub_rn(x[base + (size_t)c * inner], m)));
    const float lf = label[r];
    if (!(lf >= 0.f && lf < static_cast<float>(C))) {
      *reinterpret_cast<volatile int*>(status) = kStatusBadLabel;
      for (int c = 0; c < C; ++c) dx[base + (size_t)c * inner] = 0.f;
      continue;
    }
    const int l = static_cast<int>(lf);
    for (int c = 0; c < C; ++c) {
      const float p = __fdiv_rn(expf(__fsub_rn(x[base + (size_t)c * inner], m)), sum);
      dx[base + (size_t)c * inner] = __fmul_rn(c == l ? __fsub_rn(p, 1.f) : p, scale);
    }
    const float pl = __fdiv_rn(expf(__fsub_rn(x[base + (size_t)l * inner], m)), sum);
    part = __fsub_rn(part, logf(fmaxf(pl, FLT_MIN)));
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0) *loss = __fmul_rn(loss_weight, __fdiv_rn(part, count));
}

// ------------------------------------------------------------------ Slice and Concat (slice_layer.cu, concat_layer.cu)
// One range of a blob split along an axis: part[n, i, r] = whole[n, begin + i, r] over outer n, part_axis i and inner
// r.  Without into_whole it copies the range out of the whole (the forward of a Slice top, the backward of a Concat
// bottom); with into_whole it writes the part into its range (the backward of a Slice top, the forward of a Concat
// bottom).
__global__ void slice_copy_kernel(const float* src, float* dst, int64_t total, int64_t part_span, int64_t whole_span,
                                  int64_t offset, bool into_whole) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t b = (i / part_span) * whole_span + offset + i % part_span;
    if (into_whole) dst[b] = src[i];
    else dst[i] = src[b];
  }
}

// ------------------------------------------------------------------ Crop (crop_layer.cpp)
// The window's geometry over `rank` axes, innermost first (axis 0 is the contiguous one): the top's dims, the bottom's
// dims and the window's offset on each, in units of V (float or float4: the innermost dims and offset are divided by
// 4 for float4).  crop_geom merges an axis into the next inner one when that one is not cropped, so a crop on H and W
// of NCHW maps over three axes.
struct CropGeom {
  int rank;
  int64_t top[kCropMaxAxes], bottom[kCropMaxAxes], off[kCropMaxAxes];
};

// q = n / d and n - q d, with 32-bit arithmetic when both fit (every index of a blob under 2^32 elements)
__device__ __forceinline__ int64_t crop_divmod(int64_t n, int64_t d, int64_t* r) {
  if (((n | d) >> 32) == 0) {
    const uint32_t q = static_cast<uint32_t>(n) / static_cast<uint32_t>(d);
    *r = static_cast<uint32_t>(n) - q * static_cast<uint32_t>(d);
    return q;
  }
  const int64_t q = n / d;
  *r = n - q * d;
  return q;
}

// Forward: one thread per element (or float4) of the top, consecutive threads on consecutive innermost elements:
// y[i] = x[the bottom index of i's coordinates plus the offsets].  A copy: every bit of x arrives in y.
template <class V>
__global__ void crop_forward_kernel(const V* __restrict__ x, V* __restrict__ y, int64_t total, CropGeom g) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t rest = i, src = 0, stride = 1;
    for (int a = 0; a < g.rank; ++a) {
      int64_t c = rest;
      if (a + 1 < g.rank) rest = crop_divmod(rest, g.top[a], &c);
      src += (c + g.off[a]) * stride;
      stride *= g.bottom[a];
    }
    y[i] = x[src];
  }
}

// Backward: one thread per element (or float4) of the bottom, each written once: dy at the mapped top index inside
// the window, +0 outside it.  No memset, no scatter, no atomics.
template <class V>
__global__ void crop_backward_kernel(const V* __restrict__ dy, V* __restrict__ dx, int64_t total, CropGeom g) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t rest = i, src = 0, stride = 1;
    bool inside = true;
    for (int a = 0; a < g.rank; ++a) {
      int64_t c = rest;
      if (a + 1 < g.rank) rest = crop_divmod(rest, g.bottom[a], &c);
      const int64_t t = c - g.off[a];
      inside = inside && t >= 0 && t < g.top[a];
      src += t * stride;
      stride *= g.top[a];
    }
    dx[i] = inside ? dy[src] : V{};  // V{}: +0 in every lane
  }
}

// ------------------------------------------------------------------ Tile (tile_layer.cpp)
// The top is [outer, tiles, inner] over the bottom's [outer, inner]; every index is below 2^31 (tile_forward checks the
// top's count), so the kernels index in 32 bits.

// Forward: thread k writes top elements [V k, V k + V), as one 128-bit store for V = 4.  With kVecLoad (inner a multiple
// of 4, x 16-byte aligned) the V elements lie in one row of x and are read as one float4; otherwise each is read on its
// own, walking (o, t, d) from the first.  A copy: every bit of x arrives in y.
template <int V, bool kVecLoad>
__global__ void tile_forward_kernel(const float* __restrict__ x, float* __restrict__ y, int n, int inner, int tiles,
                                    FastDiv fd_inner, FastDiv fd_tiles) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const unsigned j = static_cast<unsigned>(k) * V;
  const unsigned q = fd_inner.div(j);  // the top's row (o, t)
  const unsigned o = fd_tiles.div(q);
  unsigned d = j - q * inner, t = q - o * tiles, src = o * inner + d;
  if constexpr (V == 1) {
    y[j] = x[src];
  } else if constexpr (kVecLoad) {
    *reinterpret_cast<float4*>(y + j) = *reinterpret_cast<const float4*>(x + src);
  } else {
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[e] = x[src];
      ++src;
      if (++d == static_cast<unsigned>(inner)) {  // the next row: the same bottom row again, or the next one after
        d = 0;                                   // the last tile
        if (++t == static_cast<unsigned>(tiles)) t = 0;
        else src -= inner;
      }
    }
    *reinterpret_cast<float4*>(y + j) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// Backward for inner >= kTileStagedMaxInner: one thread per dx element (o, d), consecutive threads on consecutive d, so
// every load of a tile row is coalesced.  dx = dy[o, 0, d], then dy[o, t, d] added in t order.
__global__ void tile_backward_direct_kernel(const float* __restrict__ dy, float* __restrict__ dx, int n, int inner,
                                            int tiles) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int o = i / inner;
  const float* p = dy + static_cast<int64_t>(o) * tiles * inner + (i - o * inner);
  float acc = p[0];
#pragma unroll 8
  for (int t = 1; t < tiles; ++t) acc = __fadd_rn(acc, p[static_cast<int64_t>(t) * inner]);
  dx[i] = acc;
}

// Backward for inner < kTileStagedMaxInner: a block owns `rows` consecutive outer rows, rows * inner <= blockDim.x
// outputs, and walks the tiles in chunks of kTileChunk.  The block copies its rows' part of the chunk (each row's part
// contiguous in dy) into shared memory, consecutive threads on consecutive floats, as stage[t][k] for output k = r *
// inner + d, at a row stride `stride` congruent to inner mod 32: neither the stores (consecutive t * inner + d) nor the
// column reads (consecutive k) meet a bank conflict.  Thread k then adds its column in t order: the first tile copied,
// each later one added.  fd_span and fd_last divide by a full chunk's row length (kTileChunk * inner) and the last's.
constexpr int kTileChunk = 32;
constexpr int kTileStageStride = kThreads + 32;  // the largest `stride` tile_backward picks
__global__ void __launch_bounds__(kThreads) tile_backward_staged_kernel(const float* __restrict__ dy,
                                                                        float* __restrict__ dx, int outer, int inner,
                                                                        int tiles, int rows, int stride,
                                                                        FastDiv fd_inner, FastDiv fd_span,
                                                                        FastDiv fd_last) {
  __shared__ float stage[kTileChunk * kTileStageStride];
  const int o0 = blockIdx.x * rows;
  const int nrows = min(rows, outer - o0), outputs = nrows * inner;
  const float* base = dy + static_cast<int64_t>(o0) * tiles * inner;
  float acc = 0.f;
  for (int t0 = 0; t0 < tiles; t0 += kTileChunk) {
    const int tc = min(kTileChunk, tiles - t0), span = tc * inner;
    const FastDiv& fd = tc == kTileChunk ? fd_span : fd_last;
    __syncthreads();  // the previous chunk's columns are read
#pragma unroll 4
    for (int e = threadIdx.x; e < nrows * span; e += blockDim.x) {
      const int r = fd.div(e), c = e - r * span;
      const int t = fd_inner.div(c), d = c - t * inner;
      stage[t * stride + r * inner + d] = base[(static_cast<int64_t>(r) * tiles + t0) * inner + c];
    }
    __syncthreads();
    if (static_cast<int>(threadIdx.x) < outputs) {
      const float* col = stage + threadIdx.x;
      int t = 0;
      if (t0 == 0) acc = col[0], t = 1;
      for (; t < tc; ++t) acc = __fadd_rn(acc, col[t * stride]);
    }
  }
  if (static_cast<int>(threadIdx.x) < outputs) dx[static_cast<int64_t>(o0) * inner + threadIdx.x] = acc;
}

// ------------------------------------------------------------------ ContrastiveLoss (contrastive_loss_layer.cpp)
// One block.  Pair r: d = a_r - b_r, dist_sq = sum over c of d_c^2 in c order.  A similar pair (static_cast<int>(sim)
// nonzero) adds dist_sq to the loss and gets da = alpha * d.  A dissimilar pair adds max(margin - dist_sq, 0)
// (legacy_version) or max(margin - dist, 0)^2, and gets da = beta * d while mdist = margin - dist_sq (legacy) or
// margin - dist is > 0, else an exact 0, with beta = -alpha (legacy) or -alpha * mdist / (dist + 1e-4).  alpha =
// loss_weight / N and db = -da.  As in Caffe, a NaN in d makes a dissimilar pair's loss NaN and its gradient 0.  Pairs
// are summed per thread in order, then by a fixed tree; *loss = loss_weight * (sum / N / 2).  A non-finite sim sets
// *status and its pair contributes neither loss nor gradient.  da / db are null for a staged bottom.
// Made for the narrow embeddings of siamese nets (C of a few to a few dozen: each thread walks its pairs' C channels
// twice).  For wide embeddings and few pairs most threads idle and the row loads are not coalesced.
__global__ void __launch_bounds__(kThreads) contrastive_loss_kernel(const float* a, const float* b, const float* sim,
                                                                    float* da, float* db, float* loss, int N, int C,
                                                                    float margin, bool legacy, float loss_weight,
                                                                    int* status) {
  __shared__ float sh[kThreads];
  const float alpha = __fdiv_rn(loss_weight, static_cast<float>(N));
  float part = 0.f;
  for (int r = threadIdx.x; r < N; r += kThreads) {
    const float* ar = a + (size_t)r * C;
    const float* br = b + (size_t)r * C;
    float dist_sq = 0.f;
    for (int c = 0; c < C; ++c) {
      const float d = __fsub_rn(ar[c], br[c]);
      dist_sq = __fadd_rn(dist_sq, __fmul_rn(d, d));
    }
    const float s = sim[r];
    float scale = 0.f;  // gradient of a = scale * d
    bool zero = true;   // gradient an exact 0 (caffe_set), not 0 * d: a NaN or infinite d stays out of it
    if (!isfinite(s)) {
      *reinterpret_cast<volatile int*>(status) = kStatusBadLabel;
    } else if (static_cast<int>(s)) {
      part = __fadd_rn(part, dist_sq);
      scale = alpha, zero = false;
    } else if (legacy) {
      // std::max(mdist, 0) returns its first argument unless mdist < 0: a NaN mdist reaches the loss
      const float mdist = __fsub_rn(margin, dist_sq);
      part = __fadd_rn(part, mdist < 0.f ? 0.f : mdist);
      if (mdist > 0.f) scale = -alpha, zero = false;
    } else {
      const float dist = __fsqrt_rn(dist_sq);
      const float mdist = __fsub_rn(margin, dist);
      const float m = mdist < 0.f ? 0.f : mdist;
      part = __fadd_rn(part, __fmul_rn(m, m));
      if (mdist > 0.f) scale = __fdiv_rn(__fmul_rn(-alpha, mdist), __fadd_rn(dist, 1e-4f)), zero = false;
    }
    for (int c = 0; c < C; ++c) {
      const float g = zero ? 0.f : __fmul_rn(scale, __fsub_rn(ar[c], br[c]));
      if (da) da[(size_t)r * C + c] = g;
      if (db) db[(size_t)r * C + c] = zero ? 0.f : -g;
    }
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0)
    *loss = __fmul_rn(loss_weight, __fdiv_rn(__fdiv_rn(part, static_cast<float>(N)), 2.f));
}

// ------------------------------------------------------------------ EuclideanLoss (euclidean_loss_layer.cpp)
// One block.  d = a - b over the `count` elements of each bottom; each thread sums d^2 over its elements in index order,
// then a fixed tree adds the threads: *loss = loss_weight * (dot / num / 2), each operation rounded once in float as
// Caffe computes it.  The gradients are alpha * d with alpha = loss_weight / num into a and -loss_weight / num into b,
// one rounding each; da / db are null for a bottom that wants none.  A NaN reaches the loss, as in Caffe.  Made for
// regression targets of a few values per row: on large blobs one block leaves most of the GPU idle.
__global__ void __launch_bounds__(kThreads) euclidean_loss_kernel(const float* a, const float* b, float* da, float* db,
                                                                  float* loss, int count, int num, float loss_weight) {
  __shared__ float sh[kThreads];
  const float alpha = __fdiv_rn(loss_weight, static_cast<float>(num));
  float part = 0.f;
  for (int i = threadIdx.x; i < count; i += kThreads) {
    const float d = __fsub_rn(a[i], b[i]);
    part = __fadd_rn(part, __fmul_rn(d, d));
    if (da) da[i] = __fmul_rn(alpha, d);
    if (db) db[i] = __fmul_rn(-alpha, d);
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0)
    *loss = __fmul_rn(loss_weight, __fdiv_rn(__fdiv_rn(part, static_cast<float>(num)), 2.f));
}

// ------------------------------------------------------------------ SigmoidCrossEntropyLoss
// (sigmoid_cross_entropy_loss_layer.cpp) Element i of the `count` scores x and targets t costs -(x * (t - [x >= 0]) -
// log(1 + exp(x - 2 * x * [x >= 0]))), Caffe's stable form, each operation rounded once in float.  Each block sums its
// threads' elements (each thread in index order, then a fixed tree) into partial[blockIdx.x]; the grid is grid_for(count),
// so the partials depend on the shape alone.  dx = (sigmoid(x) - t) * (loss_weight / num), one rounding each, with the
// Sigmoid op's sigmoid; null when the scores want no gradient.  A NaN or infinite x or t reaches the loss, as in Caffe.
__global__ void __launch_bounds__(kThreads) sigmoid_xent_loss_kernel(const float* x, const float* t, float* dx,
                                                                     float* partial, int count, int num,
                                                                     float loss_weight) {
  __shared__ float sh[kThreads];
  const float scale = __fdiv_rn(loss_weight, static_cast<float>(num));
  float part = 0.f;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < count; i += gridDim.x * kThreads) {
    const float v = x[i], target = t[i];
    const float pos = v >= 0.f ? 1.f : 0.f;
    const float e = logf(__fadd_rn(1.f, expf(__fsub_rn(v, __fmul_rn(__fmul_rn(2.f, v), pos)))));
    part = __fsub_rn(part, __fsub_rn(__fmul_rn(v, __fsub_rn(target, pos)), e));
    if (dx) dx[i] = __fmul_rn(__fsub_rn(sigmoid(v), target), scale);
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = part;
}
// *loss = loss_weight * (sum / num), the partials added in block order (also HingeLoss's)
__global__ void sigmoid_xent_loss_total_kernel(const float* partial, int blocks, int num, float loss_weight,
                                               float* loss) {
  float sum = 0.f;
  for (int b = 0; b < blocks; ++b) sum = __fadd_rn(sum, partial[b]);
  *loss = __fmul_rn(loss_weight, __fdiv_rn(sum, static_cast<float>(num)));
}

// ------------------------------------------------------------------ Split, Eltwise (split_layer.cpp, eltwise_layer.cpp)
// dst = a + b: the Split backward's first two read tops (later ones go through accumulate_kernel, in top order)
__global__ void add_kernel(const float* a, const float* b, float* dst, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = __fadd_rn(a[i], b[i]);
}
// SUM, one bottom at a time in bottom order: y = c * x for the first (caffe_set(0) + axpy), then y = fma(c, x, y)
__global__ void eltwise_axpy_kernel(const float* x, float c, float* y, int n, bool first) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    y[i] = first ? __fmul_rn(c, x[i]) : __fmaf_rn(c, x[i], y[i]);
}
// dst = c * src: SUM's backward for a coefficient other than 1
__global__ void scale_copy_kernel(const float* src, float c, float* dst, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = __fmul_rn(c, src[i]);
}
// dst = a * b: PROD's forward (y = b0 * b1, then y = y * b_i) and the stable backward's running product
__global__ void mul_kernel(const float* a, const float* b, float* dst, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = __fmul_rn(a[i], b[i]);
}
// PROD's backward without stable_prod_grad: dx = (y / x) * dy, two roundings (caffe_div, then caffe_mul)
__global__ void prod_div_backward_kernel(const float* y, const float* x, const float* dy, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dx[i] = __fmul_rn(__fdiv_rn(y[i], x[i]), dy[i]);
}
// MAX, one bottom at a time (eltwise_layer.cpp Forward_cpu).  The first call (a non-null) compares bottoms 0 and 1:
// bottom 0 wins only when strictly greater.  Every later bottom b takes over only when strictly greater than y.
__global__ void eltwise_max_kernel(const float* a, const float* b, int b_index, float* y, int* idx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = b[i];
    if (a) {
      const float u = a[i];
      y[i] = u > v ? u : v;
      idx[i] = u > v ? 0 : 1;
    } else if (v > y[i]) {
      y[i] = v;
      idx[i] = b_index;
    }
  }
}
// dx = dy where bottom `which` won, else 0
__global__ void eltwise_max_backward_kernel(const float* dy, const int* idx, int which, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dx[i] = idx[i] == which ? dy[i] : 0.f;
}

// ------------------------------------------------------------------ Scale (scale_layer.cu)
// y[o, d, i] = x[o, d, i] * s[d] (+ b[d], one fused rounding); also the data gradient dx = dy * s with b null
__global__ void scale_forward_kernel(const float* x, const float* s, const float* b, float* y, int n, int dim,
                                     int inner) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int d = (i / inner) % dim;
    y[i] = b ? __fmaf_rn(x[i], __ldg(s + d), __ldg(b + d)) : __fmul_rn(x[i], __ldg(s + d));
  }
}
// dst[d] += sum over (o, i) of dy[o, d, i] * x[o, d, i]: one block per scale element, each thread's products summed
// in index order, then a fixed tree (bias_grad_kernel's order, with the product fused into each addition)
__global__ void __launch_bounds__(kThreads) scale_grad_kernel(const float* dy, const float* x, int outer, int dim,
                                                              int inner, float* dst) {
  __shared__ float sh[kThreads];
  const int d = blockIdx.x;
  float s = 0.f;
  for (int i = threadIdx.x; i < outer * inner; i += kThreads) {
    const size_t j = ((size_t)(i / inner) * dim + d) * inner + i % inner;
    s = __fmaf_rn(dy[j], x[j], s);
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) dst[d] = __fadd_rn(dst[d], s);
}

// ------------------------------------------------------------------ the other neuron layers
// (tanh_layer.cu, elu_layer.cu, absval_layer.cu, bnll_layer.cu, power_layer.cpp, exp_layer.cpp, log_layer.cpp,
// threshold_layer.cu): Caffe's formulas, each operation rounded once in float.  x is the bottom's activation, y the
// top's; the top has storage of its own, so x is the bottom as it was even when the layer is written in place.
__global__ void tanh_forward_kernel(const float* x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = tanhf(x[i]);
}
__global__ void tanh_backward_kernel(const float* y, const float* dy, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float t = y[i];
    dx[i] = __fmul_rn(dy[i], __fsub_rn(1.f, __fmul_rn(t, t)));
  }
}
__global__ void elu_forward_kernel(const float* x, float* y, int n, float alpha) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i];
    y[i] = v > 0.f ? v : __fmul_rn(alpha, __fsub_rn(expf(v), 1.f));
  }
}
__global__ void elu_backward_kernel(const float* x, const float* y, const float* dy, float* dx, int n, float alpha) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dx[i] = x[i] > 0.f ? dy[i] : __fmul_rn(dy[i], __fadd_rn(y[i], alpha));
}
__global__ void absval_forward_kernel(const float* x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = fabsf(x[i]);
}
// dx = dy * sign(x), caffe_gpu_sign's sign: 0 for a zero (and a NaN)
__global__ void absval_backward_kernel(const float* x, const float* dy, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i];
    dx[i] = __fmul_rn(dy[i], static_cast<float>((0.f < v) - (v < 0.f)));
  }
}
constexpr float kBnllThreshold = 50.f;  // bnll_layer.cu kBNLL_THRESHOLD
__global__ void bnll_forward_kernel(const float* x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i];
    y[i] = v > 0.f ? __fadd_rn(v, logf(__fadd_rn(1.f, expf(-v)))) : logf(__fadd_rn(1.f, expf(v)));
  }
}
__global__ void bnll_backward_kernel(const float* x, const float* dy, float* dx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float e = expf(fminf(x[i], kBnllThreshold));  // CUDA's min: a NaN x takes the threshold, as in bnll_layer.cu
    dx[i] = __fdiv_rn(__fmul_rn(dy[i], e), __fadd_rn(e, 1.f));
  }
}
// Power, Exp and Log transform their input as Caffe's scal and add_scalar calls do: a factor of 1 or a shift of 0 is
// skipped (so a -0 stays -0)
__device__ __forceinline__ float scale_shift(float v, float scale, float shift) {
  if (scale != 1.f) v = __fmul_rn(scale, v);
  if (shift != 0.f) v = __fadd_rn(v, shift);
  return v;
}
// y = (shift + scale * x)^power; `constant` (power * scale == 0) writes power == 0 ? 1 : shift^power everywhere
__global__ void power_forward_kernel(const float* x, float* y, int n, float power, float scale, float shift,
                                     bool constant, float value) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (constant) {
      y[i] = value;
      continue;
    }
    const float v = scale_shift(x[i], scale, shift);
    y[i] = power != 1.f ? powf(v, power) : v;
  }
}
// power_layer.cpp Backward_cpu's four branches with diff_scale = power * scale: the constant diff_scale (power 1, or
// diff_scale 0, which is not multiplied by dy); power 2: diff_scale * scale * x (+ diff_scale * shift); shift 0:
// power * y / x (NaN at x = 0, as in Caffe); else diff_scale * y / (shift + scale * x).  Then times dy.
__global__ void power_backward_kernel(const float* x, const float* y, const float* dy, float* dx, int n, float power,
                                      float scale, float shift, float diff_scale, float ds_scale, float ds_shift) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float g;
    if (diff_scale == 0.f || power == 1.f) {
      g = diff_scale;
    } else if (power == 2.f) {
      g = __fmul_rn(ds_scale, x[i]);
      if (shift != 0.f) g = __fadd_rn(g, ds_shift);
    } else if (shift == 0.f) {
      g = __fmul_rn(__fdiv_rn(y[i], x[i]), power);
    } else {
      g = __fdiv_rn(y[i], scale_shift(x[i], scale, shift));
      if (diff_scale != 1.f) g = __fmul_rn(diff_scale, g);
    }
    dx[i] = diff_scale != 0.f ? __fmul_rn(dy[i], g) : g;
  }
}
// y = outer * exp(inner * x), each factor of 1 skipped; dx = inner * (y * dy)
__global__ void exp_forward_kernel(const float* x, float* y, int n, float inner, float outer) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float v = expf(inner != 1.f ? __fmul_rn(inner, x[i]) : x[i]);
    y[i] = outer != 1.f ? __fmul_rn(outer, v) : v;
  }
}
__global__ void exp_backward_kernel(const float* y, const float* dy, float* dx, int n, float inner) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float g = __fmul_rn(y[i], dy[i]);
    dx[i] = inner != 1.f ? __fmul_rn(inner, g) : g;
  }
}
// y = base_scale * log(shift + scale * x); dx = dy * (backward_num_scale * (shift + scale * x)^-1), the power -1 a
// correctly rounded reciprocal
__global__ void log_forward_kernel(const float* x, float* y, int n, float scale, float shift, float base_scale) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = logf(scale_shift(x[i], scale, shift));
    y[i] = base_scale != 1.f ? __fmul_rn(base_scale, v) : v;
  }
}
__global__ void log_backward_kernel(const float* x, const float* dy, float* dx, int n, float scale, float shift,
                                    float num_scale) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float g = __frcp_rn(scale_shift(x[i], scale, shift));
    if (num_scale != 1.f) g = __fmul_rn(num_scale, g);
    dx[i] = __fmul_rn(dy[i], g);
  }
}
__global__ void threshold_forward_kernel(const float* x, float* y, int n, float threshold) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    y[i] = x[i] > threshold ? 1.f : 0.f;
}

// ------------------------------------------------------------------ PReLU (prelu_layer.cpp)
// Channel c of element i is (i / dim) % C, or 0 with channel_shared.  y = max(x, 0) + a_c * min(x, 0), with std::max
// and std::min's rules for zeros and NaN; dx = dy * ((x > 0) + a_c * (x <= 0)).
__global__ void prelu_forward_kernel(const float* x, const float* slope, float* y, int n, int C, int dim, bool shared) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i], a = __ldg(slope + (shared ? 0 : (i / dim) % C));
    const float hi = v < 0.f ? 0.f : v, lo = 0.f < v ? 0.f : v;
    y[i] = __fadd_rn(hi, __fmul_rn(a, lo));
  }
}
__global__ void prelu_backward_kernel(const float* x, const float* slope, const float* dy, float* dx, int n, int C,
                                      int dim, bool shared) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i], a = __ldg(slope + (shared ? 0 : (i / dim) % C));
    const float pos = v > 0.f ? 1.f : 0.f, neg = v <= 0.f ? 1.f : 0.f;
    dx[i] = __fmul_rn(dy[i], __fadd_rn(pos, __fmul_rn(a, neg)));
  }
}
// The slope gradient sums dy * x * (x <= 0) over the M = N * dim elements of each channel (M = count with
// channel_shared) in fixed chunks of kPreluChunk: block (k, c) sums chunk k of channel c (each thread in index order,
// then block_sum's tree) into partial[c * chunks + k], and prelu_slope_total_kernel adds the partials in chunk order,
// then once into the gradient.  The order depends on the shape alone; no atomics.  The grid is (chunks, slopes):
// build_plan refuses more than kMaxPReLUChannels slopes, gridDim.y's limit.
constexpr int kPreluChunk = 8192;
__global__ void __launch_bounds__(kThreads) prelu_slope_partial_kernel(const float* x, const float* dy, float* partial,
                                                                       int M, int C, int dim, bool shared,
                                                                       int chunks) {
  __shared__ float sh[kThreads];
  const int c = blockIdx.y, k = blockIdx.x;
  const int end = min(M, (k + 1) * kPreluChunk);
  float s = 0.f;
  for (int j = k * kPreluChunk + threadIdx.x; j < end; j += kThreads) {
    const size_t i = shared ? static_cast<size_t>(j) : ((size_t)(j / dim) * C + c) * dim + j % dim;
    const float v = x[i];
    s = __fadd_rn(s, __fmul_rn(__fmul_rn(dy[i], v), v <= 0.f ? 1.f : 0.f));
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) partial[(size_t)c * chunks + k] = s;
}
__global__ void prelu_slope_total_kernel(const float* partial, int chunks, int slopes, float* dst) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < slopes; c += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < chunks; ++k) s = __fadd_rn(s, partial[(size_t)c * chunks + k]);
    dst[c] = __fadd_rn(dst[c], s);
  }
}

// ------------------------------------------------------------------ Softmax (softmax_layer.cu)
// Row r = (o, s) of x[o, c, s] (outer o, class c along the axis, inner s): max over c (from -FLT_MAX, CUDA's max),
// y = exp(x - max), their sum in c order, y / sum.  One thread per row, looping over the classes: made for
// classification heads; a wide axis over few rows leaves most of the GPU idle.
__global__ void softmax_forward_kernel(const float* x, float* y, int rows, int C, int inner) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const size_t base = (size_t)(r / inner) * C * inner + r % inner;
    float m = -FLT_MAX;
    for (int c = 0; c < C; ++c) m = fmaxf(x[base + (size_t)c * inner], m);
    float sum = 0.f;
    for (int c = 0; c < C; ++c) {
      const float e = expf(__fsub_rn(x[base + (size_t)c * inner], m));
      y[base + (size_t)c * inner] = e;
      sum = __fadd_rn(sum, e);
    }
    for (int c = 0; c < C; ++c) y[base + (size_t)c * inner] = __fdiv_rn(y[base + (size_t)c * inner], sum);
  }
}
// dx = (dy - sum over c of dy * y) * y, the dot in c order
__global__ void softmax_backward_kernel(const float* y, const float* dy, float* dx, int rows, int C, int inner) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const size_t base = (size_t)(r / inner) * C * inner + r % inner;
    float dot = 0.f;
    for (int c = 0; c < C; ++c) dot = __fadd_rn(dot, __fmul_rn(dy[base + (size_t)c * inner], y[base + (size_t)c * inner]));
    for (int c = 0; c < C; ++c) {
      const size_t i = base + (size_t)c * inner;
      dx[i] = __fmul_rn(__fsub_rn(dy[i], dot), y[i]);
    }
  }
}

// ------------------------------------------------------------------ MultinomialLogisticLoss
// (multinomial_logistic_loss_layer.cpp) One block over the num rows of x [num, dim]: p = max(x[r, label_r], 1e-20),
// the loss sums -log(p) (each thread over its rows in order, then a fixed tree) and *loss = loss_weight * (sum / num).
// dx (null when not wanted) is (-loss_weight / num) / p at the label and an exact 0 elsewhere, written whole.  A label
// outside [0, dim) (or NaN) sets *status; its row adds no loss and gets a zero gradient.  Made for classification
// heads of a few to a few thousand classes.
constexpr float kLogThreshold = 1e-20f;  // loss_layer.hpp kLOG_THRESHOLD
__global__ void __launch_bounds__(kThreads) mll_loss_kernel(const float* x, const float* label, float* dx, float* loss,
                                                            int num, int dim, float loss_weight, int* status) {
  __shared__ float sh[kThreads];
  const float scale = __fdiv_rn(-loss_weight, static_cast<float>(num));
  float part = 0.f;
  for (int r = threadIdx.x; r < num; r += kThreads) {
    const float lf = label[r];
    const bool bad = !(lf >= 0.f && lf < static_cast<float>(dim));
    if (bad) *reinterpret_cast<volatile int*>(status) = kStatusBadMultinomialLabel;
    const int l = bad ? -1 : static_cast<int>(lf);
    float p = 0.f;
    if (!bad) {
      p = x[(size_t)r * dim + l];
      p = p < kLogThreshold ? kLogThreshold : p;  // std::max(p, threshold): a NaN p stays
      part = __fsub_rn(part, logf(p));
    }
    if (dx)
      for (int j = 0; j < dim; ++j) dx[(size_t)r * dim + j] = j == l ? __fdiv_rn(scale, p) : 0.f;
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0) *loss = __fmul_rn(loss_weight, __fdiv_rn(part, static_cast<float>(num)));
}

// ------------------------------------------------------------------ HingeLoss (hinge_loss_layer.cpp)
// Element (r, j) of x [num, dim]: v = x, negated at j = label_r; h = std::max(0, 1 + v) (a NaN gives 0).  The loss sums
// h (L1) or h * h (L2): each block over its threads' elements in index order, then a fixed tree, into
// partial[blockIdx.x] (the grid is grid_for(count)); sigmoid_xent_loss_total_kernel adds the partials in block order.
// dx (null when not wanted) is g = +-h (negated at the label) times: sign(g) * (loss_weight / num) for L1, with
// sign(0) = 0; g * (loss_weight * 2 / num) for L2.  A bad label sets *status; its row adds no loss and a zero gradient.
__global__ void __launch_bounds__(kThreads) hinge_loss_kernel(const float* x, const float* label, float* dx,
                                                              float* partial, int count, int dim, int num, bool l2,
                                                              float loss_weight, int* status) {
  __shared__ float sh[kThreads];
  const float s1 = __fdiv_rn(loss_weight, static_cast<float>(num));
  const float s2 = __fdiv_rn(__fmul_rn(loss_weight, 2.f), static_cast<float>(num));
  float part = 0.f;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < count; i += gridDim.x * kThreads) {
    const float lf = label[i / dim];
    if (!(lf >= 0.f && lf < static_cast<float>(dim))) {
      *reinterpret_cast<volatile int*>(status) = kStatusBadHingeLabel;
      if (dx) dx[i] = 0.f;
      continue;
    }
    const bool at = i % dim == static_cast<int>(lf);
    const float t = __fadd_rn(1.f, at ? -x[i] : x[i]);
    const float h = 0.f < t ? t : 0.f;
    part = __fadd_rn(part, l2 ? __fmul_rn(h, h) : h);
    if (!dx) continue;
    const float g = at ? -h : h;
    dx[i] = l2 ? __fmul_rn(g, s2) : __fmul_rn(static_cast<float>((0.f < g) - (g < 0.f)), s1);
  }
  part = block_sum(part, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = part;
}

// ------------------------------------------------------------------ Embed (embed_layer.cpp semantics)
constexpr int kEmbedBlock = 1024;  // the one block of the offsets' scan and of the stable placement

// The table row of an id, or -1 when the id is not an integer in [0, K) (negative, too large, fractional, NaN, inf).
// K <= 2^24, so every integer below it is exact in fp32.
__device__ __forceinline__ int embed_row(float id, int K) {
  return id >= 0.f && id < static_cast<float>(K) && id == truncf(id) ? static_cast<int>(id) : -1;
}

// y[m, :] = w[id_m, :] (+ b, one rounding), or b (0 without a bias) for an invalid id, which sets *status.  Each thread
// copies V consecutive floats of one row (V = 4: float4, when the row length and the pointers allow), so a warp reads
// and writes contiguous memory.
template <int V>
__global__ void embed_forward_kernel(const float* ids, const float* w, const float* b, float* y, int M, int N, int K,
                                     int* status) {
  typedef typename std::conditional<V == 4, float4, float>::type Vec;
  const int nv = N / V;
  const int64_t total = static_cast<int64_t>(M) * nv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / nv), c = static_cast<int>(i % nv) * V;
    const int k = embed_row(__ldg(ids + m), K);
    if (k < 0 && c == 0) *reinterpret_cast<volatile int*>(status) = kStatusBadEmbedIndex;
    Vec v;
    if (k >= 0) {
      v = __ldg(reinterpret_cast<const Vec*>(w + static_cast<size_t>(k) * N + c));
    } else {
      float* f = reinterpret_cast<float*>(&v);
      for (int j = 0; j < V; ++j) f[j] = 0.f;
    }
    if (b) {
      const Vec bv = __ldg(reinterpret_cast<const Vec*>(b + c));
      float* f = reinterpret_cast<float*>(&v);
      const float* g = reinterpret_cast<const float*>(&bv);
      for (int j = 0; j < V; ++j) f[j] = __fadd_rn(f[j], g[j]);
    }
    *reinterpret_cast<Vec*>(y + static_cast<size_t>(m) * N + c) = v;
  }
}

// count[k] = occurrences of row k among the M ids (integer atomics: the counts do not depend on their order)
__global__ void embed_count_kernel(const float* ids, int M, int K, int* count) {
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < M; m += gridDim.x * blockDim.x) {
    const int k = embed_row(__ldg(ids + m), K);
    if (k >= 0) atomicAdd(count + k, 1);
  }
}

// a[0 .. n) becomes its exclusive prefix sum: each thread scans a contiguous range, offset by the block's scan of the
// range totals
__global__ void __launch_bounds__(kEmbedBlock) exclusive_scan_kernel(int* a, int n) {
  __shared__ int sh[kEmbedBlock];
  const int per = (n + kEmbedBlock - 1) / kEmbedBlock;
  const int lo = min(n, static_cast<int>(threadIdx.x) * per), hi = min(n, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += a[i];
  sh[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < kEmbedBlock; off <<= 1) {
    const int v = threadIdx.x >= off ? sh[threadIdx.x - off] : 0;
    __syncthreads();
    sh[threadIdx.x] += v;
    __syncthreads();
  }
  int run = sh[threadIdx.x] - sum;
  for (int i = lo; i < hi; ++i) {
    const int v = a[i];
    a[i] = run;
    run += v;
  }
}

// Stable placement: order[cursor[k] ..] receives the positions m of row k in increasing m.  One block walks the ids in
// chunks of kEmbedBlock; a position's slot is its row's cursor plus the number of earlier positions of that row in the
// chunk, and the row's last position in the chunk advances the cursor.  On return cursor[k] is the end of k's group.
__global__ void __launch_bounds__(kEmbedBlock) embed_place_kernel(const float* ids, int M, int K, int* cursor,
                                                                  int* order) {
  __shared__ int key[kEmbedBlock];
  for (int base = 0; base < M; base += kEmbedBlock) {
    const int m = base + static_cast<int>(threadIdx.x);
    const int k = m < M ? embed_row(__ldg(ids + m), K) : -1;
    key[threadIdx.x] = k;
    __syncthreads();
    int rank = 0;
    bool last = true;
    if (k >= 0) {
      for (int j = 0; j < kEmbedBlock; ++j) {
        if (key[j] != k) continue;
        if (j < static_cast<int>(threadIdx.x)) ++rank;
        else if (j > static_cast<int>(threadIdx.x)) last = false;
      }
    }
    const int slot = k >= 0 ? cursor[k] + rank : 0;
    __syncthreads();  // every cursor read of this chunk before its updates
    if (k >= 0) {
      order[slot] = m;
      if (last) cursor[k] = slot + 1;
    }
    __syncthreads();  // the updates, and key[], before the next chunk
  }
}

// dw[k, :] += the dy rows of k's positions, added one at a time in increasing m onto the value already in dw
// (embed_layer.cpp Backward_cpu's order).  end[k] is the end of k's group in order[], end[K] the number of valid ids;
// the block at a group's first slot walks the group.
__global__ void embed_weight_grad_kernel(const float* ids, const int* order, const int* end, const float* dy,
                                         float* dw, int N, int K) {
  const int valid = end[K];
  for (int j = blockIdx.x; j < valid; j += gridDim.x) {
    const int k = static_cast<int>(__ldg(ids + order[j]));
    if (j != (k ? end[k - 1] : 0)) continue;
    const int stop = end[k];
    for (int d = threadIdx.x; d < N; d += blockDim.x) {
      float* p = dw + static_cast<size_t>(k) * N + d;
      float s = *p;
#pragma unroll 4
      for (int q = j; q < stop; ++q) s = __fadd_rn(s, __ldg(dy + static_cast<size_t>(order[q]) * N + d));
      *p = s;
    }
  }
}

// ------------------------------------------------------------------ fillers (u: the cos_net_fill value in [-1, 1))
__global__ void constant_fill_kernel(float* p, int n, float v) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}
// min + (max - min) * (u + 1) / 2, one rounding per operation
__global__ void uniform_fill_kernel(float* p, int n, float lo, float hi) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    p[i] = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), __fmul_rn(__fadd_rn(p[i], 1.f), 0.5f)));
}
// Box-Muller on two independent draws: a = 1 - (u1 + 1) / 2 in (0, 1], b = (u2 + 1) / 2
__global__ void gaussian_fill_kernel(float* p, const float* u2, int n, float mean, float sd) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float a = 1.f - (p[i] + 1.f) * 0.5f, b = (u2[i] + 1.f) * 0.5f;
    p[i] = mean + sd * sqrtf(-2.f * logf(a)) * cospif(2.f * b);
  }
}

// GaussianFiller's sparse mask: p[i] stays with probability prob (u3 in [-1, 1): kept when (u3 + 1) / 2 < prob), else 0
__global__ void sparse_mask_kernel(float* p, const float* u3, int n, float prob) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (!((u3[i] + 1.f) * 0.5f < prob)) p[i] = 0.f;
}

int grid_for(int64_t n) {
  const int64_t g = (n + kThreads - 1) / kThreads;
  return static_cast<int>(g < 1 ? 1 : (g > kTargetSms * 16 ? kTargetSms * 16 : g));
}

// D and OD are 1 below three spatial axes, and H and OH are 1 for one ([N, C, L] runs as [N, C, 1, L])
struct ConvDims {
  int N, Cin, H, W, Cout, OH, OW;
  int D = 1, OD = 1;
  bool vol = false;  // three spatial axes: the Vol2col / Col2volGather instantiations
};

// Tile's outer = count(0, axis) of its bottom
int64_t tile_outer(const Op& op) {
  return shape_count(std::vector<int64_t>(op.in_shape.begin(), op.in_shape.begin() + op.tile_axis));
}
// A Deconvolution's dims are those of the convolution from its top to its bottom (the same weight blob, [Cin, Cout,
// KH, KW] of the deconvolution): its forward is that convolution's data gradient, its data gradient that
// convolution's forward, and its weight gradient that convolution's with the bottom as dy.
ConvDims conv_dims(const Op& op) {
  ConvDims d;
  const size_t axes = op.in_shape.size();
  d.vol = axes == 5;
  // a blob's spatial axes as D, H, W
  auto spatial = [axes](const std::vector<int64_t>& s, int* D, int* H, int* W) {
    *D = axes == 5 ? static_cast<int>(s[2]) : 1;
    *H = axes == 3 ? 1 : static_cast<int>(s[axes - 2]);
    *W = static_cast<int>(s[axes - 1]);
  };
  if (op.kind == OpKind::kDeconv) {
    d.N = static_cast<int>(op.in_shape[0]);
    d.Cin = static_cast<int>(op.out_shape[1]);
    spatial(op.out_shape, &d.D, &d.H, &d.W);
    d.Cout = static_cast<int>(op.in_shape[1]);
    spatial(op.in_shape, &d.OD, &d.OH, &d.OW);
    return d;
  }
  d.N = static_cast<int>(op.in_shape[0]), d.Cin = static_cast<int>(op.in_shape[1]);
  spatial(op.in_shape, &d.D, &d.H, &d.W);
  d.Cout = static_cast<int>(op.w_count / (static_cast<int64_t>(d.Cin) * op.kd * op.kh * op.kw));
  d.OD = (d.D + 2 * op.pd - op.kd) / op.sd + 1;
  d.OH = (d.H + 2 * op.ph - op.kh) / op.sh + 1;
  d.OW = (d.W + 2 * op.pw - op.kw) / op.sw + 1;
  return d;
}
ConvGeom geom(const ConvDims& d, const Op& op) {
  return ConvGeom{d.Cin, d.H, d.W, op.kh, op.kw, op.sh, op.sw, op.ph, op.pw, d.OH, d.OW};
}
// c: the channels of the blob the gather reads (Cin for Vol2col, Cout for Col2volGather)
ConvGeom3 geom3(const ConvDims& d, const Op& op, int c) {
  return ConvGeom3{c, d.D, d.H, d.W, op.kd, op.kh, op.kw, op.sd, op.sh, op.sw, op.pd, op.ph, op.pw, d.OD, d.OH, d.OW};
}
PoolGeom pool_geom(const Op& op) {
  return PoolGeom{static_cast<int>(op.in_shape[0]), static_cast<int>(op.in_shape[1]), static_cast<int>(op.in_shape[2]),
                  static_cast<int>(op.in_shape[3]), static_cast<int>(op.out_shape[2]), static_cast<int>(op.out_shape[3]),
                  op.kh, op.kw, op.sh, op.sw, op.ph, op.pw};
}
void bn_dims(const Op& op, int* n, int* c, int* hw) {
  int64_t total = 1;
  for (int64_t d : op.in_shape) total *= d;
  *n = static_cast<int>(op.in_shape[0]);
  *c = static_cast<int>(op.in_shape.size() > 1 ? op.in_shape[1] : 1);
  *hw = static_cast<int>(total / (static_cast<int64_t>(*n) * *c));
}
// Slice, Concat: elements after the axis (the same in the bottom and the top), and the elements of one outer index of a
// blob (its axis times that)
int64_t slice_inner(const Op& op) {
  int64_t n = 1;
  for (size_t a = op.slice_axis + 1; a < op.in_shape.size(); ++a) n *= op.in_shape[a];
  return n;
}
int64_t slice_span(const Op& op, const std::vector<int64_t>& shape) { return shape[op.slice_axis] * slice_inner(op); }
// InnerProduct: K = count(axis) inputs per row (the weight is [num_output, K]), and count(0, axis) rows
int ip_k(const Op& op) { return static_cast<int>(op.w_count / (op.w_count > 0 ? op.out_shape.back() : 1)); }
int ip_rows(const Op& op) { return static_cast<int>(shape_count(op.in_shape) / std::max(ip_k(op), 1)); }
// RNN: T steps of N streams, H hidden units, I = count(x, 2) inputs per step and S = count(x_static, 1)
struct RnnDims {
  int T, N, H, I, S;
};
RnnDims rnn_dims(const Op& op, const std::vector<int64_t>& tensor_count) {
  RnnDims d;
  d.T = static_cast<int>(op.in_shape[0]), d.N = static_cast<int>(op.in_shape[1]);
  d.H = static_cast<int>(op.out_shape[2]), d.I = static_cast<int>(shape_count(op.in_shape, 2));
  d.S = op.bottoms.size() > 2 ? static_cast<int>(tensor_count[op.bottoms[2]] / d.N) : 0;
  return d;
}
// PReLU: the elements each slope reduces over, the number of slopes, and the chunks of the slope gradient
int prelu_span(const Op& op) {
  return static_cast<int>(op.channel_shared ? shape_count(op.in_shape) : op.in_shape[0] * op.prelu_dim);
}
int prelu_slopes(const Op& op) { return op.channel_shared ? 1 : static_cast<int>(op.prelu_channels); }
int prelu_chunks(const Op& op) { return (prelu_span(op) + kPreluChunk - 1) / kPreluChunk; }

// The three GEMMs of a convolution of dims d: y = W * im2col(x) (+ bias); dx = W^T * dy gathered back to the input
// (+ bias); dst += dW = dy * im2col(x)^T, split over N * OH * OW in fixed chunks added in chunk order.
// Over three spatial axes the same three GEMMs run on Vol2col and Col2volGather, k and j extended by the depth axis.
cudaError_t conv_forward(const Op& op, const ConvDims& d, const float* x, const float* w, const float* bias, float* y,
                         cudaStream_t s) {
  if (d.vol) {
    const int K = d.Cin * op.kd * op.kh * op.kw, OV = d.OD * d.OH * d.OW;
    return gemm(DenseRM{w, K}, Vol2col{x, geom3(d, op, d.Cin)}, StoreNCHW{y, bias, d.Cout, OV}, d.Cout, d.N * OV, K,
                K, s);
  }
  const int K = d.Cin * op.kh * op.kw;
  return gemm(DenseRM{w, K}, Im2col{x, geom(d, op)}, StoreNCHW{y, bias, d.Cout, d.OH * d.OW}, d.Cout,
              d.N * d.OH * d.OW, K, K, s);
}
cudaError_t conv_data_grad(const Op& op, const ConvDims& d, const float* dy, const float* w, const float* bias, float* dx,
                           cudaStream_t s) {
  if (d.vol) {
    const int KK = op.kd * op.kh * op.kw, V = d.D * d.H * d.W;
    return gemm(WeightT{w, d.Cin, KK}, Col2volGather{dy, geom3(d, op, d.Cout)}, StoreNCHW{dx, bias, d.Cin, V}, d.Cin,
                d.N * V, d.Cout * KK, d.Cout * KK, s);
  }
  const int KD = d.Cout * op.kh * op.kw;
  return gemm(WeightT{w, d.Cin, op.kh * op.kw},
              Col2imGather{dy, d.Cout, d.H, d.W, op.kh, op.kw, op.sh, op.sw, op.ph, op.pw, d.OH, d.OW},
              StoreNCHW{dx, bias, d.Cin, d.H * d.W}, d.Cin, d.N * d.H * d.W, KD, KD, s);
}
cudaError_t conv_weight_grad(const Op& op, const ConvDims& d, const float* x, const float* dy, float* ws, float* dst,
                             cudaStream_t s) {
  const int K = d.N * d.OD * d.OH * d.OW, KW = d.Cin * op.kd * op.kh * op.kw;
  cudaError_t e =
      d.vol ? gemm(ChanMajor{dy, d.Cout, d.OD * d.OH * d.OW}, Transposed<Vol2col>{Vol2col{x, geom3(d, op, d.Cin)}},
                   StorePartial{ws, d.Cout, KW}, d.Cout, KW, K, split_chunk(K), s)
            : gemm(ChanMajor{dy, d.Cout, d.OH * d.OW}, Transposed<Im2col>{Im2col{x, geom(d, op)}},
                   StorePartial{ws, d.Cout, KW}, d.Cout, KW, K, split_chunk(K), s);
  if (e != cudaSuccess) return e;
  reduce_partials_kernel<<<grid_for(op.w_count), kThreads, 0, s>>>(ws, splits_of(K), static_cast<int>(op.w_count), dst);
  return cudaGetLastError();
}

// conv weight / bias gradients and the data gradient, from dy = the conv output's gradient
cudaError_t conv_backward(const Op& op, const float* x, const float* dy, float* dx, const float* w, float* diff,
                          float* ws, bool bias_grad, cudaStream_t s) {
  const ConvDims d = conv_dims(op);
  cudaError_t e = conv_weight_grad(op, d, x, dy, ws, diff + op.w_off, s);
  if (e != cudaSuccess) return e;
  if (bias_grad) bias_grad_kernel<<<d.Cout, kThreads, 0, s>>>(dy, d.N, d.Cout, d.OD * d.OH * d.OW, diff + op.b_off);
  if ((e = cudaGetLastError()) != cudaSuccess || !dx) return e;
  return conv_data_grad(op, d, dy, w, nullptr, dx, s);
}

// Deconvolution (deconv_layer.cpp) from dy = its top's gradient: the weight gradient of the convolution from top to
// bottom with the bottom x as that convolution's dy, the bias gradient over dy, and dx = that convolution's forward of dy
cudaError_t deconv_backward(const Op& op, const float* x, const float* dy, float* dx, const float* w, float* diff,
                            float* ws, cudaStream_t s) {
  const ConvDims d = conv_dims(op);
  cudaError_t e = conv_weight_grad(op, d, dy, x, ws, diff + op.w_off, s);
  if (e != cudaSuccess) return e;
  if (op.b_off >= 0) bias_grad_kernel<<<d.Cin, kThreads, 0, s>>>(dy, d.N, d.Cin, d.D * d.H * d.W, diff + op.b_off);
  if ((e = cudaGetLastError()) != cudaSuccess || !dx) return e;
  return conv_forward(op, d, dy, w, nullptr, dx, s);
}

}  // namespace

// ------------------------------------------------------------------ Crop's launches
namespace {
// The merged geometry of a crop, innermost axis first; false for a shape the kernels do not take.  *vec4 when the
// float4 kernels apply: the innermost run, the bottom's innermost dim and offset are multiples of 4 and every pointer
// is 16-byte aligned (the bottom's rows then start aligned too).
bool crop_geom(const std::vector<int64_t>& bottom, const std::vector<int64_t>& top, const std::vector<int64_t>& offsets,
               std::initializer_list<const void*> ptrs, CropGeom* g, bool* vec4) {
  const size_t n = bottom.size();
  if (n == 0 || n > static_cast<size_t>(kCropMaxAxes) || top.size() != n || offsets.size() != n) return false;
  g->rank = 0;
  for (size_t k = n; k-- > 0;) {
    if (top[k] < 1 || offsets[k] < 0 || offsets[k] + top[k] > bottom[k]) return false;
    const int r = g->rank - 1;
    if (r >= 0 && g->top[r] == g->bottom[r] && g->off[r] == 0) {  // the inner axis is whole: merge this one into it
      g->off[r] = offsets[k] * g->bottom[r];
      g->top[r] *= top[k];
      g->bottom[r] *= bottom[k];
    } else {
      g->top[g->rank] = top[k], g->bottom[g->rank] = bottom[k], g->off[g->rank] = offsets[k];
      ++g->rank;
    }
  }
  bool aligned = true;
  for (const void* p : ptrs) aligned = aligned && reinterpret_cast<uintptr_t>(p) % 16 == 0;
  *vec4 = aligned && g->top[0] % 4 == 0 && g->bottom[0] % 4 == 0 && g->off[0] % 4 == 0;
  if (*vec4) g->top[0] /= 4, g->bottom[0] /= 4, g->off[0] /= 4;
  return true;
}
}  // namespace

cudaError_t crop_forward(const float* x, float* y, const std::vector<int64_t>& bottom_shape,
                         const std::vector<int64_t>& top_shape, const std::vector<int64_t>& offsets, cudaStream_t s) {
  CropGeom g;
  bool vec4;
  if (!crop_geom(bottom_shape, top_shape, offsets, {x, y}, &g, &vec4)) return cudaErrorInvalidValue;
  const int64_t n = shape_count(top_shape) / (vec4 ? 4 : 1);
  if (vec4)
    crop_forward_kernel<float4><<<grid_for(n), kThreads, 0, s>>>(reinterpret_cast<const float4*>(x),
                                                                  reinterpret_cast<float4*>(y), n, g);
  else
    crop_forward_kernel<float><<<grid_for(n), kThreads, 0, s>>>(x, y, n, g);
  return cudaGetLastError();
}

cudaError_t crop_backward(const float* dy, float* dx, const std::vector<int64_t>& bottom_shape,
                          const std::vector<int64_t>& top_shape, const std::vector<int64_t>& offsets, cudaStream_t s) {
  CropGeom g;
  bool vec4;
  if (!crop_geom(bottom_shape, top_shape, offsets, {dy, dx}, &g, &vec4)) return cudaErrorInvalidValue;
  const int64_t n = shape_count(bottom_shape) / (vec4 ? 4 : 1);
  if (vec4)
    crop_backward_kernel<float4><<<grid_for(n), kThreads, 0, s>>>(reinterpret_cast<const float4*>(dy),
                                                                   reinterpret_cast<float4*>(dx), n, g);
  else
    crop_backward_kernel<float><<<grid_for(n), kThreads, 0, s>>>(dy, dx, n, g);
  return cudaGetLastError();
}

// ------------------------------------------------------------------ SPP's launches
namespace {
// The pyramid of spp_level() over a num x channels x height x width bottom; false for one the kernels do not take
bool spp_geom(int num, int channels, int height, int width, int levels, SppGeom* g) {
  if (num < 1 || channels < 1 || height < 1 || width < 1 || levels < 1 || levels > kSppMaxLevels) return false;
  *g = SppGeom{num, channels, height, width, levels, 0, {}, {}, {}, {}};
  int64_t per_sample = 0;
  for (int l = 0; l < levels; ++l) {
    const SppLevel v = spp_level(height, width, l);
    // pad < kernel (the parser's check) puts every window's start inside the map, so each level pools bins x bins
    if (v.pad_h >= v.kernel_h || v.pad_w >= v.kernel_w) return false;
    g->kh[l] = static_cast<int>(v.kernel_h), g->kw[l] = static_cast<int>(v.kernel_w);
    g->padh[l] = static_cast<int>(v.pad_h), g->padw[l] = static_cast<int>(v.pad_w);
    per_sample += static_cast<int64_t>(channels) * v.bins * v.bins;
  }
  const int64_t limit = int64_t(1) << 31;
  if (per_sample * num >= limit || static_cast<int64_t>(num) * channels * height * width >= limit) return false;
  g->per_sample = static_cast<int>(per_sample);
  return true;
}
}  // namespace

cudaError_t spp_forward(const float* x, float* y, int* argmax, int num, int channels, int height, int width, int levels,
                        bool max_pool, cudaStream_t s) {
  SppGeom g;
  if (!spp_geom(num, channels, height, width, levels, &g) || (max_pool && !argmax)) return cudaErrorInvalidValue;
  const int n = g.N * g.per_sample;
  spp_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, argmax, g, max_pool);
  return cudaGetLastError();
}

cudaError_t spp_backward(const float* dy, const int* argmax, float* dx, int num, int channels, int height, int width,
                         int levels, bool max_pool, cudaStream_t s) {
  SppGeom g;
  if (!spp_geom(num, channels, height, width, levels, &g) || (max_pool && !argmax)) return cudaErrorInvalidValue;
  const int n = num * channels * height * width;
  spp_backward_kernel<<<grid_for(n), kThreads, 0, s>>>(dy, argmax, dx, g, max_pool);
  return cudaGetLastError();
}

// ------------------------------------------------------------------ Tile's launches
bool tile_backward_staged(int64_t inner) { return inner < kTileStagedMaxInner; }

namespace {
bool tile_shape_ok(int64_t outer, int64_t inner, int64_t tiles) {
  return outer >= 1 && inner >= 1 && tiles >= 1 && outer <= kTileMaxTop / inner && outer * inner <= kTileMaxTop / tiles;
}
bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }
}  // namespace

cudaError_t tile_forward(const float* x, float* y, int64_t outer, int64_t inner, int64_t tiles, cudaStream_t s) {
  if (!tile_shape_ok(outer, inner, tiles)) return cudaErrorInvalidValue;
  const int64_t total = outer * tiles * inner;
  const int in = static_cast<int>(inner), ti = static_cast<int>(tiles);
  const FastDiv fi(static_cast<unsigned>(inner)), ft(static_cast<unsigned>(tiles));
  if (total % 4 == 0 && aligned16(y)) {
    const int n = static_cast<int>(total / 4);
    const int blocks = (n + kThreads - 1) / kThreads;
    if (inner % 4 == 0 && aligned16(x))
      tile_forward_kernel<4, true><<<blocks, kThreads, 0, s>>>(x, y, n, in, ti, fi, ft);
    else
      tile_forward_kernel<4, false><<<blocks, kThreads, 0, s>>>(x, y, n, in, ti, fi, ft);
  } else {
    const int n = static_cast<int>(total);
    tile_forward_kernel<1, false><<<(n + kThreads - 1) / kThreads, kThreads, 0, s>>>(x, y, n, in, ti, fi, ft);
  }
  return cudaGetLastError();
}

cudaError_t tile_backward(const float* dy, float* dx, int64_t outer, int64_t inner, int64_t tiles, cudaStream_t s) {
  if (!tile_shape_ok(outer, inner, tiles)) return cudaErrorInvalidValue;
  const int in = static_cast<int>(inner), ti = static_cast<int>(tiles);
  if (!tile_backward_staged(inner)) {
    const int n = static_cast<int>(outer * inner);
    tile_backward_direct_kernel<<<(n + kThreads - 1) / kThreads, kThreads, 0, s>>>(dy, dx, n, in, ti);
    return cudaGetLastError();
  }
  // rows per block: a block's worth of outputs, fewer when that would leave the grid under two blocks per SM
  const int64_t spread = (outer + 2 * kTargetSms - 1) / (2 * kTargetSms);
  const int rows = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(kThreads / inner, spread)));
  const int outputs = rows * in;
  const int stride = outputs + ((in - outputs) % 32 + 32) % 32;  // >= outputs, congruent to inner mod 32
  const int64_t blocks = (outer + rows - 1) / rows;
  const int last = static_cast<int>((tiles - 1) % kTileChunk + 1);  // the last chunk's tiles
  tile_backward_staged_kernel<<<static_cast<unsigned>(blocks), kThreads, 0, s>>>(
      dy, dx, static_cast<int>(outer), in, ti, rows, stride, FastDiv(static_cast<unsigned>(in)),
      FastDiv(static_cast<unsigned>(kTileChunk * in)), FastDiv(static_cast<unsigned>(last * in)));
  return cudaGetLastError();
}

// ------------------------------------------------------------------ engine

NativeProducer* NativeProducer::create(const Plan& plan, int device, float* data, float* diff, int* status,
                                       std::string* err) {
  NativeProducer* p = new NativeProducer(plan, device, data, diff, status);
  if (!p->allocate(err)) {
    delete p;
    return nullptr;
  }
  return p;
}

NativeProducer::~NativeProducer() {
  cudaSetDevice(device_);
  if (done_) {  // the last call may still run on whatever stream it was given
    cudaEventSynchronize(done_);
    cudaEventDestroy(done_);
  }
  for (void* a : allocations_) cudaFree(a);
  cudaGetLastError();
}

bool NativeProducer::allocate(std::string* err) {
  auto alloc = [&](size_t bytes, void** out) {
    cudaError_t e = cudaMalloc(out, bytes > 0 ? bytes : 4);
    if (e != cudaSuccess) {
      *err = std::string("native producer: cudaMalloc failed: ") + cudaGetErrorString(e);
      cudaGetLastError();
      return false;
    }
    allocations_.push_back(*out);
    return true;
  };
  cudaError_t e = cudaSetDevice(device_);
  if (e != cudaSuccess) {
    *err = std::string("native producer: ") + cudaGetErrorString(e) + " (this library has no CPU path)";
    cudaGetLastError();
    return false;
  }
  const size_t T = plan_.tensor_count.size();
  act_.assign(T, nullptr);
  grad_.assign(T, nullptr);
  // Every tensor owning its storage gets a gradient buffer, a staged input too: SoftmaxWithLoss writes its bottom's
  // gradient whatever that bottom is.  Activations of staged inputs are the caller's buffers, set per call.
  for (size_t t = 0; t < T; ++t) {
    if (plan_.storage[t] != static_cast<int>(t)) continue;
    const size_t bytes = plan_.tensor_count[t] * sizeof(float);
    void* g;
    if (!alloc(bytes, &g)) return false;
    // a tensor nothing reads keeps a zero gradient
    if (cudaMemset(g, 0, bytes) != cudaSuccess) {
      *err = "native producer: cudaMemset failed";
      return false;
    }
    grad_[t] = static_cast<float*>(g);
    // a Split top's activation is its bottom's, set when the forward reaches it
    if (static_cast<int>(t) < plan_.ninputs || plan_.data_alias[t]) continue;
    void* a;
    if (!alloc(bytes, &a)) return false;
    act_[t] = static_cast<float*>(a);
  }
  for (size_t t = 0; t < T; ++t) {
    const int st = plan_.storage[t];
    // a staged input is never an in-place alias (build_plan), so every alias below has device memory of its own
    if (static_cast<int>(t) >= plan_.ninputs && st < plan_.ninputs) {
      *err = "native producer: tensor " + std::to_string(t) + " aliases a staged input";
      return false;
    }
    grad_[t] = grad_[st];
    if (static_cast<int>(t) >= plan_.ninputs) act_[t] = act_[st];
    if (!grad_[t] || (static_cast<int>(t) >= plan_.ninputs && !plan_.data_alias[t] && !act_[t])) {
      *err = "native producer: tensor " + std::to_string(t) + " has no device storage";
      return false;
    }
  }
  op_aux_.assign(plan_.ops.size(), nullptr);
  op_z_.assign(plan_.ops.size(), nullptr);
  op_dz_.assign(plan_.ops.size(), nullptr);
  rnn_.assign(plan_.ops.size(), RnnBuffers());
  size_t ws = 1;
  for (size_t i = 0; i < plan_.ops.size(); ++i) {
    const Op& op = plan_.ops[i];
    const int64_t out = plan_.tensor_count[op.out];
    if (op.kind == OpKind::kConv || op.kind == OpKind::kConvBiasReluMaxPool || op.kind == OpKind::kDeconv) {
      const ConvDims d = conv_dims(op);
      const size_t K = static_cast<size_t>(d.N) * d.OD * d.OH * d.OW;
      ws = std::max(ws, static_cast<size_t>(splits_of(static_cast<int>(K))) * op.w_count);
      if (op.kind == OpKind::kConvBiasReluMaxPool) {
        const size_t zb = static_cast<size_t>(d.N) * d.Cout * d.OH * d.OW * sizeof(float);
        void *z, *dz, *idx;
        if (!alloc(zb, &z) || !alloc(zb, &dz) || !alloc(out, &idx)) return false;
        op_z_[i] = static_cast<float*>(z), op_dz_[i] = static_cast<float*>(dz), op_aux_[i] = idx;
        ws = std::max(ws, static_cast<size_t>(d.N + 1) * d.Cout);  // bias partials + dbias
      }
    } else if (((op.kind == OpKind::kPool || op.kind == OpKind::kSPP) && op.max_pool) ||
               (op.kind == OpKind::kEltwise && op.eltwise_op == kEltwiseMax)) {
      if (!alloc(out * sizeof(int), &op_aux_[i])) return false;
    } else if (op.kind == OpKind::kInnerProduct) {
      ws = std::max(ws, static_cast<size_t>(splits_of(ip_rows(op))) * op.w_count);
    } else if (op.kind == OpKind::kRNN) {
      const RnnDims d = rnn_dims(op, plan_.tensor_count);
      const size_t step = static_cast<size_t>(d.N) * d.H, seq = step * d.T;
      RnnBuffers& b = rnn_[i];
      void *g, *h, *state, *dzo, *dho, *dpre;
      if (!alloc(seq * sizeof(float), &g) || !alloc(seq * sizeof(float) + step * sizeof(float), &h) ||
          !alloc(step * sizeof(float), &state) || !alloc(seq * sizeof(float), &dzo) ||
          !alloc(seq * sizeof(float), &dho) || !alloc(seq * sizeof(float), &dpre))
        return false;
      b.g = static_cast<float*>(g), b.h = static_cast<float*>(h), b.state = static_cast<float*>(state);
      b.dzo = static_cast<float*>(dzo), b.dho = static_cast<float*>(dho), b.dpre = static_cast<float*>(dpre);
      if (cudaMemset(b.state, 0, step * sizeof(float)) != cudaSuccess) {  // the first call starts from h = 0
        *err = "native producer: cudaMemset failed";
        return false;
      }
      const size_t seq_splits = static_cast<size_t>(splits_of(d.T * d.N));
      ws = std::max(ws, seq_splits * d.H * std::max(d.H, d.I));  // dW_hh, dW_ho and dW_xh
      if (d.S > 0) {
        void *z, *dz;
        if (!alloc(step * sizeof(float), &z) || !alloc(step * sizeof(float), &dz)) return false;
        b.z = static_cast<float*>(z), b.dz = static_cast<float*>(dz);
        ws = std::max(ws, static_cast<size_t>(splits_of(d.N)) * d.H * d.S);
      }
    } else if (op.kind == OpKind::kBatchNorm) {
      int n, c, hw;
      bn_dims(op, &n, &c, &hw);
      if (!alloc(2 * static_cast<size_t>(c) * sizeof(float), &op_aux_[i])) return false;
      ws = std::max(ws, bn_workspace_floats(n, c));
    } else if (op.kind == OpKind::kMVN) {  // the per-row statistics, and the long rows' chunk partials
      if (!alloc(5 * static_cast<size_t>(op.mvn_rows) * sizeof(float), &op_aux_[i])) return false;
      ws = std::max(ws, mvn_workspace_floats(op.mvn_rows, op.mvn_dim));
    } else if (op.kind == OpKind::kSigmoidCrossEntropyLoss || op.kind == OpKind::kHingeLoss) {
      ws = std::max(ws, static_cast<size_t>(grid_for(plan_.tensor_count[op.bottoms[0]])));  // the per-block partials
    } else if (op.kind == OpKind::kPReLU) {
      ws = std::max(ws, static_cast<size_t>(prelu_slopes(op)) * prelu_chunks(op));  // the slope gradient's partials
    } else if (op.kind == OpKind::kEmbed) {  // the id grouping: K + 1 counts / group ends, then the M placed positions
      ws = std::max(ws, static_cast<size_t>(op.input_dim + 1 + plan_.tensor_count[op.bottoms[0]]));
    }
  }
  if ((e = cudaEventCreateWithFlags(&done_, cudaEventDisableTiming)) != cudaSuccess) {
    *err = std::string("native producer: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return false;
  }
  void* w;
  if (!alloc(ws * sizeof(float), &w)) return false;
  workspace_ = static_cast<float*>(w);
  workspace_floats_ = ws;
  if ((e = cudaDeviceSynchronize()) != cudaSuccess) {
    *err = std::string("native producer: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return false;
  }
  return true;
}

bool NativeProducer::fill(uint64_t seed, cudaStream_t s, std::string* err) {
  cudaSetDevice(device_);
  float* tmp = nullptr;
  int64_t most = 1;
  for (int64_t c : plan_.blob_count) most = std::max(most, c);
  cudaError_t e = cudaMalloc(&tmp, most * sizeof(float));
  for (size_t k = 0; k < plan_.blob_count.size() && e == cudaSuccess; ++k) {
    const FillerSpec& f = plan_.blob_filler[k];
    const int n = static_cast<int>(plan_.blob_count[k]);
    if (n == 0) continue;
    float* p = data_ + plan_.blob_off[k];
    const std::vector<int64_t>& sh = plan_.blob_shape[k];
    // filler.hpp: fan_in = count / shape(0), fan_out = count / shape(1) (count for a 1-axis blob)
    const int fan_in = sh.empty() ? n : static_cast<int>(n / sh[0]);  // a 0-axis (scalar) blob: its one element
    const int fan_out = sh.size() > 1 ? static_cast<int>(n / sh[1]) : n;
    const float norm = f.variance_norm == "FAN_OUT" ? static_cast<float>(fan_out)
                       : f.variance_norm == "AVERAGE" ? static_cast<float>(fan_in + fan_out) / 2.0f
                                                      : static_cast<float>(fan_in);
    if (f.type == "constant") {
      constant_fill_kernel<<<grid_for(n), kThreads, 0, s>>>(p, n, f.value);
      e = cudaGetLastError();
    } else if (f.type == "uniform") {
      e = launch_fill(p, n, seed, k, 1.f, s);
      if (e == cudaSuccess) uniform_fill_kernel<<<grid_for(n), kThreads, 0, s>>>(p, n, f.min, f.max);
    } else if (f.type == "xavier") {
      e = launch_fill(p, n, seed, k, sqrtf(3.0f / norm), s);  // uniform in [-scale, scale)
    } else {  // gaussian, msra
      const float mean = f.type == "msra" ? 0.f : f.mean, sd = f.type == "msra" ? sqrtf(2.0f / norm) : f.std;
      e = launch_fill(p, n, seed, k, 1.f, s);
      if (e == cudaSuccess) e = launch_fill(tmp, n, seed, k + (uint64_t(1) << 32), 1.f, s);
      if (e == cudaSuccess) gaussian_fill_kernel<<<grid_for(n), kThreads, 0, s>>>(p, tmp, n, mean, sd);
      // filler.hpp: sparse >= 0 keeps each weight with probability sparse / num_outputs (shape(0)), drawn under stream
      // index + 2^33
      if (e == cudaSuccess && f.type == "gaussian" && f.sparse >= 0) {
        const float prob = static_cast<float>(f.sparse) / static_cast<float>(sh.empty() ? 1 : sh[0]);
        e = launch_fill(tmp, n, seed, k + (uint64_t(2) << 32), 1.f, s);
        if (e == cudaSuccess) sparse_mask_kernel<<<grid_for(n), kThreads, 0, s>>>(p, tmp, n, prob);
      }
    }
    if (e == cudaSuccess) e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (tmp) cudaFree(tmp);
  if (e != cudaSuccess) {
    *err = std::string("native producer fill: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return false;
  }
  return true;
}

int NativeProducer::callback(void* user, int, const cos_blob* inputs, int ninputs, float* loss_dev,
                             void* cuda_stream) {
  return static_cast<NativeProducer*>(user)->forward_backward(inputs, ninputs, loss_dev,
                                                              static_cast<cudaStream_t>(cuda_stream));
}

int NativeProducer::forward_backward(const cos_blob* inputs, int ninputs, float* loss_dev, cudaStream_t s) {
  if (!inputs || !loss_dev || ninputs < plan_.ninputs) return -1;
  for (int i = 0; i < plan_.ninputs; ++i) {
    const cos_blob& b = inputs[i];
    if (!b.data || static_cast<int64_t>(b.num) * b.channels * b.height * b.width != plan_.tensor_count[i]) return -1;
    act_[i] = const_cast<float*>(b.data);
  }
  for (size_t i = 0; i < plan_.ops.size(); ++i) {
    cudaError_t e = run_op_forward(plan_.ops[i], i, loss_dev, s);
    if (e != cudaSuccess) return e;
  }
  for (size_t i = plan_.ops.size(); i-- > 0;) {
    cudaError_t e = run_op_backward(plan_.ops[i], i, s);
    if (e != cudaSuccess) return e;
  }
  return cudaEventRecord(done_, s);
}

cudaError_t NativeProducer::run_op_forward(const Op& op, size_t i, float* loss_dev, cudaStream_t s) {
  const float* x = act_[op.bottoms[0]];
  float* y = act_[op.out];
  const int n = static_cast<int>(plan_.tensor_count[op.out]);
  switch (op.kind) {
    case OpKind::kConv:
    case OpKind::kConvBiasReluMaxPool: {
      const ConvDims d = conv_dims(op);
      const bool fused = op.kind == OpKind::kConvBiasReluMaxPool;
      const float* bias = (!fused && op.b_off >= 0) ? data_ + op.b_off : nullptr;
      float* z = fused ? op_z_[i] : y;
      cudaError_t e = conv_forward(op, d, x, data_ + op.w_off, bias, z, s);
      if (e != cudaSuccess || !fused) return e;
      return bias_relu_maxpool_forward(z, data_ + op.b_off, y, static_cast<uint8_t*>(op_aux_[i]), d.N, d.Cout, d.OH,
                                       d.OW, op.pool_kernel, op.pool_stride, static_cast<int>(op.out_shape[2]),
                                       static_cast<int>(op.out_shape[3]), s);
    }
    case OpKind::kPool:
      if (op.max_pool)
        max_pool_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, static_cast<int*>(op_aux_[i]), pool_geom(op));
      else
        ave_pool_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, pool_geom(op));
      return cudaGetLastError();
    case OpKind::kInnerProduct: {
      const int B = ip_rows(op), N = static_cast<int>(op.out_shape.back()), K = ip_k(op);
      return gemm(DenseRM{x, K}, DenseCM{data_ + op.w_off, K},
                  StoreRM{y, op.b_off >= 0 ? data_ + op.b_off : nullptr, N}, B, N, K, K, s);
    }
    case OpKind::kReLU:
      relu_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.slope);
      return cudaGetLastError();
    case OpKind::kSigmoid:
      sigmoid_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n);
      return cudaGetLastError();
    case OpKind::kBatchNorm: {
      int bn, c, hw;
      bn_dims(op, &bn, &c, &hw);
      float* m = data_ + op.w_off;
      return batch_norm_forward(x, y, m, m + c, m + 2 * c, static_cast<float*>(op_aux_[i]), workspace_, bn, c, hw, 1,
                                op.global_stats, op.fraction, op.eps, s);
    }
    case OpKind::kMVN:
      return mvn_forward(x, y, static_cast<float*>(op_aux_[i]), workspace_, op.mvn_rows, op.mvn_dim,
                         op.normalize_variance, op.eps, s);
    case OpKind::kSlice:
      slice_copy_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, slice_span(op, op.out_shape), slice_span(op, op.in_shape),
                                                         op.slice_begin * slice_inner(op), false);
      return cudaGetLastError();
    case OpKind::kConcat: {
      const int64_t nin = plan_.tensor_count[op.bottoms[0]];
      slice_copy_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, y, nin, slice_span(op, op.in_shape),
                                                           slice_span(op, op.out_shape),
                                                           op.slice_begin * slice_inner(op), true);
      return cudaGetLastError();
    }
    case OpKind::kCrop:
      return crop_forward(x, y, op.in_shape, op.out_shape, op.crop_offsets, s);
    case OpKind::kSPP:
      return spp_forward(x, y, static_cast<int*>(op_aux_[i]), static_cast<int>(op.in_shape[0]),
                         static_cast<int>(op.in_shape[1]), static_cast<int>(op.in_shape[2]),
                         static_cast<int>(op.in_shape[3]), op.spp_levels, op.max_pool, s);
    case OpKind::kTile:
      return tile_forward(x, y, tile_outer(op), shape_count(op.in_shape, op.tile_axis), op.tiles, s);
    case OpKind::kDeconv:  // the data gradient of the convolution from top to bottom, with the bias in its store
      return conv_data_grad(op, conv_dims(op), x, data_ + op.w_off, op.b_off >= 0 ? data_ + op.b_off : nullptr, y, s);
    case OpKind::kSplit:  // no copy: the top reads the bottom's memory
    case OpKind::kFlatten:
    case OpKind::kReshape:
      act_[op.out] = act_[op.bottoms[0]];
      return cudaSuccess;
    case OpKind::kEltwise: {
      const size_t nb = op.bottoms.size();
      if (op.eltwise_op == kEltwiseSum) {
        for (size_t b = 0; b < nb; ++b)
          eltwise_axpy_kernel<<<grid_for(n), kThreads, 0, s>>>(act_[op.bottoms[b]], op.coeffs[b], y, n, b == 0);
      } else if (op.eltwise_op == kEltwiseProd) {
        mul_kernel<<<grid_for(n), kThreads, 0, s>>>(act_[op.bottoms[0]], act_[op.bottoms[1]], y, n);
        for (size_t b = 2; b < nb; ++b) mul_kernel<<<grid_for(n), kThreads, 0, s>>>(y, act_[op.bottoms[b]], y, n);
      } else {
        int* idx = static_cast<int*>(op_aux_[i]);
        eltwise_max_kernel<<<grid_for(n), kThreads, 0, s>>>(act_[op.bottoms[0]], act_[op.bottoms[1]], 1, y, idx, n);
        for (size_t b = 2; b < nb; ++b)
          eltwise_max_kernel<<<grid_for(n), kThreads, 0, s>>>(nullptr, act_[op.bottoms[b]], static_cast<int>(b), y, idx,
                                                              n);
      }
      return cudaGetLastError();
    }
    case OpKind::kScale:
      scale_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, data_ + op.w_off, op.b_off >= 0 ? data_ + op.b_off : nullptr,
                                                            y, n, static_cast<int>(op.scale_dim),
                                                            static_cast<int>(op.scale_inner));
      return cudaGetLastError();
    case OpKind::kLRNWithin:
      return lrn_within_forward(x, y, static_cast<int>(op.in_shape[0]), static_cast<int>(op.in_shape[1]),
                                static_cast<int>(op.in_shape[2]), static_cast<int>(op.in_shape[3]), op.lrn_size,
                                op.lrn_alpha, op.lrn_beta, s);
    // The loss kernels also write their bottoms' gradients.  SoftmaxWithLoss writes its bottom's whatever bottom_grad
    // says (a staged input's too: every tensor has a gradient buffer).
    case OpKind::kSoftmaxLoss:
      softmax_loss_kernel<<<1, kThreads, 0, s>>>(x, act_[op.bottoms[1]], grad_[op.bottoms[0]], loss_dev,
                                                 static_cast<int>(op.rows), static_cast<int>(op.classes),
                                                 static_cast<int>(op.inner), op.loss_weight, status_);
      return cudaGetLastError();
    case OpKind::kContrastiveLoss: {
      const int N = static_cast<int>(op.in_shape[0]);
      const int C = static_cast<int>(plan_.tensor_count[op.bottoms[0]] / N);
      contrastive_loss_kernel<<<1, kThreads, 0, s>>>(x, act_[op.bottoms[1]], act_[op.bottoms[2]],
                                                     op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr,
                                                     op.bottom_grad[1] ? grad_[op.bottoms[1]] : nullptr, loss_dev, N, C,
                                                     op.margin, op.legacy, op.loss_weight, status_);
      return cudaGetLastError();
    }
    case OpKind::kEuclideanLoss:
      euclidean_loss_kernel<<<1, kThreads, 0, s>>>(x, act_[op.bottoms[1]],
                                                   op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr,
                                                   op.bottom_grad[1] ? grad_[op.bottoms[1]] : nullptr, loss_dev,
                                                   static_cast<int>(plan_.tensor_count[op.bottoms[0]]),
                                                   static_cast<int>(op.in_shape[0]), op.loss_weight);
      return cudaGetLastError();
    case OpKind::kSigmoidCrossEntropyLoss: {
      const int count = static_cast<int>(plan_.tensor_count[op.bottoms[0]]), num = static_cast<int>(op.in_shape[0]);
      const int blocks = grid_for(count);
      sigmoid_xent_loss_kernel<<<blocks, kThreads, 0, s>>>(x, act_[op.bottoms[1]],
                                                           op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr,
                                                           workspace_, count, num, op.loss_weight);
      sigmoid_xent_loss_total_kernel<<<1, 1, 0, s>>>(workspace_, blocks, num, op.loss_weight, loss_dev);
      return cudaGetLastError();
    }
    case OpKind::kTanH:
      tanh_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n);
      return cudaGetLastError();
    case OpKind::kELU:
      elu_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.alpha);
      return cudaGetLastError();
    case OpKind::kAbsVal:
      absval_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n);
      return cudaGetLastError();
    case OpKind::kBNLL:
      bnll_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n);
      return cudaGetLastError();
    case OpKind::kPower: {  // power_layer.cpp: the constant is pow(shift, power) in float, on the host
      const bool constant = op.power * op.scale == 0.f;
      const float value = op.power == 0.f ? 1.f : std::pow(op.shift, op.power);
      power_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.power, op.scale, op.shift, constant, value);
      return cudaGetLastError();
    }
    case OpKind::kExp:
      exp_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.inner_scale, op.outer_scale);
      return cudaGetLastError();
    case OpKind::kLog:
      log_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.scale, op.shift, op.base_scale);
      return cudaGetLastError();
    case OpKind::kThreshold:
      threshold_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, y, n, op.threshold);
      return cudaGetLastError();
    case OpKind::kPReLU:
      prelu_forward_kernel<<<grid_for(n), kThreads, 0, s>>>(x, data_ + op.w_off, y, n,
                                                            static_cast<int>(op.prelu_channels),
                                                            static_cast<int>(op.prelu_dim), op.channel_shared);
      return cudaGetLastError();
    case OpKind::kSoftmax: {
      const int rows = static_cast<int>(op.outer * op.inner);
      softmax_forward_kernel<<<grid_for(rows), kThreads, 0, s>>>(x, y, rows, static_cast<int>(op.classes),
                                                                 static_cast<int>(op.inner));
      return cudaGetLastError();
    }
    case OpKind::kMultinomialLogisticLoss: {
      const int num = static_cast<int>(op.in_shape[0]);
      mll_loss_kernel<<<1, kThreads, 0, s>>>(x, act_[op.bottoms[1]], op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr,
                                             loss_dev, num, static_cast<int>(plan_.tensor_count[op.bottoms[0]] / num),
                                             op.loss_weight, status_);
      return cudaGetLastError();
    }
    case OpKind::kHingeLoss: {
      const int count = static_cast<int>(plan_.tensor_count[op.bottoms[0]]), num = static_cast<int>(op.in_shape[0]);
      const int blocks = grid_for(count);
      hinge_loss_kernel<<<blocks, kThreads, 0, s>>>(x, act_[op.bottoms[1]],
                                                    op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr, workspace_,
                                                    count, count / num, num, op.hinge_l2, op.loss_weight, status_);
      sigmoid_xent_loss_total_kernel<<<1, 1, 0, s>>>(workspace_, blocks, num, op.loss_weight, loss_dev);
      return cudaGetLastError();
    }
    case OpKind::kEmbed: {
      const int M = static_cast<int>(plan_.tensor_count[op.bottoms[0]]), N = static_cast<int>(op.out_shape.back());
      const int K = static_cast<int>(op.input_dim);
      const float* w = data_ + op.w_off;
      const float* b = op.b_off >= 0 ? data_ + op.b_off : nullptr;
      auto aligned = [](const float* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
      if (N % 4 == 0 && aligned(w) && (!b || aligned(b)) && aligned(y))
        embed_forward_kernel<4><<<grid_for(static_cast<int64_t>(M) * N / 4), kThreads, 0, s>>>(x, w, b, y, M, N, K,
                                                                                               status_);
      else
        embed_forward_kernel<1><<<grid_for(static_cast<int64_t>(M) * N), kThreads, 0, s>>>(x, w, b, y, M, N, K, status_);
      return cudaGetLastError();
    }
    case OpKind::kRNN: {  // recurrent_layer.cpp Forward_cpu without expose_hidden, over rnn_layer.cpp's unrolled net
      const RnnDims d = rnn_dims(op, plan_.tensor_count);
      const RnnBuffers& b = rnn_[i];
      const float* cont = act_[op.bottoms[1]];
      const float* whh = data_ + op.rnn_off[Op::kWhh];
      const size_t step = static_cast<size_t>(d.N) * d.H;
      const int TN = d.T * d.N;
      // g = x W_xh^T + b_h over every step, z = x_static W_xh_static^T, and h_{-1} = the carried state
      cudaError_t e = gemm(DenseRM{x, d.I}, DenseCM{data_ + op.rnn_off[Op::kWxh], d.I},
                           StoreRM{b.g, data_ + op.rnn_off[Op::kBh], d.H}, TN, d.H, d.I, d.I, s);
      if (e == cudaSuccess && b.z)
        e = gemm(DenseRM{act_[op.bottoms[2]], d.S}, DenseCM{data_ + op.rnn_off[Op::kWxhStatic], d.S},
                 StoreRM{b.z, nullptr, d.H}, d.N, d.H, d.S, d.S, s);
      if (e == cudaSuccess) e = cudaMemcpyAsync(b.h, b.state, step * sizeof(float), cudaMemcpyDeviceToDevice, s);
      // one launch per step: h_t from cont_t * h_{t-1}
      for (int t = 0; t < d.T && e == cudaSuccess; ++t)
        e = gemm(ContGather{b.h + t * step, cont + static_cast<size_t>(t) * d.N, d.H}, DenseCM{whh, d.H},
                 RnnStep{b.g + t * step, b.z, b.h + (t + 1) * step, d.H}, d.N, d.H, d.H, d.H, s);
      // the top o = tanh(h W_ho^T + b_o) over every step, and h_{T-1} carried to the next call
      if (e == cudaSuccess)
        e = gemm(DenseRM{b.h + step, d.H}, DenseCM{data_ + op.rnn_off[Op::kWho], d.H},
                 StoreTanhRM{y, data_ + op.rnn_off[Op::kBo], d.H}, TN, d.H, d.H, d.H, s);
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(b.state, b.h + d.T * step, step * sizeof(float), cudaMemcpyDeviceToDevice, s);
      return e;
    }
    default:
      return cudaErrorInvalidValue;
  }
}

cudaError_t NativeProducer::run_op_backward(const Op& op, size_t i, cudaStream_t s) {
  const float* x = act_[op.bottoms[0]];
  const float* dy = grad_[op.out];
  float* dx = op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr;
  const int nin = static_cast<int>(plan_.tensor_count[op.bottoms[0]]);
  if (op.no_backward) return cudaSuccess;  // no gradient reaches the top
  switch (op.kind) {
    case OpKind::kConv:
      return conv_backward(op, x, dy, dx, data_ + op.w_off, diff_, workspace_, op.b_off >= 0, s);
    case OpKind::kDeconv:
      return deconv_backward(op, x, dy, dx, data_ + op.w_off, diff_, workspace_, s);
    case OpKind::kConvBiasReluMaxPool: {
      const ConvDims d = conv_dims(op);
      float* partials = workspace_;
      float* dbias = workspace_ + static_cast<size_t>(d.N) * d.Cout;
      cudaError_t e = bias_relu_maxpool_backward(dy, static_cast<const uint8_t*>(op_aux_[i]), op_dz_[i], partials, dbias,
                                                 d.N, d.Cout, d.OH, d.OW, op.pool_kernel, op.pool_stride,
                                                 static_cast<int>(op.out_shape[2]), static_cast<int>(op.out_shape[3]), s);
      if (e != cudaSuccess) return e;
      accumulate_kernel<<<grid_for(d.Cout), kThreads, 0, s>>>(diff_ + op.b_off, dbias, d.Cout);
      if ((e = cudaGetLastError()) != cudaSuccess) return e;
      return conv_backward(op, x, op_dz_[i], dx, data_ + op.w_off, diff_, workspace_, false, s);
    }
    case OpKind::kPool:
      if (!dx) return cudaSuccess;
      if (op.max_pool)
        max_pool_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, static_cast<const int*>(op_aux_[i]), dx,
                                                                     pool_geom(op));
      else
        ave_pool_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, dx, pool_geom(op));
      return cudaGetLastError();
    case OpKind::kInnerProduct: {
      const int B = ip_rows(op), N = static_cast<int>(op.out_shape.back()), K = ip_k(op);
      cudaError_t e = gemm(DenseCM{dy, N}, DenseRM{x, K}, StorePartial{workspace_, N, K}, N, K, B, split_chunk(B), s);
      if (e != cudaSuccess) return e;
      reduce_partials_kernel<<<grid_for(op.w_count), kThreads, 0, s>>>(workspace_, splits_of(B),
                                                                         static_cast<int>(op.w_count), diff_ + op.w_off);
      if (op.b_off >= 0) bias_grad_kernel<<<N, kThreads, 0, s>>>(dy, B, N, 1, diff_ + op.b_off);
      if ((e = cudaGetLastError()) != cudaSuccess || !dx) return e;
      return gemm(DenseRM{dy, N}, DenseRM{data_ + op.w_off, K}, StoreRM{dx, nullptr, K}, B, K, N, N, s);
    }
    case OpKind::kReLU:
      if (!dx) return cudaSuccess;
      relu_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, dy, dx, nin, op.slope);
      return cudaGetLastError();
    case OpKind::kSigmoid:
      if (!dx) return cudaSuccess;
      sigmoid_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(act_[op.out], dy, dx, nin);
      return cudaGetLastError();
    case OpKind::kBatchNorm: {
      if (!dx) return cudaSuccess;
      int bn, c, hw;
      bn_dims(op, &bn, &c, &hw);
      return batch_norm_backward(x, dy, dx, static_cast<const float*>(op_aux_[i]), workspace_, bn, c, hw, 1,
                                 op.global_stats, op.eps, s);
    }
    case OpKind::kMVN:  // reads its own top y, not x
      if (!dx) return cudaSuccess;
      return mvn_backward(act_[op.out], dy, dx, static_cast<float*>(op_aux_[i]), workspace_, op.mvn_rows, op.mvn_dim,
                          op.normalize_variance, s);
    case OpKind::kLRNWithin:
      if (!dx) return cudaSuccess;
      return lrn_within_backward(x, dy, dx, static_cast<int>(op.in_shape[0]), static_cast<int>(op.in_shape[1]),
                                 static_cast<int>(op.in_shape[2]), static_cast<int>(op.in_shape[3]), op.lrn_size,
                                 op.lrn_alpha, op.lrn_beta, s);
    case OpKind::kSlice: {
      if (!dx) return cudaSuccess;
      const int64_t n = plan_.tensor_count[op.out];
      slice_copy_kernel<<<grid_for(n), kThreads, 0, s>>>(dy, dx, n, slice_span(op, op.out_shape),
                                                         slice_span(op, op.in_shape), op.slice_begin * slice_inner(op),
                                                         true);
      return cudaGetLastError();
    }
    case OpKind::kConcat:
      if (!dx) return cudaSuccess;
      slice_copy_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, dx, nin, slice_span(op, op.in_shape),
                                                           slice_span(op, op.out_shape),
                                                           op.slice_begin * slice_inner(op), false);
      return cudaGetLastError();
    case OpKind::kCrop:  // writes every element of dx: the engine's data gradients are written, not accumulated
      return dx ? crop_backward(dy, dx, op.in_shape, op.out_shape, op.crop_offsets, s) : cudaSuccess;
    case OpKind::kSPP:  // writes every element of dx
      if (!dx) return cudaSuccess;
      return spp_backward(dy, static_cast<const int*>(op_aux_[i]), dx, static_cast<int>(op.in_shape[0]),
                          static_cast<int>(op.in_shape[1]), static_cast<int>(op.in_shape[2]),
                          static_cast<int>(op.in_shape[3]), op.spp_levels, op.max_pool, s);
    case OpKind::kTile:  // writes every element of dx
      return dx ? tile_backward(dy, dx, tile_outer(op), shape_count(op.in_shape, op.tile_axis), op.tiles, s)
                : cudaSuccess;
    case OpKind::kSplit: {  // top 0's op: dx = the read tops' gradients summed in top order; the other tops' do nothing
      if (!dx || op.split_top != 0) return cudaSuccess;
      const std::vector<int>& g = op.split_sum;
      const size_t bytes = static_cast<size_t>(nin) * sizeof(float);
      if (g.empty()) return cudaMemsetAsync(dx, 0, bytes, s);
      if (g.size() == 1) return cudaMemcpyAsync(dx, grad_[g[0]], bytes, cudaMemcpyDeviceToDevice, s);
      add_kernel<<<grid_for(nin), kThreads, 0, s>>>(grad_[g[0]], grad_[g[1]], dx, nin);
      for (size_t k = 2; k < g.size(); ++k) accumulate_kernel<<<grid_for(nin), kThreads, 0, s>>>(dx, grad_[g[k]], nin);
      return cudaGetLastError();
    }
    case OpKind::kEltwise: {  // eltwise_layer.cpp Backward_cpu, bottom by bottom
      const size_t nb = op.bottoms.size();
      const size_t bytes = static_cast<size_t>(nin) * sizeof(float);
      for (size_t b = 0; b < nb; ++b) {
        if (!op.bottom_grad[b]) continue;
        float* db = grad_[op.bottoms[b]];
        cudaError_t e = cudaSuccess;
        if (op.eltwise_op == kEltwiseSum) {
          if (op.coeffs[b] == 1.f) e = cudaMemcpyAsync(db, dy, bytes, cudaMemcpyDeviceToDevice, s);
          else scale_copy_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, op.coeffs[b], db, nin);
        } else if (op.eltwise_op == kEltwiseMax) {
          eltwise_max_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, static_cast<const int*>(op_aux_[i]),
                                                                         static_cast<int>(b), db, nin);
        } else if (op.stable_prod_grad) {  // the product of the other bottoms in bottom order, then times dy
          bool first = true;
          for (size_t j = 0; j < nb && e == cudaSuccess; ++j) {
            if (j == b) continue;
            if (first) e = cudaMemcpyAsync(db, act_[op.bottoms[j]], bytes, cudaMemcpyDeviceToDevice, s);
            else mul_kernel<<<grid_for(nin), kThreads, 0, s>>>(act_[op.bottoms[j]], db, db, nin);
            first = false;
          }
          if (e == cudaSuccess) mul_kernel<<<grid_for(nin), kThreads, 0, s>>>(db, dy, db, nin);
        } else {
          prod_div_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(act_[op.out], act_[op.bottoms[b]], dy, db, nin);
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) return e;
      }
      return cudaSuccess;
    }
    case OpKind::kScale: {
      const int outer = static_cast<int>(op.scale_outer), dim = static_cast<int>(op.scale_dim);
      const int inner = static_cast<int>(op.scale_inner);
      scale_grad_kernel<<<dim, kThreads, 0, s>>>(dy, x, outer, dim, inner, diff_ + op.w_off);
      if (op.b_off >= 0) bias_grad_kernel<<<dim, kThreads, 0, s>>>(dy, outer, dim, inner, diff_ + op.b_off);
      if (dx) scale_forward_kernel<<<grid_for(nin), kThreads, 0, s>>>(dy, data_ + op.w_off, nullptr, dx, nin, dim, inner);
      return cudaGetLastError();
    }
    case OpKind::kTanH:
      if (dx) tanh_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(act_[op.out], dy, dx, nin);
      return cudaGetLastError();
    case OpKind::kELU:
      if (dx) elu_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, act_[op.out], dy, dx, nin, op.alpha);
      return cudaGetLastError();
    case OpKind::kAbsVal:
      if (dx) absval_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, dy, dx, nin);
      return cudaGetLastError();
    case OpKind::kBNLL:
      if (dx) bnll_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, dy, dx, nin);
      return cudaGetLastError();
    case OpKind::kPower: {  // the products of diff_scale are float, as Caffe forms them
      const float ds = op.power * op.scale;
      if (dx)
        power_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, act_[op.out], dy, dx, nin, op.power, op.scale,
                                                                 op.shift, ds, ds * op.scale, ds * op.shift);
      return cudaGetLastError();
    }
    case OpKind::kExp:
      if (dx) exp_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(act_[op.out], dy, dx, nin, op.inner_scale);
      return cudaGetLastError();
    case OpKind::kLog:
      if (dx)
        log_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, dy, dx, nin, op.scale, op.shift,
                                                               op.backward_num_scale);
      return cudaGetLastError();
    case OpKind::kThreshold:  // build_plan refuses a Threshold whose bottom would need a gradient
      return dx ? cudaErrorInvalidValue : cudaSuccess;
    case OpKind::kPReLU: {  // the slope gradient first, then the data gradient (prelu_layer.cpp's order)
      const int C = static_cast<int>(op.prelu_channels), dim = static_cast<int>(op.prelu_dim);
      const int chunks = prelu_chunks(op), slopes = prelu_slopes(op);
      prelu_slope_partial_kernel<<<dim3(chunks, slopes), kThreads, 0, s>>>(x, dy, workspace_, prelu_span(op), C, dim,
                                                                           op.channel_shared, chunks);
      prelu_slope_total_kernel<<<grid_for(slopes), kThreads, 0, s>>>(workspace_, chunks, slopes, diff_ + op.w_off);
      if (dx)
        prelu_backward_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, data_ + op.w_off, dy, dx, nin, C, dim,
                                                                 op.channel_shared);
      return cudaGetLastError();
    }
    case OpKind::kSoftmax:
      if (dx)
        softmax_backward_kernel<<<grid_for(op.outer * op.inner), kThreads, 0, s>>>(
            act_[op.out], dy, dx, static_cast<int>(op.outer * op.inner), static_cast<int>(op.classes),
            static_cast<int>(op.inner));
      return cudaGetLastError();
    case OpKind::kSoftmaxLoss:  // the loss kernels wrote their bottoms' gradients in the forward pass
    case OpKind::kContrastiveLoss:
    case OpKind::kEuclideanLoss:
    case OpKind::kSigmoidCrossEntropyLoss:
    case OpKind::kMultinomialLogisticLoss:
    case OpKind::kHingeLoss:
    case OpKind::kFlatten:  // the top's gradient is the bottom's memory
    case OpKind::kReshape:
      return cudaSuccess;
    case OpKind::kEmbed: {  // build_plan refuses an Embed whose ids would need a gradient
      const int N = static_cast<int>(op.out_shape.back()), K = static_cast<int>(op.input_dim);
      int* group = reinterpret_cast<int*>(workspace_);  // counts, then offsets, then group ends: K + 1 ints
      int* order = group + K + 1;
      cudaError_t e = cudaMemsetAsync(group, 0, (static_cast<size_t>(K) + 1) * sizeof(int), s);
      if (e != cudaSuccess) return e;
      embed_count_kernel<<<grid_for(nin), kThreads, 0, s>>>(x, nin, K, group);
      exclusive_scan_kernel<<<1, kEmbedBlock, 0, s>>>(group, K + 1);
      embed_place_kernel<<<1, kEmbedBlock, 0, s>>>(x, nin, K, group, order);
      const int threads = N >= kThreads ? kThreads : (N + 31) / 32 * 32;
      embed_weight_grad_kernel<<<std::min(nin, kTargetSms * 16), threads, 0, s>>>(x, order, group, dy,
                                                                                  diff_ + op.w_off, N, K);
      if (op.b_off >= 0) bias_grad_kernel<<<N, kThreads, 0, s>>>(dy, nin, N, 1, diff_ + op.b_off);
      return cudaGetLastError();
    }
    case OpKind::kRNN: {  // backpropagation through time inside this call; nothing crosses into the previous one
      const RnnDims d = rnn_dims(op, plan_.tensor_count);
      const RnnBuffers& b = rnn_[i];
      const float* cont = act_[op.bottoms[1]];
      const float* whh = data_ + op.rnn_off[Op::kWhh];
      const size_t step = static_cast<size_t>(d.N) * d.H;
      const int TN = d.T * d.N;
      // the weight gradient C[M, N] = A B over K products, split in fixed chunks and added once into dst
      auto weight_grad = [&](auto ga, auto gb, int M, int N, int K, float* dst) {
        cudaError_t e = gemm(ga, gb, StorePartial{workspace_, M, N}, M, N, K, split_chunk(K), s);
        if (e != cudaSuccess) return e;
        reduce_partials_kernel<<<grid_for(static_cast<int64_t>(M) * N), kThreads, 0, s>>>(workspace_, splits_of(K),
                                                                                          M * N, dst);
        return cudaGetLastError();
      };
      // the output: dzo = dtop (1 - top^2), then W_ho, b_o and dho over every step
      tanh_backward_kernel<<<grid_for(static_cast<int64_t>(TN) * d.H), kThreads, 0, s>>>(act_[op.out], dy, b.dzo,
                                                                                        TN * d.H);
      cudaError_t e = cudaGetLastError();
      if (e == cudaSuccess)
        e = weight_grad(DenseCM{b.dzo, d.H}, DenseRM{b.h + step, d.H}, d.H, d.H, TN, diff_ + op.rnn_off[Op::kWho]);
      if (e != cudaSuccess) return e;
      bias_grad_kernel<<<d.H, kThreads, 0, s>>>(b.dzo, TN, d.H, 1, diff_ + op.rnn_off[Op::kBo]);
      if ((e = cudaGetLastError()) != cudaSuccess) return e;
      e = gemm(DenseRM{b.dzo, d.H}, DenseRM{data_ + op.rnn_off[Op::kWho], d.H},
               RnnOutGrad{b.dho, b.dpre, b.h + step, d.H, (d.T - 1) * d.N}, TN, d.H, d.H, d.H, s);
      // one launch per step, t = T-1 .. 1: dpre_{t-1} from dpre_t (step 0's gradient at h_{-1} is not needed)
      for (int t = d.T - 1; t >= 1 && e == cudaSuccess; --t)
        e = gemm(DenseRM{b.dpre + t * step, d.H}, DenseRM{whh, d.H},
                 RnnBackStep{cont + static_cast<size_t>(t) * d.N, b.dho + (t - 1) * step, b.h + t * step,
                             b.dpre + (t - 1) * step, d.H},
                 d.N, d.H, d.H, d.H, s);
      // W_hh against hc_{t-1} = cont_t h_{t-1}, regathered; W_xh, b_h and dx over every step
      if (e == cudaSuccess)
        e = weight_grad(DenseCM{b.dpre, d.H}, ContGather{b.h, cont, d.H}, d.H, d.H, TN, diff_ + op.rnn_off[Op::kWhh]);
      if (e == cudaSuccess)
        e = weight_grad(DenseCM{b.dpre, d.H}, DenseRM{x, d.I}, d.H, d.I, TN, diff_ + op.rnn_off[Op::kWxh]);
      if (e != cudaSuccess) return e;
      bias_grad_kernel<<<d.H, kThreads, 0, s>>>(b.dpre, TN, d.H, 1, diff_ + op.rnn_off[Op::kBh]);
      if ((e = cudaGetLastError()) == cudaSuccess && dx)
        e = gemm(DenseRM{b.dpre, d.H}, DenseRM{data_ + op.rnn_off[Op::kWxh], d.I}, StoreRM{dx, nullptr, d.I}, TN, d.I,
                 d.H, d.H, s);
      if (e != cudaSuccess || !b.z) return e;
      // x_static: its transform is read by every step, so its gradient is dpre summed over t in step order
      sum_steps_kernel<<<grid_for(step), kThreads, 0, s>>>(b.dpre, d.T, static_cast<int>(step), b.dz);
      const float* xs = act_[op.bottoms[2]];
      if ((e = cudaGetLastError()) == cudaSuccess)
        e = weight_grad(DenseCM{b.dz, d.H}, DenseRM{xs, d.S}, d.H, d.S, d.N, diff_ + op.rnn_off[Op::kWxhStatic]);
      if (e == cudaSuccess && op.bottom_grad[2])
        e = gemm(DenseRM{b.dz, d.H}, DenseRM{data_ + op.rnn_off[Op::kWxhStatic], d.S},
                 StoreRM{grad_[op.bottoms[2]], nullptr, d.S}, d.N, d.S, d.H, d.H, s);
      return e;
    }
    default:
      return cudaErrorInvalidValue;
  }
}

}  // namespace cosb
