// native_producer.cu -- kernels and device side of the built-in gradient producer (DESIGN.md section 14).
//
// One fp32 GEMM core serves every convolution and inner product, forward and both backwards: a 64x64x16 shared-memory
// tile with FFMA and fp32 accumulation, templated on how it gathers its A and B operands and how it stores C.
// Convolutions are implicit GEMMs (the tile loader gathers im2col, or the transposed-convolution window for the data
// gradient, on the fly; no column buffer exists).  No TF32, no atomics: every output element is one thread's sum over
// k in increasing order, and weight gradients reduce over N*OH*OW in fixed chunks (split_chunk) whose partials a
// second kernel adds in chunk order.  Bias gradients are fixed-shape block reductions.  So a forward/backward is bitwise
// reproducible run to run.
#include <algorithm>
#include <cfloat>
#include <cmath>

#include "batch_norm.hpp"
#include "caffe_layers.hpp"
#include "fused_sync_sgd.hpp"
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

__global__ void accumulate_kernel(float* dst, const float* src, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dst[i] = __fadd_rn(dst[i], src[i]);
}

// ------------------------------------------------------------------ pooling (pooling_layer.cu semantics)
struct PoolGeom {
  int N, C, H, W, PH, PW, KH, KW, SH, SW, PADH, PADW;
};

__global__ void max_pool_forward_kernel(const float* x, float* y, int* idx, PoolGeom g) {
  const int total = g.N * g.C * g.PH * g.PW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int pw = i % g.PW, ph = (i / g.PW) % g.PH, nc = i / (g.PW * g.PH);
    int hs = ph * g.SH - g.PADH, ws = pw * g.SW - g.PADW;
    const int he = min(hs + g.KH, g.H), we = min(ws + g.KW, g.W);
    hs = max(hs, 0), ws = max(ws, 0);
    const float* plane = x + (size_t)nc * g.H * g.W;
    float m = -FLT_MAX;
    int mi = -1;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w)
        if (plane[h * g.W + w] > m) {  // the first maximum wins
          mi = h * g.W + w;
          m = plane[mi];
        }
    y[i] = m;
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
    const int size = ave_pool_size(ph, pw, g);
    int hs = ph * g.SH - g.PADH, ws = pw * g.SW - g.PADW;
    const int he = min(hs + g.KH, g.H), we = min(ws + g.KW, g.W);
    hs = max(hs, 0), ws = max(ws, 0);
    const float* plane = x + (size_t)nc * g.H * g.W;
    float s = 0.f;
    for (int h = hs; h < he; ++h)
      for (int w = ws; w < we; ++w) s = __fadd_rn(s, plane[h * g.W + w]);
    y[i] = __fdiv_rn(s, static_cast<float>(size));
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
__global__ void sigmoid_forward_kernel(const float* x, float* y, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    y[i] = __fadd_rn(__fmul_rn(0.5f, tanhf(__fmul_rn(0.5f, x[i]))), 0.5f);  // sigmoid_layer.cu
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

int grid_for(int64_t n) {
  const int64_t g = (n + kThreads - 1) / kThreads;
  return static_cast<int>(g < 1 ? 1 : (g > kTargetSms * 16 ? kTargetSms * 16 : g));
}

struct ConvDims {
  int N, Cin, H, W, Cout, OH, OW;
};
ConvDims conv_dims(const Op& op) {
  ConvDims d;
  d.N = static_cast<int>(op.in_shape[0]), d.Cin = static_cast<int>(op.in_shape[1]);
  d.H = static_cast<int>(op.in_shape[2]), d.W = static_cast<int>(op.in_shape[3]);
  d.Cout = static_cast<int>(op.w_count / (static_cast<int64_t>(d.Cin) * op.kh * op.kw));
  d.OH = (d.H + 2 * op.ph - op.kh) / op.sh + 1;
  d.OW = (d.W + 2 * op.pw - op.kw) / op.sw + 1;
  return d;
}
ConvGeom geom(const ConvDims& d, const Op& op) {
  return ConvGeom{d.Cin, d.H, d.W, op.kh, op.kw, op.sh, op.sw, op.ph, op.pw, d.OH, d.OW};
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
int ip_k(const Op& op) { return static_cast<int>(op.w_count / (op.w_count > 0 ? op.out_shape[1] : 1)); }

// conv weight / bias gradients and the data gradient, from dy = the conv output's gradient
cudaError_t conv_backward(const Op& op, const float* x, const float* dy, float* dx, const float* w, float* diff,
                          float* ws, bool bias_grad, cudaStream_t s) {
  const ConvDims d = conv_dims(op);
  const int K = d.N * d.OH * d.OW, KW = d.Cin * op.kh * op.kw;
  cudaError_t e = gemm(ChanMajor{dy, d.Cout, d.OH * d.OW}, Transposed<Im2col>{Im2col{x, geom(d, op)}},
                       StorePartial{ws, d.Cout, KW}, d.Cout, KW, K, split_chunk(K), s);
  if (e != cudaSuccess) return e;
  reduce_partials_kernel<<<grid_for(op.w_count), kThreads, 0, s>>>(ws, splits_of(K), static_cast<int>(op.w_count),
                                                                     diff + op.w_off);
  if (bias_grad) bias_grad_kernel<<<d.Cout, kThreads, 0, s>>>(dy, d.N, d.Cout, d.OH * d.OW, diff + op.b_off);
  if (dx) {
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int KD = d.Cout * op.kh * op.kw;
    return gemm(WeightT{w, d.Cin, op.kh * op.kw},
                Col2imGather{dy, d.Cout, d.H, d.W, op.kh, op.kw, op.sh, op.sw, op.ph, op.pw, d.OH, d.OW},
                StoreNCHW{dx, nullptr, d.Cin, d.H * d.W}, d.Cin, d.N * d.H * d.W, KD, KD, s);
  }
  return cudaGetLastError();
}

}  // namespace

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
  size_t ws = 1;
  for (size_t i = 0; i < plan_.ops.size(); ++i) {
    const Op& op = plan_.ops[i];
    const int64_t out = plan_.tensor_count[op.out];
    if (op.kind == OpKind::kConv || op.kind == OpKind::kConvBiasReluMaxPool) {
      const ConvDims d = conv_dims(op);
      const size_t K = static_cast<size_t>(d.N) * d.OH * d.OW;
      ws = std::max(ws, static_cast<size_t>(splits_of(static_cast<int>(K))) * op.w_count);
      if (op.kind == OpKind::kConvBiasReluMaxPool) {
        const size_t zb = static_cast<size_t>(d.N) * d.Cout * d.OH * d.OW * sizeof(float);
        void *z, *dz, *idx;
        if (!alloc(zb, &z) || !alloc(zb, &dz) || !alloc(out, &idx)) return false;
        op_z_[i] = static_cast<float*>(z), op_dz_[i] = static_cast<float*>(dz), op_aux_[i] = idx;
        ws = std::max(ws, static_cast<size_t>(d.N + 1) * d.Cout);  // bias partials + dbias
      }
    } else if ((op.kind == OpKind::kPool && op.max_pool) ||
               (op.kind == OpKind::kEltwise && op.eltwise_op == kEltwiseMax)) {
      if (!alloc(out * sizeof(int), &op_aux_[i])) return false;
    } else if (op.kind == OpKind::kInnerProduct) {
      ws = std::max(ws, static_cast<size_t>(splits_of(static_cast<int>(op.in_shape[0]))) * op.w_count);
    } else if (op.kind == OpKind::kBatchNorm) {
      int n, c, hw;
      bn_dims(op, &n, &c, &hw);
      if (!alloc(2 * static_cast<size_t>(c) * sizeof(float), &op_aux_[i])) return false;
      ws = std::max(ws, bn_workspace_floats(n, c));
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
      const int K = d.Cin * op.kh * op.kw;
      const bool fused = op.kind == OpKind::kConvBiasReluMaxPool;
      const float* bias = (!fused && op.b_off >= 0) ? data_ + op.b_off : nullptr;
      float* z = fused ? op_z_[i] : y;
      cudaError_t e = gemm(DenseRM{data_ + op.w_off, K}, Im2col{x, geom(d, op)}, StoreNCHW{z, bias, d.Cout, d.OH * d.OW},
                           d.Cout, d.N * d.OH * d.OW, K, K, s);
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
      const int B = static_cast<int>(op.in_shape[0]), N = static_cast<int>(op.out_shape[1]), K = ip_k(op);
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
    case OpKind::kSplit:  // no copy: the top reads the bottom's memory
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
    default:
      return cudaErrorInvalidValue;
  }
}

cudaError_t NativeProducer::run_op_backward(const Op& op, size_t i, cudaStream_t s) {
  const float* x = act_[op.bottoms[0]];
  const float* dy = grad_[op.out];
  float* dx = op.bottom_grad[0] ? grad_[op.bottoms[0]] : nullptr;
  const int nin = static_cast<int>(plan_.tensor_count[op.bottoms[0]]);
  switch (op.kind) {
    case OpKind::kConv:
      return conv_backward(op, x, dy, dx, data_ + op.w_off, diff_, workspace_, op.b_off >= 0, s);
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
      const int B = static_cast<int>(op.in_shape[0]), N = static_cast<int>(op.out_shape[1]), K = ip_k(op);
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
    case OpKind::kSoftmaxLoss:  // the loss kernels wrote their bottoms' gradients in the forward pass
    case OpKind::kContrastiveLoss:
    case OpKind::kEuclideanLoss:
      return cudaSuccess;
    default:
      return cudaErrorInvalidValue;
  }
}

}  // namespace cosb
