// mvn.cu -- Caffe's MVN layer on sm_90a: deterministic row statistics, forward and backward (mvn.hpp).
//
// Every element operation is the __f*_rn intrinsic of the one rounding Caffe's Forward_gpu / Backward_gpu gives it
// (no contraction into FMA), and powf(var, 0.5) is glibc's, as BatchNorm computes it (powf_half.h).  A group of G
// threads sums its row (or chunk) with each thread striding by G in element order, then a butterfly over the warp's
// lanes and, for a block, the warps' sums in warp order: all fixed by (rows, dim).
//
// Traffic: the row-local kernels read a row once per sum and once more to write (x three times in the forward with
// normalize_variance, y and dy twice in the backward); the re-reads of a row just read hit L1 or L2.  A split row is
// read by three kernels in the forward (sum, squared deviations, write) and two in the backward.
#include "mvn.hpp"

#include "powf_half.h"

namespace cosb {
namespace {

constexpr int kBlock = 256;

// the sum of v over the G threads of a group (G <= 32: aligned lanes of a warp; G == kBlock: the block), returned to
// every thread of the group.  A butterfly adds the same two operands on both sides, so all lanes agree bit for bit.
template <int G>
__device__ __forceinline__ float group_sum(float v, float* red) {
#pragma unroll
  for (int o = (G < 32 ? G : 32) / 2; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (G <= 32) return v;
  __syncthreads();  // red may still be read by an earlier call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = red[0];
#pragma unroll
  for (int w = 1; w < G / 32; ++w) t = __fadd_rn(t, red[w]);
  return t;
}

__device__ __forceinline__ float mvn_std(float syy, float alpha, float eps) {
  return __fadd_rn(cos_powf_half(__fmul_rn(syy, alpha)), eps);
}

// Row-local forward: group g of G threads owns row g.  A row-local dim is below 2^21 (mvn_regime splits longer rows
// unless rows >= kMvnSplitMaxRows, and rows * dim < 2^31), so `i += G` cannot overflow.
template <int G>
__global__ void __launch_bounds__(kBlock) mvn_forward_rows_kernel(const float* x, float* y, float* stats, int64_t rows,
                                                                  int dim, float alpha, float eps, bool variance) {
  __shared__ float red[kBlock / 32];
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x) / G;
  const int lane = threadIdx.x % G;
  const bool live = row < rows;  // a dead group still joins the shuffles
  const float* xr = x + (live ? row : 0) * dim;
  float sx = 0.f;
  if (live)
    for (int i = lane; i < dim; i += G) sx = __fadd_rn(sx, xr[i]);
  sx = group_sum<G>(sx, red);
  const float mu = __fmul_rn(sx, alpha);
  float syy = 0.f, sd = 1.f;
  if (variance) {
    if (live)
      for (int i = lane; i < dim; i += G) {
        const float d = __fsub_rn(xr[i], mu);
        syy = __fadd_rn(syy, __fmul_rn(d, d));
      }
    syy = group_sum<G>(syy, red);
    sd = mvn_std(syy, alpha, eps);
  }
  if (!live) return;
  float* yr = y + row * dim;
  for (int i = lane; i < dim; i += G) {
    const float d = __fsub_rn(xr[i], mu);
    yr[i] = variance ? __fdiv_rn(d, sd) : d;
  }
  if (lane == 0) stats[row] = sx, stats[rows + row] = syy, stats[2 * rows + row] = sd;
}

__device__ __forceinline__ float mvn_dx(float yv, float g, float a, float b, float c, float sd, float m, bool variance) {
  return variance ? __fdiv_rn(__fadd_rn(g, __fmul_rn(c, __fadd_rn(__fmul_rn(yv, a), b))), sd) : __fsub_rn(g, m);
}

template <int G>
__global__ void __launch_bounds__(kBlock) mvn_backward_rows_kernel(const float* y, const float* dy, float* dx,
                                                                   float* stats, int64_t rows, int dim, float alpha,
                                                                   float c, bool variance) {
  __shared__ float red[kBlock / 32];
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x) / G;
  const int lane = threadIdx.x % G;
  const bool live = row < rows;
  const int64_t base = (live ? row : 0) * dim;
  float a = 0.f, b = 0.f;
  if (live)
    for (int i = lane; i < dim; i += G) {
      const float g = dy[base + i];
      if (variance) a = __fadd_rn(a, __fmul_rn(y[base + i], g));
      b = __fadd_rn(b, g);
    }
  if (variance) a = group_sum<G>(a, red);
  b = group_sum<G>(b, red);
  if (!live) return;
  const float sd = stats[2 * rows + row], m = __fmul_rn(b, alpha);
  for (int i = lane; i < dim; i += G) dx[base + i] = mvn_dx(y[base + i], dy[base + i], a, b, c, sd, m, variance);
  if (lane == 0) stats[3 * rows + row] = a, stats[4 * rows + row] = b;
}

// The row's chunk partials part[0 .. chunks) added in chunk order, returned to every thread of the block.
__device__ float chunk_total(const float* part, int chunks, float* sh) {
  __syncthreads();  // sh may still be read by an earlier call
  for (int k = threadIdx.x; k < chunks; k += kBlock) sh[k] = part[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = sh[0];
    for (int k = 1; k < chunks; ++k) t = __fadd_rn(t, sh[k]);
    sh[kMvnMaxChunks] = t;
  }
  __syncthreads();
  return sh[kMvnMaxChunks];
}

// Split rows, grid (chunks, rows): the sums of one chunk.  kPass 0: Sx into pa.  1: Syy into pb (mu from pa's
// totals).  2: A into pa and B into pb.  3: B into pb.
template <int kPass>
__global__ void __launch_bounds__(kBlock) mvn_chunk_sums_kernel(const float* u, const float* v, float* pa, float* pb,
                                                                int dim, int chunk, int chunks, float alpha) {
  __shared__ float red[kBlock / 32];
  __shared__ float sh[kMvnMaxChunks + 1];
  const int64_t row = blockIdx.y, first = row * chunks;
  const int begin = blockIdx.x * chunk, n = static_cast<int>(min(static_cast<int64_t>(dim) - begin, int64_t(chunk)));
  const float* ur = u + row * dim;
  const float* vr = v ? v + row * dim : nullptr;
  const float mu = kPass == 1 ? __fmul_rn(chunk_total(pa + first, chunks, sh), alpha) : 0.f;
  float s1 = 0.f, s2 = 0.f;
  for (int k = threadIdx.x; k < n; k += kBlock) {
    const int i = begin + k;
    if (kPass == 0) s1 = __fadd_rn(s1, ur[i]);
    if (kPass == 1) {
      const float d = __fsub_rn(ur[i], mu);
      s2 = __fadd_rn(s2, __fmul_rn(d, d));
    }
    if (kPass == 2) s1 = __fadd_rn(s1, __fmul_rn(ur[i], vr[i]));
    if (kPass >= 2) s2 = __fadd_rn(s2, vr[i]);
  }
  if (kPass == 0 || kPass == 2) s1 = group_sum<kBlock>(s1, red);
  if (kPass >= 1) s2 = group_sum<kBlock>(s2, red);
  if (threadIdx.x != 0) return;
  if (kPass == 0 || kPass == 2) pa[first + blockIdx.x] = s1;
  if (kPass >= 1) pb[first + blockIdx.x] = s2;
}

__global__ void __launch_bounds__(kBlock) mvn_chunk_forward_kernel(const float* x, float* y, float* stats,
                                                                   const float* pa, const float* pb, int64_t rows,
                                                                   int dim, int chunk, int chunks, float alpha,
                                                                   float eps, bool variance) {
  __shared__ float sh[kMvnMaxChunks + 1];
  const int64_t row = blockIdx.y, first = row * chunks;
  const int begin = blockIdx.x * chunk, n = static_cast<int>(min(static_cast<int64_t>(dim) - begin, int64_t(chunk)));
  const float sx = chunk_total(pa + first, chunks, sh), mu = __fmul_rn(sx, alpha);
  const float syy = variance ? chunk_total(pb + first, chunks, sh) : 0.f;
  const float sd = variance ? mvn_std(syy, alpha, eps) : 1.f;
  const int64_t base = row * dim;
  for (int k = threadIdx.x; k < n; k += kBlock) {
    const int i = begin + k;
    const float d = __fsub_rn(x[base + i], mu);
    y[base + i] = variance ? __fdiv_rn(d, sd) : d;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) stats[row] = sx, stats[rows + row] = syy, stats[2 * rows + row] = sd;
}

__global__ void __launch_bounds__(kBlock) mvn_chunk_backward_kernel(const float* y, const float* dy, float* dx,
                                                                    float* stats, const float* pa, const float* pb,
                                                                    int64_t rows, int dim, int chunk, int chunks,
                                                                    float alpha, float c, bool variance) {
  __shared__ float sh[kMvnMaxChunks + 1];
  const int64_t row = blockIdx.y, first = row * chunks;
  const int begin = blockIdx.x * chunk, n = static_cast<int>(min(static_cast<int64_t>(dim) - begin, int64_t(chunk)));
  const float a = variance ? chunk_total(pa + first, chunks, sh) : 0.f;
  const float b = chunk_total(pb + first, chunks, sh);
  const float sd = stats[2 * rows + row], m = __fmul_rn(b, alpha);
  const int64_t base = row * dim;
  for (int k = threadIdx.x; k < n; k += kBlock) {
    const int i = begin + k;
    dx[base + i] = mvn_dx(y[base + i], dy[base + i], a, b, c, sd, m, variance);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) stats[3 * rows + row] = a, stats[4 * rows + row] = b;
}

int lanes(int64_t dim) {  // next_pow2(dim) for the lanes regime, 32 for a warp, kBlock for a block
  const MvnRegime r = mvn_regime(1, dim);
  if (r == MvnRegime::kWarp) return 32;
  if (r != MvnRegime::kLanes) return kBlock;
  int g = 1;
  while (g < dim) g <<= 1;
  return g;
}

template <int G>
void rows_forward(const float* x, float* y, float* stats, int64_t rows, int dim, float alpha, float eps, bool var,
                  cudaStream_t s) {
  const int64_t blocks = (rows * G + kBlock - 1) / kBlock;
  mvn_forward_rows_kernel<G><<<static_cast<unsigned>(blocks), kBlock, 0, s>>>(x, y, stats, rows, dim, alpha, eps, var);
}
template <int G>
void rows_backward(const float* y, const float* dy, float* dx, float* stats, int64_t rows, int dim, float alpha,
                   float c, bool var, cudaStream_t s) {
  const int64_t blocks = (rows * G + kBlock - 1) / kBlock;
  mvn_backward_rows_kernel<G><<<static_cast<unsigned>(blocks), kBlock, 0, s>>>(y, dy, dx, stats, rows, dim, alpha, c,
                                                                               var);
}

// one launch of F<G> for the group size G of (rows, dim)
template <template <int> class F, typename... Args>
void by_lanes(int g, Args... args) {
  switch (g) {
    case 1: F<1>::run(args...); break;
    case 2: F<2>::run(args...); break;
    case 4: F<4>::run(args...); break;
    case 8: F<8>::run(args...); break;
    case 16: F<16>::run(args...); break;
    case 32: F<32>::run(args...); break;
    default: F<kBlock>::run(args...); break;
  }
}
template <int G>
struct Forward {
  template <typename... Args>
  static void run(Args... args) { rows_forward<G>(args...); }
};
template <int G>
struct Backward {
  template <typename... Args>
  static void run(Args... args) { rows_backward<G>(args...); }
};

}  // namespace

MvnRegime mvn_regime(int64_t rows, int64_t dim) {
  if (dim <= kMvnLanesMaxDim) return MvnRegime::kLanes;
  if (dim <= kMvnWarpMaxDim) return MvnRegime::kWarp;
  if (dim >= kMvnSplitMinDim && rows < kMvnSplitMaxRows) return MvnRegime::kSplit;
  return MvnRegime::kBlock;
}

void mvn_chunks(int64_t rows, int64_t dim, int64_t* chunk, int64_t* chunks) {
  if (mvn_regime(rows, dim) != MvnRegime::kSplit) {
    *chunk = dim, *chunks = 1;
    return;
  }
  const int64_t least = (dim + kMvnMaxChunks - 1) / kMvnMaxChunks;  // at most kMvnMaxChunks chunks
  *chunk = least <= kMvnChunk ? kMvnChunk : (least + kBlock - 1) / kBlock * kBlock;
  *chunks = (dim + *chunk - 1) / *chunk;
}

size_t mvn_workspace_floats(int64_t rows, int64_t dim) {
  int64_t chunk, chunks;
  mvn_chunks(rows, dim, &chunk, &chunks);
  return mvn_regime(rows, dim) == MvnRegime::kSplit ? static_cast<size_t>(2 * rows * chunks) : 0;
}

cudaError_t mvn_forward(const float* x, float* y, float* stats, float* workspace, int64_t rows, int64_t dim,
                        bool variance, float eps, cudaStream_t s) {
  const float alpha = static_cast<float>(1.0 / static_cast<double>(dim));
  const int d = static_cast<int>(dim);
  if (mvn_regime(rows, dim) != MvnRegime::kSplit) {
    by_lanes<Forward>(lanes(dim), x, y, stats, rows, d, alpha, eps, variance, s);
    return cudaGetLastError();
  }
  int64_t chunk, chunks;
  mvn_chunks(rows, dim, &chunk, &chunks);
  float *pa = workspace, *pb = workspace + rows * chunks;
  const dim3 grid(static_cast<unsigned>(chunks), static_cast<unsigned>(rows));
  const int c = static_cast<int>(chunk), n = static_cast<int>(chunks);
  mvn_chunk_sums_kernel<0><<<grid, kBlock, 0, s>>>(x, nullptr, pa, pb, d, c, n, alpha);
  if (variance) mvn_chunk_sums_kernel<1><<<grid, kBlock, 0, s>>>(x, nullptr, pa, pb, d, c, n, alpha);
  mvn_chunk_forward_kernel<<<grid, kBlock, 0, s>>>(x, y, stats, pa, pb, rows, d, c, n, alpha, eps, variance);
  return cudaGetLastError();
}

cudaError_t mvn_backward(const float* y, const float* dy, float* dx, float* stats, float* workspace, int64_t rows,
                         int64_t dim, bool variance, cudaStream_t s) {
  const float alpha = static_cast<float>(1.0 / static_cast<double>(dim));
  const float c = static_cast<float>(-1.0 / static_cast<double>(dim));
  const int d = static_cast<int>(dim);
  if (mvn_regime(rows, dim) != MvnRegime::kSplit) {
    by_lanes<Backward>(lanes(dim), y, dy, dx, stats, rows, d, alpha, c, variance, s);
    return cudaGetLastError();
  }
  int64_t chunk, chunks;
  mvn_chunks(rows, dim, &chunk, &chunks);
  float *pa = workspace, *pb = workspace + rows * chunks;
  const dim3 grid(static_cast<unsigned>(chunks), static_cast<unsigned>(rows));
  const int ch = static_cast<int>(chunk), n = static_cast<int>(chunks);
  if (variance)
    mvn_chunk_sums_kernel<2><<<grid, kBlock, 0, s>>>(y, dy, pa, pb, d, ch, n, alpha);
  else
    mvn_chunk_sums_kernel<3><<<grid, kBlock, 0, s>>>(y, dy, pa, pb, d, ch, n, alpha);
  mvn_chunk_backward_kernel<<<grid, kBlock, 0, s>>>(y, dy, dx, stats, pa, pb, rows, d, ch, n, alpha, c, variance);
  return cudaGetLastError();
}

}  // namespace cosb
