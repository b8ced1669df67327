// conv_tf32.cu -- implicit-GEMM convolutions on sm_90a TF32 tensor cores (conv_tf32.hpp, DESIGN.md section 10.2).
//
// One mainloop serves the three passes: a BM x BN block tile, BK = 16 deep k-tiles, a STAGES-deep cp.async ring in
// shared memory and 64 x 32 warp tiles of mma.sync.m16n8k8 TF32 with fp32 accumulators.  The passes differ only in
// their tile loaders, which gather each element straight from the NCHW tensors with a 4-byte cp.async (zero-filled
// outside the tensor, the GEMM or the window), and in where the epilogue stores.  A loader's lanes run along the
// operand's contiguous axis in global memory: the pixel axis of a window gather (A of the forward and the data
// gradient, stored pixel-major in shared memory), the tap axis of a weight row or the pixel axis of the weight
// gradient's operands (stored k-major).  The window taps (c or filter, r, s) are decoded once per block into a
// shared-memory table, so the per-element work is a table read, two bounds tests and an address.
#include "conv_tf32.hpp"

#include <algorithm>

namespace cosb {
namespace {

constexpr int BK = 16, STAGES = 4, WM = 64, WN = 32, MT = WM / 16, NT = WN / 8;
constexpr int kTapSeg = 3584;          // taps per shared-memory table segment (28 KB of int2), a multiple of BK
constexpr int kFilterTargetBlocks = 1024;  // backward_filter splits its reduction until about this many blocks run
constexpr int kFilterMinKTiles = 8;    // ... but gives every chunk at least this many k-tiles

// operand tile of BX rows (M or N) by BK taps in shared memory: k-major [BX][BK + 4] or x-major [BK][BX + 8]; both
// paddings make the mma fragment reads conflict-free
template <bool KMAJ, int BX>
struct Tile {
  static constexpr int kFloats = KMAJ ? BX * (BK + 4) : BK * (BX + 8);
  __device__ __forceinline__ static int at(int x, int k) { return KMAJ ? x * (BK + 4) + k : k * (BX + 8) + x; }
};

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 4 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ uint32_t to_tf32(float f) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(f));
  return r;
}

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int BM, int BN>
struct Cfg {
  static constexpr int kThreads = (BM / WM) * (BN / WN) * 32;
};

template <int BM, int BN, bool AK, bool BKM>
__host__ __device__ constexpr size_t stage_bytes() {
  return sizeof(float) * STAGES * (Tile<AK, BM>::kFloats + Tile<BKM, BN>::kFloats);
}

// acc += A[., k] B[k, .] over the k-tiles [kt0, kt1); ld.load(As, Bs, kt) issues one k-tile's cp.asyncs.  Ends with
// a barrier, so the caller may rewrite shared memory afterwards.
template <int BM, int BN, bool AK, bool BKM, class Ld>
__device__ __forceinline__ void mainloop(Ld& ld, int kt0, int kt1, float* smem, float (&acc)[MT][NT][4]) {
  using TA = Tile<AK, BM>;
  using TB = Tile<BKM, BN>;
  float* As = smem;
  float* Bs = smem + STAGES * TA::kFloats;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wm = (warp % (BM / WM)) * WM, wn = (warp / (BM / WM)) * WN;
  const int gr = lane >> 2, tg = lane & 3;
  const int nkt = kt1 - kt0;
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) ld.load(As + s * TA::kFloats, Bs + s * TB::kFloats, kt0 + s);
    cp_async_commit();
  }
  for (int i = 0; i < nkt; ++i) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();  // k-tile i has landed for every thread, and slot (i - 1) % STAGES is free again
    const int nx = i + STAGES - 1;
    if (nx < nkt) ld.load(As + (nx % STAGES) * TA::kFloats, Bs + (nx % STAGES) * TB::kFloats, kt0 + nx);
    cp_async_commit();
    const float* a = As + (i % STAGES) * TA::kFloats;
    const float* b = Bs + (i % STAGES) * TB::kFloats;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 8) {
      uint32_t af[MT][4], bf[NT][2];
#pragma unroll
      for (int mi = 0; mi < MT; ++mi) {
        const int m = wm + mi * 16 + gr;
        af[mi][0] = to_tf32(a[TA::at(m, kk + tg)]);
        af[mi][1] = to_tf32(a[TA::at(m + 8, kk + tg)]);
        af[mi][2] = to_tf32(a[TA::at(m, kk + tg + 4)]);
        af[mi][3] = to_tf32(a[TA::at(m + 8, kk + tg + 4)]);
      }
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int n = wn + ni * 8 + gr;
        bf[ni][0] = to_tf32(b[TB::at(n, kk + tg)]);
        bf[ni][1] = to_tf32(b[TB::at(n, kk + tg + 4)]);
      }
#pragma unroll
      for (int mi = 0; mi < MT; ++mi)
#pragma unroll
        for (int ni = 0; ni < NT; ++ni) mma_tf32(acc[mi][ni], af[mi], bf[ni]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();
}

// stores the block's accumulators: C[m, n] goes to out[row(m) + n * col_stride] for m < M, n < N (+ bias[n])
template <int BM, int BN, class Row>
__device__ __forceinline__ void epilogue(const float (&acc)[MT][NT][4], float* out, int m0, int n0, int M, int N,
                                         long long col_stride, const float* bias, Row row) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wm = (warp % (BM / WM)) * WM, wn = (warp / (BM / WM)) * WN;
  const int gr = lane >> 2, tg = lane & 3;
#pragma unroll
  for (int mi = 0; mi < MT; ++mi)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int m = m0 + wm + mi * 16 + gr + 8 * hf;
      if (m >= M) continue;
      float* o = out + row(m);
#pragma unroll
      for (int ni = 0; ni < NT; ++ni)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = n0 + wn + ni * 8 + 2 * tg + j;
          if (n < N) o[n * col_stride] = acc[mi][ni][2 * hf + j] + (bias ? bias[n] : 0.f);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- forward
// A[m, k] = x[img, g·Cg + c, p·sh − ph + r, q·sw − pw + s]  (m = (img, p, q), k = (c, r, s)), pixel-major tile
// B[k, n] = w[g·Kg + n, c, r, s]                              k-major tile
template <int BM, int BN>
struct FwdLoad {
  static constexpr int T = Cfg<BM, BN>::kThreads;
  const float* x;
  const float* w;
  const int2* taps;  // taps [seg0, seg0 + kTapSeg): {c·H·W + r·W + s, r << 16 | s}
  int seg0, Kt, H, W;
  int xoff, h0, w0;  // this thread's A pixel: x offset of (img, g·Cg, h0, w0)
  bool mval;
  int akin;                 // this thread's first A tap row in the tile
  const float* wrow;        // this thread's first B filter row (k = 0)
  int bkin, brows;          // this thread's B tap column, and how many of its B rows are filters (< Kg)

  __device__ __forceinline__ void load(float* As, float* Bs, int kt) {
    constexpr int AE = BK * BM / T, BE = BK * BN / T;
#pragma unroll
    for (int i = 0; i < AE; ++i) {
      const int kin = akin + i * (T / BM), k = kt * BK + kin;
      bool v = mval && k < Kt;
      int off = 0;
      if (v) {
        const int2 t = taps[k - seg0];
        const int ih = h0 + (t.y >> 16), iw = w0 + (t.y & 0xffff);
        v = static_cast<unsigned>(ih) < static_cast<unsigned>(H) && static_cast<unsigned>(iw) < static_cast<unsigned>(W);
        off = xoff + t.x;
      }
      cp_async4(As + Tile<false, BM>::at(threadIdx.x % BM, kin), x + (v ? off : 0), v);
    }
    const int k = kt * BK + bkin;
#pragma unroll
    for (int i = 0; i < BE; ++i) {
      const bool v = i < brows && k < Kt;
      cp_async4(Bs + Tile<true, BN>::at(threadIdx.x / BK + i * (T / BK), bkin),
                v ? wrow + static_cast<long long>(i) * (T / BK) * Kt + k : w, v);
    }
  }
};

template <int BM, int BN>
__global__ void __launch_bounds__(Cfg<BM, BN>::kThreads, 2)
    conv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ y, ConvGeom g) {
  constexpr int T = Cfg<BM, BN>::kThreads;
  extern __shared__ __align__(16) float smem[];
  int2* taps = reinterpret_cast<int2*>(smem + stage_bytes<BM, BN, false, true>() / sizeof(float));
  const int grp = blockIdx.z, m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int Cg = g.c / g.groups, Kg = g.k / g.groups, RS = g.r * g.s, HW = g.h * g.w, PQ = g.p * g.q;
  const int M = g.n * PQ, Kt = Cg * RS;

  FwdLoad<BM, BN> ld;
  ld.x = x;
  ld.w = w;
  ld.taps = taps;
  ld.Kt = Kt;
  ld.H = g.h;
  ld.W = g.w;
  {
    const int m = m0 + static_cast<int>(threadIdx.x) % BM;
    ld.mval = m < M;
    const int mm = ld.mval ? m : 0, img = mm / PQ, pq = mm - img * PQ, p = pq / g.q, q = pq - p * g.q;
    ld.h0 = p * g.stride_h - g.pad_h;
    ld.w0 = q * g.stride_w - g.pad_w;
    ld.xoff = (img * g.c + grp * Cg) * HW + ld.h0 * g.w + ld.w0;
    ld.akin = threadIdx.x / BM;
  }
  ld.bkin = threadIdx.x % BK;
  {
    const int n = n0 + threadIdx.x / BK;
    ld.brows = n < Kg ? (Kg - n + T / BK - 1) / (T / BK) : 0;
    ld.wrow = w + static_cast<long long>(grp * Kg + (n < Kg ? n : 0)) * Kt;
  }

  float acc[MT][NT][4] = {};
  for (int seg0 = 0; seg0 < Kt; seg0 += kTapSeg) {
    const int seg1 = min(Kt, seg0 + kTapSeg);
    for (int k = seg0 + threadIdx.x; k < seg1; k += T) {
      const int c = k / RS, rs = k - c * RS, r = rs / g.s, s = rs - r * g.s;
      taps[k - seg0] = make_int2(c * HW + r * g.w + s, r << 16 | s);
    }
    __syncthreads();
    ld.seg0 = seg0;
    mainloop<BM, BN, false, true>(ld, seg0 / BK, (seg1 + BK - 1) / BK, smem, acc);
  }
  const int K = g.k;
  epilogue<BM, BN>(acc, y, m0, n0, M, Kg, PQ, bias ? bias + grp * Kg : nullptr, [&](int m) {
    const int img = m / PQ;
    return static_cast<long long>(img * K + grp * Kg) * PQ + (m - img * PQ);
  });
}

// ---------------------------------------------------------------------------------------------- backward data
// A[m, k] = dy[img, g·Kg + f, (h + ph − r) / sh, (w + pw − s) / sw]  where both divisions are exact and in range
//           (m = (img, h, w) of dx, k = (f, r, s)), pixel-major tile
// B[k, n] = w[g·Kg + f, n, r, s]                                       k-major tile
template <int BM, int BN>
struct DataLoad {
  static constexpr int T = Cfg<BM, BN>::kThreads;
  const float* dy;
  const float* w;
  const int2* taps;  // {f·P·Q, r << 16 | s}
  int seg0, Kt, P, Q, sh, sw, RS, Cg, Kg, grp;
  int dyoff, hh0, ww0;  // this thread's A pixel: dy offset of (img, g·Kg), h + ph, w + pw
  bool mval;
  int akin, bkin, bn;  // bn: this thread's first B channel (relative to the group)

  __device__ __forceinline__ void load(float* As, float* Bs, int kt) {
    constexpr int AE = BK * BM / T, BE = BK * BN / T;
    const bool unit = (sh == 1) & (sw == 1);
#pragma unroll
    for (int i = 0; i < AE; ++i) {
      const int kin = akin + i * (T / BM), k = kt * BK + kin;
      bool v = mval && k < Kt;
      int off = 0;
      if (v) {
        const int2 t = taps[k - seg0];
        int p = hh0 - (t.y >> 16), q = ww0 - (t.y & 0xffff);
        if (!unit) {
          v = p >= 0 && q >= 0 && p % sh == 0 && q % sw == 0;
          p /= sh;
          q /= sw;
        }
        v = v && static_cast<unsigned>(p) < static_cast<unsigned>(P) &&
            static_cast<unsigned>(q) < static_cast<unsigned>(Q);
        off = dyoff + t.x + p * Q + q;
      }
      cp_async4(As + Tile<false, BM>::at(threadIdx.x % BM, kin), dy + (v ? off : 0), v);
    }
    const int k = kt * BK + bkin;
    const int f = k / RS, rs = k - f * RS;
    const long long base = static_cast<long long>(grp * Kg + f) * Cg * RS + rs;
#pragma unroll
    for (int i = 0; i < BE; ++i) {
      const int n = bn + i * (T / BK);
      const bool v = k < Kt && n < Cg;
      cp_async4(Bs + Tile<true, BN>::at(threadIdx.x / BK + i * (T / BK), bkin),
                v ? w + base + static_cast<long long>(n) * RS : w, v);
    }
  }
};

template <int BM, int BN>
__global__ void __launch_bounds__(Cfg<BM, BN>::kThreads, 2)
    conv_data_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, ConvGeom g) {
  constexpr int T = Cfg<BM, BN>::kThreads;
  extern __shared__ __align__(16) float smem[];
  int2* taps = reinterpret_cast<int2*>(smem + stage_bytes<BM, BN, false, true>() / sizeof(float));
  const int grp = blockIdx.z, m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int Cg = g.c / g.groups, Kg = g.k / g.groups, RS = g.r * g.s, HW = g.h * g.w, PQ = g.p * g.q;
  const int M = g.n * HW, Kt = Kg * RS;

  DataLoad<BM, BN> ld;
  ld.dy = dy;
  ld.w = w;
  ld.taps = taps;
  ld.Kt = Kt;
  ld.P = g.p;
  ld.Q = g.q;
  ld.sh = g.stride_h;
  ld.sw = g.stride_w;
  ld.RS = RS;
  ld.Cg = Cg;
  ld.Kg = Kg;
  ld.grp = grp;
  {
    const int m = m0 + static_cast<int>(threadIdx.x) % BM;
    ld.mval = m < M;
    const int mm = ld.mval ? m : 0, img = mm / HW, hw = mm - img * HW, h = hw / g.w, wc = hw - h * g.w;
    ld.hh0 = h + g.pad_h;
    ld.ww0 = wc + g.pad_w;
    ld.dyoff = (img * g.k + grp * Kg) * PQ;
    ld.akin = threadIdx.x / BM;
  }
  ld.bkin = threadIdx.x % BK;
  ld.bn = n0 + threadIdx.x / BK;

  float acc[MT][NT][4] = {};
  for (int seg0 = 0; seg0 < Kt; seg0 += kTapSeg) {
    const int seg1 = min(Kt, seg0 + kTapSeg);
    for (int k = seg0 + threadIdx.x; k < seg1; k += T) {
      const int f = k / RS, rs = k - f * RS, r = rs / g.s, s = rs - r * g.s;
      taps[k - seg0] = make_int2(f * PQ, r << 16 | s);
    }
    __syncthreads();
    ld.seg0 = seg0;
    mainloop<BM, BN, false, true>(ld, seg0 / BK, (seg1 + BK - 1) / BK, smem, acc);
  }
  const int C = g.c;
  epilogue<BM, BN>(acc, dx, m0, n0, M, Cg, HW, nullptr, [&](int m) {
    const int img = m / HW;
    return static_cast<long long>(img * C + grp * Cg) * HW + (m - img * HW);
  });
}

// -------------------------------------------------------------------------------------------- backward filter
// A[m, k] = dy[img, g·Kg + m, p, q]                            (m = filter, k = (img, p, q)), k-major tile
// B[k, n] = x[img, g·Cg + c, p·sh − ph + r, q·sw − pw + s]     (n = (c, r, s)), k-major tile
// Block (mt, nt, chunk·G + g) reduces the k-tiles of its chunk.
template <int BM, int BN>
struct FilterLoad {
  static constexpr int T = Cfg<BM, BN>::kThreads;
  const float* x;
  const float* dy;
  const int2* taps;  // the block's BN taps: {c·H·W + r·W + s, r << 16 | s}
  int Kt, PQ, Q, H, W, C, K, sh, sw, ph, pw, grp, Cg, Kg;
  int kin, am, bn, bvalid;  // this thread's tap column in the tile, first A filter row, first B tap, valid B taps

  __device__ __forceinline__ void load(float* As, float* Bs, int kt) {
    constexpr int AE = BK * BM / T, BE = BK * BN / T;
    const int k = kt * BK + kin;
    const bool kv = k < Kt;
    const int kk = kv ? k : 0, img = kk / PQ, pq = kk - img * PQ, p = pq / Q, q = pq - p * Q;
    const int h0 = p * sh - ph, w0 = q * sw - pw;
    const long long dyoff = static_cast<long long>(img * K + grp * Kg) * PQ + pq;
    const int xoff = (img * C + grp * Cg) * H * W + h0 * W + w0;
#pragma unroll
    for (int i = 0; i < AE; ++i) {
      const int m = am + i * (T / BK);
      const bool v = kv && m < Kg;
      cp_async4(As + Tile<true, BM>::at(threadIdx.x / BK + i * (T / BK), kin),
                v ? dy + dyoff + static_cast<long long>(m) * PQ : dy, v);
    }
#pragma unroll
    for (int i = 0; i < BE; ++i) {
      const int nl = threadIdx.x / BK + i * (T / BK);
      bool v = kv && i < bvalid;
      int off = 0;
      if (v) {
        const int2 t = taps[nl];
        const int ih = h0 + (t.y >> 16), iw = w0 + (t.y & 0xffff);
        v = static_cast<unsigned>(ih) < static_cast<unsigned>(H) && static_cast<unsigned>(iw) < static_cast<unsigned>(W);
        off = xoff + t.x;
      }
      cp_async4(Bs + Tile<true, BN>::at(nl, kin), x + (v ? off : 0), v);
    }
  }
};

template <int BM, int BN>
__global__ void __launch_bounds__(Cfg<BM, BN>::kThreads, 2)
    conv_filter_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ out,
                       ConvGeom g, int chunks, int chunk_ktiles) {
  constexpr int T = Cfg<BM, BN>::kThreads;
  extern __shared__ __align__(16) float smem[];
  int2* taps = reinterpret_cast<int2*>(smem + stage_bytes<BM, BN, true, true>() / sizeof(float));
  const int grp = blockIdx.z % g.groups, chunk = blockIdx.z / g.groups;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int Cg = g.c / g.groups, Kg = g.k / g.groups, RS = g.r * g.s, HW = g.h * g.w, PQ = g.p * g.q;
  const int Ng = Cg * RS, Kt = g.n * PQ;

  for (int i = threadIdx.x; i < BN; i += T) {
    const int n = min(n0 + i, Ng - 1), c = n / RS, rs = n - c * RS, r = rs / g.s, s = rs - r * g.s;
    taps[i] = make_int2(c * HW + r * g.w + s, r << 16 | s);
  }
  __syncthreads();

  FilterLoad<BM, BN> ld;
  ld.x = x;
  ld.dy = dy;
  ld.taps = taps;
  ld.Kt = Kt;
  ld.PQ = PQ;
  ld.Q = g.q;
  ld.H = g.h;
  ld.W = g.w;
  ld.C = g.c;
  ld.K = g.k;
  ld.sh = g.stride_h;
  ld.sw = g.stride_w;
  ld.ph = g.pad_h;
  ld.pw = g.pad_w;
  ld.grp = grp;
  ld.Cg = Cg;
  ld.Kg = Kg;
  ld.kin = threadIdx.x % BK;
  ld.am = m0 + threadIdx.x / BK;
  ld.bn = n0 + threadIdx.x / BK;
  ld.bvalid = ld.bn < Ng ? (Ng - ld.bn + T / BK - 1) / (T / BK) : 0;

  const int nkt = (Kt + BK - 1) / BK, kt0 = chunk * chunk_ktiles, kt1 = min(nkt, kt0 + chunk_ktiles);
  float acc[MT][NT][4] = {};
  mainloop<BM, BN, true, true>(ld, kt0, kt1, smem, acc);
  float* o = out + static_cast<long long>(chunks > 1 ? chunk : 0) * g.k * Ng;
  epilogue<BM, BN>(acc, o, m0, n0, Kg, Ng, 1, nullptr,
                   [&](int m) { return static_cast<long long>(grp * Kg + m) * Ng; });
}

// dw[i] = part[0][i] + part[1][i] + ... in chunk order
__global__ void conv_filter_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, long long count,
                                          int chunks) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float s = part[i];
    for (int c = 1; c < chunks; ++c) s += part[c * count + i];
    dw[i] = s;
  }
}

// ---------------------------------------------------------------------------------------------------- launches
int ceil_div(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// 64 columns when that wastes fewer of them than 128 (a 48-channel group, 192 filters, 1,200 or 1,728 taps)
bool narrow(int cols) { return (ceil_div(cols, 64) * 64 - cols) < (ceil_div(cols, 128) * 128 - cols); }

template <int BM, int BN, bool AK>
size_t smem_bytes(int taps) {
  return stage_bytes<BM, BN, AK, true>() + sizeof(int2) * static_cast<size_t>(taps);
}

template <int BM, int BN>
cudaError_t fwd(const float* x, const float* w, const float* bias, float* y, const ConvGeom& g, cudaStream_t st) {
  const int Kt = g.c / g.groups * g.r * g.s;
  const size_t sm = smem_bytes<BM, BN, false>(std::min(Kt, kTapSeg));
  cudaError_t e = cudaFuncSetAttribute(conv_fwd_kernel<BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(sm));
  if (e != cudaSuccess) return e;
  dim3 grid(ceil_div(static_cast<long long>(g.n) * g.p * g.q, BM), ceil_div(g.k / g.groups, BN), g.groups);
  conv_fwd_kernel<BM, BN><<<grid, Cfg<BM, BN>::kThreads, sm, st>>>(x, w, bias, y, g);
  return cudaGetLastError();
}

template <int BM, int BN>
cudaError_t data(const float* dy, const float* w, float* dx, const ConvGeom& g, cudaStream_t st) {
  const int Kt = g.k / g.groups * g.r * g.s;
  const size_t sm = smem_bytes<BM, BN, false>(std::min(Kt, kTapSeg));
  cudaError_t e = cudaFuncSetAttribute(conv_data_kernel<BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(sm));
  if (e != cudaSuccess) return e;
  dim3 grid(ceil_div(static_cast<long long>(g.n) * g.h * g.w, BM), ceil_div(g.c / g.groups, BN), g.groups);
  conv_data_kernel<BM, BN><<<grid, Cfg<BM, BN>::kThreads, sm, st>>>(dy, w, dx, g);
  return cudaGetLastError();
}

void filter_split(const ConvGeom& g, int* chunks, int* chunk_ktiles) {
  const int Ng = g.c / g.groups * g.r * g.s, Kg = g.k / g.groups;
  const long long tiles =
      static_cast<long long>(ceil_div(Kg, 128)) * ceil_div(Ng, narrow(Ng) ? 64 : 128) * g.groups;
  const int nkt = ceil_div(static_cast<long long>(g.n) * g.p * g.q, BK);
  int want = static_cast<int>(std::max<long long>(1, (kFilterTargetBlocks + tiles - 1) / tiles));
  want = std::max(1, std::min(want, nkt / kFilterMinKTiles));
  *chunk_ktiles = ceil_div(nkt, want);
  *chunks = ceil_div(nkt, *chunk_ktiles);
}

template <int BM, int BN>
cudaError_t filter(const float* x, const float* dy, float* dw, float* ws, const ConvGeom& g, cudaStream_t st) {
  int chunks, chunk_ktiles;
  filter_split(g, &chunks, &chunk_ktiles);
  const size_t sm = smem_bytes<BM, BN, true>(BN);
  cudaError_t e = cudaFuncSetAttribute(conv_filter_kernel<BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(sm));
  if (e != cudaSuccess) return e;
  const int Ng = g.c / g.groups * g.r * g.s;
  dim3 grid(ceil_div(g.k / g.groups, BM), ceil_div(Ng, BN), chunks * g.groups);
  conv_filter_kernel<BM, BN><<<grid, Cfg<BM, BN>::kThreads, sm, st>>>(x, dy, chunks > 1 ? ws : dw, g, chunks,
                                                                       chunk_ktiles);
  if ((e = cudaGetLastError()) != cudaSuccess || chunks == 1) return e;
  const long long count = static_cast<long long>(g.k) * Ng;
  conv_filter_reduce_kernel<<<static_cast<int>(std::min<long long>(ceil_div(count, 256), 4096)), 256, 0, st>>>(
      ws, dw, count, chunks);
  return cudaGetLastError();
}

}  // namespace

const char* conv_geometry(ConvGeom* g) {
  if (g->n < 1 || g->c < 1 || g->h < 1 || g->w < 1 || g->k < 1 || g->r < 1 || g->s < 1) return "bad shape";
  if (g->stride_h < 1 || g->stride_w < 1 || g->pad_h < 0 || g->pad_w < 0) return "bad stride or pad";
  if (g->groups < 1 || g->c % g->groups || g->k % g->groups) return "groups must divide the channels and filters";
  if (g->r > 32767 || g->s > 32767 || g->pad_h > 32767 || g->pad_w > 32767) return "kernel or pad too large";
  if (g->h + 2 * static_cast<long long>(g->pad_h) < g->r || g->w + 2 * static_cast<long long>(g->pad_w) < g->s)
    return "the kernel is larger than the padded input";
  g->p = (g->h + 2 * g->pad_h - g->r) / g->stride_h + 1;
  g->q = (g->w + 2 * g->pad_w - g->s) / g->stride_w + 1;
  const long long lim = (1ll << 31) - 1;
  const long long nx = static_cast<long long>(g->n) * g->c * g->h * g->w,
                  ny = static_cast<long long>(g->n) * g->k * g->p * g->q,
                  nw = static_cast<long long>(g->k) * (g->c / g->groups) * g->r * g->s;
  if (nx > lim || ny > lim || nw > lim) return "tensors of 2^31 or more elements are not supported";
  if (static_cast<long long>(conv_filter_chunks(*g)) * nw > lim) return "weight-gradient workspace too large";
  return nullptr;
}

int conv_filter_chunks(const ConvGeom& g) {
  int chunks, chunk_ktiles;
  filter_split(g, &chunks, &chunk_ktiles);
  return chunks;
}

size_t conv_workspace_floats(const ConvGeom& g) {
  const int chunks = conv_filter_chunks(g);
  return chunks > 1 ? static_cast<size_t>(chunks) * g.k * (g.c / g.groups) * g.r * g.s : 0;
}

cudaError_t conv_forward(const float* x, const float* w, const float* bias, float* y, const ConvGeom& g,
                         cudaStream_t stream) {
  return narrow(g.k / g.groups) ? fwd<128, 64>(x, w, bias, y, g, stream) : fwd<128, 128>(x, w, bias, y, g, stream);
}

cudaError_t conv_backward_data(const float* dy, const float* w, float* dx, const ConvGeom& g, cudaStream_t stream) {
  return narrow(g.c / g.groups) ? data<128, 64>(dy, w, dx, g, stream) : data<128, 128>(dy, w, dx, g, stream);
}

cudaError_t conv_backward_filter(const float* x, const float* dy, float* dw, float* workspace, const ConvGeom& g,
                                 cudaStream_t stream) {
  return narrow(g.c / g.groups * g.r * g.s) ? filter<128, 64>(x, dy, dw, workspace, g, stream)
                                            : filter<128, 128>(x, dy, dw, workspace, g, stream);
}

}  // namespace cosb
