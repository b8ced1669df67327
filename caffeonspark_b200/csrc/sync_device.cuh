// sync_device.cuh -- building blocks shared by the five variants of the fused
// sync kernel (fused_sync_sgd.cu: vector LDG/STG, _tma.cu: cp.async.bulk
// pipeline, _push.cu: stores only, _ll.cu: flag-in-data, _nvls.cu: in-switch
// reduction): PTX wrappers, bf16 packing, the per-CTA cross-GPU barrier, the
// shard/vector partition and its scalar edges, the reduce in the reference's
// order, the blob (segment) cursor, the SGD and Adam element updates in the
// reference's operation order, and the host-side dispatch of a launch to its
// <N, BF16, ADAM, NORM> instantiation.
#ifndef COS_SYNC_DEVICE_CUH_
#define COS_SYNC_DEVICE_CUH_

#include <cuda_bf16.h>
#include <stdint.h>

#include "fused_sync_sgd.hpp"
#include "powf_half.h"

namespace cosb {
namespace {

// ------------------------------------------------------------ PTX helpers

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// streaming 128-bit load that does not allocate in L1 (each element is read once)
__device__ __forceinline__ float4 ld_stream(const float* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ uint2 ld_stream_u2(const uint16_t* p) {
  uint2 v;
  asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}

__device__ __forceinline__ void st_vec(float* p, const float4& v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// NVLS (NVLink SHARP): one load on a multicast address returns the fp32 sum of the
// word on every rank, reduced inside the NVSwitch (SASS LDGMC.E.ADD.F32x4); one
// store on it lands on every rank.
__device__ __forceinline__ float4 mc_ld_reduce(const float* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

__device__ __forceinline__ void mc_st(float* p, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

__device__ __forceinline__ float bf16_bits_to_float(uint32_t bits16) { return __uint_as_float(bits16 << 16); }

__device__ __forceinline__ uint16_t float_to_bf16_bits(float f) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

// the rounding the bf16 wire applies to a gradient element
__device__ __forceinline__ float round_bf16(float x) { return bf16_bits_to_float(float_to_bf16_bits(x)); }

__device__ __forceinline__ uint2 pack_bf16x4(const float4& v) {
  uint2 o;
  o.x = static_cast<uint32_t>(float_to_bf16_bits(v.x)) | (static_cast<uint32_t>(float_to_bf16_bits(v.y)) << 16);
  o.y = static_cast<uint32_t>(float_to_bf16_bits(v.z)) | (static_cast<uint32_t>(float_to_bf16_bits(v.w)) << 16);
  return o;
}

__device__ __forceinline__ float4 unpack_bf16x4(const uint2& u) {
  return make_float4(bf16_bits_to_float(u.x & 0xffffu), bf16_bits_to_float(u.x >> 16),
                     bf16_bits_to_float(u.y & 0xffffu), bf16_bits_to_float(u.y >> 16));
}

// ------------------------------------------------------ cross-GPU barrier

__device__ __forceinline__ uint32_t* flag_slot(uint32_t* base, int which, int cta, int src) {
  return base + (static_cast<size_t>(which) * kMaxCtas + cta) * kMaxRanks + src;
}

// Barrier between CTA blockIdx.x of every rank, split into its two halves.
// Thread t < world handles peer t.  cta_signal publishes this launch's epoch
// into the peer's flag slot [cta][rank]: the leading __syncthreads orders every
// store of the CTA (e.g. pushes into peer memory) before the releasing thread,
// and st.release.sys (= fence.acq_rel.sys + store, cumulative over the bar.sync)
// makes them visible before the flag is.  cta_wait spins on the LOCAL slot
// [cta][t] (peers store into it, so spinning costs no NVLink bandwidth) with
// relaxed loads and issues ONE acquire fence after the flag arrived.
// cta_wait returns false if a peer did not arrive within timeout_ns (status is set).
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Optional diagnostics (option "trace"): the first participating thread of CTA 0 stamps %globaltimer into
// trace[5 + 4*which ...]: barrier entered (after __syncthreads), release fence done, flag arrived, acquire done.
__device__ __forceinline__ bool barrier_tracer(const SyncParams& p) {
  return p.trace != nullptr && blockIdx.x == 0 && static_cast<int>(threadIdx.x) == (p.rank == 0 ? 1 : 0);
}

__device__ __forceinline__ void cta_signal(const SyncParams& p, int which) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < p.world && t != p.rank) {
    const bool tr = barrier_tracer(p);
    if (tr) p.trace[5 + 4 * which] = globaltimer_ns();
    asm volatile("fence.acq_rel.sys;" ::: "memory");  // release: cumulative over the bar.sync above
    if (tr) p.trace[6 + 4 * which] = globaltimer_ns();
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(flag_slot(p.flags[t], which, blockIdx.x, p.rank)),
                 "r"(p.epoch)
                 : "memory");
  }
}

__device__ __forceinline__ bool cta_wait(const SyncParams& p, int which, int* s_abort) {
  const int t = threadIdx.x;
  if (t < p.world && t != p.rank) {
    const bool tr = barrier_tracer(p);
    const uint32_t* mine = flag_slot(p.flags[p.rank], which, blockIdx.x, t);
    const unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    for (;;) {
      uint32_t v = ld_relaxed_sys(mine);
      if (static_cast<int32_t>(v - p.epoch) >= 0) break;
      if ((++spins & 0x3ffu) == 0) {
        if (*reinterpret_cast<volatile int*>(s_abort)) break;
        if (globaltimer_ns() - t0 > p.timeout_ns) {
          atomicExch(p.status, 100 + which * 32 + t);  // which barrier, which peer
          *reinterpret_cast<volatile int*>(s_abort) = 1;
          break;
        }
      }
    }
    if (tr) p.trace[7 + 4 * which] = globaltimer_ns();
    asm volatile("fence.acq_rel.sys;" ::: "memory");  // acquire: later loads see what the peer released
    if (tr) p.trace[8 + 4 * which] = globaltimer_ns();
  }
  __syncthreads();
  return *reinterpret_cast<volatile int*>(s_abort) == 0;
}

__device__ __forceinline__ bool cta_barrier(const SyncParams& p, int which, int* s_abort) {
  cta_signal(p, which);
  return cta_wait(p, which, s_abort);
}

// ------------------------------------------------------------- partition

struct ShardRange {
  uint64_t lo, hi;        // element range
  uint64_t vec_lo;        // first float4 index fully inside
  uint64_t nvec;          // number of float4 vectors fully inside
  uint64_t head_end;      // [lo, head_end) scalar head
  uint64_t tail_begin;    // [tail_begin, hi) scalar tail
  // 512-byte aligned iteration space (push / NVLS kernels): thread index a = tid + k*stride addresses vector
  // vec_base + a, valid for off <= a < off + nvec.  vec_base is a multiple of 32 vectors, so every warp's 32 float4
  // cover exactly four 128-byte lines of data_ / diff_ / the receive slot -- with the plain j = tid + k*stride walk
  // a shard that starts mid-line (CaffeNet: every shard but one) makes EVERY warp access straddle lines: partial
  // sectors over NVLink.
  uint64_t vec_base;      // (lo / 4) rounded down to a multiple of 32
  uint64_t off;           // vec_lo - vec_base, 0..32
};

// aligned index a -> element index of its vector in shard r, or ~0 when a is outside the shard's vector body
__device__ __forceinline__ uint64_t vec_elem(const ShardRange& r, uint64_t a) {
  return (a >= r.off && a - r.off < r.nvec) ? ((r.vec_base + a) << 2) : ~0ull;
}

// socket_sync_cpu.cpp:46-54 chunk(): multiply first, then divide, in 64 bit.
__device__ __forceinline__ ShardRange shard_range(uint64_t count, int world, int s) {
  ShardRange r;
  r.lo = static_cast<uint64_t>(s) * count / static_cast<uint64_t>(world);
  r.hi = (static_cast<uint64_t>(s) + 1) * count / static_cast<uint64_t>(world);
  uint64_t vlo = (r.lo + 3) >> 2, vhi = r.hi >> 2;
  if (vhi > vlo) {
    r.vec_lo = vlo;
    r.nvec = vhi - vlo;
    r.head_end = vlo << 2;
    r.tail_begin = vhi << 2;
  } else {
    r.vec_lo = vlo;
    r.nvec = 0;
    r.head_end = r.hi;  // everything scalar
    r.tail_begin = r.hi;
  }
  r.vec_base = (r.lo >> 2) & ~31ull;
  r.off = r.vec_lo - r.vec_base;
  return r;
}

// f(i) for the scalar head / tail element i of range r (ShardRange or the TMA kernel's BodyRange) that thread t of
// CTA 0 handles, if there is one
template <class Range, class F>
__device__ __forceinline__ void for_edge_element(const Range& r, unsigned t, F f) {
  const uint64_t nhead = r.head_end - r.lo, ntail = r.hi - r.tail_begin;
  if (t < nhead) f(r.lo + t);
  else if (t - nhead < ntail) f(r.tail_begin + (t - nhead));
}

// the same element as an index, ~0 when thread t has none
template <class Range>
__device__ __forceinline__ uint64_t edge_element(const Range& r, unsigned t) {
  uint64_t i = ~0ull;
  for_edge_element(r, t, [&](uint64_t e) { i = e; });
  return i;
}

// ------------------------------------------------------------- reduce

// One term of the reduce, with the 1/N scale applied BEFORE the sum (parallel_cpu.cpp:120-122 runs before
// socket_sync_cpu.cpp:112-132): the first term is scale4(inv, x), each further one add_scaled(acc, inv, x).
__device__ __forceinline__ float4 scale4(float inv, const float4& x) {
  return make_float4(__fmul_rn(inv, x.x), __fmul_rn(inv, x.y), __fmul_rn(inv, x.z), __fmul_rn(inv, x.w));
}

__device__ __forceinline__ void add_scaled(float4& acc, float inv, const float4& x) {
  acc.x = __fadd_rn(__fmul_rn(inv, x.x), acc.x);
  acc.y = __fadd_rn(__fmul_rn(inv, x.y), acc.y);
  acc.z = __fadd_rn(__fmul_rn(inv, x.z), acc.z);
  acc.w = __fadd_rn(__fmul_rn(inv, x.w), acc.w);
}

// Element i of shard s summed over the world's diff_ (or bf16 wire buffers) in the reference's order s, s+1, ...
// (mod N), each term scaled by 1/N first.
template <bool BF16>
__device__ __forceinline__ float reduce_scalar(const SyncParams& p, int s, uint64_t i) {
  float acc = 0.f;
  for (int j = 0; j < p.world; ++j) {
    int src = s + j;
    if (src >= p.world) src -= p.world;
    float x = BF16 ? bf16_bits_to_float(p.wire[src][i]) : p.diff[src][i];
    x = __fmul_rn(p.inv_scale, x);
    acc = (j == 0) ? x : __fadd_rn(x, acc);
  }
  return acc;
}

// ----------------------------------------------------------- SGD element

struct SegCursor {
  const uint64_t* end;
  const float* lr_mult;
  const float* decay_mult;
  int nseg;
  int k;
  __device__ __forceinline__ void seek(uint64_t i) {  // binary search: first k with end[k] > i
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (end[mid] > i) hi = mid; else lo = mid + 1;
    }
    k = lo;
  }
  __device__ __forceinline__ void advance(uint64_t i) {
    while (k < nseg - 1 && i >= end[k]) ++k;
  }
};

// Segments a kernel copies into dynamic shared memory at most (ends, then lr_mult, then decay_mult); with more the
// cursor reads the global table.  The TMA kernel has its own, smaller limit.
constexpr int kMaxSegSmem = 1024;

// dynamic shared memory the segment table takes when at most max_smem segments are copied
inline size_t seg_smem_bytes(int nseg, int max_smem = kMaxSegSmem) {
  return nseg <= max_smem ? static_cast<size_t>(nseg) * (sizeof(uint64_t) + 2 * sizeof(float)) : 0;
}

// Regularize + ComputeUpdateValue + Blob::Update for one element, in the
// reference's operation order with one rounding per operation:
//   L2: g = ld*w + g          (sgd_solver.cpp:155-160 caffe_axpy(local_decay, data, diff))
//   L1: g = ld*sign(w) + g    (sgd_solver.cpp:161-168 caffe_cpu_sign into temp_, then caffe_axpy; sign is
//                              (0 < w) - (w < 0): 0 for +-0 and NaN, math_functions.hpp caffe_sign)
//   h = m*h ; h = lr*g + h ; w = (-1*h) + w
template <bool L1>
__device__ __forceinline__ void sgd_element_t(float g, float& w, float& h, float lr, float ld, float m) {
  if (ld != 0.f) {
    const float x = L1 ? static_cast<float>((0.f < w) - (w < 0.f)) : w;
    g = __fadd_rn(__fmul_rn(ld, x), g);
  }
  h = __fmul_rn(m, h);
  h = __fadd_rn(__fmul_rn(lr, g), h);
  w = __fadd_rn(__fmul_rn(-1.0f, h), w);
}

// l1 is a launch-wide constant: ONE uniform branch selects the instantiation, so the (rare) L1 path adds no
// instructions to the L2 path (the TMA kernel's 8 consumer warps per SM are issue-bound).
__device__ __forceinline__ void sgd_element(float g, float& w, float& h, float lr, float ld, float m, int l1 = 0) {
  if (l1) sgd_element_t<true>(g, w, h, lr, ld, m);
  else sgd_element_t<false>(g, w, h, lr, ld, m);
}

__device__ __forceinline__ void sgd_vec(const SyncParams& p, SegCursor& c, uint64_t i, const float4& g, float4& w,
                                        float4& h) {
  c.advance(i);
  if (i + 3 < c.end[c.k]) {
    const float lr = __fmul_rn(p.rate, c.lr_mult[c.k]);
    const float ld = __fmul_rn(p.weight_decay, c.decay_mult[c.k]);
    if (p.l1) {
      sgd_element_t<true>(g.x, w.x, h.x, lr, ld, p.momentum);
      sgd_element_t<true>(g.y, w.y, h.y, lr, ld, p.momentum);
      sgd_element_t<true>(g.z, w.z, h.z, lr, ld, p.momentum);
      sgd_element_t<true>(g.w, w.w, h.w, lr, ld, p.momentum);
    } else {
      sgd_element_t<false>(g.x, w.x, h.x, lr, ld, p.momentum);
      sgd_element_t<false>(g.y, w.y, h.y, lr, ld, p.momentum);
      sgd_element_t<false>(g.z, w.z, h.z, lr, ld, p.momentum);
      sgd_element_t<false>(g.w, w.w, h.w, lr, ld, p.momentum);
    }
  } else {  // the vector straddles one or more blob boundaries
    const float gg[4] = {g.x, g.y, g.z, g.w};
    float ww[4] = {w.x, w.y, w.z, w.w};
    float hh[4] = {h.x, h.y, h.z, h.w};
    int k = c.k;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      while (k < c.nseg - 1 && i + e >= c.end[k]) ++k;
      sgd_element(gg[e], ww[e], hh[e], __fmul_rn(p.rate, c.lr_mult[k]), __fmul_rn(p.weight_decay, c.decay_mult[k]),
                  p.momentum, p.l1);
    }
    w = make_float4(ww[0], ww[1], ww[2], ww[3]);
    h = make_float4(hh[0], hh[1], hh[2], hh[3]);
  }
}

// ---------------------------------------------------------- Adam element

// The same Regularize, then AdamSolver::ComputeUpdateValue's CPU branch (adam_solver.cpp:46-73; caffe_cpu_axpby =
// scal then axpy, mkl_alternate.hpp) and Blob::Update, one rounding per operation (m = h, v = second history half):
//   m = b1*m ; m = (1-b1)*g + m
//   t = g*g ; v = b2*v ; v = (1-b2)*t + v
//   t = powf(v, 0.5) ; t = t + delta ; t = m / t        (powf as glibc rounds it, powf_half.h)
//   g = lrc*t ; w = (-1*g) + w                           lrc = (rate*lr_mult)*correction
template <bool L1>
__device__ __forceinline__ void adam_element_t(float g, float& w, float& m, float& v, float lrc, float ld,
                                               const SyncParams& p) {
  if (ld != 0.f) {
    const float x = L1 ? static_cast<float>((0.f < w) - (w < 0.f)) : w;
    g = __fadd_rn(__fmul_rn(ld, x), g);
  }
  const float b1 = p.momentum, b2 = p.beta2;
  m = __fmul_rn(b1, m);
  m = __fadd_rn(__fmul_rn(__fsub_rn(1.f, b1), g), m);
  float t = __fmul_rn(g, g);
  v = __fmul_rn(b2, v);
  v = __fadd_rn(__fmul_rn(__fsub_rn(1.f, b2), t), v);
  t = cos_powf_half(v);
  t = __fadd_rn(t, p.delta);
  t = __fdiv_rn(m, t);
  g = __fmul_rn(lrc, t);
  w = __fadd_rn(__fmul_rn(-1.0f, g), w);
}

// one element of blob k
__device__ __forceinline__ void adam_element(const SyncParams& p, float g, float& w, float& m, float& v, float lr_mult,
                                             float decay_mult) {
  const float lrc = __fmul_rn(__fmul_rn(p.rate, lr_mult), p.correction);
  const float ld = __fmul_rn(p.weight_decay, decay_mult);
  if (p.l1) adam_element_t<true>(g, w, m, v, lrc, ld, p);
  else adam_element_t<false>(g, w, m, v, lrc, ld, p);
}

__device__ __forceinline__ void adam_vec(const SyncParams& p, SegCursor& c, uint64_t i, const float4& g, float4& w,
                                         float4& m, float4& v) {
  c.advance(i);
  int k = c.k;
  // One element per trip, picked and written back with selects: the four double-precision powf evaluations are
  // not interleaved, which keeps the update inside the kernels' register budget (no spills at N = 8).
#pragma unroll 1
  for (int e = 0; e < 4; ++e) {  // the vector may straddle blob boundaries
    while (k < c.nseg - 1 && i + e >= c.end[k]) ++k;
    float ge = e == 0 ? g.x : e == 1 ? g.y : e == 2 ? g.z : g.w;
    float we = e == 0 ? w.x : e == 1 ? w.y : e == 2 ? w.z : w.w;
    float me = e == 0 ? m.x : e == 1 ? m.y : e == 2 ? m.z : m.w;
    float ve = e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w;
    adam_element(p, ge, we, me, ve, c.lr_mult[k], c.decay_mult[k]);
    if (e == 0) { w.x = we; m.x = me; v.x = ve; }
    else if (e == 1) { w.y = we; m.y = me; v.y = ve; }
    else if (e == 2) { w.z = we; m.z = me; v.z = ve; }
    else { w.w = we; m.w = me; v.w = ve; }
  }
}

// ---------------------------------------------- solver as a kernel parameter
// The kernels are templates on ADAM (false = SGD, the default).  The SGD instantiations only ever see sgd_vec /
// sgd_element; Adam loads and stores v at h's index in hist2.  hist2 = hist + P is 16-byte aligned only when P is a
// multiple of 4 (the history is Caffe's history_ laid out flat, m then v); i is, so the access width follows from
// the alignment of hist2, the same for the whole launch.

template <bool ADAM>
__device__ __forceinline__ void load_v(const SyncParams& p, uint64_t i, float4& v) {
  if (ADAM) {
    const float* q = p.hist2 + i;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p.hist2);
    if ((a & 15) == 0) {
      v = *reinterpret_cast<const float4*>(q);
    } else if ((a & 7) == 0) {
      const float2 lo = *reinterpret_cast<const float2*>(q), hi = *reinterpret_cast<const float2*>(q + 2);
      v = make_float4(lo.x, lo.y, hi.x, hi.y);
    } else {
      v = make_float4(q[0], q[1], q[2], q[3]);
    }
  }
}

template <bool ADAM>
__device__ __forceinline__ void store_v(const SyncParams& p, uint64_t i, const float4& v) {
  if (ADAM) {
    float* q = p.hist2 + i;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p.hist2);
    if ((a & 15) == 0) {
      *reinterpret_cast<float4*>(q) = v;
    } else if ((a & 7) == 0) {
      *reinterpret_cast<float2*>(q) = make_float2(v.x, v.y);
      *reinterpret_cast<float2*>(q + 2) = make_float2(v.z, v.w);
    } else {
      q[0] = v.x;
      q[1] = v.y;
      q[2] = v.z;
      q[3] = v.w;
    }
  }
}

// ------------------------------------------- Normalize as a kernel parameter
// iter_size > 1 (SGDSolver::Normalize, sgd_solver.cpp:118-142): caffe_scal(count, Dtype(1.)/iter_size, diff) on the
// reduced gradient, before Regularize, for SGD and Adam alike.  One rounding: g = accum_norm * g.  The kernels are
// templates on NORM (false = no Normalize, the default); NORM is applied to the reduced gradient right before the
// element update, so it only adds one FMUL per element.
__device__ __forceinline__ float4 normalize_vec(const SyncParams& p, const float4& g) { return scale4(p.accum_norm, g); }

template <bool ADAM, bool NORM = false>
__device__ __forceinline__ void update_vec(const SyncParams& p, SegCursor& c, uint64_t i, const float4& g, float4& w,
                                           float4& h, float4& v) {
  const float4 gn = NORM ? normalize_vec(p, g) : g;
  if (ADAM) adam_vec(p, c, i, gn, w, h, v);
  else sgd_vec(p, c, i, gn, w, h);
}

// scalar head / tail element i of blob c.k
template <bool ADAM, bool NORM = false>
__device__ __forceinline__ void update_element(const SyncParams& p, const SegCursor& c, uint64_t i, float g, float& w,
                                               float& h) {
  if (NORM) g = __fmul_rn(p.accum_norm, g);
  if (ADAM) {
    float v = p.hist2[i];
    adam_element(p, g, w, h, v, c.lr_mult[c.k], c.decay_mult[c.k]);
    p.hist2[i] = v;
  } else {
    sgd_element(g, w, h, __fmul_rn(p.rate, c.lr_mult[c.k]), __fmul_rn(p.weight_decay, c.decay_mult[c.k]),
                p.momentum, p.l1);
  }
}

// ------------------------------------------------------------ host: launch

// world size and rank a launcher accepts (its kernel needs at least min_world ranks)
inline bool valid_world(const SyncParams& p, int min_world) {
  return p.world >= min_world && p.world <= kMaxRanks && p.rank >= 0 && p.rank < p.world;
}

// Launches the <N, BF16, ADAM, NORM> instantiation of a kernel family that SyncParams selects: BF16 = grad_bf16,
// ADAM = (solver == kSolverAdam), NORM = sync_normalizes(p).  K::kernel<N, BF16, ADAM, NORM> names the family's
// kernel.  N = n for n = 2..8; any other n launches the run-time-world instantiation N = 0 when GENERIC, else is
// refused.
template <class K, int N, bool NORM>
void launch_solver(const SyncParams& p, int grid, int block, size_t smem, cudaStream_t stream) {
  if (p.solver == kSolverAdam) {
    if (p.grad_bf16) K::template kernel<N, true, true, NORM><<<grid, block, smem, stream>>>(p);
    else K::template kernel<N, false, true, NORM><<<grid, block, smem, stream>>>(p);
  } else if (p.grad_bf16) {
    K::template kernel<N, true, false, NORM><<<grid, block, smem, stream>>>(p);
  } else {
    K::template kernel<N, false, false, NORM><<<grid, block, smem, stream>>>(p);
  }
}

template <class K, int N>
cudaError_t launch_n(const SyncParams& p, int grid, int block, size_t smem, cudaStream_t stream) {
  if (sync_normalizes(p)) launch_solver<K, N, true>(p, grid, block, smem, stream);
  else launch_solver<K, N, false>(p, grid, block, smem, stream);
  return cudaGetLastError();
}

template <class K, bool GENERIC>
cudaError_t launch_sync(const SyncParams& p, int n, int grid, int block, size_t smem, cudaStream_t stream) {
  switch (n) {
    case 2: return launch_n<K, 2>(p, grid, block, smem, stream);
    case 3: return launch_n<K, 3>(p, grid, block, smem, stream);
    case 4: return launch_n<K, 4>(p, grid, block, smem, stream);
    case 5: return launch_n<K, 5>(p, grid, block, smem, stream);
    case 6: return launch_n<K, 6>(p, grid, block, smem, stream);
    case 7: return launch_n<K, 7>(p, grid, block, smem, stream);
    case 8: return launch_n<K, 8>(p, grid, block, smem, stream);
    default:
      if constexpr (GENERIC) return launch_n<K, 0>(p, grid, block, smem, stream);
      else return cudaErrorInvalidValue;
  }
}

}  // namespace
}  // namespace cosb
#endif
