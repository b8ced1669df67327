// fused_sync_sgd_ll.cu -- the LOW-LATENCY variant of the fused sync kernel for
// small nets (LeNet, CIFAR-10-quick): no barriers and no memory fences at all.
//
// In the barrier-based kernels one cross-GPU barrier costs two system-scope
// fences (release before the flag store, acquire after the poll) plus the flag
// flight, each of them microseconds; a 64 KiB..2 MiB sync is two barriers plus a
// few microseconds of real work.  Here every 8-byte word that crosses NVLink
// carries its own flag (the launch epoch) next to 4 bytes of payload, written
// and read with single 64-bit accesses, which are single-copy atomic: a reader
// that sees the flag sees the payload, so no fence and no separate barrier is
// needed (the scheme NCCL calls "LL").  Twice the wire bytes -- irrelevant while
// the message is latency-bound; AUTO uses this kernel below ll_max_bytes only.
//
// Same arithmetic and the same results, bit for bit, as the other P2P kernels
// (reference mapping in fused_sync_sgd.cu / fused_sync_sgd_push.cu):
//   phase 1  store shard q of my gradient into rank q's LL gradient slot [me]
//            (bf16 wire: two bf16 per word, cast in registers), then zero what I
//            pushed (ClearParamDiffs; nobody else reads diff_);
//   phase 2  owner: poll the N-1 slots word by word, reduce with my own gradient
//            in the reference's order s, s+1, ... (mod N) with the 1/N scale before
//            the sum, apply decay + momentum + update, store w / h locally and w
//            into every peer's LL weight slot [me];
//   phase 3  poll the N-1 weight slots and copy the peers' shards into data_ (the
//            next on_start(), socket_sync_cpu.cpp:102-105).
// Slot reuse needs no barrier: a peer can only push step t+1 after it finished
// step t, which includes receiving MY step-t weights, which I send after my last
// read of the gradient slots; and it can only push step-t+1 weights after it has
// my step-t+1 gradient, which I send after my phase 3 of step t.  Epochs grow
// monotonically, so a stale word can never carry the current flag.
#include "fused_sync_sgd.hpp"
#include "sync_device.cuh"

namespace cosb {
namespace {

constexpr int kLLThreads = 512;
constexpr int kLLMaxSeg = 1024;
constexpr int kEdgeWords = 8;  // scalar head/tail elements of a shard travel in 8 extra words behind the body

__device__ __forceinline__ void st_ll2(uint64_t* p, uint64_t a, uint64_t b) {  // two atomic 8-byte words
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void st_ll1(uint64_t* p, uint64_t a) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(a) : "memory");
}
__device__ __forceinline__ void ld_ll2(const uint64_t* p, uint64_t& a, uint64_t& b) {
  asm volatile("ld.relaxed.sys.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ uint64_t ld_ll1(const uint64_t* p) {
  uint64_t a;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(a) : "l"(p) : "memory");
  return a;
}
__device__ __forceinline__ uint64_t ll_word(uint32_t payload, uint32_t flag) {
  return static_cast<uint64_t>(payload) | (static_cast<uint64_t>(flag) << 32);
}
__device__ __forceinline__ bool ll_ok(uint64_t w, uint32_t flag) { return static_cast<uint32_t>(w >> 32) == flag; }

struct Poll {  // bounded spinning shared by all polls of a thread
  const SyncParams& p;
  int* s_abort;
  unsigned spins = 0;
  unsigned long long t0 = 0;
  __device__ Poll(const SyncParams& pp, int* a) : p(pp), s_abort(a) {}
  __device__ __forceinline__ bool give_up(int src) {  // call once per failed try
    if ((++spins & 0x3ffu) != 0) return false;
    if (*reinterpret_cast<volatile int*>(s_abort)) return true;
    const unsigned long long now = globaltimer_ns();
    if (t0 == 0) t0 = now;
    if (now - t0 > p.timeout_ns) {
      atomicExch(p.status, 200 + src);
      *reinterpret_cast<volatile int*>(s_abort) = 1;
      return true;
    }
    return false;
  }
  __device__ __forceinline__ void progress() { t0 = 0; }
};

// K independent groups of W consecutive LL words (W = 4: one float4 of fp32 payload, W = 2: four bf16).  All
// loads of a round are issued before the first flag is looked at, so K x W/2 16-byte loads are in flight per
// thread; groups whose flags are not all current are re-read.  `live` masks the groups that exist.  Returns false
// on abort (peer never arrived).
template <int K, int W>
__device__ __forceinline__ bool poll_groups(const uint64_t* const (&ptr)[K], uint32_t live, uint32_t flag, Poll& poll,
                                            int src_for_status, uint64_t (&out)[K][W]) {
  uint32_t pending = live;
  while (pending) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (pending & (1u << k)) {
#pragma unroll
        for (int w = 0; w < W; w += 2) ld_ll2(ptr[k] + w, out[k][w], out[k][w + 1]);
      }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (pending & (1u << k)) {
        bool ok = true;
#pragma unroll
        for (int w = 0; w < W; ++w) ok = ok && ll_ok(out[k][w], flag);
        if (ok) pending &= ~(1u << k);
      }
    }
    if (pending && poll.give_up(src_for_status)) return false;
  }
  poll.progress();
  return true;
}
__device__ __forceinline__ bool poll1(const uint64_t* w, uint32_t flag, Poll& poll, int src, uint32_t& out) {
  uint64_t a;
  for (;;) {
    a = ld_ll1(w);
    if (ll_ok(a, flag)) break;
    if (poll.give_up(src)) return false;
  }
  poll.progress();
  out = static_cast<uint32_t>(a);
  return true;
}

// edge (scalar head / tail) element e of shard range r -> index into the kEdgeWords edge words of a slot
__device__ __forceinline__ uint64_t edge_index(const ShardRange& r, uint64_t e) {
  return e < r.head_end ? e - r.lo : 4 + (e - r.tail_begin);
}
__device__ __forceinline__ uint64_t edge_of_thread(const ShardRange& r, unsigned t) {
  const uint64_t nhead = r.head_end - r.lo, ntail = r.hi - r.tail_begin;
  if (t < nhead) return r.lo + t;
  if (t - nhead < ntail) return r.tail_begin + (t - nhead);
  return ~0ull;
}

// N = compile-time world size, 2..8 (the N-1 polled slots live in registers)
// ADAM: Adam update with the second history half (sync_device.cuh), false = SGD.
// NORM: Normalize (iter_size > 1) before the update (sync_device.cuh), false = none.
template <int N, bool BF16, bool ADAM = false, bool NORM = false>
__global__ void __launch_bounds__(kLLThreads, 1) fused_sync_sgd_ll_kernel(const SyncParams p) {
  extern __shared__ unsigned char smem_raw[];
  __shared__ int s_abort;
  uint64_t* s_end = reinterpret_cast<uint64_t*>(smem_raw);
  float* s_lr = reinterpret_cast<float*>(s_end + p.nseg);
  float* s_dm = s_lr + p.nseg;
  const bool seg_in_smem = p.nseg <= kLLMaxSeg;
  if (seg_in_smem) {
    for (int k = threadIdx.x; k < p.nseg; k += blockDim.x) {
      s_end[k] = p.seg_end[k];
      s_lr[k] = p.seg_lr_mult[k];
      s_dm[k] = p.seg_decay_mult[k];
    }
  }
  if (threadIdx.x == 0) s_abort = 0;
  __syncthreads();
  const bool tracer = p.trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (tracer) p.trace[0] = globaltimer_ns();

  const int world = N;
  const int rank = p.rank;
  const uint32_t flag = p.epoch;
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t gslot = p.ll_grad_stride;   // 8-byte words per gradient slot (body + edge words)
  const uint64_t wslot = p.ll_weight_stride; // 8-byte words per weight slot
  float* g = const_cast<float*>(p.diff[rank]);
  const bool zero = p.zero_diff != 0;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  // body word index of element i in a slot of shard range r: fp32 wire / weights 1 element per word,
  // bf16 wire 2 elements per word; base = r.lo rounded down to a multiple of 4
  const uint64_t gedge = gslot - kEdgeWords, wedge = wslot - kEdgeWords;

  // ---- phase 1: my gradient -> the owners' LL gradient slots [rank] ---------
  // The loads for all N-1 destinations are issued before the first store: one local-memory latency per
  // iteration instead of N-1.
  constexpr int D = N - 1;
  const uint64_t max_nvec = ((p.count + N - 1) / N + 3) >> 2;  // >= nvec of every shard
  for (uint64_t j = tid; j < max_nvec; j += stride) {
    float4 v[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      int q = rank + 1 + d;
      if (q >= N) q -= N;
      const ShardRange r = shard_range(p.count, N, q);
      if (j < r.nvec) v[d] = ld_stream(g + ((r.vec_lo + j) << 2));
    }
#pragma unroll
    for (int d = 0; d < D; ++d) {
      int q = rank + 1 + d;
      if (q >= N) q -= N;
      const ShardRange r = shard_range(p.count, N, q);
      if (j < r.nvec) {
        const uint64_t i = (r.vec_lo + j) << 2, base = r.lo & ~3ull;
        uint64_t* dst = p.ll_grad[q] + static_cast<uint64_t>(rank) * gslot;
        if (BF16) {
          const uint32_t lo2 = static_cast<uint32_t>(float_to_bf16_bits(v[d].x)) | (static_cast<uint32_t>(float_to_bf16_bits(v[d].y)) << 16);
          const uint32_t hi2 = static_cast<uint32_t>(float_to_bf16_bits(v[d].z)) | (static_cast<uint32_t>(float_to_bf16_bits(v[d].w)) << 16);
          st_ll2(dst + ((i - base) >> 1), ll_word(lo2, flag), ll_word(hi2, flag));
        } else {
          uint64_t* w = dst + (i - base);
          st_ll2(w, ll_word(__float_as_uint(v[d].x), flag), ll_word(__float_as_uint(v[d].y), flag));
          st_ll2(w + 2, ll_word(__float_as_uint(v[d].z), flag), ll_word(__float_as_uint(v[d].w), flag));
        }
      }
    }
  }
  if (blockIdx.x == 0) {
    for (int d = 1; d < world; ++d) {
      int q = rank + d;
      if (q >= world) q -= world;
      const ShardRange r = shard_range(p.count, world, q);
      const uint64_t e = edge_of_thread(r, threadIdx.x);
      if (e != ~0ull) {
        float x = g[e];
        if (BF16) x = bf16_bits_to_float(float_to_bf16_bits(x));
        st_ll1(p.ll_grad[q] + static_cast<uint64_t>(rank) * gslot + gedge + edge_index(r, e), ll_word(__float_as_uint(x), flag));
      }
    }
  }
  if (tracer) p.trace[1] = globaltimer_ns();
  if (zero) {  // ClearParamDiffs of what I pushed: plain streaming stores behind the pushes, hidden in the flight time
    for (int d = 1; d < world; ++d) {
      int q = rank + d;
      if (q >= world) q -= world;
      const ShardRange r = shard_range(p.count, world, q);
      for (uint64_t j = tid; j < r.nvec; j += stride) st_vec(g + ((r.vec_lo + j) << 2), z4);
      if (blockIdx.x == 0) {
        const uint64_t e = edge_of_thread(r, threadIdx.x);
        if (e != ~0ull) g[e] = 0.f;
      }
    }
  }
  if (tracer) p.trace[2] = globaltimer_ns();

  // ---- phase 2: poll + reduce + update + push the new weights ----------------
  SegCursor cur;
  cur.end = seg_in_smem ? s_end : p.seg_end;
  cur.lr_mult = seg_in_smem ? s_lr : p.seg_lr_mult;
  cur.decay_mult = seg_in_smem ? s_dm : p.seg_decay_mult;
  cur.nseg = p.nseg;
  cur.k = 0;
  Poll poll(p, &s_abort);
  bool alive = true;
  {
    const ShardRange r = shard_range(p.count, world, rank);
    const uint64_t base = r.lo & ~3ull;
    float* wl = p.data[rank];
    float* hl = p.hist;
    const float inv = p.inv_scale;
    const uint64_t* mine = p.ll_grad[rank];
    if (tid < r.nvec) cur.seek((r.vec_lo + tid) << 2);
    for (uint64_t j = tid; alive && j < r.nvec; j += stride) {
      const uint64_t i = (r.vec_lo + j) << 2;
      float4 x = ld_stream(g + i);
      float4 w = *reinterpret_cast<const float4*>(wl + i);
      float4 h = *reinterpret_cast<const float4*>(hl + i);
      float4 v;
      load_v<ADAM>(p, i, v);
      if (BF16) {
        x.x = bf16_bits_to_float(float_to_bf16_bits(x.x)); x.y = bf16_bits_to_float(float_to_bf16_bits(x.y));
        x.z = bf16_bits_to_float(float_to_bf16_bits(x.z)); x.w = bf16_bits_to_float(float_to_bf16_bits(x.w));
      }
      float4 acc = make_float4(__fmul_rn(inv, x.x), __fmul_rn(inv, x.y), __fmul_rn(inv, x.z), __fmul_rn(inv, x.w));
      constexpr int K = N - 1;  // the N-1 slots, polled together
      constexpr int W = BF16 ? 2 : 4;
      const uint64_t* ptr[K];
      uint64_t words[K][W];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        int src = rank + 1 + k;
        if (src >= world) src -= world;
        ptr[k] = mine + src * gslot + (BF16 ? ((i - base) >> 1) : (i - base));
      }
      alive = poll_groups<K, W>(ptr, (1u << K) - 1u, flag, poll, rank, words);
      if (!alive) break;
#pragma unroll
      for (int k = 0; k < K; ++k) {  // reference order: rank+1, rank+2, ... (mod N)
        float4 y;
        if (BF16) {
          const uint32_t u0 = static_cast<uint32_t>(words[k][0]), u1 = static_cast<uint32_t>(words[k][1]);
          y = make_float4(bf16_bits_to_float(u0 & 0xffffu), bf16_bits_to_float(u0 >> 16),
                          bf16_bits_to_float(u1 & 0xffffu), bf16_bits_to_float(u1 >> 16));
        } else {
          y = make_float4(__uint_as_float(static_cast<uint32_t>(words[k][0])),
                          __uint_as_float(static_cast<uint32_t>(words[k][1])),
                          __uint_as_float(static_cast<uint32_t>(words[k][W - 2])),
                          __uint_as_float(static_cast<uint32_t>(words[k][W - 1])));
        }
        acc.x = __fadd_rn(__fmul_rn(inv, y.x), acc.x);
        acc.y = __fadd_rn(__fmul_rn(inv, y.y), acc.y);
        acc.z = __fadd_rn(__fmul_rn(inv, y.z), acc.z);
        acc.w = __fadd_rn(__fmul_rn(inv, y.w), acc.w);
      }
      if (!alive) break;
      update_vec<ADAM, NORM>(p, cur, i, acc, w, h, v);
      *reinterpret_cast<float4*>(hl + i) = h;
      store_v<ADAM>(p, i, v);
      *reinterpret_cast<float4*>(wl + i) = w;
      const uint64_t wa = ll_word(__float_as_uint(w.x), flag), wb = ll_word(__float_as_uint(w.y), flag);
      const uint64_t wc = ll_word(__float_as_uint(w.z), flag), wd = ll_word(__float_as_uint(w.w), flag);
      for (int k = 1; k < world; ++k) {
        int dst = rank + k;
        if (dst >= world) dst -= world;
        uint64_t* o = p.ll_weight[dst] + static_cast<uint64_t>(rank) * wslot + (i - base);
        st_ll2(o, wa, wb);
        st_ll2(o + 2, wc, wd);
      }
    }
    if (alive && blockIdx.x == 0) {  // scalar head / tail of my shard
      const uint64_t e = edge_of_thread(r, threadIdx.x);
      if (e != ~0ull) {
        SegCursor c2 = cur;
        c2.seek(e);
        float x = g[e];
        if (BF16) x = bf16_bits_to_float(float_to_bf16_bits(x));
        float acc = __fmul_rn(inv, x);
        for (int k = 1; alive && k < world; ++k) {
          int src = rank + k;
          if (src >= world) src -= world;
          uint32_t u;
          alive = poll1(mine + src * gslot + gedge + edge_index(r, e), flag, poll, src, u);
          if (alive) acc = __fadd_rn(__fmul_rn(inv, __uint_as_float(u)), acc);
        }
        if (alive) {
          float w = wl[e], h = hl[e];
          update_element<ADAM, NORM>(p, c2, e, acc, w, h);
          hl[e] = h;
          wl[e] = w;
          for (int k = 1; k < world; ++k) {
            int dst = rank + k;
            if (dst >= world) dst -= world;
            st_ll1(p.ll_weight[dst] + static_cast<uint64_t>(rank) * wslot + wedge + edge_index(r, e),
                   ll_word(__float_as_uint(w), flag));
          }
        }
      }
    }
    if (zero) {  // my own shard of diff_ (read above by exactly these threads)
      for (uint64_t j = tid; j < r.nvec; j += stride) st_vec(g + ((r.vec_lo + j) << 2), z4);
      if (blockIdx.x == 0) {
        const uint64_t e = edge_of_thread(r, threadIdx.x);
        if (e != ~0ull) g[e] = 0.f;
      }
    }
  }
  if (tracer) p.trace[3] = globaltimer_ns();

  // ---- phase 3: the peers' updated shards -> my data_ ------------------------
  // One vector of EVERY peer's shard per round: the 2(N-1) polling loads are in flight together.
  if (alive) {
    float* wl = p.data[rank];
    for (uint64_t j = tid; alive && j < max_nvec; j += stride) {
      const uint64_t* ptr[D];
      uint64_t words[D][4];
      uint64_t idx[D];
      uint32_t live = 0;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        int q = rank + 1 + d;
        if (q >= N) q -= N;
        const ShardRange r = shard_range(p.count, N, q);
        const bool in = j < r.nvec;
        idx[d] = (r.vec_lo + j) << 2;
        ptr[d] = p.ll_weight[rank] + static_cast<uint64_t>(q) * wslot + (in ? idx[d] - (r.lo & ~3ull) : 0);
        if (in) live |= 1u << d;
      }
      alive = poll_groups<D, 4>(ptr, live, flag, poll, rank, words);
      if (!alive) break;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        if (live & (1u << d))
          st_vec(wl + idx[d], make_float4(__uint_as_float(static_cast<uint32_t>(words[d][0])),
                                          __uint_as_float(static_cast<uint32_t>(words[d][1])),
                                          __uint_as_float(static_cast<uint32_t>(words[d][2])),
                                          __uint_as_float(static_cast<uint32_t>(words[d][3]))));
      }
    }
    if (alive && blockIdx.x == 0) {
      for (int d = 1; alive && d < world; ++d) {
        int q = rank + d;
        if (q >= world) q -= world;
        const ShardRange r = shard_range(p.count, world, q);
        const uint64_t e = edge_of_thread(r, threadIdx.x);
        if (e != ~0ull) {
          uint32_t u;
          alive = poll1(p.ll_weight[rank] + static_cast<uint64_t>(q) * wslot + wedge + edge_index(r, e), flag, poll, q, u);
          if (alive) wl[e] = __uint_as_float(u);
        }
      }
    }
  }
  if (tracer) p.trace[4] = globaltimer_ns();
}

template <int N, bool NORM>
void launch_ll_solver(const SyncParams& p, int grid, int block, size_t smem, cudaStream_t stream) {
  if (p.solver == kSolverAdam) {
    if (p.grad_bf16) fused_sync_sgd_ll_kernel<N, true, true, NORM><<<grid, block, smem, stream>>>(p);
    else fused_sync_sgd_ll_kernel<N, false, true, NORM><<<grid, block, smem, stream>>>(p);
  } else if (p.grad_bf16) {
    fused_sync_sgd_ll_kernel<N, true, false, NORM><<<grid, block, smem, stream>>>(p);
  } else {
    fused_sync_sgd_ll_kernel<N, false, false, NORM><<<grid, block, smem, stream>>>(p);
  }
}

template <int N>
cudaError_t launch_ll_n(const SyncParams& p, int grid, int block, size_t smem, cudaStream_t stream) {
  if (sync_normalizes(p)) launch_ll_solver<N, true>(p, grid, block, smem, stream);
  else launch_ll_solver<N, false>(p, grid, block, smem, stream);
  return cudaGetLastError();
}

}  // namespace

// 8-byte words per LL slot (body + kEdgeWords): gradient slots hold one (fp32) or two (bf16) elements per word,
// weight slots one.
void ll_slot_words(uint64_t count, int world, bool bf16, uint64_t* grad_words, uint64_t* weight_words) {
  const uint64_t max_shard = (count + world - 1) / world;
  const uint64_t body = (max_shard + 4 + 3) / 4 * 4;  // + up to 3 elements of alignment slack in front
  *weight_words = body + kEdgeWords;
  *grad_words = (bf16 ? body / 2 : body) + kEdgeWords;
}

cudaError_t launch_fused_sync_sgd_ll(const SyncParams& p, int grid, int block, int vecs_per_thread,
                                     cudaStream_t stream) {
  if (p.world < 2 || p.world > kMaxRanks || p.rank < 0 || p.rank >= p.world) return cudaErrorInvalidValue;
  if (p.mode != kModeTwoShot || p.ll_grad_stride == 0 || p.ll_weight_stride == 0) return cudaErrorInvalidValue;
  if (block <= 0) block = kLLThreads;
  if (block > kLLThreads || block < kMaxRanks || (block & 31)) return cudaErrorInvalidValue;
  if (vecs_per_thread <= 0) vecs_per_thread = 2;
  // Every CTA spins on peer data in phases 2 and 3 after feeding the peers in phase 1: the whole grid must be
  // co-resident (__launch_bounds__(512, 1): one CTA per SM).
  int dev = 0, sms = kTargetSms;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int cap = sms < kMaxCtas ? sms : kMaxCtas;
  if (grid <= 0) {  // sized by the larger phases (1 and 3 move (N-1)/N of the buffer)
    const uint64_t vecs = (p.count - p.count / p.world) >> 2;
    const uint64_t per_cta = static_cast<uint64_t>(block) * vecs_per_thread;
    uint64_t need = (vecs + per_cta - 1) / per_cta;
    if (need < 1) need = 1;
    grid = static_cast<int>(need > static_cast<uint64_t>(cap) ? cap : need);
  }
  if (grid > cap) grid = cap;
  const size_t smem = p.nseg <= kLLMaxSeg ? static_cast<size_t>(p.nseg) * (sizeof(uint64_t) + 2 * sizeof(float)) : 0;
  switch (p.world) {
    case 2: return launch_ll_n<2>(p, grid, block, smem, stream);
    case 3: return launch_ll_n<3>(p, grid, block, smem, stream);
    case 4: return launch_ll_n<4>(p, grid, block, smem, stream);
    case 5: return launch_ll_n<5>(p, grid, block, smem, stream);
    case 6: return launch_ll_n<6>(p, grid, block, smem, stream);
    case 7: return launch_ll_n<7>(p, grid, block, smem, stream);
    case 8: return launch_ll_n<8>(p, grid, block, smem, stream);
    default: return cudaErrorInvalidValue;  // world sizes 9..16 use the barrier-based kernels
  }
}

}  // namespace cosb
