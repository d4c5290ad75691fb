// flpr federated collectives: hand-written NVLink peer-memory kernels (no NCCL on these paths).
//
// Every rank owns a "symmetric" cudaMalloc'ed arena that all peers map through CUDA IPC. A collective is ONE
// kernel launched by every rank with the same grid: it (1) cross-GPU barriers on system-scope flags living in the
// peers' arenas, (2) pulls the operands straight out of the peers' HBM with 128-bit loads through NVSwitch,
// applying the federated arithmetic in registers, (3) writes (locally and/or pushes to peers), (4) barriers again.
//
//   fed_reduce_bcast  C1+C2  FedAvg weighted mean  out = sum_c (k_c / sum k) * p_c   (reference:
//                            methods/fedavg.py:386-397 + dispatch :413-421) as a two-shot reduce-scatter +
//                            all-gather; the k_c/sum(k) weights are formed in-kernel from the clients' counters.
//   fed_mix           C4     FedSTIL spatial-temporal mix out_i = sum_j W_ij * theta_j, a different row per
//                            receiving client (methods/fedstil.py:1146-1160), fused with the adaptive-layer
//                            re-initialisation (methods/fedstil.py:53-76): writes global_weight, theta master and
//                            the bf16 compute copy in the same pass.
//   fed_curv_moments  C3     FedCurv exchange (methods/fedcurv.py:621-646) pre-reduced to three moment buffers
//                            sum F_j, sum F_j p_j, sum F_j p_j^2 (the penalty at :79-86 is quadratic in p).
//   fed_gather_strided C5/C6 all-gather into the [..., K] trailing-client-dim layout
//                            (methods/fedstil_atten.py:1099-1121, methods/fedweit.py:999-1009).
//   fed_pull_copy     C2     first-contact dispatch / token all-gather: peer -> local copy with optional bf16 cast.
//
//   fed_reduce_bcast_nvls  C1+C2 through the NVSwitch's multicast / in-fabric reduction (NVLS): every rank first folds
//                            its own clients into a symmetric partial  sum_c k_c * p_c  (local HBM only), then
//                            multimem.ld_reduce adds the partials of all ranks INSIDE THE SWITCH for this rank's slice,
//                            the kernel scales by 1 / sum k and multimem.st broadcasts the slice to every rank's
//                            destination: each GPU sends and receives the buffer once, whatever the number of ranks.
//   fed_reduce_robust C1+C2  Byzantine-robust aggregate: coordinate-wise median or trimmed mean of the K uploads
//                            (unweighted), same two-shot structure as fed_reduce_bcast; every coordinate's K values are
//                            sorted in registers by a sorting network.
//
// Clients-per-rank is arbitrary (8 clients on 1/2/4/8 GPUs): sources are a table of K pointers, local or peer.
// Concurrent collectives (aggregation on a communication stream while the next round's mix runs on the compute stream)
// use different CHANNELS: each channel has its own arrival flags and epoch counters.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "ptx.cuh"

namespace flpr {

constexpr int MAX_RANKS = 8;
constexpr int MAX_CLIENTS = 32;
constexpr int MAX_LOCAL = 8;
constexpr int COMM_THREADS = 512;
constexpr int MAX_COMM_BLOCKS = 512;

// Layout of the flag page at the start of every rank's arena (uint32 units):
//   [0, MAX_COMM_BLOCKS*MAX_RANKS)       arrival flags  flag[block][src_rank]
//   [.., + MAX_COMM_BLOCKS)              per-block epoch counters (local use only)
//   [.., + 4)                            [0] error word (timeout), local use only; [2..3] 64-bit address of a
//                                        host-mapped mailbox that mirrors the error word (the host reads it without
//                                        any CUDA call, i.e. after every collective and without a device sync)
constexpr int MAX_CHANNELS = 4;
constexpr int FLAG_WORDS = MAX_COMM_BLOCKS * MAX_RANKS;
constexpr int EPOCH_OFF = FLAG_WORDS;
constexpr int CHANNEL_WORDS = FLAG_WORDS + MAX_COMM_BLOCKS;      // one channel: arrival flags + epoch counters
constexpr int ERR_OFF = MAX_CHANNELS * CHANNEL_WORDS;            // shared by all channels (relative to the page base)
constexpr int MAILBOX_OFF = ERR_OFF + 2;
constexpr int FLAG_PAGE_WORDS = ERR_OFF + 4;

struct CommCtx {
  int rank;
  int world;
  uint32_t* flags[MAX_RANKS];  // flags[r] = this channel's flags in rank r's flag page (peer-mapped; [rank] is local)
  uint32_t* err;               // local error word (+2: host mailbox address), shared by all channels
  unsigned long long timeout_ns;
};

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Block-granular cross-rank barrier: block b of every rank meets block b of every other rank.
// Release/acquire at system scope makes all prior global writes of the arriving block (including its P2P
// stores) visible to the waiter.
// Returns false when the watchdog fired (now or in an earlier collective of this communicator): the caller must then
// SKIP its load / store phase - a peer's operands may be incomplete, and a partial aggregate must never be pushed to
// the other ranks - but still runs its remaining barriers so that the epochs stay aligned. The error word is sticky
// and mirrored into a host-mapped mailbox, which the host polls after every collective (FedComm.check_errors).
__device__ __forceinline__ bool rank_barrier(const CommCtx& ctx, uint32_t epoch) {
  int fail = 0;
  __syncthreads();
  if (ctx.world > 1) {
    if (threadIdx.x < ctx.world) {
      const int peer = threadIdx.x;
      __threadfence_system();
      st_release_sys(ctx.flags[peer] + blockIdx.x * MAX_RANKS + ctx.rank, epoch);
      const uint32_t* mine = ctx.flags[ctx.rank] + blockIdx.x * MAX_RANKS + peer;
      const unsigned long long t0 = gtimer();
      // signed distance so that the 32-bit epoch may wrap
      while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
        if (gtimer() - t0 > ctx.timeout_ns) {
          fail = 1;
          uint32_t* err = ctx.err;
          if (atomicExch(err, 1u) == 0u) {
            volatile uint32_t* box = *reinterpret_cast<volatile uint32_t* const*>(ctx.err + (MAILBOX_OFF - ERR_OFF));
            if (box != nullptr) {
              *box = 1u;
              __threadfence_system();
            }
          }
          break;
        }
      }
    }
    if (threadIdx.x == 0 && *reinterpret_cast<volatile uint32_t*>(ctx.err) != 0u) fail = 1;
    fail = __syncthreads_or(fail);
  }
  return fail == 0;
}

__device__ __forceinline__ uint32_t block_epoch_begin(const CommCtx& ctx) {
  return ctx.flags[ctx.rank][EPOCH_OFF + blockIdx.x];
}
__device__ __forceinline__ void block_epoch_end(const CommCtx& ctx, uint32_t e) {
  __syncthreads();
  if (threadIdx.x == 0) ctx.flags[ctx.rank][EPOCH_OFF + blockIdx.x] = e;
}

__device__ __forceinline__ float4 f4_fma(float w, const float4& v, const float4& a) {
  return make_float4(fmaf(w, v.x, a.x), fmaf(w, v.y, a.y), fmaf(w, v.z, a.z), fmaf(w, v.w, a.w));
}
__device__ __forceinline__ void store_bf16x4(__nv_bfloat16* p, const float4& v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&lo);
  u.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = u;
}

// ----------------------------------------------------------------------------- C1 + C2
struct ReduceArgs {
  int K;                              // number of client sources
  const float* src[MAX_CLIENTS];      // upload buffers (local or peer)
  const float* cnt[MAX_CLIENTS];      // per-client train_cnt scalar (local or peer), or nullptr -> use w[]
  float w[MAX_CLIENTS];               // explicit weights when cnt == nullptr
  float* dst[MAX_RANKS];              // destination buffer on every rank (peer-mapped)
  size_t n4;                          // length in float4
  int one_shot;                       // small buffers: every rank reduces everything locally (no push phase)
};

__global__ void __launch_bounds__(COMM_THREADS)
fed_reduce_bcast_kernel(const CommCtx ctx, const ReduceArgs a) {
  __shared__ float s_w[MAX_CLIENTS];
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);  // all uploads (and counters) are complete on every rank

  if (threadIdx.x < 32) {
    float tot = 0.f;
    for (int c = 0; c < a.K; ++c) tot += (a.cnt[0] != nullptr) ? *a.cnt[c] : a.w[c];
    for (int c = threadIdx.x; c < a.K; c += 32) {
      const float k = (a.cnt[0] != nullptr) ? *a.cnt[c] : a.w[c];
      s_w[c] = (a.cnt[0] != nullptr) ? k / tot : k;
    }
  }
  __syncthreads();

  const size_t stride = (size_t)gridDim.x * blockDim.x;
  if (a.one_shot) {
    // latency-bound sizes (task tokens, BN statistics): every rank pulls all K sources and reduces the whole buffer
    // itself - no push phase, the only cross-rank traffic is the loads, and nobody writes into anybody's memory
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; ok && i < a.n4; i += stride) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c = 0; c < a.K; ++c)
        acc = f4_fma(s_w[c], ld_stream_f4(reinterpret_cast<const float4*>(a.src[c]) + i), acc);
      reinterpret_cast<float4*>(a.dst[ctx.rank])[i] = acc;
    }
    rank_barrier(ctx, e0 + 2);  // sources may be overwritten again
    block_epoch_end(ctx, e0 + 2);
    return;
  }
  // two-shot: this rank reduces slice [lo, hi) and pushes the result to every rank
  const size_t per = (a.n4 + ctx.world - 1) / ctx.world;
  const size_t lo = per * ctx.rank;
  const size_t hi = (lo + per < a.n4) ? lo + per : a.n4;
  for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; ok && i < hi; i += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c0 = 0; c0 < a.K; c0 += 8) {
      float4 v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) v[c] = ld_stream_f4(reinterpret_cast<const float4*>(a.src[c0 + c]) + i);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) acc = f4_fma(s_w[c0 + c], v[c], acc);
    }
#pragma unroll
    for (int r = 0; r < MAX_RANKS; ++r)
      if (r < ctx.world) st_stream_f4(reinterpret_cast<float4*>(a.dst[r]) + i, acc);
  }

  rank_barrier(ctx, e0 + 2);  // every rank's slice has landed everywhere
  block_epoch_end(ctx, e0 + 2);
}

// ----------------------------------------------------------------------------- C1 + C2 over NVLS (multimem)
// `ld_reduce` on a multicast address returns the SUM over every GPU bound to the multicast object of the word at that
// offset - the addition happens inside the NVSwitch; `st` on a multicast address writes the word to every GPU.
__device__ __forceinline__ float4 multimem_ld_reduce_add_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f4(float* mc, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

struct NvlsReduceArgs {
  int L;                            // clients hosted on THIS rank that take part in the mean
  const float* src[MAX_LOCAL];      // their upload slots (local HBM)
  const float* cnt[MAX_LOCAL];      // their train_cnt scalars (nullptr -> w[])
  float w[MAX_LOCAL];
  int K;                            // all participating clients (for sum k)
  const float* cnt_all[MAX_CLIENTS];  // every participating client's counter (local or peer), or nullptr -> w_total
  float w_total;                    // sum of the explicit weights when counters are not used
  float* partial;                   // this rank's symmetric partial buffer (local address)
  const float* mc_partial;          // multicast address of the partial buffers
  float* mc_dst;                    // multicast address of the destination buffers
  size_t n4;
};

__global__ void __launch_bounds__(COMM_THREADS)
fed_reduce_bcast_nvls_kernel(const CommCtx ctx, const NvlsReduceArgs a) {
  __shared__ float s_w[MAX_LOCAL];
  __shared__ float s_inv;
  const uint32_t e0 = block_epoch_begin(ctx);
  // (1) nobody is still reading last round's partial / destination; every counter is visible
  bool ok = rank_barrier(ctx, e0 + 1);
  if (threadIdx.x == 0) {
    float tot = 0.f;
    if (a.cnt_all[0] != nullptr) {
      for (int c = 0; c < a.K; ++c) tot += *a.cnt_all[c];
    } else {
      tot = a.w_total;
    }
    s_inv = 1.f / tot;
    for (int l = 0; l < a.L; ++l) s_w[l] = (a.cnt[0] != nullptr) ? *a.cnt[l] : a.w[l];
  }
  __syncthreads();
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  // (2) local fold: partial = sum over my clients of k_c * p_c  (zero when this rank hosts no participant)
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; ok && i < a.n4; i += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int l = 0; l < MAX_LOCAL; ++l)
      if (l < a.L) acc = f4_fma(s_w[l], ld_stream_f4(reinterpret_cast<const float4*>(a.src[l]) + i), acc);
    reinterpret_cast<float4*>(a.partial)[i] = acc;
  }
  ok = rank_barrier(ctx, e0 + 2) && ok;  // every rank's partial is complete and visible system-wide
  // (3) my slice: in-switch reduction of the partials, scale, multicast store into every rank's destination
  const size_t per = (a.n4 + ctx.world - 1) / ctx.world;
  const size_t lo = per * ctx.rank;
  const size_t hi = (lo + per < a.n4) ? lo + per : a.n4;
  const float inv = s_inv;
  // The barriers pair block b of this rank with block b of every peer, so a block may only consume what the SAME
  // block index produced on the peers: walk this block's own fold positions (b*T + t + k*stride) and keep the ones
  // that fall into my slice. The slice is still spread evenly over the grid.
  const size_t first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t skip = (lo > first) ? (lo - first + stride - 1) / stride : 0;
  for (size_t i = first + skip * stride; ok && i < hi; i += stride) {
    float4 v = multimem_ld_reduce_add_f4(a.mc_partial + 4 * i);
    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
    multimem_st_f4(a.mc_dst + 4 * i, v);
  }
  rank_barrier(ctx, e0 + 3);  // every slice has landed everywhere
  block_epoch_end(ctx, e0 + 3);
}

// ----------------------------------------------------------------------------- C1 + C2 robust (median / trimmed mean)
// Order of the K values of one coordinate: (value, position in the client list), NaN above +inf, -0.0 == +0.0 (the
// tie goes to the lower position) - what a stable sort of the K values gives. Each value becomes one 64-bit key that
// sorts in exactly that order and still holds the value's bits:
//   high word  order key of the value: NaN -> 0xFFFFFFFF, +-0 -> 0x80000000, x > 0 -> bits | 0x80000000, x < 0 -> ~bits
//   low word   [31:27] position, [23] sign bit, [22:0] mantissa
// The exponent is recovered from the high word (negative values: from ~high), so the key decodes to the original bits,
// signed zeros and NaN payloads included. The padding of a K-bucket (all ones) sorts after every real key.
constexpr int ROBUST_MEDIAN = 0;
constexpr int ROBUST_TRIMMED_MEAN = 1;

struct RobustArgs {
  int K;                              // number of client sources
  int rule;                           // ROBUST_MEDIAN / ROBUST_TRIMMED_MEAN
  int b;                              // trimmed mean: sorted positions [b, K - b) are kept
  const float* src[MAX_CLIENTS];      // upload buffers (local or peer)
  float* dst[MAX_RANKS];              // destination buffer on every rank (peer-mapped)
  size_t n4;                          // length in float4
};

__device__ __forceinline__ uint32_t f32_bits(float x) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(x);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  return u;
#endif
}

__device__ __forceinline__ unsigned long long robust_key(float x, int pos) {
  const uint32_t u = f32_bits(x);
  const uint32_t ax = u & 0x7FFFFFFFu;
  const uint32_t hi = ax > 0x7F800000u ? 0xFFFFFFFFu : (ax == 0u ? 0x80000000u : ((u >> 31) ? ~u : (u | 0x80000000u)));
  const uint32_t lo = ((uint32_t)pos << 27) | ((u >> 31) << 23) | (u & 0x007FFFFFu);
  return ((unsigned long long)hi << 32) | lo;
}

__device__ __forceinline__ float robust_value(unsigned long long key) {
  const uint32_t hi = (uint32_t)(key >> 32), lo = (uint32_t)key;
  const uint32_t e = (((hi >> 31) ? hi : ~hi) >> 23) & 0xFFu;
  return __uint_as_float((((lo >> 23) & 1u) << 31) | (e << 23) | (lo & 0x007FFFFFu));
}

__device__ __forceinline__ void cmp_swap(unsigned long long& a, unsigned long long& b) {
  const bool s = a > b;
  const unsigned long long lo = s ? b : a;
  b = s ? a : b;
  a = lo;
}

// Batcher's odd-even merge sort of P = 2^LOG keys. Stage (p, d) with p = 2^lp, d = 2^(lp - ld) compares x and x + d
// for every x with (x - d % p) mod 2d < d inside one block of 2p. Every loop has a constant trip count, so full
// unrolling turns every index into a constant and the keys stay in registers.
template <int P, int LOG>
__device__ __forceinline__ void sort_keys(unsigned long long (&k)[P]) {
#pragma unroll
  for (int lp = 0; lp < LOG; ++lp)
#pragma unroll
    for (int ld = 0; ld < LOG; ++ld)
#pragma unroll
      for (int x = 0; x < P; ++x) {
        const int p = 1 << lp, d = ld <= lp ? 1 << (lp - ld) : 1, r = d % p;
        if (ld <= lp && x + d < P && x >= r && (x - r) % (2 * d) < d && x / (2 * p) == (x + d) / (2 * p))
          cmp_swap(k[x], k[x + d]);
      }
}

// (0.5 * lo + 0.5 * hi, each product and the sum rounded on its own: no FMA contraction)
__device__ __forceinline__ float robust_midpoint(float lo, float hi) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(__fmul_rn(0.5f, lo), __fmul_rn(0.5f, hi));
#else
  return 0.5f * lo + 0.5f * hi;  // (host builds are ISO C++: no contraction)
#endif
}

template <int P, int LOG>
__device__ __forceinline__ void robust_body(const CommCtx& ctx, const RobustArgs& a, size_t e_lo, size_t e_hi) {
  const int K = a.K;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t e = e_lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < e_hi; e += stride) {
    unsigned long long k[P];
#pragma unroll
    for (int c = 0; c < P; ++c) k[c] = c < K ? robust_key(a.src[c][e], c) : ~0ull;
    sort_keys<P, LOG>(k);
    float out;
    if (a.rule == ROBUST_MEDIAN) {
      // odd K: position (K-1)/2; even K: midpoint of positions K/2-1 and K/2
      const int m_lo = (K - 1) >> 1, m_hi = K >> 1;
      unsigned long long lo = 0ull, hi = 0ull;
#pragma unroll
      for (int j = 0; j < P; ++j) {
        if (j == m_lo) lo = k[j];
        if (j == m_hi) hi = k[j];
      }
      out = (m_lo == m_hi) ? robust_value(lo) : robust_midpoint(robust_value(lo), robust_value(hi));
    } else {
      // sum of the kept positions in ascending order; -0.0 is the exact identity of the addition
      float acc = -0.f;
#pragma unroll
      for (int j = 0; j < P; ++j)
        if (j >= a.b && j < K - a.b) acc += robust_value(k[j]);
      out = acc / (float)(K - 2 * a.b);
    }
#pragma unroll
    for (int r = 0; r < MAX_RANKS; ++r)
      if (r < ctx.world) a.dst[r][e] = out;
  }
}

__global__ void __launch_bounds__(COMM_THREADS)
fed_reduce_robust_kernel(const CommCtx ctx, const RobustArgs a) {
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);  // all uploads are complete on every rank
  // two-shot: this rank reduces slice [lo, hi) (in float4 units, as fed_reduce_bcast) and pushes it to every rank
  const size_t per = (a.n4 + ctx.world - 1) / ctx.world;
  const size_t lo = per * ctx.rank;
  const size_t hi = (lo + per < a.n4) ? lo + per : a.n4;
  if (ok && lo < hi) {
    const size_t e_lo = 4 * lo, e_hi = 4 * hi;
    if (a.K <= 2) robust_body<2, 1>(ctx, a, e_lo, e_hi);
    else if (a.K <= 4) robust_body<4, 2>(ctx, a, e_lo, e_hi);
    else if (a.K <= 8) robust_body<8, 3>(ctx, a, e_lo, e_hi);
    else if (a.K <= 16) robust_body<16, 4>(ctx, a, e_lo, e_hi);
    else robust_body<32, 5>(ctx, a, e_lo, e_hi);
  }
  rank_barrier(ctx, e0 + 2);  // all robust slices are in every rank's dst; uploads may be rewritten
  block_epoch_end(ctx, e0 + 2);
}

// ----------------------------------------------------------------------------- C4
struct MixArgs {
  int K;                            // all clients
  int L;                            // local (receiving) clients on this rank
  const float* src[MAX_CLIENTS];    // theta uploads
  float w[MAX_LOCAL][MAX_CLIENTS];  // mixing rows for the local clients (host-provided)
  const float* w_dev;               // optional device-resident rows [L*K]: no host sync to launch the mix
  float* dst_g[MAX_LOCAL];          // global_weight of local client i          (nullable)
  float* dst_theta[MAX_LOCAL];      // theta master of local client i           (nullable)
  __nv_bfloat16* dst_bf16[MAX_LOCAL];  // bf16 compute copy of theta            (nullable)
  size_t n4;
};

template <int L>
__device__ __forceinline__ void mix_body(const MixArgs& a, const float (*sw)[MAX_CLIENTS]) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n4; i += stride) {
    float4 acc[L];
#pragma unroll
    for (int l = 0; l < L; ++l) acc[l] = make_float4(0.f, 0.f, 0.f, 0.f);
    // 8 sources at a time keeps 8 x 16 B per thread in flight without blowing the register file
    for (int c0 = 0; c0 < a.K; c0 += 8) {
      float4 v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) v[c] = ld_stream_f4(reinterpret_cast<const float4*>(a.src[c0 + c]) + i);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) {
#pragma unroll
          for (int l = 0; l < L; ++l) acc[l] = f4_fma(sw[l][c0 + c], v[c], acc[l]);
        }
    }
#pragma unroll
    for (int l = 0; l < L; ++l) {
      if (a.dst_g[l]) reinterpret_cast<float4*>(a.dst_g[l])[i] = acc[l];
      if (a.dst_theta[l]) reinterpret_cast<float4*>(a.dst_theta[l])[i] = acc[l];
      if (a.dst_bf16[l]) store_bf16x4(a.dst_bf16[l] + 4 * i, acc[l]);
    }
  }
}

__global__ void __launch_bounds__(COMM_THREADS) fed_mix_kernel(const CommCtx ctx, const MixArgs a) {
  __shared__ float sw[MAX_LOCAL][MAX_CLIENTS];
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);
  for (int i = threadIdx.x; i < a.L * a.K; i += blockDim.x) {
    const int l = i / a.K, c = i - l * a.K;
    sw[l][c] = a.w_dev ? a.w_dev[i] : a.w[l][c];
  }
  __syncthreads();
  switch (ok ? a.L : 0) {
    case 0: break;  // rank hosts no receiving client this round (or the watchdog fired): barriers only
    case 1: mix_body<1>(a, sw); break;
    case 2: mix_body<2>(a, sw); break;
    case 3: mix_body<3>(a, sw); break;
    case 4: mix_body<4>(a, sw); break;
    case 5: mix_body<5>(a, sw); break;
    case 6: mix_body<6>(a, sw); break;
    case 7: mix_body<7>(a, sw); break;
    default: mix_body<8>(a, sw); break;
  }
  rank_barrier(ctx, e0 + 2);  // nobody may overwrite an upload buffer while a peer is still reading it
  block_epoch_end(ctx, e0 + 2);
}

// ----------------------------------------------------------------------------- C3
struct CurvArgs {
  int K;
  const float* fisher[MAX_CLIENTS];
  const float* param[MAX_CLIENTS];
  float* dst_f[MAX_RANKS];    // sum_j F_j
  float* dst_fp[MAX_RANKS];   // sum_j F_j p_j
  float* dst_fpp[MAX_RANKS];  // sum_j F_j p_j^2
  size_t n4;
};

__global__ void __launch_bounds__(COMM_THREADS) fed_curv_moments_kernel(const CommCtx ctx, const CurvArgs a) {
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);
  const size_t per = (a.n4 + ctx.world - 1) / ctx.world;
  const size_t lo = per * ctx.rank;
  const size_t hi = (lo + per < a.n4) ? lo + per : a.n4;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; ok && i < hi; i += stride) {
    float4 sf = make_float4(0.f, 0.f, 0.f, 0.f), sfp = sf, sfpp = sf;
    for (int c0 = 0; c0 < a.K; c0 += 4) {
      float4 f[4], q[4];
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c0 + c < a.K) {
          f[c] = ld_stream_f4(reinterpret_cast<const float4*>(a.fisher[c0 + c]) + i);
          q[c] = ld_stream_f4(reinterpret_cast<const float4*>(a.param[c0 + c]) + i);
        }
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c0 + c < a.K) {
          sf.x += f[c].x; sf.y += f[c].y; sf.z += f[c].z; sf.w += f[c].w;
          const float4 fp = make_float4(f[c].x * q[c].x, f[c].y * q[c].y, f[c].z * q[c].z, f[c].w * q[c].w);
          sfp.x += fp.x; sfp.y += fp.y; sfp.z += fp.z; sfp.w += fp.w;
          sfpp.x = fmaf(fp.x, q[c].x, sfpp.x); sfpp.y = fmaf(fp.y, q[c].y, sfpp.y);
          sfpp.z = fmaf(fp.z, q[c].z, sfpp.z); sfpp.w = fmaf(fp.w, q[c].w, sfpp.w);
        }
    }
#pragma unroll
    for (int r = 0; r < MAX_RANKS; ++r)
      if (r < ctx.world) {
        st_stream_f4(reinterpret_cast<float4*>(a.dst_f[r]) + i, sf);
        st_stream_f4(reinterpret_cast<float4*>(a.dst_fp[r]) + i, sfp);
        st_stream_f4(reinterpret_cast<float4*>(a.dst_fpp[r]) + i, sfpp);
      }
  }
  rank_barrier(ctx, e0 + 2);
  block_epoch_end(ctx, e0 + 2);
}

// ----------------------------------------------------------------------------- C5 / C6
struct GatherArgs {
  int K;
  const float* src[MAX_CLIENTS];
  float* dst;  // local [n, K] (client index is the fastest dim)
  size_t n;    // elements per client
};

__global__ void __launch_bounds__(COMM_THREADS) fed_gather_strided_kernel(const CommCtx ctx, const GatherArgs a) {
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);
  const size_t n4 = ok ? a.n / 4 : 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    for (int c0 = 0; c0 < a.K; c0 += 8) {
      float4 v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) v[c] = ld_stream_f4(reinterpret_cast<const float4*>(a.src[c0 + c]) + i);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c0 + c < a.K) {
          float* o = a.dst + (4 * i) * a.K + (c0 + c);
          o[0] = v[c].x; o[a.K] = v[c].y; o[2 * (size_t)a.K] = v[c].z; o[3 * (size_t)a.K] = v[c].w;
        }
    }
  }
  for (size_t e = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; ok && e < a.n; e += stride)
    for (int c = 0; c < a.K; ++c) a.dst[e * a.K + c] = a.src[c][e];
  rank_barrier(ctx, e0 + 2);
  block_epoch_end(ctx, e0 + 2);
}

// ----------------------------------------------------------------------------- C2 (pull copy)
struct CopyArgs {
  const float* src;          // peer or local
  float* dst;                // local fp32 (nullable)
  __nv_bfloat16* dst_bf16;   // local bf16 (nullable)
  size_t n4;
};

__global__ void __launch_bounds__(COMM_THREADS) fed_pull_copy_kernel(const CommCtx ctx, const CopyArgs a) {
  const uint32_t e0 = block_epoch_begin(ctx);
  const bool ok = rank_barrier(ctx, e0 + 1);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!ok) i = a.n4;
  for (; i + 3 * stride < a.n4; i += 4 * stride) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld_stream_f4(reinterpret_cast<const float4*>(a.src) + i + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (a.dst) reinterpret_cast<float4*>(a.dst)[i + u * stride] = v[u];
      if (a.dst_bf16) store_bf16x4(a.dst_bf16 + 4 * (i + u * stride), v[u]);
    }
  }
  for (; i < a.n4; i += stride) {
    const float4 v = ld_stream_f4(reinterpret_cast<const float4*>(a.src) + i);
    if (a.dst) reinterpret_cast<float4*>(a.dst)[i] = v;
    if (a.dst_bf16) store_bf16x4(a.dst_bf16 + 4 * i, v);
  }
  rank_barrier(ctx, e0 + 2);
  block_epoch_end(ctx, e0 + 2);
}

__global__ void fed_barrier_kernel(const CommCtx ctx) {
  const uint32_t e0 = block_epoch_begin(ctx);
  rank_barrier(ctx, e0 + 1);
  block_epoch_end(ctx, e0 + 1);
}

static char g_comm_err[256] = {0};
static int g_one_shot_bytes = 1 << 20;   // reduce_bcast buffers up to this size take the one-shot path
static int comm_fail(cudaError_t e, const char* where) {
  snprintf(g_comm_err, sizeof(g_comm_err), "%s: %s", where, cudaGetErrorString(e));
  return (int)e;
}
static int clamp_blocks(int b) { return b < 1 ? 1 : (b > MAX_COMM_BLOCKS ? MAX_COMM_BLOCKS : b); }

}  // namespace flpr

using namespace flpr;

extern "C" {

const char* flpr_comm_last_error() { return g_comm_err; }
int flpr_comm_flag_page_bytes() { return FLAG_PAGE_WORDS * 4; }
int flpr_comm_max_clients() { return MAX_CLIENTS; }
int flpr_comm_max_local() { return MAX_LOCAL; }
int flpr_comm_max_ranks() { return MAX_RANKS; }

int flpr_symm_alloc(void** ptr, size_t bytes) {
  cudaError_t e = cudaMalloc(ptr, bytes);
  if (e != cudaSuccess) return comm_fail(e, "cudaMalloc(symmetric arena)");
  e = cudaMemset(*ptr, 0, bytes);
  if (e != cudaSuccess) return comm_fail(e, "cudaMemset(symmetric arena)");
  return 0;
}
int flpr_symm_free(void* ptr) { return (int)cudaFree(ptr); }
int flpr_ipc_get_handle(void* ptr, unsigned char* out64) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
  if (e != cudaSuccess) return comm_fail(e, "cudaIpcGetMemHandle");
  memcpy(out64, &h, sizeof(h));
  return 0;
}
int flpr_ipc_open_handle(const unsigned char* in64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, in64, sizeof(h));
  cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return comm_fail(e, "cudaIpcOpenMemHandle");
  return 0;
}
int flpr_ipc_close(void* ptr) { return (int)cudaIpcCloseMemHandle(ptr); }

// Same-process multi-device mode (tests / single-process multi-GPU): enable direct peer access.
int flpr_enable_peer(int dev, int peer) {
  int can = 0;
  cudaDeviceCanAccessPeer(&can, dev, peer);
  if (!can) return -1;
  int cur;
  cudaGetDevice(&cur);
  cudaSetDevice(dev);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  cudaSetDevice(cur);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return 0;
  }
  return (int)e;
}

static thread_local int t_channel = 0;   // set by flpr_comm_set_channel for the calling thread's next launches

static CommCtx make_ctx(int rank, int world, void* const* flag_pages, double timeout_s) {
  bind_device_of(flag_pages[rank]);
  CommCtx c;
  c.rank = rank;
  c.world = world;
  const int ch = (t_channel >= 0 && t_channel < MAX_CHANNELS) ? t_channel : 0;
  for (int r = 0; r < MAX_RANKS; ++r)
    c.flags[r] = r < world ? reinterpret_cast<uint32_t*>(flag_pages[r]) + (size_t)ch * CHANNEL_WORDS : nullptr;
  c.err = reinterpret_cast<uint32_t*>(flag_pages[rank]) + ERR_OFF;
  c.timeout_ns = (unsigned long long)(timeout_s * 1e9);
  return c;
}

int flpr_comm_read_error(void* local_flag_page, int* out) {
  uint32_t v = 0;
  cudaError_t e = cudaMemcpy(&v, reinterpret_cast<uint32_t*>(local_flag_page) + ERR_OFF, 4, cudaMemcpyDeviceToHost);
  *out = (int)v;
  return (int)e;
}

// Register a host-mapped (pinned, UVA) 32-bit mailbox that the watchdog mirrors the error word into.
int flpr_comm_set_mailbox(void* local_flag_page, void* host_mailbox) {
  unsigned long long addr = reinterpret_cast<unsigned long long>(host_mailbox);
  return (int)cudaMemcpy(reinterpret_cast<uint32_t*>(local_flag_page) + MAILBOX_OFF, &addr, 8, cudaMemcpyHostToDevice);
}

// Channel (0 .. MAX_CHANNELS-1) used by the collectives the CALLING THREAD launches from now on. Collectives that may
// run concurrently (different streams) must use different channels; every rank must use the same channel for the same
// collective.
int flpr_comm_set_channel(int channel) {
  if (channel < 0 || channel >= MAX_CHANNELS) return -1;
  t_channel = channel;
  return 0;
}
int flpr_comm_max_channels() { return MAX_CHANNELS; }

int flpr_comm_barrier(int rank, int world, void* const* flag_pages, double timeout_s, cudaStream_t st) {
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  fed_barrier_kernel<<<1, 32, 0, st>>>(c);
  return (int)cudaGetLastError();
}

int flpr_comm_reduce_bcast(int rank, int world, void* const* flag_pages, double timeout_s, int K,
                           const float* const* src, const float* const* cnt, const float* w, float* const* dst,
                           size_t n, int nblocks, cudaStream_t st) {
  if (K > MAX_CLIENTS || world > MAX_RANKS) return -1;
  if (n % 4) return -2;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  ReduceArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  for (int i = 0; i < K; ++i) {
    a.src[i] = src[i];
    a.cnt[i] = cnt ? cnt[i] : nullptr;
    a.w[i] = w ? w[i] : 0.f;
  }
  for (int r = 0; r < world; ++r) a.dst[r] = dst[r];
  a.n4 = n / 4;
  a.one_shot = (world > 1 && n * sizeof(float) <= (size_t)g_one_shot_bytes) ? 1 : 0;
  int blocks = clamp_blocks(nblocks);
  if (a.one_shot) {                      // a few KB .. 1 MB: don't spread 32 k floats over hundreds of barrier-ing blocks
    const int need = (int)((a.n4 + COMM_THREADS - 1) / COMM_THREADS);
    blocks = need < 1 ? 1 : (need < blocks ? need : blocks);
  }
  fed_reduce_bcast_kernel<<<blocks, COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

// NVLS variant: `src` / `cnt` are this rank's participating clients (local pointers, L <= MAX_LOCAL), `cnt_all` the
// counters of all K participants (nullable together with `cnt`: then `w` / `w_total` are used), `partial` the local
// address and `mc_partial` / `mc_dst` the MULTICAST addresses of the symmetric partial / destination buffers.
int flpr_comm_reduce_bcast_nvls(int rank, int world, void* const* flag_pages, double timeout_s, int L,
                                const float* const* src, const float* const* cnt, const float* w, int K,
                                const float* const* cnt_all, float w_total, float* partial, const float* mc_partial,
                                float* mc_dst, size_t n, int nblocks, cudaStream_t st) {
  if (L > MAX_LOCAL || L < 0 || K > MAX_CLIENTS || world > MAX_RANKS) return -1;
  if (n % 4) return -2;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  NvlsReduceArgs a;
  memset(&a, 0, sizeof(a));
  a.L = L;
  for (int l = 0; l < L; ++l) {
    a.src[l] = src[l];
    a.cnt[l] = cnt ? cnt[l] : nullptr;
    a.w[l] = w ? w[l] : 0.f;
  }
  a.K = K;
  for (int i = 0; i < K; ++i) a.cnt_all[i] = cnt_all ? cnt_all[i] : nullptr;
  a.w_total = w_total;
  a.partial = partial;
  a.mc_partial = mc_partial;
  a.mc_dst = mc_dst;
  a.n4 = n / 4;
  fed_reduce_bcast_nvls_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

void flpr_comm_set_one_shot_bytes(int bytes) { g_one_shot_bytes = bytes; }

// Robust aggregate of K uploads into every rank's `dst`: rule 0 = coordinate-wise median, 1 = trimmed mean of sorted
// positions [b, K - b). Returns -1 (K or world out of range), -2 (n % 4), -3 (unknown rule, or b outside [0, K/2) for
// the trimmed mean / not 0 for the median).
int flpr_comm_reduce_robust(int rank, int world, void* const* flag_pages, double timeout_s, int K,
                            const float* const* src, float* const* dst, int rule, int b, size_t n, int nblocks,
                            cudaStream_t st) {
  if (K < 1 || K > MAX_CLIENTS || world < 1 || world > MAX_RANKS) return -1;
  if (n % 4) return -2;
  if (rule == ROBUST_MEDIAN ? b != 0 : (rule != ROBUST_TRIMMED_MEAN || b < 0 || 2 * b >= K)) return -3;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  RobustArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  a.rule = rule;
  a.b = b;
  for (int i = 0; i < K; ++i) a.src[i] = src[i];
  for (int r = 0; r < world; ++r) a.dst[r] = dst[r];
  a.n4 = n / 4;
  fed_reduce_robust_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

int flpr_comm_mix(int rank, int world, void* const* flag_pages, double timeout_s, int K, int L,
                  const float* const* src, const float* w_rows /* host [L*K] or null */,
                  const float* w_dev /* device [L*K] or null */, float* const* dst_g,
                  float* const* dst_theta, void* const* dst_bf16, size_t n, int nblocks, cudaStream_t st) {
  if (K > MAX_CLIENTS || L > MAX_LOCAL || L < 0 || world > MAX_RANKS) return -1;
  if (n % 4) return -2;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  MixArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  a.L = L;
  for (int i = 0; i < K; ++i) a.src[i] = src[i];
  for (int l = 0; l < L; ++l) {
    for (int i = 0; i < K; ++i) a.w[l][i] = w_rows ? w_rows[l * K + i] : 0.f;
    a.dst_g[l] = dst_g ? dst_g[l] : nullptr;
    a.dst_theta[l] = dst_theta ? dst_theta[l] : nullptr;
    a.dst_bf16[l] = dst_bf16 ? reinterpret_cast<__nv_bfloat16*>(dst_bf16[l]) : nullptr;
  }
  a.w_dev = w_dev;
  a.n4 = n / 4;
  fed_mix_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

int flpr_comm_curv_moments(int rank, int world, void* const* flag_pages, double timeout_s, int K,
                           const float* const* fisher, const float* const* param, float* const* dst_f,
                           float* const* dst_fp, float* const* dst_fpp, size_t n, int nblocks, cudaStream_t st) {
  if (K > MAX_CLIENTS || world > MAX_RANKS) return -1;
  if (n % 4) return -2;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  CurvArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  for (int i = 0; i < K; ++i) {
    a.fisher[i] = fisher[i];
    a.param[i] = param[i];
  }
  for (int r = 0; r < world; ++r) {
    a.dst_f[r] = dst_f[r];
    a.dst_fp[r] = dst_fp[r];
    a.dst_fpp[r] = dst_fpp[r];
  }
  a.n4 = n / 4;
  fed_curv_moments_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

int flpr_comm_gather_strided(int rank, int world, void* const* flag_pages, double timeout_s, int K,
                             const float* const* src, float* dst, size_t n, int nblocks, cudaStream_t st) {
  if (K > MAX_CLIENTS || world > MAX_RANKS) return -1;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  GatherArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  for (int i = 0; i < K; ++i) a.src[i] = src[i];
  a.dst = dst;
  a.n = n;
  fed_gather_strided_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

int flpr_comm_pull_copy(int rank, int world, void* const* flag_pages, double timeout_s, const float* src, float* dst,
                        void* dst_bf16, size_t n, int nblocks, cudaStream_t st) {
  if (n % 4) return -2;
  CommCtx c = make_ctx(rank, world, flag_pages, timeout_s);
  CopyArgs a;
  a.src = src;
  a.dst = dst;
  a.dst_bf16 = reinterpret_cast<__nv_bfloat16*>(dst_bf16);
  a.n4 = n / 4;
  fed_pull_copy_kernel<<<clamp_blocks(nblocks), COMM_THREADS, 0, st>>>(c, a);
  return (int)cudaGetLastError();
}

}  // extern "C"
