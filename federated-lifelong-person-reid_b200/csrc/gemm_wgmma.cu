// flpr wgmma GEMM / implicit-GEMM convolution for sm_90a (H100).
//
//   D[M,N] = alpha * sum_k A[m,k] * B[n,k]  (+bias, +residual, ReLU)      bf16 operands, fp32 accumulate in registers
//
// One 128 x BN output tile at a time per CTA. Warp-specialised, 3 warpgroups (384 threads):
//   warpgroup 0   : TMA producer  (one elected thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier
//                   complete_tx), register budget handed to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2: MMA + epilogue, each owns 64 rows of the tile (wgmma m64nBNk16, accumulators in registers). The
//                   epilogue stages the accumulators through shared memory 64 columns at a time so that every warp
//                   then holds 32 consecutive columns of 32 rows (lane = row) for the fused epilogue.
// The kernel is persistent: CTAs walk tiles t = blockIdx.x, + gridDim.x, ... and the producer runs ahead across tile
// boundaries, so the next tile's operands stream in while the MMA warpgroups run the epilogue of the current one.
//
// Operand modes (per operand):
//   OP_KMAJOR  : row-major [rows, K], K contiguous           (forward GEMMs, dgrad A operand)
//   OP_MNMAJOR : row-major [K, rows], rows contiguous        (wgrad operands, dgrad B operand) -> no transposes
//   OP_CONV    : A only. NHWC activation tensor, 4-D TMA box per filter tap; zero padding comes from TMA
//                out-of-bounds fill, so a 3x3 convolution is 9*(C/64) K-blocks of a plain GEMM pipeline.
//
// This is the compute kernel behind ops/gemm.py (classifier, 1x1 / 3x3 bottleneck convs, gallery-vs-query
// similarity). Reference call sites it replaces: models/resnet.py:121-141 (bottleneck convs),
// models/resnet.py:321 (classifier), tools/evaluate.py:100 (per-query torch.mm).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "ptx.cuh"

namespace flpr {

enum { OP_KMAJOR = 0, OP_MNMAJOR = 1, OP_CONV = 2, OP_TAPFLIP = 3 };
enum { EPI_GENERIC = 0, EPI_LEAN = 1 };

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle atom row
constexpr int MMA_K = 16;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB

struct GemmParams {
  int M, N, K;          // K = total reduction length (conv: taps * C)
  int kb_per_split;     // K-blocks handled by one blockIdx.z
  int kb_total;
  // epilogue
  void* out;
  long long ldo;
  int out_bf16;
  int trans_out;
  int atomic_add;
  float alpha;
  const float* bias_n;
  const float* bias_m;
  int relu;
  const __nv_bfloat16* residual;
  // conv geometry (A operand in OP_CONV mode)
  int cH, cW, cC, cTH, cNB, cKW, cPadH, cPadW, cTilesPerImg, cSplits;
  long long tap_stride;  // conv wgrad: output column offset per filter tap
  long long split_stride;  // split-K: element offset between the per-split partial outputs (deterministic reduction)
  int cTaps;             // KH*KW (OP_TAPFLIP: B column offset = (cTaps-1-tap) * N)
  int cStride;           // convolution stride (A operand: TMA element strides), 1 or 2
  // persistent scheduling
  int tiles_m, tiles_n, tiles_z, tiles_total;
  // fused batch-norm statistics: per (m-tile, 32-row quarter) column partials of sum / sum^2 of the fp32 accumulators
  float* col_part;       // [tiles_m * 4][2][N] or nullptr
  int debug;             // FLPR_GEMM_DEBUG bit mask (bottleneck isolation, results are WRONG when set):
                         //   1 skip the epilogue body, 2 skip global stores, 4 skip TMA loads (MMA on stale smem)
};

// Shared memory: operand ring | accumulator staging (2 MMA warpgroups x 64 rows x 64 fp32 columns) | store staging
// (8 warps x 32 rows x 80 B) | barriers. Up to 227 KB per block on H100: the ring gets what the tile width leaves.
template <int BN>
struct GemmLayout {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = (BN == 64) ? 6 : (BN == 128 ? 5 : 3);
  static constexpr int THREADS = 384;
  static constexpr int ACC_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int ACC_BYTES = 2 * 64 * 64 * 4;
  static constexpr int STORE_OFFSET = ACC_OFFSET + ACC_BYTES;
  static constexpr int STORE_BYTES = 8 * 32 * 80;
  static constexpr int BAR_OFFSET = STORE_OFFSET + STORE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;  // barriers + alignment slack
  static_assert(TOTAL <= 227 * 1024, "shared memory budget of an H100 block");
};

// ------------------------------------------------------------------------------------------------- shared pieces
// TMA loads of one K-block (BK = 64) of both operands into one ring stage.
// CL == 2 (CTA pair = 2-CTA cluster on the same N tile): each CTA loads its own A tile and HALF of the shared B tile,
// multicast into the same stage of both CTAs, so every byte of B crosses L2 -> SM once per pair instead of twice.
template <int BN, int A_MODE, int B_MODE, int CL = 1>
__device__ __forceinline__ void load_kblock(const GemmParams& p, const CUtensorMap* tmA, const CUtensorMap* tmB,
                                            uint8_t* sa, uint8_t* sb, uint64_t* bar, int kb, int mt, int m0, int n0,
                                            int ztap, int rank = 0) {
  auto b2d = [&](void* d, int c0, int c1) {
    if constexpr (CL == 2) tma_load_2d_mc(d, tmB, bar, c0, c1, 0x3); else tma_load_2d(d, tmB, bar, c0, c1);
  };
  auto b4d = [&](void* d, int c0, int c1, int c2, int c3) {
    if constexpr (CL == 2) tma_load_4d_mc(d, tmB, bar, c0, c1, c2, c3, 0x3); else tma_load_4d(d, tmB, bar, c0, c1, c2, c3);
  };
  int tapA = 0;
  if constexpr (A_MODE == OP_KMAJOR) {
    tma_load_2d(sa, tmA, bar, kb * BK, m0);
  } else if constexpr (A_MODE == OP_MNMAJOR) {
    tma_load_2d(sa, tmA, bar, m0, kb * BK);
    tma_load_2d(sa + 64 * 128, tmA, bar, m0 + 64, kb * BK);
  } else {
    const int chunks = p.cC / BK;
    tapA = kb / chunks;
    const int cc = kb - tapA * chunks;
    const int kh = tapA / p.cKW;
    const int kw = tapA - kh * p.cKW;
    int img0, h0;
    if (p.cTilesPerImg <= 1) {
      img0 = mt * p.cNB;
      h0 = 0;
    } else {
      img0 = mt / p.cTilesPerImg;
      h0 = (mt - img0 * p.cTilesPerImg) * p.cTH;
    }
    tma_load_4d(sa, tmA, bar, cc * BK, kw - p.cPadW, h0 * p.cStride + kh - p.cPadH, img0);
  }
  if constexpr (B_MODE == OP_KMAJOR) {
    constexpr int ROWS = BN / CL;                         // (the tensor map's box is ROWS x 64)
    b2d(sb + rank * ROWS * 128, kb * BK, n0 + rank * ROWS);
  } else if constexpr (B_MODE == OP_MNMAJOR) {
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
      if (j % CL == rank) b2d(sb + j * 64 * 128, n0 + j * 64, kb * BK);
  } else if constexpr (B_MODE == OP_TAPFLIP) {
    // data-gradient of a convolution straight from the forward weight W[Cout, taps, Cin]: for A tap t the B operand
    // is W[:, taps-1-t, :] viewed as [K = Cout rows (stride taps*Cin), N = Cin contiguous] -> no flipped copy.
    const int chunks = p.cC / BK;                         // A channels (= Cout of the forward conv) per tap
    const int cc = kb - tapA * chunks;
    const int col0 = (p.cTaps - 1 - tapA) * p.N + n0;
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
      if (j % CL == rank) b2d(sb + j * 64 * 128, col0 + j * 64, cc * BK);
  } else {
    // weight-gradient of a convolution: K runs over pixels (64 per block), the filter tap (ztap) shifts the 4-D
    // box, zero padding comes from TMA out-of-bounds fill
    const int kh = ztap / p.cKW;
    const int kw = ztap - kh * p.cKW;
    const int p0 = kb * BK;
    const int hw = p.cH * p.cW;
    const int img = p0 / hw;
    const int h0 = (p0 - img * hw) / p.cW;
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
      if (j % CL == rank) b4d(sb + j * 64 * 128, n0 + j * 64, kw - p.cPadW, h0 + kh - p.cPadH, img);
  }
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 64) wgmma_m64n64k16<TA, TB>(acc, da, db, 1u);
  else if constexpr (BN == 128) wgmma_m64n128k16<TA, TB>(acc, da, db, 1u);
  else wgmma_m64n256k16<TA, TB>(acc, da, db, 1u);
}

// The four MMA_K = 16 steps of one K-block for the 64 rows of warpgroup `wg` (issued by the whole warpgroup).
template <int BN, int A_MODE, int B_MODE>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint32_t sa, int wg) {
  constexpr int TA = (A_MODE == OP_MNMAJOR) ? 1 : 0;
  constexpr int TB = (B_MODE != OP_KMAJOR) ? 1 : 0;
  const uint32_t a0 = sa + wg * (64 * 128);     // K-major: rows 64wg.. ; MN-major: the second 64-row TMA box
  const uint32_t sb = sa + A_STAGE_BYTES;
#pragma unroll
  for (int k = 0; k < BK / MMA_K; ++k) {
    const uint64_t da = TA ? make_smem_desc_sw128(a0 + k * (MMA_K * 128), 64 * 128, 1024)
                           : make_smem_desc_sw128(a0 + k * (MMA_K * 2), 16, 1024);
    const uint64_t db = TB ? make_smem_desc_sw128(sb + k * (MMA_K * 128), 64 * 128, 1024)
                           : make_smem_desc_sw128(sb + k * (MMA_K * 2), 16, 1024);
    wgmma_tile<BN, TA, TB>(acc, da, db);
  }
}

// Column sums over the 32 rows held by a warp (lane = row, v[j] = column j) with a butterfly of 31 shuffles:
// afterwards v[0] on lane l is the total of column l.
__device__ __forceinline__ void warp_colsum32(float (&v)[32], int lane) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const bool up = (lane & s) != 0;
#pragma unroll
    for (int j = 0; j < s; ++j) {
      const float send = up ? v[j] : v[j + s];
      const float keep = up ? v[j + s] : v[j];
      v[j] = keep + __shfl_xor_sync(0xffffffffu, send, s);
    }
  }
}

// Generic epilogue of one 32-row x 32-column chunk by one warp (q = 32-row quarter of the tile, lane = row, r[j] =
// fp32 bits of column c0 + j): alpha / bias / residual / ReLU -> global (bf16 / fp32 / transposed / atomic).
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const uint32_t (&r)[32], int mt, int m0, int n0,
                                               int c0, long long tap_off, int q, int lane, uint8_t* stage_buf,
                                               float bm, bool use_stage) {
  const int row = m0 + q * 32 + lane;
  if (n0 + c0 >= p.N) return;
  if (p.debug & 1) return;
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float x = __uint_as_float(r[j]) * p.alpha + bm;
    const int col = n0 + c0 + j;
    if (p.bias_n != nullptr && col < p.N) x += p.bias_n[col];
    v[j] = x;
  }
  const bool stats_from_stage = p.col_part != nullptr && use_stage && (n0 + c0 + 32 <= p.N);
  if (p.col_part != nullptr && !stats_from_stage) {
    // fused batch-norm statistics of the raw fp32 conv output (rows >= M are exact zeros: TMA OOB fill)
    // (of the value that is stored: bf16-rounded when the output is bf16, like the staged path below)
    float s1[32], s2[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float x = p.out_bf16 ? __bfloat162float(__float2bfloat16(v[j])) : v[j];
      s1[j] = x;
      s2[j] = x * x;
    }
    warp_colsum32(s1, lane);
    warp_colsum32(s2, lane);
    const int col = n0 + c0 + lane;
    if (col < p.N) {
      float* dst = p.col_part + ((size_t)(mt * 4 + q) * 2) * p.N + col;
      dst[0] = s1[0];
      dst[p.N] = s2[0];
    }
  }
  if (p.trans_out) {
    // out[col * ldo + row]: lanes are contiguous in memory -> coalesced per column
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int col = n0 + c0 + j;
      if (row < p.M && col < p.N) {
        const long long idx = (long long)col * p.ldo + row + tap_off;
        float x = v[j];
        if (p.residual != nullptr) x += __bfloat162float(p.residual[idx]);
        if (p.relu) x = fmaxf(x, 0.f);
        if (p.atomic_add)
          atomicAdd(reinterpret_cast<float*>(p.out) + idx, x);
        else if (p.out_bf16)
          reinterpret_cast<__nv_bfloat16*>(p.out)[idx] = __float2bfloat16(x);
        else
          reinterpret_cast<float*>(p.out)[idx] = x;
      }
    }
  } else if (row < p.M || use_stage) {
    const long long base = (long long)row * p.ldo + n0 + c0 + tap_off;
    const bool full = (n0 + c0 + 32 <= p.N);
    if (p.residual != nullptr && row < p.M) {
      if (full && ((base & 7) == 0)) {
        const uint4* rp = reinterpret_cast<const uint4*>(p.residual + base);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          uint4 u = rp[j4];
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            float2 f = __bfloat1622float2(h[t]);
            v[j4 * 8 + t * 2] += f.x;
            v[j4 * 8 + t * 2 + 1] += f.y;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (n0 + c0 + j < p.N) v[j] += __bfloat162float(p.residual[base + j]);
      }
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    if (p.atomic_add) {
      float* o = reinterpret_cast<float*>(p.out) + base;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (n0 + c0 + j < p.N) atomicAdd(o + j, v[j]);
    } else if (p.out_bf16) {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + base;
      if (full && ((base & 7) == 0)) {
        uint4 pk[4];
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&pk[j4]);
#pragma unroll
          for (int t = 0; t < 4; ++t) h[t] = __floats2bfloat162_rn(v[j4 * 8 + t * 2], v[j4 * 8 + t * 2 + 1]);
        }
        if (use_stage) {
          // transpose through this warp's private staging tile so that 4 lanes write one row's 64 B contiguously
          const uint32_t sbase = smem_u32(stage_buf);
          const uint32_t st = sbase + lane * 80;
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) sts_128(st + j4 * 16, pk[j4]);
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int rr = 8 * j + (lane >> 2);
            const uint4 u = lds_128(sbase + rr * 80 + (lane & 3) * 16);
            const int grow = m0 + q * 32 + rr;
            if (grow < p.M && !(p.debug & 2))
              *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (long long)grow * p.ldo + n0 +
                                        c0 + tap_off + (lane & 3) * 8) = u;
          }
          if (stats_from_stage) {
            // fused batch-norm statistics: lane = column, walk the 32 staged rows (the bf16 values that are stored;
            // rows >= M hold exact zeros). 32 conflict-free 2-byte smem loads instead of 62 shuffles.
            float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll
            for (int rr = 0; rr < 32; rr += 2) {
              const float x = lds_bf16(sbase + rr * 80 + lane * 2);
              const float y = lds_bf16(sbase + (rr + 1) * 80 + lane * 2);
              a1 += x;
              a2 = fmaf(x, x, a2);
              b1 += y;
              b2 = fmaf(y, y, b2);
            }
            float* dst = p.col_part + ((size_t)(mt * 4 + q) * 2) * p.N + n0 + c0 + lane;
            dst[0] = a1 + b1;
            dst[p.N] = a2 + b2;
          }
          __syncwarp();
        } else {
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) reinterpret_cast<uint4*>(o)[j4] = pk[j4];
        }
      } else if (row < p.M) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (n0 + c0 + j < p.N) o[j] = __float2bfloat16(v[j]);
      }
    } else {
      float* o = reinterpret_cast<float*>(p.out) + base;
      if (full && ((base & 3) == 0)) {
#pragma unroll
        for (int j4 = 0; j4 < 8; ++j4)
          reinterpret_cast<float4*>(o)[j4] = make_float4(v[j4 * 4], v[j4 * 4 + 1], v[j4 * 4 + 2], v[j4 * 4 + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (n0 + c0 + j < p.N) o[j] = v[j];
      }
    }
  }
}

// Lean epilogue (EPI_LEAN) of one 32 x 32 chunk: the three hot output kinds - bf16 store (+ fused BN statistics),
// fp32 store, fp32 atomic accumulate (split-K) - all row-major, no bias_m / transpose, N a multiple of 32. Every chunk
// goes through the warp's 32 x 64-byte staging tile so that one store instruction covers 8 full 64-byte row segments
// (a lane-per-row store would touch 32 different lines per instruction; the atomic path uses red.v4.f32).
// A separate, small code path: the generic epilogue above inlines several thousand instructions.
__device__ __forceinline__ void lean_chunk(const GemmParams& p, const uint32_t (&r)[32], int mt, int m0, int n0,
                                           int c0, long long tap_off, int q, int lane, uint32_t sbase) {
  if ((p.debug & 1) || n0 + c0 >= p.N) return;       // (tile wider than the matrix: nothing to store)
  const uint32_t st = sbase + lane * 80;
  const int sub_row = lane >> 2, sub_col = lane & 3;
  const float alpha = p.alpha;
  if (p.out_bf16) {
    uint4 pk[4];
    if (p.bias_n == nullptr && p.residual == nullptr && !p.relu) {
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&pk[j4]);
#pragma unroll
        for (int t = 0; t < 4; ++t)
          h[t] = __floats2bfloat162_rn(__uint_as_float(r[j4 * 8 + t * 2]) * alpha,
                                       __uint_as_float(r[j4 * 8 + t * 2 + 1]) * alpha);
      }
    } else {
      // inference epilogue of the BN-folded trunk: + bias[col] (+ residual[row, col]) -> ReLU
      const int grow_l = m0 + q * 32 + lane;
      const bool has_res = p.residual != nullptr && grow_l < p.M;
      const uint4* rp = reinterpret_cast<const uint4*>(p.residual + (long long)grow_l * p.ldo + n0 + c0 + tap_off);
      const float4* bp = reinterpret_cast<const float4*>(p.bias_n + n0 + c0);
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        float v[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) v[t] = __uint_as_float(r[j4 * 8 + t]) * alpha;
        if (p.bias_n != nullptr) {
          const float4 b0 = bp[j4 * 2], b1 = bp[j4 * 2 + 1];
          v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w;
          v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        }
        if (has_res) {
          const uint4 u = rp[j4];
          const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const float2 f = __bfloat1622float2(rh[t]);
            v[2 * t] += f.x;
            v[2 * t + 1] += f.y;
          }
        }
        if (p.relu) {
#pragma unroll
          for (int t = 0; t < 8; ++t) v[t] = fmaxf(v[t], 0.f);
        }
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&pk[j4]);
#pragma unroll
        for (int t = 0; t < 4; ++t) h[t] = __floats2bfloat162_rn(v[2 * t], v[2 * t + 1]);
      }
    }
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) sts_128(st + j4 * 16, pk[j4]);
    __syncwarp();
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + n0 + c0 + tap_off + sub_col * 8;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int rr = 8 * j + sub_row;
      const uint4 u = lds_128(sbase + rr * 80 + sub_col * 16);
      const int grow = m0 + q * 32 + rr;
      if (grow < p.M) *reinterpret_cast<uint4*>(o + (long long)grow * p.ldo) = u;
    }
    if (p.col_part != nullptr) {
      // fused batch-norm statistics of the stored (bf16) values: lane = column, 32 staged rows (rows >= M are 0)
      float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll
      for (int rr = 0; rr < 32; rr += 2) {
        const float x = lds_bf16(sbase + rr * 80 + lane * 2);
        const float y = lds_bf16(sbase + (rr + 1) * 80 + lane * 2);
        a1 += x;
        a2 = fmaf(x, x, a2);
        b1 += y;
        b2 = fmaf(y, y, b2);
      }
      float* dst = p.col_part + ((size_t)(mt * 4 + q) * 2) * p.N + n0 + c0 + lane;
      dst[0] = a1 + b1;
      dst[p.N] = a2 + b2;
    }
    __syncwarp();
  } else {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        uint4 u;
        u.x = __float_as_uint(__uint_as_float(r[half * 16 + j4 * 4 + 0]) * alpha);
        u.y = __float_as_uint(__uint_as_float(r[half * 16 + j4 * 4 + 1]) * alpha);
        u.z = __float_as_uint(__uint_as_float(r[half * 16 + j4 * 4 + 2]) * alpha);
        u.w = __float_as_uint(__uint_as_float(r[half * 16 + j4 * 4 + 3]) * alpha);
        sts_128(st + j4 * 16, u);
      }
      __syncwarp();
      float* o = reinterpret_cast<float*>(p.out) + n0 + c0 + half * 16 + tap_off + sub_col * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int rr = 8 * j + sub_row;
        const uint4 u = lds_128(sbase + rr * 80 + sub_col * 16);
        const int grow = m0 + q * 32 + rr;
        if (grow < p.M) {
          float* dst = o + (long long)grow * p.ldo;
          if (p.atomic_add)
            red_add_v4_f32(dst, u);
          else
            *reinterpret_cast<uint4*>(dst) = u;
        }
      }
      __syncwarp();
    }
  }
}

// Accumulator staging tile of one MMA warpgroup: 64 rows x 64 fp32 columns, 16-byte groups XOR-swizzled by row so
// that both the fragment stores (8-byte pairs) and the row-per-lane reads (16-byte groups) spread over the banks.
__device__ __forceinline__ uint32_t acc_off(int r, int c) {
  return (uint32_t)(r * 256 + ((((c >> 2) ^ (r & 15)) << 4) | ((c & 3) << 2)));
}

// Epilogue of the warpgroup's 64 x BN accumulator block: 64 columns at a time through the staging tile, then warp w of
// the warpgroup takes rows 32(w&1).. and columns 32(w>>1).. of the chunk (lane = row) into the chunk epilogue.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float (&acc)[BN / 2], int wg, int mt, int m0,
                                              int n0, long long tap_off, uint32_t acc_s, uint8_t* stage_buf) {
  const int t = threadIdx.x & 127, wl = t >> 5, lane = t & 31;
  const int fr = wl * 16 + (lane >> 2), fc = 2 * (lane & 3);   // fragment row / column of this thread
  const int q = wg * 2 + (wl & 1);
  const int row = m0 + q * 32 + lane;
  const float bm = (EPI == EPI_GENERIC && p.bias_m != nullptr && row < p.M) ? p.bias_m[row] : 0.f;
  // bf16 row-major output without residual: stores are staged through smem so that each store instruction writes
  // 8 full 64-byte row segments
  const bool use_stage = p.out_bf16 && !p.trans_out && !p.atomic_add && p.residual == nullptr &&
                         ((p.ldo & 7) == 0) && (((n0 + tap_off) & 7) == 0) &&
                         ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0);
#pragma unroll
  for (int ch = 0; ch < BN / 64; ++ch) {
    if (n0 + ch * 64 >= p.N) break;                            // (uniform over the CTA)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int a = (ch * 8 + j) * 4;
      const int c = j * 8 + fc;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_s + acc_off(fr, c)), "f"(acc[a]), "f"(acc[a + 1])
                   : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_s + acc_off(fr + 8, c)), "f"(acc[a + 2]),
                   "f"(acc[a + 3])
                   : "memory");
    }
    named_bar_sync(1 + wg, 128);
    const int rr = (wl & 1) * 32 + lane, cc = (wl >> 1) * 32;
    uint32_t r[32];
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const uint4 u = lds_128(acc_s + acc_off(rr, cc + 4 * g));
      r[4 * g] = u.x; r[4 * g + 1] = u.y; r[4 * g + 2] = u.z; r[4 * g + 3] = u.w;
    }
    if constexpr (EPI == EPI_LEAN)
      lean_chunk(p, r, mt, m0, n0, ch * 64 + cc, tap_off, q, lane, smem_u32(stage_buf));
    else
      epilogue_chunk(p, r, mt, m0, n0, ch * 64 + cc, tap_off, q, lane, stage_buf, bm, use_stage);
    named_bar_sync(1 + wg, 128);                               // staging tile free for the next chunk
  }
}

// ------------------------------------------------------------------------------------------------- the kernel
// grid = min(#work units, SMs) (persistent) or #units (one unit per CTA); units u = cluster index, + #clusters, ...
// with n fastest, so that concurrently running CTAs share the A rows in L2. CL = 1: a unit is one 128 x BN tile.
// CL = 2 (CTA pair): the grid is made of 2-CTA clusters, a unit is the tile pair (2 u_m, n), (2 u_m + 1, n) and the B
// tile both need is multicast (see load_kblock); a stage is free again once the MMA warpgroups of BOTH CTAs released
// it, so each consumer warpgroup arrives on the `empty` barrier of both CTAs.
template <int BN, int A_MODE, int B_MODE, int EPI, int CL>
__global__ void __launch_bounds__(GemmLayout<BN>::THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const GemmParams p) {
  using L = GemmLayout<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + L::STAGES;

  const int warp_id = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rank = (CL == 2) ? (int)cluster_ctarank() : 0;
  const int per_z = ((p.tiles_m + CL - 1) / CL) * p.tiles_n;
  const int unit0 = blockIdx.x / CL, units_step = gridDim.x / CL;

  if (warp_id == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < L::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CL);                     // one arrival per MMA warpgroup of every CTA
    }
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (CL == 2) cluster_sync_all();                 // the peer's barriers exist before any remote access

  if (warp_id < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp_id == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = unit0; t < p.tiles_total; t += units_step) {
        const int z = t / per_z;
        const int r = t - z * per_z;
        const int mt = (r / p.tiles_n) * CL + rank;         // (CL = 2, odd tiles_m: the last pair's rank 1 computes
        const int nt = r % p.tiles_n;                       //  on TMA zero fill and stores nothing)
        const int zsplit = (B_MODE == OP_CONV) ? (z % p.cSplits) : z;
        const int ztap = (B_MODE == OP_CONV) ? (z / p.cSplits) : 0;
        const int kb_begin = zsplit * p.kb_per_split;
        const int kb_end = min(kb_begin + p.kb_per_split, p.kb_total);
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          if (p.debug & 4) {
            mbar_arrive(&full_bar[stage]);
          } else {
            mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
            load_kblock<BN, A_MODE, B_MODE, CL>(p, &tmA, &tmB, sa, sa + A_STAGE_BYTES, &full_bar[stage], kb, mt,
                                                mt * BM, nt * BN, ztap, rank);
          }
          if (++stage == L::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue (two warpgroups, 64 rows each) =====================
    setmaxnreg_inc<232>();
    const int wg = (warp_id >> 2) - 1;
    const uint32_t acc_s = smem_u32(smem + L::ACC_OFFSET + wg * (64 * 64 * 4));
    uint8_t* stage_buf = smem + L::STORE_OFFSET + (warp_id - 4) * (32 * 80);
    const bool signaller = (threadIdx.x & 127) == 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    auto release = [&](int s) {
      if constexpr (CL == 2) {
        mbar_arrive_cluster(&empty_bar[s], 0);
        mbar_arrive_cluster(&empty_bar[s], 1);
      } else {
        mbar_arrive(&empty_bar[s]);
      }
    };
    for (int t = unit0; t < p.tiles_total; t += units_step) {
      const int z = t / per_z;
      const int r = t - z * per_z;
      const int mt = (r / p.tiles_n) * CL + rank;
      const int nt = r % p.tiles_n;
      const int zsplit = (B_MODE == OP_CONV) ? (z % p.cSplits) : z;
      const int ztap = (B_MODE == OP_CONV) ? (z / p.cSplits) : 0;
      const int kb_begin = zsplit * p.kb_per_split;
      const int num_kb = min(kb_begin + p.kb_per_split, p.kb_total) - kb_begin;
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int i = 0; i < num_kb; ++i) {
        mbar_wait(&full_bar[stage], phase);
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) reg_fence(acc[j]);
        wgmma_fence();
        mma_kblock<BN, A_MODE, B_MODE>(acc, smem_u32(smem + stage * L::STAGE_BYTES), wg);
        wgmma_commit();
        wgmma_wait<1>();                                       // the previous K-block's MMAs are done
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) reg_fence(acc[j]);
        if (prev >= 0 && signaller) release(prev);
        prev = stage;
        if (++stage == L::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) reg_fence(acc[j]);
      if (prev >= 0 && signaller) release(prev);
      const long long tap_off =
          ((B_MODE == OP_CONV) ? (long long)ztap * p.tap_stride : 0) + (long long)zsplit * p.split_stride;
      if (mt < p.tiles_m) epilogue_tile<BN, EPI>(p, acc, wg, mt, mt * BM, nt * BN, tap_off, acc_s, stage_buf);
    }
  }
  if constexpr (CL == 2) {
    __syncwarp();
    cluster_sync_all();              // no CTA leaves while its peer may still multicast into it or arrive on its barriers
  }
}

// Deterministic split-K: out[r, c] += sum over s (in order) of part[s][r, c], r < rows, c < cols (row stride ld).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(float* out, const float* part, long long rows, long long cols,
                                                           long long ld, long long split_stride, int splits) {
  const long long n = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    const long long off = r * ld + c;
    float acc = part[off];
    for (int s = 1; s < splits; ++s) acc += part[s * split_stride + off];
    out[off] += acc;
  }
}

// =============================================================================== host side
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static std::mutex g_mu;
static char g_err[512] = {0};

static int set_err(const char* what, int code) {
  snprintf(g_err, sizeof(g_err), "%s (code %d)", what, code);
  return code ? code : -1;
}

static bool load_encode() {
  if (g_encode) return true;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr) return false;
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  return true;
}

struct MapKey {
  const void* ptr;
  uint64_t d0, d1, d2, d3, s1, s2, s3;
  uint32_t b0, b1, b2, b3, rank, estride, pad_;
  bool operator==(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(MapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// rank-2 or rank-4 bf16 tensor map with 128B swizzle, zero OOB fill.
static int get_map(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, uint32_t spatial_stride = 1) {
  MapKey k;
  memset(&k, 0, sizeof(k));
  k.ptr = ptr;
  k.rank = rank;
  k.estride = spatial_stride;
  k.d0 = dims[0];
  k.d1 = dims[1];
  k.b0 = box[0];
  k.b1 = box[1];
  k.s1 = strides_bytes[0];
  if (rank == 4) {
    k.d2 = dims[2];
    k.d3 = dims[3];
    k.b2 = box[2];
    k.b3 = box[3];
    k.s2 = strides_bytes[1];
    k.s3 = strides_bytes[2];
  }
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_maps.find(k);
  if (it != g_maps.end()) {
    *out = it->second;
    return 0;
  }
  if (!load_encode()) return set_err("cuTensorMapEncodeTiled entry point unavailable", -2);
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t bx[4];
  cuuint32_t es[4] = {1, 1, 1, 1};
  if (rank == 4 && spatial_stride > 1) es[1] = es[2] = spatial_stride;   // strided convolution: every s-th pixel
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
  }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_bytes[i];
  CUtensorMap m;
  CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_err("cuTensorMapEncodeTiled failed", (int)r);
  if (g_maps.size() > 4096) g_maps.clear();
  g_maps.emplace(k, m);
  *out = m;
  return 0;
}

static int g_persist = -1;   // FLPR_GEMM_PERSIST (default 1): persistent grid, operand loads overlap the epilogue
static int g_sms = 0;

static bool use_persist() {
  if (g_persist < 0) {
    const char* e = getenv("FLPR_GEMM_PERSIST");
    g_persist = (e == nullptr || e[0] != '0') ? 1 : 0;
  }
  return g_persist == 1;
}

static int sm_count() {
  if (g_sms == 0) {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    g_sms = n;
  }
  return g_sms;
}

// FLPR_GEMM_2CTA=1: CTA-pair (2-CTA cluster, multicast B) kernel where eligible. Off by default: on an H100 it measured
// 2-12 % slower than the single-CTA kernel on the head-step GEMM / convolution shapes (scripts/gemm_pair_bench.py) -
// B-operand L2 traffic is not what bounds these tiles, and the pair runs at the pace of its slower CTA.
static int g_pair = -1;

static bool use_pair() {
  if (g_pair < 0) {
    const char* e = getenv("FLPR_GEMM_2CTA");
    g_pair = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return g_pair == 1;
}

// CTA pairs need two M tiles to share a B tile.
static bool pair_ok(int M) { return use_pair() && (M + BM - 1) / BM >= 2; }

// FLPR_GEMM_GENERIC_EPI / FLPR_GEMM_DEBUG are read ONCE (no getenv on the launch path: launches come from several
// client threads, and getenv is not safe against a concurrent setenv elsewhere in the process).
static int g_generic_epi = -1;
static int g_debug = -1;

static bool force_generic_epi() {
  if (g_generic_epi < 0) g_generic_epi = getenv("FLPR_GEMM_GENERIC_EPI") != nullptr ? 1 : 0;
  return g_generic_epi == 1;
}

static int debug_flags() {
  if (g_debug < 0) {
    const char* e = getenv("FLPR_GEMM_DEBUG");
    g_debug = e ? atoi(e) : 0;
  }
  return g_debug;
}

// lean epilogue: plain row-major bf16 / fp32 / fp32-atomic output, every 32-column chunk full and 16-byte aligned
static bool lean_ok(const GemmParams& p) {
  const long long esz = p.out_bf16 ? 2 : 4;
  const bool act = p.residual != nullptr || p.bias_n != nullptr || p.relu;
  return !p.trans_out && p.bias_m == nullptr && (!act || (p.out_bf16 && !p.atomic_add)) &&
         (reinterpret_cast<uintptr_t>(p.bias_n) % 16) == 0 && (reinterpret_cast<uintptr_t>(p.residual) % 16) == 0 &&
         (p.N % 32) == 0 && ((p.ldo * esz) % 16) == 0 && ((p.tap_stride * esz) % 16) == 0 &&
         (reinterpret_cast<uintptr_t>(p.out) % 16) == 0 && !(p.atomic_add && p.out_bf16) &&
         !(p.col_part != nullptr && !p.out_bf16) && !force_generic_epi();
}

template <int BN, int A_MODE, int B_MODE, int EPI, int CL>
static int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int grid, cudaStream_t st) {
  using L = GemmLayout<BN>;
  auto kern = gemm_bf16_wgmma_kernel<BN, A_MODE, B_MODE, EPI, CL>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return set_err("cudaFuncSetAttribute(smem)", (int)e);
    configured = true;
  }
  if constexpr (CL == 1) {
    kern<<<grid, L::THREADS, L::TOTAL, st>>>(ta, tb, p);
  } else {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(L::THREADS);
    cfg.dynamicSmemBytes = L::TOTAL;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, p);
    if (e != cudaSuccess) return set_err(cudaGetErrorString(e), (int)e);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_err(cudaGetErrorString(e), (int)e);
  return 0;
}

template <int BN, int A_MODE, int B_MODE>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p_in, int splits, cudaStream_t st,
                  bool pair) {
  GemmParams p = p_in;
  p.debug = debug_flags();
  p.tiles_m = (p.M + BM - 1) / BM;
  p.tiles_n = (p.N + BN - 1) / BN;
  p.tiles_z = splits;
  const int cl = pair ? 2 : 1;
  p.tiles_total = ((p.tiles_m + cl - 1) / cl) * p.tiles_n * splits;     // work units (tiles or tile pairs)
  // persistent: one CTA per SM walks the units; otherwise one CTA (cluster) per unit
  const int slots = sm_count() / cl;
  const int grid = cl * ((use_persist() && p.tiles_total > slots) ? slots : p.tiles_total);
  const bool lean = lean_ok(p);
  if (pair)
    return lean ? launch_kernel<BN, A_MODE, B_MODE, EPI_LEAN, 2>(ta, tb, p, grid, st)
                : launch_kernel<BN, A_MODE, B_MODE, EPI_GENERIC, 2>(ta, tb, p, grid, st);
  return lean ? launch_kernel<BN, A_MODE, B_MODE, EPI_LEAN, 1>(ta, tb, p, grid, st)
              : launch_kernel<BN, A_MODE, B_MODE, EPI_GENERIC, 1>(ta, tb, p, grid, st);
}

template <int BN>
static int dispatch_modes(int a_mode, int b_mode, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          int splits, cudaStream_t st, bool pair) {
  if (a_mode == OP_KMAJOR && b_mode == OP_KMAJOR) return launch<BN, OP_KMAJOR, OP_KMAJOR>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_KMAJOR && b_mode == OP_MNMAJOR) return launch<BN, OP_KMAJOR, OP_MNMAJOR>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_MNMAJOR && b_mode == OP_KMAJOR) return launch<BN, OP_MNMAJOR, OP_KMAJOR>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_MNMAJOR && b_mode == OP_MNMAJOR) return launch<BN, OP_MNMAJOR, OP_MNMAJOR>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_CONV && b_mode == OP_KMAJOR) return launch<BN, OP_CONV, OP_KMAJOR>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_CONV && b_mode == OP_TAPFLIP) return launch<BN, OP_CONV, OP_TAPFLIP>(ta, tb, p, splits, st, pair);
  if (a_mode == OP_MNMAJOR && b_mode == OP_CONV) return launch<BN, OP_MNMAJOR, OP_CONV>(ta, tb, p, splits, st, pair);
  return set_err("unsupported operand mode combination", -3);
}

static int dispatch_bn(int BN, int a_mode, int b_mode, const CUtensorMap& ta, const CUtensorMap& tb,
                       const GemmParams& p, int splits, cudaStream_t st, bool pair) {
  if (BN == 64) return dispatch_modes<64>(a_mode, b_mode, ta, tb, p, splits, st, pair);
  if (BN == 128) return dispatch_modes<128>(a_mode, b_mode, ta, tb, p, splits, st, pair);
  return dispatch_modes<256>(a_mode, b_mode, ta, tb, p, splits, st, pair);
}

// Split-K without atomics: the kernel stores the partial product of split s to ws + s * split_stride (plain stores),
// then splitk_reduce_kernel adds the partials to `out` in split order - the result does not depend on which CTA
// finished first, so a run is bitwise reproducible. out: `rows` x `cols` valid elements, row stride p.ldo; ws holds
// splits x ceil4(rows * ldo) floats.
// zcount: grid z extent (splits, or taps x splits for the convolution weight gradient).
static int dispatch_split(int BN, int a_mode, int b_mode, const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p,
                          int zcount, int splits, float* ws, long long rows, long long cols, cudaStream_t st,
                          bool pair) {
  if (splits <= 1) return dispatch_bn(BN, a_mode, b_mode, ta, tb, p, zcount, st, pair);
  if (ws == nullptr) return set_err("split-K needs a workspace of splits x ceil4(rows * ldo) floats", -14);
  float* out = reinterpret_cast<float*>(p.out);
  p.out = ws;
  p.atomic_add = 0;
  p.split_stride = (rows * p.ldo + 3) & ~3LL;
  int rc = dispatch_bn(BN, a_mode, b_mode, ta, tb, p, zcount, st, pair);
  if (rc) return rc;
  const long long n = rows * cols;
  long long grid = (n + 255) / 256;
  if (grid > (long long)sm_count() * 8) grid = (long long)sm_count() * 8;
  splitk_reduce_kernel<<<(int)grid, 256, 0, st>>>(out, ws, rows, cols, p.ldo, p.split_stride, splits);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_err(cudaGetErrorString(e), (int)e);
  return 0;
}

// Tile width. 128 x 256 tiles halve the A-operand smem traffic per MMA relative to 128 x 128 tiles but take the
// whole ring of shallower stages, so they are used when they still give ~a full wave of the 132 SMs.
static int pick_bn(int M, int N, int z, int requested) {
  if (requested == 64 || requested == 128 || requested == 256) return requested;
  if (N <= 64) return 64;
  if (!use_persist()) return 128;
  const long long mt = (M + BM - 1) / BM;
  const long long t256 = mt * ((N + 255) / 256) * (z > 0 ? z : 1);
  if (N >= 256 && t256 >= 120) return 256;
  return 128;
}

}  // namespace flpr

using namespace flpr;

extern "C" {

const char* flpr_gemm_last_error() { return g_err; }

// 1: persistent grid (default), 0: one CTA per tile, -1: re-read FLPR_GEMM_PERSIST.
void flpr_gemm_set_persistent(int on) { g_persist = on; }

// 1: use the CTA-pair (2-CTA cluster, multicast B operand) kernel where eligible, 0: never, -1: re-read FLPR_GEMM_2CTA.
void flpr_gemm_set_pair(int on) { g_pair = on; }

// bottleneck-isolation switches of scripts/gemm_*: debug bit mask (see GemmParams::debug) and forced generic epilogue;
// -1 re-reads the FLPR_GEMM_DEBUG / FLPR_GEMM_GENERIC_EPI environment variables at the next launch.
void flpr_gemm_set_debug(int flags) { g_debug = flags; }
void flpr_gemm_set_generic_epilogue(int on) { g_generic_epi = on; }

// D = alpha * op(A) * op(B)^T.  a_mode/b_mode: 0 = [rows,K] (ld = row stride), 1 = [K,rows] (ld = K-row stride).
// split_k > 1: fp32 `out` is accumulated into (out += D), deterministically, through `split_ws` (see dispatch_split).
// col_part (optional, fp32 [ceil(M/128)*4][2][N]): per-32-row partial column sums / sums of squares of the fp32
// result (fused batch-norm statistics); requires split_k <= 1 and no transposed output.
int flpr_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, long long lda, long long ldb,
                   long long ldo, int a_mode, int b_mode, int out_bf16, int trans_out, float alpha,
                   const float* bias_n, const float* bias_m, int relu, const void* residual, int split_k, int bn_req,
                   float* col_part, float* split_ws, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  bind_device_of(A);
  if ((lda % 8) || (ldb % 8)) return set_err("lda/ldb must be multiples of 8 elements (16B TMA stride)", -4);
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return set_err("A/B must be 16B aligned", -5);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.kb_total = (K + BK - 1) / BK;
  int splits = split_k > 1 ? split_k : 1;
  if (splits > p.kb_total) splits = p.kb_total;
  p.kb_per_split = (p.kb_total + splits - 1) / splits;
  splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  const int BN = pick_bn(M, N, splits, bn_req);
  const bool pair = pair_ok(M);
  p.out = out; p.ldo = ldo; p.out_bf16 = out_bf16; p.trans_out = trans_out;
  if (splits > 1 && out_bf16) return set_err("split-K requires fp32 output", -6);
  if (col_part != nullptr && (splits > 1 || trans_out)) return set_err("col_part needs split_k=1, no transpose", -12);
  p.col_part = col_part;
  p.alpha = alpha; p.bias_n = bias_n; p.bias_m = bias_m; p.relu = relu;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(residual);
  CUtensorMap ta, tb;
  int rc;
  {
    uint64_t dims[2], str[1];
    uint32_t box[2];
    if (a_mode == OP_KMAJOR) {
      dims[0] = (uint64_t)K; dims[1] = (uint64_t)M; box[0] = BK; box[1] = BM;
    } else {
      dims[0] = (uint64_t)M; dims[1] = (uint64_t)K; box[0] = 64; box[1] = BK;
    }
    str[0] = (uint64_t)lda * 2;
    if ((rc = get_map(&ta, A, 2, dims, str, box))) return rc;
    if (b_mode == OP_KMAJOR) {
      dims[0] = (uint64_t)K; dims[1] = (uint64_t)N; box[0] = BK; box[1] = (uint32_t)(pair ? BN / 2 : BN);
    } else {
      dims[0] = (uint64_t)N; dims[1] = (uint64_t)K; box[0] = 64; box[1] = BK;
    }
    str[0] = (uint64_t)ldb * 2;
    if ((rc = get_map(&tb, B, 2, dims, str, box))) return rc;
  }
  return dispatch_split(BN, a_mode, b_mode, ta, tb, p, splits, splits, split_ws, trans_out ? N : M, trans_out ? M : N,
                        stream, pair);
}

static int conv_tiling(int H, int W, int* TH, int* NB, int* tiles_per_img) {
  if (W > 128 || (128 % W)) return set_err("conv: W must divide 128", -8);
  if (H * W <= 128) {
    if (128 % (H * W)) return set_err("conv: H*W must divide 128", -9);
    *TH = H; *NB = 128 / (H * W); *tiles_per_img = 1;
  } else {
    *TH = 128 / W;
    if (H % *TH) return set_err("conv: 128/W must divide H", -10);
    *NB = 1; *tiles_per_img = H / *TH;
  }
  return 0;
}

// Implicit-GEMM convolution (stride 1 or 2): X [NIMG,H,W,C] bf16 NHWC, Wt [Cout, KH*KW*C] bf16 (tap-major, then C),
// out [NIMG*Ho*Wo, Cout]. Requires C % 64 == 0, Wo a power of two <= 128 and (Ho*Wo) | 128 or 128/Wo | Ho.
// A strided convolution is the same pipeline: the TMA tensor map walks the input with element strides {1,s,s,1}.
// col_part: see flpr_gemm_bf16 (fused batch-norm statistics of the conv output).
int flpr_conv_nhwc_bf16(const void* X, const void* Wt, void* out, int NIMG, int H, int W, int C, int Cout, int KH,
                        int KW, int pad_h, int pad_w, int out_bf16, float alpha, const float* bias_n, int relu,
                        const void* residual, int bn_req, float* col_part, int stride, long long x_stride_w,
                        long long x_stride_h, long long x_stride_n, cudaStream_t stream) {
  // x_stride_{w,h,n}: element strides of X (0 = dense NHWC). A W stride smaller than C makes the per-pixel "channel"
  // vectors overlap: that is how the 7x7 stem convolution runs on 4-cell windows of a space-to-depth input.
  bind_device_of(X);
  if (C % 64) return set_err("conv: C must be a multiple of 64", -7);
  if (stride != 1 && stride != 2) return set_err("conv: stride must be 1 or 2", -13);
  const int Ho = (H + 2 * pad_h - KH) / stride + 1;
  const int Wo = (W + 2 * pad_w - KW) / stride + 1;
  int TH, NB, tiles_per_img, rc;
  if ((rc = conv_tiling(Ho, Wo, &TH, &NB, &tiles_per_img))) return rc;
  const int M = NIMG * Ho * Wo;
  const int K = KH * KW * C;
  const int BN = pick_bn(M, Cout, 1, bn_req);
  const bool pair = pair_ok(M);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = Cout; p.K = K;
  p.kb_total = K / BK; p.kb_per_split = p.kb_total;
  p.out = out; p.ldo = Cout; p.out_bf16 = out_bf16; p.alpha = alpha; p.bias_n = bias_n; p.relu = relu;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(residual);
  p.col_part = col_part;
  p.cH = Ho; p.cW = Wo; p.cC = C; p.cTH = TH; p.cNB = NB; p.cKW = KW; p.cPadH = pad_h; p.cPadW = pad_w;
  p.cTilesPerImg = tiles_per_img; p.cTaps = KH * KW; p.cStride = stride;
  CUtensorMap ta, tb;
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NIMG};
    uint64_t str[3] = {(uint64_t)(x_stride_w ? x_stride_w : C) * 2,
                       (uint64_t)(x_stride_h ? x_stride_h : (long long)W * C) * 2,
                       (uint64_t)(x_stride_n ? x_stride_n : (long long)H * W * C) * 2};
    uint32_t box[4] = {64, (uint32_t)(Wo * stride), (uint32_t)(TH * stride), (uint32_t)NB};
    if ((rc = get_map(&ta, X, 4, dims, str, box, (uint32_t)stride))) return rc;
    uint64_t d2[2] = {(uint64_t)K, (uint64_t)Cout};
    uint64_t s2[1] = {(uint64_t)K * 2};
    uint32_t b2[2] = {BK, (uint32_t)(pair ? BN / 2 : BN)};
    if ((rc = get_map(&tb, Wt, 2, d2, s2, b2))) return rc;
  }
  return dispatch_bn(BN, OP_CONV, OP_KMAJOR, ta, tb, p, 1, stream, pair);
}

// Data gradient of a stride-1 convolution, straight from the FORWARD weight Wt [Cout, KH*KW*Cin] (no flipped /
// transposed copy): dX[NIMG*H*W, Cin] = sum_taps dY(shifted by the mirrored tap)[., Cout] x Wt[:, tap, :].
// dY: [NIMG,H,W,Cout] bf16. pad_h/pad_w are the FORWARD paddings (dgrad pads with K-1-pad).
int flpr_conv_dgrad_nhwc_bf16(const void* dY, const void* Wt, void* out, int NIMG, int H, int W, int Cin, int Cout,
                              int KH, int KW, int pad_h, int pad_w, int out_bf16, int bn_req, cudaStream_t stream) {
  bind_device_of(dY);
  if (Cout % 64) return set_err("conv dgrad: Cout must be a multiple of 64", -7);
  if (Cin % 64) return set_err("conv dgrad: Cin must be a multiple of 64", -7);
  int TH, NB, tiles_per_img, rc;
  if ((rc = conv_tiling(H, W, &TH, &NB, &tiles_per_img))) return rc;
  const int M = NIMG * H * W;
  const int K = KH * KW * Cout;
  const int BN = pick_bn(M, Cin, 1, bn_req);
  CUtensorMap ta, tb;
  {
    uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NIMG};
    uint64_t str[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
    uint32_t box[4] = {64, (uint32_t)W, (uint32_t)TH, (uint32_t)NB};
    if ((rc = get_map(&ta, dY, 4, dims, str, box))) return rc;
    uint64_t d2[2] = {(uint64_t)KH * KW * Cin, (uint64_t)Cout};
    uint64_t s2[1] = {(uint64_t)KH * KW * Cin * 2};
    uint32_t b2[2] = {64, BK};
    if ((rc = get_map(&tb, Wt, 2, d2, s2, b2))) return rc;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = Cin; p.K = K;
  p.kb_total = K / BK; p.kb_per_split = p.kb_total;
  p.out = out; p.ldo = Cin; p.out_bf16 = out_bf16; p.alpha = 1.f;
  p.cH = H; p.cW = W; p.cC = Cout; p.cTH = TH; p.cNB = NB; p.cKW = KW;
  p.cPadH = KH - 1 - pad_h; p.cPadW = KW - 1 - pad_w;
  p.cTilesPerImg = tiles_per_img; p.cTaps = KH * KW; p.cStride = 1;
  return dispatch_bn(BN, OP_CONV, OP_TAPFLIP, ta, tb, p, 1, stream, pair_ok(M));
}

// Weight gradient of a stride-1 convolution: out[Cout, KH*KW*C] (fp32, tap-major then C) +=
//   sum over pixels dY[p, cout] * Xshift_tap[p, c].  One launch covers every tap (grid.z = taps * split_k).
// dY: [NIMG*H*W, Cout] bf16, X: [NIMG,H,W,C] bf16. split_k > 1: `out` is accumulated into (out += dW) through
// `split_ws` (splits x ceil4(Cout * KH*KW*C) floats), deterministically (see dispatch_split).
int flpr_conv_wgrad_nhwc_bf16(const void* X, const void* dY, float* out, int NIMG, int H, int W, int C, int Cout,
                              int KH, int KW, int pad_h, int pad_w, int split_k, int bn_req, float* split_ws,
                              cudaStream_t stream) {
  bind_device_of(X);
  if (C % 64) return set_err("conv wgrad: C must be a multiple of 64", -7);
  if (Cout % 8) return set_err("conv wgrad: Cout must be a multiple of 8", -11);
  if (W > 64 || (64 % W)) return set_err("conv wgrad: W must divide 64", -8);
  int TH, NB;
  if (H * W >= 64) {
    if ((H * W) % 64) return set_err("conv wgrad: H*W must be a multiple of 64", -9);
    TH = 64 / W; NB = 1;
  } else {
    if (64 % (H * W)) return set_err("conv wgrad: H*W must divide 64", -9);
    TH = H; NB = 64 / (H * W);
  }
  const int M = Cout, N = C, K = NIMG * H * W;
  const int BN = (bn_req == 64 || bn_req == 128 || bn_req == 256) ? bn_req : (N >= 128 ? 128 : 64);
  CUtensorMap ta, tb;
  int rc;
  {
    uint64_t d2[2] = {(uint64_t)M, (uint64_t)K};
    uint64_t s2[1] = {(uint64_t)Cout * 2};
    uint32_t b2[2] = {64, BK};
    if ((rc = get_map(&ta, dY, 2, d2, s2, b2))) return rc;
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NIMG};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, (uint32_t)W, (uint32_t)TH, (uint32_t)NB};
    if ((rc = get_map(&tb, X, 4, dims, str, box))) return rc;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.kb_total = (K + BK - 1) / BK;
  int splits = split_k > 1 ? split_k : 1;
  if (splits > p.kb_total) splits = p.kb_total;
  p.kb_per_split = (p.kb_total + splits - 1) / splits;
  splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  p.out = out; p.ldo = (long long)KH * KW * C; p.out_bf16 = 0; p.alpha = 1.f;
  p.cH = H; p.cW = W; p.cC = C; p.cTH = TH; p.cNB = NB; p.cKW = KW; p.cPadH = pad_h; p.cPadW = pad_w;
  p.cSplits = splits; p.tap_stride = C; p.cTaps = KH * KW;
  const int gz = KH * KW * splits;
  return dispatch_split(BN, OP_MNMAJOR, OP_CONV, ta, tb, p, gz, splits, split_ws, M, p.ldo, stream, pair_ok(M));
}

}  // extern "C"
