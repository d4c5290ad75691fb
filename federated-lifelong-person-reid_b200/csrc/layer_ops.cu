// flpr layer-level fused element-wise kernels (memory-bound passes that used to be chains of ATen ops):
//
//   wcompose_fwd / wcompose_bwd   decomposed-weight composition of FedWeIT (methods/fedweit.py:122-136 of the reference)
//                                 and fedstil-atten (methods/fedstil_atten.py:88-96):
//                                     theta[e] = prune(aw[e]) + sum_k atten[k] * stack[e, k] + prune(mask[row(e)]) * sw[e]
//                                 one pass writes theta in fp32 (autograd master) and bf16 (tensor-core operand); the
//                                 backward pass produces d aw (pruned pass-through), d mask (one value per output unit)
//                                 and d atten (deterministic two-stage reduction) from d theta in one sweep.
//   ln_rows                       LayerNorm over the channel dim of bf16 token rows, one warp per token, fp32 statistics;
//                                 optionally the destination is the (cyclically shifted) window layout of a Swin block
//                                 (models/swin_transformer.py:358-380: norm1 -> roll -> window_partition in one pass).
//   ln_rows_train / ln_rows_bwd   the same LayerNorm for the TRAINABLE stage: the forward keeps (mean, rstd) per row, the
//                                 backward is one sweep (dx in the source layout, per-block dgamma / dbeta partials
//                                 folded in a fixed order by ln_colsum: deterministic, no atomics).
//   window_merge_add              window_reverse -> roll back -> + shortcut (models/swin_transformer.py:383-391) in one pass.
//   gelu_rows                     exact (erf) GELU over bf16 rows (models/swin_transformer.py:118-140, frozen stages).
//   apply_global                  receiving end of the FedAvg-family dispatch (methods/fedavg.py:413-430,
//                                 fedprox.py:351-364): master <- global, bf16 copy, FedProx anchor snapshot, one pass.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ptx.cuh"

namespace flpr {

constexpr int WC_MAXK = 16;

__device__ __forceinline__ float prune_val(float v, float thr, int prune) {
  return (prune && !(fabsf(v) > thr)) ? 0.f : v;
}

// ------------------------------------------------------------------------------------------------- compose forward
__global__ void __launch_bounds__(256) wcompose_fwd_kernel(const float* __restrict__ aw, const float* __restrict__ stack,
                                                           const float* __restrict__ atten, int kb, int ks,
                                                           const float* __restrict__ sw, const float* __restrict__ mask,
                                                           long long row_len, float thr_aw, float thr_mask, int prune,
                                                           float* __restrict__ out_f32,
                                                           __nv_bfloat16* __restrict__ out_bf16, long long n) {
  __shared__ float s_att[WC_MAXK];
  if (threadIdx.x < kb) s_att[threadIdx.x] = atten[threadIdx.x];
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    float acc = prune_val(aw[e], thr_aw, prune);
    if (kb > 0) {
      const float* sp = stack + e * ks;
      float kacc = 0.f;
      for (int k = 0; k < kb; ++k) kacc = fmaf(s_att[k], sp[k], kacc);
      acc += kacc;
    }
    if (sw != nullptr) acc = fmaf(prune_val(mask[e / row_len], thr_mask, prune), sw[e], acc);
    if (out_f32 != nullptr) out_f32[e] = acc;
    if (out_bf16 != nullptr) out_bf16[e] = __float2bfloat16(acc);
  }
}

// ------------------------------------------------------------------------------------------------- compose backward
// One block per row r (FedWeIT: one output unit; fedstil-atten: an arbitrary chunk): d_aw element-wise, the row's
// partial sums of d theta * stack[., k] into part_att[r, k] and of d theta * sw into d_mask[r].
__global__ void __launch_bounds__(256) wcompose_bwd_kernel(const float* __restrict__ dth, const float* __restrict__ aw,
                                                           const float* __restrict__ stack, int kb, int ks,
                                                           const float* __restrict__ sw, const float* __restrict__ mask,
                                                           long long row_len, float thr_aw, float thr_mask, int prune,
                                                           float* __restrict__ d_aw, float* __restrict__ part_att,
                                                           float* __restrict__ d_mask, long long n) {
  __shared__ float sh[8][WC_MAXK + 1];
  const long long r = blockIdx.x;
  const long long beg = r * row_len;
  long long end = beg + row_len;
  if (end > n) end = n;
  float acc[WC_MAXK];
#pragma unroll
  for (int k = 0; k < WC_MAXK; ++k) acc[k] = 0.f;
  float am = 0.f;
  for (long long e = beg + threadIdx.x; e < end; e += blockDim.x) {
    const float g = dth[e];
    if (d_aw != nullptr) d_aw[e] = (prune && !(fabsf(aw[e]) > thr_aw)) ? 0.f : g;
    if (kb > 0) {
      const float* sp = stack + e * ks;
#pragma unroll
      for (int k = 0; k < WC_MAXK; ++k)
        if (k < kb) acc[k] = fmaf(g, sp[k], acc[k]);
    }
    if (sw != nullptr) am = fmaf(g, sw[e], am);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < WC_MAXK; ++k) {
    const float v = warp_sum(acc[k]);
    if (l == 0) sh[w][k] = v;
  }
  {
    const float v = warp_sum(am);
    if (l == 0) sh[w][WC_MAXK] = v;
  }
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  if (threadIdx.x <= WC_MAXK) {
    float t = 0.f;
    for (int i = 0; i < nw; ++i) t += sh[i][threadIdx.x];
    if (threadIdx.x < kb && part_att != nullptr) part_att[r * kb + threadIdx.x] = t;
    if (threadIdx.x == WC_MAXK && d_mask != nullptr) d_mask[r] = (prune && !(fabsf(mask[r]) > thr_mask)) ? 0.f : t;
  }
}

// d_att[k] = sum_r part[r, k]   (one block per k, fixed summation order -> deterministic)
__global__ void __launch_bounds__(256) wcompose_colsum_kernel(const float* __restrict__ part, long long rows, int kb,
                                                              float* __restrict__ d_att) {
  __shared__ float sh[8];
  const int k = blockIdx.x;
  float t = 0.f;
  for (long long r = threadIdx.x; r < rows; r += blockDim.x) t += part[r * kb + k];
  t = warp_sum(t);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < (int)((blockDim.x + 31) >> 5); ++i) s += sh[i];
    d_att[k] = s;
  }
}

// ------------------------------------------------------------------------------------------------- Swin token kernels
// window layout row (b, wh, ww, ph, pw)  <->  image row (b, (wh*ws+ph + shift) % H, (ww*ws+pw + shift) % W)
__device__ __forceinline__ long long window_row_to_image_row(long long r, int H, int W, int ws, int shift) {
  const int ws2 = ws * ws, nWw = W / ws, nWh = H / ws;
  const long long win = r / ws2;
  const int pos = (int)(r - win * ws2);
  const int ph = pos / ws, pw = pos - ph * ws;
  const int wwi = (int)(win % nWw);
  const long long t = win / nWw;
  const int whi = (int)(t % nWh);
  const long long b = t / nWh;
  const int hh = (whi * ws + ph + shift) % H, ww = (wwi * ws + pw + shift) % W;
  return (b * H + hh) * W + ww;
}

__device__ __forceinline__ long long image_row_to_window_row(long long r, int H, int W, int ws, int shift) {
  const int ws2 = ws * ws, nWw = W / ws, nWh = H / ws;
  const long long b = r / ((long long)H * W);
  const int rem = (int)(r - b * (long long)H * W);
  const int hh = rem / W, ww = rem - hh * W;
  const int h2 = (hh - shift + H) % H, w2 = (ww - shift + W) % W;
  const long long win = (b * nWh + h2 / ws) * nWw + w2 / ws;
  return win * ws2 + (h2 % ws) * ws + (w2 % ws);
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 p = __bfloat1622float2(h[t]);
    f[2 * t] = p.x;
    f[2 * t + 1] = p.y;
  }
}

__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int t = 0; t < 4; ++t) h[t] = __floats2bfloat162_rn(f[2 * t], f[2 * t + 1]);
  return u;
}

// One warp per destination row; VPL = 16-byte vectors per lane (C <= 256 * VPL). window != 0: the destination rows are
// in window layout and row r normalises the image row window_row_to_image_row(r).
template <int VPL>
__global__ void __launch_bounds__(256) ln_rows_kernel(const __nv_bfloat16* __restrict__ x,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      __nv_bfloat16* __restrict__ out, long long rows, int C, float eps,
                                                      int window, int H, int W, int ws, int shift,
                                                      float2* __restrict__ stats) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + warp;
  if (r >= rows) return;
  const long long src = window ? window_row_to_image_row(r, H, W, ws, shift) : r;
  const uint4* xp = reinterpret_cast<const uint4*>(x + src * C);
  const int nvec = C >> 3;
  float v[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      const uint4 u = xp[idx];
      unpack8(u, v[i]);
#pragma unroll
      for (int t = 0; t < 8; ++t) s += v[i][t];
    } else {
#pragma unroll
      for (int t = 0; t < 8; ++t) v[i][t] = 0.f;
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (lane + 32 * i < nvec) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float d = v[i][t] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
  if (stats != nullptr && lane == 0) stats[r] = make_float2(mean, rstd);       // saved for ln_rows_bwd_kernel
  uint4* op = reinterpret_cast<uint4*>(out + r * C);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      const float4 g0 = reinterpret_cast<const float4*>(gamma)[2 * idx], g1 = reinterpret_cast<const float4*>(gamma)[2 * idx + 1];
      const float4 b0 = reinterpret_cast<const float4*>(beta)[2 * idx], b1 = reinterpret_cast<const float4*>(beta)[2 * idx + 1];
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float y[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) y[t] = fmaf((v[i][t] - mean) * rstd, gg[t], bb[t]);
      op[idx] = pack8(y);
    }
  }
}

// LayerNorm backward for the TRAINABLE Swin stage (bf16 token rows, fp32 statistics saved by the forward kernel).
// One warp per destination row (the layout dy arrives in; window != 0: the forward wrote the shifted-window layout, so
// row r belongs to image row window_row_to_image_row(r), which is where dx goes - the map is a bijection, every image
// row is written exactly once). With xhat = (x - mean) * rstd and g = dy * gamma:
//     dx = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)),   dgamma += dy * xhat,   dbeta += dy.
// x and dy stay packed (bf16) in registers; each block walks its rows with a grid stride, folds the per-warp dgamma /
// dbeta partials through shared memory and writes ONE [2, C] partial per block: part[block][0] = dgamma, [1] = dbeta
// (ln_colsum_kernel adds the blocks in a fixed order: deterministic, no atomics).
template <int VPL>
__global__ void __launch_bounds__(256) ln_rows_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                          const __nv_bfloat16* __restrict__ x,
                                                          const float* __restrict__ gamma,
                                                          const float2* __restrict__ stats,
                                                          __nv_bfloat16* __restrict__ dx, float* __restrict__ part,
                                                          long long rows, int C, int window, int H, int W, int ws,
                                                          int shift) {
  __shared__ float sh[2][8][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  const float inv_c = 1.f / (float)C;
  // gamma stays in registers up to C = 1024; the widest instantiation (C <= 2048: Swin-L) re-reads it from L1 instead -
  // 64 more live registers there would spill
  constexpr bool kCacheGamma = VPL <= 4;
  constexpr int GV = kCacheGamma ? VPL : 1;
  float dg[VPL][8], db[VPL][8], gm[GV][8];
  auto load_gamma = [&](int idx, float* g8) {
    const float4 g0 = reinterpret_cast<const float4*>(gamma)[2 * idx], g1 = reinterpret_cast<const float4*>(gamma)[2 * idx + 1];
    g8[0] = g0.x; g8[1] = g0.y; g8[2] = g0.z; g8[3] = g0.w;
    g8[4] = g1.x; g8[5] = g1.y; g8[6] = g1.z; g8[7] = g1.w;
  };
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int idx = lane + 32 * i;
    if (kCacheGamma) {
      if (idx < nvec) {
        load_gamma(idx, gm[i % GV]);
      } else {
#pragma unroll
        for (int t = 0; t < 8; ++t) gm[i % GV][t] = 0.f;
      }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) dg[i][t] = db[i][t] = 0.f;
  }
  for (long long r = (long long)blockIdx.x * 8 + warp; r < rows; r += (long long)gridDim.x * 8) {
    const long long src = window ? window_row_to_image_row(r, H, W, ws, shift) : r;
    const uint4* xp = reinterpret_cast<const uint4*>(x + src * C);
    const uint4* yp = reinterpret_cast<const uint4*>(dy + r * C);
    const float2 st = stats[r];
    uint4 xu[VPL], yu[VPL];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) {
        xu[i] = xp[idx];
        yu[i] = yp[idx];
        float xv[8], yv[8], gl[8];
        unpack8(xu[i], xv);
        unpack8(yu[i], yv);
        if (!kCacheGamma) load_gamma(idx, gl);
        const float* gv = kCacheGamma ? gm[i % GV] : gl;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float xh = (xv[t] - st.x) * st.y;
          const float g = yv[t] * gv[t];
          s1 += g;
          s2 = fmaf(g, xh, s2);
          dg[i][t] = fmaf(yv[t], xh, dg[i][t]);
          db[i][t] += yv[t];
        }
      }
    }
    s1 = warp_sum(s1) * inv_c;
    s2 = warp_sum(s2) * inv_c;
    uint4* op = reinterpret_cast<uint4*>(dx + src * C);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) {
        float xv[8], yv[8], o[8], gl[8];
        unpack8(xu[i], xv);
        unpack8(yu[i], yv);
        if (!kCacheGamma) load_gamma(idx, gl);
        const float* gv = kCacheGamma ? gm[i % GV] : gl;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float xh = (xv[t] - st.x) * st.y;
          o[t] = st.y * (yv[t] * gv[t] - s1 - xh * s2);
        }
        op[idx] = pack8(o);
      }
    }
  }
  // fold the 8 warps' partials (every thread reaches these barriers: the row loop has no early exit)
  float* pg = part + (long long)blockIdx.x * 2 * C;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      sh[0][warp][lane * 8 + t] = dg[i][t];
      sh[1][warp][lane * 8 + t] = db[i][t];
    }
    __syncthreads();
    const int c = 256 * i + threadIdx.x;
    if (c < C) {
      float a = 0.f, b = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) {
        a += sh[0][w8][threadIdx.x];
        b += sh[1][w8][threadIdx.x];
      }
      pg[c] = a;
      pg[C + c] = b;
    }
    __syncthreads();
  }
}

// out[j] = sum_b part[b, j] over the per-block partials (j in [0, 2C): dgamma then dbeta), fixed order
__global__ void __launch_bounds__(256) ln_colsum_kernel(const float* __restrict__ part, int blocks, int n2,
                                                        float* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n2) return;
  float t = 0.f;
  for (int b = 0; b < blocks; ++b) t += part[(long long)b * n2 + j];
  out[j] = t;
}

// out[image row r] = shortcut[r] + scale[b(r)] * win[image_row_to_window_row(r)]   (8 channels per thread; scale: the
// per-sample drop-path factor 0 or 1 / keep of a TRAINABLE block, nullptr = 1)
__global__ void __launch_bounds__(256) window_merge_add_kernel(const __nv_bfloat16* __restrict__ win,
                                                               const __nv_bfloat16* __restrict__ shortcut,
                                                               __nv_bfloat16* __restrict__ out, long long rows, int C,
                                                               int H, int W, int ws, int shift,
                                                               const float* __restrict__ scale) {
  const int nvec = C >> 3;
  const long long total = rows * nvec;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long r = i / nvec;
    const int vi = (int)(i - r * nvec);
    const long long src = image_row_to_window_row(r, H, W, ws, shift);
    const uint4 a = reinterpret_cast<const uint4*>(shortcut + r * C)[vi];
    const uint4 b = reinterpret_cast<const uint4*>(win + src * C)[vi];
    float fa[8], fb[8];
    unpack8(a, fa);
    unpack8(b, fb);
    const float sc = scale != nullptr ? scale[r / ((long long)H * W)] : 1.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) fa[t] = fmaf(sc, fb[t], fa[t]);
    reinterpret_cast<uint4*>(out + r * C)[vi] = pack8(fa);
  }
}

// Backward of the merge w.r.t. the window-layout operand: dwin[window row r] = scale[b(r)] * dy[window_row_to_image_row(r)]
// (a pure gather; the gradient of the shortcut operand is dy itself).
__global__ void __launch_bounds__(256) window_gather_scale_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                  __nv_bfloat16* __restrict__ dwin, long long rows,
                                                                  int C, int H, int W, int ws, int shift,
                                                                  const float* __restrict__ scale) {
  const int nvec = C >> 3;
  const long long total = rows * nvec;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long r = i / nvec;
    const int vi = (int)(i - r * nvec);
    const long long src = window_row_to_image_row(r, H, W, ws, shift);
    uint4 v = reinterpret_cast<const uint4*>(dy + src * C)[vi];
    if (scale != nullptr) {
      float f[8];
      unpack8(v, f);
      const float sc = scale[src / ((long long)H * W)];
#pragma unroll
      for (int t = 0; t < 8; ++t) f[t] *= sc;
      v = pack8(f);
    }
    reinterpret_cast<uint4*>(dwin + r * C)[vi] = v;
  }
}

// exact GELU, 8 bf16 per thread
__global__ void __launch_bounds__(256) gelu_rows_kernel(const __nv_bfloat16* __restrict__ x,
                                                        __nv_bfloat16* __restrict__ out, long long nvec) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 u = reinterpret_cast<const uint4*>(x)[i];
    float f[8];
    unpack8(u, f);
#pragma unroll
    for (int t = 0; t < 8; ++t) f[t] = 0.5f * f[t] * (1.f + erff(f[t] * 0.70710678118654752440f));
    reinterpret_cast<uint4*>(out)[i] = pack8(f);
  }
}

// d/dx GELU(x) = Phi(x) + x * phi(x)   (exact form; x is the saved pre-activation), 8 bf16 per thread
__global__ void __launch_bounds__(256) gelu_bwd_rows_kernel(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ dy,
                                                            __nv_bfloat16* __restrict__ dx, long long nvec) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float f[8], g[8];
    unpack8(reinterpret_cast<const uint4*>(x)[i], f);
    unpack8(reinterpret_cast<const uint4*>(dy)[i], g);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float cdf = 0.5f * (1.f + erff(f[t] * 0.70710678118654752440f));
      const float pdf = 0.39894228040143267794f * expf(-0.5f * f[t] * f[t]);
      g[t] *= fmaf(f[t], pdf, cdf);
    }
    reinterpret_cast<uint4*>(dx)[i] = pack8(g);
  }
}

// C2 tail on the receiving client: master <- aggregated parameters, bf16 compute copy refreshed and the FedProx anchor
// snapshotted in the same pass (snap_mode 1: the weights being replaced = the reference's order of operations,
// methods/fedprox.py:351-364; 2: the incoming global model = textbook FedProx). 4 floats per thread.
__global__ void __launch_bounds__(256) apply_global_kernel(const float4* __restrict__ flat, float4* __restrict__ master,
                                                           uint2* __restrict__ shadow, float4* __restrict__ p_old,
                                                           int snap_mode, long long n4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = flat[i];
    if (p_old != nullptr) {
      if (snap_mode == 1) p_old[i] = master[i];
      else if (snap_mode == 2) p_old[i] = v;
    }
    master[i] = v;
    if (shadow != nullptr) {
      uint2 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
      h[0] = __floats2bfloat162_rn(v.x, v.y);
      h[1] = __floats2bfloat162_rn(v.z, v.w);
      shadow[i] = u;
    }
  }
}

static int grid_for(long long work_items, int threads) {
  long long g = (work_items + threads - 1) / threads;
  const long long cap = 132LL * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace flpr

using namespace flpr;

extern "C" {

int flpr_wcompose_max_k() { return WC_MAXK; }

// n must be a multiple of 4 and every pointer 16-byte aligned (8 for shadow): arena prefixes are.
int flpr_apply_global(const float* flat, float* master, void* shadow, float* p_old, int snap_mode, long long n,
                      cudaStream_t st) {
  if (n <= 0) return 0;
  if (n % 4) return -25;
  if (((uintptr_t)flat | (uintptr_t)master | (uintptr_t)p_old) & 15 || ((uintptr_t)shadow & 7)) return -26;
  bind_device_of(master);
  apply_global_kernel<<<grid_for(n / 4, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(flat),
                                                            reinterpret_cast<float4*>(master),
                                                            reinterpret_cast<uint2*>(shadow),
                                                            reinterpret_cast<float4*>(p_old), snap_mode, n / 4);
  return (int)cudaGetLastError();
}

int flpr_wcompose_fwd(const float* aw, const float* stack, const float* atten, int kb, int ks, const float* sw,
                      const float* mask, long long row_len, float thr_aw, float thr_mask, int prune, float* out_f32,
                      void* out_bf16, long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  if (kb < 0 || kb > WC_MAXK || (kb > 0 && ks < kb) || row_len <= 0) return -21;
  bind_device_of(aw);
  wcompose_fwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(aw, stack, atten, kb, ks, sw, mask, row_len, thr_aw, thr_mask,
                                                        prune, out_f32, reinterpret_cast<__nv_bfloat16*>(out_bf16), n);
  return (int)cudaGetLastError();
}

// part_att: [rows, kb] scratch; d_att: [kb]; d_aw may be null (no pruning: d aw == d theta); d_mask null without sw.
int flpr_wcompose_bwd(const float* dth, const float* aw, const float* stack, int kb, int ks, const float* sw,
                      const float* mask, long long row_len, float thr_aw, float thr_mask, int prune, float* d_aw,
                      float* part_att, float* d_mask, float* d_att, long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  if (kb < 0 || kb > WC_MAXK || (kb > 0 && ks < kb) || row_len <= 0) return -21;
  bind_device_of(dth);
  const long long rows = (n + row_len - 1) / row_len;
  if (rows > 0x7fffffffLL) return -22;
  wcompose_bwd_kernel<<<(unsigned)rows, 256, 0, st>>>(dth, aw, stack, kb, ks, sw, mask, row_len, thr_aw, thr_mask, prune,
                                                      d_aw, part_att, d_mask, n);
  int rc = (int)cudaGetLastError();
  if (rc) return rc;
  if (kb > 0 && d_att != nullptr) {
    wcompose_colsum_kernel<<<kb, 256, 0, st>>>(part_att, rows, kb, d_att);
    rc = (int)cudaGetLastError();
  }
  return rc;
}

// LayerNorm over rows of C bf16 channels (C % 8 == 0, C <= 2048). window != 0: see ln_rows_kernel.
static int ln_rows_launch(const void* x, const float* gamma, const float* beta, void* out, long long rows, int C,
                          float eps, int window, int H, int W, int ws, int shift, float2* stats, cudaStream_t st);

int flpr_ln_rows(const void* x, const float* gamma, const float* beta, void* out, long long rows, int C, float eps,
                 int window, int H, int W, int ws, int shift, cudaStream_t st) {
  return ln_rows_launch(x, gamma, beta, out, rows, C, eps, window, H, W, ws, shift, nullptr, st);
}

// Training forward: same kernel, the per-row (mean, rstd) pairs are kept for flpr_ln_rows_bwd (stats: [rows, 2] fp32).
int flpr_ln_rows_train(const void* x, const float* gamma, const float* beta, void* out, float* stats, long long rows,
                       int C, float eps, int window, int H, int W, int ws, int shift, cudaStream_t st) {
  if (stats == nullptr || ((uintptr_t)stats & 7)) return -27;
  return ln_rows_launch(x, gamma, beta, out, rows, C, eps, window, H, W, ws, shift, reinterpret_cast<float2*>(stats), st);
}

// Blocks the backward kernel is launched with for `rows` rows (= rows of the partial buffer the caller allocates).
int flpr_ln_rows_bwd_blocks(long long rows) {
  long long g = (rows + 7) / 8;
  if (g > 132LL * 2) g = 132LL * 2;
  if (g < 1) g = 1;
  return (int)g;
}

// dy: [rows, C] bf16 in the forward's DESTINATION layout; x: the forward's input; dx: same layout as x;
// part: [flpr_ln_rows_bwd_blocks(rows), 2, C] fp32 scratch; dgb: [2, C] fp32 (dgamma, dbeta).
int flpr_ln_rows_bwd(const void* dy, const void* x, const float* gamma, const float* stats, void* dx, float* part,
                     float* dgb, long long rows, int C, int window, int H, int W, int ws, int shift, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8 || C <= 0 || C > 2048) return -23;
  if (window && (ws <= 0 || H % ws || W % ws || shift < 0 || shift >= ws || rows % ((long long)H * W))) return -24;
  if (((uintptr_t)stats & 7) || ((uintptr_t)gamma & 15)) return -27;
  bind_device_of(x);
  const int grid = flpr_ln_rows_bwd_blocks(rows);
  const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(dy);
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(dx);
  const float2* sp = reinterpret_cast<const float2*>(stats);
  const int nvec = C / 8;
  if (nvec <= 32)
    ln_rows_bwd_kernel<1><<<grid, 256, 0, st>>>(yp, xp, gamma, sp, op, part, rows, C, window, H, W, ws, shift);
  else if (nvec <= 64)
    ln_rows_bwd_kernel<2><<<grid, 256, 0, st>>>(yp, xp, gamma, sp, op, part, rows, C, window, H, W, ws, shift);
  else if (nvec <= 128)
    ln_rows_bwd_kernel<4><<<grid, 256, 0, st>>>(yp, xp, gamma, sp, op, part, rows, C, window, H, W, ws, shift);
  else
    ln_rows_bwd_kernel<8><<<grid, 256, 0, st>>>(yp, xp, gamma, sp, op, part, rows, C, window, H, W, ws, shift);
  int rc = (int)cudaGetLastError();
  if (rc) return rc;
  ln_colsum_kernel<<<(2 * C + 255) / 256, 256, 0, st>>>(part, grid, 2 * C, dgb);
  return (int)cudaGetLastError();
}

static int ln_rows_launch(const void* x, const float* gamma, const float* beta, void* out, long long rows, int C,
                          float eps, int window, int H, int W, int ws, int shift, float2* stats, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8 || C <= 0 || C > 2048) return -23;
  if (window && (ws <= 0 || H % ws || W % ws || shift < 0 || shift >= ws || rows % ((long long)H * W))) return -24;
  bind_device_of(x);
  const unsigned grid = (unsigned)((rows + 7) / 8);
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(out);
  const int nvec = C / 8;
  if (nvec <= 32)
    ln_rows_kernel<1><<<grid, 256, 0, st>>>(xp, gamma, beta, op, rows, C, eps, window, H, W, ws, shift, stats);
  else if (nvec <= 64)
    ln_rows_kernel<2><<<grid, 256, 0, st>>>(xp, gamma, beta, op, rows, C, eps, window, H, W, ws, shift, stats);
  else if (nvec <= 128)
    ln_rows_kernel<4><<<grid, 256, 0, st>>>(xp, gamma, beta, op, rows, C, eps, window, H, W, ws, shift, stats);
  else
    ln_rows_kernel<8><<<grid, 256, 0, st>>>(xp, gamma, beta, op, rows, C, eps, window, H, W, ws, shift, stats);
  return (int)cudaGetLastError();
}

int flpr_window_merge_add(const void* win, const void* shortcut, void* out, long long rows, int C, int H, int W, int ws,
                          int shift, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8 || ws <= 0 || H % ws || W % ws || shift < 0 || shift >= ws || rows % ((long long)H * W)) return -24;
  bind_device_of(win);
  window_merge_add_kernel<<<grid_for(rows * (C / 8), 256), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(win), reinterpret_cast<const __nv_bfloat16*>(shortcut),
      reinterpret_cast<__nv_bfloat16*>(out), rows, C, H, W, ws, shift, nullptr);
  return (int)cudaGetLastError();
}

// Trainable block: out = shortcut + scale[sample] * merge(win)  (scale: [rows / (H*W)] fp32, nullable).
int flpr_window_merge_add_scaled(const void* win, const void* shortcut, const float* scale, void* out, long long rows,
                                 int C, int H, int W, int ws, int shift, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8 || ws <= 0 || H % ws || W % ws || shift < 0 || shift >= ws || rows % ((long long)H * W)) return -24;
  bind_device_of(win);
  window_merge_add_kernel<<<grid_for(rows * (C / 8), 256), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(win), reinterpret_cast<const __nv_bfloat16*>(shortcut),
      reinterpret_cast<__nv_bfloat16*>(out), rows, C, H, W, ws, shift, scale);
  return (int)cudaGetLastError();
}

// Its backward w.r.t. win: dwin = scale[sample] * gather(dy) in window layout.
int flpr_window_gather_scale(const void* dy, const float* scale, void* dwin, long long rows, int C, int H, int W, int ws,
                             int shift, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8 || ws <= 0 || H % ws || W % ws || shift < 0 || shift >= ws || rows % ((long long)H * W)) return -24;
  bind_device_of(dy);
  window_gather_scale_kernel<<<grid_for(rows * (C / 8), 256), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<__nv_bfloat16*>(dwin), rows, C, H, W, ws, shift,
      scale);
  return (int)cudaGetLastError();
}

int flpr_gelu_bwd_rows(const void* x, const void* dy, void* dx, long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  if (n % 8) return -23;
  bind_device_of(x);
  gelu_bwd_rows_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                            reinterpret_cast<const __nv_bfloat16*>(dy),
                                                            reinterpret_cast<__nv_bfloat16*>(dx), n / 8);
  return (int)cudaGetLastError();
}

int flpr_gelu_rows(const void* x, void* out, long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  if (n % 8) return -23;
  bind_device_of(x);
  gelu_rows_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                         reinterpret_cast<__nv_bfloat16*>(out), n / 8);
  return (int)cudaGetLastError();
}

}  // extern "C"
