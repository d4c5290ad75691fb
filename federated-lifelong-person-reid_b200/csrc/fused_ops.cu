// flpr fused memory-bound kernels for the local training step (all flat-arena, multi-tensor by construction:
// every client keeps its trainable state in ONE contiguous fp32 arena, so "multi-tensor apply" is one launch).
//
//   adam / sgd        optimizer step fused with (a) the continual-learning quadratic penalty gradient
//                     2*lam*(Q*p - R)  [EWC ewc.py:80-85, MAS mas.py:78-83, FedProx fedprox.py:52-57,
//                     FedCurv fedcurv.py:79-86 all reduce to this form], (b) FedSTIL's L1 sparseness gradient
//                     lam1*sign(theta - G) and adaptive-weight decay (fedstil.py:639-644), (c) the bf16 compute
//                     copy of the updated weights, (d) the penalty / L1 *values* for loss reporting, (e) with the SI
//                     flag, the Synaptic Intelligence path integral omega += -g * (p_new - p_old).
//   importance_accum  Fisher (g^2) / MAS (|g|) accumulation (ewc.py:56-78, mas.py:55-76, fedcurv.py:56-77).
//   ce_label_smooth   fused log-softmax + label-smoothing CE + gradient + top-1 hit count
//                     (criterions/cross_entropy.py:35-40 and the per-step accuracy at baseline.py:47).
//   bn_*              NHWC bf16 batch-norm training kernels (stats, apply+residual+ReLU, backward).
//   rank_eval         CMC first-hit + average precision per query straight from the similarity matrix
//                     (tools/evaluate.py:11-142) without sorting.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ptx.cuh"

namespace flpr {

__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  v = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) v = warp_sum(v);
  return v;  // valid in warp 0
}

struct OptArgs {
  float* p;             // fp32 master
  const float* g;       // fp32 gradient
  float* m;             // exp_avg / momentum buffer
  float* v;             // exp_avg_sq (adam)
  const float* Q;       // penalty curvature (nullable)
  const float* R;       // penalty linear term (nullable)
  const float* G;       // FedSTIL global weight (nullable)
  __nv_bfloat16* p_bf16;  // compute copy (nullable)
  float* stats;         // [0] += sum(Q p^2 - 2 R p), [1] += sum |p - G|   (nullable)
  float* stats_part;    // per-block partials of the two sums, folded into stats in block order by opt_stats_kernel
  size_t n;
  float lr, beta1, beta2, eps, wd, bc1, bc2_sqrt;
  float lam2;           // penalty strength (gradient gets 2*lam2*(Q p - R))
  float lam1;           // L1 strength
  float atten;          // FedSTIL attention scalar a: adaptive weight A = p - a*G (weight decay acts on A)
  float momentum;
  int penalty_ones;     // FedProx: Q == 1 without materialising it
  const float* hyper;   // optional device-resident [lr, step]: keeps a captured CUDA graph valid across steps
  // FedSTIL trained L1 anchor (reference quirk, methods/fedstil.py:53-76,639-647): `initial_adaptive_weight` is a bare
  // Parameter whose requires_grad is never cleared, so the reference's optimizer trains the anchor of the L1 term too
  // (gradient -lam1*sign(aw - aw0) + wd*aw0, own moments). `anchor` holds theta0 = atten*G + aw0 (nullable = constant
  // anchor G); am / av are its exp_avg (or momentum buffer) / exp_avg_sq.
  float* anchor;
  float* am;
  float* av;
  // Synaptic Intelligence path integral (Zenke et al. 2017, Eq. 4), read and written by the SI instantiation only:
  // omega += -g * (p_new - p_old) per element, with g the loss gradient as passed in (before the L1, penalty and
  // weight-decay terms). Last field, so the offsets of the others are those of the non-SI kernels.
  float* omega;
};

template <bool ADAM, bool SI>
__global__ void __launch_bounds__(256) fused_opt_kernel(const OptArgs a) {
  __shared__ float sh[8];
  float pen = 0.f, l1 = 0.f;
  float lr = a.lr, bc1 = a.bc1, bc2_sqrt = a.bc2_sqrt;
  if (a.hyper != nullptr) {
    lr = a.hyper[0];
    const float step = a.hyper[1];
    bc1 = 1.f - powf(a.beta1, step);
    bc2_sqrt = sqrtf(1.f - powf(a.beta2, step));
  }
  const size_t n4 = a.n >> 2;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 p4 = reinterpret_cast<const float4*>(a.p)[i];
    const float4 g4 = reinterpret_cast<const float4*>(a.g)[i];
    float4 m4 = make_float4(0.f, 0.f, 0.f, 0.f), v4 = m4, q4 = m4, r4 = m4, G4 = m4;
    if (ADAM || a.momentum != 0.f) m4 = reinterpret_cast<const float4*>(a.m)[i];
    if (ADAM) v4 = reinterpret_cast<const float4*>(a.v)[i];
    if (a.Q) q4 = reinterpret_cast<const float4*>(a.Q)[i];
    if (a.R) r4 = reinterpret_cast<const float4*>(a.R)[i];
    if (a.G) G4 = reinterpret_cast<const float4*>(a.G)[i];
    float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (SI) w4 = reinterpret_cast<const float4*>(a.omega)[i];
    float* ww = reinterpret_cast<float*>(&w4);
    float4 c4 = G4, cm4 = make_float4(0.f, 0.f, 0.f, 0.f), cv4 = cm4;
    if (a.anchor) {
      c4 = reinterpret_cast<const float4*>(a.anchor)[i];
      if (ADAM || a.momentum != 0.f) cm4 = reinterpret_cast<const float4*>(a.am)[i];
      if (ADAM) cv4 = reinterpret_cast<const float4*>(a.av)[i];
    }
    float* cc = reinterpret_cast<float*>(&c4);
    float* cmm = reinterpret_cast<float*>(&cm4);
    float* cvv = reinterpret_cast<float*>(&cv4);
    float* pp = reinterpret_cast<float*>(&p4);
    const float* gg = reinterpret_cast<const float*>(&g4);
    float* mm = reinterpret_cast<float*>(&m4);
    float* vv = reinterpret_cast<float*>(&v4);
    const float* qq = reinterpret_cast<const float*>(&q4);
    const float* rr = reinterpret_cast<const float*>(&r4);
    const float* GG = reinterpret_cast<const float*>(&G4);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float p = pp[t];
      float g = gg[t];
      float decay_base = p;
      if (a.G) {
        const float d = p - cc[t];                         // cc = G unless the anchor is trained
        l1 += fabsf(d);
        float sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
        // Where the loss gradient is exactly zero weight and anchor receive the same update and stay identical in the
        // reference (sign(0) = 0); differently fused update formulas cannot promise that bit for bit, so differences
        // at rounding level (1e-6 of a step) count as zero.
        if (a.anchor && fabsf(d) <= 1e-6f * lr) sgn = 0.f;
        g += a.lam1 * sgn;
        decay_base = p - a.atten * GG[t];
        if (a.anchor) {
          const float c = cc[t];
          const float g0 = -a.lam1 * sgn + a.wd * (c - a.atten * GG[t]);
          if (ADAM) {
            const float m0 = a.beta1 * cmm[t] + (1.f - a.beta1) * g0;
            const float v0 = a.beta2 * cvv[t] + (1.f - a.beta2) * g0 * g0;
            cmm[t] = m0;
            cvv[t] = v0;
            cc[t] = c - (lr / bc1) * (m0 / (sqrtf(v0) / bc2_sqrt + a.eps));
          } else {
            float d0 = g0;
            if (a.momentum != 0.f) {
              d0 = a.momentum * cmm[t] + g0;
              cmm[t] = d0;
            }
            cc[t] = c - lr * d0;
          }
        }
      }
      if (a.R) {
        const float q = a.penalty_ones ? 1.f : qq[t];
        pen += q * p * p - 2.f * rr[t] * p;
        g += 2.f * a.lam2 * (q * p - rr[t]);
      }
      g += a.wd * decay_base;
      float np;
      if (ADAM) {
        const float m = a.beta1 * mm[t] + (1.f - a.beta1) * g;
        const float v = a.beta2 * vv[t] + (1.f - a.beta2) * g * g;
        mm[t] = m;
        vv[t] = v;
        const float denom = sqrtf(v) / bc2_sqrt + a.eps;
        np = p - (lr / bc1) * (m / denom);
      } else {
        float d = g;
        if (a.momentum != 0.f) {
          d = a.momentum * mm[t] + g;
          mm[t] = d;
        }
        np = p - lr * d;
      }
      pp[t] = np;
      if (SI) ww[t] = fmaf(-gg[t], np - p, ww[t]);
    }
    reinterpret_cast<float4*>(a.p)[i] = p4;
    if (SI) reinterpret_cast<float4*>(a.omega)[i] = w4;
    if (ADAM || a.momentum != 0.f) reinterpret_cast<float4*>(a.m)[i] = m4;
    if (ADAM) reinterpret_cast<float4*>(a.v)[i] = v4;
    if (a.anchor) {
      reinterpret_cast<float4*>(a.anchor)[i] = c4;
      if (ADAM || a.momentum != 0.f) reinterpret_cast<float4*>(a.am)[i] = cm4;
      if (ADAM) reinterpret_cast<float4*>(a.av)[i] = cv4;
    }
    if (a.p_bf16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&lo);
      u.y = *reinterpret_cast<uint32_t*>(&hi);
      reinterpret_cast<uint2*>(a.p_bf16)[i] = u;
    }
  }
  if (a.stats) {
    const float s0 = block_sum(pen, sh);
    const float s1 = block_sum(l1, sh);
    if (threadIdx.x == 0) {
      a.stats_part[2 * blockIdx.x] = s0;
      a.stats_part[2 * blockIdx.x + 1] = s1;
    }
  }
}

// stats[0] += sum of the blocks' penalty partials (when R is given), stats[1] += L1 partials (when G is given), in
// block order: the reported penalty is reproducible.
__global__ void opt_stats_kernel(const float* part, float* stats, int blocks, int has_r, int has_g) {
  if (threadIdx.x != 0) return;
  float s0 = 0.f, s1 = 0.f;
  for (int b = 0; b < blocks; ++b) {
    s0 += part[2 * b];
    s1 += part[2 * b + 1];
  }
  if (has_r) stats[0] += s0;
  if (has_g) stats[1] += s1;
}

// F += scale * g^2 (mode 0) or scale * |g| (mode 1)
__global__ void __launch_bounds__(256) importance_accum_kernel(float* F, const float* g, size_t n, float scale,
                                                               int mode) {
  const size_t n4 = n >> 2, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 f = reinterpret_cast<float4*>(F)[i];
    const float4 x = reinterpret_cast<const float4*>(g)[i];
    if (mode == 0) {
      f.x = fmaf(scale * x.x, x.x, f.x); f.y = fmaf(scale * x.y, x.y, f.y);
      f.z = fmaf(scale * x.z, x.z, f.z); f.w = fmaf(scale * x.w, x.w, f.w);
    } else {
      f.x += scale * fabsf(x.x); f.y += scale * fabsf(x.y); f.z += scale * fabsf(x.z); f.w += scale * fabsf(x.w);
    }
    reinterpret_cast<float4*>(F)[i] = f;
  }
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* x, __nv_bfloat16* y, size_t n) {
  const size_t n4 = n >> 2, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
    reinterpret_cast<uint2*>(y)[i] = u;
  }
}

// theta = a * G + A   (adaptive compose, fedstil.py:85,120) with bf16 compute copy; scalar attention
__global__ void __launch_bounds__(256) compose_kernel(const float* G, const float* A, float a, float* theta,
                                                      __nv_bfloat16* theta_bf16, size_t n) {
  const size_t n4 = n >> 2, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 g = reinterpret_cast<const float4*>(G)[i];
    const float4 w = reinterpret_cast<const float4*>(A)[i];
    const float4 t = make_float4(fmaf(a, g.x, w.x), fmaf(a, g.y, w.y), fmaf(a, g.z, w.z), fmaf(a, g.w, w.w));
    if (theta) reinterpret_cast<float4*>(theta)[i] = t;
    if (theta_bf16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(t.x, t.y), hi = __floats2bfloat162_rn(t.z, t.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&lo);
      u.y = *reinterpret_cast<uint32_t*>(&hi);
      reinterpret_cast<uint2*>(theta_bf16)[i] = u;
    }
  }
}

// ----------------------------------------------------------------------------- server optimizer
// One step of the server optimizer of adaptive federated optimization (Reddi et al., ICLR 2021, Algorithm 2, without
// bias correction; FedAvgM, Hsu et al. 2019). x: the server replica's upload prefix, mean: the aggregated uploads.
// The pseudo-gradient d = mean - x lives in registers only; m, v are fp32.
//   SOPT_SGD      m = momentum*m + d                                      x += lr*m
//   SOPT_ADAGRAD  m = b1*m + (1-b1)*d   v = v + d^2                       x += lr*m / (sqrt(v) + tau)
//   SOPT_ADAM     m = b1*m + (1-b1)*d   v = b2*v + (1-b2)*d^2             x += lr*m / (sqrt(v) + tau)
//   SOPT_YOGI     m = b1*m + (1-b1)*d   v = v - (1-b2)*d^2*sign(v - d^2)  x += lr*m / (sqrt(v) + tau)
// The bf16 compute copy of x (nullable) is written in the same pass. This is not fused_opt_kernel: that one is the
// client hot path (gradient buffer, Adam bias correction, penalties), and sharing it would make it branch on its caller.
enum { SOPT_SGD = 0, SOPT_ADAGRAD = 1, SOPT_ADAM = 2, SOPT_YOGI = 3 };

struct ServerOptArgs {
  float* x;
  const float* mean;
  float* m;
  float* v;                  // unused by SOPT_SGD
  __nv_bfloat16* x_bf16;     // nullable
  size_t n;
  float lr, momentum, beta1, beta2, tau;
};

template <int RULE>
__device__ __forceinline__ void server_opt_elem(const ServerOptArgs& a, float& x, const float mean, float& m,
                                                float& v) {
  const float d = mean - x;
  if (RULE == SOPT_SGD) {
    m = a.momentum * m + d;
    x = x + a.lr * m;
    return;
  }
  m = a.beta1 * m + (1.f - a.beta1) * d;
  const float d2 = d * d;
  if (RULE == SOPT_ADAGRAD) {
    v = v + d2;
  } else if (RULE == SOPT_ADAM) {
    v = a.beta2 * v + (1.f - a.beta2) * d2;
  } else {
    const float s = v - d2;
    const float sgn = (s > 0.f) ? 1.f : ((s < 0.f) ? -1.f : 0.f);
    v = v - (1.f - a.beta2) * d2 * sgn;
  }
  x = x + a.lr * m / (sqrtf(v) + a.tau);
}

// vec: every operand is 16-byte aligned (x_bf16: 8-byte) - float4 accesses over n / 4 quads, then a scalar tail;
// otherwise scalar accesses throughout.
template <int RULE>
__global__ void __launch_bounds__(256) server_opt_kernel(const ServerOptArgs a, const int vec) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t head = 0;
  if (vec) {
    const size_t n4 = a.n >> 2;
    for (size_t i = tid; i < n4; i += stride) {
      float4 x4 = reinterpret_cast<const float4*>(a.x)[i];
      const float4 u4 = reinterpret_cast<const float4*>(a.mean)[i];
      float4 m4 = reinterpret_cast<const float4*>(a.m)[i];
      float4 v4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (RULE != SOPT_SGD) v4 = reinterpret_cast<const float4*>(a.v)[i];
      server_opt_elem<RULE>(a, x4.x, u4.x, m4.x, v4.x);
      server_opt_elem<RULE>(a, x4.y, u4.y, m4.y, v4.y);
      server_opt_elem<RULE>(a, x4.z, u4.z, m4.z, v4.z);
      server_opt_elem<RULE>(a, x4.w, u4.w, m4.w, v4.w);
      reinterpret_cast<float4*>(a.x)[i] = x4;
      reinterpret_cast<float4*>(a.m)[i] = m4;
      if (RULE != SOPT_SGD) reinterpret_cast<float4*>(a.v)[i] = v4;
      if (a.x_bf16) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(x4.x, x4.y), hi = __floats2bfloat162_rn(x4.z, x4.w);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&lo);
        u.y = *reinterpret_cast<uint32_t*>(&hi);
        reinterpret_cast<uint2*>(a.x_bf16)[i] = u;
      }
    }
    head = n4 << 2;
  }
  for (size_t i = head + tid; i < a.n; i += stride) {
    float x = a.x[i], m = a.m[i], v = 0.f;
    if (RULE != SOPT_SGD) v = a.v[i];
    server_opt_elem<RULE>(a, x, a.mean[i], m, v);
    a.x[i] = x;
    a.m[i] = m;
    if (RULE != SOPT_SGD) a.v[i] = v;
    if (a.x_bf16) a.x_bf16[i] = __float2bfloat16_rn(x);
  }
}

// ----------------------------------------------------------------------------- label-smoothing CE
// One block per sample. logits: [B, C] (bf16 or fp32, row stride ld). dlogits same layout (bf16 or fp32).
// row_part[2 row] = loss_row / B, row_part[2 row + 1] = (argmax == target); ce_stats_kernel folds them into stats.
template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256) ce_ls_kernel(const TIn* logits, const long long* target, TOut* dlogits,
                                                    float* row_part, int B, int C, long long ld, float eps,
                                                    float grad_scale) {
  __shared__ float sh[8];
  __shared__ float s_bcast[2];
  __shared__ int s_arg;
  const int row = blockIdx.x;
  const TIn* z = logits + (long long)row * ld;
  // pass 1: max (+ argmax) and sum of logits
  float mx = -INFINITY, sumz = 0.f;
  int arg = 0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float x = static_cast<float>(z[c]);
    sumz += x;
    if (x > mx) { mx = x; arg = c; }
  }
  // block argmax (first index wins on ties, like torch.max)
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
  }
  __shared__ float s_mx[8];
  __shared__ int s_ai[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_mx[w] = mx; s_ai[w] = arg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float bm = s_mx[0];
    int ba = s_ai[0];
    for (int i = 1; i < (blockDim.x >> 5); ++i)
      if (s_mx[i] > bm || (s_mx[i] == bm && s_ai[i] < ba)) { bm = s_mx[i]; ba = s_ai[i]; }
    s_bcast[0] = bm;
    s_arg = ba;
  }
  __syncthreads();
  mx = s_bcast[0];
  const float tot_z = block_sum(sumz, sh);
  // pass 2: sum exp
  float se = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) se += __expf(static_cast<float>(z[c]) - mx);
  const float tot_e = block_sum(se, sh);
  if (threadIdx.x == 0) s_bcast[1] = tot_e;
  __syncthreads();
  const float lse = mx + logf(s_bcast[1]);
  const long long y = target[row];
  if (threadIdx.x == 0) {
    const float zy = static_cast<float>(z[y]);
    // -(1-eps)*(z_y - lse) - eps/C * (sum z - C*lse)
    const float loss = -(1.f - eps) * (zy - lse) - (eps / C) * (tot_z - C * lse);
    row_part[2 * row] = loss / B;
    row_part[2 * row + 1] = s_arg == (int)y ? 1.f : 0.f;
  }
  if (dlogits != nullptr) {
    TOut* d = dlogits + (long long)row * ld;
    const float smooth = eps / C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const float pr = __expf(static_cast<float>(z[c]) - lse);
      const float t = smooth + ((c == (int)y) ? (1.f - eps) : 0.f);
      d[c] = static_cast<TOut>((pr - t) * grad_scale);
    }
  }
}

// stats[0] += sum of the rows' losses, stats[1] += hits, summed in row order (a reproducible loss value).
__global__ void ce_stats_kernel(const float* row_part, float* stats, int B) {
  if (threadIdx.x != 0) return;
  float loss = 0.f, hits = 0.f;
  for (int r = 0; r < B; ++r) {
    loss += row_part[2 * r];
    hits += row_part[2 * r + 1];
  }
  stats[0] += loss;
  stats[1] += hits;
}

// ----------------------------------------------------------------------------- batch norm (NHWC, [M, C] bf16)
// Column statistics of x[M, C] (bf16): every thread owns 8 adjacent channels (one 16-byte load per row), the rows
// are split over blockIdx.y (and threadIdx.y when C/8 < 256); per-block partial sums go to part[gridDim.y][2][C]
// (no atomics, deterministic) and bn_finalize_kernel folds the partials.
__global__ void __launch_bounds__(256) bn_stats_kernel(const __nv_bfloat16* x, float* part, int M, int C,
                                                       int rows_per_block) {
  __shared__ float sh[16 * 256];
  const int c8n = C / 8;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c8 = blockIdx.x * blockDim.x + tx;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, M);
  float s[8], q[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { s[t] = 0.f; q[t] = 0.f; }
  if (c8 < c8n) {
    const uint4* xp = reinterpret_cast<const uint4*>(x);
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += blockDim.y) {
      const uint4 u = xp[(size_t)r * c8n + c8];
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = __bfloat1622float2(h[t]);
        s[2 * t] += f.x; s[2 * t + 1] += f.y;
        q[2 * t] = fmaf(f.x, f.x, q[2 * t]); q[2 * t + 1] = fmaf(f.y, f.y, q[2 * t + 1]);
      }
    }
  }
  const int tid = ty * blockDim.x + tx;
  for (int off = blockDim.y >> 1; off > 0; off >>= 1) {   // fold the row-lanes of this block
    __syncthreads();
    if (ty >= off && ty < 2 * off) {
#pragma unroll
      for (int t = 0; t < 8; ++t) { sh[(t * 2) * 256 + tid - off * blockDim.x] = s[t]; sh[(t * 2 + 1) * 256 + tid - off * blockDim.x] = q[t]; }
    }
    __syncthreads();
    if (ty < off) {
#pragma unroll
      for (int t = 0; t < 8; ++t) { s[t] += sh[(t * 2) * 256 + tid]; q[t] += sh[(t * 2 + 1) * 256 + tid]; }
    }
  }
  if (ty == 0 && c8 < c8n) {
    float* ps = part + (size_t)blockIdx.y * 2 * C + c8 * 8;
    float* pq = ps + C;
    reinterpret_cast<float4*>(ps)[0] = make_float4(s[0], s[1], s[2], s[3]);
    reinterpret_cast<float4*>(ps)[1] = make_float4(s[4], s[5], s[6], s[7]);
    reinterpret_cast<float4*>(pq)[0] = make_float4(q[0], q[1], q[2], q[3]);
    reinterpret_cast<float4*>(pq)[1] = make_float4(q[4], q[5], q[6], q[7]);
  }
}

// Fold per-block partials part[nparts][2][C] -> two per-channel sums. blockDim = (32 channels, FOLD_LANES part-lanes).
constexpr int FOLD_LANES = 32;
__device__ __forceinline__ void fold_partials(const float* part, int nparts, int C, int c, float& s0, float& s1,
                                              float (*sh)[FOLD_LANES][33]) {
  float a = 0.f, b = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int i = threadIdx.y; i < nparts; i += FOLD_LANES) {
      a += part[(size_t)i * 2 * C + c];
      b += part[(size_t)i * 2 * C + C + c];
    }
  }
  sh[0][threadIdx.y][threadIdx.x] = a;
  sh[1][threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  s0 = 0.f; s1 = 0.f;
  if (threadIdx.y == 0) {
#pragma unroll
    for (int j = 0; j < FOLD_LANES; ++j) { s0 += sh[0][j][threadIdx.x]; s1 += sh[1][j][threadIdx.x]; }
  }
}

// finalize: fold partials, mean/rstd, running stats (momentum, unbiased var), scale/shift for the apply pass
__global__ void __launch_bounds__(32 * FOLD_LANES) bn_finalize_kernel(const float* part, int nparts, const float* gamma,
                                                          const float* beta, float* mean, float* rstd, float* scale,
                                                          float* shift, float* running_mean, float* running_var, int M,
                                                          int C, float eps, float momentum) {
  __shared__ float sh[2][FOLD_LANES][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float sm, sq;
  fold_partials(part, nparts, C, c, sm, sq, sh);
  if (threadIdx.y != 0 || c >= C) return;
  const float mu = sm / M;
  float var = sq / M - mu * mu;
  var = fmaxf(var, 0.f);
  const float rs = rsqrtf(var + eps);
  mean[c] = mu;
  rstd[c] = rs;
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  scale[c] = g * rs;
  shift[c] = b - mu * g * rs;
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
    const float unb = (M > 1) ? var * ((float)M / (float)(M - 1)) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unb;
  }
}

// y = relu?(x * ca[c] + cb[c] (+ residual)); row-strided: every thread keeps its 8 channels' coefficients in
// registers and walks the rows of its block (grid = (channel groups, row blocks), block = (bx, by)).
__global__ void __launch_bounds__(256) bn_affine_rows_kernel(const __nv_bfloat16* x, const float* ca, const float* cb,
                                                             const __nv_bfloat16* residual, __nv_bfloat16* y, int M,
                                                             int C, int rows_per_block, int relu) {
  const int c8n = C / 8;
  const int c8 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c8 >= c8n) return;
  float a[8], b[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { a[t] = ca[c8 * 8 + t]; b[t] = cb[c8 * 8 + t]; }
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, M);
  const uint4* xp = reinterpret_cast<const uint4*>(x);
  const uint4* rp = reinterpret_cast<const uint4*>(residual);
  uint4* yp = reinterpret_cast<uint4*>(y);
#pragma unroll 4
  for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
    const size_t idx = (size_t)r * c8n + c8;
    uint4 u = xp[idx];
    uint4 ru = make_uint4(0, 0, 0, 0);
    if (residual) ru = rp[idx];
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
    const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&ru);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float2 f = __bfloat1622float2(h[t]);
      f.x = fmaf(f.x, a[2 * t], b[2 * t]);
      f.y = fmaf(f.y, a[2 * t + 1], b[2 * t + 1]);
      if (residual) {
        const float2 rr = __bfloat1622float2(rh[t]);
        f.x += rr.x; f.y += rr.y;
      }
      if (relu) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); }
      h[t] = __floats2bfloat162_rn(f.x, f.y);
    }
    yp[idx] = u;
  }
}

// y = relu?( x*scale[c] + shift[c] (+ residual) ), 8 channels per thread
__global__ void __launch_bounds__(256) bn_apply_kernel(const __nv_bfloat16* x, const float* scale, const float* shift,
                                                       const __nv_bfloat16* residual, __nv_bfloat16* y, size_t total8,
                                                       int C, int relu) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += stride) {
    const int c0 = (int)((i * 8) % C);
    uint4 u = reinterpret_cast<const uint4*>(x)[i];
    uint4 ru = make_uint4(0, 0, 0, 0);
    if (residual) ru = reinterpret_cast<const uint4*>(residual)[i];
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
    const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&ru);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float2 f = __bfloat1622float2(h[t]);
      f.x = fmaf(f.x, scale[c0 + 2 * t], shift[c0 + 2 * t]);
      f.y = fmaf(f.y, scale[c0 + 2 * t + 1], shift[c0 + 2 * t + 1]);
      if (residual) {
        const float2 r = __bfloat1622float2(rh[t]);
        f.x += r.x; f.y += r.y;
      }
      if (relu) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); }
      h[t] = __floats2bfloat162_rn(f.x, f.y);
    }
    reinterpret_cast<uint4*>(y)[i] = u;
  }
}

// backward reduce: dy_eff = dy * (y > 0 if relu); per-block partials of sum dy_eff * xhat and sum dy_eff go to
// part[gridDim.y][2][C]; also writes dy_eff (masked) to dres when requested so the residual branch gets its gradient.
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const __nv_bfloat16* dy, const __nv_bfloat16* y,
                                                            const __nv_bfloat16* x, const float* mean,
                                                            const float* rstd, float* part, __nv_bfloat16* dres,
                                                            int M, int C, int rows_per_block, int relu) {
  __shared__ float sh[16 * 256];
  const int c8n = C / 8;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c8 = blockIdx.x * blockDim.x + tx;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, M);
  float g[8], b[8], mu[8], rs[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { g[t] = 0.f; b[t] = 0.f; mu[t] = 0.f; rs[t] = 0.f; }
  if (c8 < c8n) {
#pragma unroll
    for (int t = 0; t < 8; ++t) { mu[t] = mean[c8 * 8 + t]; rs[t] = rstd[c8 * 8 + t]; }
    const uint4* dyp = reinterpret_cast<const uint4*>(dy);
    const uint4* yp = reinterpret_cast<const uint4*>(y);
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    uint4* dr = reinterpret_cast<uint4*>(dres);
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += blockDim.y) {
      const size_t idx = (size_t)r * c8n + c8;
      uint4 du = dyp[idx];
      const uint4 xu = xp[idx];
      __nv_bfloat162* dh = reinterpret_cast<__nv_bfloat162*>(&du);
      const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xu);
      if (relu) {
        const uint4 yu = yp[idx];
        const __nv_bfloat162* yh = reinterpret_cast<const __nv_bfloat162*>(&yu);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float2 d = __bfloat1622float2(dh[t]);
          const float2 o = __bfloat1622float2(yh[t]);
          if (o.x <= 0.f) d.x = 0.f;
          if (o.y <= 0.f) d.y = 0.f;
          dh[t] = __floats2bfloat162_rn(d.x, d.y);
        }
      }
      if (dr) dr[idx] = du;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 d = __bfloat1622float2(dh[t]);
        const float2 xv = __bfloat1622float2(xh[t]);
        g[2 * t] = fmaf(d.x, (xv.x - mu[2 * t]) * rs[2 * t], g[2 * t]);
        g[2 * t + 1] = fmaf(d.y, (xv.y - mu[2 * t + 1]) * rs[2 * t + 1], g[2 * t + 1]);
        b[2 * t] += d.x; b[2 * t + 1] += d.y;
      }
    }
  }
  const int tid = ty * blockDim.x + tx;
  for (int off = blockDim.y >> 1; off > 0; off >>= 1) {
    __syncthreads();
    if (ty >= off && ty < 2 * off) {
#pragma unroll
      for (int t = 0; t < 8; ++t) { sh[(t * 2) * 256 + tid - off * blockDim.x] = g[t]; sh[(t * 2 + 1) * 256 + tid - off * blockDim.x] = b[t]; }
    }
    __syncthreads();
    if (ty < off) {
#pragma unroll
      for (int t = 0; t < 8; ++t) { g[t] += sh[(t * 2) * 256 + tid]; b[t] += sh[(t * 2 + 1) * 256 + tid]; }
    }
  }
  if (ty == 0 && c8 < c8n) {
    float* pg = part + (size_t)blockIdx.y * 2 * C + c8 * 8;
    float* pb = pg + C;
    reinterpret_cast<float4*>(pg)[0] = make_float4(g[0], g[1], g[2], g[3]);
    reinterpret_cast<float4*>(pg)[1] = make_float4(g[4], g[5], g[6], g[7]);
    reinterpret_cast<float4*>(pb)[0] = make_float4(b[0], b[1], b[2], b[3]);
    reinterpret_cast<float4*>(pb)[1] = make_float4(b[4], b[5], b[6], b[7]);
  }
}

// dgamma / dbeta totals and the coefficients of  dx = ca*dy_eff + cb*x + cc  (cc folded below):
//   ca = gamma*rstd, cb = -ca*rstd*dgamma/M, cc = -ca*dbeta/M - cb*mean
__global__ void __launch_bounds__(32 * FOLD_LANES) bn_fold_partials_kernel(const float* part, int nparts, const float* gamma,
                                                               const float* mean, const float* rstd, float* dgamma,
                                                               float* dbeta, float* coef /* [3][C] */, int M, int C,
                                                               int accumulate) {
  __shared__ float sh[2][FOLD_LANES][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float g, b;
  fold_partials(part, nparts, C, c, g, b, sh);
  if (threadIdx.y != 0 || c >= C) return;
  // accumulate: dgamma / dbeta point into the (zeroed) flat gradient arena of the optimizer
  if (dgamma) dgamma[c] = accumulate ? dgamma[c] + g : g;
  if (dbeta) dbeta[c] = accumulate ? dbeta[c] + b : b;
  const float ga = gamma ? gamma[c] : 1.f;
  const float ca = ga * rstd[c];
  const float cb = -ca * rstd[c] * g / M;
  coef[c] = ca;
  coef[C + c] = cb;
  coef[2 * C + c] = -ca * b / M - cb * mean[c];
}

// dx = ca*dy_eff + cb*x + cc ; dy_eff = dy masked by (y > 0) when relu (row-strided like bn_affine_rows_kernel)
__global__ void __launch_bounds__(256) bn_bwd_rows_kernel(const __nv_bfloat16* dy, const __nv_bfloat16* y,
                                                          const __nv_bfloat16* x, const float* coef,
                                                          __nv_bfloat16* dx, int M, int C, int rows_per_block,
                                                          int relu) {
  const int c8n = C / 8;
  const int c8 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c8 >= c8n) return;
  float ca[8], cb[8], cc[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { ca[t] = coef[c8 * 8 + t]; cb[t] = coef[C + c8 * 8 + t]; cc[t] = coef[2 * C + c8 * 8 + t]; }
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(r0 + rows_per_block, M);
  const uint4* dyp = reinterpret_cast<const uint4*>(dy);
  const uint4* yp = reinterpret_cast<const uint4*>(y);
  const uint4* xp = reinterpret_cast<const uint4*>(x);
  uint4* dxp = reinterpret_cast<uint4*>(dx);
#pragma unroll 4
  for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
    const size_t idx = (size_t)r * c8n + c8;
    uint4 du = dyp[idx];
    const uint4 xu = xp[idx];
    uint4 yu = make_uint4(0, 0, 0, 0);
    if (relu) yu = yp[idx];
    __nv_bfloat162* dh = reinterpret_cast<__nv_bfloat162*>(&du);
    const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xu);
    const __nv_bfloat162* yh = reinterpret_cast<const __nv_bfloat162*>(&yu);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float2 d = __bfloat1622float2(dh[t]);
      const float2 xv = __bfloat1622float2(xh[t]);
      if (relu) {
        const float2 o = __bfloat1622float2(yh[t]);
        if (o.x <= 0.f) d.x = 0.f;
        if (o.y <= 0.f) d.y = 0.f;
      }
      d.x = fmaf(ca[2 * t], d.x, fmaf(cb[2 * t], xv.x, cc[2 * t]));
      d.y = fmaf(ca[2 * t + 1], d.y, fmaf(cb[2 * t + 1], xv.y, cc[2 * t + 1]));
      dh[t] = __floats2bfloat162_rn(d.x, d.y);
    }
    dxp[idx] = du;
  }
}

// global average pool over HW rows: x [N, HW, C] bf16 -> out [N, C] fp32 (+ optional bf16)
__global__ void __launch_bounds__(256) gap_fwd_kernel(const __nv_bfloat16* x, float* out, __nv_bfloat16* out_bf16,
                                                      int HW, int C) {
  const int n = blockIdx.y;
  const int c2 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c2 * 2 >= C) return;
  const __nv_bfloat162* xp = reinterpret_cast<const __nv_bfloat162*>(x) + (size_t)n * HW * (C / 2);
  float s0 = 0.f, s1 = 0.f;
  for (int r = 0; r < HW; ++r) {
    const float2 f = __bfloat1622float2(xp[(size_t)r * (C / 2) + c2]);
    s0 += f.x; s1 += f.y;
  }
  s0 /= HW; s1 /= HW;
  if (out) { out[(size_t)n * C + 2 * c2] = s0; out[(size_t)n * C + 2 * c2 + 1] = s1; }
  if (out_bf16) reinterpret_cast<__nv_bfloat162*>(out_bf16)[(size_t)n * (C / 2) + c2] = __floats2bfloat162_rn(s0, s1);
}
// dx[n, r, c] = dout[n, c] / HW
__global__ void __launch_bounds__(256) gap_bwd_kernel(const float* dout, __nv_bfloat16* dx, int HW, int C) {
  const int n = blockIdx.y;
  const int c2 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c2 * 2 >= C) return;
  const float a = dout[(size_t)n * C + 2 * c2] / HW, b = dout[(size_t)n * C + 2 * c2 + 1] / HW;
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  __nv_bfloat162* dp = reinterpret_cast<__nv_bfloat162*>(dx) + (size_t)n * HW * (C / 2);
  for (int r = 0; r < HW; ++r) dp[(size_t)r * (C / 2) + c2] = v;
}

// ----------------------------------------------------------------------------- CMC / AP without sorting
// One block per query. S: [Q, G] similarity (higher = closer). An item g' precedes g iff
// S[g'] > S[g] or (S[g'] == S[g] and g' > g)   (== np.argsort(sim)[::-1] with a stable sort).
// out_ap[q] = AP (trapezoid form, tools/evaluate.py:75-82), out_first[q] = rank of first hit (or -1: no match).
__global__ void __launch_bounds__(256) rank_eval_kernel(const float* S, const long long* qlab, const long long* glab,
                                                        float* out_ap, int* out_first, int G, long long lds) {
  extern __shared__ int s_match[];  // indices of matching gallery items (capacity = blockDim-independent, G max)
  __shared__ int s_nmatch;
  __shared__ float shf[8];
  __shared__ float s_ap;
  __shared__ int s_first;
  const int q = blockIdx.x;
  const float* row = S + (long long)q * lds;
  const long long ql = qlab[q];
  if (threadIdx.x == 0) { s_nmatch = 0; s_ap = 0.f; s_first = 0x7fffffff; }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x)
    if (glab[g] == ql) s_match[atomicAdd(&s_nmatch, 1)] = g;
  __syncthreads();
  const int R = s_nmatch;
  if (R == 0) {
    if (threadIdx.x == 0) { out_ap[q] = 0.f; out_first[q] = -1; }
    return;
  }
  for (int mi = 0; mi < R; ++mi) {
    const int gm = s_match[mi];
    const float sm = row[gm];
    float higher = 0.f, higher_match = 0.f;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
      const float s = row[g];
      const bool before = (s > sm) || (s == sm && g > gm);
      if (before) {
        higher += 1.f;
        if (glab[g] == ql) higher_match += 1.f;
      }
    }
    const float loc = block_sum(higher, shf);
    __syncthreads();
    const float im = block_sum(higher_match, shf);
    if (threadIdx.x == 0) {
      const float precision = (im + 1.f) / (loc + 1.f);
      const float old_precision = (loc != 0.f) ? im / loc : 1.f;
      s_ap += (old_precision + precision) * 0.5f / R;
      s_first = min(s_first, (int)loc);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out_ap[q] = s_ap; out_first[q] = s_first; }
}


// ----------------------------------------------------------------------------- input pipeline: fused augmentation
// uint8 NHWC crops -> normalise -> horizontal flip -> random erasing (value 0) -> bf16 / fp32 NHWC, one pass.
// Reference: datasets/image_augmentation.py:6-71 (ToTensor, Normalize, RandomHorizontalFlip, RandomErasing).
// u: [7][B] uniforms in [0,1) (flip, erase-select, area, log-ratio, top, left, spare); the per-sample rectangle is
// derived here exactly as torchvision does (area in `scale`, aspect log-uniform in `ratio`, one attempt).
struct AugArgs {
  const uint8_t* in;
  void* out;
  const float* u;
  int B, H, W;
  float mean[3], inv_std[3];
  float flip_p, erase_p, s0, s1, lr0, lr1;
  int out_bf16;
};

__global__ void __launch_bounds__(256) augment_u8_kernel(const AugArgs a) {
  const int b = blockIdx.y;
  const int quads_per_img = a.H * (a.W / 4);
  __shared__ int s_flip, s_sel, s_top, s_left, s_eh, s_ew;
  if (threadIdx.x == 0) {
    const float* u = a.u + b;
    const int B = a.B;
    s_flip = u[0] < a.flip_p;
    s_sel = u[1 * B] < a.erase_p;
    const float area = (u[2 * B] * (a.s1 - a.s0) + a.s0) * a.H * a.W;
    const float ar = __expf(u[3 * B] * (a.lr1 - a.lr0) + a.lr0);
    const float eh = fminf(fmaxf(rintf(sqrtf(area * ar)), 1.f), (float)(a.H - 1));
    const float ew = fminf(fmaxf(rintf(sqrtf(area / ar)), 1.f), (float)(a.W - 1));
    s_eh = (int)eh;
    s_ew = (int)ew;
    s_top = (int)floorf(u[4 * B] * (a.H - eh + 1.f));
    s_left = (int)floorf(u[5 * B] * (a.W - ew + 1.f));
  }
  __syncthreads();
  const int flip = s_flip, sel = s_sel, top = s_top, left = s_left, eh = s_eh, ew = s_ew;
  const uint8_t* src = a.in + (size_t)b * a.H * a.W * 3;
  for (int qd = blockIdx.x * blockDim.x + threadIdx.x; qd < quads_per_img; qd += gridDim.x * blockDim.x) {
    const int y = qd / (a.W / 4);
    const int x0 = (qd - y * (a.W / 4)) * 4;
    const int sx0 = flip ? (a.W - 4 - x0) : x0;                     // 4 source pixels (12 B, 4-byte aligned)
    const uint32_t* sp = reinterpret_cast<const uint32_t*>(src + ((size_t)y * a.W + sx0) * 3);
    const uint32_t w0 = sp[0], w1 = sp[1], w2 = sp[2];
    uint8_t px[12];
    *reinterpret_cast<uint32_t*>(px) = w0;
    *reinterpret_cast<uint32_t*>(px + 4) = w1;
    *reinterpret_cast<uint32_t*>(px + 8) = w2;
    float v[12];
    const bool yin = sel && y >= top && y < top + eh;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int si = flip ? (3 - i) : i;
      const int x = x0 + i;
      const bool erase = yin && x >= left && x < left + ew;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[i * 3 + c] = erase ? 0.f : ((float)px[si * 3 + c] - a.mean[c]) * a.inv_std[c];
    }
    const size_t o = ((size_t)b * a.H * a.W + (size_t)y * a.W + x0) * 3;
    if (a.out_bf16) {
      __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(a.out) + o);
#pragma unroll
      for (int i = 0; i < 6; ++i) op[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    } else {
      float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(a.out) + o);
#pragma unroll
      for (int i = 0; i < 3; ++i) op[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
  }
}

// ----------------------------------------------------------------------------- herding (iCaRL exemplar selection)
// One block per identity. feats [n_total, D] fp32, rows of identity g are idx[g*nmax .. g*nmax+cnt[g]).
// Step t picks argmin_i || mean - (S + f_i)/(t+1) ||  <=>  argmin_i ( |f_i|^2 - 2 f_i . c ),  c = (t+1) mean - S
// (duplicates allowed, first index wins ties) - methods/fedstil.py:378-395, methods/icarl.py:122-139.
// The whole m-step loop runs inside the kernel: no per-step launches, no host round trips.
__global__ void __launch_bounds__(256) herding_kernel(const float* feats, const long long* idx, const int* cnt,
                                                      long long* picks, int nmax, int D, int m) {
  extern __shared__ float sh[];          // mean[D] | S[D] | c[D] | score[nmax] | sq[nmax]
  float* mean = sh;
  float* S = sh + D;
  float* c = sh + 2 * D;
  float* score = sh + 3 * D;
  float* sq = score + nmax;
  __shared__ int s_best;
  const int g = blockIdx.x;
  const int n = cnt[g];
  const long long* rows = idx + (size_t)g * nmax;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  for (int d = tid; d < D; d += blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < n; ++i) s += feats[(size_t)rows[i] * D + d];
    mean[d] = n > 0 ? s / n : 0.f;
    S[d] = 0.f;
  }
  for (int i = warp; i < n; i += nwarps) {
    const float* f = feats + (size_t)rows[i] * D;
    float s = 0.f;
    for (int d = lane; d < D; d += 32) s = fmaf(f[d], f[d], s);
    s = warp_sum(s);
    if (lane == 0) sq[i] = s;
  }
  __syncthreads();
  for (int t = 0; t < m; ++t) {
    for (int d = tid; d < D; d += blockDim.x) c[d] = (t + 1) * mean[d] - S[d];
    __syncthreads();
    for (int i = warp; i < n; i += nwarps) {
      const float* f = feats + (size_t)rows[i] * D;
      float s = 0.f;
      for (int d = lane; d < D; d += 32) s = fmaf(f[d], c[d], s);
      s = warp_sum(s);
      if (lane == 0) score[i] = sq[i] - 2.f * s;
    }
    __syncthreads();
    if (tid == 0) {
      int best = 0;
      float bv = n > 0 ? score[0] : 0.f;
      for (int i = 1; i < n; ++i)
        if (score[i] < bv) { bv = score[i]; best = i; }
      s_best = best;
      picks[(size_t)g * m + t] = best;
    }
    __syncthreads();
    if (n > 0) {
      const float* f = feats + (size_t)rows[s_best] * D;
      for (int d = tid; d < D; d += blockDim.x) S[d] += f[d];
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------- frozen-trunk stem helpers
// Space-to-depth + zero padding of the stem input: x [B,H,W,3] bf16 (NHWC) -> y [B, H/2+3, W/2+3, 16] bf16 where
// cell (i, j) holds the 2x2 pixel block ((i-2)*2 + bh, (j-2)*2 + bw), channel index (bh*2 + bw)*3 + c, channels
// 12..15 and the border cells are zero. A 7x7 / stride-2 / pad-3 convolution on x is then a 4x4 / stride-1
// convolution on y whose 4-cell windows are CONTIGUOUS 128-byte runs: the implicit-GEMM kernel loads them with one
// TMA box per kernel row (tensor map with a 32-byte cell stride, i.e. overlapping 128-byte rows).
__global__ void __launch_bounds__(256) s2d_pad_kernel(const __nv_bfloat16* x, __nv_bfloat16* y, int B, int H, int W) {
  const int H2 = H / 2 + 3, W2 = W / 2 + 3;
  const size_t cells = (size_t)B * H2 * W2;
  for (size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x; cell < cells;
       cell += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(cell % W2);
    const int i = (int)((cell / W2) % H2);
    const int b = (int)(cell / ((size_t)W2 * H2));
    __align__(16) __nv_bfloat16 v[16];
#pragma unroll
    for (int t = 0; t < 16; ++t) v[t] = __float2bfloat16(0.f);
    const int ci = i - 2, cj = j - 2;
    if (ci >= 0 && ci < H / 2 && cj >= 0 && cj < W / 2) {
#pragma unroll
      for (int bh = 0; bh < 2; ++bh)
#pragma unroll
        for (int bw = 0; bw < 2; ++bw) {
          const __nv_bfloat16* src = x + (((size_t)b * H + (ci * 2 + bh)) * W + (cj * 2 + bw)) * 3;
#pragma unroll
          for (int c = 0; c < 3; ++c) v[(bh * 2 + bw) * 3 + c] = src[c];
        }
    }
    uint4* dst = reinterpret_cast<uint4*>(y + cell * 16);
    dst[0] = reinterpret_cast<const uint4*>(v)[0];
    dst[1] = reinterpret_cast<const uint4*>(v)[1];
  }
}

// 3x3 / stride 2 / pad 1 max-pool over NHWC bf16, 8 channels (16 bytes) per thread.
__global__ void __launch_bounds__(256) maxpool3x3s2_nhwc_kernel(const __nv_bfloat16* x, __nv_bfloat16* y, int B,
                                                                int H, int W, int C) {
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1, c8n = C / 8;
  const size_t total = (size_t)B * Ho * Wo * c8n;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % c8n);
    const int ow = (int)((t / c8n) % Wo);
    const int oh = (int)((t / ((size_t)c8n * Wo)) % Ho);
    const int b = (int)(t / ((size_t)c8n * Wo * Ho));
    float m[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) m[k] = -3.0e38f;
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int ih = oh * 2 - 1 + dh;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int iw = ow * 2 - 1 + dw;
        if (iw < 0 || iw >= W) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(x + (((size_t)b * H + ih) * W + iw) * C + c8 * 8);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(h[k]);
          m[2 * k] = fmaxf(m[2 * k], f.x);
          m[2 * k + 1] = fmaxf(m[2 * k + 1], f.y);
        }
      }
    }
    uint4 o;
    __nv_bfloat162* oh2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) oh2[k] = __floats2bfloat162_rn(m[2 * k], m[2 * k + 1]);
    *reinterpret_cast<uint4*>(y + (((size_t)b * Ho + oh) * Wo + ow) * C + c8 * 8) = o;
  }
}

// ----------------------------------------------------------------------------- Swin window attention (fused)
// One block per (window, head): S = scale * Q K^T + bias (relative-position bias [+ shift mask]) -> softmax -> P V,
// everything in shared memory / registers (N <= 64 tokens per window, head dim D <= 64; Swin: N = 49, D = 32).
// Reference: models/swin_transformer.py:255-286 (QK^T, bias table gather, mask add, softmax, attn @ v as five
// separate library calls materialising the [B*nW, heads, N, N] score tensor twice).
// qkv: [BW, N, 3, H, D] (the qkv projection's output), bias: [nWb, H, N, N] fp32 (nWb = 1 or #windows per image;
// window index = bw % nWb), out: [BW, N, H*D].
template <typename T>
__device__ __forceinline__ float attn_ld(const T* p) { return static_cast<float>(*p); }
template <>
__device__ __forceinline__ float attn_ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T>
__device__ __forceinline__ void attn_st(T* p, float v) { *p = static_cast<T>(v); }
template <>
__device__ __forceinline__ void attn_st<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

constexpr int ATT_MAXN = 64;
constexpr int ATT_MAXD = 64;

template <typename T>
__global__ void __launch_bounds__(64) window_attn_fwd_kernel(const T* qkv, const float* bias, T* out, int N, int H,
                                                             int D, int nWb, float scale) {
  extern __shared__ float sm[];                 // K[N][D+1] | V[N][D+1] | S[N][N+1]
  const int bw = blockIdx.x, h = blockIdx.y, i = threadIdx.x;
  const int ld = D + 1;
  float* Ks = sm;
  float* Vs = sm + N * ld;
  float* s = Vs + N * ld + (size_t)i * (N + 1);  // this thread's score row
  const size_t row_stride = (size_t)3 * H * D;
  const T* base = qkv + (size_t)bw * N * row_stride + (size_t)h * D;
  for (int t = threadIdx.x; t < N * D; t += blockDim.x) {
    const int j = t / D, d = t - j * D;
    Ks[j * ld + d] = attn_ld(base + j * row_stride + (size_t)H * D + d);
    Vs[j * ld + d] = attn_ld(base + j * row_stride + (size_t)2 * H * D + d);
  }
  __syncthreads();
  if (i >= N) return;
  float q[ATT_MAXD];
#pragma unroll
  for (int d = 0; d < ATT_MAXD; ++d) q[d] = d < D ? attn_ld(base + i * row_stride + d) * scale : 0.f;
  const float* brow = bias + (((size_t)(bw % nWb) * H + h) * N + i) * N;
  float mx = -3.0e38f;
#pragma unroll 1
  for (int j = 0; j < N; ++j) {
    float a = brow[j];
#pragma unroll
    for (int d = 0; d < ATT_MAXD; ++d)
      if (d < D) a = fmaf(q[d], Ks[j * ld + d], a);
    s[j] = a;
    mx = fmaxf(mx, a);
  }
  float sum = 0.f;
#pragma unroll 1
  for (int j = 0; j < N; ++j) {
    s[j] = __expf(s[j] - mx);
    sum += s[j];
  }
  const float inv = 1.f / sum;
  float o[ATT_MAXD];
#pragma unroll
  for (int d = 0; d < ATT_MAXD; ++d) o[d] = 0.f;
#pragma unroll 1
  for (int j = 0; j < N; ++j) {
    const float pj = s[j] * inv;
#pragma unroll
    for (int d = 0; d < ATT_MAXD; ++d)
      if (d < D) o[d] = fmaf(pj, Vs[j * ld + d], o[d]);
  }
  T* orow = out + ((size_t)bw * N + i) * H * D + (size_t)h * D;
#pragma unroll
  for (int d = 0; d < ATT_MAXD; ++d)
    if (d < D) attn_st(orow + d, o[d]);
}

// Backward: recompute P, then dV = P^T dO, dP = dO V^T, dS = P (.) (dP - rowsum(dP (.) P)), dQ = scale dS K,
// dK = scale dS^T Q, dBias += dS (atomic over the images that share a window index).

// ----------------------------------------------------------------------------- Swin window attention on wgmma
// Forward only (the frozen stages never need a gradient; the trainable stage's backward keeps the kernel above).
// A persistent CTA of one warpgroup (128 threads) walks (window, head) pairs. Per pair:
//   * Q [N x 32], K [N x 32] are copied into 128B-swizzled K-major operand tiles (rows = tokens padded to 64, the
//     K extent padded 32 -> 64 with zeros written once), V is TRANSPOSED on the way in (Vt [32 x N], K extent = keys);
//   * S = Q K^T: two wgmma m64n64k16 into 32 fp32 registers per thread;
//   * softmax on the accumulator fragment: each row lives in the 4 lanes of a quad (two rows per thread), so max / sum
//     take two shuffles; + relative-position bias (+ shift mask), exp2 with the scale folded in; P (bf16,
//     un-normalised) is written back as the next A operand, 1 / sum stays in a register;
//   * O = P V: four wgmma m64n32k16; the epilogue scales by 1 / sum and stores bf16 pairs.
// Swin: N = 49 (or 16), D = 32 for every model size. Reference: models/swin_transformer.py:255-286.
constexpr int WA_THREADS = 128;
constexpr int WA_SQ = 0;                       // 64 rows x 128 B
constexpr int WA_SK = 64 * 128;                // 64 rows x 128 B
constexpr int WA_SVT = WA_SK + 64 * 128;       // 32 rows x 128 B
constexpr int WA_SP = WA_SVT + 32 * 128;       // 64 rows x 128 B   (WA_SVT is 4 KB: WA_SP stays 1024-aligned)
constexpr int WA_END = WA_SP + 64 * 128;
constexpr int WA_SMEM = WA_END + 1024;

// byte offset of 16-byte chunk `c` (0..7) of row `r` in a K-major SWIZZLE_128B tile (8-row x 128 B atoms)
__device__ __forceinline__ uint32_t wa_swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

__global__ void __launch_bounds__(WA_THREADS, 4)
window_attn_fwd_tc_kernel(const __nv_bfloat16* qkv, const float* bias, __nv_bfloat16* out, int N, int H, int nWb,
                          float scale, int total_pairs) {
  extern __shared__ uint8_t wa_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wa_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int D = 32;

  for (int i = tid; i < WA_END / 16; i += WA_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const uint32_t sQ = smem_u32(smem + WA_SQ), sK = smem_u32(smem + WA_SK), sVt = smem_u32(smem + WA_SVT),
                 sP = smem_u32(smem + WA_SP);
  const size_t row_stride = (size_t)3 * H * D;
  const float sl2 = scale * 1.4426950408889634f;            // exp(x) = exp2(x * log2 e)
  // accumulator fragment of this thread: rows r0 and r0 + 8, columns 8j + c0 + {0, 1}
  const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);

  for (int p = blockIdx.x; p < total_pairs; p += gridDim.x) {
    const int bw = p / H, h = p - bw * H;
    const __nv_bfloat16* base = qkv + (size_t)bw * N * row_stride + (size_t)h * D;
    // ---- operands: Q, K row-wise (4 chunks of 16 B per token), V transposed
    for (int t = tid; t < N * 4; t += WA_THREADS) {
      const int r = t >> 2, c = t & 3;
      const __nv_bfloat16* src = base + (size_t)r * row_stride + c * 8;
      const uint4 q = *reinterpret_cast<const uint4*>(src);
      const uint4 k = *reinterpret_cast<const uint4*>(src + (size_t)H * D);
      const uint4 v = *reinterpret_cast<const uint4*>(src + (size_t)2 * H * D);
      sts_128(sQ + wa_swz(r, c), q);
      sts_128(sK + wa_swz(r, c), k);
      const __nv_bfloat16* ve = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int d = c * 8 + e;                             // Vt[d][r]
        *reinterpret_cast<__nv_bfloat16*>(smem + WA_SVT + wa_swz(d, r >> 3) + (r & 7) * 2) = ve[e];
      }
    }
    fence_proxy_async();                                     // generic-proxy smem writes -> visible to wgmma
    __syncthreads();
    float s[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k)                              // D = 32 -> two K = 16 steps (the padded half is unused)
      wgmma_m64n64k16<0, 0>(s, make_smem_desc_sw128(sQ + k * 32, 16, 1024),
                            make_smem_desc_sw128(sK + k * 32, 16, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 32; ++j) reg_fence(s[j]);
    // ---- softmax on the fragment: half 0 = row r0, half 1 = row r0 + 8
    float inv[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = r0 + hf * 8;
      const float* brow = bias + (((size_t)(bw % nWb) * H + h) * N + (r < N ? r : 0)) * N;
      float mx = -3.0e38f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * j + c0 + e;
          const float x = (col < N && r < N) ? fmaf(s[4 * j + 2 * hf + e], sl2, brow[col] * 1.4426950408889634f)
                                             : -3.0e38f;
          s[4 * j + 2 * hf + e] = x;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * j + c0 + e;
          const float ex = (col < N && r < N) ? exp2f(s[4 * j + 2 * hf + e] - mx) : 0.f;
          s[4 * j + 2 * hf + e] = ex;
          sum += ex;
        }
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      inv[hf] = r < N ? 1.f / sum : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __nv_bfloat162 pk = __floats2bfloat162_rn(s[4 * j + 2 * hf], s[4 * j + 2 * hf + 1]);
        // column 8j + c0 of row r: 16-byte chunk j, byte 2 * c0 inside it
        *reinterpret_cast<__nv_bfloat162*>(smem + WA_SP + wa_swz(r, j) + c0 * 2) = pk;
      }
    }
    fence_proxy_async();
    __syncthreads();
    float o[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)                              // K = 64 keys -> four K = 16 steps
      wgmma_m64n32k16<0, 0>(o, make_smem_desc_sw128(sP + k * 32, 16, 1024),
                            make_smem_desc_sw128(sVt + k * 32, 16, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 16; ++j) reg_fence(o[j]);
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = r0 + hf * 8;
      if (r < N) {
        __nv_bfloat16* dst = out + ((size_t)bw * N + r) * H * D + (size_t)h * D + c0;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<__nv_bfloat162*>(dst + 8 * j) =
              __floats2bfloat162_rn(o[4 * j + 2 * hf] * inv[hf], o[4 * j + 2 * hf + 1] * inv[hf]);
      }
    }
    __syncthreads();                                         // operands free for the next pair
  }
}

template <typename T>
__global__ void __launch_bounds__(64) window_attn_bwd_kernel(const T* qkv, const float* bias, const T* dout, T* dqkv,
                                                             float* dbias, int N, int H, int D, int nWb,
                                                             float scale) {
  extern __shared__ float sm[];                 // Q | K | V | dO : [N][D+1] each ; P | dS : [N][N+1] each
  const int bw = blockIdx.x, h = blockIdx.y, i = threadIdx.x;
  const int ld = D + 1, ln = N + 1;
  float* Qs = sm;
  float* Ks = Qs + N * ld;
  float* Vs = Ks + N * ld;
  float* Os = Vs + N * ld;
  float* Ps = Os + N * ld;
  float* Ss = Ps + N * ln;
  const size_t row_stride = (size_t)3 * H * D;
  const T* base = qkv + (size_t)bw * N * row_stride + (size_t)h * D;
  const T* dob = dout + (size_t)bw * N * H * D + (size_t)h * D;
  for (int t = threadIdx.x; t < N * D; t += blockDim.x) {
    const int j = t / D, d = t - j * D;
    Qs[j * ld + d] = attn_ld(base + j * row_stride + d);
    Ks[j * ld + d] = attn_ld(base + j * row_stride + (size_t)H * D + d);
    Vs[j * ld + d] = attn_ld(base + j * row_stride + (size_t)2 * H * D + d);
    Os[j * ld + d] = attn_ld(dob + (size_t)j * H * D + d);
  }
  __syncthreads();
  if (i < N) {
    const float* brow = bias + (((size_t)(bw % nWb) * H + h) * N + i) * N;
    float mx = -3.0e38f;
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
      float a = brow[j];
      for (int d = 0; d < D; ++d) a = fmaf(Qs[i * ld + d] * scale, Ks[j * ld + d], a);
      Ps[i * ln + j] = a;
      mx = fmaxf(mx, a);
    }
    float sum = 0.f;
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
      const float e = __expf(Ps[i * ln + j] - mx);
      Ps[i * ln + j] = e;
      sum += e;
    }
    const float inv = 1.f / sum;
    float delta = 0.f;
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
      const float pj = Ps[i * ln + j] * inv;
      float dp = 0.f;
      for (int d = 0; d < D; ++d) dp = fmaf(Os[i * ld + d], Vs[j * ld + d], dp);
      Ps[i * ln + j] = pj;
      Ss[i * ln + j] = dp;
      delta = fmaf(pj, dp, delta);
    }
    float* dbrow = dbias ? dbias + (((size_t)(bw % nWb) * H + h) * N + i) * N : nullptr;
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
      const float ds = Ps[i * ln + j] * (Ss[i * ln + j] - delta);
      Ss[i * ln + j] = ds;
      if (dbrow) atomicAdd(dbrow + j, ds);
    }
    // dQ_i = scale * sum_j dS_ij K_j
    T* dq = dqkv + ((size_t)bw * N + i) * row_stride + (size_t)h * D;
    for (int d = 0; d < D; ++d) {
      float a = 0.f;
      for (int j = 0; j < N; ++j) a = fmaf(Ss[i * ln + j], Ks[j * ld + d], a);
      attn_st(dq + d, a * scale);
    }
  }
  __syncthreads();
  if (i < N) {
    // column pass (thread = key index j): dK_j = scale * sum_i dS_ij Q_i ; dV_j = sum_i P_ij dO_i
    const int j = i;
    T* dk = dqkv + ((size_t)bw * N + j) * row_stride + (size_t)H * D + (size_t)h * D;
    T* dv = dk + (size_t)H * D;
    for (int d = 0; d < D; ++d) {
      float a = 0.f, b = 0.f;
      for (int r = 0; r < N; ++r) {
        a = fmaf(Ss[r * ln + j], Qs[r * ld + d], a);
        b = fmaf(Ps[r * ln + j], Os[r * ld + d], b);
      }
      attn_st(dk + d, a * scale);
      attn_st(dv + d, b);
    }
  }
}

static inline int grid_for(size_t n_items, int threads, int cap = 132 * 8) {
  size_t b = (n_items + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > (size_t)cap) b = cap;
  return (int)b;
}

}  // namespace flpr

using namespace flpr;

extern "C" {

// stats_part (required with stats): 2 x 1056 floats of scratch (2 per block, at most 132 * 8 blocks).
// omega (nullable): Synaptic Intelligence path integral, accumulated by the SI instantiation of the kernel.
int flpr_fused_opt(int adam, float* p, const float* g, float* m, float* v, const float* Q, const float* R,
                   const float* G, void* p_bf16, float* stats, size_t n, float lr, float beta1, float beta2, float eps,
                   float wd, int step, float lam2, float lam1, float atten, float momentum, int penalty_ones,
                   const float* hyper, float* anchor, float* anchor_m, float* anchor_v, float* stats_part,
                   float* omega, cudaStream_t st) {
  bind_device_of(p);
  if (n % 4) return -2;
  OptArgs a;
  a.p = p; a.g = g; a.m = m; a.v = v; a.Q = Q; a.R = R; a.G = G;
  a.p_bf16 = reinterpret_cast<__nv_bfloat16*>(p_bf16); a.stats = stats; a.stats_part = stats_part; a.n = n;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  a.bc1 = 1.f - powf(beta1, (float)step);
  a.bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  a.lam2 = lam2; a.lam1 = lam1; a.atten = atten; a.momentum = momentum; a.penalty_ones = penalty_ones;
  a.hyper = hyper;
  a.omega = omega;
  a.anchor = G != nullptr ? anchor : nullptr; a.am = anchor_m; a.av = anchor_v;
  if (a.anchor != nullptr && ((adam && (anchor_m == nullptr || anchor_v == nullptr)) ||
                              (!adam && momentum != 0.f && anchor_m == nullptr)))
    return -3;
  if (stats != nullptr && stats_part == nullptr) return -4;
  const int grid = grid_for(n / 4, 256);
  if (omega != nullptr) {
    if (adam) fused_opt_kernel<true, true><<<grid, 256, 0, st>>>(a);
    else fused_opt_kernel<false, true><<<grid, 256, 0, st>>>(a);
  } else {
    if (adam) fused_opt_kernel<true, false><<<grid, 256, 0, st>>>(a);
    else fused_opt_kernel<false, false><<<grid, 256, 0, st>>>(a);
  }
  if (stats != nullptr) opt_stats_kernel<<<1, 32, 0, st>>>(stats_part, stats, grid, R != nullptr, G != nullptr);
  return (int)cudaGetLastError();
}

int flpr_importance_accum(float* F, const float* g, size_t n, float scale, int mode, cudaStream_t st) {
  bind_device_of(F);
  if (n % 4) return -2;
  importance_accum_kernel<<<grid_for(n / 4, 256), 256, 0, st>>>(F, g, n, scale, mode);
  return (int)cudaGetLastError();
}

int flpr_cast_bf16(const float* x, void* y, size_t n, cudaStream_t st) {
  bind_device_of(x);
  if (n % 4) return -2;
  cast_bf16_kernel<<<grid_for(n / 4, 256), 256, 0, st>>>(x, reinterpret_cast<__nv_bfloat16*>(y), n);
  return (int)cudaGetLastError();
}

int flpr_compose(const float* G, const float* A, float a, float* theta, void* theta_bf16, size_t n, cudaStream_t st) {
  bind_device_of(G);
  if (n % 4) return -2;
  compose_kernel<<<grid_for(n / 4, 256), 256, 0, st>>>(G, A, a, theta, reinterpret_cast<__nv_bfloat16*>(theta_bf16), n);
  return (int)cudaGetLastError();
}

// rule: SOPT_SGD 0, SOPT_ADAGRAD 1, SOPT_ADAM 2, SOPT_YOGI 3 (see server_opt_kernel). x, mean, m are required, v for
// every rule but SOPT_SGD; x_bf16 is nullable. Any length and alignment. -2: unknown rule, -3: a required pointer is null.
int flpr_server_opt(int rule, float* x, const float* mean, float* m, float* v, void* x_bf16, size_t n, float lr,
                    float momentum, float beta1, float beta2, float tau, cudaStream_t st) {
  if (rule < SOPT_SGD || rule > SOPT_YOGI) return -2;
  if (x == nullptr || mean == nullptr || m == nullptr || (rule != SOPT_SGD && v == nullptr)) return -3;
  if (n == 0) return 0;
  bind_device_of(x);
  ServerOptArgs a;
  a.x = x; a.mean = mean; a.m = m; a.v = v; a.x_bf16 = reinterpret_cast<__nv_bfloat16*>(x_bf16); a.n = n;
  a.lr = lr; a.momentum = momentum; a.beta1 = beta1; a.beta2 = beta2; a.tau = tau;
  const auto al = [](const void* p, uintptr_t b) { return (reinterpret_cast<uintptr_t>(p) & (b - 1)) == 0; };
  const int vec = al(x, 16) && al(mean, 16) && al(m, 16) && (rule == SOPT_SGD || al(v, 16)) && al(x_bf16, 8);
  const int grid = grid_for(vec ? (n + 3) / 4 : n, 256);
  switch (rule) {
    case SOPT_SGD: server_opt_kernel<SOPT_SGD><<<grid, 256, 0, st>>>(a, vec); break;
    case SOPT_ADAGRAD: server_opt_kernel<SOPT_ADAGRAD><<<grid, 256, 0, st>>>(a, vec); break;
    case SOPT_ADAM: server_opt_kernel<SOPT_ADAM><<<grid, 256, 0, st>>>(a, vec); break;
    default: server_opt_kernel<SOPT_YOGI><<<grid, 256, 0, st>>>(a, vec); break;
  }
  return (int)cudaGetLastError();
}

// in_bf16 / out_bf16 select the logits / dlogits dtypes. stats: float[2] (loss mean accum, correct count accum);
// row_part: float[2 B] scratch.
int flpr_ce_label_smooth(const void* logits, const long long* target, void* dlogits, float* stats, float* row_part,
                         int B, int C, long long ld, float eps, float grad_scale, int in_bf16, int out_bf16, cudaStream_t st) {
  if (in_bf16 && out_bf16)
    ce_ls_kernel<__nv_bfloat16, __nv_bfloat16><<<B, 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(logits), target, reinterpret_cast<__nv_bfloat16*>(dlogits), row_part, B, C,
        ld, eps, grad_scale);
  else if (in_bf16)
    ce_ls_kernel<__nv_bfloat16, float><<<B, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(logits), target,
                                                           reinterpret_cast<float*>(dlogits), row_part, B, C, ld, eps,
                                                           grad_scale);
  else if (out_bf16)
    ce_ls_kernel<float, __nv_bfloat16><<<B, 256, 0, st>>>(reinterpret_cast<const float*>(logits), target,
                                                           reinterpret_cast<__nv_bfloat16*>(dlogits), row_part, B, C, ld,
                                                           eps, grad_scale);
  else
    ce_ls_kernel<float, float><<<B, 256, 0, st>>>(reinterpret_cast<const float*>(logits), target,
                                                   reinterpret_cast<float*>(dlogits), row_part, B, C, ld, eps, grad_scale);
  ce_stats_kernel<<<1, 32, 0, st>>>(row_part, stats, B);
  return (int)cudaGetLastError();
}

static void bn_launch_geometry(int M, int C, dim3& grid, dim3& block, int& rpb) {
  const int c8n = C / 8;
  const int bx = c8n >= 256 ? 256 : c8n;              // channel groups per block
  int by = 1;                                         // row-lanes per block (power of two, <= 16)
  while (by * 2 * bx <= 256 && by < 16) by *= 2;
  const int gx = (c8n + bx - 1) / bx;
  int gy = (132 * 4) / gx;
  if (gy < 1) gy = 1;
  rpb = (M + gy - 1) / gy;
  if (rpb < by * 4) rpb = by * 4;
  gy = (M + rpb - 1) / rpb;
  grid = dim3(gx, gy);
  block = dim3(bx, by);
}

int flpr_bn_partials_floats(int M, int C) {
  dim3 g, b; int rpb;
  bn_launch_geometry(M, C, g, b, rpb);
  return (int)g.y * 2 * C + 3 * C;   // partials + backward coefficients
}

// `part` is scratch of flpr_bn_partials_floats(M, C) floats (no zeroing needed).
// pre_part / pre_nparts: column partials [pre_nparts][2][C] already produced by the convolution's epilogue
// (gemm_wgmma.cu, `col_part`): the statistics pass over x is skipped.
int flpr_bn_fwd(const void* x, const float* gamma, const float* beta, const void* residual, void* y, float* part,
                float* mean, float* rstd, float* scale, float* shift, float* running_mean,
                float* running_var, int M, int C, float eps, float momentum, int relu, const float* pre_part,
                int pre_nparts, cudaStream_t st) {
  bind_device_of(x);
  if (C % 8) return -2;
  dim3 grid, block; int rpb;
  bn_launch_geometry(M, C, grid, block, rpb);
  if (pre_part != nullptr && pre_nparts > 0) {
    bn_finalize_kernel<<<(C + 31) / 32, dim3(32, FOLD_LANES), 0, st>>>(pre_part, pre_nparts, gamma, beta, mean, rstd, scale,
                                                              shift, running_mean, running_var, M, C, eps, momentum);
  } else {
    bn_stats_kernel<<<grid, block, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), part, M, C, rpb);
    bn_finalize_kernel<<<(C + 31) / 32, dim3(32, FOLD_LANES), 0, st>>>(part, (int)grid.y, gamma, beta, mean, rstd, scale,
                                                              shift, running_mean, running_var, M, C, eps, momentum);
  }
  bn_affine_rows_kernel<<<grid, block, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), scale, shift,
                                                reinterpret_cast<const __nv_bfloat16*>(residual),
                                                reinterpret_cast<__nv_bfloat16*>(y), M, C, rpb, relu);
  return (int)cudaGetLastError();
}

// eval-mode / folded affine: y = relu?(x*scale + shift (+res))
int flpr_affine_act(const void* x, const float* scale, const float* shift, const void* residual, void* y, int M, int C,
                    int relu, cudaStream_t st) {
  bind_device_of(x);
  if (C % 8) return -2;
  dim3 grid, block; int rpb;
  bn_launch_geometry(M, C, grid, block, rpb);
  bn_affine_rows_kernel<<<grid, block, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), scale, shift,
                                                reinterpret_cast<const __nv_bfloat16*>(residual),
                                                reinterpret_cast<__nv_bfloat16*>(y), M, C, rpb, relu);
  return (int)cudaGetLastError();
}

// `part` is scratch of flpr_bn_partials_floats(M, C) floats. dres (nullable) receives the ReLU-masked dy for the
// residual branch.
int flpr_bn_bwd(const void* dy, const void* y, const void* x, const float* mean, const float* rstd, const float* gamma,
                float* dgamma, float* dbeta, float* part, void* dres, void* dx, int M, int C, int relu,
                int accumulate, cudaStream_t st) {
  bind_device_of(dy);
  if (C % 8) return -2;
  dim3 grid, block; int rpb;
  bn_launch_geometry(M, C, grid, block, rpb);
  bn_bwd_reduce_kernel<<<grid, block, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(y),
      reinterpret_cast<const __nv_bfloat16*>(x), mean, rstd, part, reinterpret_cast<__nv_bfloat16*>(dres), M, C, rpb,
      relu);
  float* coef = part + (size_t)grid.y * 2 * C;
  bn_fold_partials_kernel<<<(C + 31) / 32, dim3(32, FOLD_LANES), 0, st>>>(part, (int)grid.y, gamma, mean, rstd, dgamma, dbeta,
                                                                 coef, M, C, accumulate);
  // when the masked dy was materialised in dres, read it back (no second ReLU-mask pass over y)
  const __nv_bfloat16* dy_in = dres ? reinterpret_cast<const __nv_bfloat16*>(dres)
                                    : reinterpret_cast<const __nv_bfloat16*>(dy);
  bn_bwd_rows_kernel<<<grid, block, 0, st>>>(dy_in, reinterpret_cast<const __nv_bfloat16*>(y),
                                             reinterpret_cast<const __nv_bfloat16*>(x), coef,
                                             reinterpret_cast<__nv_bfloat16*>(dx), M, C, rpb, dres ? 0 : relu);
  return (int)cudaGetLastError();
}

int flpr_gap_fwd(const void* x, float* out, void* out_bf16, int N, int HW, int C, cudaStream_t st) {
  bind_device_of(x);
  const int threads = 128;
  gap_fwd_kernel<<<dim3((C / 2 + threads - 1) / threads, N), threads, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), out, reinterpret_cast<__nv_bfloat16*>(out_bf16), HW, C);
  return (int)cudaGetLastError();
}
int flpr_gap_bwd(const float* dout, void* dx, int N, int HW, int C, cudaStream_t st) {
  bind_device_of(dout);
  const int threads = 128;
  gap_bwd_kernel<<<dim3((C / 2 + threads - 1) / threads, N), threads, 0, st>>>(
      dout, reinterpret_cast<__nv_bfloat16*>(dx), HW, C);
  return (int)cudaGetLastError();
}

int flpr_rank_eval(const float* S, const long long* qlab, const long long* glab, float* out_ap, int* out_first, int Q,
                   int G, long long lds, cudaStream_t st) {
  bind_device_of(S);
  const size_t smem = (size_t)G * sizeof(int);
  if (smem > 200 * 1024) return -3;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(rank_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  rank_eval_kernel<<<Q, 256, smem, st>>>(S, qlab, glab, out_ap, out_first, G, lds);
  return (int)cudaGetLastError();
}

// in: uint8 [B,H,W,3]; out: bf16 / fp32 [B,H,W,3]; u: fp32 [7][B] uniforms; mean / inv_std in 0..255 units.
int flpr_augment_u8(const void* in, void* out, const float* u, int B, int H, int W, const float* mean3,
                    const float* inv_std3, float flip_p, float erase_p, float s0, float s1, float r0, float r1,
                    int out_bf16, cudaStream_t st) {
  bind_device_of(in);
  if (W % 4) return -2;
  if (B <= 0) return 0;
  AugArgs a;
  a.in = reinterpret_cast<const uint8_t*>(in); a.out = out; a.u = u; a.B = B; a.H = H; a.W = W;
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean3[c]; a.inv_std[c] = inv_std3[c]; }
  a.flip_p = flip_p; a.erase_p = erase_p; a.s0 = s0; a.s1 = s1; a.lr0 = logf(r0); a.lr1 = logf(r1);
  a.out_bf16 = out_bf16;
  const int quads = H * (W / 4);
  int gx = (quads + 255) / 256;
  if (gx > 16) gx = 16;
  augment_u8_kernel<<<dim3(gx, B), 256, 0, st>>>(a);
  return (int)cudaGetLastError();
}

// picks [P, m] (positions within each identity's row list). feats fp32 [n, D], idx int64 [P, nmax], cnt int32 [P].
int flpr_herding(const float* feats, const long long* idx, const int* cnt, long long* picks, int P, int nmax, int D,
                 int m, cudaStream_t st) {
  bind_device_of(feats);
  if (P <= 0 || m <= 0) return 0;
  const size_t smem = (size_t)(3 * D + 2 * nmax) * sizeof(float);
  if (smem > 200 * 1024) return -3;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(herding_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  herding_kernel<<<P, 256, smem, st>>>(feats, idx, cnt, picks, nmax, D, m);
  return (int)cudaGetLastError();
}

// x [B,H,W,3] bf16 -> y [B, H/2+3, W/2+3, 16] bf16 (space-to-depth cells, zero borders); H, W even.
int flpr_s2d_pad(const void* x, void* y, int B, int H, int W, cudaStream_t st) {
  bind_device_of(x);
  if ((H & 1) || (W & 1)) return -2;
  const size_t cells = (size_t)B * (H / 2 + 3) * (W / 2 + 3);
  s2d_pad_kernel<<<grid_for(cells, 256, 132 * 16), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                                reinterpret_cast<__nv_bfloat16*>(y), B, H, W);
  return (int)cudaGetLastError();
}

// 3x3 / 2 / pad 1 max-pool, NHWC bf16, C multiple of 8.
int flpr_maxpool3x3s2(const void* x, void* y, int B, int H, int W, int C, cudaStream_t st) {
  bind_device_of(x);
  if (C % 8) return -2;
  const size_t total = (size_t)B * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * (C / 8);
  maxpool3x3s2_nhwc_kernel<<<grid_for(total, 256, 132 * 16), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y), B, H, W, C);
  return (int)cudaGetLastError();
}

// Fused Swin window attention. qkv [BW,N,3,H,D], bias fp32 [nWb,H,N,N], out [BW,N,H*D]; bf16 != 0: bf16 tensors.
static int g_window_attn_tc = 1;
void flpr_window_attn_set_tc(int on) { g_window_attn_tc = on; }

int flpr_window_attn_fwd(const void* qkv, const float* bias, void* out, int BW, int N, int H, int D, int nWb,
                         float scale, int bf16, cudaStream_t st) {
  bind_device_of(qkv);
  if (N > ATT_MAXN || D > ATT_MAXD || N < 1) return -2;
  if (bf16 && D == 32 && g_window_attn_tc && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    // tensor-core path: persistent CTAs over (window, head) pairs, QK^T and PV on wgmma
    static bool configured = false;
    if (!configured) {
      cudaError_t e = cudaFuncSetAttribute(window_attn_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           WA_SMEM);
      if (e != cudaSuccess) return (int)e;
      configured = true;
    }
    const long long pairs = (long long)BW * H;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long cap = (long long)sms * 4;
    const int grid_tc = (int)(pairs < cap ? pairs : cap);
    window_attn_fwd_tc_kernel<<<grid_tc, WA_THREADS, WA_SMEM, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), bias,
                                                                    reinterpret_cast<__nv_bfloat16*>(out), N, H, nWb,
                                                                    scale, (int)pairs);
    return (int)cudaGetLastError();
  }
  const size_t smem = ((size_t)2 * N * (D + 1) + (size_t)N * (N + 1)) * sizeof(float);
  dim3 grid(BW, H);
  if (bf16)
    window_attn_fwd_kernel<__nv_bfloat16><<<grid, 64, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), bias,
                                                                   reinterpret_cast<__nv_bfloat16*>(out), N, H, D, nWb,
                                                                   scale);
  else
    window_attn_fwd_kernel<float><<<grid, 64, smem, st>>>(reinterpret_cast<const float*>(qkv), bias,
                                                          reinterpret_cast<float*>(out), N, H, D, nWb, scale);
  return (int)cudaGetLastError();
}

// dqkv [BW,N,3,H,D] is fully written; dbias (nullable, fp32 [nWb,H,N,N]) must be zeroed by the caller.
int flpr_window_attn_bwd(const void* qkv, const float* bias, const void* dout, void* dqkv, float* dbias, int BW, int N,
                         int H, int D, int nWb, float scale, int bf16, cudaStream_t st) {
  bind_device_of(qkv);
  if (N > ATT_MAXN || D > ATT_MAXD || N < 1) return -2;
  const size_t smem = ((size_t)4 * N * (D + 1) + (size_t)2 * N * (N + 1)) * sizeof(float);
  dim3 grid(BW, H);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(window_attn_bwd_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(window_attn_bwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    configured = true;
  }
  if (bf16)
    window_attn_bwd_kernel<__nv_bfloat16><<<grid, 64, smem, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(qkv), bias, reinterpret_cast<const __nv_bfloat16*>(dout),
        reinterpret_cast<__nv_bfloat16*>(dqkv), dbias, N, H, D, nWb, scale);
  else
    window_attn_bwd_kernel<float><<<grid, 64, smem, st>>>(reinterpret_cast<const float*>(qkv), bias,
                                                          reinterpret_cast<const float*>(dout),
                                                          reinterpret_cast<float*>(dqkv), dbias, N, H, D, nWb, scale);
  return (int)cudaGetLastError();
}

}  // extern "C"
