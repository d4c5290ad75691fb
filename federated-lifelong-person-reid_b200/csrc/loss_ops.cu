// flpr metric / distillation losses (criterions/triplet_loss.py:89-127, tools/distance.py:9-30,
// criterions/kd_loss.py:10-27, methods/icarl.py:216-236 of the reference), fused around the wgmma Gram matrix:
//
//   triplet_mine_fwd   one block per anchor: distance row from the Gram matrix (squared euclidean  |xi|^2 + |xj|^2 -
//                      2 G_ij  or cosine  1 - G_ij), positive / negative masks from the labels, hard (arg-max / arg-min)
//                      or softmax-weighted mining -> dist_ap[i], dist_an[i] and the mining Jacobians
//                      d dist_ap[i] / d dist[i,j],  d dist_an[i] / d dist[i,j]   (two B x B fp32 matrices).
//   triplet_mine_bwd   W = g_ap (.) J_ap + g_an (.) J_an  ->  S = W + W^T (bf16, the operand of the gradient GEMM
//                      dX = 2 (rowsum(S) (.) X - S X)  /  - S X  that runs on the wgmma kernel) and rowsum(S).
//   kd_kl              KL( softmax(t / T) || softmax(s / T) ) * T^2 / B  with gradient w.r.t. the student logits.
//   bce_distill        iCaRL: BCEWithLogits(score, one-hot) + BCEWithLogits(score[:, :P], sigmoid(prev logits)),
//                      mean-reduced, with gradient.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ptx.cuh"

namespace flpr {

__device__ __forceinline__ float blk_reduce(float v, float* sh, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = is_max ? -INFINITY : 0.f;
  for (int i = 0; i < nw; ++i) r = is_max ? fmaxf(r, sh[i]) : r + sh[i];
  return r;  // valid in every thread
}

// G: [B, ldg] fp32 Gram matrix X X^T; sq: [B] |x_i|^2 (euclid only); lab: [B].
__global__ void __launch_bounds__(128) triplet_mine_fwd_kernel(const float* G, long long ldg, const float* sq,
                                                               const long long* lab, int B, int cosine, int hard,
                                                               float* dist_ap, float* dist_an, float* Jap,
                                                               float* Jan) {
  __shared__ float sh[8];
  __shared__ int s_arg[2];
  const int i = blockIdx.x;
  const long long li = lab[i];
  const float sqi = cosine ? 0.f : sq[i];
  auto dist_of = [&](int j) -> float {
    const float g = G[(long long)i * ldg + j];
    return cosine ? 1.f - g : sqi + sq[j] - 2.f * g;
  };
  float* jap = Jap + (long long)i * B;
  float* jan = Jan + (long long)i * B;
  if (hard) {
    // dist_ap = max_j dist*pos ; dist_an = min_j (dist*neg + pos*1e9)   (first index wins a tie, like torch.max / min)
    float bp = -INFINITY, bn = INFINITY;
    int ip = B, in_ = B;
    for (int j = threadIdx.x; j < B; j += blockDim.x) {
      const bool pos = lab[j] == li;
      const float d = dist_of(j);
      const float vp = pos ? d : 0.f;
      const float vn = pos ? 1e9f : d;
      if (vp > bp) { bp = vp; ip = j; }
      if (vn < bn) { bn = vn; in_ = j; }
      jap[j] = 0.f;
      jan[j] = 0.f;
    }
    const float mp = blk_reduce(bp, sh, true);
    const float mn = -blk_reduce(-bn, sh, true);
    if (threadIdx.x == 0) { s_arg[0] = B; s_arg[1] = B; }
    __syncthreads();
    if (bp == mp) atomicMin(&s_arg[0], ip);
    if (bn == mn) atomicMin(&s_arg[1], in_);
    __syncthreads();
    if (threadIdx.x == 0) {
      dist_ap[i] = mp;
      dist_an[i] = mn;
      const int p = s_arg[0], n = s_arg[1];
      if (p < B && lab[p] == li) jap[p] = 1.f;      // (an all-masked max is the constant 0: no gradient)
      if (n < B && lab[n] != li) jan[n] = 1.f;
    }
    return;
  }
  // softmax-weighted mining (fast-reid): w = softmax over the masked entries, +1e-6 in the denominator
  float mxp = -INFINITY, mxn = -INFINITY;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const bool pos = lab[j] == li;
    const float d = dist_of(j);
    mxp = fmaxf(mxp, pos ? d : 0.f);               // max over (dist * is_pos): masked entries count as 0
    mxn = fmaxf(mxn, pos ? 0.f : -d);              // max over (-dist * is_neg)
  }
  mxp = blk_reduce(mxp, sh, true);
  mxn = blk_reduce(mxn, sh, true);
  float zp = 0.f, zn = 0.f, sp = 0.f, sn = 0.f;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const bool pos = lab[j] == li;
    const float d = dist_of(j);
    if (pos) {
      const float e = __expf(d - mxp);
      zp += e;
      sp += d * e;
    } else {
      const float e = __expf(-d - mxn);
      zn += e;
      sn += d * e;
    }
  }
  zp = blk_reduce(zp, sh, false) + 1e-6f;
  zn = blk_reduce(zn, sh, false) + 1e-6f;
  const float ap = blk_reduce(sp, sh, false) / zp;
  const float an = blk_reduce(sn, sh, false) / zn;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const bool pos = lab[j] == li;
    const float d = dist_of(j);
    if (pos) {
      const float w = __expf(d - mxp) / zp;
      jap[j] = w * (1.f + d - ap);
      jan[j] = 0.f;
    } else {
      const float w = __expf(-d - mxn) / zn;
      jap[j] = 0.f;
      jan[j] = w * (1.f - d + an);
    }
  }
  if (threadIdx.x == 0) {
    dist_ap[i] = ap;
    dist_an[i] = an;
  }
}

// S[i, j] = W_ij + W_ji with W = g_ap[i] Jap[i, j] + g_an[i] Jan[i, j];  S is written bf16 with row stride lds
// (padded columns zero-filled); rs[i] = sum_j S[i, j] (fp32).
__global__ void __launch_bounds__(128) triplet_mine_bwd_kernel(const float* Jap, const float* Jan, const float* g_ap,
                                                               const float* g_an, int B, __nv_bfloat16* S,
                                                               long long lds, float* rs) {
  __shared__ float sh[8];
  const int i = blockIdx.x;
  const float gpi = g_ap[i], gni = g_an[i];
  float acc = 0.f;
  for (int j = threadIdx.x; j < (int)lds; j += blockDim.x) {
    float s = 0.f;
    if (j < B) {
      s = gpi * Jap[(long long)i * B + j] + gni * Jan[(long long)i * B + j] +
          g_ap[j] * Jap[(long long)j * B + i] + g_an[j] * Jan[(long long)j * B + i];
      acc += s;
    }
    S[(long long)i * lds + j] = __float2bfloat16(s);
  }
  acc = blk_reduce(acc, sh, false);
  if (threadIdx.x == 0) rs[i] = acc;
}

// One block per row. loss[0] += scale * sum_c p_t (log p_t - log p_s);  ds = scale / T * (p_s - p_t)   (scale = T^2/B)
template <typename T>
__global__ void __launch_bounds__(256) kd_kl_kernel(const T* s, const T* t, float* ds, float* loss, int C,
                                                    long long lds_, long long ldt, float invT, float scale) {
  __shared__ float sh[8];
  const int row = blockIdx.x;
  const T* sp = s + (long long)row * lds_;
  const T* tp = t + (long long)row * ldt;
  float ms = -INFINITY, mt = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    ms = fmaxf(ms, (float)sp[c] * invT);
    mt = fmaxf(mt, (float)tp[c] * invT);
  }
  ms = blk_reduce(ms, sh, true);
  mt = blk_reduce(mt, sh, true);
  float zs = 0.f, zt = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    zs += __expf((float)sp[c] * invT - ms);
    zt += __expf((float)tp[c] * invT - mt);
  }
  zs = blk_reduce(zs, sh, false);
  zt = blk_reduce(zt, sh, false);
  const float lzs = logf(zs), lzt = logf(zt);
  float kl = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float ls = (float)sp[c] * invT - ms - lzs;
    const float lt = (float)tp[c] * invT - mt - lzt;
    const float pt = __expf(lt);
    if (pt > 0.f) kl += pt * (lt - ls);
    ds[(long long)row * C + c] = scale * invT * (__expf(ls) - pt);
  }
  kl = blk_reduce(kl, sh, false);
  if (threadIdx.x == 0) atomicAdd(loss, scale * kl);
}

// iCaRL distillation pass over [B, C] logits: mean over B*C of BCE(z, onehot(target))  +  mean over B*P of
// BCE(z[:, :P], sigmoid(prev[:, :P])).  dz gets both gradients.
template <typename T>
__global__ void __launch_bounds__(256) bce_distill_kernel(const T* z, const long long* target, const float* prev,
                                                          float* dz, float* loss, int B, int C, int P, long long ldz,
                                                          long long ldp) {
  __shared__ float sh[8];
  const long long n = (long long)B * C;
  const float w1 = 1.f / (float)n;
  const float w2 = P > 0 ? 1.f / ((float)B * (float)P) : 0.f;
  float acc = 0.f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / C), c = (int)(e - (long long)r * C);
    const float x = (float)z[(long long)r * ldz + c];
    const float sp = fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x)));   // softplus(x) = -log(1 - sigmoid(x))
    const float sg = 1.f / (1.f + __expf(-x));
    const float y = (target[r] == c) ? 1.f : 0.f;
    acc += w1 * (sp - x * y);
    float g = w1 * (sg - y);
    if (c < P) {
      const float q = 1.f / (1.f + __expf(-prev[(long long)r * ldp + c]));
      acc += w2 * (sp - x * q);
      g += w2 * (sg - q);
    }
    dz[(long long)r * C + c] = g;
  }
  acc = blk_reduce(acc, sh, false);
  if (threadIdx.x == 0) atomicAdd(loss, acc);
}

}  // namespace flpr

using namespace flpr;

extern "C" {

int flpr_triplet_mine_fwd(const float* G, long long ldg, const float* sq, const long long* lab, int B, int cosine,
                          int hard, float* dist_ap, float* dist_an, float* Jap, float* Jan, cudaStream_t st) {
  if (B <= 0) return 0;
  bind_device_of(G);
  triplet_mine_fwd_kernel<<<B, 128, 0, st>>>(G, ldg, sq, lab, B, cosine, hard, dist_ap, dist_an, Jap, Jan);
  return (int)cudaGetLastError();
}

int flpr_triplet_mine_bwd(const float* Jap, const float* Jan, const float* g_ap, const float* g_an, int B, void* S,
                          long long lds, float* rs, cudaStream_t st) {
  if (B <= 0) return 0;
  bind_device_of(Jap);
  triplet_mine_bwd_kernel<<<B, 128, 0, st>>>(Jap, Jan, g_ap, g_an, B, reinterpret_cast<__nv_bfloat16*>(S), lds, rs);
  return (int)cudaGetLastError();
}

int flpr_kd_kl(const void* s, const void* t, float* ds, float* loss, int B, int C, long long lds_, long long ldt,
               float temperature, int is_bf16, cudaStream_t st) {
  if (B <= 0) return 0;
  bind_device_of(s);
  const float invT = 1.f / temperature, scale = temperature * temperature / (float)B;
  if (is_bf16)
    kd_kl_kernel<__nv_bfloat16><<<B, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(s),
                                                   reinterpret_cast<const __nv_bfloat16*>(t), ds, loss, C, lds_, ldt,
                                                   invT, scale);
  else
    kd_kl_kernel<float><<<B, 256, 0, st>>>(reinterpret_cast<const float*>(s), reinterpret_cast<const float*>(t), ds,
                                           loss, C, lds_, ldt, invT, scale);
  return (int)cudaGetLastError();
}

int flpr_bce_distill(const void* z, const long long* target, const float* prev, float* dz, float* loss, int B, int C,
                     int P, long long ldz, long long ldp, int is_bf16, cudaStream_t st) {
  if (B <= 0 || C <= 0) return 0;
  bind_device_of(z);
  const long long n = (long long)B * C;
  int grid = (int)((n + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  if (is_bf16)
    bce_distill_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(z), target, prev, dz,
                                                            loss, B, C, P, ldz, ldp);
  else
    bce_distill_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(z), target, prev, dz, loss, B, C, P,
                                                    ldz, ldp);
  return (int)cudaGetLastError();
}

}  // extern "C"
