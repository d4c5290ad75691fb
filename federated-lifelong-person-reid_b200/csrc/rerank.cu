// k-reciprocal re-ranking (Zhong et al., CVPR 2017) on the GPU, as separately callable stages over X = cat(query,
// gallery), N = Q + G rows. The similarity matrix S = X X^T comes from the hi/lo wgmma GEMM (ops/rank.py:similarity);
// everything after it lives here:
//
//   sqnorm    |x_i|^2 in fp32, one warp per row (fixed shuffle-tree order).
//   distance  S -> D in place: D_ij = max(|x_i|^2 + |x_j|^2 - 2 S_ij, 0), D_ii = 0, every row divided by its maximum.
//   topk      R[i, :K]: the K = min(k1 + 1, N) smallest entries of D[i, :], ascending, ties to the lower index
//             (== np.argsort(kind="stable")[:K]); K passes of a block-wide lexicographic arg-min.
//   encode    k-reciprocal set K(i), its 2/3-overlap expansion E(i) and the weights exp(-D_ij) / sum_E exp(-D_ie):
//             one fixed-capacity sparse row per i (cap = K (h + 1)), column indices ascending.
//   expand    local query expansion V'_i = mean_{r in R[i, :k2]} V_r: a k2-way merge of sorted sparse rows, one warp
//             per row, each output column summed in rank order.
//   index     inverted index of the gallery rows of V': column j -> (gallery row, value) pairs. Counts (integer
//             atomics), one-block exclusive scan, fill.
//   jaccard   one block per query (x gallery tile): sum_j min(V'_qj, V'_gj) accumulated in shared memory, then
//             J = 1 - m / (2 - m) and final = (1 - lambda) J + lambda D[q, Q + g].
//
// No floating-point atomics anywhere: every floating-point sum has an order fixed by the code, so the result is
// bitwise reproducible from run to run.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ptx.cuh"

namespace flpr {

constexpr int RR_INT_MAX = 0x7fffffff;

// ----------------------------------------------------------------------------- squared norms
// X [N, C] fp32 (row stride ldx). One warp per row: lane-strided partial sums, then the fixed xor-shuffle tree.
__global__ void __launch_bounds__(256) rr_sqnorm_kernel(const float* X, float* out, int N, int C, long long ldx) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  const float* x = X + (long long)row * ldx;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += x[c] * x[c];
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

// ----------------------------------------------------------------------------- distance (in place)
__global__ void __launch_bounds__(256) rr_distance_kernel(float* D, const float* sqn, int N, long long ldd) {
  __shared__ float s_red[32];
  const int i = blockIdx.x;
  float* row = D + (long long)i * ldd;
  const float ni = sqn[i];
  float mx = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    float d = fmaxf(ni + sqn[j] - 2.f * row[j], 0.f);
    if (j == i) d = 0.f;
    row[j] = d;
    mx = fmaxf(mx, d);
  }
  mx = warp_max(mx);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) s_red[w] = mx;
  __syncthreads();
  mx = 0.f;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) mx = fmaxf(mx, s_red[k]);
  if (mx > 0.f)
    for (int j = threadIdx.x; j < N; j += blockDim.x) row[j] = row[j] / mx;
}

// ----------------------------------------------------------------------------- top-K per row
// (v, j) < (v', j')  <=>  v < v' or (v == v' and j < j'): a total order on the row, so the t-th pass picks the least
// element after the (t-1)-th pick. That is exactly a stable ascending sort's first K entries.
__device__ __forceinline__ bool rr_less(float a, int ia, float b, int ib) { return a < b || (a == b && ia < ib); }

__global__ void __launch_bounds__(256) rr_topk_kernel(const float* D, int* R, int N, int K, long long ldd) {
  __shared__ float s_v[32];
  __shared__ int s_j[32];
  const int i = blockIdx.x;
  const float* row = D + (long long)i * ldd;
  float pv = -INFINITY;
  int pj = -1;
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int t = 0; t < K; ++t) {
    float bv = INFINITY;
    int bj = RR_INT_MAX;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float v = row[j];
      if (rr_less(pv, pj, v, j) && rr_less(v, j, bv, bj)) { bv = v; bj = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (rr_less(ov, oj, bv, bj)) { bv = ov; bj = oj; }
    }
    if (l == 0) { s_v[w] = bv; s_j[w] = bj; }
    __syncthreads();
    bv = s_v[0];
    bj = s_j[0];
    for (int k = 1; k < nw; ++k)
      if (rr_less(s_v[k], s_j[k], bv, bj)) { bv = s_v[k]; bj = s_j[k]; }
    __syncthreads();                       // s_v / s_j are rewritten by the next pass
    if (threadIdx.x == 0) R[(long long)i * K + t] = bj;
    pv = bv;
    pj = bj;
  }
}

// ----------------------------------------------------------------------------- encode one row
// R [N, K] (K = min(k1 + 1, N)), hh = min(round(k1 / 2) + 1, K). Output row i: cols[i, :nnz[i]] ascending, vals.
// Shared memory (ints unless noted): F[K], recip[K], kc_n[K], accept[K], kc[K * hh], list[cap], first[cap],
// ocol[cap], w[cap] (float), red[32] (float), counters.
__global__ void __launch_bounds__(128) rr_encode_kernel(const float* D, const int* R, int* cols, float* vals, int* nnz,
                                                        int N, int K, int hh, int cap, long long ldd) {
  extern __shared__ int s_mem[];
  int* F = s_mem;
  int* recip = F + K;
  int* kc_n = recip + K;
  int* accept = kc_n + K;
  int* kc = accept + K;
  int* list = kc + K * hh;
  int* first = list + cap;
  int* ocol = first + cap;
  float* w = reinterpret_cast<float*>(ocol + cap);
  float* red = w + cap;
  __shared__ int s_m, s_n;
  const int i = blockIdx.x;
  const int tid = threadIdx.x;
  (void)N;
  if (tid < K) F[tid] = R[(long long)i * K + tid];
  __syncthreads();
  // K(i): the neighbours f whose own first K neighbours contain i
  if (tid < K) {
    const int* rf = R + (long long)F[tid] * K;
    int r = 0;
    for (int u = 0; u < K; ++u) r |= rf[u] == i;
    recip[tid] = r;
  }
  __syncthreads();
  // candidate sets K_c(c) over the first hh neighbours, for every c in K(i), and the 2/3-overlap test
  if (tid < K) {
    int n = 0, inter = 0;
    if (recip[tid]) {
      const int c = F[tid];
      const int* rc = R + (long long)c * K;
      for (int u = 0; u < hh; ++u) {
        const int f = rc[u];
        const int* rf = R + (long long)f * K;
        int back = 0;
        for (int v = 0; v < hh; ++v) back |= rf[v] == c;
        if (!back) continue;
        kc[tid * hh + n++] = f;
        int in_k = 0;
        for (int v = 0; v < K; ++v) in_k |= (F[v] == f) & recip[v];
        inter += in_k;
      }
    }
    kc_n[tid] = n;
    accept[tid] = recip[tid] && 3 * inter > 2 * n;     // |Kc n K(i)| > (2/3) |Kc|, exactly in integers
  }
  __syncthreads();
  // E(i) with duplicates: K(i), then every accepted K_c (at most K + K * hh <= cap entries)
  if (tid == 0) {
    int m = 0;
    for (int t = 0; t < K; ++t)
      if (recip[t]) list[m++] = F[t];
    for (int t = 0; t < K; ++t)
      if (accept[t])
        for (int u = 0; u < kc_n[t]; ++u) list[m++] = kc[t * hh + u];
    s_m = m;
    s_n = 0;
  }
  __syncthreads();
  const int m = s_m;
  // de-duplicate and sort by counting: an entry is kept at its first occurrence, its output slot is the number of kept
  // entries with a smaller column index
  for (int p = tid; p < m; p += blockDim.x) {
    const int e = list[p];
    int f = 1;
    for (int q = 0; q < p; ++q) f &= list[q] != e;
    first[p] = f;
    if (f) atomicAdd(&s_n, 1);
  }
  __syncthreads();
  const int n_out = s_n;
  for (int p = tid; p < m; p += blockDim.x) {
    if (!first[p]) continue;
    const int e = list[p];
    int pos = 0;
    for (int q = 0; q < m; ++q) pos += first[q] && list[q] < e;
    ocol[pos] = e;
  }
  __syncthreads();
  // weights and their sum (thread-strided partials in ascending slot order, then the fixed shuffle tree)
  const float* drow = D + (long long)i * ldd;
  float part = 0.f;
  for (int p = tid; p < n_out; p += blockDim.x) {
    w[p] = expf(-drow[ocol[p]]);
    part += w[p];
  }
  part = warp_sum(part);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  float total = 0.f;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) total += red[k];
  int* crow = cols + (long long)i * cap;
  float* vrow = vals + (long long)i * cap;
  for (int p = tid; p < n_out; p += blockDim.x) {
    crow[p] = ocol[p];
    vrow[p] = w[p] / total;
  }
  if (tid == 0) nnz[i] = n_out;
}

// ----------------------------------------------------------------------------- local query expansion
// One warp per row; lane l merges the rows of ranks l and l + 32 (k2 <= 64). Each step takes the smallest head column
// over all k2 rows; the contributions of the rows that hold it are summed by lane 0 in rank order (a row that does not
// hold the column adds +0, which leaves the sum unchanged), then divided by k2.
constexpr int RR_EXP_WARPS = 4;

__global__ void __launch_bounds__(RR_EXP_WARPS * 32) rr_expand_kernel(const int* cols, const float* vals,
                                                                     const int* nnz, const int* R, int* ocols,
                                                                     float* ovals, int* onnz, int N, int K, int k2,
                                                                     int cap, int ocap) {
  __shared__ float s_c[RR_EXP_WARPS][64];
  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * RR_EXP_WARPS + wi;
  if (i >= N) return;                                  // warp-uniform
  int row[2], p[2], end[2];
  for (int s = 0; s < 2; ++s) {
    const int r = lane + 32 * s;
    row[s] = r < k2 ? R[(long long)i * K + r] : 0;
    p[s] = 0;
    end[s] = r < k2 ? nnz[row[s]] : 0;
  }
  const float div = (float)k2;
  int n = 0;
  int* orow = ocols + (long long)i * ocap;
  float* vrow = ovals + (long long)i * ocap;
  for (;;) {
    int h[2];
    for (int s = 0; s < 2; ++s) h[s] = p[s] < end[s] ? cols[(long long)row[s] * cap + p[s]] : RR_INT_MAX;
    int mcol = min(h[0], h[1]);
    for (int o = 16; o > 0; o >>= 1) mcol = min(mcol, __shfl_xor_sync(0xffffffffu, mcol, o));
    if (mcol == RR_INT_MAX) break;
    for (int s = 0; s < 2; ++s) {
      float c = 0.f;
      if (h[s] == mcol) {
        c = vals[(long long)row[s] * cap + p[s]];
        p[s]++;
      }
      s_c[wi][lane + 32 * s] = c;
    }
    __syncwarp();
    if (lane == 0) {
      float acc = 0.f;
      for (int r = 0; r < k2; ++r) acc += s_c[wi][r];
      orow[n] = mcol;
      vrow[n] = acc / div;
    }
    n++;
    __syncwarp();
  }
  if (lane == 0) onnz[i] = n;
}

// ----------------------------------------------------------------------------- inverted index (gallery rows)
__global__ void rr_zero_kernel(int* p, int n) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) p[k] = 0;
}

__global__ void __launch_bounds__(128) rr_count_kernel(const int* cols, const int* nnz, int row0, int G, int cap,
                                                       int* cnt) {
  const int g = blockIdx.x;
  if (g >= G) return;
  const int r = row0 + g;
  const int* c = cols + (long long)r * cap;
  for (int p = threadIdx.x; p < nnz[r]; p += blockDim.x) atomicAdd(&cnt[c[p]], 1);
}

// one block: off[0] = 0, off[j + 1] = off[j] + cnt[j]; cnt is reset to zero (the fill cursors)
__global__ void __launch_bounds__(1024) rr_scan_kernel(int* cnt, int* off, int N) {
  __shared__ int s_part[1024];
  const int t = threadIdx.x, nt = blockDim.x;
  const int per = (N + nt - 1) / nt;
  const int lo = min(N, t * per), hi = min(N, lo + per);
  int s = 0;
  for (int j = lo; j < hi; ++j) s += cnt[j];
  s_part[t] = s;
  __syncthreads();
  if (t == 0) {
    int acc = 0;
    for (int k = 0; k < nt; ++k) {
      const int v = s_part[k];
      s_part[k] = acc;
      acc += v;
    }
    off[N] = acc;
  }
  __syncthreads();
  int acc = s_part[t];
  for (int j = lo; j < hi; ++j) {
    off[j] = acc;
    acc += cnt[j];
    cnt[j] = 0;
  }
}

__global__ void __launch_bounds__(128) rr_fill_kernel(const int* cols, const float* vals, const int* nnz, int row0,
                                                      int G, int cap, const int* off, int* cursor, int* idx_row,
                                                      float* idx_val) {
  const int g = blockIdx.x;
  if (g >= G) return;
  const int r = row0 + g;
  const int* c = cols + (long long)r * cap;
  const float* v = vals + (long long)r * cap;
  for (int p = threadIdx.x; p < nnz[r]; p += blockDim.x) {
    const int j = c[p];
    const int at = off[j] + atomicAdd(&cursor[j], 1);
    idx_row[at] = g;
    idx_val[at] = v[p];
  }
}

// ----------------------------------------------------------------------------- Jaccard distance + blend
// Block (q, tile): acc[k] = sum_j min(V'_qj, V'_(Q+t0+k),j) for the gallery items t0 .. t0 + tn of this tile.
//
// Why the sums are reproducible without atomics: the block walks query q's non-zero columns j in ascending order, one
// column at a time, with a barrier after each. Inside column j, the list holds each gallery row at most once (a sparse
// row has one entry per column), so the threads that share the list write DISTINCT accumulator slots - no two updates of
// one slot happen in the same column phase. Across phases the barrier orders them. Hence slot k receives its terms in
// ascending column order, whatever order the fill kernel's atomics gave the rows inside a column and whichever thread
// handles which row.
__global__ void __launch_bounds__(256) rr_jaccard_kernel(const int* qcols, const float* qvals, const int* qnnz,
                                                         int qcap, const int* off, const int* idx_row,
                                                         const float* idx_val, const float* D, long long ldd,
                                                         float* out, int Q, int G, int tile, float lambda) {
  extern __shared__ float s_acc[];
  const int q = blockIdx.x;
  const int t0 = blockIdx.y * tile;
  const int tn = min(tile, G - t0);
  for (int k = threadIdx.x; k < tn; k += blockDim.x) s_acc[k] = 0.f;
  __syncthreads();
  const int* qc = qcols + (long long)q * qcap;
  const float* qv = qvals + (long long)q * qcap;
  const int n = qnnz[q];
  for (int p = 0; p < n; ++p) {
    const int j = qc[p];
    const float a = qv[p];
    const int e1 = off[j + 1];
    for (int e = off[j] + threadIdx.x; e < e1; e += blockDim.x) {
      const int k = idx_row[e] - t0;
      if (k >= 0 && k < tn) s_acc[k] += fminf(a, idx_val[e]);
    }
    __syncthreads();
  }
  const float* drow = D + (long long)q * ldd + Q + t0;
  float* orow = out + (long long)q * G + t0;
  for (int k = threadIdx.x; k < tn; k += blockDim.x) {
    const float m = s_acc[k];
    const float jac = 1.f - m / (2.f - m);
    orow[k] = (1.f - lambda) * jac + lambda * drow[k];
  }
}

}  // namespace flpr

using namespace flpr;

extern "C" {

int flpr_rr_sqnorm(const float* X, float* out, int N, int C, long long ldx, cudaStream_t st) {
  if (N <= 0) return 0;
  bind_device_of(X);
  rr_sqnorm_kernel<<<(N + 7) / 8, 256, 0, st>>>(X, out, N, C, ldx);
  return (int)cudaGetLastError();
}

int flpr_rr_distance(float* D, const float* sqn, int N, long long ldd, cudaStream_t st) {
  if (N <= 0) return 0;
  bind_device_of(D);
  rr_distance_kernel<<<N, 256, 0, st>>>(D, sqn, N, ldd);
  return (int)cudaGetLastError();
}

int flpr_rr_topk(const float* D, int* R, int N, int K, long long ldd, cudaStream_t st) {
  if (N <= 0) return 0;
  if (K < 1 || K > N || K > 64) return -2;
  bind_device_of(D);
  rr_topk_kernel<<<N, 256, 0, st>>>(D, R, N, K, ldd);
  return (int)cudaGetLastError();
}

// cap must be >= K * (hh + 1)
int flpr_rr_encode(const float* D, const int* R, int* cols, float* vals, int* nnz, int N, int K, int hh, int cap,
                   long long ldd, cudaStream_t st) {
  if (N <= 0) return 0;
  if (K < 1 || K > 64 || hh < 1 || hh > K || cap < K * (hh + 1)) return -2;
  bind_device_of(D);
  const size_t smem = (size_t)(4 * K + K * hh + 4 * cap + 32) * sizeof(int);
  if (smem > 200 * 1024) return -3;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(rr_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  rr_encode_kernel<<<N, 128, smem, st>>>(D, R, cols, vals, nnz, N, K, hh, cap, ldd);
  return (int)cudaGetLastError();
}

// ocap must be >= k2 * cap (the union of k2 rows)
int flpr_rr_expand(const int* cols, const float* vals, const int* nnz, const int* R, int* ocols, float* ovals,
                   int* onnz, int N, int K, int k2, int cap, int ocap, cudaStream_t st) {
  if (N <= 0) return 0;
  if (k2 < 1 || k2 > K || k2 > 64 || ocap < k2 * cap) return -2;
  bind_device_of(cols);
  rr_expand_kernel<<<(N + RR_EXP_WARPS - 1) / RR_EXP_WARPS, RR_EXP_WARPS * 32, 0, st>>>(
      cols, vals, nnz, R, ocols, ovals, onnz, N, K, k2, cap, ocap);
  return (int)cudaGetLastError();
}

// Inverted index of rows row0 .. row0 + G of a sparse matrix with N columns. cnt: int [N] scratch, off: int [N + 1];
// idx_row / idx_val hold at least sum(nnz[row0 : row0 + G]) entries. Gallery rows are stored as 0 .. G - 1.
int flpr_rr_index(const int* cols, const float* vals, const int* nnz, int row0, int G, int N, int cap, int* cnt,
                  int* off, int* idx_row, float* idx_val, cudaStream_t st) {
  if (N <= 0) return 0;
  bind_device_of(cols);
  rr_zero_kernel<<<min((N + 255) / 256, 1024), 256, 0, st>>>(cnt, N);
  if (G > 0) rr_count_kernel<<<G, 128, 0, st>>>(cols, nnz, row0, G, cap, cnt);
  rr_scan_kernel<<<1, 1024, 0, st>>>(cnt, off, N);
  if (G > 0) rr_fill_kernel<<<G, 128, 0, st>>>(cols, vals, nnz, row0, G, cap, off, cnt, idx_row, idx_val);
  return (int)cudaGetLastError();
}

// out [Q, G] fp32; tile = gallery items per block (0: the largest that fits in shared memory).
int flpr_rr_jaccard(const int* qcols, const float* qvals, const int* qnnz, int qcap, const int* off, const int* idx_row,
                    const float* idx_val, const float* D, long long ldd, float* out, int Q, int G, int tile,
                    float lambda, cudaStream_t st) {
  if (Q <= 0 || G <= 0) return 0;
  bind_device_of(D);
  const int max_tile = 48 * 1024;                      // 192 KB of fp32 accumulators
  if (tile <= 0 || tile > max_tile) tile = max_tile;
  if (tile > G) tile = G;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(rr_jaccard_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  const int tiles = (G + tile - 1) / tile;
  if (tiles > 65535) return -2;
  rr_jaccard_kernel<<<dim3(Q, tiles), 256, (size_t)tile * sizeof(float), st>>>(qcols, qvals, qnnz, qcap, off, idx_row,
                                                                               idx_val, D, ldd, out, Q, G, tile, lambda);
  return (int)cudaGetLastError();
}

}  // extern "C"
