// Compressed scene export (DESIGN 3.24; the fp64 model is oracle/compress_oracle.py): the k-means
// vector quantiser of the higher-order SH rows and the 8 / 16-bit scalar quantiser of the others.
//
//  k_kmeans_prep     the codebook transposed into ws = ct[D + 1][Kp] (Kp = K rounded up to 128):
//                    rows 0..D-1 the coordinates, row D the norms |c|^2 (a fixed fmaf chain over d).
//                    Padding centroids have coordinates 0 and norm NaN, so they never win.
//  k_kmeans_assign   a register-tiled SGEMM: a CTA holds 128 points (transposed in shared memory) and
//                    streams the codebook through two 128-centroid shared tiles by cp.async; each of
//                    its 16 x 16 threads owns 8 points x 8 centroids and keeps a running (score, index)
//                    per point, score = |c|^2 - 2 x.c (fmaf chain over d from 0).  The 16 threads that
//                    share a point reduce by shuffles, lowest index on ties.  No N x K value is stored.
//  k_kmeans_update   one warp per cluster over the label-sorted (stable) permutation: the members are
//                    summed in fp64 in ascending point index, lane d owning columns d and d + 32.  An
//                    empty cluster keeps its previous centroid.
//  k_quant_range     per-column min / max of the transformed values: shared-memory then global integer
//                    atomics on the order-preserving key of the float bits (order-free, so exact).
//  k_quantize / k_dequantize   elementwise over [N, D]; a thread always sees the same column because
//                    the block size and the grid stride are multiples of D.  The code is formed in fp64
//                    (16-bit codes are too fine for fp32's rounding of (t - lo) (2^b - 1) / (hi - lo)).
#include <climits>

#include "common.cuh"
#include "kernels.h"

namespace gsb {

namespace {

constexpr int KM_TILE = 128;    // points and centroids of one CTA tile
constexpr int KM_THREADS = 256; // 16 x 16 threads, 8 x 8 (point, centroid) pairs each
constexpr int KM_UPDATE_THREADS = 256;
constexpr int Q_THREADS = 256;

__global__ void __launch_bounds__(256) k_kmeans_prep(int K, int Kp, int D, const float *__restrict__ c,
                                                     float *__restrict__ ct) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= Kp) return;
  float n = 0.f;
  for (int d = 0; d < D; d++) {
    const float v = k < K ? c[(size_t)k * D + d] : 0.f;
    ct[(size_t)d * Kp + k] = v;
    n = fmaf(v, v, n);
  }
  ct[(size_t)D * Kp + k] = k < K ? n : __int_as_float(0x7fc00000);
}

// the 4 + 4 columns a thread owns of a 128-wide tile: 4 t .. 4 t + 3 and 64 + 4 t .. 64 + 4 t + 3
__device__ __forceinline__ int km_col(int t, int j) { return (j < 4 ? 0 : 64 - 4) + 4 * t + j; }

__global__ void __launch_bounds__(KM_THREADS, 2) k_kmeans_assign(int N, int Kp, int D, const float *__restrict__ x,
                                                                 int64_t ldx, const float *__restrict__ ct,
                                                                 int32_t *__restrict__ labels,
                                                                 float *__restrict__ dist) {
  extern __shared__ __align__(16) float km_smem[];
  __shared__ float xnorm[KM_TILE];
  float *xs = km_smem;                 // [D][128] points, transposed
  float *cs = km_smem + D * KM_TILE;   // 2 x [D + 1][128] centroid tiles
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int p0 = blockIdx.x * KM_TILE;
  const int tile_floats = (D + 1) * KM_TILE;
  const int ntiles = Kp / KM_TILE;

  auto stage = [&](int t, int buf) {
    const float *src = ct + (size_t)t * KM_TILE;
    float *dst = cs + buf * tile_floats;
    for (int e = tid; e < (D + 1) * (KM_TILE / 4); e += KM_THREADS) {
      const int r = e >> 5, q = e & 31;
      cp_async16_sa(smem_u32(dst + r * KM_TILE + q * 4), src + (size_t)r * Kp + q * 4);
    }
    cp_async_commit();
  };
  stage(0, 0);
  for (int e = tid; e < KM_TILE * D; e += KM_THREADS) {
    const int p = e / D, d = e - p * D;
    xs[d * KM_TILE + p] = p0 + p < N ? x[(int64_t)(p0 + p) * ldx + d] : 0.f;
  }
  __syncthreads();
  if (tid < KM_TILE) {
    float s = 0.f;
    for (int d = 0; d < D; d++) s = fmaf(xs[d * KM_TILE + tid], xs[d * KM_TILE + tid], s);
    xnorm[tid] = s;
  }

  float best[8];
  int bidx[8];
#pragma unroll
  for (int i = 0; i < 8; i++) best[i] = INFINITY, bidx[i] = INT_MAX;

  for (int t = 0; t < ntiles; t++) {
    if (t + 1 < ntiles) {
      stage(t + 1, (t + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float *cb = cs + (t & 1) * tile_floats;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
#pragma unroll 2
    for (int d = 0; d < D; d++) {
      const float4 a0 = *reinterpret_cast<const float4 *>(xs + d * KM_TILE + 4 * ty);
      const float4 a1 = *reinterpret_cast<const float4 *>(xs + d * KM_TILE + 64 + 4 * ty);
      const float4 b0 = *reinterpret_cast<const float4 *>(cb + d * KM_TILE + 4 * tx);
      const float4 b1 = *reinterpret_cast<const float4 *>(cb + d * KM_TILE + 64 + 4 * tx);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    const float4 n0 = *reinterpret_cast<const float4 *>(cb + D * KM_TILE + 4 * tx);
    const float4 n1 = *reinterpret_cast<const float4 *>(cb + D * KM_TILE + 64 + 4 * tx);
    const float nn[8] = {n0.x, n0.y, n0.z, n0.w, n1.x, n1.y, n1.z, n1.w};
    // j ascends with the centroid index, and tiles ascend: a strict < keeps the lowest index
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float s = fmaf(-2.f, acc[i][j], nn[j]);
        if (s < best[i]) best[i] = s, bidx[i] = t * KM_TILE + km_col(tx, j);
      }
    __syncthreads();  // the next stage overwrites the buffer just read
  }

#pragma unroll
  for (int i = 0; i < 8; i++) {
    float s = best[i];
    int k = bidx[i];
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      const float s2 = __shfl_xor_sync(0xffffffffu, s, off);
      const int k2 = __shfl_xor_sync(0xffffffffu, k, off);
      if (s2 < s || (s2 == s && k2 < k)) s = s2, k = k2;
    }
    const int p = km_col(ty, i);
    if (tx == 0 && p0 + p < N) {
      labels[p0 + p] = k == INT_MAX ? 0 : k;  // INT_MAX: every score was NaN (non-finite input)
      dist[p0 + p] = fmaxf(s + xnorm[p], 0.f);
    }
  }
}

// first position i of the label-sorted order with labels[perm[i]] >= v
__device__ __forceinline__ int km_lower(int N, const int32_t *__restrict__ labels, const int32_t *__restrict__ perm,
                                        int v) {
  int lo = 0, hi = N;
  while (lo < hi) {
    const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
    const int p = perm[mid];
    const int l = (unsigned)p < (unsigned)N ? labels[p] : INT_MAX;
    if (l < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(KM_UPDATE_THREADS) k_kmeans_update(int N, int K, int D, const float *__restrict__ x,
                                                                     int64_t ldx, const int32_t *__restrict__ labels,
                                                                     const int32_t *__restrict__ perm,
                                                                     const float *__restrict__ cin,
                                                                     float *__restrict__ cout,
                                                                     int32_t *__restrict__ counts) {
  const int k = (int)(((int64_t)blockIdx.x * KM_UPDATE_THREADS + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (k >= K) return;
  const int b = km_lower(N, labels, perm, k), e = km_lower(N, labels, perm, k + 1);
  double s0 = 0.0, s1 = 0.0;
#pragma unroll 4
  for (int i = b; i < e; i++) {
    const int p = perm[i];
    if ((unsigned)p >= (unsigned)N) continue;
    const float *r = x + (int64_t)p * ldx;
    if (lane < D) s0 += (double)r[lane];
    if (lane + 32 < D) s1 += (double)r[lane + 32];
  }
  const int n = e - b;
  if (lane == 0) counts[k] = n;
  const size_t row = (size_t)k * D;
  if (n == 0) {
    if (lane < D) cout[row + lane] = cin[row + lane];
    if (lane + 32 < D) cout[row + lane + 32] = cin[row + lane + 32];
  } else {
    if (lane < D) cout[row + lane] = (float)(s0 / (double)n);
    if (lane + 32 < D) cout[row + lane + 32] = (float)(s1 / (double)n);
  }
}

// the positions' transform sign(v) log1p(|v|) and its inverse
__device__ __forceinline__ float q_fwd(float v, int log_t) { return log_t ? copysignf(log1pf(fabsf(v)), v) : v; }
__device__ __forceinline__ float q_inv(float y, int log_t) { return log_t ? copysignf(expm1f(fabsf(y)), y) : y; }
// float bits -> an unsigned key with the float order (negative values flipped whole, positive ones
// get the sign bit), and back
__device__ __forceinline__ unsigned q_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float q_unkey(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// range[2][D] holds the keys: row 0 the minima (set to 0xff bytes first), row 1 the maxima (0)
__global__ void __launch_bounds__(Q_THREADS) k_quant_range(int64_t n, int D, const float *__restrict__ x, int64_t ldx,
                                                           int log_t, unsigned *__restrict__ keys) {
  __shared__ unsigned smin[64], smax[64];
  const int bd = blockDim.x;  // a multiple of D
  const int d = threadIdx.x % D;
  if (threadIdx.x < D) smin[threadIdx.x] = 0xffffffffu, smax[threadIdx.x] = 0u;
  __syncthreads();
  unsigned lo = 0xffffffffu, hi = 0u;
  for (int64_t e = (int64_t)blockIdx.x * bd + threadIdx.x; e < n; e += (int64_t)gridDim.x * bd) {
    const unsigned k = q_key(q_fwd(x[(e / D) * ldx + d], log_t));
    lo = min(lo, k);
    hi = max(hi, k);
  }
  if (lo <= hi) {
    atomicMin(&smin[d], lo);
    atomicMax(&smax[d], hi);
  }
  __syncthreads();
  if (threadIdx.x < D && smin[threadIdx.x] <= smax[threadIdx.x]) {
    atomicMin(&keys[threadIdx.x], smin[threadIdx.x]);
    atomicMax(&keys[D + threadIdx.x], smax[threadIdx.x]);
  }
}

// keys -> floats in place; a column that saw no value (N = 0) gets lo = hi = 0
__global__ void k_quant_unkey(int D, float *__restrict__ range) {
  const int d = threadIdx.x;
  if (d >= D) return;
  const unsigned a = __float_as_uint(range[d]), b = __float_as_uint(range[D + d]);
  range[d] = a <= b ? q_unkey(a) : 0.f;
  range[D + d] = a <= b ? q_unkey(b) : 0.f;
}

template <typename Q>
__global__ void __launch_bounds__(Q_THREADS) k_quantize(int64_t n, int D, const float *__restrict__ x, int64_t ldx,
                                                        int log_t, float qmax, const float *__restrict__ range,
                                                        Q *__restrict__ codes) {
  const int bd = blockDim.x;
  const int d = threadIdx.x % D;
  // the code in fp64 from the fp32 value and range: the formula's rounding, not fp32's, decides it
  const double lo = range[d], hi = range[D + d];
  const double scale = hi > lo ? (double)qmax / (hi - lo) : 0.0;
  for (int64_t e = (int64_t)blockIdx.x * bd + threadIdx.x; e < n; e += (int64_t)gridDim.x * bd) {
    const double v = q_fwd(x[(e / D) * ldx + d], log_t);
    const double q = floor((v - lo) * scale + 0.5);
    codes[e] = (Q)fmin(fmax(q, 0.0), (double)qmax);  // fmax also sends NaN to 0
  }
}

template <typename Q>
__global__ void __launch_bounds__(Q_THREADS) k_dequantize(int64_t n, int D, const Q *__restrict__ codes, float qmax,
                                                          const float *__restrict__ range, int log_t,
                                                          float *__restrict__ out) {
  const int bd = blockDim.x;
  const int d = threadIdx.x % D;
  const float lo = range[d];
  const float step = (range[D + d] - lo) / qmax;
  for (int64_t e = (int64_t)blockIdx.x * bd + threadIdx.x; e < n; e += (int64_t)gridDim.x * bd)
    out[e] = q_inv(fmaf((float)codes[e], step, lo), log_t);
}

// block size (a multiple of D) and grid of the elementwise kernels over n = N D elements
struct QLaunch {
  int threads, blocks;
};
QLaunch q_launch(int64_t n, int D) {
  const int threads = Q_THREADS / D * D;
  const int64_t want = (n + threads - 1) / threads;
  return {threads, (int)(want < 4 * 132 ? want : 4 * 132)};
}

size_t kmeans_smem(int D) { return ((size_t)D * KM_TILE + 2 * (size_t)(D + 1) * KM_TILE) * sizeof(float); }

}  // namespace

int kmeans_padded(int K) { return (K + KM_TILE - 1) / KM_TILE * KM_TILE; }

size_t kmeans_assign_workspace_bytes(int K, int D) { return (size_t)(D + 1) * kmeans_padded(K) * sizeof(float); }

int launch_kmeans_assign(int N, int K, int D, const float *x, int64_t ldx, const float *centroids, int32_t *labels,
                         float *dist, void *ws, cudaStream_t st) {
  if (N == 0) return 0;
  const int Kp = kmeans_padded(K);
  float *ct = static_cast<float *>(ws);
  const size_t smem = kmeans_smem(D);
  if (smem > 48 * 1024)
    GSB_CUDA_TRY(cudaFuncSetAttribute(k_kmeans_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfScope ps(K_KMEANS_ASSIGN, st);
  k_kmeans_prep<<<Kp / 256 + 1, 256, 0, st>>>(K, Kp, D, centroids, ct);
  GSB_CUDA_TRY(cudaGetLastError());
  k_kmeans_assign<<<(N + KM_TILE - 1) / KM_TILE, KM_THREADS, smem, st>>>(N, Kp, D, x, ldx, ct, labels, dist);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_kmeans_update(int N, int K, int D, const float *x, int64_t ldx, const int32_t *labels, const int32_t *perm,
                         const float *centroids, float *centroids_out, int32_t *counts, cudaStream_t st) {
  const int64_t blocks = ((int64_t)K * 32 + KM_UPDATE_THREADS - 1) / KM_UPDATE_THREADS;
  ProfScope ps(K_KMEANS_UPDATE, st);
  k_kmeans_update<<<(unsigned)blocks, KM_UPDATE_THREADS, 0, st>>>(N, K, D, x, ldx, labels, perm, centroids,
                                                                  centroids_out, counts);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_quantize(int N, int D, const float *x, int64_t ldx, int bits, int log_t, int fit_range, float *range,
                    void *codes, cudaStream_t st) {
  const int64_t n = (int64_t)N * D;
  const QLaunch L = q_launch(n, D);
  const float qmax = (float)((1 << bits) - 1);
  ProfScope ps(K_QUANTIZE, st);
  if (fit_range) {
    GSB_CUDA_TRY(cudaMemsetAsync(range, 0xff, D * sizeof(float), st));
    GSB_CUDA_TRY(cudaMemsetAsync(range + D, 0, D * sizeof(float), st));
    if (n > 0) {
      k_quant_range<<<L.blocks, L.threads, 0, st>>>(n, D, x, ldx, log_t, reinterpret_cast<unsigned *>(range));
      GSB_CUDA_TRY(cudaGetLastError());
    }
    k_quant_unkey<<<1, 64, 0, st>>>(D, range);
    GSB_CUDA_TRY(cudaGetLastError());
  }
  if (n == 0) return 0;
  if (bits == 8)
    k_quantize<uint8_t><<<L.blocks, L.threads, 0, st>>>(n, D, x, ldx, log_t, qmax, range, (uint8_t *)codes);
  else
    k_quantize<uint16_t><<<L.blocks, L.threads, 0, st>>>(n, D, x, ldx, log_t, qmax, range, (uint16_t *)codes);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_dequantize(int N, int D, const void *codes, int bits, const float *range, int log_t, float *out,
                      cudaStream_t st) {
  const int64_t n = (int64_t)N * D;
  if (n == 0) return 0;
  const QLaunch L = q_launch(n, D);
  const float qmax = (float)((1 << bits) - 1);
  ProfScope ps(K_DEQUANTIZE, st);
  if (bits == 8)
    k_dequantize<uint8_t><<<L.blocks, L.threads, 0, st>>>(n, D, (const uint8_t *)codes, qmax, range, log_t, out);
  else
    k_dequantize<uint16_t><<<L.blocks, L.threads, 0, st>>>(n, D, (const uint16_t *)codes, qmax, range, log_t, out);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
