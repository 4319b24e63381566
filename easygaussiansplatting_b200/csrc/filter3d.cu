// Mip-Splatting's 3D smoothing filter (pg_fused_math.h filter3d_*): the per-Gaussian sampling-rate
// bound from the training cameras, and the two elementwise passes that put it around the fused
// per-Gaussian kernels without touching them.
//   k_filter3d_depth   d_i = the smallest camera-frame depth over the cameras that see Gaussian i
//                      (0 when none does), the largest such d and the largest positive fx.  Grid-stride over
//                      the Gaussians; the camera table goes through shared memory F3_CHUNK rows at
//                      a time and every lane of a warp reads the same row (a broadcast).  Each CTA
//                      folds its two maxima into the workspace with one atomicMax each on the float
//                      bits: the values are >= 0, so the integer order is the float order and the
//                      result does not depend on the CTAs' order.
//   k_filter3d_finish  filter3d_i = sqrt(variance) d_i / f_max (unseen rows take the largest d;
//                      all 0 when no row is seen or no camera has fx > 0)
//   k_filter3d_apply   (s, alpha) -> (s', alpha'), 28 B in / 16 B out per Gaussian
//   k_filter3d_bwd     (dL/ds', dL/dalpha') -> (dL/ds, dL/dalpha), 36 B in / 16 B out; may run in place
#include "common.cuh"
#include "kernels.h"
#include "pg_fused_math.h"

namespace gsb {

constexpr int F3T = 256;  // threads per CTA of every filter kernel
static_assert(F3_CHUNK * pg::kCamRow % 4 == 0, "the staged chunk is read as float4 rows");

__device__ __forceinline__ float block_max(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = 0.f;
  for (int w = 0; w < F3T / 32; w++) m = fmaxf(m, red[w]);
  return m;
}

// ws[0] = bits of the largest d over the seen rows, ws[1] = bits of the largest fx (both zeroed by
// the launcher).  The loop bounds are the same for every thread of a CTA, so all of them stage.
__global__ void __launch_bounds__(F3T) k_filter3d_depth(int N, const float *__restrict__ pws, int C,
                                                        const float *__restrict__ cams, float *__restrict__ dmin,
                                                        unsigned int *__restrict__ ws) {
  __shared__ __align__(16) float cs[F3_CHUNK * pg::kCamRow];
  __shared__ float red[2][F3T / 32];
  const int tid = threadIdx.x;
  float dmax = 0.f, fxmax = 0.f;
  for (long long base = (long long)blockIdx.x * F3T; base < N; base += (long long)gridDim.x * F3T) {
    const long long i = base + tid;
    const bool valid = i < N;
    float pw[3] = {0.f, 0.f, 0.f};
    if (valid) {
      pw[0] = __ldg(pws + 3 * i); pw[1] = __ldg(pws + 3 * i + 1); pw[2] = __ldg(pws + 3 * i + 2);
    }
    float best = INFINITY;
    for (int c0 = 0; c0 < C; c0 += F3_CHUNK) {
      const int nc = min(F3_CHUNK, C - c0);
      __syncthreads();  // the previous chunk is no longer read
      for (int e = tid; e < nc * pg::kCamRow; e += F3T) {
        const float v = __ldg(cams + (size_t)c0 * pg::kCamRow + e);
        cs[e] = v;
        if (e % pg::kCamRow == 12) fxmax = fmaxf(fxmax, v);
      }
      __syncthreads();
      if (valid) {
        for (int k = 0; k < nc; k++) {
          float row[18];  // Rcw, tcw, fx, fy, cx, cy, W, H (the pad is not read)
          const float4 *r4 = reinterpret_cast<const float4 *>(cs + k * pg::kCamRow);
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const float4 x = r4[q];
            row[4 * q] = x.x; row[4 * q + 1] = x.y; row[4 * q + 2] = x.z; row[4 * q + 3] = x.w;
          }
          const float2 wh = *reinterpret_cast<const float2 *>(cs + k * pg::kCamRow + 16);
          row[16] = wh.x; row[17] = wh.y;
          float z;
          if (pg::filter3d_sees(row, pw, z)) best = fminf(best, z);
        }
      }
    }
    if (valid) {
      const float d = best < INFINITY ? best : 0.f;
      dmin[i] = d;
      dmax = fmaxf(dmax, d);
    }
  }
  const float m = block_max(dmax, red[0]);
  const float f = block_max(fxmax, red[1]);
  if (tid == 0) {
    if (m > 0.f) atomicMax(ws, __float_as_uint(m));
    if (f > 0.f) atomicMax(ws + 1, __float_as_uint(f));
  }
}

__global__ void __launch_bounds__(F3T) k_filter3d_finish(int N, float variance, const unsigned int *__restrict__ ws,
                                                         float *__restrict__ filter3d) {
  const long long i = (long long)blockIdx.x * F3T + threadIdx.x;
  if (i >= N) return;
  const float dmax = __uint_as_float(__ldg(ws)), fmax = __uint_as_float(__ldg(ws + 1));
  // no camera sees any Gaussian (or C == 0: no depth pass ran), or no camera has fx > 0 (fmax only
  // collects positive fx): all 0 rather than d / 0
  if (!(dmax > 0.f && fmax > 0.f)) {
    filter3d[i] = 0.f;
    return;
  }
  const float d = filter3d[i];
  filter3d[i] = pg::filter3d_value(d > 0.f ? d : dmax, fmax, variance);
}

__global__ void __launch_bounds__(F3T) k_filter3d_apply(int N, const float *scales, const float *alphas,
                                                        const float *__restrict__ filter3d, float *scales_f,
                                                        float *alphas_f) {
  const long long i = (long long)blockIdx.x * F3T + threadIdx.x;
  if (i >= N) return;
  const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
  const float a = alphas[i];
  float sf[3], t[3];
  const float c = pg::filter3d_apply(s, __ldg(filter3d + i), sf, t);
  scales_f[3 * i] = sf[0]; scales_f[3 * i + 1] = sf[1]; scales_f[3 * i + 2] = sf[2];
  alphas_f[i] = c * a;
}

// the gradient outputs may alias the inputs (dscales == dscales_f, dalphas == dalphas_f): each
// thread reads its row completely before it writes it
__global__ void __launch_bounds__(F3T) k_filter3d_bwd(int N, const float *__restrict__ scales,
                                                      const float *__restrict__ alphas,
                                                      const float *__restrict__ filter3d, const float *dscales_f,
                                                      const float *dalphas_f, float *dscales, float *dalphas) {
  const long long i = (long long)blockIdx.x * F3T + threadIdx.x;
  if (i >= N) return;
  const float s[3] = {__ldg(scales + 3 * i), __ldg(scales + 3 * i + 1), __ldg(scales + 3 * i + 2)};
  const float gsf[3] = {dscales_f[3 * i], dscales_f[3 * i + 1], dscales_f[3 * i + 2]};
  const float gaf = dalphas_f[i];
  float gs[3];
  const float ga = pg::filter3d_backward(s, __ldg(alphas + i), __ldg(filter3d + i), gsf, gaf, gs);
  dscales[3 * i] = gs[0]; dscales[3 * i + 1] = gs[1]; dscales[3 * i + 2] = gs[2];
  dalphas[i] = ga;
}

int launch_filter3d(int N, const float *pws, int C, const float *cams, float variance, float *filter3d,
                    unsigned int *ws, cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_FILTER3D, st);
  GSB_CUDA_TRY(cudaMemsetAsync(ws, 0, 2 * sizeof(unsigned int), st));
  const int nb = (N + F3T - 1) / F3T;
  if (C > 0) {
    // one wave of resident CTAs (more would only re-stage the camera table in a partial second wave)
    int dev = 0, sms = 0, per_sm = 0;
    GSB_CUDA_TRY(cudaGetDevice(&dev));
    GSB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    GSB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_filter3d_depth, F3T, 0));
    const int grid = min(nb, max(1, per_sm) * sms);
    k_filter3d_depth<<<grid, F3T, 0, st>>>(N, pws, C, cams, filter3d, ws);
  }
  k_filter3d_finish<<<nb, F3T, 0, st>>>(N, variance, ws, filter3d);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_filter3d_apply(int N, const float *scales, const float *alphas, const float *filter3d, float *scales_f,
                          float *alphas_f, cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_FILTER3D_APPLY, st);
  k_filter3d_apply<<<(N + F3T - 1) / F3T, F3T, 0, st>>>(N, scales, alphas, filter3d, scales_f, alphas_f);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_filter3d_bwd(int N, const float *scales, const float *alphas, const float *filter3d,
                        const float *dscales_f, const float *dalphas_f, float *dscales, float *dalphas,
                        cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_FILTER3D_BWD, st);
  k_filter3d_bwd<<<(N + F3T - 1) / F3T, F3T, 0, st>>>(N, scales, alphas, filter3d, dscales_f, dalphas_f, dscales,
                                                       dalphas);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
