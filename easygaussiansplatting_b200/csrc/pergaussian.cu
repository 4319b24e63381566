// Per-Gaussian stages: project, computeCov3D, computeCov2D, sh2Color, inverseCov2D.
//
// One thread per Gaussian, 128 Gaussians per CTA.  These kernels are pure HBM streaming
// (SURVEY 8d: 832 B/Gaussian with Jacobians), so the only thing that matters is that every
// global access is a full, aligned 128-bit transaction: array-of-struct inputs (float3
// means, 48-float SH rows) and outputs (up to 24 floats per Gaussian) are staged through a
// shared-memory tile with an odd row stride (bank-conflict free) and moved with coalesced
// float4 loads/stores.  Culled Gaussians write their zeros in-kernel, so outputs can be
// torch.empty (the reference pre-fills every output with torch::full, gausplat.cu:176-178).
//
// The values (means, covariances, colours, conics, radii) are computed by the stage functions of
// pg_fused_math.h, the same ones the fused kernels (fused.cu) compose; each kernel here adds only
// its shared-memory staging, the gate on the caller's depths and its Jacobian outputs, whose math
// follows docs/backward.md B.1-B.5.3 of the reference.  Each kernel cites the reference kernel it
// replaces.
#include "common.cuh"
#include "kernels.h"
#include "pg_fused_math.h"
#include "tile_io.cuh"

namespace gsb {


// ------------------------------------------------------------------ project
// replaces kernel.cu:553-617
__global__ void __launch_bounds__(PG) k_project(int N, const float *__restrict__ pws,
                                                const float *__restrict__ Rcw,
                                                const float *__restrict__ tcw, float fx,
                                                float fy, float cx, float cy,
                                                float *__restrict__ us, float *__restrict__ pcs,
                                                float *__restrict__ depths,
                                                float *__restrict__ du_dpcs) {
  __shared__ float sm[TileT<6>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  tile_fetch<3>(pws, base, nv, sm, tid);
  __syncthreads();
  float pc[3] = {0.f, 0.f, 0.f};
  bool keep = false;
  if (valid) {
    float R[9], t[3];
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = __ldg(Rcw + k);
#pragma unroll
    for (int k = 0; k < 3; k++) t[k] = __ldg(tcw + k);
    keep = pg::camera_point(R, t, ROW(3), pc);
  }
  float zi = 0.f, xf = 0.f, yf = 0.f, u[2] = {0.f, 0.f};
  if (keep) {
    zi = 1.0f / pc[2];
    xf = pc[0] * fx;  // for du/dpc; the same products project_mean forms
    yf = pc[1] * fy;
    pg::project_mean(pc, zi, fx, fy, cx, cy, u);
  }
  __syncthreads();
  {  // pcs
    float *r = ROW(3);
    r[0] = keep ? pc[0] : 0.f; r[1] = keep ? pc[1] : 0.f; r[2] = keep ? pc[2] : 0.f;
  }
  __syncthreads();
  tile_flush<3>(pcs, base, nv, sm, tid);
  __syncthreads();
  {  // us
    float *r = ROW(2);
    r[0] = u[0];
    r[1] = u[1];
  }
  __syncthreads();
  tile_flush<2>(us, base, nv, sm, tid);
  if (valid) depths[base + tid] = keep ? pc[2] : BAD_MARKER;
  if (du_dpcs != nullptr) {
    __syncthreads();
    float *r = ROW(6);
    float zi2 = zi * zi;
    r[0] = keep ? fx * zi : 0.f; r[1] = 0.f; r[2] = keep ? -xf * zi2 : 0.f;
    r[3] = 0.f; r[4] = keep ? fy * zi : 0.f; r[5] = keep ? -yf * zi2 : 0.f;
    __syncthreads();
    tile_flush<6>(du_dpcs, base, nv, sm, tid);
  }
}

// ------------------------------------------------------------------ computeCov3D
// replaces kernel.cu:326-423.  dSigma/dp = dM M^T + (dM M^T)^T.
__global__ void __launch_bounds__(PG) k_cov3d(int N, const float *__restrict__ rots,
                                              const float *__restrict__ scales,
                                              const float *__restrict__ depths,
                                              float *__restrict__ cov3ds,
                                              float *__restrict__ dcov3d_drots,
                                              float *__restrict__ dcov3d_dscales) {
  __shared__ float sm[TileT<24>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  tile_fetch<3>(scales, base, nv, sm, tid);
  __syncthreads();
  bool keep = false;
  float q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {0.f, 0.f, 0.f};
  if (valid) {
    keep = !(__ldg(depths + base + tid) < MIN_DEPTH);
    const float *r = ROW(3);
    s[0] = r[0]; s[1] = r[1]; s[2] = r[2];
    const float *rq = rots + (base + tid) * 4;
    if (aligned16(rots)) {
      float4 v = __ldg(reinterpret_cast<const float4 *>(rq));
      q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
    } else {
      q[0] = __ldg(rq); q[1] = __ldg(rq + 1); q[2] = __ldg(rq + 2); q[3] = __ldg(rq + 3);
    }
  }
  float R[9], M[9], S6[6];
  pg::cov3d(q, s, R, M, S6);
  __syncthreads();
  {
    float *o = ROW(6);
#pragma unroll
    for (int n = 0; n < 6; n++) o[n] = keep ? S6[n] : 0.f;
  }
  __syncthreads();
  tile_flush<6>(cov3ds, base, nv, sm, tid);
  if (dcov3d_drots == nullptr || dcov3d_dscales == nullptr) return;
  __syncthreads();
  {
    // dR/dq_p (times 2), rows as in pg::quat_to_R
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float dR[4][9] = {{0.f, -z, y, z, 0.f, -x, -y, x, 0.f},
                            {0.f, y, z, y, -2.f * x, -w, z, w, -2.f * x},
                            {-2.f * y, x, w, x, 0.f, z, -w, z, -2.f * y},
                            {-2.f * z, -w, x, w, -2.f * z, y, x, y, 0.f}};
    float *o = ROW(24);
#pragma unroll
    for (int p = 0; p < 4; p++) {
      float A[9];
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
          float a = 0.f;
#pragma unroll
          for (int k = 0; k < 3; k++) a = fmaf(2.f * dR[p][3 * i + k] * s[k], M[3 * j + k], a);
          A[3 * i + j] = a;
        }
      int n = 0;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = i; j < 3; j++) {
          o[4 * n + p] = keep ? A[3 * i + j] + A[3 * j + i] : 0.f;
          n++;
        }
    }
  }
  __syncthreads();
  tile_flush<24>(dcov3d_drots, base, nv, sm, tid);
  __syncthreads();
  {
    float *o = ROW(18);
#pragma unroll
    for (int p = 0; p < 3; p++) {
      int n = 0;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = i; j < 3; j++) {
          // A_ij = R_ip M_jp  (dM has only column p)
          float v = R[3 * i + p] * M[3 * j + p] + R[3 * j + p] * M[3 * i + p];
          o[3 * n + p] = keep ? v : 0.f;
          n++;
        }
    }
  }
  __syncthreads();
  tile_flush<18>(dcov3d_dscales, base, nv, sm, tid);
}

// ------------------------------------------------------------------ computeCov2D
// replaces kernel.cu:425-551.  tan_fov = width/(2 fx) computed by the caller as on the
// reference host side (gausplat.cu:225-226).
__global__ void __launch_bounds__(PG) k_cov2d(int N, const float *__restrict__ cov3ds,
                                              const float *__restrict__ pcs,
                                              const float *__restrict__ Rcw,
                                              const float *__restrict__ depths, float fx,
                                              float fy, float tan_fovx, float tan_fovy,
                                              float *__restrict__ cov2ds,
                                              float *__restrict__ dcov2d_dcov3ds,
                                              float *__restrict__ dcov2d_dpcs) {
  __shared__ float sm[TileT<18>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float c3[6] = {0, 0, 0, 0, 0, 0}, pc[3] = {0, 0, 1};
  tile_fetch<6>(cov3ds, base, nv, sm, tid);
  __syncthreads();
  if (valid) {
    const float *r = ROW(6);
#pragma unroll
    for (int k = 0; k < 6; k++) c3[k] = r[k];
  }
  __syncthreads();
  tile_fetch<3>(pcs, base, nv, sm, tid);
  __syncthreads();
  bool keep = false;
  if (valid) {
    keep = !(__ldg(depths + base + tid) < MIN_DEPTH);
    const float *r = ROW(3);
    pc[0] = r[0]; pc[1] = r[1]; pc[2] = r[2];
  }
  float R[9];
#pragma unroll
  for (int k = 0; k < 9; k++) R[k] = __ldg(Rcw + k);
  pg::Cov2d g;
  pg::cov2d(pc, keep, c3, R, fx, fy, tan_fovx, tan_fovy, g);
  const float *M = g.M, *MS = g.MS;
  const float x = g.xc, y = g.yc, zi2 = g.zi * g.zi, zi3 = zi2 * g.zi;
  __syncthreads();
  {
    float *o = ROW(3);
    o[0] = keep ? g.c2[0] : 0.f; o[1] = keep ? g.c2[1] : 0.f; o[2] = keep ? g.c2[2] : 0.f;
  }
  __syncthreads();
  tile_flush<3>(cov2ds, base, nv, sm, tid);
  if (dcov2d_dcov3ds == nullptr || dcov2d_dpcs == nullptr) return;
  __syncthreads();
  {
    float *o = ROW(18);
    // dSigma'_ab / dsigma_ij = M_ai M_bj + (i != j) M_aj M_bi
    const int AB[3][2] = {{0, 0}, {0, 1}, {1, 1}};
#pragma unroll
    for (int t = 0; t < 3; t++) {
      const int a = AB[t][0], b = AB[t][1];
      int n = 0;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = i; j < 3; j++) {
          float v = M[3 * a + i] * M[3 * b + j];
          if (i != j) v = fmaf(M[3 * a + j], M[3 * b + i], v);
          o[6 * t + n] = keep ? v : 0.f;
          n++;
        }
    }
  }
  __syncthreads();
  tile_flush<18>(dcov2d_dcov3ds, base, nv, sm, tid);
  __syncthreads();
  {
    float *o = ROW(9);
    // dJ/dx, dJ/dy, dJ/dz with the clamped x, y (kernel.cu:527-534)
    const float dJ[3][6] = {{0.f, 0.f, -fx * zi2, 0.f, 0.f, 0.f},
                            {0.f, 0.f, 0.f, 0.f, 0.f, -fy * zi2},
                            {-fx * zi2, 0.f, 2.f * fx * x * zi3, 0.f, -fy * zi2, 2.f * fy * y * zi3}};
#pragma unroll
    for (int p = 0; p < 3; p++) {
      float dM[6];
#pragma unroll
      for (int a = 0; a < 2; a++)
#pragma unroll
        for (int c = 0; c < 3; c++)
          dM[3 * a + c] = dJ[p][3 * a] * R[c] + dJ[p][3 * a + 1] * R[3 + c] + dJ[p][3 * a + 2] * R[6 + c];
      float d00 = 2.f * (dM[0] * MS[0] + dM[1] * MS[1] + dM[2] * MS[2]);
      float d01 = dM[0] * MS[3] + dM[1] * MS[4] + dM[2] * MS[5] + MS[0] * dM[3] + MS[1] * dM[4] + MS[2] * dM[5];
      float d11 = 2.f * (dM[3] * MS[3] + dM[4] * MS[4] + dM[5] * MS[5]);
      o[0 + p] = keep ? d00 : 0.f;
      o[3 + p] = keep ? d01 : 0.f;
      o[6 + p] = keep ? d11 : 0.f;
    }
  }
  __syncthreads();
  tile_flush<9>(dcov2d_dpcs, base, nv, sm, tid);
}

// ------------------------------------------------------------------ sh2Color
// replaces kernel.cu:619-807.  K3 = coefficients per channel (1,4,9,16).
template <int K3>
__global__ void __launch_bounds__(PG) k_sh2color(int N, const float *__restrict__ shs,
                                                 const float *__restrict__ pws,
                                                 const float *__restrict__ twc,
                                                 float *__restrict__ colors,
                                                 float *__restrict__ dcolor_dshs,
                                                 float *__restrict__ dcolor_dpws) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<9>::FLOATS ? TileT<KS>::FLOATS : TileT<9>::FLOATS;
  __shared__ float sm[SMF];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, tw[3] = {0.f, 0.f, 0.f};
  if (K3 > 1) {
    tile_fetch<3>(pws, base, nv, sm, tid);
    __syncthreads();
    if (valid) {
      const float *r = ROW(3);
#pragma unroll
      for (int k = 0; k < 3; k++) { pw[k] = r[k]; tw[k] = __ldg(twc + k); }
    }
    __syncthreads();
  }
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  const float *sh = ROW(KS);  // [coef][rgb]
  float d[3], r[3] = {0.f, 0.f, 0.f}, ninv = 1.f;
  if (K3 > 1) ninv = pg::view_dir<K3 == 16>(pw, tw, d, r);
  float Y[K3], dY[K3][3];
  pg::sh_basis<K3>(r[0], r[1], r[2], Y, dY);
  float col[3] = {0.5f, 0.5f, 0.5f};
  float dc_dr[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (valid) {
#pragma unroll
    for (int l = 0; l < K3; l++) {
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float v = sh[3 * l + c];
        col[c] = fmaf(Y[l], v, col[c]);
        if (l > 0) {
          dc_dr[3 * c + 0] = fmaf(v, dY[l][0], dc_dr[3 * c + 0]);
          dc_dr[3 * c + 1] = fmaf(v, dY[l][1], dc_dr[3 * c + 1]);
          dc_dr[3 * c + 2] = fmaf(v, dY[l][2], dc_dr[3 * c + 2]);
        }
      }
    }
  }
  __syncthreads();
  {
    float *o = ROW(3);
    o[0] = col[0]; o[1] = col[1]; o[2] = col[2];
  }
  __syncthreads();
  tile_flush<3>(colors, base, nv, sm, tid);
  if (dcolor_dshs == nullptr || dcolor_dpws == nullptr) return;
  __syncthreads();
  {
    float *o = ROW(K3);
#pragma unroll
    for (int l = 0; l < K3; l++) o[l] = Y[l];
  }
  __syncthreads();
  tile_flush<K3>(dcolor_dshs, base, nv, sm, tid);
  __syncthreads();
  {
    float *o = ROW(9);
    float dr[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (K3 > 1) {
      const float n3 = ninv * ninv * ninv;
#pragma unroll
      for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b = 0; b < 3; b++) dr[3 * a + b] = (a == b ? ninv : 0.f) - d[a] * d[b] * n3;
    }
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int b = 0; b < 3; b++)
        o[3 * c + b] = dc_dr[3 * c] * dr[b] + dc_dr[3 * c + 1] * dr[3 + b] + dc_dr[3 * c + 2] * dr[6 + b];
  }
  __syncthreads();
  tile_flush<9>(dcolor_dpws, base, nv, sm, tid);
}

// ------------------------------------------------------------------ inverseCov2D
// replaces kernel.cu:274-324
__global__ void __launch_bounds__(PG) k_inv_cov2d(int N, const float *__restrict__ cov2ds,
                                                  float *__restrict__ depths,
                                                  float *__restrict__ cinv2ds,
                                                  int32_t *__restrict__ areas,
                                                  float *__restrict__ dcinv2d_dcov2ds) {
  __shared__ float sm[TileT<9>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  tile_fetch<3>(cov2ds, base, nv, sm, tid);
  __syncthreads();
  bool keep = false;
  float c2[3] = {1.f, 0.f, 1.f}, di = 0.f, cn[3];
  if (valid) {
    keep = !(depths[base + tid] < MIN_DEPTH);
    const float *r = ROW(3);
    if (keep) {
      c2[0] = r[0]; c2[1] = r[1]; c2[2] = r[2];
      if (!pg::conic(c2, di, cn)) {
        depths[base + tid] = BAD_MARKER;
        keep = false;
      }
    }
  }
  __syncthreads();
  {
    float *o = ROW(3);
    o[0] = keep ? cn[0] : 0.f; o[1] = keep ? cn[1] : 0.f; o[2] = keep ? cn[2] : 0.f;
  }
  __syncthreads();
  tile_flush<3>(cinv2ds, base, nv, sm, tid);
  __syncthreads();
  {
    float *o = ROW(2);
    int area[2] = {0, 0};
    if (keep) pg::radius(c2, area);
    o[0] = __int_as_float(area[0]); o[1] = __int_as_float(area[1]);
  }
  __syncthreads();
  tile_flush<2>(reinterpret_cast<float *>(areas), base, nv, sm, tid);
  if (dcinv2d_dcov2ds == nullptr) return;
  __syncthreads();
  {
    float *o = ROW(9);
    const float a = c2[0], b = c2[1], c = c2[2], d2 = di * di;
    o[0] = keep ? -c * c * d2 : 0.f;      o[1] = keep ? 2.f * b * c * d2 : 0.f;       o[2] = keep ? di - a * c * d2 : 0.f;
    o[3] = keep ? b * c * d2 : 0.f;       o[4] = keep ? -di - 2.f * b * b * d2 : 0.f; o[5] = keep ? a * b * d2 : 0.f;
    o[6] = keep ? di - a * c * d2 : 0.f;  o[7] = keep ? 2.f * a * b * d2 : 0.f;       o[8] = keep ? -a * a * d2 : 0.f;
  }
  __syncthreads();
  tile_flush<9>(dcinv2d_dcov2ds, base, nv, sm, tid);
}

// ------------------------------------------------------------------ launchers
static inline int nblocks(int N) { return (N + PG - 1) / PG; }

int launch_project(int N, const float *pws, const float *Rcw, const float *tcw, float fx, float fy,
                   float cx, float cy, float *us, float *pcs, float *depths, float *du_dpcs,
                   cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_PROJECT, st);
  k_project<<<nblocks(N), PG, 0, st>>>(N, pws, Rcw, tcw, fx, fy, cx, cy, us, pcs, depths, du_dpcs);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}
int launch_cov3d(int N, const float *rots, const float *scales, const float *depths, float *cov3ds,
                 float *Jr, float *Js, cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_COV3D, st);
  k_cov3d<<<nblocks(N), PG, 0, st>>>(N, rots, scales, depths, cov3ds, Jr, Js);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}
int launch_cov2d(int N, const float *cov3ds, const float *pcs, const float *Rcw, const float *depths,
                 float fx, float fy, float width, float height, float *cov2ds, float *Jc, float *Jp,
                 cudaStream_t st) {
  if (N <= 0) return 0;
  const float tan_fovx = width / (2 * fx), tan_fovy = height / (2 * fy);  // gausplat.cu:225-226
  ProfScope ps(K_COV2D, st);
  k_cov2d<<<nblocks(N), PG, 0, st>>>(N, cov3ds, pcs, Rcw, depths, fx, fy, tan_fovx, tan_fovy, cov2ds,
                                     Jc, Jp);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}
int launch_sh2color(int N, int k3, const float *shs, const float *pws, const float *twc, float *colors,
                    float *Js, float *Jp, cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_SH2COLOR, st);
  switch (k3) {
    case 1: k_sh2color<1><<<nblocks(N), PG, 0, st>>>(N, shs, pws, twc, colors, Js, Jp); break;
    case 4: k_sh2color<4><<<nblocks(N), PG, 0, st>>>(N, shs, pws, twc, colors, Js, Jp); break;
    case 9: k_sh2color<9><<<nblocks(N), PG, 0, st>>>(N, shs, pws, twc, colors, Js, Jp); break;
    case 16: k_sh2color<16><<<nblocks(N), PG, 0, st>>>(N, shs, pws, twc, colors, Js, Jp); break;
    default: return set_arg_error("sh2color: shs.shape[1]/3 must be 1, 4, 9 or 16");
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}
int launch_inv_cov2d(int N, const float *cov2ds, float *depths, float *cinv2ds, int32_t *areas,
                     float *J, cudaStream_t st) {
  if (N <= 0) return 0;
  ProfScope ps(K_INVCOV, st);
  k_inv_cov2d<<<nblocks(N), PG, 0, st>>>(N, cov2ds, depths, cinv2ds, areas, J);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
