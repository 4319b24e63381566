// Fused per-Gaussian path (SURVEY 8f row N1): one forward kernel that does the work of
// project + computeCov3D + computeCov2D + sh2Color + inverseCov2D without materialising
// their 109 floats/Gaussian of Jacobians, and one backward kernel that recomputes the
// intermediates and applies the vector-Jacobian products in registers (pg_fused_math.h)
// instead of the reference's materialise -> torch.bmm chain (gsmodel.py:21-49,72-85).
// HBM traffic: forward 232 B in / 44 B out, backward 268 B in / 232 B out per Gaussian
// (SH degree 3).  The 192-byte SH rows go through the coalescing shared-memory tile of
// tile_io.cuh; the 3/4-float rows are read and written straight from registers, so all loads
// of a CTA are in flight at once.
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "pg_fused_math.h"
#include "tile_io.cuh"

namespace gsb {

__device__ __forceinline__ pg::Cam load_cam(const float *__restrict__ Rcw, const float *__restrict__ tcw,
                                            const float *__restrict__ twc, float fx, float fy, float cx,
                                            float cy, float tan_fovx, float tan_fovy) {
  pg::Cam c;
#pragma unroll
  for (int i = 0; i < 9; i++) c.R[i] = __ldg(Rcw + i);
#pragma unroll
  for (int i = 0; i < 3; i++) { c.t[i] = __ldg(tcw + i); c.twc[i] = __ldg(twc + i); }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy; c.tan_fovx = tan_fovx; c.tan_fovy = tan_fovy;
  return c;
}

#define ROWK(K) (sm + tid * TileT<K>::S)

// row o of the forward's per-Gaussian outputs (not the record, nor the effective opacity)
__device__ __forceinline__ void store_fwd_rows(float *__restrict__ us, float *__restrict__ cinv2ds,
                                               float *__restrict__ colors, int32_t *__restrict__ areas,
                                               float *__restrict__ depths, long long o, const float (&u)[2],
                                               const float (&conic)[3], const float (&col)[3], const int (&area)[2],
                                               float depth) {
  st_pair(us, o, u[0], u[1]);
  cinv2ds[3 * o] = conic[0]; cinv2ds[3 * o + 1] = conic[1]; cinv2ds[3 * o + 2] = conic[2];
  colors[3 * o] = col[0]; colors[3 * o + 1] = col[1]; colors[3 * o + 2] = col[2];
  st_pair(areas, o, area[0], area[1]);
  depths[o] = depth;
}

// row o of the 10 small gradient floats: direct strided stores (no staging, no barriers)
__device__ __forceinline__ void store_grad_rows(float *g_pws, float *g_scales, float *g_rots, long long o,
                                                const float (&gpw)[3], const float (&gs)[3], const float (&gq)[4]) {
  g_pws[3 * o] = gpw[0]; g_pws[3 * o + 1] = gpw[1]; g_pws[3 * o + 2] = gpw[2];
  g_scales[3 * o] = gs[0]; g_scales[3 * o + 1] = gs[1]; g_scales[3 * o + 2] = gs[2];
  if (aligned16(g_rots)) {
    reinterpret_cast<float4 *>(g_rots)[o] = make_float4(gq[0], gq[1], gq[2], gq[3]);
  } else {
    g_rots[4 * o] = gq[0]; g_rots[4 * o + 1] = gq[1]; g_rots[4 * o + 2] = gq[2]; g_rots[4 * o + 3] = gq[3];
  }
}

// the first step of the camera kernels' CTA sum of the NE camera terms (15 pose, 23 pose +
// intrinsics): the warp's sum, by shuffles, into lane 0's `row`
template <int NE>
__device__ __forceinline__ void warp_sum_pose(float (&gcam)[NE], float *row) {
#pragma unroll
  for (int e = 0; e < NE; e++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gcam[e] += __shfl_down_sync(0xffffffffu, gcam[e], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int e = 0; e < NE; e++) row[e] = gcam[e];
  }
}

__device__ __forceinline__ void load_small_rows(const float *__restrict__ pws, const float *__restrict__ scales,
                                                const float *__restrict__ rots, long long i, bool valid,
                                                float (&pw)[3], float (&s)[3], float (&q)[4]) {
  if (!valid) return;
  pw[0] = __ldg(pws + 3 * i); pw[1] = __ldg(pws + 3 * i + 1); pw[2] = __ldg(pws + 3 * i + 2);
  s[0] = __ldg(scales + 3 * i); s[1] = __ldg(scales + 3 * i + 1); s[2] = __ldg(scales + 3 * i + 2);
  if (aligned16(rots)) {
    const float4 r = __ldg(reinterpret_cast<const float4 *>(rots) + i);
    q[0] = r.x; q[1] = r.y; q[2] = r.z; q[3] = r.w;
  } else {
    q[0] = __ldg(rots + 4 * i); q[1] = __ldg(rots + 4 * i + 1); q[2] = __ldg(rots + 4 * i + 2); q[3] = __ldg(rots + 4 * i + 3);
  }
}

// AA = antialiasing (pg::aa_scale): alphas is read, alpha_eff = rho alpha goes to alphas_eff[N]
// and into the record's alpha word (so its culling threshold follows); every other output is the
// non-AA kernel's.
// MODEL = pg::CamModel; lk = FISHEYE's k1..k4 or OPENCV's k1, k2, p1, p2 (unread by the other models)
template <int K3, bool AA, int MODEL>
__global__ void __launch_bounds__(PG) k_preprocess_fwd(
    int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const float *__restrict__ Rcw, const float *__restrict__ tcw,
    const float *__restrict__ twc, float fx, float fy, float cx, float cy, float tan_fovx, float tan_fovy,
    float *__restrict__ us, float *__restrict__ cinv2ds, float *__restrict__ colors,
    float *__restrict__ depths, int32_t *__restrict__ areas, const float *__restrict__ alphas,
    Rec *__restrict__ recs, float *__restrict__ alphas_eff, float4 lk) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  __shared__ float sm[SMF];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  pg::Cam cam = load_cam(Rcw, tcw, twc, fx, fy, cx, cy, tan_fovx, tan_fovy);
  if (MODEL == pg::FISHEYE || MODEL == pg::OPENCV) { cam.k[0] = lk.x; cam.k[1] = lk.y; cam.k[2] = lk.z; cam.k[3] = lk.w; }
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  // The 10 floats of position / scale / rotation go straight from global memory to registers
  // (a warp's strided loads use every byte of the sectors they touch; L1 serves the repeats) and
  // are in flight together with the SH tile -- one exposed memory latency per CTA instead of
  // one per array.
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  float u[2] = {0.f, 0.f}, conic[3] = {0.f, 0.f, 0.f}, col[3] = {0.f, 0.f, 0.f}, depth = -1.f;
  int area[2] = {0, 0};
  if (valid) {
    const float rho = pg::forward_one<K3, AA, MODEL>(pw, q, s, ROWK(KS), cam, u, conic, col, &depth, area);
    const long long i = base + tid;
    store_fwd_rows(us, cinv2ds, colors, areas, depths, i, u, conic, col, area, depth);
    float al = 0.f;
    if (AA) {
      al = rho * __ldg(alphas + i);
      alphas_eff[i] = al;
    }
    // the rasterizers' per-Gaussian record, straight from registers (saves the k_pack pass)
    if (recs != nullptr)
      recs[i] = build_record(u[0], u[1], conic[0], conic[1], conic[2], AA ? al : __ldg(alphas + i), col[0], col[1],
                             col[2], depth, (int)i);
  }
}

// PUSH = the multi-GPU variant (SURVEY 8e): instead of writing the gradient tile to local
// buffers, the CTA stores it straight into the staging slot `rank` of the GPU that owns this
// tile's Gaussians (peer memory over NVLink -- posted stores, so the transfer of tile t
// overlaps the math of tile t+1), together with dL/dalpha from the rasterizer backward.  The
// last CTA to finish raises this rank's arrival flag on every peer; k_grad_reduce_bcast
// (comm.cu) then sums the slots of the rows it owns and broadcasts the result.
// MOM = the upstream gradients come as the rasterizer backward's raw moment rows [N,9] (see
// raster_bwd.cu): the conversion k_finalize_grads would do (dL/du = -(A Sx + B Sy, B Sx + C Sy),
// dL/dconic = (-Sxx/2, -Sxy, -Syy/2), dL/dcolor, dL/dalpha) happens here in registers, dL/du and
// dL/dalpha are still written out (the caller's densification statistics / alpha gradient), and
// the separate finalize pass with its 36 B/Gaussian round trip disappears.
// DEPTH = the RGB-D rasterizer's dL/dz[N] (g_depths) is a fourth upstream gradient (not with PUSH).
// POSE = the camera gradient instead of the per-Gaussian ones (not with PUSH): everything is read
// as before, the CTA sums its threads' 15 contributions (pg::backward_one) -- warp shuffles, then
// the 4 warps through shared memory, fp32 -- into row blockIdx.x of pose_part[nb][16] (summed by
// k_pose_reduce), and no per-Gaussian gradient (nor, with MOM, dL/du or dL/dalpha) is written, nor
// the SH tile flushed.  A caller that wants both runs the non-POSE form as well: the compiler
// fuses multiply-adds differently in a kernel that also carries the camera terms, and the
// per-Gaussian gradients have to be the same bits with and without the pose.
// AA = antialiasing (only with MOM, not with PUSH): the moment rows' dL/dalpha is dL/dalpha_eff of
// the forward's alpha_eff = rho alpha; alphas (raw, 4 B/Gaussian) is read, dL/dalpha = rho m[5]
// is written and alpha m[5] drho feeds the geometry (and camera) gradients (pg::backward_one).
// MODEL, lk: as for k_preprocess_fwd (ORTHO, FISHEYE and OPENCV only with MOM, not with PUSH).
template <int K3, bool PUSH, bool MOM, bool DEPTH, bool POSE, bool AA, int MODEL>
__global__ void __launch_bounds__(PG) k_preprocess_bwd(
    int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const float *__restrict__ Rcw, const float *__restrict__ tcw,
    const float *__restrict__ twc, float fx, float fy, float cx, float cy, float tan_fovx, float tan_fovy,
    const float *__restrict__ g_us, const float *__restrict__ g_cinv2ds, const float *__restrict__ g_colors,
    float *__restrict__ g_pws, float *__restrict__ g_shs, float *__restrict__ g_scales,
    float *__restrict__ g_rots, GradPush gp, MomentsIn mi, const float *__restrict__ g_depths,
    float *__restrict__ pose_part, const float *__restrict__ alphas, float4 lk) {
  static_assert(!AA || (MOM && !PUSH), "antialiasing takes the moment rows and no exchange");
  static_assert(MODEL == pg::PINHOLE || (MOM && !PUSH), "camera models take the moment rows and no exchange");
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  __shared__ float sm[SMF];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  pg::Cam cam = load_cam(Rcw, tcw, twc, fx, fy, cx, cy, tan_fovx, tan_fovy);
  if (MODEL == pg::FISHEYE || MODEL == pg::OPENCV) { cam.k[0] = lk.x; cam.k[1] = lk.y; cam.k[2] = lk.z; cam.k[3] = lk.w; }
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  float gu[2] = {0.f, 0.f}, gci[3] = {0.f, 0.f, 0.f}, gcol[3] = {0.f, 0.f, 0.f};
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);  // see k_preprocess_fwd
  float galpha = 0.f, al = 0.f;
  if (MOM) {
    if (valid) {
      const long long i = base + tid;
      float m[9];
#pragma unroll
      for (int k = 0; k < 9; k++) m[k] = __ldg(mi.moments + 9 * i + k);
      const float A = __ldg(mi.cinv2ds + 3 * i), B = __ldg(mi.cinv2ds + 3 * i + 1), C = __ldg(mi.cinv2ds + 3 * i + 2);
      // untouched Gaussians stay exactly 0 even if their conic is inf/NaN (k_finalize_grads)
      const bool none = (m[0] == 0.f) && (m[1] == 0.f);
      gu[0] = none ? 0.f : -(A * m[0] + B * m[1]);
      gu[1] = none ? 0.f : -(B * m[0] + C * m[1]);
      gci[0] = -0.5f * m[2]; gci[1] = -m[3]; gci[2] = -0.5f * m[4];
      gcol[0] = m[6]; gcol[1] = m[7]; gcol[2] = m[8];
      galpha = m[5];
      if (AA) al = __ldg(alphas + i);  // in flight with the moment row
      if (!POSE) st_pair(mi.dus_out, i, gu[0], gu[1]);
      if (!POSE && !AA && mi.dalphas_out != nullptr) mi.dalphas_out[i] = galpha;  // AA: after the math
    }
  } else if (valid) {
    const long long i = base + tid;
    const float2 g2 = ld_pair(g_us, i);
    gu[0] = g2.x; gu[1] = g2.y;
    gci[0] = __ldg(g_cinv2ds + 3 * i); gci[1] = __ldg(g_cinv2ds + 3 * i + 1); gci[2] = __ldg(g_cinv2ds + 3 * i + 2);
    gcol[0] = __ldg(g_colors + 3 * i); gcol[1] = __ldg(g_colors + 3 * i + 1); gcol[2] = __ldg(g_colors + 3 * i + 2);
  }
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  float gpw[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f};
  if (POSE) {
    float gcam[15];
#pragma unroll
    for (int e = 0; e < 15; e++) gcam[e] = 0.f;
    if (valid) {
      const float gz = DEPTH ? __ldg(g_depths + base + tid) : 0.f;
      float xpw[3], xq[4], xs[3], xsh[KS];  // the per-Gaussian outputs: not written by this form
      pg::backward_one<K3, DEPTH, true, AA, MODEL>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, xpw, xq, xs, xsh, gz, gcam,
                                            galpha, al);
    }
    __shared__ float red[PG / 32][16];
    warp_sum_pose(gcam, red[tid >> 5]);
    __syncthreads();
    if (tid < 16) {
      float v = 0.f;
      if (tid < 15) {
#pragma unroll
        for (int w = 0; w < PG / 32; w++) v += red[w][tid];
      }
      pose_part[(size_t)blockIdx.x * 16 + tid] = v;
    }
    return;  // nothing per Gaussian leaves the CTA
  }
  // dL/dsh overwrites the thread's own SH row in place, then the tile is flushed
  float gal = galpha;
  if (DEPTH) {
    const float gz = valid ? __ldg(g_depths + base + tid) : 0.f;
    if (valid)
      gal = pg::backward_one<K3, true, false, AA, MODEL>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, gpw, gq, gs, ROWK(KS), gz,
                                                  nullptr, galpha, al);
  } else if (valid) {
    gal = pg::backward_one<K3, false, false, AA, MODEL>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, gpw, gq, gs, ROWK(KS), 0.f,
                                                 nullptr, galpha, al);
  }
  if (AA && valid && mi.dalphas_out != nullptr) mi.dalphas_out[base + tid] = gal;
  __syncthreads();
  long long drow = base;
  if (PUSH) {  // destination = slot `rank` on the owner of this tile, rows relative to its range
    // tiles are dealt round-robin over the ranks, so peer and local stores interleave for the
    // whole kernel instead of one NVLink burst at one end of it
    const int owner = (int)(blockIdx.x % gp.world);
    float *sb = gp.slot[owner];
    drow = (long long)(blockIdx.x / gp.world) * PG;
    g_shs = sb;
    g_rots = sb + gp.off_rots;
    g_pws = sb + gp.off_pws;
    g_scales = sb + gp.off_scales;
    if (valid) (sb + gp.off_alphas)[drow + tid] = MOM ? galpha : __ldg(gp.g_alphas + base + tid);
  }
  // g_shs == nullptr: the caller re-expands dL/dsh = sum over views of Y(dir_v) (x) dL/dcolor_v itself
  // (multi-view data parallel: 12 B/view travel instead of the 192 B row, k_sh_expand below)
  if (g_shs != nullptr) tile_flush<KS>(g_shs, drow, nv, sm, tid);
  if (valid) store_grad_rows(g_pws, g_scales, g_rots, drow + tid, gpw, gs, gq);
  if (PUSH) {
    __threadfence_system();  // this thread's peer stores are ordered before the flag below
    __syncthreads();
    if (tid == 0) {
      const unsigned done = atomicAdd(gp.counter, 1u);
      if (done == gridDim.x - 1) {  // last tile of this rank
        *gp.counter = 0;            // re-armed for the next launch (stream-ordered)
        __threadfence_system();
        for (int p = 0; p < gp.world; p++) st_release_sys(gp.flags[p] + gp.rank, gp.epoch);
      }
    }
  }
}

// The camera gradient: the nrows partial rows of NE + 1 floats (NE = 15: k_preprocess_bwd<..., POSE>,
// 23: k_preprocess_bwd_intrinsics) summed in fp64 by one CTA in a fixed order (thread t takes rows t,
// t + PR, ...; then a fixed shuffle tree and the warps in index order), so the result is the same bits
// on every run.  Columns 0-14 go to gcam, 15-22 to gint.  nrows == 0 writes zeros.
constexpr int PR = 512;
template <int NE>
__device__ __forceinline__ void pose_reduce(int nrows, const float *__restrict__ part, float *__restrict__ gcam,
                                            float *__restrict__ gint) {
  constexpr int RW = NE + 1;  // the row width: 16 or 24 floats, whole float4s
  const int tid = threadIdx.x;
  double acc[NE];
#pragma unroll
  for (int e = 0; e < NE; e++) acc[e] = 0.0;
  for (int r = tid; r < nrows; r += PR) {
    const float4 *row = reinterpret_cast<const float4 *>(part + (size_t)r * RW);
    float v[RW];
#pragma unroll
    for (int c = 0; c < RW / 4; c++) {
      const float4 x = __ldg(row + c);
      v[4 * c] = x.x; v[4 * c + 1] = x.y; v[4 * c + 2] = x.z; v[4 * c + 3] = x.w;
    }
#pragma unroll
    for (int e = 0; e < NE; e++) acc[e] += (double)v[e];
  }
#pragma unroll
  for (int e = 0; e < NE; e++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[e] += __shfl_down_sync(0xffffffffu, acc[e], o);
  }
  __shared__ double red[PR / 32][NE];
  if ((tid & 31) == 0) {
#pragma unroll
    for (int e = 0; e < NE; e++) red[tid >> 5][e] = acc[e];
  }
  __syncthreads();
  if (tid < NE) {
    double t = 0.0;
    for (int w = 0; w < PR / 32; w++) t += red[w][tid];
    if (tid < 15)
      gcam[tid] = (float)t;
    else
      gint[tid - 15] = (float)t;
  }
}
__global__ void __launch_bounds__(PR) k_pose_reduce(int nrows, const float *__restrict__ part,
                                                    float *__restrict__ gcam) {
  pose_reduce<15>(nrows, part, gcam, nullptr);
}
// the batch's: CTA c sums camera c's nrows rows of part[C][nrows][16] into gcam[c][15]
__global__ void __launch_bounds__(PR) k_pose_reduce_batch(int nrows, const float *__restrict__ part,
                                                          float *__restrict__ gcam) {
  pose_reduce<15>(nrows, part + (size_t)blockIdx.x * nrows * 16, gcam + (size_t)blockIdx.x * 15, nullptr);
}
// pose + intrinsics (DESIGN 3.23), one camera or a batch: CTA c sums camera c's nrows rows of
// part[C][nrows][24] into gcam[c][15] and gint[c][8]
__global__ void __launch_bounds__(PR) k_intrinsics_reduce(int nrows, const float *__restrict__ part,
                                                          float *__restrict__ gcam, float *__restrict__ gint) {
  pose_reduce<23>(nrows, part + (size_t)blockIdx.x * nrows * 24, gcam + (size_t)blockIdx.x * 15,
                  gint + (size_t)blockIdx.x * 8);
}

// dL/dsh of one Gaussian summed over V views from the views' dL/dcolor:
//   colour = 0.5 + sum_l Y_l(dir) sh_l is linear in sh and never clamped (kernel.cu:735-774), so
//   dL/dsh[l][c] = sum_v Y_l(dir_v) dL/dcolor_v[c]   with dir_v = (pw - twc_v) / |pw - twc_v|,
// the same Y as backward_one evaluates (for V = 1 the result equals the dL/dsh row the per-Gaussian
// backward writes up to the compiler's FMA contraction of the basis polynomials).  Multi-view data parallel
// training exchanges the 12-byte dL/dcolor per view instead of the 192-byte dL/dsh row and
// expands on every rank (parallel.MultiViewStep).  Views are summed in index order.
template <int K3>
__global__ void __launch_bounds__(PG) k_sh_expand(int N, int V, const float *__restrict__ pws,
                                                  const float *__restrict__ twcs, const float *__restrict__ gcols,
                                                  float *__restrict__ g_shs) {
  constexpr int KS = 3 * K3;
  __shared__ float sm[TileT<KS>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float acc[KS];
#pragma unroll
  for (int i = 0; i < KS; i++) acc[i] = 0.f;
  if (valid) {
    const long long i = base + tid;
    const float pw[3] = {__ldg(pws + 3 * i), __ldg(pws + 3 * i + 1), __ldg(pws + 3 * i + 2)};
    for (int v = 0; v < V; v++) {
      const float *gc = gcols + ((size_t)v * N + i) * 3;
      const float g0 = __ldg(gc), g1 = __ldg(gc + 1), g2 = __ldg(gc + 2);
      float Y[K3], dY[K3][3];
      float d[3], r[3] = {0.f, 0.f, 0.f};
      if (K3 > 1) {
        const float twc[3] = {__ldg(twcs + 3 * v), __ldg(twcs + 3 * v + 1), __ldg(twcs + 3 * v + 2)};
        pg::view_dir(pw, twc, d, r);
      }
      pg::sh_basis<K3>(r[0], r[1], r[2], Y, dY);
#pragma unroll
      for (int l = 0; l < K3; l++) {
        acc[3 * l] += g0 * Y[l];
        acc[3 * l + 1] += g1 * Y[l];
        acc[3 * l + 2] += g2 * Y[l];
      }
    }
    float *row = ROWK(KS);
#pragma unroll
    for (int e = 0; e < KS; e++) row[e] = acc[e];
  }
  __syncthreads();
  tile_flush<KS>(g_shs, base, nv, sm, tid);
}

// ---- batched per-Gaussian path (DESIGN 3.21): C cameras in one launch.  A thread loads its
// Gaussian's rows once (the 10 small floats to registers, the SH row through the shared tile) and
// runs pg::forward_one / pg::backward_one once per camera, camera c from poses[c] (Rcw 9, tcw 3,
// twc 3 floats, device memory) and cams (its intrinsics, kernel parameter memory).  Outputs of
// camera c go to rows c N + n of the [C, N, ...] arrays; record c N + n carries id c N + n.
__device__ __forceinline__ pg::Cam batch_cam(const float *__restrict__ poses, const BatchCams &bc, int c, bool lens) {
  const float *p = poses + 15 * c;
  const float4 f = bc.f[c];
  const float2 tf = bc.tf[c];
  pg::Cam cam = load_cam(p, p + 9, p + 12, f.x, f.y, f.z, f.w, tf.x, tf.y);
  if (lens) {
    const float4 lk = bc.k[c];
    cam.k[0] = lk.x; cam.k[1] = lk.y; cam.k[2] = lk.z; cam.k[3] = lk.w;
  }
  return cam;
}

// the forward: k_preprocess_fwd's outputs per camera (alphas and records required)
template <int K3, bool AA, int MODEL>
__global__ void __launch_bounds__(PG) k_preprocess_fwd_batch(
    int C, int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const float *__restrict__ poses, const __grid_constant__ BatchCams bc,
    float *__restrict__ us, float *__restrict__ cinv2ds, float *__restrict__ colors, float *__restrict__ depths,
    int32_t *__restrict__ areas, const float *__restrict__ alphas, Rec *__restrict__ recs,
    float *__restrict__ alphas_eff) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  __shared__ float sm[SMF];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  if (!valid) return;
  const long long i = base + tid;
  const float alpha = __ldg(alphas + i);
  for (int c = 0; c < C; c++) {
    const pg::Cam cam = batch_cam(poses, bc, c, MODEL == pg::FISHEYE || MODEL == pg::OPENCV);
    float u[2] = {0.f, 0.f}, conic[3] = {0.f, 0.f, 0.f}, col[3] = {0.f, 0.f, 0.f}, depth = -1.f;
    int area[2] = {0, 0};
    const float rho = pg::forward_one<K3, AA, MODEL>(pw, q, s, ROWK(KS), cam, u, conic, col, &depth, area);
    const long long o = (long long)c * N + i;
    store_fwd_rows(us, cinv2ds, colors, areas, depths, o, u, conic, col, area, depth);
    float al = alpha;
    if (AA) {
      al = rho * alpha;
      alphas_eff[o] = al;
    }
    recs[o] = build_record(u[0], u[1], conic[0], conic[1], conic[2], al, col[0], col[1], col[2], depth, (int)o);
  }
}

// the backward from the C moment rows [C, N, 9] (and dL/dz [C, N] with DEPTH): the C contributions
// to each per-Gaussian gradient, dL/dsh included, are summed in fp32 registers in camera order; one
// gradient row per Gaussian, dL/du per camera [C, N, 2] and the summed dL/dalpha [N].  AA: as
// k_preprocess_bwd's (dL/dalpha = sum_c rho_c m_c[5]).
template <int K3, bool DEPTH, bool AA, int MODEL>
__global__ void __launch_bounds__(PG) k_preprocess_bwd_batch(
    int C, int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const float *__restrict__ poses, const __grid_constant__ BatchCams bc,
    const float *__restrict__ moments, const float *__restrict__ cinv2ds, const float *__restrict__ g_depths,
    const float *__restrict__ alphas, float *__restrict__ dus_out, float *__restrict__ dalphas_out,
    float *__restrict__ g_pws, float *__restrict__ g_shs, float *__restrict__ g_scales, float *__restrict__ g_rots) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  __shared__ float sm[SMF];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  float gpw[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gsh[KS], gal = 0.f;
#pragma unroll
  for (int e = 0; e < KS; e++) gsh[e] = 0.f;
  const long long i = base + tid;
  if (valid) {
    const float al = AA ? __ldg(alphas + i) : 0.f;
    for (int c = 0; c < C; c++) {
      const long long o = (long long)c * N + i;
      float m[9];
#pragma unroll
      for (int k = 0; k < 9; k++) m[k] = __ldg(moments + 9 * o + k);
      const float A = __ldg(cinv2ds + 3 * o), B = __ldg(cinv2ds + 3 * o + 1), Cc = __ldg(cinv2ds + 3 * o + 2);
      const bool none = (m[0] == 0.f) && (m[1] == 0.f);  // as k_preprocess_bwd's MOM form
      const float gu[2] = {none ? 0.f : -(A * m[0] + B * m[1]), none ? 0.f : -(B * m[0] + Cc * m[1])};
      const float gci[3] = {-0.5f * m[2], -m[3], -0.5f * m[4]}, gcol[3] = {m[6], m[7], m[8]};
      st_pair(dus_out, o, gu[0], gu[1]);
      const float gz = DEPTH ? __ldg(g_depths + o) : 0.f;
      const pg::Cam cam = batch_cam(poses, bc, c, MODEL == pg::FISHEYE || MODEL == pg::OPENCV);
      float xpw[3], xq[4], xs[3], xsh[KS];
      gal += pg::backward_one<K3, DEPTH, false, AA, MODEL>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, xpw, xq, xs, xsh,
                                                           gz, nullptr, m[5], al);
#pragma unroll
      for (int e = 0; e < 3; e++) { gpw[e] += xpw[e]; gs[e] += xs[e]; }
#pragma unroll
      for (int e = 0; e < 4; e++) gq[e] += xq[e];
#pragma unroll
      for (int e = 0; e < KS; e++) gsh[e] += xsh[e];
    }
    // dL/dsh replaces the thread's own SH row (no other thread reads it before the barrier)
    float *row = ROWK(KS);
#pragma unroll
    for (int e = 0; e < KS; e++) row[e] = gsh[e];
    dalphas_out[i] = gal;
  }
  __syncthreads();
  tile_flush<KS>(g_shs, base, nv, sm, tid);
  if (valid) store_grad_rows(g_pws, g_scales, g_rots, i, gpw, gs, gq);
}

// The camera gradients of the batch (DESIGN 3.22): k_preprocess_bwd_batch's reads and
// k_preprocess_bwd<..., POSE>'s math per camera.  Camera c's 15 contributions are summed over the
// CTA's Gaussians with that kernel's tree (warp shuffles, then the 4 warps in index order, fp32):
// each warp's sum waits in red[c][warp] (dynamic shared memory, C x 256 B) and one barrier at the end
// hands the C rows to the CTA, which writes row part[c][blockIdx.x][16] (summed by
// k_pose_reduce_batch).  Nothing per Gaussian is written.  Every thread runs the camera loop (the
// shuffles take the whole warp); a thread past N contributes zeros.  (The minimum of 1 CTA per SM in
// the launch bounds lets ptxas keep the values that live across the lens's and the divisions'
// slow-path calls in registers: without it a third of the instantiations save 1-3 of them on the stack.
// They use 51-96 registers either way.)
template <int K3, bool DEPTH, bool AA, int MODEL>
__global__ void __launch_bounds__(PG, 1) k_preprocess_bwd_batch_pose(
    int C, int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const float *__restrict__ poses, const __grid_constant__ BatchCams bc,
    const float *__restrict__ moments, const float *__restrict__ cinv2ds, const float *__restrict__ g_depths,
    const float *__restrict__ alphas, float *__restrict__ part) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  __shared__ float sm[SMF];
  extern __shared__ float red[];  // [C][PG / 32][16]
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  const long long i = base + tid;
  const float al = AA && valid ? __ldg(alphas + i) : 0.f;
  for (int c = 0; c < C; c++) {
    float gcam[15];
#pragma unroll
    for (int e = 0; e < 15; e++) gcam[e] = 0.f;
    if (valid) {
      const long long o = (long long)c * N + i;
      float m[9];
#pragma unroll
      for (int k = 0; k < 9; k++) m[k] = __ldg(moments + 9 * o + k);
      const float A = __ldg(cinv2ds + 3 * o), B = __ldg(cinv2ds + 3 * o + 1), Cc = __ldg(cinv2ds + 3 * o + 2);
      const bool none = (m[0] == 0.f) && (m[1] == 0.f);  // as k_preprocess_bwd's MOM form
      const float gu[2] = {none ? 0.f : -(A * m[0] + B * m[1]), none ? 0.f : -(B * m[0] + Cc * m[1])};
      const float gci[3] = {-0.5f * m[2], -m[3], -0.5f * m[4]}, gcol[3] = {m[6], m[7], m[8]};
      const float gz = DEPTH ? __ldg(g_depths + o) : 0.f;
      const pg::Cam cam = batch_cam(poses, bc, c, MODEL == pg::FISHEYE || MODEL == pg::OPENCV);
      float xpw[3], xq[4], xs[3], xsh[KS];  // the per-Gaussian outputs: not written by this form
      pg::backward_one<K3, DEPTH, true, AA, MODEL>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, xpw, xq, xs, xsh, gz, gcam,
                                                   m[5], al);
    }
    warp_sum_pose(gcam, red + ((size_t)c * (PG / 32) + (tid >> 5)) * 16);
  }
  __syncthreads();
  for (int k = tid; k < C * 16; k += PG) {
    const int c = k >> 4, e = k & 15;
    float v = 0.f;
    if (e < 15) {
#pragma unroll
      for (int w = 0; w < PG / 32; w++) v += red[((size_t)c * (PG / 32) + w) * 16 + e];
    }
    part[((size_t)c * gridDim.x + blockIdx.x) * 16 + e] = v;
  }
}

// The camera gradients with the intrinsics' (DESIGN 3.23), for one camera (C = 1) or a batch:
// k_preprocess_bwd_batch_pose's reads, math and CTA tree with 23 terms per camera
// (pg::backward_one<..., POSE, ..., INTR>) -- dL/dRcw, dL/dtcw, dL/dtwc, then dL/d(fx, fy, cx, cy,
// k[4]) -- into part[c][blockIdx.x][24] (summed by k_intrinsics_reduce).  Camera c's pose is read
// from pp (Rcw, tcw, twc + c stride: the single camera's three arrays, or the batch's [C, 15] rows), its
// intrinsics, lens and tan_fov from bc.  red: [C][PG / 32][24] floats of dynamic shared memory.
// Nothing per Gaussian is written.
struct PosePtrs {
  const float *Rcw, *tcw, *twc;
  int stride;  // floats from one camera's pose to the next
};
template <int K3, bool DEPTH, bool AA, int MODEL>
__global__ void __launch_bounds__(PG, 1) k_preprocess_bwd_intrinsics(
    int C, int N, const float *__restrict__ pws, const float *__restrict__ rots, const float *__restrict__ scales,
    const float *__restrict__ shs, const PosePtrs pp, const __grid_constant__ BatchCams bc,
    const float *__restrict__ moments, const float *__restrict__ cinv2ds, const float *__restrict__ g_depths,
    const float *__restrict__ alphas, float *__restrict__ part) {
  constexpr int KS = 3 * K3;
  constexpr int SMF = TileT<KS>::FLOATS > TileT<4>::FLOATS ? TileT<KS>::FLOATS : TileT<4>::FLOATS;
  constexpr bool LENS = MODEL == pg::FISHEYE || MODEL == pg::OPENCV;
  __shared__ float sm[SMF];
  extern __shared__ float red[];  // [C][PG / 32][24]
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  load_small_rows(pws, scales, rots, base + tid, valid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  const long long i = base + tid;
  const float al = AA && valid ? __ldg(alphas + i) : 0.f;
  for (int c = 0; c < C; c++) {
    float gcam[23];
#pragma unroll
    for (int e = 0; e < 23; e++) gcam[e] = 0.f;
    if (valid) {
      const long long o = (long long)c * N + i;
      float m[9];
#pragma unroll
      for (int k = 0; k < 9; k++) m[k] = __ldg(moments + 9 * o + k);
      const float A = __ldg(cinv2ds + 3 * o), B = __ldg(cinv2ds + 3 * o + 1), Cc = __ldg(cinv2ds + 3 * o + 2);
      const bool none = (m[0] == 0.f) && (m[1] == 0.f);  // as k_preprocess_bwd's MOM form
      const float gu[2] = {none ? 0.f : -(A * m[0] + B * m[1]), none ? 0.f : -(B * m[0] + Cc * m[1])};
      const float gci[3] = {-0.5f * m[2], -m[3], -0.5f * m[4]}, gcol[3] = {m[6], m[7], m[8]};
      const float gz = DEPTH ? __ldg(g_depths + o) : 0.f;
      const size_t po = (size_t)c * pp.stride;
      const float4 f = bc.f[c];
      const float2 tf = bc.tf[c];
      pg::Cam cam = load_cam(pp.Rcw + po, pp.tcw + po, pp.twc + po, f.x, f.y, f.z, f.w, tf.x, tf.y);
      if (LENS) {
        const float4 lk = bc.k[c];
        cam.k[0] = lk.x; cam.k[1] = lk.y; cam.k[2] = lk.z; cam.k[3] = lk.w;
      }
      float xpw[3], xq[4], xs[3], xsh[KS];  // the per-Gaussian outputs: not written by this form
      pg::backward_one<K3, DEPTH, true, AA, MODEL, true>(pw, q, s, ROWK(KS), cam, gu, gci, gcol, xpw, xq, xs, xsh,
                                                         gz, gcam, m[5], al);
    }
    warp_sum_pose(gcam, red + ((size_t)c * (PG / 32) + (tid >> 5)) * 24);
  }
  __syncthreads();
  for (int k = tid; k < C * 24; k += PG) {
    const int c = k / 24, e = k - 24 * c;
    float v = 0.f;
    if (e < 23) {
#pragma unroll
      for (int w = 0; w < PG / 32; w++) v += red[((size_t)c * (PG / 32) + w) * 24 + e];
    }
    part[((size_t)c * gridDim.x + blockIdx.x) * 24 + e] = v;
  }
}

#define GSB_DISPATCH_K3(k3, CALL)                                           \
  switch (k3) {                                                             \
    case 1: { constexpr int K3 = 1; CALL; } break;                          \
    case 4: { constexpr int K3 = 4; CALL; } break;                          \
    case 9: { constexpr int K3 = 9; CALL; } break;                          \
    case 16: { constexpr int K3 = 16; CALL; } break;                        \
    default: return set_arg_error("sh_dim3 must be 1, 4, 9 or 16");         \
  }

// f(std::bool_constant<b>...) for the runtime flags b...: each flag becomes a compile-time constant
template <class F>
static int with_flags(F &&f) { return f(); }
template <class F, class... B>
static int with_flags(F &&f, bool b, B... rest) {
  const auto bind = [&](auto c) { return with_flags([&](auto... cs) { return f(c, cs...); }, rest...); };
  return b ? bind(std::true_type{}) : bind(std::false_type{});
}
// f(std::integral_constant<int, pg::CamModel>) for the camera model `model`.  The deduced return
// type has the compiler instantiate f, and its kernels, where this is called: the forward's kernels
// stay ahead of k_sh_expand in the cubin.
template <class F>
static auto with_model(int model, const char *unknown, F &&f) {
  switch (model) {
    case pg::PINHOLE: return f(std::integral_constant<int, pg::PINHOLE>{});
    case pg::ORTHO: return f(std::integral_constant<int, pg::ORTHO>{});
    case pg::FISHEYE: return f(std::integral_constant<int, pg::FISHEYE>{});
    case pg::OPENCV: return f(std::integral_constant<int, pg::OPENCV>{});
    default: return set_arg_error(unknown);
  }
}
// the kernels' lk
static float4 lens_k(const CamLens *lens) {
  return lens ? make_float4(lens->k[0], lens->k[1], lens->k[2], lens->k[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
}
// the kernels' tan_fovx, tan_fovy: W / (2 fx), H / (2 fy), stretched by OPENCV's lens (exactly 1 otherwise)
float2 lens_tan_fov(const FusedScene &sc) {
  const float c = sc.lens ? sc.lens->stretch : 1.f;
  return make_float2(sc.width / (2 * sc.fx) * c, sc.height / (2 * sc.fy) * c);
}

int launch_preprocess_fwd(const FusedScene &sc, const FusedFwd &f, cudaStream_t st) {
  const int N = sc.N;
  if (N <= 0) return 0;
  const float2 tf = lens_tan_fov(sc);
  const float tfx = tf.x, tfy = tf.y;
  const int nb = (N + PG - 1) / PG;
  const float4 lk = lens_k(sc.lens);
  ProfScope ps(K_PRE_FWD, st);
  const auto launch = [&](auto aa) {
    return with_model(sc.lens ? sc.lens->model : pg::PINHOLE, "preprocess: unknown camera model", [&](auto mdl) -> int {
      constexpr bool AA = decltype(aa)::value;
      constexpr int MODEL = decltype(mdl)::value;
      GSB_DISPATCH_K3(sc.k3, (k_preprocess_fwd<K3, AA, MODEL><<<nb, PG, 0, st>>>(
                                 N, sc.pws, sc.rots, sc.scales, sc.shs, sc.Rcw, sc.tcw, sc.twc, sc.fx, sc.fy, sc.cx,
                                 sc.cy, tfx, tfy, f.us, f.cinv2ds, f.colors, f.depths, f.areas, f.alphas, f.recs,
                                 AA ? f.alphas_eff : nullptr, lk)));
      return 0;
    });
  };
  const int rc = f.alphas_eff != nullptr ? launch(std::true_type{}) : launch(std::false_type{});
  if (rc) return rc;
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_sh_expand(int N, int k3, int V, const float *pws, const float *twcs, const float *gcols, float *g_shs,
                     cudaStream_t st) {
  if (N <= 0) return 0;
  const int nb = (N + PG - 1) / PG;
  ProfScope ps(K_SH_EXPAND, st);
  GSB_DISPATCH_K3(k3, (k_sh_expand<K3><<<nb, PG, 0, st>>>(N, V, pws, twcs, gcols, g_shs)));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// one launch of k_preprocess_bwd_intrinsics.  Its static SH tile (25 KB at K3 = 16) and `red` (24 KB at
// C = 64) together pass the 48 KB a kernel gets without asking, so it asks for `red`.
template <int K3, bool DEPTH, bool AA, int MODEL>
static int launch_intrinsics_kernel(int nb, size_t red, int C, int N, const float *pws, const float *rots,
                                    const float *scales, const float *shs, const PosePtrs &pp, const BatchCams &bc,
                                    const float *moments, const float *cinv2ds, const float *g_depths,
                                    const float *alphas, float *part, cudaStream_t st) {
  GSB_CUDA_TRY(cudaFuncSetAttribute(k_preprocess_bwd_intrinsics<K3, DEPTH, AA, MODEL>,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)red));
  k_preprocess_bwd_intrinsics<K3, DEPTH, AA, MODEL><<<nb, PG, red, st>>>(C, N, pws, rots, scales, shs, pp, bc, moments,
                                                                         cinv2ds, g_depths, alphas, part);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// the pose + intrinsics pass and its reduction, for launch_preprocess_bwd (C = 1) and
// launch_preprocess_bwd_batch: moment rows, dL/dz and alphas as k_preprocess_bwd_intrinsics reads them
static int launch_intrinsics_pass(int C, int N, int k3, int model, const float *pws, const float *rots,
                                  const float *scales, const float *shs, const PosePtrs &pp, const BatchCams &bc,
                                  const float *moments, const float *cinv2ds, const float *g_depths,
                                  const float *alphas, const PoseOut &po, cudaStream_t st) {
  const int nb = N > 0 ? (N + PG - 1) / PG : 0;
  if (nb > 0) {
    const size_t red = (size_t)C * (PG / 32) * 24 * sizeof(float);
    const int rc = with_model(model, "preprocessB_intrinsics: unknown camera model", [&](auto mdl) {
      return with_flags(
          [&](auto depth, auto aa) -> int {
            constexpr bool DEPTH = decltype(depth)::value, AA = decltype(aa)::value;
            constexpr int MODEL = decltype(mdl)::value;
            GSB_DISPATCH_K3(k3, return (launch_intrinsics_kernel<K3, DEPTH, AA, MODEL>(
                                    nb, red, C, N, pws, rots, scales, shs, pp, bc, moments, cinv2ds, g_depths,
                                    alphas, po.part, st)));
            return 0;
          },
          g_depths != nullptr, alphas != nullptr);
    });
    if (rc) return rc;
  }
  k_intrinsics_reduce<<<C, PR, 0, st>>>(nb, po.part, po.gcam, po.gint);
  return 0;
}

int launch_preprocess_bwd(const FusedScene &sc, const FusedBwd &b, cudaStream_t st) {
  const int N = sc.N;
  const PoseOut *po = b.po;
  if (N <= 0 && po == nullptr) return 0;
  const float2 tf = lens_tan_fov(sc);
  const float tfx = tf.x, tfy = tf.y;
  const int nb = N > 0 ? (N + PG - 1) / PG : 0;
  const bool moments = b.mi.moments != nullptr;
  const GradPush p = b.gp ? *b.gp : GradPush{};
  const MomentsIn m = moments ? b.mi : MomentsIn{};
  float *part = po ? po->part : nullptr;
  const float4 lk = lens_k(sc.lens);
  // one pass of k_preprocess_bwd<K3, PUSH, MOM, DEPTH, POSE, AA, MODEL>, PUSH, MOM, DEPTH and AA set
  // by which optional inputs are given.  The exchange carries neither a depth nor a camera gradient,
  // so no PUSH form with DEPTH or POSE exists (api.cu never asks for one); AA exists only with the
  // moment rows and without the exchange, and so do the camera models other than PINHOLE.
  const auto pass = [&](auto pose) -> int {
    return with_model(sc.lens ? sc.lens->model : pg::PINHOLE, "preprocessB: unknown camera model", [&](auto mdl) {
      return with_flags(
          [&](auto push, auto mom, auto depth, auto aa) -> int {
            constexpr bool PUSH = decltype(push)::value, MOM = decltype(mom)::value, DEPTH = decltype(depth)::value,
                           POSE = decltype(pose)::value, AA = decltype(aa)::value;
            constexpr int MODEL = decltype(mdl)::value;
            if constexpr (PUSH && (DEPTH || POSE)) {
              return set_arg_error("preprocessB: no depth or camera gradient with the exchange");
            } else if constexpr (AA && (PUSH || !MOM)) {
              return set_arg_error("preprocessB: antialiasing needs the moment rows and no exchange");
            } else if constexpr (MODEL != pg::PINHOLE && (PUSH || !MOM)) {
              return set_arg_error("preprocessB: camera models need the moment rows and no exchange");
            } else {
              GSB_DISPATCH_K3(sc.k3, (k_preprocess_bwd<K3, PUSH, MOM, DEPTH, POSE, AA, MODEL><<<nb, PG, 0, st>>>(
                                         N, sc.pws, sc.rots, sc.scales, sc.shs, sc.Rcw, sc.tcw, sc.twc, sc.fx, sc.fy,
                                         sc.cx, sc.cy, tfx, tfy, b.g_us, b.g_cinv2ds, b.g_colors, b.g_pws, b.g_shs,
                                         b.g_scales, b.g_rots, p, m, b.g_depths, part, b.alphas, lk)));
              return 0;
            }
          },
          b.gp != nullptr, moments, b.g_depths != nullptr, b.alphas != nullptr);
    });
  };
  ProfScope ps(K_PRE_BWD, st);
  // the camera gradient first; then, unless g_pws is NULL (pose only), the per-Gaussian gradients
  // from the form without POSE
  if (po != nullptr && po->gint != nullptr) {  // with the intrinsics' (DESIGN 3.23): a one-camera batch
    BatchCams bc;
    bc.f[0] = make_float4(sc.fx, sc.fy, sc.cx, sc.cy);
    bc.k[0] = lk;
    bc.tf[0] = tf;
    if (int rc = launch_intrinsics_pass(1, N, sc.k3, sc.lens ? sc.lens->model : pg::PINHOLE, sc.pws, sc.rots,
                                        sc.scales, sc.shs, PosePtrs{sc.Rcw, sc.tcw, sc.twc, 0}, bc, m.moments,
                                        m.cinv2ds, b.g_depths, b.alphas, *po, st))
      return rc;
  } else if (po != nullptr) {
    if (nb > 0)
      if (int rc = pass(std::true_type{})) return rc;
    k_pose_reduce<<<1, PR, 0, st>>>(nb, part, po->gcam);
  }
  if (nb > 0 && (po == nullptr || b.g_pws != nullptr))
    if (int rc = pass(std::false_type{})) return rc;
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_preprocess_fwd_batch(const BatchScene &b, const FusedFwd &f, cudaStream_t st) {
  if (b.N <= 0) return 0;
  const int nb = (b.N + PG - 1) / PG;
  ProfScope ps(K_PRE_FWD_BATCH, st);
  const auto launch = [&](auto aa) {
    return with_model(b.model, "preprocess_batch: unknown camera model", [&](auto mdl) -> int {
      constexpr bool AA = decltype(aa)::value;
      constexpr int MODEL = decltype(mdl)::value;
      GSB_DISPATCH_K3(b.k3, (k_preprocess_fwd_batch<K3, AA, MODEL><<<nb, PG, 0, st>>>(
                                b.C, b.N, b.pws, b.rots, b.scales, b.shs, b.poses, *b.cams, f.us, f.cinv2ds, f.colors,
                                f.depths, f.areas, f.alphas, f.recs, f.alphas_eff)));
      return 0;
    });
  };
  const int rc = f.alphas_eff != nullptr ? launch(std::true_type{}) : launch(std::false_type{});
  if (rc) return rc;
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_preprocess_bwd_batch(const BatchScene &b, const BatchBwd &g, cudaStream_t st) {
  const PoseOut *po = g.po;
  if (b.N <= 0 && po == nullptr) return 0;
  const int nb = b.N > 0 ? (b.N + PG - 1) / PG : 0;
  // one pass: k_preprocess_bwd_batch_pose (pose) or k_preprocess_bwd_batch, DEPTH and AA set by which
  // optional inputs are given
  const auto pass = [&](auto pose) {
    return with_model(b.model, "preprocessB_batch: unknown camera model", [&](auto mdl) {
      return with_flags(
          [&](auto depth, auto aa) -> int {
            constexpr bool DEPTH = decltype(depth)::value, AA = decltype(aa)::value;
            constexpr int MODEL = decltype(mdl)::value;
            if constexpr (decltype(pose)::value) {
              const size_t red = (size_t)b.C * (PG / 32) * 16 * sizeof(float);
              GSB_DISPATCH_K3(b.k3, (k_preprocess_bwd_batch_pose<K3, DEPTH, AA, MODEL><<<nb, PG, red, st>>>(
                                        b.C, b.N, b.pws, b.rots, b.scales, b.shs, b.poses, *b.cams, g.moments,
                                        g.cinv2ds, g.g_depths, g.alphas, po->part)));
            } else {
              GSB_DISPATCH_K3(b.k3, (k_preprocess_bwd_batch<K3, DEPTH, AA, MODEL><<<nb, PG, 0, st>>>(
                                        b.C, b.N, b.pws, b.rots, b.scales, b.shs, b.poses, *b.cams, g.moments,
                                        g.cinv2ds, g.g_depths, g.alphas, g.dus_out, g.dalphas_out, g.g_pws, g.g_shs,
                                        g.g_scales, g.g_rots)));
            }
            return 0;
          },
          g.g_depths != nullptr, g.alphas != nullptr);
    });
  };
  ProfScope ps(K_PRE_BWD_BATCH, st);
  // the camera gradients first (DESIGN 3.22); then, unless g_pws is NULL (pose only), the per-Gaussian
  // gradients from the kernel without the camera terms, so that they are the same bits either way
  if (po != nullptr && po->gint != nullptr) {  // with the intrinsics' (DESIGN 3.23)
    if (int rc = launch_intrinsics_pass(b.C, b.N, b.k3, b.model, b.pws, b.rots, b.scales, b.shs,
                                        PosePtrs{b.poses, b.poses + 9, b.poses + 12, 15}, *b.cams, g.moments,
                                        g.cinv2ds, g.g_depths, g.alphas, *po, st))
      return rc;
  } else if (po != nullptr) {
    if (nb > 0)
      if (int rc = pass(std::true_type{})) return rc;
    k_pose_reduce_batch<<<b.C, PR, 0, st>>>(nb, po->part, po->gcam);
  }
  if (nb > 0 && (po == nullptr || g.g_pws != nullptr))
    if (int rc = pass(std::false_type{})) return rc;
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
