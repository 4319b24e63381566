// 2D Gaussian Splatting (DESIGN 3.15): surfels rendered by ray-splat intersection.
//
//  k_surfel_fwd<K3>    one pass per surfel (surfel_math.h forward_one): us, depths, areas, colours and
//                      one 80-byte record [M (9), alpha, u (2), cull half-extents (2), colour (3), n (3)]
//  (binning)           launch_bin + launch_sort_and_pack(pack = false), unchanged: they read only
//                      us, areas and depths
//  k_draw_surfel       the persistent record walk of the colour rasterizer (raster_walk.cuh: work list,
//                      cp.async chunk ring, exact per-block culling into a survivor list) over 80-byte
//                      records; composites image, depth = sum w z(p), alpha = sum w, normal = sum w n
//  k_draw_surfel_bwd   back to front from final_tau and contrib, the recurrence of k_draw_bwd over
//                      3 + 1 + 1 + 3 channels; each (record, 8x8 block) is reduced in the warp and added
//                      to the surfel's gradient row [dM (9), dalpha, dcolour (3), dn (3), ddelta (2)]
//  k_draw_2dgs         k_draw_surfel's walk (draw_walk<true>) that also composites the 2DGS geometry
//                      planes (DESIGN 3.16): depth distortion, its moments and the median depth
//  k_draw_2dgs_bwd     k_draw_surfel_bwd's walk (draw_bwd_walk<true>) with the geometry terms added to
//                      the alpha' recurrence and to the hit-depth gradient; the rows are the same
//  k_surfel_bwd<K3>    the rows -> dL/dpws, dL/dshs, dL/dalphas, dL/dscales, dL/drots, dL/dus (= ddelta)
//  k_draw_stats_2dgs   per-surfel sums, maxima and counts of a drawn frame's weights (DESIGN 3.18)
//  k_disk_fwd_batch<K3>, k_disk_bwd_batch<K3>, k_draw_disk_batch, k_draw_2dgs_batch, k_draw_disk_bwd_batch,
//  k_draw_2dgs_bwd_batch: the batch forms of k_surfel_fwd, k_surfel_bwd and the four rasterizers for C
//                      cameras drawn as one tall frame (DESIGN 3.25)
#include "common.cuh"
#include "kernels.h"
#include "raster_walk.cuh"
#include "surfel_math.h"
#include "tile_io.cuh"

namespace gsb {

#ifndef DRAW_SURFEL_MINBLOCKS
#define DRAW_SURFEL_MINBLOCKS 4
#endif
#ifndef DRAW_SURFEL_BWD_MINBLOCKS
#define DRAW_SURFEL_BWD_MINBLOCKS 4
#endif
#ifndef DRAW_2DGS_BWD_MINBLOCKS
#define DRAW_2DGS_BWD_MINBLOCKS 4
#endif
// k_draw_stats_2dgs: 56 registers and 21 KiB of shared memory without spills (-Xptxas -v), so 8
// CTAs of 128 threads fit the register file
#ifndef DRAW_STATS_2DGS_MINBLOCKS
#define DRAW_STATS_2DGS_MINBLOCKS 8
#endif

constexpr int SREC_BYTES = sf::kRecFloats * 4;  // 80
static_assert(SREC_BYTES == 80, "surfel record must be 80 bytes");

__device__ __forceinline__ pg::Cam surfel_cam(const float *__restrict__ Rcw, const float *__restrict__ tcw,
                                              const float *__restrict__ twc, float fx, float fy, float cx, float cy) {
  pg::Cam c;
#pragma unroll
  for (int i = 0; i < 9; i++) c.R[i] = __ldg(Rcw + i);
#pragma unroll
  for (int i = 0; i < 3; i++) { c.t[i] = __ldg(tcw + i); c.twc[i] = __ldg(twc + i); }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy; c.tan_fovx = 0.f; c.tan_fovy = 0.f;
  return c;
}

__device__ __forceinline__ void surfel_rows(const float *__restrict__ pws, const float *__restrict__ scales,
                                            const float *__restrict__ rots, long long i, float (&pw)[3],
                                            float (&s)[3], float (&q)[4]) {
  pw[0] = __ldg(pws + 3 * i); pw[1] = __ldg(pws + 3 * i + 1); pw[2] = __ldg(pws + 3 * i + 2);
  s[0] = __ldg(scales + 3 * i); s[1] = __ldg(scales + 3 * i + 1); s[2] = __ldg(scales + 3 * i + 2);
  q[0] = __ldg(rots + 4 * i); q[1] = __ldg(rots + 4 * i + 1); q[2] = __ldg(rots + 4 * i + 2); q[3] = __ldg(rots + 4 * i + 3);
}

#define ROWK(K) (sm + tid * TileT<K>::S)

template <int K3>
__global__ void __launch_bounds__(PG) k_surfel_fwd(int N, const float *__restrict__ pws, const float *__restrict__ rots,
                                                   const float *__restrict__ scales, const float *__restrict__ shs,
                                                   const float *__restrict__ Rcw, const float *__restrict__ tcw,
                                                   const float *__restrict__ twc, float fx, float fy, float cx, float cy,
                                                   const float *__restrict__ alphas, float *__restrict__ us,
                                                   float *__restrict__ depths, int32_t *__restrict__ areas,
                                                   float *__restrict__ colors, float4 *__restrict__ recs) {
  constexpr int KS = 3 * K3;
  __shared__ float sm[TileT<KS>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  const pg::Cam cam = surfel_cam(Rcw, tcw, twc, fx, fy, cx, cy);
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f}, al = 0.f;
  if (valid) {
    surfel_rows(pws, scales, rots, base + tid, pw, s, q);
    al = __ldg(alphas + base + tid);
  }
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  if (!valid) return;
  float u[2], depth, col[3], rec[sf::kRecFloats];
  int area[2];
  sf::forward_one<K3>(pw, q, s, ROWK(KS), al, cam, u, &depth, area, col, rec);
  const long long i = base + tid;
  st_pair(us, i, u[0], u[1]);
  depths[i] = depth;
  st_pair(areas, i, area[0], area[1]);
  colors[3 * i] = col[0]; colors[3 * i + 1] = col[1]; colors[3 * i + 2] = col[2];
#pragma unroll
  for (int k = 0; k < 5; k++) recs[5 * i + k] = make_float4(rec[4 * k], rec[4 * k + 1], rec[4 * k + 2], rec[4 * k + 3]);
}

template <int K3>
__global__ void __launch_bounds__(PG) k_surfel_bwd(int N, const float *__restrict__ pws, const float *__restrict__ rots,
                                                   const float *__restrict__ scales, const float *__restrict__ shs,
                                                   const float *__restrict__ Rcw, const float *__restrict__ tcw,
                                                   const float *__restrict__ twc, float fx, float fy, float cx, float cy,
                                                   const float *__restrict__ rows, float *__restrict__ g_pws,
                                                   float *__restrict__ g_shs, float *__restrict__ g_alphas,
                                                   float *__restrict__ g_scales, float *__restrict__ g_rots,
                                                   float *__restrict__ g_us) {
  constexpr int KS = 3 * K3;
  __shared__ float sm[TileT<KS>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  const pg::Cam cam = surfel_cam(Rcw, tcw, twc, fx, fy, cx, cy);
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  float row[sf::kRowFloats];
  if (valid) {
    const long long i = base + tid;
    surfel_rows(pws, scales, rots, i, pw, s, q);
#pragma unroll
    for (int k = 0; k < sf::kRowFloats; k++) row[k] = __ldg(rows + sf::kRowFloats * i + k);
  }
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  float gpw[3], gq[4], gs[3];
  if (valid) sf::backward_one<K3>(pw, q, s, ROWK(KS), cam, row, gpw, gq, gs, ROWK(KS));  // dL/dsh in place
  __syncthreads();
  tile_flush<KS>(g_shs, base, nv, sm, tid);
  if (!valid) return;
  const long long o = base + tid;
  g_pws[3 * o] = gpw[0]; g_pws[3 * o + 1] = gpw[1]; g_pws[3 * o + 2] = gpw[2];
  g_scales[3 * o] = gs[0]; g_scales[3 * o + 1] = gs[1]; g_scales[3 * o + 2] = 0.f;
  g_rots[4 * o] = gq[0]; g_rots[4 * o + 1] = gq[1]; g_rots[4 * o + 2] = gq[2]; g_rots[4 * o + 3] = gq[3];
  g_alphas[o] = row[9];
  st_pair(g_us, o, row[16], row[17]);
}

// ---- batched per-surfel kernels (DESIGN 3.25): C pinhole cameras in one launch, as
// k_preprocess_fwd_batch / k_preprocess_bwd_batch (fused.cu).  A thread loads its surfel's rows once
// (pw, q, s, alpha to registers, the SH row through the shared tile) and runs sf::forward_one /
// sf::backward_one once per camera: camera c's pose from poses[c] (Rcw 9, tcw 3, twc 3 floats), its
// intrinsics from the kernel parameters.  Camera c's outputs go to rows c N + n of [C, N, ...].
__device__ __forceinline__ pg::Cam disk_batch_cam(const float *__restrict__ poses, const BatchCams &bc, int c) {
  const float *p = poses + 15 * c;
  const float4 f = bc.f[c];
  return surfel_cam(p, p + 9, p + 12, f.x, f.y, f.z, f.w);
}

// the forward: k_surfel_fwd's outputs per camera; record c N + n of recs [C N, 20]
template <int K3>
__global__ void __launch_bounds__(PG) k_disk_fwd_batch(int C, int N, const float *__restrict__ pws,
                                                       const float *__restrict__ rots, const float *__restrict__ scales,
                                                       const float *__restrict__ shs, const float *__restrict__ poses,
                                                       const __grid_constant__ BatchCams bc,
                                                       const float *__restrict__ alphas, float *__restrict__ us,
                                                       float *__restrict__ depths, int32_t *__restrict__ areas,
                                                       float *__restrict__ colors, float4 *__restrict__ recs) {
  constexpr int KS = 3 * K3;
  __shared__ float sm[TileT<KS>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f}, al = 0.f;
  if (valid) {
    surfel_rows(pws, scales, rots, base + tid, pw, s, q);
    al = __ldg(alphas + base + tid);
  }
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  if (!valid) return;
  const long long i = base + tid;
  for (int c = 0; c < C; c++) {
    const pg::Cam cam = disk_batch_cam(poses, bc, c);
    float u[2], depth, col[3], rec[sf::kRecFloats];
    int area[2];
    sf::forward_one<K3>(pw, q, s, ROWK(KS), al, cam, u, &depth, area, col, rec);
    const long long o = (long long)c * N + i;
    st_pair(us, o, u[0], u[1]);
    depths[o] = depth;
    st_pair(areas, o, area[0], area[1]);
    colors[3 * o] = col[0]; colors[3 * o + 1] = col[1]; colors[3 * o + 2] = col[2];
#pragma unroll
    for (int k = 0; k < 5; k++) recs[5 * o + k] = make_float4(rec[4 * k], rec[4 * k + 1], rec[4 * k + 2], rec[4 * k + 3]);
  }
}

// the backward from the rows [C N, 18]: the C contributions to each per-surfel gradient summed in
// fp32 registers in camera order.  dL/dsh goes to registers, not over the SH tile as in
// k_surfel_bwd: the next camera still reads the SH row.  One gradient row per surfel (dL/dalpha the
// sum of the rows' dalpha), dL/dus per camera [C, N, 2].
template <int K3>
__global__ void __launch_bounds__(PG) k_disk_bwd_batch(int C, int N, const float *__restrict__ pws,
                                                       const float *__restrict__ rots, const float *__restrict__ scales,
                                                       const float *__restrict__ shs, const float *__restrict__ poses,
                                                       const __grid_constant__ BatchCams bc,
                                                       const float *__restrict__ rows, float *__restrict__ g_pws,
                                                       float *__restrict__ g_shs, float *__restrict__ g_alphas,
                                                       float *__restrict__ g_scales, float *__restrict__ g_rots,
                                                       float *__restrict__ g_us) {
  constexpr int KS = 3 * K3;
  __shared__ float sm[TileT<KS>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float pw[3] = {0.f, 0.f, 1.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
  if (valid) surfel_rows(pws, scales, rots, base + tid, pw, s, q);
  tile_fetch<KS>(shs, base, nv, sm, tid);
  __syncthreads();
  float gpw[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gsh[KS], gal = 0.f;
#pragma unroll
  for (int e = 0; e < KS; e++) gsh[e] = 0.f;
  const long long i = base + tid;
  if (valid) {
    for (int c = 0; c < C; c++) {
      const long long o = (long long)c * N + i;
      float row[sf::kRowFloats];
#pragma unroll
      for (int k = 0; k < sf::kRowFloats; k++) row[k] = __ldg(rows + sf::kRowFloats * o + k);
      const pg::Cam cam = disk_batch_cam(poses, bc, c);
      float xpw[3], xq[4], xs[3], xsh[KS];
      sf::backward_one<K3>(pw, q, s, ROWK(KS), cam, row, xpw, xq, xs, xsh);
#pragma unroll
      for (int e = 0; e < 3; e++) { gpw[e] += xpw[e]; gs[e] += xs[e]; }
#pragma unroll
      for (int e = 0; e < 4; e++) gq[e] += xq[e];
#pragma unroll
      for (int e = 0; e < KS; e++) gsh[e] += xsh[e];
      gal += row[9];
      st_pair(g_us, o, row[16], row[17]);
    }
    // dL/dsh replaces the thread's own SH row (no other thread reads it before the barrier)
    float *row = ROWK(KS);
#pragma unroll
    for (int e = 0; e < KS; e++) row[e] = gsh[e];
  }
  __syncthreads();
  tile_flush<KS>(g_shs, base, nv, sm, tid);
  if (!valid) return;
  g_pws[3 * i] = gpw[0]; g_pws[3 * i + 1] = gpw[1]; g_pws[3 * i + 2] = gpw[2];
  g_scales[3 * i] = gs[0]; g_scales[3 * i + 1] = gs[1]; g_scales[3 * i + 2] = 0.f;
  g_rots[4 * i] = gq[0]; g_rots[4 * i + 1] = gq[1]; g_rots[4 * i + 2] = gq[2]; g_rots[4 * i + 3] = gq[3];
  g_alphas[i] = gal;
}

// ---- the rasterizers' 80-byte record walk: raster_walk.cuh's protocol and chunk helpers at
// SREC_BYTES, with the surfel record's own cull

// Can the record reach alpha' >= 0.002 in the block [bx0, bx1] x [by0, by1]?  Its cull box (u +-
// the half-extents of sf::cull_extent) bounds {G3 <= t} and {G2 <= t}: outside it min(G3, G2) > t.
__device__ __forceinline__ bool surfel_can_touch(uint32_t rec, float bx0, float bx1, float by0, float by1) {
  const float4 q2 = lds128(rec + 32), q3 = lds128(rec + 48);
  return (q2.z + q3.x >= bx0) && (q2.z - q3.x <= bx1) && (q2.w + q3.y >= by0) && (q2.w - q3.y <= by1);
}

// The record's fields in registers
struct SRecRegs {
  float M[9], al, u[2], col[3], n[3];
};
__device__ __forceinline__ void load_srec(uint32_t a, SRecRegs &r) {
  const float4 q0 = lds128(a), q1 = lds128(a + 16), q2 = lds128(a + 32), q3 = lds128(a + 48), q4 = lds128(a + 64);
  r.M[0] = q0.x; r.M[1] = q0.y; r.M[2] = q0.z; r.M[3] = q0.w;
  r.M[4] = q1.x; r.M[5] = q1.y; r.M[6] = q1.z; r.M[7] = q1.w;
  r.M[8] = q2.x; r.al = q2.y; r.u[0] = q2.z; r.u[1] = q2.w;
  r.col[0] = q3.z; r.col[1] = q3.w; r.col[2] = q4.x;
  r.n[0] = q4.y; r.n[1] = q4.z; r.n[2] = q4.w;
}

// alpha' of a record at one pixel, the one operation sequence both rasterizers replay; g = the
// Gaussian factor, clamped = alpha g above 0.99
__device__ __forceinline__ float surfel_alpha(const SRecRegs &r, float x, float y, sf::PixEval &pe, float &g,
                                              bool &clamped) {
  sf::pixel_eval(r.M, r.u, x, y, pe);
  g = ex2_approx(-0.5f * LOG2E * pe.G);
  const float ag = r.al * g;
  clamped = ag > ALPHA_CLAMP;
  return fminf(ALPHA_CLAMP, ag);
}

// Cull and compact one chunk: survivors as (record address, patch index) in walk order; returns n.
// back: list back to front (the backward's order).
__device__ __forceinline__ int surfel_compact(uint32_t my_rec, int my_idx, int lim, float bx0, float bx1, float by0,
                                              float by1, uint32_t list, int lane, bool back) {
  const bool hit = my_idx < lim && surfel_can_touch(my_rec, bx0, bx1, by0, by1);
  const unsigned mask = __ballot_sync(0xffffffffu, hit);
  if (hit) {
    const int pos = back ? __popc(mask & ~((2u << lane) - 1u)) : __popc(mask & ((1u << lane) - 1u));
    sts64u(list + pos * 8, my_rec, (uint32_t)my_idx);
  }
  __syncwarp();
  return __popc(mask);
}

// one 8x8 block of a work-list entry: pixel coordinates of the lane's pair.  BATCH: the tall frame
// of a batch (DESIGN 3.25, as draw_body's in raster_fwd.cu): tile row r is row r - f gy of frame
// f = r / gy, the pixels are that frame's own coordinates, fo = f H W is the frame's offset in every
// [H,W] plane and pix includes it; a block in a pad row lies below the frame and is skipped.
struct BlockPix {
  int rx0, ry0, px, py;
  bool in0, in1;
  size_t pix, fo;
};
template <bool BATCH>
__device__ __forceinline__ bool block_pix(int W, int H, int gx, int gy, int tile, int blk, int lane, BlockPix &b) {
  int tx = tile % gx, ty = tile / gx;
  b.fo = 0;
  if constexpr (BATCH) {
    const int f = ty / gy;
    ty -= f * gy;
    b.fo = (size_t)f * H * W;
  }
  b.rx0 = tx * TILE + (blk & 1) * 8;
  b.ry0 = ty * TILE + (blk >> 1) * 8;
  if (b.rx0 >= W || b.ry0 >= H) return false;
  b.px = b.rx0 + 2 * (lane & 3);
  b.py = b.ry0 + (lane >> 2);
  b.in0 = b.px < W && b.py < H;
  b.in1 = b.px + 1 < W && b.py < H;
  b.pix = b.fo + (size_t)b.py * W + b.px;
  return true;
}

// the NDC-mapped hit depth of the geometry planes and its derivative (0 at and below near)
__device__ __forceinline__ float geo_m(float z, float near, float mscale) {
  return mscale * (1.0f - near / fmaxf(z, near));
}
__device__ __forceinline__ float geo_dm(float z, float near, float mscale) {
  return z > near ? mscale * near / (z * z) : 0.f;
}

// The forward walk of k_draw_surfel and (GEO) k_draw_2dgs: GEO also accumulates the moments
// D = sum w m, D2 = sum w m^2, the distortion sum_{j<i} w_i w_j (m_i - m_j)^2 and the median.
// BATCH: the tall frame of a batch of frames (k_draw_disk_batch, k_draw_2dgs_batch; block_pix): every
// plane is frame f's of [C, ..., H, W]
template <bool GEO, bool BATCH>
__device__ __forceinline__ void draw_walk(int W, int H, int gx, int gy, const int2 *__restrict__ ranges,
                                          const float4 *__restrict__ recs, const int32_t *__restrict__ gsid,
                                          float *__restrict__ image, int32_t *__restrict__ contrib,
                                          float *__restrict__ final_tau, float *__restrict__ depth_image,
                                          float *__restrict__ alpha_image, float *__restrict__ normal_image,
                                          const GeoPlanes &geo, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<SREC_BYTES>];
  __shared__ __align__(16) uint2 s_list[4][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const int items = work[1];
  const int *__restrict__ entries = work + 2;
  for (;;) {
    const int item = pull_item(work, lane);
    if (item >= items) break;
    const int ent = __ldg(entries + item);
    const int tile = ent >> 3, code = ent & 7;
    const int2 range = __ldg(ranges + tile);
    const int len = range.y - range.x;
    const int32_t *ids = gsid + range.x;
    for (int blk = code == 4 ? 0 : code; blk < (code == 4 ? 4 : code + 1); blk++) {
      BlockPix bp;
      if (!block_pix<BATCH>(W, H, gx, gy, tile, blk, lane, bp)) continue;
      const float xs[2] = {(float)bp.px, (float)(bp.px + 1)}, y = (float)bp.py;
      float tau[2] = {bp.in0 ? 1.0f : 0.0f, bp.in1 ? 1.0f : 0.0f};
      float acc[2][8];  // r, g, b, depth, alpha, nx, ny, nz
      int cont[2] = {0, 0};
#pragma unroll
      for (int p = 0; p < 2; p++)
#pragma unroll
        for (int k = 0; k < 8; k++) acc[p][k] = 0.f;
      float mD[2] = {0.f, 0.f}, mD2[2] = {0.f, 0.f}, dist[2] = {0.f, 0.f}, medz[2] = {0.f, 0.f};
      int medc[2] = {0, 0};
      if (len > 0) {
        const int nch = (len + 31) >> 5;
        auto issue = [&](int c) {
          if (c < nch && c * 32 + lane < len)
            gather_record<SREC_BYTES>(recs + 5 * (size_t)__ldg(ids + c * 32 + lane),
                                      ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<SREC_BYTES> +
                                          lane * SREC_BYTES);
          cp_async_commit();
        };
#pragma unroll
        for (int r = 0; r < WALK_RING; r++) issue(r);
        const float bx0 = (float)bp.rx0, bx1 = (float)(bp.rx0 + 7), by0 = (float)bp.ry0, by1 = (float)(bp.ry0 + 7);
        for (int c = 0; c < nch; c++) {
          const int n = surfel_compact(wait_chunk<SREC_BYTES>(ring_addr, c, lane), c * 32 + lane, len, bx0, bx1, by0,
                                       by1, list_addr, lane, false);
          for (int i = 0; i < n; i++) {
            const uint2 e = lds64u(list_addr + i * 8);
            SRecRegs r;
            load_srec(e.x, r);
#pragma unroll
            for (int p = 0; p < 2; p++) {
              sf::PixEval pe;
              float g;
              bool clamped;
              const float ap = surfel_alpha(r, xs[p], y, pe, g, clamped);
              if (tau[p] >= TAU_STOP && ap >= ALPHA_SKIP) {
                const float w = tau[p] * ap;
                if constexpr (GEO) {
                  // before this record joins the totals: w (m^2 A + D2 - 2 m D), A = acc[p][4]
                  const float m = geo_m(pe.z, geo.near, geo.mscale);
                  dist[p] = fmaf(w, fmaf(m, fmaf(m, acc[p][4], -2.0f * mD[p]), mD2[p]), dist[p]);
                  mD[p] = fmaf(w, m, mD[p]);
                  mD2[p] = fmaf(w * m, m, mD2[p]);
                  if (tau[p] > 0.5f) {
                    medz[p] = pe.z;
                    medc[p] = (int)e.y + 1;
                  }
                }
                acc[p][0] = fmaf(w, r.col[0], acc[p][0]);
                acc[p][1] = fmaf(w, r.col[1], acc[p][1]);
                acc[p][2] = fmaf(w, r.col[2], acc[p][2]);
                acc[p][3] = fmaf(w, pe.z, acc[p][3]);
                acc[p][4] += w;
                acc[p][5] = fmaf(w, r.n[0], acc[p][5]);
                acc[p][6] = fmaf(w, r.n[1], acc[p][6]);
                acc[p][7] = fmaf(w, r.n[2], acc[p][7]);
                tau[p] = tau[p] * (1.0f - ap);
                cont[p] = (int)e.y + 1;
              }
            }
          }
          const bool done = __all_sync(0xffffffffu, tau[0] < TAU_STOP && tau[1] < TAU_STOP);
          if (done) break;
          __syncwarp();  // every lane is done with this ring slot and with the list
          issue(c + WALK_RING);
        }
        walk_drain();
      }
      // the frame's [3,H,W] planes start at 3 fo and its moments [2,H,W] at 2 fo (pix holds fo)
      float *const image_f = BATCH ? image + 2 * bp.fo : image;
      float *const normal_f = BATCH ? normal_image + 2 * bp.fo : normal_image;
      float *const moments_f = BATCH ? geo.moments + bp.fo : geo.moments;
#pragma unroll
      for (int p = 0; p < 2; p++) {
        if (!(p ? bp.in1 : bp.in0)) continue;
        const size_t q = bp.pix + p;
        image_f[q] = acc[p][0]; image_f[HW + q] = acc[p][1]; image_f[2 * HW + q] = acc[p][2];
        contrib[q] = cont[p]; final_tau[q] = tau[p];
        depth_image[q] = acc[p][3]; alpha_image[q] = acc[p][4];
        normal_f[q] = acc[p][5]; normal_f[HW + q] = acc[p][6]; normal_f[2 * HW + q] = acc[p][7];
        if constexpr (GEO) {
          geo.distortion[q] = dist[p];
          moments_f[q] = mD[p]; moments_f[HW + q] = mD2[p];
          geo.median_depth[q] = medz[p]; geo.median_contrib[q] = medc[p];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(128, DRAW_SURFEL_MINBLOCKS) k_draw_surfel(
    int W, int H, int gx, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, float *__restrict__ image, int32_t *__restrict__ contrib,
    float *__restrict__ final_tau, float *__restrict__ depth_image, float *__restrict__ alpha_image,
    float *__restrict__ normal_image, int *__restrict__ work) {
  draw_walk<false, false>(W, H, gx, 0, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                          normal_image, GeoPlanes{}, work);
}

// 2DGS (DESIGN 3.16): k_draw_surfel's planes, bit for bit, and the geometry planes
__global__ void __launch_bounds__(128, DRAW_SURFEL_MINBLOCKS) k_draw_2dgs(
    int W, int H, int gx, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, float *__restrict__ image, int32_t *__restrict__ contrib,
    float *__restrict__ final_tau, float *__restrict__ depth_image, float *__restrict__ alpha_image,
    float *__restrict__ normal_image, GeoPlanes geo, int *__restrict__ work) {
  draw_walk<true, false>(W, H, gx, 0, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                         normal_image, geo, work);
}

// ---- the batched rasterizers (DESIGN 3.25): the C frames of a batch binned as one tall frame of
// C gy tile rows, drawn from the records [C N, 20] (record c N + n: surfel n seen by camera c) into
// image / normal [C,3,H,W], contrib / final_tau / depth / alpha [C,H,W] and the geometry planes
// [C,...,H,W].  Frame c is the single frame of camera c, bit for bit.  (The kernels carry no
// "surfel" in their names: that name stays with the single-camera kernels.)
__global__ void __launch_bounds__(128, DRAW_SURFEL_MINBLOCKS) k_draw_disk_batch(
    int W, int H, int gx, int gy, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, float *__restrict__ image, int32_t *__restrict__ contrib,
    float *__restrict__ final_tau, float *__restrict__ depth_image, float *__restrict__ alpha_image,
    float *__restrict__ normal_image, int *__restrict__ work) {
  draw_walk<false, true>(W, H, gx, gy, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                         normal_image, GeoPlanes{}, work);
}

__global__ void __launch_bounds__(128, DRAW_SURFEL_MINBLOCKS) k_draw_2dgs_batch(
    int W, int H, int gx, int gy, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, float *__restrict__ image, int32_t *__restrict__ contrib,
    float *__restrict__ final_tau, float *__restrict__ depth_image, float *__restrict__ alpha_image,
    float *__restrict__ normal_image, GeoPlanes geo, int *__restrict__ work) {
  draw_walk<true, true>(W, H, gx, gy, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                        normal_image, geo, work);
}

// the upstream gradient planes of the backward; NULL reads as zero
struct SurfelGrads {
  const float *img, *depth, *alpha, *normal;
};

__device__ __forceinline__ float ld_plane(const float *__restrict__ p, size_t q) { return p ? __ldg(p + q) : 0.f; }

// The backward walk of k_draw_surfel_bwd and (GEO) k_draw_2dgs_bwd: GEO adds dL/ddistortion's
// dDelta/dw_i to the per-record value of the alpha' recurrence and its dDelta/dz_i, with dL/dmedian
// at the median record, to the hit-depth coefficient.  BATCH: as draw_walk's; the upstream planes
// and the forward's alpha, moments and median_contrib are frame f's of [C, ..., H, W] as well
template <bool GEO, bool BATCH>
__device__ __forceinline__ void draw_bwd_walk(int W, int H, int gx, int gy, const int2 *__restrict__ ranges,
                                              const float4 *__restrict__ recs, const int32_t *__restrict__ gsid,
                                              const int32_t *__restrict__ contrib,
                                              const float *__restrict__ final_tau, const SurfelGrads &dl,
                                              const GeoGrads &geo, float *__restrict__ rows, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<SREC_BYTES>];
  __shared__ __align__(16) uint2 s_list[4][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const int items = work[1];
  const int *__restrict__ entries = work + 2;
  for (;;) {
    const int item = pull_item(work, lane);
    if (item >= items) break;
    const int ent = __ldg(entries + item);
    const int tile = ent >> 3, code = ent & 7;
    const int2 range = __ldg(ranges + tile);
    const int len = range.y - range.x;
    const int32_t *ids = gsid + range.x;
    for (int blk = code == 4 ? 0 : code; blk < (code == 4 ? 4 : code + 1); blk++) {
      BlockPix bp;
      if (!block_pix<BATCH>(W, H, gx, gy, tile, blk, lane, bp)) continue;
      const float xs[2] = {(float)bp.px, (float)(bp.px + 1)}, y = (float)bp.py;
      int cont[2] = {0, 0};
      float tau[2] = {0.f, 0.f}, sdot[2] = {0.f, 0.f};
      float d[2][8];  // dL/d(r, g, b, depth, alpha, nx, ny, nz) of the pixel
      // the frame's [3,H,W] upstream planes start at 3 fo (pix holds fo)
      const float *img = dl.img, *nrm = dl.normal;
      if constexpr (BATCH) {
        if (img) img += 2 * bp.fo;
        if (nrm) nrm += 2 * bp.fo;
      }
#pragma unroll
      for (int p = 0; p < 2; p++) {
        const bool in = p ? bp.in1 : bp.in0;
        const size_t q = bp.pix + p;
        cont[p] = in ? min(__ldg(contrib + q), len) : 0;
        tau[p] = in ? __ldg(final_tau + q) : 0.f;
        d[p][0] = in ? ld_plane(img, q) : 0.f;
        d[p][1] = in ? ld_plane(img ? img + HW : nullptr, q) : 0.f;
        d[p][2] = in ? ld_plane(img ? img + 2 * HW : nullptr, q) : 0.f;
        d[p][3] = in ? ld_plane(dl.depth, q) : 0.f;
        d[p][4] = in ? ld_plane(dl.alpha, q) : 0.f;
        d[p][5] = in ? ld_plane(nrm, q) : 0.f;
        d[p][6] = in ? ld_plane(nrm ? nrm + HW : nullptr, q) : 0.f;
        d[p][7] = in ? ld_plane(nrm ? nrm + 2 * HW : nullptr, q) : 0.f;
      }
      // GEO: dL/ddistortion, dL/dmedian, the final A, D, D2 and the median record of each pixel
      float gdist[2] = {0.f, 0.f}, gmed[2] = {0.f, 0.f}, fA[2] = {0.f, 0.f}, fD[2] = {0.f, 0.f},
            fD2[2] = {0.f, 0.f};
      int medc[2] = {0, 0};
      if constexpr (GEO) {
#pragma unroll
        for (int p = 0; p < 2; p++) {
          if (!(p ? bp.in1 : bp.in0)) continue;
          const size_t q = bp.pix + p;
          gdist[p] = ld_plane(geo.distortion, q);
          gmed[p] = ld_plane(geo.median, q);
          const float *moments_f = BATCH ? geo.moments + bp.fo : geo.moments;  // [2,H,W] at 2 fo
          fA[p] = __ldg(geo.alpha + q);
          fD[p] = __ldg(moments_f + q);
          fD2[p] = __ldg(moments_f + HW + q);
          medc[p] = __ldg(geo.median_contrib + q);
        }
      }
      int wmax = max(cont[0], cont[1]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
      if (wmax <= 0) continue;
      const int nch = (wmax + 31) >> 5;
      auto issue = [&](int c) {
        if (c >= 0 && c * 32 + lane < wmax)
          gather_record<SREC_BYTES>(recs + 5 * (size_t)__ldg(ids + c * 32 + lane),
                                    ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<SREC_BYTES> +
                                        lane * SREC_BYTES);
        cp_async_commit();
      };
#pragma unroll
      for (int r = 0; r < WALK_RING; r++) issue(nch - 1 - r);
      const float bx0 = (float)bp.rx0, bx1 = (float)(bp.rx0 + 7), by0 = (float)bp.ry0, by1 = (float)(bp.ry0 + 7);
      for (int c = nch - 1; c >= 0; c--) {
        const int n = surfel_compact(wait_chunk<SREC_BYTES>(ring_addr, c, lane), c * 32 + lane, wmax, bx0, bx1, by0,
                                     by1, list_addr, lane, true);
        for (int i = 0; i < n; i++) {
          const uint2 e = lds64u(list_addr + i * 8);
          const int idx = (int)e.y;
          SRecRegs r;
          load_srec(e.x, r);
          float gM[9], gd[2] = {0.f, 0.f}, gu[2] = {0.f, 0.f}, gal = 0.f, gc[3] = {0.f, 0.f, 0.f},
                gn[3] = {0.f, 0.f, 0.f};
#pragma unroll
          for (int k = 0; k < 9; k++) gM[k] = 0.f;
          bool any = false;
#pragma unroll
          for (int p = 0; p < 2; p++) {
            sf::PixEval pe;
            float g;
            bool clamped;
            const float ap = surfel_alpha(r, xs[p], y, pe, g, clamped);
            if (idx < cont[p] && ap >= ALPHA_SKIP) {
              any = true;
              tau[p] = tau[p] / (1.0f - ap);
              const float *dp = d[p];
              float v = fmaf(dp[0], r.col[0], fmaf(dp[1], r.col[1], fmaf(dp[2], r.col[2],
                        fmaf(dp[3], pe.z, fmaf(dp[5], r.n[0], fmaf(dp[6], r.n[1], fmaf(dp[7], r.n[2], dp[4])))))));
              float m = 0.f;
              if constexpr (GEO) {
                m = geo_m(pe.z, geo.near, geo.mscale);
                v = fmaf(gdist[p], fmaf(m, fmaf(m, fA[p], -2.0f * fD[p]), fD2[p]), v);
              }
              const float diff = v - sdot[p];
              sdot[p] = fmaf(ap, diff, sdot[p]);
              const float dap = tau[p] * diff;  // dL/dalpha'
              const float w = tau[p] * ap;
#pragma unroll
              for (int k = 0; k < 3; k++) {
                gc[k] = fmaf(w, dp[k], gc[k]);
                gn[k] = fmaf(w, dp[5 + k], gn[k]);
              }
              float dG = 0.f;
              if (!clamped) {
                gal = fmaf(dap, g, gal);
                dG = -0.5f * dap * ap;
              }
              float dz = w * dp[3];
              if constexpr (GEO) {
                dz = fmaf(2.0f * gdist[p] * w * fmaf(m, fA[p], -fD[p]), geo_dm(pe.z, geo.near, geo.mscale), dz);
                if (idx == medc[p] - 1) dz += gmed[p];
              }
              sf::pixel_grad(r.M, xs[p], y, pe, dG, dz, gM, gd, gu);
            }
          }
          if (!__any_sync(0xffffffffu, any)) continue;
          // the (record, block) sums: butterfly over the warp, then one row update from lane 0
          float v[20];
#pragma unroll
          for (int k = 0; k < 9; k++) v[k] = gM[k];
          v[9] = gal; v[10] = gc[0]; v[11] = gc[1]; v[12] = gc[2];
          v[13] = gn[0]; v[14] = gn[1]; v[15] = gn[2]; v[16] = gd[0]; v[17] = gd[1]; v[18] = gu[0]; v[19] = gu[1];
#pragma unroll
          for (int k = 0; k < 20; k++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
          }
          if (lane == 0) {
            const float gu2[2] = {v[18], v[19]};
            sf::fold_du(r.M, gu2, v);
            float *row = rows + (size_t)__ldg(ids + idx) * sf::kRowFloats;
#pragma unroll
            for (int k = 0; k < sf::kRowFloats; k++)
              if (v[k] != 0.f) atomicAdd(row + k, v[k]);
          }
        }
        __syncwarp();  // every lane is done with this ring slot and with the list
        issue(c - WALK_RING);
      }
      walk_drain();
    }
  }
}

__global__ void __launch_bounds__(128, DRAW_SURFEL_BWD_MINBLOCKS) k_draw_surfel_bwd(
    int W, int H, int gx, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    SurfelGrads dl, float *__restrict__ rows, int *__restrict__ work) {
  draw_bwd_walk<false, false>(W, H, gx, 0, ranges, recs, gsid, contrib, final_tau, dl, GeoGrads{}, rows, work);
}

// the upstream planes of k_draw_2dgs_bwd: k_draw_surfel_bwd's and the geometry terms' (one struct,
// so the kernel's name stays its own)
struct GeoBwdArgs {
  SurfelGrads dl;
  GeoGrads geo;
};

__global__ void __launch_bounds__(128, DRAW_2DGS_BWD_MINBLOCKS) k_draw_2dgs_bwd(
    int W, int H, int gx, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    GeoBwdArgs a, float *__restrict__ rows, int *__restrict__ work) {
  draw_bwd_walk<true, false>(W, H, gx, 0, ranges, recs, gsid, contrib, final_tau, a.dl, a.geo, rows, work);
}

// the batched backward rasterizers (DESIGN 3.25): rows [C N, 18], one per record of the tall frame
__global__ void __launch_bounds__(128, DRAW_SURFEL_BWD_MINBLOCKS) k_draw_disk_bwd_batch(
    int W, int H, int gx, int gy, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    SurfelGrads dl, float *__restrict__ rows, int *__restrict__ work) {
  draw_bwd_walk<false, true>(W, H, gx, gy, ranges, recs, gsid, contrib, final_tau, dl, GeoGrads{}, rows, work);
}

__global__ void __launch_bounds__(128, DRAW_2DGS_BWD_MINBLOCKS) k_draw_2dgs_bwd_batch(
    int W, int H, int gx, int gy, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    GeoBwdArgs a, float *__restrict__ rows, int *__restrict__ work) {
  draw_bwd_walk<true, true>(W, H, gx, gy, ranges, recs, gsid, contrib, final_tau, a.dl, a.geo, rows, work);
}

// Contribution statistics of a drawn surfel frame (DESIGN 3.18): k_draw_stats' three reductions
// (raster_stats.cu) over the 80-byte records.  One CTA per tile, warp = 8x8 block, front to back to
// the block's largest contrib; a record reaches a pixel exactly when its patch index is below the
// pixel's contrib and alpha' >= 0.002 (k_draw_surfel's stop rule: tau only falls, so every record
// before the last contributing one met tau >= 1e-4), and alpha' (surfel_alpha), tau and w are
// k_draw_surfel's fp32 operations, so the weights are its bits.  The record has no id word: the
// surfel's id is the patch list's entry at the survivor's patch index.
__global__ void __launch_bounds__(128, DRAW_STATS_2DGS_MINBLOCKS) k_draw_stats_2dgs(
    int W, int H, int gx, const int2 *__restrict__ ranges, const float4 *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, float *__restrict__ weight_sum,
    uint32_t *__restrict__ weight_max, unsigned long long *__restrict__ hit_count) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<SREC_BYTES>];
  __shared__ __align__(16) uint2 s_list[4][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned F = 0xffffffffu;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const int tile = blockIdx.x;
  const int2 range = __ldg(ranges + tile);
  const int len = range.y - range.x;
  const int32_t *ids = gsid + range.x;
  BlockPix bp;
  if (len <= 0 || !block_pix<false>(W, H, gx, 0, tile, warp, lane, bp)) return;
  const float xs[2] = {(float)bp.px, (float)(bp.px + 1)}, y = (float)bp.py;
  const int cont[2] = {bp.in0 ? min(__ldg(contrib + bp.pix), len) : 0,
                       bp.in1 ? min(__ldg(contrib + bp.pix + 1), len) : 0};
  int wmax = max(cont[0], cont[1]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(F, wmax, o));
  if (wmax <= 0) return;
  const int nch = (wmax + 31) >> 5;
  auto issue = [&](int c) {
    if (c < nch && c * 32 + lane < wmax)
      gather_record<SREC_BYTES>(recs + 5 * (size_t)__ldg(ids + c * 32 + lane),
                                ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<SREC_BYTES> + lane * SREC_BYTES);
    cp_async_commit();
  };
#pragma unroll
  for (int r = 0; r < WALK_RING; r++) issue(r);
  const float bx0 = (float)bp.rx0, bx1 = (float)(bp.rx0 + 7), by0 = (float)bp.ry0, by1 = (float)(bp.ry0 + 7);
  float tau[2] = {1.0f, 1.0f};
  for (int c = 0; c < nch; c++) {
    const int n = surfel_compact(wait_chunk<SREC_BYTES>(ring_addr, c, lane), c * 32 + lane, wmax, bx0, bx1, by0, by1,
                                 list_addr, lane, false);
    for (int i = 0; i < n; i++) {
      const uint2 e = lds64u(list_addr + i * 8);
      SRecRegs r;
      load_srec(e.x, r);
      float w[2];
#pragma unroll
      for (int p = 0; p < 2; p++) {
        sf::PixEval pe;
        float g;
        bool clamped;
        const float ap = surfel_alpha(r, xs[p], y, pe, g, clamped);
        w[p] = 0.0f;
        if ((int)e.y < cont[p] && ap >= ALPHA_SKIP) {
          w[p] = tau[p] * ap;
          tau[p] = tau[p] * (1.0f - ap);
        }
      }
      const unsigned cnt = __reduce_add_sync(F, (unsigned)(w[0] > 0.0f) + (unsigned)(w[1] > 0.0f));
      if (cnt == 0) continue;  // warp-uniform
      const unsigned mx = __reduce_max_sync(F, max(__float_as_uint(w[0]), __float_as_uint(w[1])));
      float s = w[0] + w[1];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(F, s, o);
      if (lane == 0) {
        const int id = __ldg(ids + (int)e.y);
        atomicAdd(weight_sum + id, s);
        atomicMax(weight_max + id, mx);
        atomicAdd(hit_count + id, (unsigned long long)cnt);
      }
    }
    __syncwarp();  // every lane is done with this ring slot and with the list
    issue(c + WALK_RING);
  }
  walk_drain();
}

// ---- launchers

#define GSB_SURFEL_K3(k3, CALL)                                           \
  switch (k3) {                                                             \
    case 1: { constexpr int K3 = 1; CALL; } break;                          \
    case 4: { constexpr int K3 = 4; CALL; } break;                          \
    case 9: { constexpr int K3 = 9; CALL; } break;                          \
    case 16: { constexpr int K3 = 16; CALL; } break;                        \
    default: return set_arg_error("sh_dim3 must be 1, 4, 9 or 16");         \
  }

int launch_surfel_fwd(const FusedScene &sc, const float *alphas, float *us, float *depths, int32_t *areas, float *colors,
                      float *recs, cudaStream_t st) {
  const int N = sc.N;
  if (N <= 0) return 0;
  const int nb = (N + PG - 1) / PG;
  ProfScope ps(K_SURFEL_FWD, st);
  GSB_SURFEL_K3(sc.k3, (k_surfel_fwd<K3><<<nb, PG, 0, st>>>(N, sc.pws, sc.rots, sc.scales, sc.shs, sc.Rcw, sc.tcw,
                                                            sc.twc, sc.fx, sc.fy, sc.cx, sc.cy, alphas, us, depths,
                                                            areas, colors, reinterpret_cast<float4 *>(recs))));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_surfel_bwd(const FusedScene &sc, const float *rows, float *g_pws, float *g_shs, float *g_alphas,
                      float *g_scales, float *g_rots, float *g_us, cudaStream_t st) {
  const int N = sc.N;
  if (N <= 0) return 0;
  const int nb = (N + PG - 1) / PG;
  ProfScope ps(K_SURFEL_BWD, st);
  GSB_SURFEL_K3(sc.k3, (k_surfel_bwd<K3><<<nb, PG, 0, st>>>(N, sc.pws, sc.rots, sc.scales, sc.shs, sc.Rcw, sc.tcw,
                                                            sc.twc, sc.fx, sc.fy, sc.cx, sc.cy, rows, g_pws, g_shs,
                                                            g_alphas, g_scales, g_rots, g_us)));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_surfel_fwd_batch(const BatchScene &b, const float *alphas, float *us, float *depths, int32_t *areas,
                            float *colors, float *recs, cudaStream_t st) {
  if (b.N <= 0) return 0;
  const int nb = (b.N + PG - 1) / PG;
  ProfScope ps(K_SURFEL_FWD_BATCH, st);
  GSB_SURFEL_K3(b.k3, (k_disk_fwd_batch<K3><<<nb, PG, 0, st>>>(b.C, b.N, b.pws, b.rots, b.scales, b.shs, b.poses,
                                                               *b.cams, alphas, us, depths, areas, colors,
                                                               reinterpret_cast<float4 *>(recs))));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_surfel_bwd_batch(const BatchScene &b, const float *rows, float *g_pws, float *g_shs, float *g_alphas,
                            float *g_scales, float *g_rots, float *g_us, cudaStream_t st) {
  if (b.N <= 0) return 0;
  const int nb = (b.N + PG - 1) / PG;
  ProfScope ps(K_SURFEL_BWD_BATCH, st);
  GSB_SURFEL_K3(b.k3, (k_disk_bwd_batch<K3><<<nb, PG, 0, st>>>(b.C, b.N, b.pws, b.rots, b.scales, b.shs, b.poses,
                                                               *b.cams, rows, g_pws, g_shs, g_alphas, g_scales, g_rots,
                                                               g_us)));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_draw_surfel(int H, int W, const int32_t *ranges, const float *recs, const int32_t *gsid, float *image,
                       int32_t *contrib, float *final_tau, float *depth_image, float *alpha_image, float *normal_image,
                       const GeoPlanes *geo, int *work, cudaStream_t st, int frames) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0) return 0;
  if (work == nullptr) return set_arg_error("draw_surfel: work area missing");
  // the normal (and geometry) planes of empty tiles, of every frame: k_tile_list zeroes the other
  // five planes
  const size_t HW = (size_t)H * W * (frames > 0 ? frames : 1);
  GSB_CUDA_TRY(cudaMemsetAsync(normal_image, 0, sizeof(float) * 3 * HW, st));
  if (geo) {
    GSB_CUDA_TRY(cudaMemsetAsync(geo->distortion, 0, sizeof(float) * HW, st));
    GSB_CUDA_TRY(cudaMemsetAsync(geo->moments, 0, sizeof(float) * 2 * HW, st));
    GSB_CUDA_TRY(cudaMemsetAsync(geo->median_depth, 0, sizeof(float) * HW, st));
    GSB_CUDA_TRY(cudaMemsetAsync(geo->median_contrib, 0, sizeof(int32_t) * HW, st));
  }
  int rc = launch_tile_list(H, W, ranges, image, contrib, final_tau, depth_image, alpha_image, work, st, frames);
  if (rc || recs == nullptr) return rc;
  int grid = 0;
  rc = persistent_grid(gx * gy * (frames > 0 ? frames : 1), DRAW_SURFEL_MINBLOCKS, grid);
  if (rc) return rc;
  const int2 *r2 = reinterpret_cast<const int2 *>(ranges);
  const float4 *r4 = reinterpret_cast<const float4 *>(recs);
  if (frames > 0 && geo) {
    ProfScope ps(K_DRAW_2DGS_BATCH, st);
    k_draw_2dgs_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, r2, r4, gsid, image, contrib, final_tau, depth_image,
                                            alpha_image, normal_image, *geo, work);
  } else if (frames > 0) {
    ProfScope ps(K_DRAW_SURFEL_BATCH, st);
    k_draw_disk_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, r2, r4, gsid, image, contrib, final_tau, depth_image,
                                            alpha_image, normal_image, work);
  } else if (geo) {
    ProfScope ps(K_DRAW_2DGS, st);
    k_draw_2dgs<<<grid, 128, 0, st>>>(W, H, gx, r2, r4, gsid, image, contrib, final_tau, depth_image, alpha_image,
                                      normal_image, *geo, work);
  } else {
    ProfScope ps(K_DRAW_SURFEL, st);
    k_draw_surfel<<<grid, 128, 0, st>>>(W, H, gx, r2, r4, gsid, image, contrib, final_tau, depth_image, alpha_image,
                                        normal_image, work);
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_draw_surfel_backward(int H, int W, int N, const int32_t *ranges, const float *recs, const int32_t *gsid,
                                const int32_t *contrib, const float *final_tau, const float *dl_image,
                                const float *dl_depth, const float *dl_alpha, const float *dl_normal,
                                const GeoGrads *geo, float *rows, int *work, cudaStream_t st, int frames) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || N <= 0) return 0;
  GSB_CUDA_TRY(cudaMemsetAsync(rows, 0, sizeof(float) * sf::kRowFloats * (size_t)N, st));
  if (recs == nullptr) return 0;
  const bool with_geo = geo != nullptr && (geo->distortion != nullptr || geo->median != nullptr);
  if (dl_image == nullptr && dl_depth == nullptr && dl_alpha == nullptr && dl_normal == nullptr && !with_geo) return 0;
  if (work == nullptr) return set_arg_error("draw_surfel_backward: work area missing");
  int rc = launch_tile_list(H, W, ranges, nullptr, nullptr, nullptr, nullptr, nullptr, work, st, frames);
  if (rc) return rc;
  int grid = 0;
  rc = persistent_grid(gx * gy * (frames > 0 ? frames : 1),
                       with_geo ? DRAW_2DGS_BWD_MINBLOCKS : DRAW_SURFEL_BWD_MINBLOCKS, grid);
  if (rc) return rc;
  const int2 *r2 = reinterpret_cast<const int2 *>(ranges);
  const float4 *r4 = reinterpret_cast<const float4 *>(recs);
  const SurfelGrads dl{dl_image, dl_depth, dl_alpha, dl_normal};
  if (frames > 0 && with_geo) {
    ProfScope ps(K_DRAW_2DGS_BWD_BATCH, st);
    k_draw_2dgs_bwd_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, r2, r4, gsid, contrib, final_tau, GeoBwdArgs{dl, *geo},
                                                rows, work);
  } else if (frames > 0) {
    ProfScope ps(K_DRAW_SURFEL_BWD_BATCH, st);
    k_draw_disk_bwd_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, r2, r4, gsid, contrib, final_tau, dl, rows, work);
  } else if (with_geo) {
    ProfScope ps(K_DRAW_2DGS_BWD, st);
    k_draw_2dgs_bwd<<<grid, 128, 0, st>>>(W, H, gx, r2, r4, gsid, contrib, final_tau, GeoBwdArgs{dl, *geo}, rows,
                                          work);
  } else {
    ProfScope ps(K_DRAW_SURFEL_BWD, st);
    k_draw_surfel_bwd<<<grid, 128, 0, st>>>(W, H, gx, r2, r4, gsid, contrib, final_tau, dl, rows, work);
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_draw_surfel_stats(int H, int W, const int32_t *ranges, const float *recs, const int32_t *gsid,
                             const int32_t *contrib, float *weight_sum, float *weight_max, int64_t *hit_count,
                             cudaStream_t st) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || recs == nullptr) return 0;  // no patches: nothing to add
  ProfScope ps(K_DRAW_SURFEL_STATS, st);
  k_draw_stats_2dgs<<<gx * gy, 128, 0, st>>>(W, H, gx, reinterpret_cast<const int2 *>(ranges),
                                               reinterpret_cast<const float4 *>(recs), gsid, contrib, weight_sum,
                                               reinterpret_cast<uint32_t *>(weight_max),
                                               reinterpret_cast<unsigned long long *>(hit_count));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
