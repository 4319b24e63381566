// Forward tile rasterizer: warp-autonomous 8x8 blocks and a list-driven two-record loop.
//
// Every warp of the persistent grid walks its blocks' records by the protocol of raster_walk.cuh
// (work list, cp.async chunk ring, exact culling into a survivor list); the compositing loop walks
// the survivors two at a time (two independent alpha' chains in flight per warp).  A lane owns two
// horizontally adjacent pixels; the quadratic form, the alpha multiply and the compositing update
// are fp32 pair ops (common.cuh).  The backward (raster_bwd.cu) replays alpha' with the same
// operation sequence (raster_eval.cuh), so both take identical skip decisions.
// Replaces reference kernel.cu:152-271 (draw).
#include "common.cuh"
#include "kernels.h"
#include "raster_walk.cuh"
#include "tile_io.cuh"

namespace gsb {

#ifndef DRAW_MINBLOCKS
#define DRAW_MINBLOCKS 8
#endif

// Work list of the two rasterizers (work[0] = the kernels' item counter, work[1] = number of
// entries, work[2..] = entries): a tile with more than 32 patches contributes four entries
// `tile * 8 + block` (one 8x8 block each), a tile with 1..32 patches ONE entry `tile * 8 + 4` --
// the warp that pulls it gathers the tile's single chunk of records once and renders all four
// blocks from it (a block of a sparse tile is bounded by the latency of its queue pull, range
// load, id load and gather, not by work: this quarters them).  A tile without patches keeps
// image 0, contrib 0, tau 0 (kernel.cu:182-183): when outputs are given this pass writes those
// zeros itself with 16-byte stores -- one warp per empty tile -- so the sparse corner of BASELINE config 4
// (50k Gaussians at 4K: 32 400 tiles, most of them empty) costs one streaming pass over the
// frame instead of one queue item per 8x8 block.
// BATCH: a batch of frames binned as one tall frame (DESIGN 3.21): tile row r belongs to frame
// r / gy (gy = tile rows per frame), and its empty tiles are zeroed in that frame's planes.
template <bool BATCH>
__device__ __forceinline__ void tile_list_body(int W, int H, int gx, int gy, int T, const int32_t *__restrict__ ranges,
                                               float *__restrict__ image, int32_t *__restrict__ contrib,
                                               float *__restrict__ final_tau, float *__restrict__ depth_image,
                                               float *__restrict__ alpha_image, int *__restrict__ work) {
  __shared__ unsigned s_empty[8];  // per warp: which of its 32 tiles have no patches
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tile = blockIdx.x * 256 + threadIdx.x;  // phase 1: one thread per tile
  int len = 0;
  if (tile < T) {
    const int2 r = ld_pair(ranges, tile);  // splatB takes the ranges from its caller: any alignment
    len = r.y - r.x;
  }
  const bool has = len > 0;
  const int n_ent = !has ? 0 : (len <= 32 ? 1 : 4);
  int incl = n_ent;  // warp prefix sum of the entry counts -> one atomic per 32 tiles
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  const unsigned m = __ballot_sync(0xffffffffu, has);
  int base = 0;
  if (lane == 31 && incl) base = atomicAdd(work + 1, incl);
  base = __shfl_sync(0xffffffffu, base, 31) + incl - n_ent;
  if (n_ent == 1) work[2 + base] = tile * 8 + 4;
  if (n_ent == 4) {
#pragma unroll
    for (int b = 0; b < 4; b++) work[2 + base + b] = tile * 8 + b;
  }
  if (image == nullptr) return;
  if (lane == 0) s_empty[warp] = ~m;
  __syncthreads();
  // phase 2: the CTA's empty tiles, one warp per tile, 16-byte stores
  const size_t HW = (size_t)H * W;
  for (int w = 0; w < 8; w++) {
    unsigned e = s_empty[w];
    // warp `warp` takes every 8th empty tile of the CTA's list; simple static split
    for (int k = 0; e; k++) {
      const int bit = __ffs(e) - 1;
      e &= e - 1;
      if ((k & 7) != warp) continue;
      const int t = blockIdx.x * 256 + w * 32 + bit;
      if (t >= T) break;
      const int x0 = (t % gx) * TILE + (lane & 1) * 8, y = (BATCH ? t / gx % gy : t / gx) * TILE + (lane >> 1);
      if (y >= H || x0 >= W) continue;
      const size_t fo = BATCH ? (size_t)(t / gx / gy) * HW : 0;  // BATCH: the tile's frame in every [H,W] plane
      const size_t pix = fo + (size_t)y * W + x0;
      float *const image_f = image + 2 * fo;  // pix holds fo; the frame's [3,H,W] planes start at 3 fo
      if ((W & 3) == 0 && x0 + 8 <= W) {  // 8 pixels = two 16-byte stores per plane
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          *reinterpret_cast<float4 *>(image_f + pix + 4 * h) = z;
          *reinterpret_cast<float4 *>(image_f + HW + pix + 4 * h) = z;
          *reinterpret_cast<float4 *>(image_f + 2 * HW + pix + 4 * h) = z;
          *reinterpret_cast<int4 *>(contrib + pix + 4 * h) = make_int4(0, 0, 0, 0);
          *reinterpret_cast<float4 *>(final_tau + pix + 4 * h) = z;
          if (depth_image != nullptr) {  // (the RGB-D frame's D and A planes: zero too)
            *reinterpret_cast<float4 *>(depth_image + pix + 4 * h) = z;
            *reinterpret_cast<float4 *>(alpha_image + pix + 4 * h) = z;
          }
        }
      } else {
        for (int x = x0; x < min(x0 + 8, W); x++) {
          const size_t q = fo + (size_t)y * W + x;
          image_f[q] = 0.f; image_f[HW + q] = 0.f; image_f[2 * HW + q] = 0.f;
          contrib[q] = 0; final_tau[q] = 0.f;
          if (depth_image != nullptr) { depth_image[q] = 0.f; alpha_image[q] = 0.f; }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_tile_list(int W, int H, int gx, int T, const int32_t *__restrict__ ranges,
                                                   float *__restrict__ image, int32_t *__restrict__ contrib,
                                                   float *__restrict__ final_tau, float *__restrict__ depth_image,
                                                   float *__restrict__ alpha_image, int *__restrict__ work) {
  tile_list_body<false>(W, H, gx, 0, T, ranges, image, contrib, final_tau, depth_image, alpha_image, work);
}

__global__ void __launch_bounds__(256) k_tile_list_batch(int W, int H, int gx, int gy, int T,
                                                         const int32_t *__restrict__ ranges, float *__restrict__ image,
                                                         int32_t *__restrict__ contrib, float *__restrict__ final_tau,
                                                         float *__restrict__ depth_image,
                                                         float *__restrict__ alpha_image, int *__restrict__ work) {
  tile_list_body<true>(W, H, gx, gy, T, ranges, image, contrib, final_tau, depth_image, alpha_image, work);
}

int launch_tile_list(int H, int W, const int32_t *ranges, float *image, int32_t *contrib, float *final_tau,
                     float *depth_image, float *alpha_image, int *work, cudaStream_t st, int frames) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const int T = gx * gy * (frames > 0 ? frames : 1);
  GSB_CUDA_TRY(cudaMemsetAsync(work, 0, 2 * sizeof(int), st));
  if (frames > 0)
    k_tile_list_batch<<<(T + 255) / 256, 256, 0, st>>>(W, H, gx, gy, T, ranges, image, contrib, final_tau, depth_image,
                                                       alpha_image, work);
  else
    k_tile_list<<<(T + 255) / 256, 256, 0, st>>>(W, H, gx, T, ranges, image, contrib,
                                             final_tau, depth_image, alpha_image, work);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// The rasterizer's body, shared by the colour kernel (k_draw) and the RGB-D kernel (k_draw_rgbd).
// RGBD: depth and opacity composite like two more colour channels whose per-record values are
// z = q2.w and 1 -- D = sum w z, A = sum w with the image's weights w = tau alpha' -- two more
// pair accumulators and two more [H,W] planes.
// BATCH: the tall frame of a batch (DESIGN 3.21): tile row r is row r - f gy of frame f = r / gy; the
// pixels are that frame's own coordinates (the records' means are camera-local) and its planes are
// frame f of image[C,3,H,W], contrib / final_tau / depth / alpha [C,H,W].
template <bool RGBD, bool BATCH>
__device__ __forceinline__ void draw_body(int W, int H, int gx, int gy, int T, const int2 *__restrict__ ranges,
                                          const Rec *__restrict__ recs, const int32_t *__restrict__ gsid,
                                          float *__restrict__ image, int32_t *__restrict__ contrib,
                                          float *__restrict__ final_tau, float *__restrict__ depth_image,
                                          float *__restrict__ alpha_image, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<>];  // gathered records, per warp
  __shared__ __align__(16) uint2 s_list[4][34];  // (record address, patch index + 1) of a chunk's survivors
  __shared__ __align__(16) Rec s_dummy;          // all-zero record (alpha = 0): pads an odd survivor count

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const bool vec2 = (W & 1) == 0;  // pixel pairs are 8-byte aligned in every plane
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const uint32_t dummy_addr = smem_u32(&s_dummy);
  zero_dummy(s_dummy);
  (void)T;
  const int items = work[1];  // entries of the work list (k_tile_list)
  const int *__restrict__ entries = work + 2;

  for (;;) {
    const int item = pull_item(work, lane);
    if (item >= items) break;
    const int ent = __ldg(entries + item);
    const int tile = ent >> 3, code = ent & 7;
    const bool whole_tile = code == 4;  // <= 32 patches: this warp renders all four blocks from one gather
    const int2 range = __ldg(ranges + tile);
    const int len = range.y - range.x;
    if (whole_tile) gather_whole_tile(ring_addr, recs, gsid + range.x, len, lane);
   for (int blk = whole_tile ? 0 : code; blk < (whole_tile ? 4 : code + 1); blk++) {
    int tx = tile % gx, ty = tile / gx;
    size_t fo = 0;  // BATCH: offset of the tile's frame in every [H,W] plane
    if (BATCH) {
      const int f = ty / gy;
      ty -= f * gy;
      fo = (size_t)f * HW;
    }
    const int rx0 = tx * TILE + (blk & 1) * 8, ry0 = ty * TILE + (blk >> 1) * 8;
    if (rx0 >= W || ry0 >= H) continue;  // block entirely outside the image (BATCH: or in a pad row)
    const int px = rx0 + 2 * (lane & 3), py = ry0 + (lane >> 2);
    const bool in0 = px < W && py < H, in1 = px + 1 < W && py < H;
    const size_t pix = fo + (size_t)py * W + px;
    float *const image_f = image + 2 * fo;  // pix holds fo; the frame's [3,H,W] planes start at 3 fo

    float2 tau = p2s(0.f), cr = p2s(0.f), cg = p2s(0.f), cb = p2s(0.f);
    float2 cd = p2s(0.f), ca = p2s(0.f);  // RGBD only: D and A
    int cont0 = 0, cont1 = 0;
    if (len > 0) {  // (a tile without patches keeps image 0, contrib 0, tau 0: kernel.cu:182-183)
      const int nch = (len + 31) >> 5;
      const int32_t *ids = gsid + range.x;
      auto issue = [&](int c, int id) {
        if (c < nch && c * 32 + lane < len)
          gather_record(recs + id, ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<> + lane * 48);
        cp_async_commit();
      };
      auto load_id = [&](int c) { return (c < nch && c * 32 + lane < len) ? __ldg(ids + c * 32 + lane) : 0; };
      int id_next = 0;
      if (!whole_tile) {
#pragma unroll
        for (int r = 0; r < WALK_RING; r++) issue(r, load_id(r));
        id_next = load_id(WALK_RING);
      }

      const float2 npx = p2(-(float)px, -(float)(px + 1));
      const float fpy = (float)py;
      const float bx0 = (float)rx0, bx1 = (float)(rx0 + 7), by0 = (float)ry0, by1 = (float)(ry0 + 7);
      // a pixel is finished exactly when tau < 1e-4; pixels outside the image start finished
      tau = p2(in0 ? 1.0f : 0.0f, in1 ? 1.0f : 0.0f);

      for (int c = 0; c < nch; c++) {
        // survivors of the chunk, front to back, as (record address, patch index + 1); the pad
        // record has alpha = 0 and never contributes
        const int n = cull_compact(wait_chunk(ring_addr, c, lane), c * 32 + lane, len, bx0, bx1, by0, by1,
                                          list_addr, dummy_addr, 1u, 0u, lane, no_hit_work, no_pad_work);
        for (int i = 0; i < n; i += 2) {
          const uint4 ent = lds128u(list_addr + i * 8);
          const float4 q0a = lds128(ent.x), q0b = lds128(ent.z);
          const float4 q1a = lds128(ent.x + 16), q1b = lds128(ent.z + 16);
          const float4 q2a = lds128(ent.x + 32), q2b = lds128(ent.z + 32);
          const float2 apa = fwd_alpha(q0a, q1a, npx, fpy), apb = fwd_alpha(q0b, q1b, npx, fpy);
          {  // first record; a pixel that skips it composites alpha' = 0: w = 0, tau unchanged
            const bool c0 = (tau.x >= TAU_STOP) && (apa.x >= ALPHA_SKIP);
            const bool c1 = (tau.y >= TAU_STOP) && (apa.y >= ALPHA_SKIP);
            const float2 e = p2(c0 ? apa.x : 0.0f, c1 ? apa.y : 0.0f);
            const float2 w = mul2_rn(tau, e);
            cr = fma2_rn(w, p2s(q2a.x), cr);
            cg = fma2_rn(w, p2s(q2a.y), cg);
            cb = fma2_rn(w, p2s(q2a.z), cb);
            if (RGBD) {
              cd = fma2_rn(w, p2s(q2a.w), cd);
              ca = add2_rn(ca, w);
            }
            tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
            if (c0) cont0 = (int)ent.y;
            if (c1) cont1 = (int)ent.y;
          }
          {  // second record (the pad record when the count is odd)
            const bool c0 = (tau.x >= TAU_STOP) && (apb.x >= ALPHA_SKIP);
            const bool c1 = (tau.y >= TAU_STOP) && (apb.y >= ALPHA_SKIP);
            const float2 e = p2(c0 ? apb.x : 0.0f, c1 ? apb.y : 0.0f);
            const float2 w = mul2_rn(tau, e);
            cr = fma2_rn(w, p2s(q2b.x), cr);
            cg = fma2_rn(w, p2s(q2b.y), cg);
            cb = fma2_rn(w, p2s(q2b.z), cb);
            if (RGBD) {
              cd = fma2_rn(w, p2s(q2b.w), cd);
              ca = add2_rn(ca, w);
            }
            tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
            if (c0) cont0 = (int)ent.w;
            if (c1) cont1 = (int)ent.w;
          }
        }
        // per-warp early out: every pixel of the block has reached tau < 1e-4 (kernel.cu:256)
        const bool done = __all_sync(0xffffffffu, tau.x < TAU_STOP && tau.y < TAU_STOP);
        if (done) break;
        __syncwarp();  // every lane is done with this ring slot and with the list
        issue(c + WALK_RING, id_next);
        id_next = load_id(c + WALK_RING + 1);
      }
      walk_drain();
    }
    if (in0 && in1 && vec2) {
      *reinterpret_cast<float2 *>(image_f + pix) = cr;
      *reinterpret_cast<float2 *>(image_f + HW + pix) = cg;
      *reinterpret_cast<float2 *>(image_f + 2 * HW + pix) = cb;
      *reinterpret_cast<int2 *>(contrib + pix) = make_int2(cont0, cont1);
      *reinterpret_cast<float2 *>(final_tau + pix) = tau;
      if (RGBD) {
        *reinterpret_cast<float2 *>(depth_image + pix) = cd;
        *reinterpret_cast<float2 *>(alpha_image + pix) = ca;
      }
    } else {
      if (in0) {
        image_f[pix] = cr.x; image_f[HW + pix] = cg.x; image_f[2 * HW + pix] = cb.x;
        contrib[pix] = cont0; final_tau[pix] = tau.x;
        if (RGBD) { depth_image[pix] = cd.x; alpha_image[pix] = ca.x; }
      }
      if (in1) {
        image_f[pix + 1] = cr.y; image_f[HW + pix + 1] = cg.y; image_f[2 * HW + pix + 1] = cb.y;
        contrib[pix + 1] = cont1; final_tau[pix + 1] = tau.y;
        if (RGBD) { depth_image[pix + 1] = cd.y; alpha_image[pix + 1] = ca.y; }
      }
    }
   }  // blocks of the entry
  }
}

__global__ void __launch_bounds__(128, DRAW_MINBLOCKS) k_draw(int W, int H, int gx, int T,
                                                              const int2 *__restrict__ ranges,
                                                              const Rec *__restrict__ recs,
                                                              const int32_t *__restrict__ gsid,
                                                              float *__restrict__ image,
                                                              int32_t *__restrict__ contrib,
                                                              float *__restrict__ final_tau,
                                                              int *__restrict__ work) {
  draw_body<false, false>(W, H, gx, 0, T, ranges, recs, gsid, image, contrib, final_tau, nullptr, nullptr, work);
}

__global__ void __launch_bounds__(128, DRAW_MINBLOCKS) k_draw_rgbd(int W, int H, int gx, int T,
                                                                   const int2 *__restrict__ ranges,
                                                                   const Rec *__restrict__ recs,
                                                                   const int32_t *__restrict__ gsid,
                                                                   float *__restrict__ image,
                                                                   int32_t *__restrict__ contrib,
                                                                   float *__restrict__ final_tau,
                                                                   float *__restrict__ depth_image,
                                                                   float *__restrict__ alpha_image,
                                                                   int *__restrict__ work) {
  draw_body<true, false>(W, H, gx, 0, T, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                         work);
}

__global__ void __launch_bounds__(128, DRAW_MINBLOCKS) k_draw_batch(int W, int H, int gx, int gy, int T,
                                                                    const int2 *__restrict__ ranges,
                                                                    const Rec *__restrict__ recs,
                                                                    const int32_t *__restrict__ gsid,
                                                                    float *__restrict__ image,
                                                                    int32_t *__restrict__ contrib,
                                                                    float *__restrict__ final_tau,
                                                                    int *__restrict__ work) {
  draw_body<false, true>(W, H, gx, gy, T, ranges, recs, gsid, image, contrib, final_tau, nullptr, nullptr, work);
}

__global__ void __launch_bounds__(128, DRAW_MINBLOCKS) k_draw_rgbd_batch(int W, int H, int gx, int gy, int T,
                                                                         const int2 *__restrict__ ranges,
                                                                         const Rec *__restrict__ recs,
                                                                         const int32_t *__restrict__ gsid,
                                                                         float *__restrict__ image,
                                                                         int32_t *__restrict__ contrib,
                                                                         float *__restrict__ final_tau,
                                                                         float *__restrict__ depth_image,
                                                                         float *__restrict__ alpha_image,
                                                                         int *__restrict__ work) {
  draw_body<true, true>(W, H, gx, gy, T, ranges, recs, gsid, image, contrib, final_tau, depth_image, alpha_image,
                        work);
}

int launch_draw(int H, int W, const int32_t *ranges, const Rec *recs, const int32_t *gsid, float *image,
                int32_t *contrib, float *final_tau, float *depth_image, float *alpha_image, int *work,
                cudaStream_t st, int frames) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0) return 0;
  const int T = gx * gy * (frames > 0 ? frames : 1);
  if (work == nullptr) return set_arg_error("draw: work area missing");
  // (k_draw reads `ranges` as int2: the splat entry points only accept an 8-byte aligned
  // patch_range_per_tile, which the binning just wrote)
  // work list (and the zeros of the empty tiles) first; it also clears the item counter
  int rc = launch_tile_list(H, W, ranges, image, contrib, final_tau, depth_image, alpha_image, work, st, frames);
  if (rc) return rc;
  int grid = 0;
  rc = persistent_grid(T, DRAW_MINBLOCKS, grid);
  if (rc) return rc;
  if (frames > 0 && depth_image != nullptr) {
    ProfScope ps(K_DRAW_RGBD_BATCH, st);
    k_draw_rgbd_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, T, reinterpret_cast<const int2 *>(ranges), recs, gsid,
                                            image, contrib, final_tau, depth_image, alpha_image, work);
  } else if (frames > 0) {
    ProfScope ps(K_DRAW_BATCH, st);
    k_draw_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, T, reinterpret_cast<const int2 *>(ranges), recs, gsid, image,
                                       contrib, final_tau, work);
  } else if (depth_image != nullptr) {
    ProfScope ps(K_DRAW_RGBD, st);
    k_draw_rgbd<<<grid, 128, 0, st>>>(W, H, gx, T, reinterpret_cast<const int2 *>(ranges), recs, gsid, image,
                                      contrib, final_tau, depth_image, alpha_image, work);
  } else {
    ProfScope ps(K_DRAW, st);
    k_draw<<<grid, 128, 0, st>>>(W, H, gx, T, reinterpret_cast<const int2 *>(ranges), recs, gsid, image, contrib,
                                 final_tau, work);
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
