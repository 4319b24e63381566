// Feature rasterizers: per-Gaussian feature vectors f_i in R^D composited with the image's weights,
//   F[c, p] = sum_i w_i(p) f_i[c],   w_i(p) = tau_i(p) alpha'_i(p),
// and the backward of that map.  Both are replays over the colour forward's binning (ranges, the
// sorted patch list, the packed 48-byte records) and its per-pixel state (contrib, final_tau); the
// colour rasterizers (raster_fwd.cu, raster_bwd.cu) are not changed.  One launch composites G
// channels (G = 8, or 4 for a last group of at most 4 channels), so D channels take ceil(D / 8)
// replays or fewer.
//
// Mapping: the rasterizers' own, through the record walk of raster_walk.cuh.  A surviving record's
// G feature floats are loaded by the lane that gathered it into a small per-warp shared table next
// to the survivor list.
//
// Weights: a record contributes to a pixel exactly when its patch index is below the pixel's
// contrib and alpha' >= 0.002 -- the forward's skip and stop rules, since tau >= 1e-4 holds for every
// record before the last contributing one -- so both passes walk only to the block's largest
// contrib.  alpha' (raster_eval.cuh), tau and w = tau alpha' are the same fp32 operation sequence
// as k_draw's, so a feature equal to a colour channel composites to the image's bits.
//
// Backward (k_draw_feat_bwd), as k_draw_bwd: phase A replays back to front from final_tau with the
// feature recurrence s <- alpha' (dL/dF . f) + (1 - alpha') s, dL/dalpha' = tau (dL/dF . f - s), and
// leaves w = dL/dalpha' alpha' and wc = tau alpha' per (pixel, record) in shared memory.  Phase B
// (feat_flush): four lanes per record sum over the block's 64 pixels the six moments
//   w dx, w dy, w dx^2, w dx dy, w dy^2, dL/dalpha' g
// -- added to moment rows 0-5 in exactly k_draw_bwd's form (row 5 = (sum w) / alpha, the clamped
// records reduced in phase A), so the unchanged conversion (k_finalize_grads or the fused
// per-Gaussian backward) yields the summed gradients -- and the G sums wc dL/dF[c], added to
// dL/dfeatures[id, c] with scalar float atomics (DESIGN 3.10).
#include "common.cuh"
#include "kernels.h"
#include "raster_walk.cuh"
#include "tile_io.cuh"

namespace gsb {

constexpr int FEAT_G = 8;     // channels per replay (a last group of <= 4 channels takes the G = 4 form)
// CTAs per SM, the most that build without spills (-Xptxas -v): the forward at 71 / 68 registers
// (G = 8 / 4); the backward keeps dL/dF of both pixels in registers through phase A and its 6 + G
// sums in phase B (152 / 121 registers)
#ifndef DRAW_FEAT_MINBLOCKS
#define DRAW_FEAT_MINBLOCKS 7
#endif
template <int G>
constexpr int feat_bwd_minblocks() { return G == 4 ? 4 : 3; }

namespace {
__device__ __forceinline__ void sts128f(uint32_t a, float x, float y, float z, float w) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}

// channels c0 .. c0 + G - 1 of Gaussian `id` (0 past D) into the feature table entry at `dst`
template <int G>
__device__ __forceinline__ void load_features(uint32_t dst, const float *__restrict__ features, int D, int c0, int id) {
  const float *src = features + (size_t)id * D + c0;
  float v[G];
#pragma unroll
  for (int k = 0; k < G; k++) v[k] = c0 + k < D ? __ldg(src + k) : 0.0f;
#pragma unroll
  for (int k = 0; k < G; k += 4) sts128f(dst + 4 * k, v[k], v[k + 1], v[k + 2], v[k + 3]);
}
template <int G>
__device__ __forceinline__ void zero_features(uint32_t dst) {
#pragma unroll
  for (int k = 0; k < G; k += 4) sts128f(dst + 4 * k, 0.f, 0.f, 0.f, 0.f);
}

// Zeros of channels c0 .. c0 + G - 1 on the tiles without patches: one warp per tile, grid-stride
// (a lane writes 8 pixels of one row, 16-byte stores where the row allows).
template <int G>
__device__ __forceinline__ void zero_empty_tiles(int W, int H, int gx, int T, int D, int c0,
                                                 const int32_t *__restrict__ ranges, float *__restrict__ image) {
  const int lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  for (int t = blockIdx.x * 4 + (threadIdx.x >> 5); t < T; t += gridDim.x * 4) {
    const int2 r = ld_pair(ranges, t);
    if (r.y > r.x) continue;
    const int x0 = (t % gx) * TILE + (lane & 1) * 8, y = (t / gx) * TILE + (lane >> 1);
    if (y >= H || x0 >= W) continue;
    const size_t pix = (size_t)y * W + x0;
#pragma unroll
    for (int k = 0; k < G; k++) {
      if (c0 + k >= D) break;
      float *plane = image + (size_t)(c0 + k) * HW;
      if ((W & 3) == 0 && x0 + 8 <= W) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4 *>(plane + pix) = z;
        *reinterpret_cast<float4 *>(plane + pix + 4) = z;
      } else {
        for (int x = x0; x < min(x0 + 8, W); x++) plane[(size_t)y * W + x] = 0.f;
      }
    }
  }
}

// the lane's two pixels of channels c0 .. c0 + G - 1 (pair store when both are in and W is even)
template <int G>
__device__ __forceinline__ void store_pixels(float *__restrict__ image, size_t HW, size_t pix, int D, int c0, bool in0,
                                             bool in1, bool vec2, const float2 *acc) {
#pragma unroll
  for (int k = 0; k < G; k++) {
    if (c0 + k >= D) break;
    float *plane = image + (size_t)(c0 + k) * HW;
    if (in0 && in1 && vec2) {
      *reinterpret_cast<float2 *>(plane + pix) = acc[k];
    } else {
      if (in0) plane[pix] = acc[k].x;
      if (in1) plane[pix + 1] = acc[k].y;
    }
  }
}

// Phase B of the backward: the six moment sums and the G feature-gradient sums of up to 8 records
// over the warp's 8x8 block.  lane = slot * 4 + part; part covers x in [4 (part & 1), +4) of rows
// (part >> 1) + {0, 2, 4, 6} (k_draw_bwd's bwd_flush).  inf = record word q0 (u_x, u_y, id, alpha)
// of the lane's slot.  The 6 + G sums are reduced over the four parts with butterflies; part p then
// adds sums p, p + 4, ... (moment rows first, then dL/dfeatures[id, c0 + k]).
template <int G>
__device__ __forceinline__ void feat_flush(uint32_t w_addr, const float4 &inf, uint32_t dl_addr, int nslots,
                                           float fbx0, float fby0, int D, int c0, float *__restrict__ moments,
                                           float *__restrict__ dfeat, int lane) {
  const int slot = lane >> 2, part = lane & 3;
  const float U = inf.x - (fbx0 + (float)((part & 1) * 4));
  const float V = inf.y - (fby0 + (float)(part >> 1));
  const float2 dx01 = p2(U, U - 1.0f), dx23 = p2(U - 2.0f, U - 3.0f);
  const uint32_t a = w_addr + slot * WALK_SLOT_BYTES + part * 16;
  const uint32_t d = dl_addr + part * 16;
  float2 m0 = p2s(0.f), m1 = p2s(0.f), m2 = p2s(0.f), m3 = p2s(0.f), m4 = p2s(0.f), m5 = p2s(0.f);
  float2 mf[G];
#pragma unroll
  for (int k = 0; k < G; k++) mf[k] = p2s(0.f);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float dy = V - (float)(2 * j);
    const float dy2 = dy * dy;
    const float4 w = lds128(a + j * 64);
    const float4 wc = lds128(a + 256 + j * 64);
    const float2 t01 = mul2_rn(lo(w), dx01), t23 = mul2_rn(hi(w), dx23);
    const float2 r1 = add2_rn(t01, t23), r0 = add2_rn(lo(w), hi(w));
    m0 = add2_rn(m0, r1);
    m2 = fma2_rn(t01, dx01, m2);
    m2 = fma2_rn(t23, dx23, m2);
    m1 = fma2_rn(p2s(dy), r0, m1);
    m3 = fma2_rn(p2s(dy), r1, m3);
    m4 = fma2_rn(p2s(dy2), r0, m4);
    m5 = add2_rn(m5, r0);
#pragma unroll
    for (int k = 0; k < G; k++) {
      const float4 dk = lds128(d + k * 256 + j * 64);
      mf[k] = fma2_rn(lo(wc), lo(dk), mf[k]);
      mf[k] = fma2_rn(hi(wc), hi(dk), mf[k]);
    }
  }
  // sum dL/dalpha' g = (sum w) / alpha; records above the clamp were reduced in phase A
  const float inv_alpha = inf.w <= ALPHA_CLAMP ? __fdividef(1.0f, inf.w) : 0.0f;
  float v[6 + G] = {m0.x + m0.y, m1.x + m1.y, m2.x + m2.y, m3.x + m3.y, m4.x + m4.y, (m5.x + m5.y) * inv_alpha};
#pragma unroll
  for (int k = 0; k < G; k++) v[6 + k] = mf[k].x + mf[k].y;
  const unsigned F = 0xffffffffu;
#pragma unroll
  for (int q = 0; q < 6 + G; q++) {
    v[q] += __shfl_xor_sync(F, v[q], 1);
    v[q] += __shfl_xor_sync(F, v[q], 2);
  }
  if (slot < nslots) {
    const int id = __float_as_int(inf.z);
    float *row = moments + (size_t)id * 9;
    float *frow = dfeat + (size_t)id * D + c0;
#pragma unroll
    for (int q = 0; q < 6 + G; q++) {
      if ((q & 3) != part) continue;
      if (q < 6) {
        atomicAdd(row + q, v[q]);
      } else if (c0 + q - 6 < D) {
        atomicAdd(frow + q - 6, v[q]);
      }
    }
  }
}
}  // namespace

template <int G>
__global__ void __launch_bounds__(128, DRAW_FEAT_MINBLOCKS) k_draw_feat(
    int W, int H, int gx, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ features, int D,
    int c0, float *__restrict__ feature_image, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<>];  // gathered records, per warp
  __shared__ __align__(16) uint2 s_list[4][34];       // (record address, patch index) of a chunk's survivors
  __shared__ __align__(16) float s_feat[4][34][G];    // their features, same order
  __shared__ __align__(16) Rec s_dummy;               // all-zero record: pads an odd survivor count

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const bool vec2 = (W & 1) == 0;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const uint32_t feat_addr = opaque_u32(smem_u32(&s_feat[warp][0][0]));
  const uint32_t dummy_addr = smem_u32(&s_dummy);
  zero_dummy(s_dummy);
  zero_empty_tiles<G>(W, H, gx, T, D, c0, ranges, feature_image);
  const int items = work[1];
  const int *__restrict__ entries = work + 2;

  for (;;) {
    const int item = pull_item(work, lane);
    walk_drain();  // a whole-tile gather whose blocks all had nothing to composite was never waited for
    if (item >= items) break;
    const int ent = __ldg(entries + item);
    const int tile = ent >> 3, code = ent & 7;
    const bool whole_tile = code == 4;
    const int2 range = ld_pair(ranges, tile);
    const int len = range.y - range.x;
    if (whole_tile) gather_whole_tile(ring_addr, recs, gsid + range.x, len, lane);
    for (int blk = whole_tile ? 0 : code; blk < (whole_tile ? 4 : code + 1); blk++) {
      const int tx = tile % gx, ty = tile / gx;
      const int rx0 = tx * TILE + (blk & 1) * 8, ry0 = ty * TILE + (blk >> 1) * 8;
      if (rx0 >= W || ry0 >= H) continue;
      const int px = rx0 + 2 * (lane & 3), py = ry0 + (lane >> 2);
      const bool in0 = px < W && py < H, in1 = px + 1 < W && py < H;
      const size_t pix = (size_t)py * W + px;
      const int cont0 = in0 ? min(__ldg(contrib + pix), len) : 0;
      const int cont1 = in1 ? min(__ldg(contrib + pix + 1), len) : 0;
      int wmax = max(cont0, cont1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));

      float2 acc[G];
#pragma unroll
      for (int k = 0; k < G; k++) acc[k] = p2s(0.f);
      if (wmax > 0) {
        const int nch = (wmax + 31) >> 5;  // chunks [0, nch) hold every record a pixel of the block composites
        const int32_t *ids = gsid + range.x;
        auto issue = [&](int c, int id) {
          if (c < nch && c * 32 + lane < wmax)
            gather_record(recs + id, ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<> + lane * 48);
          cp_async_commit();
        };
        auto load_id = [&](int c) { return (c < nch && c * 32 + lane < wmax) ? __ldg(ids + c * 32 + lane) : 0; };
        int id_next = 0;
        if (!whole_tile) {
#pragma unroll
          for (int r = 0; r < WALK_RING; r++) issue(r, load_id(r));
          id_next = load_id(WALK_RING);
        }
        const float2 npx = p2(-(float)px, -(float)(px + 1));
        const float fpy = (float)py;
        const float bx0 = (float)rx0, bx1 = (float)(rx0 + 7), by0 = (float)ry0, by1 = (float)(ry0 + 7);
        float2 tau = p2s(1.0f);

        for (int c = 0; c < nch; c++) {
          // survivors front to back: (record address, patch index) and their G features; the pad has
          // alpha 0, an index beyond every contrib and zero features
          const int n = cull_compact(
              wait_chunk(ring_addr, c, lane), c * 32 + lane, wmax, bx0, bx1, by0, by1, list_addr, dummy_addr, 0u,
              0x7fffffffu, lane,
              [&](int pos, const float4 &q0) {
                load_features<G>(feat_addr + pos * G * 4, features, D, c0, __float_as_int(q0.z));
              },
              [&](int n) { zero_features<G>(feat_addr + n * G * 4); });
          for (int i = 0; i < n; i += 2) {
            const uint4 ent2 = lds128u(list_addr + i * 8);
            const float4 q0a = lds128(ent2.x), q0b = lds128(ent2.z);
            const float4 q1a = lds128(ent2.x + 16), q1b = lds128(ent2.z + 16);
            const float2 apa = fwd_alpha(q0a, q1a, npx, fpy), apb = fwd_alpha(q0b, q1b, npx, fpy);
            const uint32_t fa = feat_addr + i * G * 4, fb = fa + G * 4;
            {  // first record (k_draw's weight: w = tau e, tau <- tau (1 - e))
              const bool c0a = ((int)ent2.y < cont0) && (apa.x >= ALPHA_SKIP);
              const bool c1a = ((int)ent2.y < cont1) && (apa.y >= ALPHA_SKIP);
              const float2 e = p2(c0a ? apa.x : 0.0f, c1a ? apa.y : 0.0f);
              const float2 w = mul2_rn(tau, e);
#pragma unroll
              for (int k = 0; k < G; k += 4) {
                const float4 f = lds128(fa + 4 * k);
                acc[k] = fma2_rn(w, p2s(f.x), acc[k]);
                acc[k + 1] = fma2_rn(w, p2s(f.y), acc[k + 1]);
                acc[k + 2] = fma2_rn(w, p2s(f.z), acc[k + 2]);
                acc[k + 3] = fma2_rn(w, p2s(f.w), acc[k + 3]);
              }
              tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
            }
            {  // second record (the pad record when the count is odd)
              const bool c0b = ((int)ent2.w < cont0) && (apb.x >= ALPHA_SKIP);
              const bool c1b = ((int)ent2.w < cont1) && (apb.y >= ALPHA_SKIP);
              const float2 e = p2(c0b ? apb.x : 0.0f, c1b ? apb.y : 0.0f);
              const float2 w = mul2_rn(tau, e);
#pragma unroll
              for (int k = 0; k < G; k += 4) {
                const float4 f = lds128(fb + 4 * k);
                acc[k] = fma2_rn(w, p2s(f.x), acc[k]);
                acc[k + 1] = fma2_rn(w, p2s(f.y), acc[k + 1]);
                acc[k + 2] = fma2_rn(w, p2s(f.z), acc[k + 2]);
                acc[k + 3] = fma2_rn(w, p2s(f.w), acc[k + 3]);
              }
              tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
            }
          }
          __syncwarp();  // every lane is done with this ring slot, the list and the features
          issue(c + WALK_RING, id_next);
          id_next = load_id(c + WALK_RING + 1);
        }
        walk_drain();
      }
      store_pixels<G>(feature_image, HW, pix, D, c0, in0, in1, vec2, acc);
    }
  }
}

template <int G>
__global__ void __launch_bounds__(128, feat_bwd_minblocks<G>()) k_draw_feat_bwd(
    int W, int H, int gx, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ features, int D, int c0, const float *__restrict__ dloss_dfeature_image,
    float *__restrict__ moments, float *__restrict__ dfeat, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<>];  // gathered records, per warp
  __shared__ __align__(16) unsigned char s_w[4][WALK_W_BYTES];                    // weight rows, per warp
  __shared__ __align__(16) float s_dl[4][G][64];       // dL/dF of the block, channel-major
  __shared__ __align__(16) uint2 s_list[4][34];        // (record address, patch index) of a chunk's survivors
  __shared__ __align__(16) float s_feat[4][34][G];     // their features, same order
  __shared__ __align__(16) Rec s_dummy;                // all-zero record: pads an odd survivor count

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t w_addr = opaque_u32(smem_u32(&s_w[warp][0]));
  const uint32_t dl_addr = opaque_u32(smem_u32(&s_dl[warp][0][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const uint32_t feat_addr = opaque_u32(smem_u32(&s_feat[warp][0][0]));
  const uint32_t dummy_addr = smem_u32(&s_dummy);
  zero_dummy(s_dummy);
  const int items = work[1];
  const int *__restrict__ entries = work + 2;

  // one flat loop over 8x8 blocks, a new work-list entry pulled when the current one is used up
  int tile = 0, len = 0, blk = 0, blk_end = 0;
  bool whole_tile = false;
  int2 range = make_int2(0, 0);
  for (;;) {
    if (blk == blk_end) {
      const int item = pull_item(work, lane);
      walk_drain();  // (an unused whole-tile gather: drained before the ring is reused)
      if (item >= items) break;
      const int ent = __ldg(entries + item);
      const int code = ent & 7;
      tile = ent >> 3;
      whole_tile = code == 4;
      range = ld_pair(ranges, tile);
      len = range.y - range.x;
      if (len <= 0) continue;
      blk = whole_tile ? 0 : code;
      blk_end = whole_tile ? 4 : code + 1;
      if (whole_tile) gather_whole_tile(ring_addr, recs, gsid + range.x, len, lane);
    }
    const int cur = blk++;
    const int tx = tile % gx, ty = tile / gx;
    const int rx0 = tx * TILE + (cur & 1) * 8, ry0 = ty * TILE + (cur >> 1) * 8;
    if (rx0 >= W || ry0 >= H) continue;
    const int px = rx0 + 2 * (lane & 3), py = ry0 + (lane >> 2);
    const bool in0 = px < W && py < H, in1 = px + 1 < W && py < H;
    const size_t pix = (size_t)py * W + px;

    int cont0 = 0, cont1 = 0;
    float2 tau = p2s(0.f);
    if (in0) { cont0 = min(__ldg(contrib + pix), len); tau.x = __ldg(final_tau + pix); }
    if (in1) { cont1 = min(__ldg(contrib + pix + 1), len); tau.y = __ldg(final_tau + pix + 1); }
    int wmax = max(cont0, cont1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (wmax <= 0) continue;
    float2 dl[G];  // dL/dF at the lane's two pixels (0 past D)
#pragma unroll
    for (int k = 0; k < G; k++) {
      dl[k] = p2s(0.f);
      if (c0 + k < D) {
        const float *plane = dloss_dfeature_image + (size_t)(c0 + k) * HW;
        if (in0) dl[k].x = __ldg(plane + pix);
        if (in1) dl[k].y = __ldg(plane + pix + 1);
      }
      sts64(dl_addr + k * 256 + lane * 8, dl[k]);  // phase B's table; the flush's __syncwarp orders it
    }

    const int nch = (wmax + 31) >> 5;
    const int32_t *ids = gsid + range.x;
    auto issue = [&](int c, int id) {
      if (c >= 0 && c * 32 + lane < wmax)
        gather_record(recs + id, ring_addr + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<> + lane * 48);
      cp_async_commit();
    };
    auto load_id = [&](int c) { return (c >= 0 && c * 32 + lane < wmax) ? __ldg(ids + c * 32 + lane) : 0; };
    int id_next = 0;
    if (!whole_tile) {
#pragma unroll
      for (int r = 0; r < WALK_RING; r++) issue(nch - 1 - r, load_id(nch - 1 - r));
      id_next = load_id(nch - 1 - WALK_RING);
    }

    const float2 npx = p2(-(float)px, -(float)(px + 1));
    const float fpy = (float)py;
    const float bx0 = (float)rx0, bx1 = (float)(rx0 + 7), by0 = (float)ry0, by1 = (float)(ry0 + 7);
    float2 sdot = p2s(0.f);  // dL/dF . F_next, per pixel
    uint32_t wa = w_addr + lane * 8;
    const uint32_t wa_pair_limit = w_addr + lane * 8 + (WALK_SLOTS - 2) * WALK_SLOT_BYTES;
    int to_my_slot = lane >> 2;
    float4 inf = make_float4(0.f, 0.f, 0.f, 1.f);

    for (int c = nch - 1; c >= 0; c--) {
      const uint32_t my_rec = wait_chunk(ring_addr, c, lane);
      const int my_idx = c * 32 + lane;
      bool hit = false;
      float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (my_idx < wmax) {
        q0 = lds128(my_rec);
        hit = rec_can_touch(q0, lds128(my_rec + 16), bx0, bx1, by0, by1);
      }
      // survivors back to front, and their features
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      const int n = __popc(mask);
      if (hit) {
        const int pos = __popc(mask & ~((2u << lane) - 1u));
        sts64u(list_addr + pos * 8, my_rec, (uint32_t)my_idx);
        load_features<G>(feat_addr + pos * G * 4, features, D, c0, __float_as_int(q0.z));
      }
      if (lane == 0) {
        sts64u(list_addr + n * 8, dummy_addr, 0x7fffffffu);
        zero_features<G>(feat_addr + n * G * 4);
      }
      __syncwarp();
      for (int i = 0; i < n; i += 2) {
        if (wa > wa_pair_limit) {  // no room for a pair
          __syncwarp();
          feat_flush<G>(w_addr, inf, dl_addr, (lane >> 2) - to_my_slot, bx0, by0, D, c0, moments, dfeat, lane);
          __syncwarp();
          wa = w_addr + lane * 8;
          to_my_slot = lane >> 2;
        }
        const uint4 ent = lds128u(list_addr + i * 8);  // ent.x / ent.z: the record further back first
        const float4 q0a = lds128(ent.x), q0b = lds128(ent.z);
        const float4 q1a = lds128(ent.x + 16), q1b = lds128(ent.z + 16);
        const BwdEval A = bwd_eval(q0a, q1a, npx, fpy, (int)ent.y, cont0, cont1);
        const BwdEval B = bwd_eval(q0b, q1b, npx, fpy, (int)ent.w, cont0, cont1);
        // dL/dF . f, last channel innermost (k_draw_bwd's order for the three colour channels)
        const uint32_t fa = feat_addr + i * G * 4, fb = fa + G * 4;
        float2 dfa = p2s(0.f), dfb = p2s(0.f);
#pragma unroll
        for (int k = G - 4; k >= 0; k -= 4) {
          const float4 f = lds128(fa + 4 * k), g = lds128(fb + 4 * k);
          if (k == G - 4) {
            dfa = mul2_rn(dl[k + 3], p2s(f.w));
            dfb = mul2_rn(dl[k + 3], p2s(g.w));
          } else {
            dfa = fma2_rn(dl[k + 3], p2s(f.w), dfa);
            dfb = fma2_rn(dl[k + 3], p2s(g.w), dfb);
          }
          dfa = fma2_rn(dl[k], p2s(f.x), fma2_rn(dl[k + 1], p2s(f.y), fma2_rn(dl[k + 2], p2s(f.z), dfa)));
          dfb = fma2_rn(dl[k], p2s(g.x), fma2_rn(dl[k + 1], p2s(g.y), fma2_rn(dl[k + 2], p2s(g.z), dfb)));
        }
        // first record
        tau = mul2_rn(tau, A.rc);
        const float2 diffa = add2_rn(dfa, p2(-sdot.x, -sdot.y));
        sdot = fma2_rn(A.e, diffa, sdot);
        const float2 dapa = mul2_rn(tau, diffa);
        sts64(wa, mul2_rn(dapa, A.e));       // w
        sts64(wa + 256, mul2_rn(A.e, tau));  // wc
        if (to_my_slot == 0) inf = q0a;
        // second record (the all-zero pad record when the count is odd: e = 0, weights 0)
        tau = mul2_rn(tau, B.rc);
        const float2 diffb = add2_rn(dfb, p2(-sdot.x, -sdot.y));
        sdot = fma2_rn(B.e, diffb, sdot);
        const float2 dapb = mul2_rn(tau, diffb);
        sts64(wa + WALK_SLOT_BYTES, mul2_rn(dapb, B.e));
        sts64(wa + WALK_SLOT_BYTES + 256, mul2_rn(B.e, tau));
        if (to_my_slot == 1) inf = q0b;
        if (fmaxf(q0a.w, q0b.w) > ALPHA_CLAMP) {  // opacity above the clamp: row 5 reduced here
          float va = q0a.w > ALPHA_CLAMP ? fmaf(A.e.x > 0.f ? dapa.x : 0.f, A.gg.x, (A.e.y > 0.f ? dapa.y : 0.f) * A.gg.y) : 0.0f;
          float vb = q0b.w > ALPHA_CLAMP ? fmaf(B.e.x > 0.f ? dapb.x : 0.f, B.gg.x, (B.e.y > 0.f ? dapb.y : 0.f) * B.gg.y) : 0.0f;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            va += __shfl_xor_sync(0xffffffffu, va, o);
            vb += __shfl_xor_sync(0xffffffffu, vb, o);
          }
          if (lane == 0 && va != 0.0f) atomicAdd(moments + (size_t)__float_as_int(q0a.z) * 9 + 5, va);
          if (lane == 0 && vb != 0.0f) atomicAdd(moments + (size_t)__float_as_int(q0b.z) * 9 + 5, vb);
        }
        const bool pair = i + 2 <= n;
        wa += pair ? 2 * WALK_SLOT_BYTES : WALK_SLOT_BYTES;
        to_my_slot -= pair ? 2 : 1;
      }
      __syncwarp();  // every lane is done with this ring slot, the list and the features
      issue(c - WALK_RING, id_next);
      id_next = load_id(c - WALK_RING - 1);
    }
    cp_async_wait<0>();
    if (wa != w_addr + lane * 8) {
      __syncwarp();
      feat_flush<G>(w_addr, inf, dl_addr, (lane >> 2) - to_my_slot, bx0, by0, D, c0, moments, dfeat, lane);
    }
    __syncwarp();  // the flush has read s_dl / s_w before the next block rewrites them
  }
}

FeatLayout feat_layout(int N, int H, int W, int64_t P, uintptr_t base) {
  FeatLayout L{};
  const size_t T = (size_t)((W + TILE - 1) / TILE) * (size_t)((H + TILE - 1) / TILE);
  auto up = [](uintptr_t x) { return (x + 255) & ~(uintptr_t)255; };
  L.recs = up(base) - base;  // (cp.async gathers the records 16 bytes at a time)
  L.work = L.recs + (size_t)up((P > 0 && N > 0 ? (size_t)N : 1) * sizeof(Rec));
  L.bytes = L.work + (4 * T + 2) * sizeof(int);  // launch_tile_list's work area
  return L;
}

int launch_draw_features(int H, int W, int D, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                         const int32_t *contrib, const float *features, float *feature_image, int *work,
                         cudaStream_t st) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || D <= 0) return 0;
  const int T = gx * gy;
  if (work == nullptr) return set_arg_error("draw_features: work area missing");
  if (recs == nullptr) {  // no patches: every tile is empty
    GSB_CUDA_TRY(cudaMemsetAsync(feature_image, 0, sizeof(float) * (size_t)D * H * W, st));
    return 0;
  }
  int rc = launch_tile_list(H, W, ranges, nullptr, nullptr, nullptr, nullptr, nullptr, work, st);
  if (rc) return rc;
  int grid = 0;
  rc = persistent_grid(T, DRAW_FEAT_MINBLOCKS, grid);
  if (rc) return rc;
  for (int c0 = 0; c0 < D; c0 += FEAT_G) {
    if (c0 > 0) GSB_CUDA_TRY(cudaMemsetAsync(work, 0, sizeof(int), st));  // the item counter, per replay
    ProfScope ps(K_DRAW_FEAT, st);
    if (D - c0 <= 4)
      k_draw_feat<4><<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib, features, D, c0, feature_image,
                                           work);
    else
      k_draw_feat<FEAT_G><<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib, features, D, c0,
                                                feature_image, work);
    GSB_CUDA_TRY(cudaGetLastError());
  }
  return 0;
}

int launch_draw_features_backward(int H, int W, int N, int D, const int32_t *ranges, const Rec *recs,
                                  const int32_t *gsid, const int32_t *contrib, const float *final_tau,
                                  const float *features, const float *dloss_dfeature_image, float *moments,
                                  float *dloss_dfeatures, int *work, cudaStream_t st) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || N <= 0 || D <= 0) return 0;
  GSB_CUDA_TRY(cudaMemsetAsync(dloss_dfeatures, 0, sizeof(float) * (size_t)N * D, st));
  if (recs == nullptr) return 0;  // nothing was drawn: no terms, zero feature gradients
  const int T = gx * gy;
  if (work == nullptr) return set_arg_error("draw_features_backward: work area missing");
  int rc = launch_tile_list(H, W, ranges, nullptr, nullptr, nullptr, nullptr, nullptr, work, st);
  if (rc) return rc;
  int grid4 = 0, grid = 0;
  rc = persistent_grid(T, feat_bwd_minblocks<4>(), grid4);
  if (rc == 0) rc = persistent_grid(T, feat_bwd_minblocks<FEAT_G>(), grid);
  if (rc) return rc;
  for (int c0 = 0; c0 < D; c0 += FEAT_G) {
    if (c0 > 0) GSB_CUDA_TRY(cudaMemsetAsync(work, 0, sizeof(int), st));
    ProfScope ps(K_DRAW_FEAT_BWD, st);
    if (D - c0 <= 4)
      k_draw_feat_bwd<4><<<grid4, 128, 0, st>>>(W, H, gx, ranges, recs, gsid, contrib, final_tau, features, D, c0,
                                               dloss_dfeature_image, moments, dloss_dfeatures, work);
    else
      k_draw_feat_bwd<FEAT_G><<<grid, 128, 0, st>>>(W, H, gx, ranges, recs, gsid, contrib, final_tau, features, D,
                                                    c0, dloss_dfeature_image, moments, dloss_dfeatures, work);
    GSB_CUDA_TRY(cudaGetLastError());
  }
  return 0;
}

}  // namespace gsb
