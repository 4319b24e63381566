// Contribution statistics (DESIGN 3.18): a replay of a frame the colour or RGB-D forward drew that
// sums, per Gaussian, what its blending weights w = tau alpha' were over the frame's pixels:
//   weight_sum[i] += sum_p w_i(p),   weight_max[i] = max(weight_max[i], max_p w_i(p)),
//   hit_count[i]  += #{p : w_i(p) > 0}.
// The replay is k_draw_feat's (raster_feat.cu) without the feature table: the record walk of
// raster_walk.cuh over the frame's ranges, sorted patch list and packed 48-byte records, to the
// block's largest contrib.  A record reaches a pixel exactly when its patch index is below the
// pixel's contrib and alpha' >= 0.002, and alpha' (raster_eval.cuh), tau and w are k_draw's fp32
// operation sequence, so every w is the bit pattern k_draw composited.
//
// Per (surviving record, 8x8 block) the warp reduces its 64 weights once: a shuffle tree for the
// sum, redux.sync on the weights' bits for the maximum (w >= 0, so the uint order of the bits is the
// float order), redux.sync for the count; lane 0 then adds them with one atomic each, only when the
// count is non-zero.  The maximum and the count are exact and independent of the order of the
// atomics; the sum is an fp32 sum in atomic order.
#include "common.cuh"
#include "kernels.h"
#include "raster_walk.cuh"
#include "tile_io.cuh"

namespace gsb {

// CTAs per SM: 55 registers and 13.1 KiB of shared memory without spills (-Xptxas -v, nvcc 12.9);
// 8 x 128 threads x 56 registers fit the 64K register file
#ifndef DRAW_STATS_MINBLOCKS
#define DRAW_STATS_MINBLOCKS 8
#endif

namespace {
// the warp's reductions of one record's weights at its 64 pixels, and lane 0's atomics
__device__ __forceinline__ void stats_add(float2 w, int id, float *__restrict__ weight_sum,
                                          uint32_t *__restrict__ weight_max,
                                          unsigned long long *__restrict__ hit_count, int lane) {
  const unsigned F = 0xffffffffu;
  const unsigned cnt = __reduce_add_sync(F, (unsigned)(w.x > 0.0f) + (unsigned)(w.y > 0.0f));
  if (cnt == 0) return;  // warp-uniform
  const unsigned mx = __reduce_max_sync(F, max(__float_as_uint(w.x), __float_as_uint(w.y)));
  float s = w.x + w.y;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(F, s, o);
  if (lane == 0) {
    atomicAdd(weight_sum + id, s);
    atomicMax(weight_max + id, mx);
    atomicAdd(hit_count + id, (unsigned long long)cnt);
  }
}
}  // namespace

__global__ void __launch_bounds__(128, DRAW_STATS_MINBLOCKS) k_draw_stats(
    int W, int H, int gx, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, float *__restrict__ weight_sum,
    uint32_t *__restrict__ weight_max, unsigned long long *__restrict__ hit_count, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<>];  // gathered records, per warp
  __shared__ __align__(16) uint2 s_list[4][34];       // (record address, patch index) of a chunk's survivors
  __shared__ __align__(16) Rec s_dummy;               // all-zero record: pads an odd survivor count

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const uint32_t dummy_addr = smem_u32(&s_dummy);
  zero_dummy(s_dummy);
  const int items = work[1];
  const int *__restrict__ entries = work + 2;

  for (;;) {
    const int item = pull_item(work, lane);
    walk_drain();  // a whole-tile gather whose blocks all had nothing to replay was never waited for
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
      if (wmax <= 0) continue;

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
        // survivors front to back; the pad has alpha 0 and an index beyond every contrib
        const int n = cull_compact(wait_chunk(ring_addr, c, lane), c * 32 + lane, wmax, bx0, bx1, by0, by1, list_addr,
                                   dummy_addr, 0u, 0x7fffffffu, lane, no_hit_work, no_pad_work);
        for (int i = 0; i < n; i += 2) {
          const uint4 ent2 = lds128u(list_addr + i * 8);
          const float4 q0a = lds128(ent2.x), q0b = lds128(ent2.z);
          const float4 q1a = lds128(ent2.x + 16), q1b = lds128(ent2.z + 16);
          const float2 apa = fwd_alpha(q0a, q1a, npx, fpy), apb = fwd_alpha(q0b, q1b, npx, fpy);
          {  // first record (k_draw's weight: w = tau e, tau <- tau (1 - e))
            const bool c0a = ((int)ent2.y < cont0) && (apa.x >= ALPHA_SKIP);
            const bool c1a = ((int)ent2.y < cont1) && (apa.y >= ALPHA_SKIP);
            const float2 e = p2(c0a ? apa.x : 0.0f, c1a ? apa.y : 0.0f);
            stats_add(mul2_rn(tau, e), __float_as_int(q0a.z), weight_sum, weight_max, hit_count, lane);
            tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
          }
          {  // second record (the pad record when the count is odd: no hits, nothing added)
            const bool c0b = ((int)ent2.w < cont0) && (apb.x >= ALPHA_SKIP);
            const bool c1b = ((int)ent2.w < cont1) && (apb.y >= ALPHA_SKIP);
            const float2 e = p2(c0b ? apb.x : 0.0f, c1b ? apb.y : 0.0f);
            stats_add(mul2_rn(tau, e), __float_as_int(q0b.z), weight_sum, weight_max, hit_count, lane);
            tau = mul2_rn(tau, add2_rn(p2s(1.0f), p2(-e.x, -e.y)));
          }
        }
        __syncwarp();  // every lane is done with this ring slot and the list
        issue(c + WALK_RING, id_next);
        id_next = load_id(c + WALK_RING + 1);
      }
      walk_drain();
    }
  }
}

int launch_draw_stats(int H, int W, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                      const int32_t *contrib, float *weight_sum, float *weight_max, int64_t *hit_count, int *work,
                      cudaStream_t st) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || recs == nullptr) return 0;  // no patches: nothing to add
  if (work == nullptr) return set_arg_error("draw_stats: work area missing");
  const int T = gx * gy;
  int rc = launch_tile_list(H, W, ranges, nullptr, nullptr, nullptr, nullptr, nullptr, work, st);
  if (rc) return rc;
  int grid = 0;
  rc = persistent_grid(T, DRAW_STATS_MINBLOCKS, grid);
  if (rc) return rc;
  ProfScope ps(K_DRAW_STATS, st);
  k_draw_stats<<<grid, 128, 0, st>>>(W, H, gx, ranges, recs, gsid, contrib, weight_sum,
                                     reinterpret_cast<uint32_t *>(weight_max),
                                     reinterpret_cast<unsigned long long *>(hit_count), work);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
