// Backward tile rasterizer ("drawB").  Replaces reference kernel.cu:809-950.
//
// The record walk of raster_walk.cuh, back to front from the last chunk any pixel of the block
// replays (max contrib), so a warp stops at its own block's last contributing record, not the
// tile's.  The records are read 4x (once per block) instead of once per tile; they come from L2.
//
// Phase A, pixel-parallel replay: each pixel replays its saved (final_tau, contrib) state:
// tau <- tau / (1 - alpha'), dL/dalpha' = tau (c - gamma_next) . dL/dgamma, with gamma_next kept as
// the scalar s = dL/dgamma . gamma_next (s <- alpha' (dL/dgamma . c) + (1 - alpha') s).  Two
// surviving records per iteration: their alpha' evaluations are independent chains (LDS -> FFMA ->
// ex2 -> min -> rcp), only the short tau / s recurrences are sequential, so an in-order warp
// overlaps their latencies.  Each (pixel, record) leaves two weights in shared memory,
// w = dL/dalpha' alpha' and wc = alpha' tau.
//
// Phase B, record-parallel moments (bwd_flush): geometry gradients are linear in per-pixel
// moments, so four lanes per record sum, over the block's 64 pixels, the nine numbers
//   w dx, w dy, w dx^2, w dx dy, w dy^2,  dL/dalpha' g,  wc dL/dgamma_rgb
// and add them into the Gaussian's contiguous 9-float moment row (red.global.add).
// k_finalize_grads turns moment rows into the four gradient tensors:
//   dL/du = -(A Sx + B Sy, B Sx + C Sy),  dL/dconic = (-Sxx/2, -Sxy, -Syy/2).
//
// The _abs kernels (absolute-gradient densification, DESIGN 3.13) also sum, per Gaussian, the
// absolute value of every pixel's term of dL/du: sum_p |w (A dx + B dy)|, sum_p |w (B dx + C dy)|.
// |.| is not linear, so these cannot come from the moment rows; phase B forms them from the same
// w it reads for the moments.
#include "common.cuh"
#include "kernels.h"
#include "raster_walk.cuh"
#include "tile_io.cuh"

namespace gsb {

#ifndef DRAW_BWD_MINBLOCKS
#define DRAW_BWD_MINBLOCKS 6
#endif
#ifndef DRAW_BWD_RGBD_MINBLOCKS
#define DRAW_BWD_RGBD_MINBLOCKS 5
#endif
// the _abs kernels: 96 registers and a small spill at 5 CTAs/SM, measured faster than 128
// registers without spills at 4 (DESIGN 3.13)
#ifndef DRAW_BWD_ABS_MINBLOCKS
#define DRAW_BWD_ABS_MINBLOCKS 5
#endif
#ifndef DRAW_BWD_RGBD_ABS_MINBLOCKS
#define DRAW_BWD_RGBD_ABS_MINBLOCKS 5
#endif

namespace {
__device__ __forceinline__ float2 abs2(float2 a) { return make_float2(fabsf(a.x), fabsf(a.y)); }

// Phase B: moment sums of up to 8 records over the warp's 8x8 block.
//   lane = slot * 4 + part; part covers x in [4 (part & 1), +4) of rows (part >> 1) + {0, 2, 4, 6}.
//   inf = record word q0 = (u_x, u_y, gaussian id, alpha) of the lane's slot.  It travels in registers:
//   shared-memory wavefronts are this kernel's scarcest resource, and a 16-byte shared store
//   costs 4 of them even from one lane (benchmarks/micro/redux_bench.cu).
//   RGBD: a tenth sum, wc dL/dD = dL/dz, over a fourth dL/d-plane at dl_addr + 768; it goes to
//   ddepths[id] from the part-3 lane (which carries only one other reduction).
//   ABS: cq = record word q1 = log2e (-A/2, -B, -C/2) of the slot, carried next to inf; two more sums
//   sum |w| |2 q1.x dx + q1.y dy|, sum |w| |q1.y dx + 2 q1.z dy|, scaled by 1/log2e once, go to
//   dus_abs[id] from the part-2 (x) and part-3 (y) lanes, which carry the fewest other reductions.
template <bool RGBD, bool ABS>
__device__ __forceinline__ void bwd_flush(uint32_t w_addr, const float4 &inf, const float4 &cq, uint32_t dl_addr,
                                          int nslots, float fbx0, float fby0, float *__restrict__ moments,
                                          float *__restrict__ ddepths, float *__restrict__ dus_abs, int lane) {
  const int slot = lane >> 2, part = lane & 3;
  const float U = inf.x - (fbx0 + (float)((part & 1) * 4));
  const float V = inf.y - (fby0 + (float)(part >> 1));
  const float2 dx01 = p2(U, U - 1.0f), dx23 = p2(U - 2.0f, U - 3.0f);
  const uint32_t a = w_addr + slot * WALK_SLOT_BYTES + part * 16;
  const uint32_t d = dl_addr + part * 16;
  float2 m0 = p2s(0.f), m1 = p2s(0.f), m2 = p2s(0.f), m3 = p2s(0.f), m4 = p2s(0.f), m5 = p2s(0.f),
         m6 = p2s(0.f), m7 = p2s(0.f), m8 = p2s(0.f), m9 = p2s(0.f);
  float2 ax = p2s(0.f), ay = p2s(0.f);  // ABS only
  const float cx2 = 2.0f * cq.x, cz2 = 2.0f * cq.z;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float dy = V - (float)(2 * j);
    const float dy2 = dy * dy;
    const float4 w = lds128(a + j * 64);
    const float4 wc = lds128(a + 256 + j * 64);
    const float4 dr = lds128(d + j * 64);
    const float4 dg = lds128(d + 256 + j * 64);
    const float4 db = lds128(d + 512 + j * 64);
    const float2 t01 = mul2_rn(lo(w), dx01), t23 = mul2_rn(hi(w), dx23);
    const float2 r1 = add2_rn(t01, t23), r0 = add2_rn(lo(w), hi(w));
    m0 = add2_rn(m0, r1);
    m2 = fma2_rn(t01, dx01, m2);
    m2 = fma2_rn(t23, dx23, m2);
    m1 = fma2_rn(p2s(dy), r0, m1);
    m3 = fma2_rn(p2s(dy), r1, m3);
    m4 = fma2_rn(p2s(dy2), r0, m4);
    m5 = add2_rn(m5, r0);
    m6 = fma2_rn(lo(wc), lo(dr), m6);
    m6 = fma2_rn(hi(wc), hi(dr), m6);
    m7 = fma2_rn(lo(wc), lo(dg), m7);
    m7 = fma2_rn(hi(wc), hi(dg), m7);
    m8 = fma2_rn(lo(wc), lo(db), m8);
    m8 = fma2_rn(hi(wc), hi(db), m8);
    if (RGBD) {
      const float4 dd = lds128(d + 768 + j * 64);
      m9 = fma2_rn(lo(wc), lo(dd), m9);
      m9 = fma2_rn(hi(wc), hi(dd), m9);
    }
    if (ABS) {
      const float2 bx = p2s(cq.y * dy), by = p2s(cz2 * dy);
      ax = add2_rn(ax, abs2(mul2_rn(lo(w), fma2_rn(p2s(cx2), dx01, bx))));
      ax = add2_rn(ax, abs2(mul2_rn(hi(w), fma2_rn(p2s(cx2), dx23, bx))));
      ay = add2_rn(ay, abs2(mul2_rn(lo(w), fma2_rn(p2s(cq.y), dx01, by))));
      ay = add2_rn(ay, abs2(mul2_rn(hi(w), fma2_rn(p2s(cq.y), dx23, by))));
    }
  }
  // sum dL/dalpha' g = (sum w) / alpha; records above the clamp were reduced in phase A
  const float inv_alpha = inf.w <= ALPHA_CLAMP ? __fdividef(1.0f, inf.w) : 0.0f;
  const float v[9] = {m0.x + m0.y, m1.x + m1.y, m2.x + m2.y, m3.x + m3.y, m4.x + m4.y,
                      (m5.x + m5.y) * inv_alpha, m6.x + m6.y, m7.x + m7.y, m8.x + m8.y};
  // split exchange between the four parts of a slot: part 0 -> v0 v1 v2, part 2 -> v3 v4,
  // part 1 -> v5 v6 v7, part 3 -> v8
  const unsigned F = 0xffffffffu;
  const bool u1 = part & 1, u2 = part & 2;
  float s[5], b[3];
#pragma unroll
  for (int i = 0; i < 4; i++) s[i] = (u1 ? v[i + 5] : v[i]) + __shfl_xor_sync(F, u1 ? v[i] : v[i + 5], 1);
  s[4] = (u1 ? 0.f : v[4]) + __shfl_xor_sync(F, u1 ? v[4] : 0.f, 1);
  b[0] = (u2 ? s[3] : s[0]) + __shfl_xor_sync(F, u2 ? s[0] : s[3], 2);
  b[1] = (u2 ? s[4] : s[1]) + __shfl_xor_sync(F, u2 ? s[1] : s[4], 2);
  b[2] = (u2 ? 0.f : s[2]) + __shfl_xor_sync(F, u2 ? s[2] : 0.f, 2);
  if (slot < nslots) {
    const int first = u1 ? (u2 ? 8 : 5) : (u2 ? 3 : 0);
    float *row = moments + (size_t)__float_as_int(inf.z) * 9 + first;
    atomicAdd(row, b[0]);
    if (part != 3) atomicAdd(row + 1, b[1]);
    if (!u2) atomicAdd(row + 2, b[2]);
  }
  if (RGBD) {
    float z = m9.x + m9.y;
    z += __shfl_xor_sync(F, z, 1);
    z += __shfl_xor_sync(F, z, 2);
    if (slot < nslots && part == 3) atomicAdd(ddepths + __float_as_int(inf.z), z);
  }
  if (ABS) {  // parts 0 and 2 gather the x sums, parts 1 and 3 the y sums
    const float sx = ax.x + ax.y, sy = ay.x + ay.y;
    float h = (u1 ? sy : sx) + __shfl_xor_sync(F, u1 ? sx : sy, 1);
    h += __shfl_xor_sync(F, h, 2);
    if (slot < nslots && u2)
      atomicAdd(dus_abs + (size_t)__float_as_int(inf.z) * 2 + (part & 1), h * (1.0f / LOG2E));
  }
}
}  // namespace

// The backward's body, shared by k_draw_bwd and k_draw_bwd_rgbd.  RGBD: the upstream gradient of a
// pixel also has dL/dD and dL/dA, so in phase A dL/dalpha' gains (dL/dD z + dL/dA) next to
// dL/dgamma . c (the sdot recurrence carries the sum of all five channels), and phase B sums
// wc dL/dD into dL/dz from a fourth per-pixel table.  dL/dA needs no table: opacity has no
// per-Gaussian value to differentiate.  ABS: the _abs kernels; phase A also keeps the lane's slot's
// record word q1 (the conic) for bwd_flush's absolute sums into dus_abs.  BATCH: the tall frame of a
// batch, as draw_body's BATCH (raster_fwd.cu): the per-pixel planes are frame r / gy's of [C,...,H,W].
template <bool RGBD, bool ABS, bool BATCH>
__device__ __forceinline__ void draw_bwd_body(
    int W, int H, int gx, int gy, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, const float *__restrict__ dloss_ddepth_image,
    const float *__restrict__ dloss_dalpha_image, float *__restrict__ moments, float *__restrict__ ddepths,
    float *__restrict__ dus_abs, int *__restrict__ work) {
  __shared__ __align__(16) unsigned char s_ring[4][WALK_RING * WALK_CHUNK_BYTES<>];  // gathered records, per warp
  __shared__ __align__(16) unsigned char s_w[4][WALK_W_BYTES];                   // weight rows, per warp
  __shared__ __align__(16) float s_dl[4][RGBD ? 4 : 3][64];                    // dL/dgamma (dL/dD) of the block
  __shared__ __align__(16) uint2 s_list[4][34];  // (record address, patch index) of a chunk's survivors
  __shared__ __align__(16) Rec s_dummy;          // all-zero record: pads an odd survivor count

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W;
  const uint32_t ring_addr = opaque_u32(smem_u32(&s_ring[warp][0]));
  const uint32_t w_addr = opaque_u32(smem_u32(&s_w[warp][0]));
  const uint32_t dl_addr = opaque_u32(smem_u32(&s_dl[warp][0][0]));
  const uint32_t list_addr = opaque_u32(smem_u32(&s_list[warp][0]));
  const uint32_t dummy_addr = smem_u32(&s_dummy);
  zero_dummy(s_dummy);
  (void)T;
  const int items = work[1];  // entries of the work list (k_tile_list, raster_fwd.cu)
  const int *__restrict__ entries = work + 2;

  // One flat loop over 8x8 blocks: a new work-list entry is pulled when the current one is used up
  // (an entry is one block of a dense tile, or all four blocks of a tile with <= 32 patches).
  int tile = 0, len = 0, blk = 0, blk_end = 0;
  bool whole_tile = false;
  int2 range = make_int2(0, 0);
  for (;;) {
    if (blk == blk_end) {
      const int item = pull_item(work, lane);
      // a whole-tile gather whose four blocks all skipped (outside the image / nothing composited)
      // was never waited for: drain it before the next gather reuses the ring, or the warp exits
      walk_drain();
      if (item >= items) break;
      const int ent = __ldg(entries + item);
      const int code = ent & 7;
      tile = ent >> 3;
      whole_tile = code == 4;  // <= 32 patches: all four blocks from one gather
      range = ld_pair(ranges, tile);  // the caller's patch_range_per_tile: any alignment
      len = range.y - range.x;
      if (len <= 0) continue;
      blk = whole_tile ? 0 : code;
      blk_end = whole_tile ? 4 : code + 1;
      if (whole_tile) gather_whole_tile(ring_addr, recs, gsid + range.x, len, lane);
    }
    const int cur = blk++;
    int tx = tile % gx, ty = tile / gx;
    size_t fo = 0;  // BATCH: offset of the tile's frame in every [H,W] plane
    if (BATCH) {
      const int f = ty / gy;
      ty -= f * gy;
      fo = (size_t)f * HW;
    }
    const int rx0 = tx * TILE + (cur & 1) * 8, ry0 = ty * TILE + (cur >> 1) * 8;
    if (rx0 >= W || ry0 >= H) continue;  // block entirely outside the image (BATCH: or in a pad row)
    const int px = rx0 + 2 * (lane & 3), py = ry0 + (lane >> 2);
    const bool in0 = px < W && py < H, in1 = px + 1 < W && py < H;
    const size_t pix = fo + (size_t)py * W + px;
    const float *const dl_f = dloss_dgammas + 2 * fo;  // pix holds fo; the frame's [3,H,W] planes start at 3 fo

    int cont0 = 0, cont1 = 0;
    float2 tau = p2s(0.f), dlr = p2s(0.f), dlg = p2s(0.f), dlb = p2s(0.f);
    float2 dld = p2s(0.f), dla = p2s(0.f);  // RGBD only: dL/dD, dL/dA
    if (RGBD) {
      if (in0) { dld.x = __ldg(dloss_ddepth_image + pix); dla.x = __ldg(dloss_dalpha_image + pix); }
      if (in1) { dld.y = __ldg(dloss_ddepth_image + pix + 1); dla.y = __ldg(dloss_dalpha_image + pix + 1); }
    }
    if (in0) {
      cont0 = min(__ldg(contrib + pix), len);
      tau.x = __ldg(final_tau + pix);
      dlr.x = __ldg(dl_f + pix);
      dlg.x = __ldg(dl_f + HW + pix);
      dlb.x = __ldg(dl_f + 2 * HW + pix);
    }
    if (in1) {
      cont1 = min(__ldg(contrib + pix + 1), len);
      tau.y = __ldg(final_tau + pix + 1);
      dlr.y = __ldg(dl_f + pix + 1);
      dlg.y = __ldg(dl_f + HW + pix + 1);
      dlb.y = __ldg(dl_f + 2 * HW + pix + 1);
    }
    int wmax = max(cont0, cont1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (wmax <= 0) continue;
    // the block's dL/dgamma table for phase B (pixel p = 8 row + x = 2 lane + {0, 1}); the
    // __syncwarp before the first flush orders it
    sts64(dl_addr + lane * 8, dlr);
    sts64(dl_addr + 256 + lane * 8, dlg);
    sts64(dl_addr + 512 + lane * 8, dlb);
    if (RGBD) sts64(dl_addr + 768 + lane * 8, dld);

    const int nch = (wmax + 31) >> 5;  // chunks [0, nch) hold the records any pixel replays
    const int32_t *ids = gsid + range.x;
    // gather of chunk c: lane j copies the record of patch 32 c + j (if below wmax) into ring slot c & 1
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
      id_next = load_id(nch - 1 - WALK_RING);  // id of the chunk the first refill gathers
    }

    const float2 npx = p2(-(float)px, -(float)(px + 1));
    const float fpy = (float)py;
    const float bx0 = (float)rx0, bx1 = (float)(rx0 + 7), by0 = (float)ry0, by1 = (float)(ry0 + 7);
    float2 sdot = p2s(0.f);  // dL/dgamma . gamma_next, per pixel
    uint32_t wa = w_addr + lane * 8;  // where the next record's weight rows go
    const uint32_t wa_pair_limit = w_addr + lane * 8 + (WALK_SLOTS - 2) * WALK_SLOT_BYTES;
    int to_my_slot = lane >> 2;  // free slots before the one whose moments this lane sums in phase B
    float4 inf = make_float4(0.f, 0.f, 0.f, 1.f);
    float4 cq = make_float4(0.f, 0.f, 0.f, 0.f);  // ABS only

    for (int c = nch - 1; c >= 0; c--) {
      // survivors of the chunk, back to front, as (record address, patch index); the pad's index
      // lies beyond every contrib
      const uint32_t my_rec = wait_chunk(ring_addr, c, lane);
      const int my_idx = c * 32 + lane;
      bool hit = false;
      if (my_idx < wmax) hit = rec_can_touch(lds128(my_rec), lds128(my_rec + 16), bx0, bx1, by0, by1);
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      const int n = __popc(mask);
      if (hit) sts64u(list_addr + __popc(mask & ~((2u << lane) - 1u)) * 8, my_rec, (uint32_t)my_idx);
      if (lane == 0) sts64u(list_addr + n * 8, dummy_addr, 0x7fffffffu);  // pad: index beyond every contrib
      __syncwarp();
      for (int i = 0; i < n; i += 2) {
        if (wa > wa_pair_limit) {  // no room for a pair
          __syncwarp();
          bwd_flush<RGBD, ABS>(w_addr, inf, cq, dl_addr, (lane >> 2) - to_my_slot, bx0, by0, moments, ddepths,
                               dus_abs, lane);
          __syncwarp();
          wa = w_addr + lane * 8;
          to_my_slot = lane >> 2;
        }
        const uint4 ent = lds128u(list_addr + i * 8);  // two records: ent.x / ent.z further back first
        const float4 q0a = lds128(ent.x), q0b = lds128(ent.z);
        const float4 q1a = lds128(ent.x + 16), q1b = lds128(ent.z + 16);
        const float4 q2a = lds128(ent.x + 32), q2b = lds128(ent.z + 32);
        const BwdEval A = bwd_eval(q0a, q1a, npx, fpy, (int)ent.y, cont0, cont1);
        const BwdEval B = bwd_eval(q0b, q1b, npx, fpy, (int)ent.w, cont0, cont1);
        float2 dca, dcb;
        if (RGBD) {  // dL/dgamma . c + dL/dD z + dL/dA
          dca = fma2_rn(dlr, p2s(q2a.x), fma2_rn(dlg, p2s(q2a.y), fma2_rn(dlb, p2s(q2a.z), fma2_rn(dld, p2s(q2a.w), dla))));
          dcb = fma2_rn(dlr, p2s(q2b.x), fma2_rn(dlg, p2s(q2b.y), fma2_rn(dlb, p2s(q2b.z), fma2_rn(dld, p2s(q2b.w), dla))));
        } else {
          dca = fma2_rn(dlr, p2s(q2a.x), fma2_rn(dlg, p2s(q2a.y), mul2_rn(dlb, p2s(q2a.z))));
          dcb = fma2_rn(dlr, p2s(q2b.x), fma2_rn(dlg, p2s(q2b.y), mul2_rn(dlb, p2s(q2b.z))));
        }
        // first record
        tau = mul2_rn(tau, A.rc);
        const float2 diffa = add2_rn(dca, p2(-sdot.x, -sdot.y));
        sdot = fma2_rn(A.e, diffa, sdot);
        const float2 dapa = mul2_rn(tau, diffa);  // dL/dalpha' (where active; times e = 0 elsewhere)
        sts64(wa, mul2_rn(dapa, A.e));        // w
        sts64(wa + 256, mul2_rn(A.e, tau));   // wc
        if (to_my_slot == 0) inf = q0a;
        if (ABS && to_my_slot == 0) cq = q1a;
        // second record (the all-zero pad record when the count is odd: e = 0, weights 0)
        tau = mul2_rn(tau, B.rc);
        const float2 diffb = add2_rn(dcb, p2(-sdot.x, -sdot.y));
        sdot = fma2_rn(B.e, diffb, sdot);
        const float2 dapb = mul2_rn(tau, diffb);
        sts64(wa + WALK_SLOT_BYTES, mul2_rn(dapb, B.e));
        sts64(wa + WALK_SLOT_BYTES + 256, mul2_rn(B.e, tau));
        if (to_my_slot == 1) inf = q0b;
        if (ABS && to_my_slot == 1) cq = q1b;
        if (fmaxf(q0a.w, q0b.w) > ALPHA_CLAMP) {  // opacity above the clamp (rare):
          // sum dL/dalpha' g is not (sum w) / alpha on clamped pixels -- reduce it with shuffles
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
        const bool pair = i + 2 <= n;  // false: the second record was the pad, its slot is reused
        wa += pair ? 2 * WALK_SLOT_BYTES : WALK_SLOT_BYTES;
        to_my_slot -= pair ? 2 : 1;
      }
      __syncwarp();  // every lane is done with this ring slot and with the list
      issue(c - WALK_RING, id_next);
      id_next = load_id(c - WALK_RING - 1);
    }
    cp_async_wait<0>();
    if (wa != w_addr + lane * 8) {
      __syncwarp();
      bwd_flush<RGBD, ABS>(w_addr, inf, cq, dl_addr, (lane >> 2) - to_my_slot, bx0, by0, moments, ddepths, dus_abs,
                           lane);
    }
    __syncwarp();  // the flush has read s_dl / s_w before the next block rewrites them
  }
}

__global__ void __launch_bounds__(128, DRAW_BWD_MINBLOCKS) k_draw_bwd(
    int W, int H, int gx, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, float *__restrict__ moments, int *__restrict__ work) {
  draw_bwd_body<false, false, false>(W, H, gx, 0, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, nullptr, nullptr,
                              moments, nullptr, nullptr, work);
}

__global__ void __launch_bounds__(128, DRAW_BWD_RGBD_MINBLOCKS) k_draw_bwd_rgbd(
    int W, int H, int gx, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, const float *__restrict__ dloss_ddepth_image,
    const float *__restrict__ dloss_dalpha_image, float *__restrict__ moments, float *__restrict__ ddepths,
    int *__restrict__ work) {
  draw_bwd_body<true, false, false>(W, H, gx, 0, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, dloss_ddepth_image,
                             dloss_dalpha_image, moments, ddepths, nullptr, work);
}

__global__ void __launch_bounds__(128, DRAW_BWD_ABS_MINBLOCKS) k_draw_bwd_abs(
    int W, int H, int gx, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, float *__restrict__ moments, float *__restrict__ dus_abs,
    int *__restrict__ work) {
  draw_bwd_body<false, true, false>(W, H, gx, 0, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, nullptr, nullptr,
                             moments, nullptr, dus_abs, work);
}

__global__ void __launch_bounds__(128, DRAW_BWD_RGBD_ABS_MINBLOCKS) k_draw_bwd_rgbd_abs(
    int W, int H, int gx, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, const float *__restrict__ dloss_ddepth_image,
    const float *__restrict__ dloss_dalpha_image, float *__restrict__ moments, float *__restrict__ ddepths,
    float *__restrict__ dus_abs, int *__restrict__ work) {
  draw_bwd_body<true, true, false>(W, H, gx, 0, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, dloss_ddepth_image,
                            dloss_dalpha_image, moments, ddepths, dus_abs, work);
}

__global__ void __launch_bounds__(128, DRAW_BWD_MINBLOCKS) k_draw_bwd_batch(
    int W, int H, int gx, int gy, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, float *__restrict__ moments, int *__restrict__ work) {
  draw_bwd_body<false, false, true>(W, H, gx, gy, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, nullptr,
                                    nullptr, moments, nullptr, nullptr, work);
}

__global__ void __launch_bounds__(128, DRAW_BWD_RGBD_MINBLOCKS) k_draw_bwd_rgbd_batch(
    int W, int H, int gx, int gy, int T, const int32_t *__restrict__ ranges, const Rec *__restrict__ recs,
    const int32_t *__restrict__ gsid, const int32_t *__restrict__ contrib, const float *__restrict__ final_tau,
    const float *__restrict__ dloss_dgammas, const float *__restrict__ dloss_ddepth_image,
    const float *__restrict__ dloss_dalpha_image, float *__restrict__ moments, float *__restrict__ ddepths,
    int *__restrict__ work) {
  draw_bwd_body<true, false, true>(W, H, gx, gy, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas,
                                   dloss_ddepth_image, dloss_dalpha_image, moments, ddepths, nullptr, work);
}

constexpr int MOM = 9;  // floats per moment row

// moment rows [N,9] -> dloss_dus[N,2], dloss_dcinv2ds[N,3], dloss_dalphas[N], dloss_dcolors[N,3]
__global__ void __launch_bounds__(PG) k_finalize_grads(int N, const float *__restrict__ moments,
                                                       const float *__restrict__ cinv2ds,
                                                       float *__restrict__ dus, float *__restrict__ dcinv,
                                                       float *__restrict__ dalphas, float *__restrict__ dcolors) {
  __shared__ float sm[TileT<MOM>::FLOATS];
  const int tid = threadIdx.x;
  const long long base = (long long)blockIdx.x * PG;
  const int nv = min(PG, (int)(N - base));
  const bool valid = tid < nv;
  float A = 0.f, B = 0.f, Cc = 0.f, m[MOM];
  tile_fetch<3>(cinv2ds, base, nv, sm, tid);
  __syncthreads();
  if (valid) { const float *r = sm + tid * TileT<3>::S; A = r[0]; B = r[1]; Cc = r[2]; }
  __syncthreads();
  tile_fetch<MOM>(moments, base, nv, sm, tid);
  __syncthreads();
#pragma unroll
  for (int i = 0; i < MOM; i++) m[i] = valid ? sm[tid * TileT<MOM>::S + i] : 0.f;
  __syncthreads();
  {
    // untouched Gaussians stay exactly 0 even if their conic is inf/NaN (reference: no atomics ran)
    const bool none = (m[0] == 0.f) && (m[1] == 0.f);
    float *o = sm + tid * TileT<2>::S;
    o[0] = none ? 0.f : -(A * m[0] + B * m[1]);
    o[1] = none ? 0.f : -(B * m[0] + Cc * m[1]);
  }
  __syncthreads();
  tile_flush<2>(dus, base, nv, sm, tid);
  __syncthreads();
  { float *o = sm + tid * TileT<3>::S; o[0] = -0.5f * m[2]; o[1] = -m[3]; o[2] = -0.5f * m[4]; }
  __syncthreads();
  tile_flush<3>(dcinv, base, nv, sm, tid);
  __syncthreads();
  { float *o = sm + tid * TileT<3>::S; o[0] = m[6]; o[1] = m[7]; o[2] = m[8]; }
  __syncthreads();
  tile_flush<3>(dcolors, base, nv, sm, tid);
  if (valid) dalphas[base + tid] = m[5];
}

int launch_draw_backward(int H, int W, int N, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                         const int32_t *contrib, const float *final_tau, const float *dloss_dgammas,
                         const DepthGrads *dg, const float *cinv2ds, float *moments, int *work, float *dloss_dus,
                         float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, bool finalize,
                         float *dus_abs, cudaStream_t st, int frames) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  if (gx <= 0 || gy <= 0 || N <= 0) return 0;
  if (frames > 0 && dus_abs != nullptr) return set_arg_error("drawB: no absolute gradients for a batch of frames");
  GSB_CUDA_TRY(cudaMemsetAsync(moments, 0, sizeof(float) * MOM * (size_t)N, st));
  if (dg != nullptr) GSB_CUDA_TRY(cudaMemsetAsync(dg->ddepths, 0, sizeof(float) * (size_t)N, st));
  if (dus_abs != nullptr) GSB_CUDA_TRY(cudaMemsetAsync(dus_abs, 0, sizeof(float) * 2 * (size_t)N, st));
  if (recs != nullptr) {
    const int T = gx * gy * (frames > 0 ? frames : 1);
    if (work == nullptr) return set_arg_error("drawB: work area missing");
    // tiles with patches
    int rc = launch_tile_list(H, W, ranges, nullptr, nullptr, nullptr, nullptr, nullptr, work, st, frames);
    if (rc) return rc;
    int grid = 0;
    const int per_sm = dus_abs != nullptr ? (dg != nullptr ? DRAW_BWD_RGBD_ABS_MINBLOCKS : DRAW_BWD_ABS_MINBLOCKS)
                                          : (dg != nullptr ? DRAW_BWD_RGBD_MINBLOCKS : DRAW_BWD_MINBLOCKS);
    rc = persistent_grid(T, per_sm, grid);
    if (rc) return rc;
    if (frames > 0 && dg != nullptr) {
      ProfScope ps(K_DRAW_BWD_RGBD_BATCH, st);
      k_draw_bwd_rgbd_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, T, ranges, recs, gsid, contrib, final_tau,
                                                  dloss_dgammas, dg->dloss_ddepth_image, dg->dloss_dalpha_image,
                                                  moments, dg->ddepths, work);
    } else if (frames > 0) {
      ProfScope ps(K_DRAW_BWD_BATCH, st);
      k_draw_bwd_batch<<<grid, 128, 0, st>>>(W, H, gx, gy, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas,
                                             moments, work);
    } else if (dus_abs != nullptr && dg != nullptr) {
      ProfScope ps(K_DRAW_BWD_RGBD_ABS, st);
      k_draw_bwd_rgbd_abs<<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas,
                                                dg->dloss_ddepth_image, dg->dloss_dalpha_image, moments, dg->ddepths,
                                                dus_abs, work);
    } else if (dus_abs != nullptr) {
      ProfScope ps(K_DRAW_BWD_ABS, st);
      k_draw_bwd_abs<<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas, moments,
                                           dus_abs, work);
    } else if (dg != nullptr) {
      ProfScope ps(K_DRAW_BWD_RGBD, st);
      k_draw_bwd_rgbd<<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib, final_tau, dloss_dgammas,
                                            dg->dloss_ddepth_image, dg->dloss_dalpha_image, moments, dg->ddepths,
                                            work);
    } else {
      ProfScope ps(K_DRAW_BWD, st);
      k_draw_bwd<<<grid, 128, 0, st>>>(W, H, gx, T, ranges, recs, gsid, contrib,
                                       final_tau, dloss_dgammas, moments, work);
    }
    GSB_CUDA_TRY(cudaGetLastError());
  }
  if (finalize) {  // otherwise the caller consumes the moment rows (gsb_preprocess_backward)
    ProfScope ps(K_FINALIZE, st);
    k_finalize_grads<<<(N + PG - 1) / PG, PG, 0, st>>>(N, moments, cinv2ds, dloss_dus, dloss_dcinv2ds,
                                                       dloss_dalphas, dloss_dcolors);
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
