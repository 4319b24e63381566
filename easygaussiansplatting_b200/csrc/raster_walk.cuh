// The record walk of every rasterizer (raster_fwd.cu, raster_bwd.cu, raster_feat.cu), the one home
// of its steps (DESIGN 3.0):
//  - a warp of the persistent grid pulls entries `tile * 8 + code` from k_tile_list's work list
//    (pull_item): code 0..3 is one 8x8 block of a dense tile, code 4 all four blocks of a tile with
//    <= 32 patches, whose single chunk of records is gathered once (gather_whole_tile: two commits,
//    so that the chunk loop's first wait<WALK_RING - 1> still covers it);
//  - it streams the tile's 48-byte records itself in 32-record chunks: lane j gathers the record of
//    patch 32 c + j with three 16-byte cp.async (gather_record) into ring slot c % WALK_RING, one
//    cp.async group per chunk and lane, WALK_RING chunks in flight, cp.async groups + __syncwarp
//    (wait_chunk) and no CTA barrier after start-up (zero_dummy).  The forward passes walk the chunks
//    front to back, the backward passes back to front from the block's largest contrib.  The surfel
//    rasterizers (surfel.cu) walk their 80-byte records with the same chunk helpers at that width;
//  - each lane tests its record against the warp's block with rec_can_touch (exact: no output
//    changes), a ballot compacts the survivors in walk order into a list of (record address, patch
//    index), and an entry pointing at the all-zero record (alpha = 0) pads an odd count, so the
//    compositing loops walk the list two records at a time (cull_compact);
//  - outstanding cp.async groups are drained (walk_drain) before the ring is reused or the warp exits.
// Every piece is __forceinline__: the kernels compile to the SASS of the copies they replace.
#pragma once
#include "common.cuh"
#include "raster_eval.cuh"

namespace gsb {

constexpr int WALK_RING = 2;  // 32-record chunks in flight per warp
template <int RecBytes = sizeof(Rec)>
constexpr int WALK_CHUNK_BYTES = 32 * RecBytes;  // one chunk of RecBytes-byte records
// phase-B weight rows of the backward passes: a slot = 2 rows of 64 floats (w, wc) + 16 floats of
// padding; a stride of 16 (mod 32) floats makes the 128-bit reads (2 slots x 4 parts per 8-lane
// wavefront) conflict-free
constexpr int WALK_SLOTS = 8;
constexpr int WALK_SLOT_BYTES = (2 * 64 + 16) * 4;        // 576
constexpr int WALK_W_BYTES = WALK_SLOTS * WALK_SLOT_BYTES;  // 4608

__device__ __forceinline__ void sts64(uint32_t a, float2 v) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ float2 lo(const float4 &v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi(const float4 &v) { return make_float2(v.z, v.w); }

// The all-zero record that pads an odd survivor count; the kernels' only CTA-wide barrier.
__device__ __forceinline__ void zero_dummy(Rec &dummy) {
  if (threadIdx.x < 12) reinterpret_cast<float *>(&dummy)[threadIdx.x] = 0.0f;
  __syncthreads();
}

// The warp's next work-list position (work[0] is the item counter, work[2..] the entries).
__device__ __forceinline__ int pull_item(int *__restrict__ work, int lane) {
  int item = 0;
  if (lane == 0) item = atomicAdd(work, 1);
  return __shfl_sync(0xffffffffu, item, 0);
}

// cp.async groups the warp has outstanding: all landed, in every lane.
__device__ __forceinline__ void walk_drain() {
  cp_async_wait<0>();
  __syncwarp();
}

// The RecBytes-byte record at `rec` (the 48-byte Rec, or the 80-byte surfel record of surfel.cu)
// into shared memory at `dst`, 16 bytes per cp.async.
template <int RecBytes = sizeof(Rec)>
__device__ __forceinline__ void gather_record(const void *rec, uint32_t dst) {
  const char *src = static_cast<const char *>(rec);
#pragma unroll
  for (int k = 0; k < RecBytes / 16; k++) cp_async16_sa(dst + 16 * k, src + 16 * k);
}

// A tile of <= 32 patches: its single chunk into ring slot 0, gathered once for all four blocks.
// Two groups, so that the chunk loop's first wait<WALK_RING - 1> covers it.
__device__ __forceinline__ void gather_whole_tile(uint32_t ring, const Rec *__restrict__ recs,
                                                  const int32_t *__restrict__ ids, int len, int lane) {
  if (lane < len) gather_record(recs + __ldg(ids + lane), ring + lane * 48);
  cp_async_commit();
  cp_async_commit();
}

// The lane's record of chunk c in a ring of WALK_RING slots, once the chunk has landed in every lane
// (a chunk is one cp.async group per lane, empty where the lane has no record in it).
template <int RecBytes = sizeof(Rec)>
__device__ __forceinline__ uint32_t wait_chunk(uint32_t ring, int c, int lane) {
  cp_async_wait<WALK_RING - 1>();  // this lane's copy of chunk c has landed ...
  __syncwarp();                   // ... and so have the other lanes'
  return ring + (c & (WALK_RING - 1)) * WALK_CHUNK_BYTES<RecBytes> + lane * RecBytes;
}

// Cull and compact one chunk of a front-to-back walk: the lane's record my_rec (patch index my_idx,
// none when my_idx >= lim) is tested against the block's rectangle [bx0, bx1] x [by0, by1]; the
// survivors are listed in order as (record address, my_idx + idx_bias), then a pad entry (dummy,
// pad_idx).  on_hit(pos, q0) runs in each surviving lane with its list position and record word q0,
// on_pad(n) in lane 0, both before the closing __syncwarp.  Returns the survivor count n.
// (The backward passes list back to front with the same steps written out: through this helper
// nvcc schedules them differently.)
template <class OnHit, class OnPad>
__device__ __forceinline__ int cull_compact(uint32_t my_rec, int my_idx, int lim, float bx0, float bx1, float by0,
                                            float by1, uint32_t list, uint32_t dummy, uint32_t idx_bias,
                                            uint32_t pad_idx, int lane, OnHit on_hit, OnPad on_pad) {
  bool hit = false;
  float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (my_idx < lim) {
    q0 = lds128(my_rec);
    hit = rec_can_touch(q0, lds128(my_rec + 16), bx0, bx1, by0, by1);
  }
  const unsigned mask = __ballot_sync(0xffffffffu, hit);
  const int n = __popc(mask);
  if (hit) {
    const int pos = __popc(mask & ((1u << lane) - 1u));
    sts64u(list + pos * 8, my_rec, (uint32_t)my_idx + idx_bias);
    on_hit(pos, q0);
  }
  if (lane == 0) {
    sts64u(list + n * 8, dummy, pad_idx);
    on_pad(n);
  }
  __syncwarp();
  return n;
}
__device__ __forceinline__ void no_hit_work(int, const float4 &) {}
__device__ __forceinline__ void no_pad_work(int) {}

// Grid of a persistent rasterizer launch: per_sm CTAs on every SM, at most one per tile.  A CUDA
// error is reported as GSB_CUDA_TRY does.
inline int persistent_grid(int T, int per_sm, int &grid) {
  int dev = 0, sms = 132;
  GSB_CUDA_TRY(cudaGetDevice(&dev));
  GSB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const long long want = (long long)sms * per_sm;
  grid = (int)(T < want ? T : want);
  return 0;
}

}  // namespace gsb
