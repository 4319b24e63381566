// Tile binning: per-Gaussian tile rectangles + exclusive offsets (one fused kernel with a
// decoupled look-back scan), (tile | depth-mm) keys emitted warp-cooperatively, a hand-written
// LSD radix sort (per pass: per-tile digit counts, one look-back scan of them, one
// rank-and-scatter kernel), per-tile ranges and the packed per-Gaussian record stream.
//
// Replaces getRects / thrust::inclusive_scan / createKeys / thrust::sort_by_key / getRanges
// (reference kernel.cu:46-150, gausplat.cu:50-91).  No library kernels: round 1 used CUB's
// DeviceScan / DeviceRadixSort, whose tile sizes gave 1.05-wave launches at this problem size
// (2.5 M pairs: 29 us per pass, 16 us for a 1 M-element scan).  Everything is stream-ordered in
// caller-provided workspace and every kernel takes the patch count P from DEVICE memory, so the
// same kernels serve the synchronous operator surface (P read back once, like the reference,
// gausplat.cu:67) and the capacity-based path without a host round trip (api.cu).
//
// Sort width.  The reference sorts all 64 bits of (tile << 32 | (uint32)(depth*1000)).  Only
// ceil(log2(tiles)) + ceil(log2(max depth key + 1)) of them can differ; when the two fields
// fit 32 bits the keys are packed as (tile << dbits | depth key) in 32-bit words -- the same
// (tile, depth-mm, id) order with half the key traffic -- and only the digits that can be
// non-zero are sorted (9-bit digits when that saves a pass: 27 bits at 1080p = 3 passes).
// Every pass is stable, so ties keep ascending Gaussian id exactly like thrust::sort_by_key.
#include <atomic>

#include "../../include/gsplat_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "rect_math.h"
#include "tile_io.cuh"

namespace gsb {

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int bits_for(uint64_t n_values) {  // bits needed to represent 0 .. n_values-1
  int b = 0;
  while (((uint64_t)1 << b) < n_values) b++;
  return b;
}
static int sm_count() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
    sms = 132;
  return sms;
}

// ---- relaxed / acquire-release device-scope accesses for the look-back descriptors
__device__ __forceinline__ void st_relaxed_u32(uint32_t *p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Single-pass decoupled look-back of Merrill & Garland, shared by the two scans of this file
// (k_rects_scan, k_colscan): a CTA publishes its aggregate, then its inclusive prefix, in one
// 64-bit word (2 flag bits | value), and a warp walks back over its predecessors 32 at a time.
// CTAs take their index `blk` from an atomic claim counter, so every predecessor is already
// running: the walk cannot deadlock.  Called by one whole warp; returns the exclusive prefix.
constexpr unsigned long long DESC_AGG = 1ull << 62, DESC_INC = 2ull << 62, DESC_VAL = (1ull << 62) - 1;
__device__ unsigned long long scan_lookback(unsigned long long *desc, int blk, unsigned long long run) {
  const int lane = threadIdx.x & 31;
  unsigned long long excl = 0;
  if (blk > 0) {
    if (lane == 0) st_relaxed_u64(desc + blk, DESC_AGG | run);
    int p = blk - 1;  // lane l inspects predecessor p - l
    for (;;) {
      const int q = p - lane;
      unsigned long long v = DESC_INC;  // virtual predecessor before block 0: inclusive 0
      if (q >= 0) {
        do { v = ld_relaxed_u64(desc + q); } while ((v >> 62) == 0);
      }
      const unsigned inc_mask = __ballot_sync(0xffffffffu, (v >> 62) == 2);
      const int first_inc = inc_mask ? __ffs(inc_mask) - 1 : 32;  // nearest predecessor with an inclusive value
      unsigned long long part = (lane <= first_inc) ? (v & DESC_VAL) : 0ull;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      excl += part;
      if (inc_mask) break;
      p -= 32;
    }
  }
  if (lane == 0) st_relaxed_u64(desc + blk, DESC_INC | (excl + run));
  return excl;
}

// =================================================================== phase 1: rects + scan
// One CTA = 1024 consecutive Gaussians (4 per thread, strided so every access is coalesced).
// Rectangle arithmetic: rect_math.h tile_rect (explicitly rounded: it decides the patch list).
// The inclusive prefix sum of the patch counts uses the decoupled look-back above.
constexpr int RS_CTA = 256, RS_ITEMS = 4, RS_SPAN = RS_CTA * RS_ITEMS;

// BATCH: the N = C nc records of a batch of C frames, record i = c nc + n in frame c (DESIGN 3.21):
// its rectangle is the single frame's (the same operations on its camera-local mean), clamped to
// frame c's gy tile rows [0, gy] and then moved down by c gy rows of the tall frame.
template <bool BATCH>
__device__ __forceinline__ void rects_scan_body(int N, const float *__restrict__ us, int32_t *__restrict__ areas,
                                                float *__restrict__ depths, int gx, int gy, int nc,
                                                uint2 *__restrict__ rects, uint32_t *__restrict__ incl,
                                                uint32_t *__restrict__ total, unsigned long long *__restrict__ desc,
                                                uint32_t *__restrict__ claim) {
  __shared__ uint32_t s_warp[RS_CTA / 32];
  __shared__ unsigned long long s_prefix;
  __shared__ uint32_t s_max[RS_CTA / 32];
  __shared__ int s_blk;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_blk = (int)atomicAdd(claim, 1u);  // claim order = data order: look-back cannot deadlock
  __syncthreads();
  const int blk = s_blk;
  const int nblk = (N + RS_SPAN - 1) / RS_SPAN;
  uint32_t cnt[RS_ITEMS], dkmax = 0;
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    const int i = blk * RS_SPAN + k * RS_CTA + tid;
    uint32_t n = 0;
    if (i < N) {
      uint2 rect = make_uint2(0u, 0u);
      const float d = depths[i];
      if (!(d < MIN_DEPTH)) {
        const float2 u = ld_pair(us, i);  // us / areas: any contiguous [N,2] view (tile_io.cuh)
        const int2 ar = ld_pair_rw(areas, i);
        const float xs = (float)ar.x, ys = (float)ar.y;
        int x0, x1, y0, y1;  // BATCH: in frame i / nc's rows of the tall frame
        tile_rect(u.x, u.y, xs, ys, gx, gy, BATCH ? (i / nc) * gy : 0, x0, x1, y0, y1);
        n = (uint32_t)(y1 - y0) * (uint32_t)(x1 - x0);
        if (n == 0) {  // kernel.cu:114-119: in-place cull
          depths[i] = BAD_MARKER;
          st_pair(areas, i, 0, 0);
        } else {
          rect = make_uint2((uint32_t)x0 | ((uint32_t)x1 << 16), (uint32_t)y0 | ((uint32_t)y1 << 16));
          dkmax = max(dkmax, __float2uint_rz(__fmul_rn(d, 1000.0f)));  // kernel.cu:73
        }
      }
      rects[i] = rect;  // rect packed as (x0 | x1 << 16, y0 | y1 << 16); grids up to 65535 x 65535 (api.cu)
    }
    cnt[k] = n;
  }
  // CTA-local inclusive scan in data order (sub-tile k holds elements k*256 .. k*256+255)
  uint32_t loc[RS_ITEMS], run = 0;
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    uint32_t v = cnt[k];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    uint32_t wbase = 0, sub = 0;
#pragma unroll
    for (int w = 0; w < RS_CTA / 32; w++) {
      const uint32_t t = s_warp[w];
      if (w < warp) wbase += t;
      sub += t;
    }
    loc[k] = run + wbase + v;
    run += sub;
    __syncthreads();
  }
  // look-back (warp 0): exclusive prefix of this CTA over all earlier CTAs
  if (warp == 0) {
    const unsigned long long excl = scan_lookback(desc, blk, run);
    if (lane == 0) {
      s_prefix = excl;
      if (blk == nblk - 1) total[0] = (uint32_t)min(excl + run, 0xffffffffull);  // P (saturating)
    }
  }
  const uint32_t wmax = __reduce_max_sync(0xffffffffu, dkmax);
  if (lane == 0) s_max[warp] = wmax;
  __syncthreads();
  const uint32_t prefix = (uint32_t)s_prefix;
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    const int i = blk * RS_SPAN + k * RS_CTA + tid;
    if (i < N) incl[i] = prefix + loc[k];
  }
  if (tid == 0) {
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < RS_CTA / 32; w++) m = max(m, s_max[w]);
    if (m > 0) atomicMax(total + 1, m);  // largest depth key of a binned Gaussian
    if (s_prefix + run > 0xffffffffull) atomicOr(total + 2, GSB_STATUS_TOO_MANY_PATCHES);  // P does not fit 32 bits
  }
}

__global__ void __launch_bounds__(RS_CTA) k_rects_scan(int N, const float *__restrict__ us,
                                                       int32_t *__restrict__ areas, float *__restrict__ depths,
                                                       int gx, int gy, uint2 *__restrict__ rects,
                                                       uint32_t *__restrict__ incl, uint32_t *__restrict__ total,
                                                       unsigned long long *__restrict__ desc,
                                                       uint32_t *__restrict__ claim) {
  rects_scan_body<false>(N, us, areas, depths, gx, gy, 0, rects, incl, total, desc, claim);
}

__global__ void __launch_bounds__(RS_CTA) k_rects_scan_batch(int N, const float *__restrict__ us,
                                                             int32_t *__restrict__ areas, float *__restrict__ depths,
                                                             int gx, int gy, int nc, uint2 *__restrict__ rects,
                                                             uint32_t *__restrict__ incl, uint32_t *__restrict__ total,
                                                             unsigned long long *__restrict__ desc,
                                                             uint32_t *__restrict__ claim) {
  rects_scan_body<true>(N, us, areas, depths, gx, gy, nc, rects, incl, total, desc, claim);
}

// =================================================================== phase 2: keys
// Sort plan: which bit ranges of the key are sorted, in which order (LSD).
constexpr int MAX_PASSES = 8;
struct PassPlan {
  int n, bits;  // passes, digit width (8 or 9)
  int shift[MAX_PASSES];
};
struct KeyPlan {
  bool narrow;     // 32-bit keys
  int shift;       // tile field starts at this bit
  int depth_bits;  // low bits of the depth key the passes order (32: all of it)
  PassPlan pp;
};
static KeyPlan key_plan(int H, int W, uint32_t depth_key_max) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const int tbits = bits_for((uint64_t)gx * (uint64_t)gy);
  const int dbits = depth_key_max == 0xffffffffu ? 32 : bits_for((uint64_t)depth_key_max + 1);
  KeyPlan p{};
  p.narrow = dbits < 32 && tbits + dbits <= 32;  // (dbits == 32 would need a shift by the word width)
  p.shift = p.narrow ? dbits : 32;
  PassPlan &pp = p.pp;
  if (p.narrow) {
    const int end = dbits + tbits;
    pp.bits = (end > 0 && (end + 8) / 9 < (end + 7) / 8) ? 9 : 8;
    for (int s = 0; s < end; s += pp.bits) pp.shift[pp.n++] = s;
    p.depth_bits = dbits;  // a deeper key would run into the tile field
  } else {  // 64-bit layout: depth bits [0, dbits), tile bits [32, 32 + tbits); the gap is all zero
    pp.bits = 8;
    for (int s = 0; s < dbits; s += 8) pp.shift[pp.n++] = s;
    for (int s = 0; s < tbits; s += 8) pp.shift[pp.n++] = 32 + s;
    p.depth_bits = (dbits + 7) / 8 * 8;  // the depth passes cover whole digits
  }
  return p;
}

// Warp-cooperative: the patches of a warp's 32 consecutive Gaussians are one contiguous range
// of the key array (exclusive offsets from the scan), and the lanes walk that range 32 keys at a
// time.  Each lane finds the Gaussian that owns its position by a binary search over the warp's
// 32 offsets (shuffles) and builds the key row-major inside that Gaussian's rectangle
// (== reference order), so every store is coalesced and no lane waits for a large rectangle.
// 64-bit: tile << 32 | dk (kernel.cu:71-74); 32-bit: tile << dbits | dk.
// *status |= GSB_STATUS_P_CAP when a Gaussian's patches do not fit the capacity (it is dropped whole
// and nothing is written at or past `capacity`), |= GSB_STATUS_DEPTH_KEY when a depth key needs more than the
// `depth_bits` the passes order, in either layout (both only possible on the capacity-based
// path, gsb_splat_forward, whose plan comes from an earlier frame's depth keys).
template <typename KeyT>
__global__ void __launch_bounds__(256) k_keys(int N, const float *__restrict__ depths,
                                              const uint32_t *__restrict__ incl, const uint2 *__restrict__ rects,
                                              int gx, int shift, int depth_bits, uint32_t capacity,
                                              KeyT *__restrict__ keys, int32_t *__restrict__ vals,
                                              uint32_t *__restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int first = (blockIdx.x * blockDim.x + threadIdx.x) & ~31;  // the warp's first Gaussian
  if (first >= N) return;
  const int i = first + lane;
  const uint32_t inc = __ldg(incl + min(i, N - 1));  // lanes past N: no patches
  uint32_t off = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) off = first == 0 ? 0u : __ldg(incl + first - 1);
  uint32_t n = inc - off, rx = 0, ry = 0;
  KeyT dk = 0;
  if (i < N) {
    const float d = __ldg(depths + i);
    if (!(d < MIN_DEPTH)) {
      const uint2 r = __ldg(rects + i);
      rx = r.x; ry = r.y;  // (x0 | x1 << 16, y0 | y1 << 16)
      dk = (KeyT)__float2uint_rz(__fmul_rn(d, 1000.0f));
      if (depth_bits < 32 && (dk >> depth_bits) != 0) {  // deeper than the plan sorts (capacity path)
        atomicOr(status, GSB_STATUS_DEPTH_KEY);
        dk &= ((KeyT)1 << depth_bits) - 1;  // (keeps the tile field of a 32-bit key intact)
      }
    }
  }
  if (n > 0 && (off > capacity || n > capacity - off)) {  // does not fit: drop, flag
    atomicOr(status, GSB_STATUS_P_CAP);
    n = 0;
  }
  const uint32_t start = __shfl_sync(0xffffffffu, off, 0);
  const uint32_t span = __shfl_sync(0xffffffffu, inc, 31) - start;
  const uint32_t rel = off - start;  // non-decreasing over the lanes
  // positions at or past the capacity belong to dropped Gaussians only
  const uint32_t todo = start < capacity ? min(span, capacity - start) : 0u;
  for (uint32_t t0 = 0; t0 < todo; t0 += 32) {
    const uint32_t t = t0 + lane;
    int o = 0;  // owner: the last lane whose range starts at or before t
#pragma unroll
    for (int s = 16; s > 0; s >>= 1)
      if (__shfl_sync(0xffffffffu, rel, o + s) <= t) o += s;
    const uint32_t on = __shfl_sync(0xffffffffu, n, o), orel = __shfl_sync(0xffffffffu, rel, o);
    const uint32_t ox = __shfl_sync(0xffffffffu, rx, o), oy = __shfl_sync(0xffffffffu, ry, o);
    const KeyT odk = __shfl_sync(0xffffffffu, dk, o);
    const uint32_t local = t - orel;
    if (t < todo && local < on) {
      const uint32_t x0 = ox & 0xffffu, w = (ox >> 16) - x0;
      const uint32_t y = (oy & 0xffffu) + local / w, x = x0 + local % w;
      keys[start + t] = ((KeyT)(y * (uint32_t)gx + x) << shift) | odk;
      vals[start + t] = first + o;
    }
  }
}

// =================================================================== phase 2: radix sort
// LSD radix sort over sort tiles of RX_TILE consecutive pairs; one pass = three kernels, no
// global atomics and no inter-CTA waiting except the look-back of the scan:
//   k_digit_counts  one CTA per sort tile counts the pass's digit of its keys in shared memory and
//               writes the counts digit-major: C[digit][tile];
//   k_colscan   one exclusive scan over all of C in that order turns it into the scatter bases
//               B[digit][tile] = (keys with a smaller digit) + (keys with this digit in earlier
//               tiles), spread over enough CTAs to use the whole GPU (decoupled look-back);
//   k_radix_pass  one CTA per sort tile ranks its keys (stable: warps own contiguous 32 RX_IPT-
//               element spans, the lanes of a round are ordered by ballots over the digit bits)
//               and scatters them to B + rank.
// k_digit_counts re-reads the keys the previous kernel has just written (L2 resident).  It
// replaces one global RED per key and pass into the next pass's counts, which capped the
// scatter kernel.  (A single-kernel pass with decoupled look-back per digit was tried before:
// with every CTA of a 2.5 M-pair pass starting in lockstep the look-back walked ~40 tiles back
// on average -- 50 us per pass, slower than the library it replaced.)
#ifndef RX_MINBLOCKS
#define RX_MINBLOCKS 3
#endif
// 4096-pair sort tiles: 614 tiles at config 2 (P = 2.51M).  Measured on an H100 80GB HBM3 (700 W
// limit) against 2048-, 3072-, 5120- and 6144-pair tiles: 2048 and 3072 (at 4 or 6 CTAs per SM)
// were slower; 5120 and 6144 sorted config 2 a few us per pass faster, but made the whole step
// no faster and the 50k-Gaussian 4K frame slower.
constexpr int RX_THREADS = 256, RX_WARPS = RX_THREADS / 32, RX_IPT = 16, RX_TILE = RX_THREADS * RX_IPT;
constexpr int CS_CTA = 256, CS_ITEMS = 8, CS_SPAN = CS_CTA * CS_ITEMS;  // k_colscan: values per CTA

template <typename KeyT, int BITS>
__global__ void __launch_bounds__(RX_THREADS) k_digit_counts(const KeyT *__restrict__ keys,
                                                             const uint32_t *__restrict__ P_dev, uint32_t capacity,
                                                             int shift, uint32_t tiles, uint32_t *__restrict__ C,
                                                             unsigned long long *__restrict__ desc, uint32_t ndesc,
                                                             uint32_t *__restrict__ claim) {
  constexpr int BINS = 1 << BITS;
  __shared__ uint32_t s_cnt[BINS];
  // reset the look-back state of the k_colscan that follows (ndesc <= tiles descriptors)
  if (threadIdx.x == 0) {
    if (blockIdx.x < ndesc) desc[blockIdx.x] = 0;
    if (blockIdx.x == 0) *claim = 0;
  }
  if (P_dev[2] != 0) return;  // [P, max key, flags]: capacity overflow, the frame is abandoned (see k_ranges)
  const uint32_t P = min(*P_dev, capacity);
  const uint32_t tile = blockIdx.x;  // tiles past P (capacity path) write zero counts
  for (int d = threadIdx.x; d < BINS; d += RX_THREADS) s_cnt[d] = 0;
  KeyT key[RX_IPT];  // all loads in flight before the first count
#pragma unroll
  for (int r = 0; r < RX_IPT; r++) {
    const uint32_t idx = tile * RX_TILE + r * RX_THREADS + threadIdx.x;
    key[r] = idx < P ? keys[idx] : (KeyT)0;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < RX_IPT; r++)
    if (tile * RX_TILE + r * RX_THREADS + threadIdx.x < P) atomicAdd(&s_cnt[(uint32_t)(key[r] >> shift) & (BINS - 1)], 1u);
  __syncthreads();
  for (int d = threadIdx.x; d < BINS; d += RX_THREADS) C[(size_t)d * tiles + tile] = s_cnt[d];
}

// In-place exclusive scan of n values (n a multiple of CS_ITEMS); claim / desc reset by k_digit_counts
__global__ void __launch_bounds__(CS_CTA) k_colscan(const uint32_t *__restrict__ flags, uint32_t n,
                                                    uint32_t *__restrict__ C, unsigned long long *__restrict__ desc,
                                                    uint32_t *__restrict__ claim) {
  __shared__ uint32_t s_warp[CS_CTA / 32];
  __shared__ uint32_t s_prefix;
  __shared__ int s_blk;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (*flags != 0) return;
  if (tid == 0) s_blk = (int)atomicAdd(claim, 1u);
  __syncthreads();
  const int blk = s_blk;
  const uint32_t i0 = (uint32_t)blk * CS_SPAN + tid * CS_ITEMS;  // this thread's CS_ITEMS consecutive values
  uint4 v[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  if (i0 < n) {
    v[0] = *reinterpret_cast<const uint4 *>(C + i0);
    v[1] = *reinterpret_cast<const uint4 *>(C + i0 + 4);
  }
  const uint32_t sum = v[0].x + v[0].y + v[0].z + v[0].w + v[1].x + v[1].y + v[1].z + v[1].w;
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  uint32_t wbase = 0, run = 0;
#pragma unroll
  for (int w = 0; w < CS_CTA / 32; w++) {
    const uint32_t t = s_warp[w];
    if (w < warp) wbase += t;
    run += t;
  }
  if (warp == 0) {
    const unsigned long long excl = scan_lookback(desc, blk, run);
    if (lane == 0) s_prefix = (uint32_t)excl;
  }
  __syncthreads();
  if (i0 < n) {
    uint32_t e = s_prefix + wbase + inc - sum;
    uint4 o[2];
    o[0].x = e; e += v[0].x; o[0].y = e; e += v[0].y; o[0].z = e; e += v[0].z; o[0].w = e; e += v[0].w;
    o[1].x = e; e += v[1].x; o[1].y = e; e += v[1].y; o[1].z = e; e += v[1].z; o[1].w = e;
    *reinterpret_cast<uint4 *>(C + i0) = o[0];
    *reinterpret_cast<uint4 *>(C + i0 + 4) = o[1];
  }
}

template <typename KeyT, int BITS>
__global__ void __launch_bounds__(RX_THREADS, sizeof(KeyT) == 8 ? 2 : RX_MINBLOCKS) k_radix_pass(const KeyT *__restrict__ keys_in,
                                                              const int32_t *__restrict__ vals_in,
                                                              KeyT *__restrict__ keys_out,
                                                              int32_t *__restrict__ vals_out,
                                                              const uint32_t *__restrict__ P_dev,
                                                              uint32_t capacity, int shift, uint32_t tiles,
                                                              const uint32_t *__restrict__ base) {
  constexpr int BINS = 1 << BITS, PER = BINS / RX_THREADS;
  __shared__ uint32_t s_whist[RX_WARPS][BINS];  // per-warp digit counts -> tile-local offsets
  __shared__ uint32_t s_gofs[BINS];             // global position of a digit's run minus its local start
  __shared__ uint32_t s_scan[RX_WARPS];
  extern __shared__ __align__(16) unsigned char s_dyn[];  // the tile in sorted order: coalesced write-out
  KeyT *const s_keys = reinterpret_cast<KeyT *>(s_dyn);
  int32_t *const s_vals = reinterpret_cast<int32_t *>(s_dyn + RX_TILE * sizeof(KeyT));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // Capacity overflow: k_keys left holes with stale keys that no histogram counted, so scatter
  // positions could run past the buffers.  Nothing is sorted; k_ranges leaves every range empty.
  if (P_dev[2] != 0) return;
  const uint32_t P = min(*P_dev, capacity);
  const uint32_t tile = blockIdx.x;  // one sort tile per CTA; tiles past P (capacity path) have nothing to do
  if (tile * RX_TILE >= P) return;
  for (int i = tid; i < RX_WARPS * BINS; i += RX_THREADS) (&s_whist[0][0])[i] = 0;
  __syncthreads();
  const uint32_t first = (uint32_t)tile * RX_TILE + warp * (32 * RX_IPT) + lane;
  const uint32_t tile_n = min((uint32_t)RX_TILE, P - (uint32_t)tile * RX_TILE);
  KeyT key[RX_IPT];
  uint32_t rank[RX_IPT];
#pragma unroll
  for (int r = 0; r < RX_IPT; r++) {
    const uint32_t idx = first + r * 32;
    key[r] = idx < P ? keys_in[idx] : (KeyT)0;
  }
  uint32_t gbase[PER];  // scatter bases of this thread's digits (below), loaded under the ranking
#pragma unroll
  for (int k = 0; k < PER; k++) gbase[k] = base[(size_t)(tid * PER + k) * tiles + tile];
#pragma unroll
  for (int r = 0; r < RX_IPT; r++) {
    const bool valid = first + r * 32 < P;
    const uint32_t d = (uint32_t)(key[r] >> shift) & (BINS - 1);
    // lanes of this round with the same digit (ballot per digit bit: __match_any_sync is a
    // data-dependent loop in hardware)
    unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int b = 0; b < BITS; b++) {
      const bool bit = (d >> b) & 1u;
      const unsigned m = __ballot_sync(0xffffffffu, bit);
      peers &= bit ? m : ~m;
    }
    const int leader = __ffs(peers) - 1;
    uint32_t old = 0;
    if (valid && lane == leader) {
      old = s_whist[warp][d];
      s_whist[warp][d] = old + __popc(peers);
    }
    old = __shfl_sync(0xffffffffu, old, leader < 0 ? 0 : leader);
    rank[r] = old + __popc(peers & ((1u << lane) - 1u));
    __syncwarp();
  }
  __syncthreads();
  {  // per digit (thread t owns digits [PER t, PER t + PER)): offsets of the warps, local start
    uint32_t cnt[PER], sum = 0;
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int d = tid * PER + k;
      uint32_t run = 0;
#pragma unroll
      for (int w = 0; w < RX_WARPS; w++) {
        const uint32_t t = s_whist[w][d];
        s_whist[w][d] = run;
        run += t;
      }
      cnt[k] = run;
      sum += run;
    }
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_scan[warp] = inc;
    __syncthreads();
    uint32_t start = inc - sum;  // tile-local start of this thread's first digit
    for (int w = 0; w < warp; w++) start += s_scan[w];
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int d = tid * PER + k;
#pragma unroll
      for (int w = 0; w < RX_WARPS; w++) s_whist[w][d] += start;
      s_gofs[d] = gbase[k] - start;
      start += cnt[k];
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < RX_IPT; r++) {
    if (first + r * 32 < P) {
      const uint32_t lp = s_whist[warp][(uint32_t)(key[r] >> shift) & (BINS - 1)] + rank[r];
      s_keys[lp] = key[r];
      s_vals[lp] = vals_in[first + r * 32];  // (read here, not held in registers through the ranking)
    }
  }
  __syncthreads();
  for (uint32_t j = tid; j < tile_n; j += RX_THREADS) {  // sorted order: runs of equal digits are contiguous
    const KeyT k = s_keys[j];
    const uint32_t pos = s_gofs[(uint32_t)(k >> shift) & (BINS - 1)] + j;
    keys_out[pos] = k;
    vals_out[pos] = s_vals[j];
  }
}

template <typename KeyT>
__global__ void __launch_bounds__(256) k_ranges(const uint32_t *__restrict__ P_dev, uint32_t capacity,
                                                const uint32_t *__restrict__ flags,
                                                const KeyT *__restrict__ keys, int shift, uint32_t T,
                                                int2 *__restrict__ ranges) {
  // After a capacity overflow (k_keys dropped the Gaussians that did not fit) the key / id arrays
  // have holes with stale contents and were not sorted: every range stays empty (the memset before
  // the sort), so that the rasterizer enqueued behind this kernel touches no patch and gathers no
  // record through a stale id.  The frame is discarded and redone by the caller anyway.
  if (*flags != 0) return;
  const uint32_t P = min(*P_dev, capacity);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
    const uint32_t t = (uint32_t)(keys[p] >> shift);
    if (t >= T) continue;  // (only after a capacity overflow, when the result is discarded anyway)
    if (p == 0 || (uint32_t)(keys[p - 1] >> shift) != t) ranges[t].x = (int)p;
    if (p == P - 1 || (uint32_t)(keys[p + 1] >> shift) != t) ranges[t].y = (int)(p + 1);
  }
}

// Gathers the four per-Gaussian attribute arrays (all L2 resident: 36 B/Gaussian) into the
// 48-B records the rasterizers gather with cp.async (gsid == nullptr: one record per Gaussian);
// the depth word is depths[g], or 0 when depths is NULL (only the RGB-D rasterizers read it).
__global__ void __launch_bounds__(256) k_pack(int64_t P, const int32_t *__restrict__ gsid,
                                              const float *__restrict__ us,
                                              const float *__restrict__ cinv2ds,
                                              const float *__restrict__ alphas,
                                              const float *__restrict__ colors,
                                              const float *__restrict__ depths, Rec *__restrict__ recs) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int g = gsid != nullptr ? __ldg(gsid + p) : (int)p;  // nullptr: one record per Gaussian
  const float2 u = ld_pair(us, g);
  recs[p] = build_record(u.x, u.y, __ldg(cinv2ds + 3 * (size_t)g), __ldg(cinv2ds + 3 * (size_t)g + 1),
                         __ldg(cinv2ds + 3 * (size_t)g + 2), __ldg(alphas + g), __ldg(colors + 3 * (size_t)g),
                         __ldg(colors + 3 * (size_t)g + 1), __ldg(colors + 3 * (size_t)g + 2),
                         depths != nullptr ? __ldg(depths + g) : 0.0f, g);
}

// ---------------------------------------------------------------- phase 1 host side
BinLayout bin_layout(int N) {
  BinLayout L{};
  const size_t n = (size_t)(N > 0 ? N : 1);
  size_t o = 0;
  L.rects = o;   o = align_up(o + n * sizeof(uint2), 256);
  L.offsets = o; o = align_up(o + n * sizeof(uint32_t), 256);
  L.total = o;   o = align_up(o + 4 * sizeof(uint32_t), 256);  // [P, max depth key, flags, scan claim]
  L.scan_desc = o;
  o = align_up(o + ((n + RS_SPAN - 1) / RS_SPAN) * sizeof(unsigned long long), 256);
  L.bytes = o;
  return L;
}

int launch_bin(int H, int W, int N, const float *us, float *depths, int32_t *areas, void *ws,
               const BinLayout &L, cudaStream_t st) {
  char *b = static_cast<char *>(ws);
  uint32_t *total = reinterpret_cast<uint32_t *>(b + L.total);
  // [P, max key, flags, claim] and the look-back descriptors start at zero
  GSB_CUDA_TRY(cudaMemsetAsync(total, 0, L.bytes - L.total, st));
  if (N <= 0) return 0;
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  ProfScope ps(K_RECTS, st);
  k_rects_scan<<<(N + RS_SPAN - 1) / RS_SPAN, RS_CTA, 0, st>>>(
      N, us, areas, depths, gx, gy,
      reinterpret_cast<uint2 *>(b + L.rects), reinterpret_cast<uint32_t *>(b + L.offsets), total,
      reinterpret_cast<unsigned long long *>(b + L.scan_desc), total + 3);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_bin_batch(int C, int H, int W, int N, const float *us, float *depths, int32_t *areas, void *ws,
                     const BinLayout &L, cudaStream_t st) {
  char *b = static_cast<char *>(ws);
  uint32_t *total = reinterpret_cast<uint32_t *>(b + L.total);
  GSB_CUDA_TRY(cudaMemsetAsync(total, 0, L.bytes - L.total, st));
  const int NT = C * N;  // (C N < 2^31: checked by the entry points)
  if (NT <= 0) return 0;
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  ProfScope ps(K_RECTS_BATCH, st);
  k_rects_scan_batch<<<(NT + RS_SPAN - 1) / RS_SPAN, RS_CTA, 0, st>>>(
      NT, us, areas, depths, gx, gy, N, reinterpret_cast<uint2 *>(b + L.rects),
      reinterpret_cast<uint32_t *>(b + L.offsets), total, reinterpret_cast<unsigned long long *>(b + L.scan_desc),
      total + 3);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------- phase 2 host side
SortLayout sort_layout(int N, int H, int W, int64_t P) {
  SortLayout L{};
  const size_t T = (size_t)((W + TILE - 1) / TILE) * (size_t)((H + TILE - 1) / TILE);
  const size_t n = (size_t)(P > 0 ? P : 1);
  const size_t ng = (size_t)(N > 0 ? N : 1);
  const size_t tiles = (n + RX_TILE - 1) / RX_TILE;
  size_t o = 0;
  L.keys_a = o; o = align_up(o + n * sizeof(uint64_t), 256);
  L.keys_b = o; o = align_up(o + n * sizeof(uint64_t), 256);
  L.vals_a = o; o = align_up(o + n * sizeof(int32_t), 256);
  L.vals_b = o; o = align_up(o + n * sizeof(int32_t), 256);
  L.recs = o;   o = align_up(o + ng * sizeof(Rec), 256);  // one record per Gaussian
  L.counters = o; o = align_up(o + (4 * T + 2) * sizeof(int), 256);  // rasterizer work area (launch_tile_list)
  // k_colscan's claim counter and look-back descriptors, reset before every pass by k_digit_counts
  L.sort_state = o;
  L.desc = o + 8;
  o = align_up(L.desc + (tiles * 512 + CS_SPAN - 1) / CS_SPAN * sizeof(unsigned long long), 256);
  L.counts = o; o = align_up(o + tiles * 512 * sizeof(uint32_t), 256);  // digit counts / scatter bases of a pass
  L.bytes = o;
  return L;
}

BwdLayout bwd_layout(int N, int H, int W, int64_t P, uintptr_t base) {
  BwdLayout L{};
  const size_t T = (size_t)((W + TILE - 1) / TILE) * (size_t)((H + TILE - 1) / TILE);
  L.recs = align_up(base, 256) - base;  // (cp.async gathers the records 16 bytes at a time)
  L.moments = L.recs + align_up((size_t)(P > 0 && N > 0 ? N : 1) * sizeof(Rec), 256);
  L.work = L.moments + align_up((size_t)(N > 0 ? N : 1) * 9 * sizeof(float), 256);
  L.bytes = L.work + (4 * T + 2) * sizeof(int);  // launch_tile_list's work area
  return L;
}

int launch_pack_only(int64_t P, const int32_t *gsid_per_patch, const float *us, const float *cinv2ds,
                     const float *alphas, const float *colors, const float *depths, Rec *recs, cudaStream_t st) {
  if (P <= 0) return 0;
  ProfScope ps(K_PACK, st);
  k_pack<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(P, gsid_per_patch, us, cinv2ds, alphas, colors, depths, recs);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// k_radix_pass stages its tile in dynamic shared memory, past the 48 KB default with 64-bit keys.
// That opt-in is a function attribute of the device's context: set on each device before its
// first pass (a process that sorts on two devices needs it twice).
template <typename KeyT, int BITS>
static cudaError_t radix_pass_smem_opt_in(int bytes) {
  static std::atomic<unsigned long long> done{0};  // bit d: set on device d (devices past 63: every call)
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
  if (done.load(std::memory_order_relaxed) & bit) return cudaSuccess;
  e = cudaFuncSetAttribute(k_radix_pass<KeyT, BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_relaxed);
  return e;
}

template <typename KeyT>
static int keys_sort_ranges(int N, int64_t P_cap, const float *depths, const uint32_t *incl, const uint2 *rects,
                            uint32_t *total, int gx, int T, const KeyPlan &kp, char *b, const SortLayout &SL,
                            int32_t *ranges, int32_t *gsid_per_patch, const StatusRead *sr, cudaStream_t st) {
  const uint32_t *P_dev = total;
  KeyT *ka = reinterpret_cast<KeyT *>(b + SL.keys_a), *kb = reinterpret_cast<KeyT *>(b + SL.keys_b);
  int32_t *va = reinterpret_cast<int32_t *>(b + SL.vals_a), *vb = reinterpret_cast<int32_t *>(b + SL.vals_b);
  uint32_t *claim = reinterpret_cast<uint32_t *>(b + SL.sort_state);
  unsigned long long *desc = reinterpret_cast<unsigned long long *>(b + SL.desc);
  uint32_t *counts = reinterpret_cast<uint32_t *>(b + SL.counts);
  const PassPlan &pp = kp.pp;
  const int sms = sm_count();
  // one sort tile per CTA; sized for the capacity, the kernels skip the tiles past the device's P
  const uint32_t tiles = (uint32_t)((P_cap + RX_TILE - 1) / RX_TILE);
  const uint32_t nscan = tiles << pp.bits;  // values k_colscan scans (a multiple of CS_ITEMS)
  const int scan_grid = (int)((nscan + CS_SPAN - 1) / CS_SPAN);
  // k_keys writes (ka, va); pass p reads what pass p-1 wrote; keys alternate ka <-> kb, values
  // va <-> vb except that the last pass (or k_keys itself when nothing has to be sorted) writes
  // the caller's gsid_per_patch
  KeyT *kin = ka;
  int32_t *vin = pp.n == 0 ? gsid_per_patch : va;
  {
    ProfScope ps(K_KEYS, st);
    k_keys<KeyT><<<(N + 255) / 256, 256, 0, st>>>(N, depths, incl, rects, gx, kp.shift, kp.depth_bits,
                                                  (uint32_t)P_cap, kin, vin, total + 2);
  }
  GSB_CUDA_TRY(cudaGetLastError());
  if (sr != nullptr) {  // everything the host has to validate is known now; the sort and the
    // rasterizer are enqueued behind this copy and run while the host waits for it
    GSB_CUDA_TRY(cudaMemcpyAsync(sr->host, total, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (sr->ready != nullptr) GSB_CUDA_TRY(cudaEventRecord(sr->ready, st));
  }
  {
    ProfScope ps(K_SORT, st);
    for (int p = 0; p < pp.n; p++) {
      KeyT *kout = (kin == ka) ? kb : ka;
      int32_t *vout = (p == pp.n - 1) ? gsid_per_patch : ((vin == va) ? vb : va);
      constexpr size_t dyn = RX_TILE * (sizeof(KeyT) + sizeof(int32_t));  // staging of the sorted tile
      if (pp.bits == 9) {  // (only 32-bit plans use 9-bit digits: key_plan)
        constexpr int B9 = sizeof(KeyT) == 4 ? 9 : 8;
        GSB_CUDA_TRY((radix_pass_smem_opt_in<KeyT, B9>((int)dyn)));
        k_digit_counts<KeyT, B9><<<tiles, RX_THREADS, 0, st>>>(kin, P_dev, (uint32_t)P_cap, pp.shift[p], tiles, counts,
                                                                 desc, (uint32_t)scan_grid, claim);
        k_colscan<<<scan_grid, CS_CTA, 0, st>>>(total + 2, nscan, counts, desc, claim);
        k_radix_pass<KeyT, B9><<<tiles, RX_THREADS, dyn, st>>>(kin, vin, kout, vout, P_dev, (uint32_t)P_cap,
                                                              pp.shift[p], tiles, counts);
      } else {
        GSB_CUDA_TRY((radix_pass_smem_opt_in<KeyT, 8>((int)dyn)));
        k_digit_counts<KeyT, 8><<<tiles, RX_THREADS, 0, st>>>(kin, P_dev, (uint32_t)P_cap, pp.shift[p], tiles, counts,
                                                                 desc, (uint32_t)scan_grid, claim);
        k_colscan<<<scan_grid, CS_CTA, 0, st>>>(total + 2, nscan, counts, desc, claim);
        k_radix_pass<KeyT, 8><<<tiles, RX_THREADS, dyn, st>>>(kin, vin, kout, vout, P_dev, (uint32_t)P_cap,
                                                              pp.shift[p], tiles, counts);
      }
      kin = kout;
      vin = vout;
    }
  }
  GSB_CUDA_TRY(cudaGetLastError());
  {
    ProfScope ps(K_RANGES, st);
    const size_t want = (size_t)((P_cap + 255) / 256);
    const int grid = (int)(want < (size_t)sms * 8 ? want : (size_t)sms * 8);
    k_ranges<KeyT><<<grid, 256, 0, st>>>(P_dev, (uint32_t)P_cap, total + 2, kin, kp.shift, (uint32_t)T,
                                         reinterpret_cast<int2 *>(ranges));
  }
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_sort_and_pack(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                         const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                         const void *bin_ws, const BinLayout &BL, void *ws, const SortLayout &SL,
                         int32_t *ranges, int32_t *gsid_per_patch, bool pack, const StatusRead *sr,
                         cudaStream_t st) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  GSB_CUDA_TRY(cudaMemsetAsync(ranges, 0, sizeof(int32_t) * 2 * (size_t)gx * gy, st));
  if (P <= 0 || N <= 0) return 0;
  if (P >= ((int64_t)1 << 30)) return set_arg_error("splat: more than 2^30 patches");
  const char *bb = static_cast<const char *>(bin_ws);
  char *b = static_cast<char *>(ws);
  const uint32_t *incl = reinterpret_cast<const uint32_t *>(bb + BL.offsets);
  const uint2 *rects = reinterpret_cast<const uint2 *>(bb + BL.rects);
  uint32_t *total = reinterpret_cast<uint32_t *>(const_cast<char *>(bb) + BL.total);  // [P, max key, flags]
  const KeyPlan kp = key_plan(H, W, depth_key_max);
  int rc = kp.narrow ? keys_sort_ranges<uint32_t>(N, P, depths, incl, rects, total, gx, gx * gy, kp, b, SL, ranges,
                                                  gsid_per_patch, sr, st)
                     : keys_sort_ranges<uint64_t>(N, P, depths, incl, rects, total, gx, gx * gy, kp, b, SL, ranges,
                                                  gsid_per_patch, sr, st);
  if (rc || !pack) return rc;  // !pack: the caller already holds the per-Gaussian records
  return launch_pack_only(N, nullptr, us, cinv2ds, alphas, colors, depths, reinterpret_cast<Rec *>(b + SL.recs), st);
}

}  // namespace gsb
