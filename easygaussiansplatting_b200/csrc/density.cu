// Density control (prune / clone / split with the Adam moments carried along) and Gaussian
// record conversion (PLY rows <-> .npy rows <-> the six training tensors).  SURVEY 8f row N3.
//
// Reference: gsplat/gsmodel.py:132-166 (update_params / prune_params), :219-234
// (update_density_info), :236-318 (update_gaussian_density), :320-331 (reset_alpha);
// gsplat/gau_io.py:60-107 (load_ply), :138-153 (save_training_params); gsmodel.py:95-113
// (get_training_params).
//
// The reference rebuilds all 18 tensors (6 parameters + exp_avg + exp_avg_sq) with boolean
// indexing and torch.cat, one tensor at a time, plus ~20 temporaries.  Here it is three
// streaming passes: classify (one byte per Gaussian) + per-CTA counts, a two-kernel exclusive
// scan of the three class counters (the output slot of every survivor / clone / split), and one
// apply kernel that moves every surviving row once and writes the new rows at the tail.  All of it is HBM-bound:
// algorithmic bytes = 24 N (classify + scan) + 2 * 708 * K + 708 * (C + S) for the full state
// (59 floats x 3 sets = 708 B per Gaussian).
//
// Transcendentals are the accurate expf / logf / sqrtf / IEEE division (no fast-math here):
// torch's CUDA kernels use the same libdevice routines, which keeps the clone / split values
// within an ulp of the reference's.
#include "common.cuh"
#include "kernels.h"
#include "pg_fused_math.h"
#include "plan_scan.cuh"
#include "tile_io.cuh"

namespace gsb {

namespace {

constexpr int kWidth[6] = {3, 3, 45, 1, 3, 4};  // pws, low_shs, high_shs, alphas_raw, scales_raw, rots_raw
enum : uint8_t { CLS_KEEP = 0, CLS_CLONE = 1, CLS_SPLIT = 2, CLS_PRUNE = 3 };

struct Slot3 {  // exclusive counts of survivors / clones / splits before this Gaussian
  int k, c, s;
};
// gsmodel.py:219-234.  init != 0 is the first call after a density update: the norm of every
// Gaussian is stored and the counter starts from the mask (:228-229).
__global__ void k_density_accumulate(int64_t N, const float *__restrict__ dus, const uint8_t *__restrict__ mask,
                                     float *__restrict__ acc, int32_t *__restrict__ cnt, int init) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float2 d = ld_pair(dus, i);  // any contiguous [N,2] view (tile_io.cuh)
  const float g = sqrtf(d.x * d.x + d.y * d.y);
  const bool m = mask[i] != 0;
  if (init) {
    acc[i] = g;
    cnt[i] = m;
  } else if (m) {
    acc[i] += g;
    cnt[i] += 1;
  }
}

// max that returns NaN when either input is NaN, like torch.max (fmaxf drops the NaN)
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// gsmodel.py:238-262.  Both maxima propagate NaN: a row with a NaN scale is neither pruned for
// size (NaN > thr is false) nor small enough to clone (NaN <= thr is false), as in the reference.
__device__ __forceinline__ uint8_t classify_row(int64_t i, const float *__restrict__ alphas_raw,
                                                const float *__restrict__ scales_raw, const float *__restrict__ acc,
                                                const int32_t *__restrict__ cnt, float alpha_raw_min,
                                                float scale_raw_max, float grad_min, float scale_clone_max) {
  const float a = alphas_raw[i];
  const float s0 = scales_raw[3 * i], s1 = scales_raw[3 * i + 1], s2 = scales_raw[3 * i + 2];
  const float smax = fmax_nan(s0, fmax_nan(s1, s2));
  uint8_t c;
  if (a < alpha_raw_min || smax > scale_raw_max) {
    c = CLS_PRUNE;
  } else {
    float g = acc[i] / (float)cnt[i];
    if (isnan(g)) g = 0.f;
    // max over exp(s) (the reference compares the activated scales, :257)
    const float big = fmax_nan(expf(s0), fmax_nan(expf(s1), expf(s2)));
    c = g >= grad_min ? (big <= scale_clone_max ? CLS_CLONE : CLS_SPLIT) : CLS_KEEP;
  }
  return c;
}

// ---- the plan scans.  Both plans (density slots, MCMC sampler) are an exclusive scan in row
// order, hand-written as three launches (plan_scan.cuh) and no library scan:
//   a row kernel      classifies / weighs 1024 rows per CTA and leaves the CTA's counters;
//   scan_blocks       one CTA turns the per-CTA counters into exclusive offsets + totals;
//   a row kernel      re-reads its CTA's rows (4 consecutive rows per thread), scans them
//                     locally and writes the per-row results.
// The counter tuples: inside a CTA the density kernels count (survivors | clones << 16, splits),
// at most SC_ROWS each, so a shuffle ladder step is two shuffles, not three; the density block
// counts are three int32 (Slot3); MCMC counts (uint64 weight, int32 dead) everywhere.
constexpr int SC_THREADS = 256, SC_PER = 4, SC_ROWS = SC_THREADS * SC_PER;

struct KcSp {
  uint32_t kc, sp;
};
struct WDead {
  uint64_t w;
  int32_t d;
};
__device__ __forceinline__ KcSp operator+(KcSp a, KcSp b) { return {a.kc + b.kc, a.sp + b.sp}; }
__device__ __forceinline__ KcSp operator-(KcSp a, KcSp b) { return {a.kc - b.kc, a.sp - b.sp}; }
__device__ __forceinline__ Slot3 operator+(Slot3 a, Slot3 b) { return {a.k + b.k, a.c + b.c, a.s + b.s}; }
__device__ __forceinline__ Slot3 operator-(Slot3 a, Slot3 b) { return {a.k - b.k, a.c - b.c, a.s - b.s}; }
__device__ __forceinline__ WDead operator+(WDead a, WDead b) { return {a.w + b.w, a.d + b.d}; }
__device__ __forceinline__ WDead operator-(WDead a, WDead b) { return {a.w - b.w, a.d - b.d}; }
__device__ __forceinline__ KcSp shfl_up(KcSp x, int o) {
  return {__shfl_up_sync(0xffffffffu, x.kc, o), __shfl_up_sync(0xffffffffu, x.sp, o)};
}
__device__ __forceinline__ Slot3 shfl_up(Slot3 x, int o) {
  return {__shfl_up_sync(0xffffffffu, x.k, o), __shfl_up_sync(0xffffffffu, x.c, o),
          __shfl_up_sync(0xffffffffu, x.s, o)};
}
__device__ __forceinline__ WDead shfl_up(WDead x, int o) {
  return {__shfl_up_sync(0xffffffffu, x.w, o), __shfl_up_sync(0xffffffffu, x.d, o)};
}
__device__ __forceinline__ KcSp warp_sum(KcSp x) {
  return {__reduce_add_sync(0xffffffffu, x.kc), __reduce_add_sync(0xffffffffu, x.sp)};
}
__device__ __forceinline__ WDead warp_sum(WDead x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x.w += __shfl_xor_sync(0xffffffffu, x.w, o);
  return {x.w, (int32_t)__reduce_add_sync(0xffffffffu, (uint32_t)x.d)};
}

// the density block counts: three int32 per CTA
struct DensityBlocks {
  using T = Slot3;
  int32_t *c;
  __device__ Slot3 load(int b) const { return {c[3 * b], c[3 * b + 1], c[3 * b + 2]}; }
  __device__ void store(int b, Slot3 x) const { c[3 * b] = x.k, c[3 * b + 1] = x.c, c[3 * b + 2] = x.s; }
  __device__ void totals(int64_t *t, Slot3 x) const { t[0] = x.k, t[1] = x.c, t[2] = x.s; }
};

__global__ void __launch_bounds__(1024) k_density_scan_blocks(int nb, DensityBlocks B, int64_t *__restrict__ totals) {
  scan_blocks(nb, B, totals);
}

__device__ __forceinline__ KcSp class_count(uint8_t c) {
  return {(c != CLS_PRUNE) + ((uint32_t)(c == CLS_CLONE) << 16), (uint32_t)(c == CLS_SPLIT)};
}

__global__ void __launch_bounds__(SC_THREADS) k_density_classify_count(
    int64_t N, const float *__restrict__ alphas_raw, const float *__restrict__ scales_raw,
    const float *__restrict__ acc, const int32_t *__restrict__ cnt, float alpha_raw_min, float scale_raw_max,
    float grad_min, float scale_clone_max, uint8_t *__restrict__ cls, int32_t *__restrict__ block_counts) {
  __shared__ KcSp red[SC_THREADS / 32];
  KcSp n{0, 0};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    const int64_t i = (int64_t)blockIdx.x * SC_ROWS + j * SC_THREADS + threadIdx.x;
    if (i < N) {
      const uint8_t c =
          classify_row(i, alphas_raw, scales_raw, acc, cnt, alpha_raw_min, scale_raw_max, grad_min, scale_clone_max);
      cls[i] = c;
      n = n + class_count(c);
    }
  }
  n = cta_sum<SC_THREADS>(n, red);
  if (threadIdx.x == 0)
    DensityBlocks{block_counts}.store(blockIdx.x, {(int)(n.kc & 0xffffu), (int)(n.kc >> 16), (int)n.sp});
}

// the classify pass of a prune by mask (gsb_density_plan_keep): keep[i] != 0 -> CLS_KEEP, else CLS_PRUNE
__global__ void __launch_bounds__(SC_THREADS) k_density_keep_count(int64_t N, const uint8_t *__restrict__ keep,
                                                                   uint8_t *__restrict__ cls,
                                                                   int32_t *__restrict__ block_counts) {
  __shared__ KcSp red[SC_THREADS / 32];
  KcSp n{0, 0};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    const int64_t i = (int64_t)blockIdx.x * SC_ROWS + j * SC_THREADS + threadIdx.x;
    if (i < N) {
      const uint8_t c = keep[i] != 0 ? CLS_KEEP : CLS_PRUNE;
      cls[i] = c;
      n = n + class_count(c);
    }
  }
  n = cta_sum<SC_THREADS>(n, red);
  if (threadIdx.x == 0) DensityBlocks{block_counts}.store(blockIdx.x, {(int)(n.kc & 0xffffu), 0, 0});
}

__global__ void __launch_bounds__(SC_THREADS) k_density_slots(int64_t N, const uint8_t *__restrict__ cls,
                                                              const DensityBlocks block_offsets,
                                                              Slot3 *__restrict__ slots) {
  __shared__ KcSp warp_tot[SC_THREADS / 32];
  const int64_t row0 = (int64_t)blockIdx.x * SC_ROWS + (int64_t)threadIdx.x * SC_PER;
  uint8_t c[SC_PER];
  KcSp n{0, 0};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    c[j] = row0 + j < N ? cls[row0 + j] : (uint8_t)CLS_PRUNE;
    n = n + class_count(c[j]);
  }
  KcSp total;
  const KcSp b = cta_exclusive_scan<SC_THREADS>(n, warp_tot, total);
  Slot3 run = block_offsets.load(blockIdx.x) + Slot3{(int)(b.kc & 0xffffu), (int)(b.kc >> 16), (int)b.sp};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    if (row0 + j < N) slots[row0 + j] = run;
    run.k += c[j] != CLS_PRUNE, run.c += c[j] == CLS_CLONE, run.s += c[j] == CLS_SPLIT;
  }
}

// One per-Gaussian tensor and its Adam moments (m, v: both or neither, NULL without optimizer
// state), source and destination; the six training tensors are Jobs::j[0..5] (kWidth).  An extra
// tensor [N, D] (per-Gaussian features) is one Job of width D.
struct Job {
  const float *p, *m, *v;  // sources
  float *dp, *dm, *dv;     // destinations (relocate: the sources)
  int w;
};
struct Jobs {
  Job j[6];
};
// from the six-pointer tables of gsb_gaussians; NULL moment tables give NULL moments
Jobs jobs(float *const *src, float *const *src_m, float *const *src_v, float *const *dst, float *const *dst_m,
          float *const *dst_v) {
  Jobs J;
  for (int a = 0; a < 6; a++)
    J.j[a] = Job{src[a], src_m ? src_m[a] : nullptr, src_v ? src_v[a] : nullptr, dst[a],
                 dst_m ? dst_m[a] : nullptr, dst_v ? dst_v[a] : nullptr, kWidth[a]};
  return J;
}

__device__ __forceinline__ float logit_of_sigmoid(float x) {
  const float a = 1.f / (1.f + expf(-x));  // get_alphas
  return logf(a / (1.f - a));              // get_alphas_raw
}

// utils.py:46-54 on the normalised quaternion, v = z * exp(scales_raw)
__device__ __forceinline__ float split_offset(const float *__restrict__ q4, const float *__restrict__ s3,
                                              const float *__restrict__ z3, int comp) {
  float w = q4[0], x = q4[1], y = q4[2], z = q4[3];
  float n = fmaxf(sqrtf(w * w + x * x + y * y + z * z), 1e-12f);  // get_rots
  w /= n, x /= n, y /= n, z /= n;
  n = fmaxf(sqrtf(w * w + x * x + y * y + z * z), 1e-12f);        // normalize() inside rotate_vector
  w /= n, x /= n, y /= n, z /= n;
  const float v0 = z3[0] * expf(s3[0]), v1 = z3[1] * expf(s3[1]), v2 = z3[2] * expf(s3[2]);
  const float uv = x * v0 + y * v1 + z * v2, uu = x * x + y * y + z * z;
  const float c0 = y * v2 - z * v1, c1 = z * v0 - x * v2, c2 = x * v1 - y * v0;
  const float u = comp == 0 ? x : (comp == 1 ? y : z);
  const float v = comp == 0 ? v0 : (comp == 1 ? v1 : v2);
  const float c = comp == 0 ? c0 : (comp == 1 ? c1 : c2);
  return 2.f * u * uv + v * (w * w - uu) + 2.f * c * w;
}

// ---- the rebuild: one job per (tensor, set) pair -- 6 tensors x {parameter, exp_avg,
// exp_avg_sq} = 18 jobs on blockIdx.y.  Survivors move to their compacted row; clones / splits
// additionally produce a new row at K + slot (clones) or K + C + slot (splits): the recomputed
// value for a parameter, zero for an Adam moment.  A warp moves 32 consecutive Gaussians of one
// array.  The per-Gaussian plan (class, survivor slot, new-row slot) is read once per group into
// a 32-entry shared-memory table instead of once per element.  Loads and stores are 4-byte but
// fully coalesced: lane l handles elements
// l, l + 32, ... of the group's contiguous source span, 12 loads in flight per lane for the wide
// arrays; consecutive survivors are consecutive in the destination too, so a store instruction
// writes whole 32-byte sectors.  (Reading the span with float4 loads would force the four
// components out with stride-16-byte stores: quarter-filled sectors.)  Elements of pruned Gaussians are not loaded.
constexpr int DG_WARPS = 8;
constexpr int DG_PAIRS = 4;  // pairs of 45-wide rows in flight per lane (3 loads each)

// the value a clone / split writes at its new row (parameters; Adam moments start at 0)
template <int A>
__device__ __forceinline__ float new_row_value(float val, bool split, int64_t i, int s, int c, const Jobs &J,
                                               const float *__restrict__ z) {
  float nv = val;
  if (A == 0) {
    if (split) nv += split_offset(J.j[5].p + 4 * i, J.j[4].p + 3 * i, z + 3 * (int64_t)s, c);
  } else if (A == 3) {
    nv = logit_of_sigmoid(nv);
  } else if (A == 4) {
    const float e = expf(nv);          // get_scales
    nv = logf(split ? e * 0.6f : e);   // gsmodel.py:281 then get_scales_raw
  } else if (A == 5) {
    const float *q = J.j[5].p + 4 * i;
    nv = nv / fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
  }
  return nv;
}

template <class Off, int A, int SET>
__device__ __forceinline__ void rows_job(int row0, const int2 *__restrict__ tab, int K, int C, const Jobs &J,
                                         const float *__restrict__ z, int lane) {
  constexpr int w = kWidth[A];
  const float *__restrict__ src = SET == 0 ? J.j[A].p : (SET == 1 ? J.j[A].m : J.j[A].v);
  float *__restrict__ dst = SET == 0 ? J.j[A].dp : (SET == 1 ? J.j[A].dm : J.j[A].dv);
  if (src == nullptr) return;
  const float *__restrict__ gsrc = src + (size_t)row0 * w;
  // element (row r of the group, column col) with plan entry `info`
  auto emit = [&](int r, int col, int2 info, float val) {
    const unsigned cl = (unsigned)info.x >> 30;
    if (cl == CLS_PRUNE) return;
    dst[(Off)(info.x & 0x3fffffff) * w + col] = val;
    if (cl == CLS_KEEP) return;
    float nv = 0.f;
    if (SET == 0) nv = new_row_value<A>(val, cl == CLS_SPLIT, (int64_t)row0 + r, info.y - K - C, col, J, z);
    dst[(Off)info.y * w + col] = nv;
  };
  const int2 pruned = make_int2((int)((unsigned)CLS_PRUNE << 30), 0);
  // Fixed lane -> (row, column) maps: table entries of rows past the end of the array are
  // CLS_PRUNE, so no row bound is checked; destination element offsets (up to 2 N * 45) are Off
  constexpr bool plain = SET != 0 || A == 1 || A == 2;  // the new row is a copy (parameters) or zero (moments)
  auto emit_fixed = [&](int r, int col, int2 info, float val) {
    if constexpr (plain) {  // two predicated stores, no branches
      const unsigned cl = (unsigned)info.x >> 30;
      if (cl != CLS_PRUNE) dst[(Off)(info.x & 0x3fffffff) * w + col] = val;
      if (cl == CLS_CLONE || cl == CLS_SPLIT) dst[(Off)info.y * w + col] = SET == 0 ? val : 0.f;
    } else {
      emit(r, col, info, val);
    }
  };
  if constexpr (w == 45) {
    // Two rows = 90 elements = three rounds of 32 lanes (94 % of the lanes busy): which of the two
    // rows and which column a lane handles in each round does not depend on the pair, so no
    // element index is divided by 45; DG_PAIRS pairs (3 DG_PAIRS loads) in flight per lane.
    const int rsel[3] = {0, lane >= 13, 1};
    const int col[3] = {lane, lane < 13 ? 32 + lane : lane - 13, 19 + lane};
#pragma unroll 1
    for (int p0 = 0; p0 < 16; p0 += DG_PAIRS) {
      float v[DG_PAIRS][3];
      int2 info[DG_PAIRS][3];
#pragma unroll
      for (int q = 0; q < DG_PAIRS; q++)
#pragma unroll
        for (int rd = 0; rd < 3; rd++) {
          info[q][rd] = tab[2 * (p0 + q) + rsel[rd]];
          if (rd == 2 && lane >= 26) info[q][rd] = pruned;  // 90 elements: the third round has 26
        }
#pragma unroll
      for (int q = 0; q < DG_PAIRS; q++)
#pragma unroll
        for (int rd = 0; rd < 3; rd++) {  // all loads are issued before any is consumed
          v[q][rd] = 0.f;
          if (((unsigned)info[q][rd].x >> 30) != CLS_PRUNE)
            v[q][rd] = __ldg(gsrc + (2 * (p0 + q) + rsel[rd]) * w + col[rd]);
        }
#pragma unroll
      for (int q = 0; q < DG_PAIRS; q++)
#pragma unroll
        for (int rd = 0; rd < 3; rd++) emit_fixed(2 * (p0 + q) + rsel[rd], col[rd], info[q][rd], v[q][rd]);
    }
  } else {
    // w = 1, 3, 4: the whole group is w rounds of 32 lanes, row and column of a lane's element in
    // round u are the same for every group (hoisted out of the group loop by the compiler)
    float v[w];
    int2 info[w];
#pragma unroll
    for (int u = 0; u < w; u++) info[u] = tab[(32 * u + lane) / w];
#pragma unroll
    for (int u = 0; u < w; u++) {
      v[u] = 0.f;
      if (((unsigned)info[u].x >> 30) != CLS_PRUNE) v[u] = __ldg(gsrc + 32 * u + lane);
    }
#pragma unroll
    for (int u = 0; u < w; u++) {
      const int e = 32 * u + lane, r = e / w;
      emit_fixed(r, e - r * w, info[u], v[u]);
    }
  }
}

template <class Off, int A, int SET>
__device__ __noinline__ void rows_loop(int N, const uint8_t *__restrict__ cls, const Slot3 *__restrict__ slots, int K,
                                       int C, const Jobs &J, const float *__restrict__ z, int2 *tab) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int groups = (N + 31) / 32;
  for (int g = blockIdx.x * DG_WARPS + wid; g < groups; g += gridDim.x * DG_WARPS) {
    const int row0 = g * 32, row = row0 + lane;
    uint8_t c = CLS_PRUNE;
    Slot3 sl{0, 0, 0};
    if (row < N) {
      c = cls[row];
      sl = slots[row];
    }
    // (class | survivor slot, new-row slot); slots < N < 2^30 (gsb_density_apply checks N)
    tab[lane] = make_int2((int)((unsigned)c << 30) | sl.k, c == CLS_SPLIT ? K + C + sl.s : K + sl.c);
    __syncwarp();
    rows_job<Off, A, SET>(row0, tab, K, C, J, z, lane);
    __syncwarp();  // the table is rewritten for the next group
  }
}

// Off: the type of the destination element offsets.  uint32_t while they stay below 2^31 (2 N * 45 <
// 2^31 for N < 23 M): the narrower address arithmetic makes the rebuild ~7 % faster at N = 1 M
// (DESIGN §3, kernel table); size_t above
template <class Off>
__global__ void __launch_bounds__(32 * DG_WARPS) k_density_apply_rows(int N, const uint8_t *__restrict__ cls,
                                                                       const Slot3 *__restrict__ slots, int K, int C,
                                                                       const __grid_constant__ Jobs J,
                                                                       const float *__restrict__ z) {
  __shared__ int2 tabs[DG_WARPS][32];
  int2 *tab = tabs[threadIdx.x >> 5];
#define GSB_JOB(y, a, s) \
  case y: rows_loop<Off, a, s>(N, cls, slots, K, C, J, z, tab); break;
  switch (blockIdx.y) {
    GSB_JOB(0, 2, 0) GSB_JOB(1, 2, 1) GSB_JOB(2, 2, 2) GSB_JOB(3, 0, 0) GSB_JOB(4, 0, 1) GSB_JOB(5, 0, 2)
    GSB_JOB(6, 1, 0) GSB_JOB(7, 1, 1) GSB_JOB(8, 1, 2) GSB_JOB(9, 3, 0) GSB_JOB(10, 3, 1) GSB_JOB(11, 3, 2)
    GSB_JOB(12, 4, 0) GSB_JOB(13, 4, 1) GSB_JOB(14, 4, 2) GSB_JOB(15, 5, 0) GSB_JOB(16, 5, 1) GSB_JOB(17, 5, 2)
  }
#undef GSB_JOB
}

// gsb_density_apply_rows: the plan applied to one more [N, D] tensor of any width D (per-Gaussian
// features), blockIdx.y = the set (parameter, exp_avg, exp_avg_sq).  Grid-stride over the N D
// elements; a survivor's element moves to its compacted row, a clone's or split's element is also
// written at its new row -- a copy for the parameter, 0 for an Adam moment.  Elements of pruned
// Gaussians are not loaded.
__global__ void __launch_bounds__(256) k_density_copy_rows(int64_t N, int D, const uint8_t *__restrict__ cls,
                                                           const Slot3 *__restrict__ slots, int64_t K, int64_t C,
                                                           const float *__restrict__ src0,
                                                           const float *__restrict__ src1,
                                                           const float *__restrict__ src2, float *__restrict__ dst0,
                                                           float *__restrict__ dst1, float *__restrict__ dst2) {
  const int set = blockIdx.y;
  const float *__restrict__ src = set == 0 ? src0 : (set == 1 ? src1 : src2);
  float *__restrict__ dst = set == 0 ? dst0 : (set == 1 ? dst1 : dst2);
  if (src == nullptr) return;
  const int64_t total = N * D, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const int64_t i = e / D;
    const int c = (int)(e - i * D);
    const uint8_t cl = cls[i];
    if (cl == CLS_PRUNE) continue;
    const Slot3 sl = slots[i];
    const float v = src[e];
    dst[(int64_t)sl.k * D + c] = v;
    if (cl == CLS_KEEP) continue;
    const int64_t r = cl == CLS_SPLIT ? K + C + sl.s : K + sl.c;
    dst[r * D + c] = set == 0 ? v : 0.f;
  }
}

// gsmodel.py:320-331
__global__ void k_reset_alpha(int64_t N, float *__restrict__ alphas_raw, float *__restrict__ m,
                              float *__restrict__ v, float val) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (alphas_raw[i] > val) alphas_raw[i] = val;
  if (m) m[i] = 0.f;
  if (v) v[i] = 0.f;
}

// ---- record conversion.  A "gs row" is the reference's .npy record (gau_io.py:7-12):
// pw[3] rot[4] scale[3] alpha sh[sh_dim], 11 + sh_dim floats, activated values.

// gau_io.py:60-107.  rows: the PLY vertex block [N, stride] f32; colmap[j] = source column of
// output column j (the f_rest channel-major -> coefficient-major transpose of :91 is folded
// into the map by the host).  rot is divided by its norm (no epsilon, :80), scale -> exp,
// opacity -> sigmoid.
__global__ void k_ply_rows_to_gs(int64_t N, int stride, int J, const float *__restrict__ rows,
                                 const int32_t *__restrict__ colmap, float *__restrict__ out) {
  const int64_t total = N * J;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / J;
    const int j = (int)(e - i * J);
    const float *__restrict__ row = rows + i * stride;
    float v = row[colmap[j]];
    if (j >= 3 && j < 7) {
      const float a = row[colmap[3]], b = row[colmap[4]], c = row[colmap[5]], d = row[colmap[6]];
      v = v / sqrtf(a * a + b * b + c * c + d * d);
    } else if (j >= 7 && j < 10) {
      v = expf(v);
    } else if (j == 10) {
      v = 1.f / (1.f + expf(-v));
    }
    out[e] = v;
  }
}

// gsmodel.py:95-113: gs rows -> raw training tensors; high_shs padded with 0.001 up to 45
__global__ void k_gs_to_params(int64_t N, int sh_dim, const float *__restrict__ gs, float *__restrict__ pws,
                               float *__restrict__ low, float *__restrict__ high, float *__restrict__ alphas_raw,
                               float *__restrict__ scales_raw, float *__restrict__ rots_raw) {
  const int J = 11 + sh_dim;
  const int64_t total = N * 59;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / 59;
    const int c = (int)(e - i * 59);
    const float *__restrict__ row = gs + i * J;
    if (c < 3) {
      pws[3 * i + c] = row[c];
    } else if (c < 7) {
      rots_raw[4 * i + c - 3] = row[c];
    } else if (c < 10) {
      scales_raw[3 * i + c - 7] = logf(row[c]);
    } else if (c == 10) {
      const float a = row[10];
      alphas_raw[i] = logf(a / (1.f - a));
    } else if (c < 14) {
      low[3 * i + c - 11] = row[c];
    } else {
      const int h = c - 14;
      high[45 * i + h] = (h + 3 < sh_dim) ? row[c] : 0.001f;
    }
  }
}

// gau_io.py:138-153: training tensors -> gs rows with sh_dim = 48
__global__ void k_params_to_gs(int64_t N, const float *__restrict__ pws, const float *__restrict__ low,
                               const float *__restrict__ high, const float *__restrict__ alphas_raw,
                               const float *__restrict__ scales_raw, const float *__restrict__ rots_raw,
                               float *__restrict__ gs) {
  const int64_t total = N * 59;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / 59;
    const int c = (int)(e - i * 59);
    float v;
    if (c < 3) {
      v = pws[3 * i + c];
    } else if (c < 7) {
      const float *q = rots_raw + 4 * i;
      v = q[c - 3] / fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
    } else if (c < 10) {
      v = expf(scales_raw[3 * i + c - 7]);
    } else if (c == 10) {
      v = 1.f / (1.f + expf(-alphas_raw[i]));
    } else if (c < 14) {
      v = low[3 * i + c - 11];
    } else {
      v = high[45 * i + c - 14];
    }
    gs[e] = v;
  }
}

inline int stream_grid(int64_t total, int block) {
  int64_t b = (total + block - 1) / block;
  const int64_t cap = 132 * 16;  // grid-stride: a few waves of the 132 SMs
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---- MCMC densification (Kheradmand et al. 2024): relocate dead Gaussians onto live ones, grow
// to a budget, covariance-shaped position noise.  DESIGN 3.11.
//
// The sampler is integer arithmetic so that its ids do not depend on summation order: row i has
// the weight q_i = floor(o_i 2^32) (o_i = sigmoid of the fp32 raw value, in fp64; 0 for excluded
// rows), W = the uint64 inclusive prefix sum, and a uniform u picks the first i with
// W_i > floor(u W_total).  The scan is a plan scan (above):
//   k_mcmc_weight_count         per-CTA weight sum and dead count of 1024 rows;
//   k_mcmc_scan_blocks          one CTA turns them into exclusive offsets and the totals;
//   k_mcmc_prefix               every CTA rescans its rows, writes W, the dead-row list, and
//                               clears the per-row sample counts.
enum : int { MCMC_RELOCATE = 0, MCMC_GROW = 1 };

// relocate samples alive rows (dead = !(a > alpha_raw_min), NaN included); grow samples every
// row that is not NaN
__device__ __forceinline__ uint64_t mcmc_weight(float a, float alpha_raw_min, int mode, bool &dead) {
  dead = !(a > alpha_raw_min);
  if (isnan(a) || (mode == MCMC_RELOCATE && dead)) return 0;
  const double o = 1.0 / (1.0 + exp(-(double)a));
  return (uint64_t)floor(o * 4294967296.0);
}

// the MCMC block counters: a uint64 weight sum and an int32 dead count per CTA, in two arrays
struct McmcBlocks {
  using T = WDead;
  uint64_t *w;
  int32_t *d;
  __device__ WDead load(int b) const { return {w[b], d[b]}; }
  __device__ void store(int b, WDead x) const { w[b] = x.w, d[b] = x.d; }
  __device__ void totals(int64_t *t, WDead x) const { t[0] = (int64_t)x.w, t[1] = x.d; }
};

__global__ void __launch_bounds__(1024) k_mcmc_scan_blocks(int nb, McmcBlocks B, int64_t *__restrict__ totals) {
  scan_blocks(nb, B, totals);
}

__global__ void __launch_bounds__(SC_THREADS) k_mcmc_weight_count(int64_t N, const float *__restrict__ alphas_raw,
                                                                   float alpha_raw_min, int mode,
                                                                   const McmcBlocks blocks) {
  __shared__ WDead red[SC_THREADS / 32];
  WDead n{0, 0};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    const int64_t i = (int64_t)blockIdx.x * SC_ROWS + j * SC_THREADS + threadIdx.x;
    if (i < N) {
      bool dd;
      n.w += mcmc_weight(alphas_raw[i], alpha_raw_min, mode, dd);
      n.d += dd;
    }
  }
  n = cta_sum<SC_THREADS>(n, red);
  if (threadIdx.x == 0) blocks.store(blockIdx.x, n);
}

__global__ void __launch_bounds__(SC_THREADS) k_mcmc_prefix(int64_t N, const float *__restrict__ alphas_raw,
                                                             float alpha_raw_min, int mode, const McmcBlocks blocks,
                                                             uint64_t *__restrict__ W, int32_t *__restrict__ dead,
                                                             int32_t *__restrict__ count) {
  __shared__ WDead warp_tot[SC_THREADS / 32];
  const int64_t row0 = (int64_t)blockIdx.x * SC_ROWS + (int64_t)threadIdx.x * SC_PER;
  uint64_t w[SC_PER];
  bool dd[SC_PER];
  WDead n{0, 0};
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    w[j] = 0, dd[j] = false;
    if (row0 + j < N) w[j] = mcmc_weight(alphas_raw[row0 + j], alpha_raw_min, mode, dd[j]);
    n.w += w[j], n.d += dd[j];
  }
  WDead total;
  const WDead before = blocks.load(blockIdx.x) + cta_exclusive_scan<SC_THREADS>(n, warp_tot, total);
  uint64_t rw = before.w;
  int rd = before.d;
#pragma unroll
  for (int j = 0; j < SC_PER; j++) {
    const int64_t i = row0 + j;
    if (i >= N) break;
    rw += w[j];
    W[i] = rw;
    count[i] = 0;
    if (mode == MCMC_RELOCATE && dd[j]) dead[rd++] = (int)i;
  }
}

// sampled[j] = the first i with W_i > t_j, t_j = min(floor(u_j W_total), W_total - 1); count[i] =
// how many draws hit row i
__global__ void k_mcmc_sample(int64_t N, int64_t n, const double *__restrict__ u, const uint64_t *__restrict__ W,
                              const int64_t *__restrict__ totals, int32_t *__restrict__ sampled,
                              int32_t *__restrict__ count) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t total = (uint64_t)totals[0];
  uint64_t t = (uint64_t)floor(u[j] * (double)total);
  if (t >= total) t = total - 1;
  int64_t lo = 0, hi = N - 1;  // W_{N-1} = total > t: the answer is in [lo, hi]
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (W[mid] > t) hi = mid;
    else lo = mid + 1;
  }
  sampled[j] = (int32_t)lo;
  atomicAdd(count + lo, 1);
}

// The relocation value of a source hit c times, in fp64 (DESIGN 3.11): r = min(c + 1, n_max) copies
// share its opacity, o' = 1 - (1 - o)^(1/r), and its scale shrinks by o / sum_m C(r,m) (-1)^(m+1)
// o'^m / sqrt(m), so that the r copies together render what the source did.  The alternating sum's
// terms reach ~2e5 at r = 51 against a result of order 1: an fp32 evaluation would lose most of
// its digits.  Each output is rounded to fp32 once.
__device__ __forceinline__ float4 relocation_value(float a, const float *__restrict__ s3, int c, double min_opacity,
                                                   int n_max) {
  const int r = min(c + 1, n_max);
  // o and 1 - o each from its own sigmoid: 1 - o formed from o would keep no digits of a nearly
  // opaque source's transparency, and o' and logit(o') are made from it
  const double o = 1.0 / (1.0 + exp(-(double)a)), om = 1.0 / (1.0 + exp((double)a));
  double op = o, q = om;  // o' and 1 - o'; r = 1 keeps o exactly (the scale factor is then 1)
  if (r > 1) q = pow(om, 1.0 / r), op = 1.0 - q;
  if (op < min_opacity) op = min_opacity, q = 1.0 - min_opacity;
  else if (q < 0x1p-23) q = 0x1p-23, op = 1.0 - 0x1p-23;
  double denom = 0.0, binom = 1.0, p = 1.0;
  for (int m = 1; m <= r; m++) {
    binom = binom * (double)(r - m + 1) / (double)m;  // C(r, m), exact for r <= 51
    p *= op;
    const double term = binom * p / sqrt((double)m);
    denom += (m & 1) ? term : -term;
  }
  const double f = log(o / denom);
  return make_float4((float)log(op / q), (float)((double)s3[0] + f), (float)((double)s3[1] + f),
                     (float)((double)s3[2] + f));
}

// vals[j] = the relocation value of sampled[j], from the unmodified source, before any row moves
__global__ void k_mcmc_values(int64_t n, const int32_t *__restrict__ sampled, const int32_t *__restrict__ count,
                              const float *__restrict__ alphas_raw, const float *__restrict__ scales_raw,
                              double min_opacity, int n_max, float4 *__restrict__ vals) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t i = sampled[j];
  vals[j] = relocation_value(alphas_raw[i], scales_raw + 3 * i, count[i], min_opacity, n_max);
}

// the value a sampled source row gets at column c (alphas_raw, scales_raw: the relocation value)
template <int A>
__device__ __forceinline__ float source_value(const float *__restrict__ p, int64_t src, int c, int w,
                                              const float4 &val) {
  if (A == 3) return val.x;
  if (A == 4) return c == 0 ? val.y : (c == 1 ? val.z : val.w);
  return p[src * w + c];
}

// relocate, in place: the source's opacity and scale become the relocation value, dead row dead[j]
// becomes a copy of the updated source sampled[j]; the moments of both rows are zeroed.  The new
// values come from vals[] and every other column of a source is only read (a source is alive, a
// destination dead), so several dead rows may copy one source in any order.
template <int A>
__device__ __forceinline__ void relocate_job(int64_t n, const int32_t *__restrict__ sampled,
                                             const int32_t *__restrict__ dead, const float4 *__restrict__ vals,
                                             const Job &J) {
  const int w = A < 6 ? kWidth[A < 6 ? A : 0] : J.w;
  const int64_t total = n * w, stride = (int64_t)gridDim.x * blockDim.x;
  float *__restrict__ p = J.dp;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const int64_t j = e / w;
    const int c = (int)(e - j * w);
    const int64_t src = sampled[j], dst = dead[j];
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (A == 3 || A == 4) val = vals[j];
    const float x = source_value<A>(p, src, c, w, val);
    p[dst * w + c] = x;
    if (A == 3 || A == 4) p[src * w + c] = x;
    if (J.dm) {
      J.dm[src * w + c] = 0.f, J.dm[dst * w + c] = 0.f;
      J.dv[src * w + c] = 0.f, J.dv[dst * w + c] = 0.f;
    }
  }
}

__global__ void __launch_bounds__(256) k_mcmc_relocate(int64_t n, const int32_t *__restrict__ sampled,
                                                       const int32_t *__restrict__ dead,
                                                       const float4 *__restrict__ vals,
                                                       const __grid_constant__ Jobs J) {
  switch (blockIdx.y) {
    case 0: relocate_job<0>(n, sampled, dead, vals, J.j[0]); break;
    case 1: relocate_job<1>(n, sampled, dead, vals, J.j[1]); break;
    case 2: relocate_job<2>(n, sampled, dead, vals, J.j[2]); break;
    case 3: relocate_job<3>(n, sampled, dead, vals, J.j[3]); break;
    case 4: relocate_job<4>(n, sampled, dead, vals, J.j[4]); break;
    case 5: relocate_job<5>(n, sampled, dead, vals, J.j[5]); break;
  }
}

__global__ void __launch_bounds__(256) k_mcmc_relocate_rows(int64_t n, const int32_t *__restrict__ sampled,
                                                            const int32_t *__restrict__ dead,
                                                            const __grid_constant__ Job J) {
  relocate_job<6>(n, sampled, dead, nullptr, J);
}

// grow, part 1: rows [0, N) of the fresh tensors are the old rows; a sampled source (count > 0)
// gets zero moments.  blockIdx.y = the set (parameter, exp_avg, exp_avg_sq); four independent
// elements in flight per thread.
template <int A>
__device__ __forceinline__ void grow_copy_job(int64_t N, const int32_t *__restrict__ count, const Job &J,
                                              int set) {
  const int w = A < 6 ? kWidth[A < 6 ? A : 0] : J.w;
  const float *__restrict__ src = set == 0 ? J.p : (set == 1 ? J.m : J.v);
  float *__restrict__ dst = set == 0 ? J.dp : (set == 1 ? J.dm : J.dv);
  if (src == nullptr) return;
  constexpr int U = 4;
  const int64_t total = N * w, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e0 < total; e0 += stride * U) {
    float x[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int64_t e = e0 + u * stride;
      x[u] = 0.f;
      if (e < total && (set == 0 || count[e / w] == 0)) x[u] = src[e];
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int64_t e = e0 + u * stride;
      if (e < total) dst[e] = x[u];
    }
  }
}

__global__ void __launch_bounds__(256) k_mcmc_grow_copy(int64_t N, const int32_t *__restrict__ count,
                                                        const __grid_constant__ Jobs J) {
  const int set = blockIdx.y % 3;
  switch (blockIdx.y / 3) {
    case 0: grow_copy_job<0>(N, count, J.j[0], set); break;
    case 1: grow_copy_job<1>(N, count, J.j[1], set); break;
    case 2: grow_copy_job<2>(N, count, J.j[2], set); break;
    case 3: grow_copy_job<3>(N, count, J.j[3], set); break;
    case 4: grow_copy_job<4>(N, count, J.j[4], set); break;
    case 5: grow_copy_job<5>(N, count, J.j[5], set); break;
  }
}

// grow, part 2 (after part 1): row N + j is a copy of the updated source sampled[j] with zero
// moments, and the source row itself gets the relocation value
template <int A>
__device__ __forceinline__ void grow_append_job(int64_t N, int64_t n, const int32_t *__restrict__ sampled,
                                                const float4 *__restrict__ vals, const Job &J) {
  const int w = A < 6 ? kWidth[A < 6 ? A : 0] : J.w;
  const int64_t total = n * w, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const int64_t j = e / w;
    const int c = (int)(e - j * w);
    const int64_t src = sampled[j], dst = N + j;
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (A == 3 || A == 4) val = vals[j];
    const float x = source_value<A>(J.p, src, c, w, val);
    J.dp[dst * w + c] = x;
    if (A == 3 || A == 4) J.dp[src * w + c] = x;
    if (J.dm) J.dm[dst * w + c] = 0.f, J.dv[dst * w + c] = 0.f;
  }
}

__global__ void __launch_bounds__(256) k_mcmc_grow_append(int64_t N, int64_t n, const int32_t *__restrict__ sampled,
                                                          const float4 *__restrict__ vals,
                                                          const __grid_constant__ Jobs J) {
  switch (blockIdx.y) {
    case 0: grow_append_job<0>(N, n, sampled, vals, J.j[0]); break;
    case 1: grow_append_job<1>(N, n, sampled, vals, J.j[1]); break;
    case 2: grow_append_job<2>(N, n, sampled, vals, J.j[2]); break;
    case 3: grow_append_job<3>(N, n, sampled, vals, J.j[3]); break;
    case 4: grow_append_job<4>(N, n, sampled, vals, J.j[4]); break;
    case 5: grow_append_job<5>(N, n, sampled, vals, J.j[5]); break;
  }
}

__global__ void __launch_bounds__(256) k_mcmc_grow_rows(int64_t N, int64_t n, const int32_t *__restrict__ count,
                                                        const int32_t *__restrict__ sampled,
                                                        const __grid_constant__ Job J, int part) {
  if (part == 0) grow_copy_job<6>(N, count, J, blockIdx.y);
  else if (blockIdx.y == 0) grow_append_job<6>(N, n, sampled, nullptr, J);
}

// pws += Sigma(q, s) z * scale / (1 + exp(-k ((1 - o) - x0))), Sigma = R S^2 R^T of the normalised
// quaternion and the raw scales (pg_fused_math.h), scale = lr * noise_lr.  68 B per Gaussian.
__global__ void __launch_bounds__(256) k_mcmc_noise(int64_t N, float *__restrict__ pws,
                                                    const float *__restrict__ alphas_raw,
                                                    const float *__restrict__ scales_raw,
                                                    const float *__restrict__ rots_raw, const float *__restrict__ z,
                                                    float scale, float k, float x0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  // the gate in fp64: it is steep (slope k / 4) where 1 - o crosses x0, so an fp32 1 - o would
  // carry ~1e-5 relative error into it; ~40 fp64 operations per Gaussian are hidden by the loads
  const double one_minus_o = 1.0 / (1.0 + exp((double)alphas_raw[i]));
  const float gate = (float)(1.0 / (1.0 + exp(-(double)k * (one_minus_o - (double)x0))));
  float q[4] = {rots_raw[4 * i], rots_raw[4 * i + 1], rots_raw[4 * i + 2], rots_raw[4 * i + 3]};
  const float nq = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
#pragma unroll
  for (int c = 0; c < 4; c++) q[c] /= nq;
  const float s[3] = {expf(scales_raw[3 * i]), expf(scales_raw[3 * i + 1]), expf(scales_raw[3 * i + 2])};
  float R3[9], M3[9], S6[6];
  pg::cov3d(q, s, R3, M3, S6);
  const float z0 = z[3 * i], z1 = z[3 * i + 1], z2 = z[3 * i + 2];
  const float f = scale * gate;
  pws[3 * i] += f * (S6[0] * z0 + S6[1] * z1 + S6[2] * z2);
  pws[3 * i + 1] += f * (S6[1] * z0 + S6[3] * z1 + S6[4] * z2);
  pws[3 * i + 2] += f * (S6[2] * z0 + S6[4] * z1 + S6[5] * z2);
}

// [totals: W_total, dead count; 256 B][block weight sums: nb u64][block dead counts: nb i32, 256-B
// padded][W: N u64][count: N i32][dead: N i32][vals: n float4]
struct McmcLayout {
  size_t block_w, block_dead, W, count, dead, vals, bytes;
};
inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }
McmcLayout mcmc_layout(int64_t N, int64_t n) {
  McmcLayout L;
  const size_t nb = (size_t)((N + SC_ROWS - 1) / SC_ROWS) + 1;
  L.block_w = 256;
  L.block_dead = up256(L.block_w + nb * 8);
  L.W = up256(L.block_dead + nb * 4);
  L.count = up256(L.W + (size_t)N * 8);
  L.dead = up256(L.count + (size_t)N * 4);
  L.vals = up256(L.dead + (size_t)N * 4);
  L.bytes = up256(L.vals + (size_t)n * 16);
  return L;
}

}  // namespace

size_t density_workspace_bytes(int64_t N) {
  // [three int64 totals, padded to 256 B][three counts per 1024-row CTA]
  return 256 + (size_t)((N + SC_ROWS - 1) / SC_ROWS + 1) * 3 * sizeof(int32_t);
}

int launch_density_accumulate(int64_t N, const float *dloss_dus, const uint8_t *mask, float *grad_accum,
                              int32_t *cunt, int init, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_DENSITY_ACC, st);
  k_density_accumulate<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, dloss_dus, mask, grad_accum, cunt, init);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// the scan of both plans once cls and the per-CTA counts are written: slots, then the three totals
// read back (the plan's one host synchronisation)
static int density_slots(int64_t N, int nb, const uint8_t *cls, int64_t *totals, int32_t *block_counts,
                         int32_t *slots, int64_t *counts_host, cudaStream_t st) {
  {
    ProfScope ps(K_DENSITY_SCAN, st);
    k_density_scan_blocks<<<1, 1024, 0, st>>>(nb, DensityBlocks{block_counts}, totals);
    k_density_slots<<<nb, SC_THREADS, 0, st>>>(N, cls, DensityBlocks{block_counts}, reinterpret_cast<Slot3 *>(slots));
    GSB_CUDA_TRY(cudaGetLastError());
  }
  GSB_CUDA_TRY(cudaMemcpyAsync(counts_host, totals, 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  GSB_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int launch_density_plan(int64_t N, const float *alphas_raw, const float *scales_raw, const float *grad_accum,
                        const int32_t *cunt, float alpha_raw_min, float scale_raw_max, float grad_min,
                        float scale_clone_max, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                        int64_t *counts_host, cudaStream_t st) {
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (N == 0) return 0;
  int64_t *totals = static_cast<int64_t *>(ws);
  int32_t *block_counts = reinterpret_cast<int32_t *>(static_cast<char *>(ws) + 256);
  const int nb = (int)((N + SC_ROWS - 1) / SC_ROWS);
  {
    ProfScope ps(K_DENSITY_CLASSIFY, st);
    k_density_classify_count<<<nb, SC_THREADS, 0, st>>>(N, alphas_raw, scales_raw, grad_accum, cunt, alpha_raw_min,
                                                       scale_raw_max, grad_min, scale_clone_max, cls, block_counts);
    GSB_CUDA_TRY(cudaGetLastError());
  }
  return density_slots(N, nb, cls, totals, block_counts, slots, counts_host, st);
}

int launch_density_plan_keep(int64_t N, const uint8_t *keep, void *ws, uint8_t *cls, int32_t *slots,
                             int64_t *counts_host, cudaStream_t st) {
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (N == 0) return 0;
  int64_t *totals = static_cast<int64_t *>(ws);
  int32_t *block_counts = reinterpret_cast<int32_t *>(static_cast<char *>(ws) + 256);
  const int nb = (int)((N + SC_ROWS - 1) / SC_ROWS);
  {
    ProfScope ps(K_DENSITY_CLASSIFY, st);
    k_density_keep_count<<<nb, SC_THREADS, 0, st>>>(N, keep, cls, block_counts);
    GSB_CUDA_TRY(cudaGetLastError());
  }
  return density_slots(N, nb, cls, totals, block_counts, slots, counts_host, st);
}

int launch_density_apply(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C,
                         float *const *src, float *const *src_m, float *const *src_v, const float *z,
                         float *const *dst, float *const *dst_m, float *const *dst_v, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_DENSITY_APPLY, st);
  int dev = 0, sms = 132;
  GSB_CUDA_TRY(cudaGetDevice(&dev));
  GSB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t blocks = (N + 32 * DG_WARPS - 1) / (32 * DG_WARPS);
  const dim3 grid((int)(blocks < (int64_t)sms * 8 ? blocks : (int64_t)sms * 8), 18);
  auto *kernel = N < 23000000 ? k_density_apply_rows<uint32_t> : k_density_apply_rows<size_t>;
  kernel<<<grid, 32 * DG_WARPS, 0, st>>>((int)N, cls, reinterpret_cast<const Slot3 *>(slots), (int)K, (int)C,
                                         jobs(src, src_m, src_v, dst, dst_m, dst_v), z);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_density_apply_rows(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int D,
                              const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                              float *dst_v, cudaStream_t st) {
  if (N == 0 || D == 0) return 0;
  ProfScope ps(K_DENSITY_ROWS, st);
  const dim3 grid(stream_grid(N * D, 256), 3);
  k_density_copy_rows<<<grid, 256, 0, st>>>(N, D, cls, reinterpret_cast<const Slot3 *>(slots), K, C, src, src_m, src_v,
                                            dst, dst_m, dst_v);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_reset_alpha(int64_t N, float *alphas_raw, float *m, float *v, float val, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_RESET_ALPHA, st);
  k_reset_alpha<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, alphas_raw, m, v, val);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_ply_rows_to_gs(int64_t N, int stride, int sh_dim, const float *rows, const int32_t *colmap, float *gs,
                          cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_GS_DECODE, st);
  const int J = 11 + sh_dim;
  k_ply_rows_to_gs<<<stream_grid(N * J, 256), 256, 0, st>>>(N, stride, J, rows, colmap, gs);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_gs_to_params(int64_t N, int sh_dim, const float *gs, float *const *dst, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_GS_TO_PARAMS, st);
  k_gs_to_params<<<stream_grid(N * 59, 256), 256, 0, st>>>(N, sh_dim, gs, dst[0], dst[1], dst[2], dst[3], dst[4],
                                                          dst[5]);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_params_to_gs(int64_t N, float *const *src, float *gs, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_PARAMS_TO_GS, st);
  k_params_to_gs<<<stream_grid(N * 59, 256), 256, 0, st>>>(N, src[0], src[1], src[2], src[3], src[4], src[5], gs);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---- MCMC densification
size_t mcmc_workspace_bytes(int64_t N, int64_t n) { return mcmc_layout(N, n).bytes; }

int launch_mcmc_plan(int64_t N, const float *alphas_raw, float alpha_raw_min, int mode, void *ws,
                     int64_t *counts_host, cudaStream_t st) {
  counts_host[0] = counts_host[1] = 0;
  if (N == 0) return 0;
  const McmcLayout L = mcmc_layout(N, 0);
  char *b = static_cast<char *>(ws);
  int64_t *totals = reinterpret_cast<int64_t *>(b);
  const McmcBlocks blocks{reinterpret_cast<uint64_t *>(b + L.block_w), reinterpret_cast<int32_t *>(b + L.block_dead)};
  const int nb = (int)((N + SC_ROWS - 1) / SC_ROWS);
  {
    ProfScope ps(K_MCMC_SCAN, st);
    k_mcmc_weight_count<<<nb, SC_THREADS, 0, st>>>(N, alphas_raw, alpha_raw_min, mode, blocks);
    k_mcmc_scan_blocks<<<1, 1024, 0, st>>>(nb, blocks, totals);
    k_mcmc_prefix<<<nb, SC_THREADS, 0, st>>>(N, alphas_raw, alpha_raw_min, mode, blocks,
                                             reinterpret_cast<uint64_t *>(b + L.W),
                                             reinterpret_cast<int32_t *>(b + L.dead),
                                             reinterpret_cast<int32_t *>(b + L.count));
    GSB_CUDA_TRY(cudaGetLastError());
  }
  GSB_CUDA_TRY(cudaMemcpyAsync(counts_host, totals, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  GSB_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int launch_mcmc_sample(int64_t N, int64_t n, const double *u, void *ws, int32_t *sampled, cudaStream_t st) {
  if (n == 0) return 0;
  const McmcLayout L = mcmc_layout(N, 0);
  char *b = static_cast<char *>(ws);
  ProfScope ps(K_MCMC_SAMPLE, st);
  k_mcmc_sample<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(N, n, u, reinterpret_cast<const uint64_t *>(b + L.W),
                                                             reinterpret_cast<const int64_t *>(b), sampled,
                                                             reinterpret_cast<int32_t *>(b + L.count));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_mcmc_values(int64_t N, int64_t n, const int32_t *sampled, void *ws, const float *alphas_raw,
                              const float *scales_raw, double min_opacity, int n_max, cudaStream_t st) {
  const McmcLayout L = mcmc_layout(N, n);
  char *b = static_cast<char *>(ws);
  k_mcmc_values<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, sampled, reinterpret_cast<const int32_t *>(b + L.count),
                                                             alphas_raw, scales_raw, min_opacity, n_max,
                                                             reinterpret_cast<float4 *>(b + L.vals));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_mcmc_relocate(int64_t N, int64_t n, const int32_t *sampled, void *ws, double min_opacity, int n_max,
                         float *const *p, float *const *m, float *const *v, cudaStream_t st) {
  if (n == 0) return 0;
  ProfScope ps(K_MCMC_RELOCATE, st);
  if (int rc = launch_mcmc_values(N, n, sampled, ws, p[3], p[4], min_opacity, n_max, st)) return rc;
  const McmcLayout L = mcmc_layout(N, n);
  char *b = static_cast<char *>(ws);
  const dim3 grid(stream_grid(n * 45, 256), 6);
  k_mcmc_relocate<<<grid, 256, 0, st>>>(n, sampled, reinterpret_cast<const int32_t *>(b + L.dead),
                                        reinterpret_cast<const float4 *>(b + L.vals), jobs(p, m, v, p, m, v));
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_mcmc_relocate_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, int D, float *x,
                              float *m, float *v, cudaStream_t st) {
  if (n == 0) return 0;
  ProfScope ps(K_MCMC_ROWS, st);
  const McmcLayout L = mcmc_layout(N, 0);
  const Job J{x, m, v, x, m, v, D};
  k_mcmc_relocate_rows<<<stream_grid(n * D, 256), 256, 0, st>>>(
      n, sampled, reinterpret_cast<const int32_t *>(static_cast<const char *>(ws) + L.dead), J);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_mcmc_grow(int64_t N, int64_t n, const int32_t *sampled, void *ws, double min_opacity, int n_max,
                     float *const *src, float *const *src_m, float *const *src_v, float *const *dst,
                     float *const *dst_m, float *const *dst_v, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_MCMC_GROW, st);
  const McmcLayout L = mcmc_layout(N, n);
  char *b = static_cast<char *>(ws);
  const Jobs J = jobs(src, src_m, src_v, dst, dst_m, dst_v);
  const dim3 grid(stream_grid((N * 45 + 3) / 4, 256), 18);
  k_mcmc_grow_copy<<<grid, 256, 0, st>>>(N, reinterpret_cast<const int32_t *>(b + L.count), J);
  GSB_CUDA_TRY(cudaGetLastError());
  if (n == 0) return 0;
  if (int rc = launch_mcmc_values(N, n, sampled, ws, src[3], src[4], min_opacity, n_max, st)) return rc;
  k_mcmc_grow_append<<<dim3(stream_grid(n * 45, 256), 6), 256, 0, st>>>(
      N, n, sampled, reinterpret_cast<const float4 *>(b + L.vals), J);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_mcmc_grow_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, int D, const float *src,
                          const float *src_m, const float *src_v, float *dst, float *dst_m, float *dst_v,
                          cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_MCMC_ROWS, st);
  const McmcLayout L = mcmc_layout(N, 0);
  const int32_t *count = reinterpret_cast<const int32_t *>(static_cast<const char *>(ws) + L.count);
  const Job J{src, src_m, src_v, dst, dst_m, dst_v, D};
  k_mcmc_grow_rows<<<dim3(stream_grid((N * D + 3) / 4, 256), 3), 256, 0, st>>>(N, n, count, sampled, J, 0);
  GSB_CUDA_TRY(cudaGetLastError());
  if (n == 0) return 0;
  k_mcmc_grow_rows<<<stream_grid(n * D, 256), 256, 0, st>>>(N, n, count, sampled, J, 1);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_mcmc_noise(int64_t N, float *pws, const float *alphas_raw, const float *scales_raw, const float *rots_raw,
                      const float *z, float scale, float k, float x0, cudaStream_t st) {
  if (N == 0) return 0;
  ProfScope ps(K_MCMC_NOISE, st);
  k_mcmc_noise<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, pws, alphas_raw, scales_raw, rots_raw, z, scale, k, x0);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
