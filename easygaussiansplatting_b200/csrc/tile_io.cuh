// Shared-memory staging of array-of-struct rows: coalesced float4 global traffic, odd row
// stride in shared memory so a thread can walk its own row without bank conflicts.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsb {

constexpr int PG = 128;  // Gaussians (threads) per CTA

template <int K>
struct TileT {
  static constexpr int S = (K & 1) ? K : K + 1;  // odd row stride -> conflict-free rows
  static constexpr int FLOATS = PG * S;
};

__device__ __forceinline__ bool aligned16(const void *p) {
  return (reinterpret_cast<uintptr_t>(p) & 15u) == 0;
}

__device__ __forceinline__ bool aligned8(const void *p) {
  return (reinterpret_cast<uintptr_t>(p) & 7u) == 0;
}

// Row i of a caller's [N,2] array: one 8-byte access when the array is 8-byte aligned, two
// scalar ones otherwise (a contiguous view at an odd float offset, e.g. a slice of a flat
// buffer).  The test is on the base pointer, so the branch is uniform over a launch.
__device__ __forceinline__ float2 ld_pair(const float *__restrict__ p, long long i) {
  if (aligned8(p)) return __ldg(reinterpret_cast<const float2 *>(p) + i);
  return make_float2(__ldg(p + 2 * i), __ldg(p + 2 * i + 1));
}
__device__ __forceinline__ int2 ld_pair(const int32_t *__restrict__ p, long long i) {
  if (aligned8(p)) return __ldg(reinterpret_cast<const int2 *>(p) + i);
  return make_int2(__ldg(p + 2 * i), __ldg(p + 2 * i + 1));
}
// (plain loads: for arrays a kernel also writes)
__device__ __forceinline__ int2 ld_pair_rw(const int32_t *p, long long i) {
  if (aligned8(p)) return reinterpret_cast<const int2 *>(p)[i];
  return make_int2(p[2 * i], p[2 * i + 1]);
}
__device__ __forceinline__ void st_pair(float *p, long long i, float x, float y) {
  if (aligned8(p)) {
    reinterpret_cast<float2 *>(p)[i] = make_float2(x, y);
  } else {
    p[2 * i] = x; p[2 * i + 1] = y;
  }
}
__device__ __forceinline__ void st_pair(int32_t *p, long long i, int x, int y) {
  if (aligned8(p)) {
    reinterpret_cast<int2 *>(p)[i] = make_int2(x, y);
  } else {
    p[2 * i] = x; p[2 * i + 1] = y;
  }
}

// global [rows, K] (contiguous) -> smem tile
template <int K>
__device__ __forceinline__ void tile_fetch(const float *__restrict__ g, long long base_row,
                                           int n_valid, float *sm, int tid) {
  constexpr int S = TileT<K>::S;
  const float *src = g + base_row * K;
  if (n_valid == PG && aligned16(src)) {
    const float4 *src4 = reinterpret_cast<const float4 *>(src);
#pragma unroll 4
    for (int v = tid; v < PG * K / 4; v += PG) {
      float4 x = __ldg(src4 + v);
      int e = 4 * v;
      sm[((e + 0) / K) * S + (e + 0) % K] = x.x;
      sm[((e + 1) / K) * S + (e + 1) % K] = x.y;
      sm[((e + 2) / K) * S + (e + 2) % K] = x.z;
      sm[((e + 3) / K) * S + (e + 3) % K] = x.w;
    }
  } else {
    for (int e = tid; e < n_valid * K; e += PG) sm[(e / K) * S + e % K] = __ldg(src + e);
  }
}

// smem tile -> global [rows, K]
template <int K>
__device__ __forceinline__ void tile_flush(float *__restrict__ g, long long base_row,
                                           int n_valid, const float *sm, int tid) {
  constexpr int S = TileT<K>::S;
  float *dst = g + base_row * K;
  if (n_valid == PG && aligned16(dst)) {
    float4 *dst4 = reinterpret_cast<float4 *>(dst);
#pragma unroll 4
    for (int v = tid; v < PG * K / 4; v += PG) {
      int e = 4 * v;
      float4 x;
      x.x = sm[((e + 0) / K) * S + (e + 0) % K];
      x.y = sm[((e + 1) / K) * S + (e + 1) % K];
      x.z = sm[((e + 2) / K) * S + (e + 2) % K];
      x.w = sm[((e + 3) / K) * S + (e + 3) % K];
      dst4[v] = x;
    }
  } else {
    for (int e = tid; e < n_valid * K; e += PG) dst[e] = sm[(e / K) * S + e % K];
  }
}

#define ROW(K) (sm + tid * TileT<K>::S)

}  // namespace gsb
