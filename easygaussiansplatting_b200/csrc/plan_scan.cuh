// The plan scans' building blocks, shared by density control and MCMC (density.cu) and the TSDF
// extraction (tsdf.cu): an exclusive scan in row order, hand-written as three launches and no
// library scan -- a row kernel leaves per-CTA counters, one CTA of scan_blocks turns them into
// exclusive offsets and totals, and a row kernel rescans its CTA's rows with cta_exclusive_scan.
// T is any counter tuple with +, -, a zero T{}, and shfl_up(T, int) / warp_sum(T) found by
// argument-dependent lookup next to the type.
#pragma once
#include <stdint.h>

namespace gsb {

// the sum of x over the CTA of NT threads, valid in thread 0; warp_tot: NT / 32 entries
template <int NT, class T>
__device__ __forceinline__ T cta_sum(T x, T *warp_tot) {
  x = warp_sum(x);
  if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = x;
  __syncthreads();
  T s = warp_tot[0];
#pragma unroll
  for (int w = 1; w < NT / 32; w++) s = s + warp_tot[w];
  return s;
}

// the sum of x over the CTA's threads before this one (thread order) and, in `total`, over all of
// them; warp_tot: NT / 32 entries, which the caller may rewrite only after a __syncthreads
template <int NT, class T>
__device__ __forceinline__ T cta_exclusive_scan(T x, T *warp_tot, T &total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = shfl_up(inc, o);
    if (lane >= o) inc = inc + y;
  }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  T before = inc - x;
  total = T{};
#pragma unroll
  for (int w = 0; w < NT / 32; w++) {
    if (w < wid) before = before + warp_tot[w];
    total = total + warp_tot[w];
  }
  return before;
}

// The body of the block-scan kernels (one CTA of 1024 threads), in place: the counters of CTA b ->
// the counters of the CTAs before b; the totals = their sums.  The CTA walks the counters 1024
// CTAs at a time, carrying the sum from pass to pass.
template <class Blocks>
__device__ __forceinline__ void scan_blocks(int nb, Blocks B, int64_t *__restrict__ totals) {
  using T = typename Blocks::T;
  __shared__ T warp_tot[32];
  T carry{};
  for (int base = 0; base < nb; base += 1024) {
    const int b = base + threadIdx.x;
    const T v = b < nb ? B.load(b) : T{};
    T pass;
    const T before = cta_exclusive_scan<1024>(v, warp_tot, pass);
    if (b < nb) B.store(b, carry + before);
    carry = carry + pass;
    __syncthreads();  // warp_tot is rewritten by the next pass
  }
  if (threadIdx.x == 0) B.totals(totals, carry);
}

}  // namespace gsb
