// Shared device helpers for the sm_90a kernels: constants fixed by the reference, fast math,
// the rasterizers' record format and their shared-memory / cp.async PTX wrappers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "pg_fused_math.h"

namespace gsb {

constexpr int TILE = 16;              // reference common.cuh:13
constexpr float MIN_DEPTH = pg::kMinDepth;
constexpr float BAD_MARKER = -1.0f;   // kernel.cu:11
constexpr float ALPHA_CLAMP = 0.99f;  // kernel.cu:245
constexpr float ALPHA_SKIP = 0.002f;  // kernel.cu:246
constexpr float TAU_STOP = 0.0001f;   // kernel.cu:256
constexpr float LOG2E = 1.4426950408889634f;

// Packed record, 48 B, one per Gaussian and indexed by Gaussian id (build_record below): the
// rasterizers gather a tile's records through its sorted id list, three 16-byte cp.async each.
//   q0 = (ux, uy, gsid bits, alpha)   mean in pixels, Gaussian id, opacity -- exactly the four
//                              words the backward's moment phase needs per record (one 16-byte copy)
//   q1 = (a, b, c, thr)        log2(g) = a dx^2 + b dx dy + c dy^2  (conic pre-scaled by
//                              -0.5*log2e, -log2e, -0.5*log2e); thr = log2(alpha / 0.002) (+margin):
//                              a pixel can reach alpha' >= 0.002 only where -log2(g) <= thr
//                              (+inf: never cull, -inf: never contributes)
//   q2 = (r, g, b, z)          colour; camera-frame depth (the `depths` value), read only by the
//                              RGB-D rasterizers (k_draw_rgbd, k_draw_bwd_rgbd)
struct __align__(16) Rec {
  float4 q0, q1, q2;
};
static_assert(sizeof(Rec) == 48, "record must be 48 bytes");

// GSB_EXACT_MATH=1 (variant builds only, benchmarks/compare_ref_gpu.py --three-way): IEEE reciprocal
// and an exp2 evaluated in double precision instead of the MUFU approximations, to show how much
// of the distance to the fp64 oracle comes from them (CUDA's own exp2f is MUFU.EX2 plus range
// scaling, i.e. the same 2-ulp function).
#ifndef GSB_EXACT_MATH
#define GSB_EXACT_MATH 0
#endif
__device__ __forceinline__ float rcp_approx(float x) {
#if GSB_EXACT_MATH
  return __frcp_rn(x);
#else
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
#endif
}
__device__ __forceinline__ float ex2_approx(float x) {
#if GSB_EXACT_MATH
  return (float)exp2((double)x);
#else
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
#endif
}

// fp32 pair arithmetic: the rasterizers and the loss carry two pixels (or two channels) per lane
// as a float2.  Hopper has no packed fp32 instruction, so each pair op is two scalar FFMA / FMUL
// / FADD; the _rn intrinsics keep nvcc from contracting or reassociating them, so every lane
// rounds exactly once per op.
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}

// Can this record reach alpha' >= 0.002 anywhere in the pixel rectangle [bx0,bx1] x [by0,by1]?
// Exact minimum of the (positive definite) quadratic Q = -log2(g) over the continuous
// rectangle: 0 if the mean lies inside, otherwise the smallest of the four edge minima (each a
// clamped 1-D parabola).  Conservative by construction (continuous rectangle >= pixel centres)
// plus an fp32 error allowance proportional to the largest term magnitude, so a record is only
// dropped when every pixel of the rectangle would take the reference's `continue`
// (kernel.cu:246) -- image, contrib and final_tau are unaffected.
__device__ __forceinline__ bool rec_can_touch(const float4 &q0, const float4 &q1, float bx0, float bx1,
                                              float by0, float by1) {
  const float A = -q1.x, B = -q1.y, C = -q1.z;
  const float dxl = q0.x - bx1, dxh = q0.x - bx0, dyl = q0.y - by1, dyh = q0.y - by0;
  const bool inside = (dxl <= 0.f) && (dxh >= 0.f) && (dyl <= 0.f) && (dyh >= 0.f);
  const float kx = __fdividef(-0.5f * B, C), ky = __fdividef(-0.5f * B, A);
  float qmin = 3.0e38f;
#pragma unroll
  for (int e = 0; e < 2; e++) {
    const float ex = e ? dxh : dxl;
    const float dy = fminf(fmaxf(kx * ex, dyl), dyh);
    qmin = fminf(qmin, fmaf(fmaf(B, ex, C * dy), dy, A * ex * ex));
    const float ey = e ? dyh : dyl;
    const float dx = fminf(fmaxf(ky * ey, dxl), dxh);
    qmin = fminf(qmin, fmaf(fmaf(B, ey, A * dx), dx, C * ey * ey));
  }
  if (inside) qmin = 0.f;
  const float X = fmaxf(fabsf(dxl), fabsf(dxh)), Y = fmaxf(fabsf(dyl), fabsf(dyh));
  const float S = fmaf(A * X, X, fmaf(fabsf(B) * X, Y, C * Y * Y));
  return !(qmin > q1.w + fmaf(2.0e-6f, S, 1.0e-5f));  // NaN anywhere keeps the record
}

// The 48-byte record the rasterizers work from (one per Gaussian).
// thr = log2(alpha / 0.002): -log2(g) <= thr is necessary for alpha' >= 0.002 -- the bound of the
// warp-level culling test (rec_can_touch); the positive-definiteness check carries a safety
// factor against fp32 cancellation in A C - B^2.
__device__ __forceinline__ Rec build_record(float ux, float uy, float A, float B, float C, float al, float cr,
                                            float cg, float cb, float z, int id) {
  float thr = INFINITY;  // never cull unless the conic is a proper positive definite form
  if (al < ALPHA_SKIP) {
    thr = -INFINITY;  // alpha * g < 0.002 everywhere: never contributes
  } else {
    const float ac = A * C;
    const float det = fmaf(A, C, -B * B);
    if (A > 0.f && C > 0.f && det > 1e-4f * ac && ac < 3.0e38f) {
      const float t = __log2f(al * 500.0f) + 1e-4f;  // log2(alpha / 0.002), lg2.approx error << margin
      if (t < 3.0e38f) thr = t;
    }
  }
  Rec r;
  r.q0 = make_float4(ux, uy, __int_as_float(id), al);
  r.q1 = make_float4(-0.5f * LOG2E * A, -LOG2E * B, -0.5f * LOG2E * C, thr);
  r.q2 = make_float4(cr, cg, cb, z);
  return r;
}

// ---- system-scope flags for the multi-GPU gradient exchange (peer memory over NVLink)
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- the rasterizers' shared-memory accesses and record gather (raster_fwd.cu, raster_bwd.cu).
// Shared memory is addressed by 32-bit shared-window addresses; a record is gathered with three
// 16-byte cp.async (SASS LDGSTS), tracked per lane by cp.async groups.
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t opaque_u32(uint32_t x) {  // keep an address in a register
  uint32_t y;
  asm volatile("mov.u32 %0, %1;" : "=r"(y) : "r"(x));
  return y;
}
__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint2 lds64u(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ uint4 lds128u(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts64u(uint32_t a, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void cp_async16_sa(uint32_t dst, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ float2 p2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 p2s(float a) { return make_float2(a, a); }

}  // namespace gsb

#define GSB_CUDA_TRY(expr)                                 \
  do {                                                     \
    cudaError_t _e = (expr);                               \
    if (_e != cudaSuccess) return gsb::set_cuda_error(_e, #expr, __FILE__, __LINE__); \
  } while (0)

namespace gsb {
int set_cuda_error(cudaError_t e, const char *what, const char *file, int line);
int set_arg_error(const char *msg);
}  // namespace gsb
