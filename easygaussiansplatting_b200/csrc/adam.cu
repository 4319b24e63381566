// Fused Adam step (DESIGN 3.12): one launch over every tensor of an optimizer step, dense or
// selective (visibility-masked rows).  Memory-bound: 28 bytes per updated element (read p, g, m, v;
// write p, m, v).
#include "../../include/gsplat_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace gsb {
namespace {

// One table entry.  The tensor's elements are cut into units of at most 4: for a tensor whose four
// pointers share their offset mod 16, unit 0 is the scalar head up to the first 16-byte boundary
// of p (when there is one) and every later full unit is one float4 access per array; otherwise
// every unit is scalar.  off = head - 4 (head > 0) or 0, so unit k covers [off + 4k, off + 4k + 4)
// clamped to [0, numel).
struct AdamSlot {
  float *p;
  const float *g;
  float *m;
  float *v;
  int64_t n;
  int64_t unit0;  // first unit of this tensor in the launch
  int D;
  int off;
  int vec;
  float step_size, bc2;
};
constexpr int kAdamMaxTensors = 24;  // 64-byte slots: the table stays well inside the 4 KiB of kernel parameters
struct AdamTable {
  AdamSlot t[kAdamMaxTensors];
  int count;
  int64_t units;
};
struct AdamCoef {
  float w1, w1c, b2, w2, eps;  // w1 = 1 - beta1 (fp32 of the double), w1c = 1 - w1 in fp32
  int small;                   // |w1| < 0.5: torch's lerp branch
};
static_assert(sizeof(AdamTable) <= 4000, "kernel parameter space");

// torch.optim.adam._multi_tensor_adam for one element: lerp_, mul_, addcmul_, sqrt, div_, add_,
// addcdiv_, each rounded once (torch's CUDA build contracts a + b * c into one FMA, as here).
__device__ __forceinline__ void adam_elem(float &p, float g, float &m, float &v, const AdamCoef &c, float step_size,
                                          float bc2) {
  const float d = __fsub_rn(g, m);
  m = c.small ? __fmaf_rn(c.w1, d, m) : __fmaf_rn(-d, c.w1c, g);
  v = __fmaf_rn(c.w2, __fmul_rn(g, g), __fmul_rn(v, c.b2));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2), c.eps);
  p = __fmaf_rn(-step_size, __fdiv_rn(m, denom), p);
}

// row of element e in a tensor of row width D (32-bit division where the tensor allows it)
__device__ __forceinline__ int64_t row_of(int64_t e, int D, int64_t n) {
  return n <= 0xffffffffll ? (int64_t)((uint32_t)e / (uint32_t)D) : e / D;
}

template <bool SELECTIVE>
__global__ void __launch_bounds__(256) k_adam(const __grid_constant__ AdamTable T, AdamCoef c, const uint8_t *vis) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int ti = 0;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < T.units; u += stride) {
    while (ti + 1 < T.count && u >= T.t[ti + 1].unit0) ti++;  // units grow with u: the slot index only advances
    const AdamSlot &S = T.t[ti];
    const int64_t s4 = (int64_t)S.off + 4 * (u - S.unit0);
    const int64_t s = s4 > 0 ? s4 : 0;
    const int64_t e = s4 + 4 < S.n ? s4 + 4 : S.n;
    const int cnt = (int)(e - s);
    bool on[4] = {true, true, true, true};
    bool any = true, all = true;
    if (SELECTIVE) {
      int64_t r = row_of(s, S.D, S.n);
      int col = (int)(s - r * S.D);
      any = false;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        on[i] = i < cnt && vis[r] != 0;
        any |= on[i];
        if (++col == S.D) {
          r++;
          col = 0;
        }
      }
      all = on[0] && on[1] && on[2] && on[3];
    }
    if (!any) continue;  // an invisible unit: nothing read, nothing written
    if (S.vec && s == s4 && cnt == 4) {
      float4 p = *reinterpret_cast<const float4 *>(S.p + s);
      const float4 g = *reinterpret_cast<const float4 *>(S.g + s);
      float4 m = *reinterpret_cast<const float4 *>(S.m + s);
      float4 v = *reinterpret_cast<const float4 *>(S.v + s);
      adam_elem(p.x, g.x, m.x, v.x, c, S.step_size, S.bc2);
      adam_elem(p.y, g.y, m.y, v.y, c, S.step_size, S.bc2);
      adam_elem(p.z, g.z, m.z, v.z, c, S.step_size, S.bc2);
      adam_elem(p.w, g.w, m.w, v.w, c, S.step_size, S.bc2);
      if (all) {
        *reinterpret_cast<float4 *>(S.p + s) = p;
        *reinterpret_cast<float4 *>(S.m + s) = m;
        *reinterpret_cast<float4 *>(S.v + s) = v;
      } else {  // a quad shared with invisible rows: write only the visible elements
        const float pp[4] = {p.x, p.y, p.z, p.w}, mm[4] = {m.x, m.y, m.z, m.w}, vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
          if (on[i]) {
            S.p[s + i] = pp[i];
            S.m[s + i] = mm[i];
            S.v[s + i] = vv[i];
          }
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        if (i < cnt && on[i]) {
          float p = S.p[s + i], m = S.m[s + i], v = S.v[s + i];
          adam_elem(p, S.g[s + i], m, v, c, S.step_size, S.bc2);
          S.p[s + i] = p;
          S.m[s + i] = m;
          S.v[s + i] = v;
        }
      }
    }
  }
}

int launch_table(AdamTable &T, const AdamCoef &c, const uint8_t *vis, int sms, cudaStream_t st) {
  if (T.units == 0) return 0;
  const int64_t blocks = (T.units + 255) / 256;
  const int grid = (int)(blocks < (int64_t)sms * 8 ? blocks : (int64_t)sms * 8);
  if (vis)
    k_adam<true><<<grid, 256, 0, st>>>(T, c, vis);
  else
    k_adam<false><<<grid, 256, 0, st>>>(T, c, nullptr);
  GSB_CUDA_TRY(cudaGetLastError());
  T.count = 0;
  T.units = 0;
  return 0;
}

}  // namespace

int launch_adam(int n_tensors, const gsb_adam_tensor *table, const uint8_t *visibility, double beta1, double beta2,
                double eps, cudaStream_t st) {
  AdamCoef c;
  c.w1 = (float)(1.0 - beta1);
  c.w1c = 1.0f - c.w1;
  c.small = fabsf(c.w1) < 0.5f;
  c.b2 = (float)beta2;
  c.w2 = (float)(1.0 - beta2);
  c.eps = (float)eps;
  int dev = 0, sms = 132;
  GSB_CUDA_TRY(cudaGetDevice(&dev));
  GSB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  ProfScope ps(K_ADAM, st);
  AdamTable T;
  T.count = 0;
  T.units = 0;
  for (int i = 0; i < n_tensors; i++) {
    const gsb_adam_tensor &a = table[i];
    if (a.numel == 0) continue;
    const uintptr_t q = reinterpret_cast<uintptr_t>(a.param) & 15;
    const bool vec = (reinterpret_cast<uintptr_t>(a.grad) & 15) == q && (reinterpret_cast<uintptr_t>(a.exp_avg) & 15) == q &&
                     (reinterpret_cast<uintptr_t>(a.exp_avg_sq) & 15) == q;
    const int head = vec ? (int)((16 - q) & 15) / 4 : 0;
    AdamSlot &S = T.t[T.count++];
    S.p = a.param;
    S.g = a.grad;
    S.m = a.exp_avg;
    S.v = a.exp_avg_sq;
    S.n = a.numel;
    S.unit0 = T.units;
    S.D = a.D > 0 ? a.D : 1;
    S.off = head > 0 ? head - 4 : 0;
    S.vec = vec;
    S.step_size = a.step_size;
    S.bc2 = a.bc2_sqrt;
    T.units += (a.numel - S.off + 3) / 4;
    if (T.count == kAdamMaxTensors)
      if (int rc = launch_table(T, c, visibility, sms, st)) return rc;
  }
  return launch_table(T, c, visibility, sms, st);
}

}  // namespace gsb
