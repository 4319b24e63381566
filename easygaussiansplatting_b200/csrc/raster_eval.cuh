// alpha' of one record at a lane's two pixels, the one operation sequence every rasterizer replays
// (raster_fwd.cu, raster_bwd.cu, raster_feat.cu): a forward and a backward that evaluate it the
// same way take identical skip decisions, and a feature replay composites with the image's weights.
#pragma once
#include "common.cuh"

namespace gsb {

// alpha' = min(0.99, alpha * exp2(a dx^2 + b dx dy + c dy^2)) at the lane's two pixels
// (kernel.cu:236-245; same operation sequence as bwd_eval below)
__device__ __forceinline__ float2 fwd_alpha(const float4 &q0, const float4 &q1, const float2 &npx, float fpy) {
  const float2 dx = add2_rn(p2s(q0.x), npx);
  const float dy = q0.y - fpy;
  const float cdy2 = (q1.z * dy) * dy;
  const float2 t = fma2_rn(p2s(q1.y), p2s(dy), mul2_rn(p2s(q1.x), dx));
  const float2 p = fma2_rn(t, dx, p2s(cdy2));
  const float2 ag = mul2_rn(p2s(q0.w), p2(ex2_approx(fminf(p.x, 0.0f)), ex2_approx(fminf(p.y, 0.0f))));
  return p2(fminf(ALPHA_CLAMP, ag.x), fminf(ALPHA_CLAMP, ag.y));
}

// alpha' of one record at the lane's pixel pair, with the skip decisions of kernel.cu:909-913.
// e = alpha' where the pixel replays the record (patch index idx < the pixel's contrib), else 0.
// An inactive pixel needs no further predication: 1 - 0 = 1 and rcp.approx.ftz(1) = 1 exactly
// (benchmarks/micro/rcp_check.cu, on the H100), so tau stays bit-identical, and both weights are
// (finite) * 0 = 0.
struct BwdEval {
  float2 dx, gg, e, rc;  // rc = 1 / (1 - e)
  float dy;
};
__device__ __forceinline__ BwdEval bwd_eval(const float4 &q0, const float4 &q1, const float2 &npx, float fpy, int idx,
                                            int cont0, int cont1) {
  BwdEval r;
  r.dx = add2_rn(p2s(q0.x), npx);
  r.dy = q0.y - fpy;
  const float cdy2 = (q1.z * r.dy) * r.dy;
  const float2 t = fma2_rn(p2s(q1.y), p2s(r.dy), mul2_rn(p2s(q1.x), r.dx));
  const float2 p = fma2_rn(t, r.dx, p2s(cdy2));
  r.gg = p2(ex2_approx(fminf(p.x, 0.0f)), ex2_approx(fminf(p.y, 0.0f)));
  const float2 ag = mul2_rn(p2s(q0.w), r.gg);
  const float ap0 = fminf(ALPHA_CLAMP, ag.x), ap1 = fminf(ALPHA_CLAMP, ag.y);
  r.e = p2(((idx < cont0) && (ap0 >= ALPHA_SKIP)) ? ap0 : 0.0f, ((idx < cont1) && (ap1 >= ALPHA_SKIP)) ? ap1 : 0.0f);
  const float2 om = add2_rn(p2s(1.0f), p2(-r.e.x, -r.e.y));
  r.rc = p2(rcp_approx(om.x), rcp_approx(om.y));
  return r;
}

}  // namespace gsb
