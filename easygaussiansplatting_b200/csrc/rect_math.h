// The tile rectangle of one record, the arithmetic of the binning's phase 1 (binning.cu
// k_rects_scan / k_rects_scan_batch; reference kernel.cu:105-110, DIV_ROUND_UP(X,16) on floats is
// ((X) + 16 - 1) / 16, common.cuh:15).  Every operation is explicitly rounded (the _rn intrinsics on the
// device, IEEE single operations on the host, built without contraction), so a host build computes the
// same tiles (tests/host_shim/rect_host.cpp).
#pragma once

#ifdef __CUDACC__
#define GSB_RECT_HD __host__ __device__ __forceinline__
#else
#define GSB_RECT_HD inline
#endif

namespace gsb {

GSB_RECT_HD float rect_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
GSB_RECT_HD float rect_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
GSB_RECT_HD float rect_div16(float a) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, 16.0f);
#else
  return a / 16.0f;
#endif
}
GSB_RECT_HD int rect_clamp(int v, int hi) {
#ifdef __CUDA_ARCH__
  return min(hi, max(0, v));
#else
  return v < 0 ? 0 : (v > hi ? hi : v);
#endif
}

// Tiles [x0, x1) x [y0, y1) of a record with mean (ux, uy) and half-extent (xs, ys) pixels in a frame of
// gx x gy tiles, clamped to that frame; row0: the frame's first tile row in the binned grid (0 for a
// single frame, c gy for frame c of a batch's tall frame, DESIGN 3.21), added after the clamp so that
// a record never reaches another frame's rows.
GSB_RECT_HD void tile_rect(float ux, float uy, float xs, float ys, int gx, int gy, int row0, int &x0, int &x1,
                           int &y0, int &y1) {
  x0 = rect_clamp((int)rect_div16(rect_sub(ux, xs)), gx);
  y0 = rect_clamp((int)rect_div16(rect_sub(uy, ys)), gy) + row0;
  x1 = rect_clamp((int)rect_div16(rect_sub(rect_add(rect_add(ux, xs), 16.0f), 1.0f)), gx);
  y1 = rect_clamp((int)rect_div16(rect_sub(rect_add(rect_add(uy, ys), 16.0f), 1.0f)), gy) + row0;
}

}  // namespace gsb
