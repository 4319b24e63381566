// TEST-ONLY host build of the Mip-Splatting 3D filter (pg::filter3d_sees, filter3d_value,
// filter3d_apply, filter3d_backward of easygaussiansplatting_b200/csrc/pg_fused_math.h), composed
// the way the kernels of filter3d.cu compose them, so the CPU suite can check the visibility
// decisions, the chosen depths and the apply / backward rows against the oracle.  Never part of
// the product library.
#include <math.h>
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

extern "C" {

// k_filter3d_depth: dmin[i] = the smallest z over the cameras cams[C,20] that see pws[i], 0 if none
void filter3d_depth_host(int N, const float *pws, int C, const float *cams, float *dmin) {
  for (int i = 0; i < N; i++) {
    float best = INFINITY;
    for (int k = 0; k < C; k++) {
      float z;
      if (filter3d_sees(cams + (size_t)k * kCamRow, pws + 3 * (size_t)i, z)) best = fminf(best, z);
    }
    dmin[i] = best < INFINITY ? best : 0.f;
  }
}

// k_filter3d_depth + k_filter3d_finish
void filter3d_host(int N, const float *pws, int C, const float *cams, float variance, float *filter3d) {
  filter3d_depth_host(N, pws, C, cams, filter3d);
  float dmax = 0.f, fmax = 0.f;
  for (int i = 0; i < N; i++) dmax = fmaxf(dmax, filter3d[i]);
  for (int k = 0; k < C; k++) fmax = fmaxf(fmax, cams[(size_t)k * kCamRow + 12]);  // positive fx only
  for (int i = 0; i < N; i++)
    filter3d[i] = dmax > 0.f && fmax > 0.f ? filter3d_value(filter3d[i] > 0.f ? filter3d[i] : dmax, fmax, variance) : 0.f;
}

void filter3d_apply_host(int N, const float *scales, const float *alphas, const float *filter3d, float *scales_f,
                         float *alphas_f) {
  for (int i = 0; i < N; i++) {
    float t[3];
    const float c = filter3d_apply(scales + 3 * i, filter3d[i], scales_f + 3 * i, t);
    alphas_f[i] = c * alphas[i];
  }
}

void filter3d_backward_host(int N, const float *scales, const float *alphas, const float *filter3d,
                            const float *gsf, const float *gaf, float *gs, float *ga) {
  for (int i = 0; i < N; i++)
    ga[i] = filter3d_backward(scales + 3 * i, alphas[i], filter3d[i], gsf + 3 * i, gaf[i], gs + 3 * i);
}
}
