// TEST-ONLY host build of the fused backward's intrinsics mode (pg::backward_one<K3, true, true, AA, MODEL,
// true>, easygaussiansplatting_b200/csrc/pg_fused_math.h, DESIGN 3.23), so the CPU suite can check the
// 23 camera terms of every camera model against the fp64 oracle.  The clamp's tan_fovx, tan_fovy are
// given directly (the library derives them from the frame and the lens).  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

template <int K3, bool AA, int MODEL>
static void bwd(int N, const float *pws, const float *rots, const float *scales, const float *shs, const Cam &cam,
                const float *gu, const float *gci, const float *gcol, const float *gz, const float *galpha,
                const float *alphas, float *gcam) {
  for (int i = 0; i < N; i++) {
    float gpw[3], gq[4], gs[3], gsh[3 * K3];
    backward_one<K3, true, true, AA, MODEL, true>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i,
                                                  cam, gu + 2 * i, gci + 3 * i, gcol + 3 * i, gpw, gq, gs, gsh, gz[i],
                                                  gcam + 23 * (size_t)i, galpha[i], alphas[i]);
  }
}

template <int K3, int MODEL>
static void bwd_aa(bool aa, int N, const float *pws, const float *rots, const float *scales, const float *shs,
                   const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                   const float *galpha, const float *alphas, float *gcam) {
  if (aa)
    bwd<K3, true, MODEL>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gcam);
  else
    bwd<K3, false, MODEL>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gcam);
}

template <int K3>
static int bwd_model(int model, bool aa, int N, const float *pws, const float *rots, const float *scales,
                     const float *shs, const Cam &cam, const float *gu, const float *gci, const float *gcol,
                     const float *gz, const float *galpha, const float *alphas, float *gcam) {
#define GSB_IN_MODEL(M) bwd_aa<K3, M>(aa, N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gcam)
  switch (model) {
    case PINHOLE: GSB_IN_MODEL(PINHOLE); return 0;
    case ORTHO: GSB_IN_MODEL(ORTHO); return 0;
    case FISHEYE: GSB_IN_MODEL(FISHEYE); return 0;
    case OPENCV: GSB_IN_MODEL(OPENCV); return 0;
  }
#undef GSB_IN_MODEL
  return -1;
}

extern "C" {

// gcam[N, 23]: each Gaussian's dL/dRcw (9), dL/dtcw (3), dL/dtwc (3), dL/d(fx, fy, cx, cy, k[4]) with
// DEPTH (gz) and, when aa != 0, antialiasing (galpha = dL/dalpha_eff, alphas raw)
int intrinsics_backward_host(int N, int k3, int model, int aa, const float *pws, const float *rots,
                             const float *scales, const float *shs, const float *Rcw, const float *tcw,
                             const float *twc, float fx, float fy, float cx, float cy, float tan_fovx,
                             float tan_fovy, const float *k, const float *gu, const float *gci, const float *gcol,
                             const float *gz, const float *galpha, const float *alphas, float *gcam) {
  Cam cam;
  for (int i = 0; i < 9; i++) cam.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { cam.t[i] = tcw[i]; cam.twc[i] = twc[i]; }
  cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy;
  cam.tan_fovx = tan_fovx; cam.tan_fovy = tan_fovy;
  for (int i = 0; i < 4; i++) cam.k[i] = k[i];
#define GSB_IN_K3(K) bwd_model<K>(model, aa != 0, N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gcam)
  switch (k3) {
    case 1: return GSB_IN_K3(1);
    case 4: return GSB_IN_K3(4);
    case 9: return GSB_IN_K3(9);
    case 16: return GSB_IN_K3(16);
  }
#undef GSB_IN_K3
  return -1;
}
}
