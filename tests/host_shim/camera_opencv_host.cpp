// TEST-ONLY host build of the OPENCV forms of the fused per-Gaussian math
// (pg::forward_one<K3, true, OPENCV>, pg::backward_one<K3, true, POSE, AA, OPENCV>,
// easygaussiansplatting_b200/csrc/pg_fused_math.h), so the CPU suite can check the radial-tangential
// projection, its gradients and camera terms against the oracle.  The camera is camera_model_host.cpp's,
// with the clamp's tan_fovx, tan_fovy given directly (the library derives them from the frame and
// the lens).  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

static Cam make_cam(const float *Rcw, const float *tcw, const float *twc, float fx, float fy, float cx,
                    float cy, float tan_fovx, float tan_fovy, const float *k) {
  Cam c;
  for (int i = 0; i < 9; i++) c.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { c.t[i] = tcw[i]; c.twc[i] = twc[i]; }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy;
  c.tan_fovx = tan_fovx;
  c.tan_fovy = tan_fovy;
  for (int i = 0; i < 4; i++) c.k[i] = k[i];
  return c;
}

template <int K3>
static void fwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, float *us, float *cinv, float *cols, float *depths, int32_t *areas, float *rho) {
  for (int i = 0; i < N; i++)
    rho[i] = forward_one<K3, true, OPENCV>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam,
                                           us + 2 * i, cinv + 3 * i, cols + 3 * i, depths + i, areas + 2 * i);
}

template <int K3, bool POSE, bool AA>
static void bwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs, float *gq,
                float *gal, float *gcam) {
  for (int i = 0; i < N; i++)
    gal[i] = backward_one<K3, true, POSE, AA, OPENCV>(
        pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam, gu + 2 * i, gci + 3 * i,
        gcol + 3 * i, gpw + 3 * i, gq + 4 * i, gs + 3 * i, gsh + (size_t)3 * K3 * i, gz[i],
        POSE ? gcam + 15 * (size_t)i : nullptr, galpha[i], alphas[i]);
}

template <int K3>
static void bwd_flags(bool pose, bool aa, int N, const float *pws, const float *rots, const float *scales,
                      const float *shs, const Cam &cam, const float *gu, const float *gci, const float *gcol,
                      const float *gz, const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs,
                      float *gq, float *gal, float *gcam) {
#define GSB_CV_BWD(P, A) \
  bwd<K3, P, A>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, gq, gal, gcam)
  if (pose && aa) GSB_CV_BWD(true, true);
  else if (pose) GSB_CV_BWD(true, false);
  else if (aa) GSB_CV_BWD(false, true);
  else GSB_CV_BWD(false, false);
#undef GSB_CV_BWD
}

extern "C" {

// camera_model_forward_host's arguments with tan_fovx, tan_fovy for width, height and no model;
// k = (k1, k2, p1, p2); rho[N] is the AA scale
int camera_opencv_forward_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                               const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                               float fy, float cx, float cy, float tan_fovx, float tan_fovy, float *us, float *cinv,
                               float *cols, float *depths, int32_t *areas, float *rho, const float *k) {
  const Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, tan_fovx, tan_fovy, k);
  switch (k3) {
    case 1: fwd<1>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 4: fwd<4>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 9: fwd<9>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 16: fwd<16>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
  }
  return -1;
}

// camera_model_backward_host's arguments likewise (DEPTH always; gcam NULL = no POSE; aa = the AA form)
int camera_opencv_backward_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                                const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                float fy, float cx, float cy, float tan_fovx, float tan_fovy, const float *gu,
                                const float *gci, const float *gcol, const float *gz, const float *galpha,
                                const float *alphas, float *gpw, float *gsh, float *gs, float *gq, float *gal,
                                float *gcam, int aa, const float *k) {
  const Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, tan_fovx, tan_fovy, k);
  const bool pose = gcam != nullptr;
#define GSB_CV_K3(K)                                                                                        \
  bwd_flags<K>(pose, aa != 0, N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, \
               gq, gal, gcam)
  switch (k3) {
    case 1: GSB_CV_K3(1); return 0;
    case 4: GSB_CV_K3(4); return 0;
    case 9: GSB_CV_K3(9); return 0;
    case 16: GSB_CV_K3(16); return 0;
  }
#undef GSB_CV_K3
  return -1;
}
}
