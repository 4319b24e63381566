// TEST-ONLY host build of the camera-model forms of the fused per-Gaussian math
// (pg::forward_one<K3, AA, MODEL>, pg::backward_one<K3, true, POSE, AA, MODEL>,
// easygaussiansplatting_b200/csrc/pg_fused_math.h), so the CPU suite can check the ortho and
// fisheye projections, their gradients and camera terms against the oracle.  Same camera set-up as
// fused_host.cpp plus the model and k1..k4.  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

static Cam make_cam(const float *Rcw, const float *tcw, const float *twc, float fx, float fy, float cx,
                    float cy, float width, float height, const float *k) {
  Cam c;
  for (int i = 0; i < 9; i++) c.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { c.t[i] = tcw[i]; c.twc[i] = twc[i]; }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy;
  c.tan_fovx = width / (2 * fx);
  c.tan_fovy = height / (2 * fy);
  for (int i = 0; i < 4; i++) c.k[i] = k[i];
  return c;
}

template <int K3, int MODEL>
static void fwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, float *us, float *cinv, float *cols, float *depths, int32_t *areas, float *rho) {
  for (int i = 0; i < N; i++)
    rho[i] = forward_one<K3, true, MODEL>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam,
                                          us + 2 * i, cinv + 3 * i, cols + 3 * i, depths + i, areas + 2 * i);
}

template <int K3, bool POSE, bool AA, int MODEL>
static void bwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs, float *gq,
                float *gal, float *gcam) {
  for (int i = 0; i < N; i++)
    gal[i] = backward_one<K3, true, POSE, AA, MODEL>(
        pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam, gu + 2 * i, gci + 3 * i,
        gcol + 3 * i, gpw + 3 * i, gq + 4 * i, gs + 3 * i, gsh + (size_t)3 * K3 * i, gz[i],
        POSE ? gcam + 15 * (size_t)i : nullptr, galpha[i], alphas[i]);
}

template <int MODEL>
static int fwd_k3(int N, int k3, const float *pws, const float *rots, const float *scales, const float *shs,
                  const Cam &cam, float *us, float *cinv, float *cols, float *depths, int32_t *areas, float *rho) {
  switch (k3) {
    case 1: fwd<1, MODEL>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 4: fwd<4, MODEL>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 9: fwd<9, MODEL>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
    case 16: fwd<16, MODEL>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); return 0;
  }
  return -1;
}

template <int K3, int MODEL>
static void bwd_flags(bool pose, bool aa, int N, const float *pws, const float *rots, const float *scales,
                      const float *shs, const Cam &cam, const float *gu, const float *gci, const float *gcol,
                      const float *gz, const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs,
                      float *gq, float *gal, float *gcam) {
#define GSB_CM_BWD(P, A) \
  bwd<K3, P, A, MODEL>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, gq, gal, gcam)
  if (pose && aa) GSB_CM_BWD(true, true);
  else if (pose) GSB_CM_BWD(true, false);
  else if (aa) GSB_CM_BWD(false, true);
  else GSB_CM_BWD(false, false);
#undef GSB_CM_BWD
}

template <int MODEL>
static int bwd_k3(int k3, bool pose, bool aa, int N, const float *pws, const float *rots, const float *scales,
                  const float *shs, const Cam &cam, const float *gu, const float *gci, const float *gcol,
                  const float *gz, const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs,
                  float *gq, float *gal, float *gcam) {
#define GSB_CM_K3(K)                                                                                           \
  bwd_flags<K, MODEL>(pose, aa, N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, \
                      gq, gal, gcam)
  switch (k3) {
    case 1: GSB_CM_K3(1); return 0;
    case 4: GSB_CM_K3(4); return 0;
    case 9: GSB_CM_K3(9); return 0;
    case 16: GSB_CM_K3(16); return 0;
  }
#undef GSB_CM_K3
  return -1;
}

extern "C" {

// fused_forward_aa_host's arguments plus model (pg::CamModel) and k[4]; rho[N] is the AA scale
int camera_model_forward_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                              const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                              float fy, float cx, float cy, float width, float height, float *us, float *cinv,
                              float *cols, float *depths, int32_t *areas, float *rho, int model, const float *k) {
  const Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, width, height, k);
  switch (model) {
    case PINHOLE: return fwd_k3<PINHOLE>(N, k3, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho);
    case ORTHO: return fwd_k3<ORTHO>(N, k3, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho);
    case FISHEYE: return fwd_k3<FISHEYE>(N, k3, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho);
  }
  return -1;
}

// fused_backward_aa_host's arguments (DEPTH always; gcam NULL = no POSE; aa = the AA form) plus model, k[4]
int camera_model_backward_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                               const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                               float fy, float cx, float cy, float width, float height, const float *gu,
                               const float *gci, const float *gcol, const float *gz, const float *galpha,
                               const float *alphas, float *gpw, float *gsh, float *gs, float *gq, float *gal,
                               float *gcam, int aa, int model, const float *k) {
  const Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, width, height, k);
  const bool pose = gcam != nullptr;
#define GSB_CM_ARGS \
  k3, pose, aa != 0, N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, gq, gal, gcam
  switch (model) {
    case PINHOLE: return bwd_k3<PINHOLE>(GSB_CM_ARGS);
    case ORTHO: return bwd_k3<ORTHO>(GSB_CM_ARGS);
    case FISHEYE: return bwd_k3<FISHEYE>(GSB_CM_ARGS);
  }
#undef GSB_CM_ARGS
  return -1;
}
}
