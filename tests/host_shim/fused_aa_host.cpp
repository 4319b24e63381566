// TEST-ONLY host build of the antialiased forms of the fused per-Gaussian math
// (pg::forward_one<K3, true>, pg::backward_one<K3, true, POSE, true>,
// easygaussiansplatting_b200/csrc/pg_fused_math.h), so the CPU suite can check rho, dL/dalpha and
// the geometry and camera terms against the oracle.  Same camera set-up as fused_host.cpp.
// Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

static Cam make_cam(const float *Rcw, const float *tcw, const float *twc, float fx, float fy, float cx,
                    float cy, float width, float height) {
  Cam c;
  for (int i = 0; i < 9; i++) c.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { c.t[i] = tcw[i]; c.twc[i] = twc[i]; }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy;
  c.tan_fovx = width / (2 * fx);
  c.tan_fovy = height / (2 * fy);
  return c;
}

template <int K3>
static void fwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, float *us, float *cinv, float *cols, float *depths, int32_t *areas, float *rho) {
  for (int i = 0; i < N; i++)
    rho[i] = forward_one<K3, true>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam,
                                   us + 2 * i, cinv + 3 * i, cols + 3 * i, depths + i, areas + 2 * i);
}

template <int K3, bool POSE>
static void bwd(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                const float *galpha, const float *alphas, float *gpw, float *gsh, float *gs, float *gq,
                float *gal, float *gcam) {
  for (int i = 0; i < N; i++)
    gal[i] = backward_one<K3, true, POSE, true>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i,
                                                cam, gu + 2 * i, gci + 3 * i, gcol + 3 * i, gpw + 3 * i, gq + 4 * i,
                                                gs + 3 * i, gsh + (size_t)3 * K3 * i, gz[i],
                                                POSE ? gcam + 15 * (size_t)i : nullptr, galpha[i], alphas[i]);
}

extern "C" {

// fused_forward_host's arguments plus rho[N] (alpha_eff = rho alpha)
int fused_forward_aa_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                          const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                          float fy, float cx, float cy, float width, float height, float *us, float *cinv,
                          float *cols, float *depths, int32_t *areas, float *rho) {
  Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, width, height);
  switch (k3) {
    case 1: fwd<1>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); break;
    case 4: fwd<4>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); break;
    case 9: fwd<9>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); break;
    case 16: fwd<16>(N, pws, rots, scales, shs, cam, us, cinv, cols, depths, areas, rho); break;
    default: return -1;
  }
  return 0;
}

// fused_backward_depth_host's arguments plus galpha[N] = dL/dalpha_eff, alphas[N] (raw), outputs
// gal[N] = dL/dalpha and, when gcam is not NULL, gcam[N,15] (the POSE form)
int fused_backward_aa_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                           const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                           float fy, float cx, float cy, float width, float height, const float *gu,
                           const float *gci, const float *gcol, const float *gz, const float *galpha,
                           const float *alphas, float *gpw, float *gsh, float *gs, float *gq, float *gal,
                           float *gcam) {
  Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy, width, height);
#define GSB_AA_BWD(K)                                                                                    \
  if (gcam)                                                                                              \
    bwd<K, true>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, gq, gal, gcam); \
  else                                                                                                   \
    bwd<K, false>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, galpha, alphas, gpw, gsh, gs, gq, gal, gcam);
  switch (k3) {
    case 1: GSB_AA_BWD(1) break;
    case 4: GSB_AA_BWD(4) break;
    case 9: GSB_AA_BWD(9) break;
    case 16: GSB_AA_BWD(16) break;
    default: return -1;
  }
#undef GSB_AA_BWD
  return 0;
}
}
