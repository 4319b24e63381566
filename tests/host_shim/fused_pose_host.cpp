// TEST-ONLY host build of the camera-gradient form of the fused per-Gaussian backward
// (pg::backward_one<K3, true, true>, easygaussiansplatting_b200/csrc/pg_fused_math.h), so the
// CPU suite can check each Gaussian's contribution against the oracle.  Same camera set-up as
// fused_host.cpp.  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

template <int K3>
static void bwd_pose(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                     const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                     float *gpw, float *gsh, float *gs, float *gq, float *gcam) {
  for (int i = 0; i < N; i++)
    backward_one<K3, true, true>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam,
                                 gu + 2 * i, gci + 3 * i, gcol + 3 * i, gpw + 3 * i, gq + 4 * i, gs + 3 * i,
                                 gsh + (size_t)3 * K3 * i, gz[i], gcam + 15 * (size_t)i);
}

extern "C" {

// fused_backward_depth_host's arguments plus gcam[N,15]: each Gaussian's dL/dRcw (9), dL/dtcw (3),
// dL/dtwc (3)
int fused_backward_pose_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                             const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                             float fy, float cx, float cy, float width, float height, const float *gu,
                             const float *gci, const float *gcol, const float *gz, float *gpw, float *gsh, float *gs,
                             float *gq, float *gcam) {
  Cam cam;
  for (int i = 0; i < 9; i++) cam.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { cam.t[i] = tcw[i]; cam.twc[i] = twc[i]; }
  cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy;
  cam.tan_fovx = width / (2 * fx);
  cam.tan_fovy = height / (2 * fy);
  switch (k3) {
    case 1: bwd_pose<1>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq, gcam); break;
    case 4: bwd_pose<4>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq, gcam); break;
    case 9: bwd_pose<9>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq, gcam); break;
    case 16: bwd_pose<16>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq, gcam); break;
    default: return -1;
  }
  return 0;
}
}
