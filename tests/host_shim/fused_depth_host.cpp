// TEST-ONLY host build of the depth term of the fused per-Gaussian backward
// (pg::backward_one<K3, true>, easygaussiansplatting_b200/csrc/pg_fused_math.h), so the CPU
// suite can check it against the oracle's chain.  Same camera set-up as fused_host.cpp.
// Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/pg_fused_math.h"

using namespace gsb::pg;

template <int K3>
static void bwd_depth(int N, const float *pws, const float *rots, const float *scales, const float *shs,
                      const Cam &cam, const float *gu, const float *gci, const float *gcol, const float *gz,
                      float *gpw, float *gsh, float *gs, float *gq) {
  for (int i = 0; i < N; i++)
    backward_one<K3, true>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam, gu + 2 * i,
                           gci + 3 * i, gcol + 3 * i, gpw + 3 * i, gq + 4 * i, gs + 3 * i, gsh + (size_t)3 * K3 * i,
                           gz[i]);
}

extern "C" {

// fused_backward_host's arguments plus gz[N] = dL/dz
int fused_backward_depth_host(int N, int k3, const float *pws, const float *rots, const float *scales,
                              const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                              float fy, float cx, float cy, float width, float height, const float *gu,
                              const float *gci, const float *gcol, const float *gz, float *gpw, float *gsh, float *gs,
                              float *gq) {
  Cam cam;
  for (int i = 0; i < 9; i++) cam.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { cam.t[i] = tcw[i]; cam.twc[i] = twc[i]; }
  cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy;
  cam.tan_fovx = width / (2 * fx);
  cam.tan_fovy = height / (2 * fy);
  switch (k3) {
    case 1: bwd_depth<1>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq); break;
    case 4: bwd_depth<4>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq); break;
    case 9: bwd_depth<9>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq); break;
    case 16: bwd_depth<16>(N, pws, rots, scales, shs, cam, gu, gci, gcol, gz, gpw, gsh, gs, gq); break;
    default: return -1;
  }
  return 0;
}
}
