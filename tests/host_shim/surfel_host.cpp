// TEST-ONLY host build of the 2D Gaussian Splatting math (easygaussiansplatting_b200/csrc/surfel_math.h):
// the per-surfel forward and backward, the footprint / cull box and the per-pixel evaluation and its
// gradient, exactly as the surfel kernels compute them, so the CPU suite can check them against the
// fp64 oracle (oracle/surfel_oracle.py).  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/surfel_math.h"

using namespace gsb;

static pg::Cam make_cam(const float *Rcw, const float *tcw, const float *twc, float fx, float fy, float cx, float cy) {
  pg::Cam c;
  for (int i = 0; i < 9; i++) c.R[i] = Rcw[i];
  for (int i = 0; i < 3; i++) { c.t[i] = tcw[i]; c.twc[i] = twc[i]; }
  c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy; c.tan_fovx = 0.f; c.tan_fovy = 0.f;
  for (int i = 0; i < 4; i++) c.k[i] = 0.f;
  return c;
}

template <int K3>
static void fwd(int N, const float *pws, const float *rots, const float *scales, const float *shs, const float *alphas,
                const pg::Cam &cam, float *us, float *depths, int32_t *areas, float *cols, float *recs) {
  for (int i = 0; i < N; i++) {
    int a[2];
    sf::forward_one<K3>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, alphas[i], cam, us + 2 * i,
                        depths + i, a, cols + 3 * i, recs + (size_t)sf::kRecFloats * i);
    areas[2 * i] = a[0];
    areas[2 * i + 1] = a[1];
  }
}

template <int K3>
static void bwd(int N, const float *pws, const float *rots, const float *scales, const float *shs, const pg::Cam &cam,
                const float *rows, float *gpw, float *gsh, float *gs, float *gq) {
  for (int i = 0; i < N; i++)
    sf::backward_one<K3>(pws + 3 * i, rots + 4 * i, scales + 3 * i, shs + (size_t)3 * K3 * i, cam,
                         rows + (size_t)sf::kRowFloats * i, gpw + 3 * i, gq + 4 * i, gs + 3 * i,
                         gsh + (size_t)3 * K3 * i);
}

extern "C" {

int surfel_forward(int N, int k3, const float *pws, const float *rots, const float *scales, const float *shs,
                   const float *alphas, const float *Rcw, const float *tcw, const float *twc, float fx, float fy,
                   float cx, float cy, float *us, float *depths, int32_t *areas, float *cols, float *recs) {
  const pg::Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy);
  switch (k3) {
    case 1: fwd<1>(N, pws, rots, scales, shs, alphas, cam, us, depths, areas, cols, recs); return 0;
    case 4: fwd<4>(N, pws, rots, scales, shs, alphas, cam, us, depths, areas, cols, recs); return 0;
    case 9: fwd<9>(N, pws, rots, scales, shs, alphas, cam, us, depths, areas, cols, recs); return 0;
    case 16: fwd<16>(N, pws, rots, scales, shs, alphas, cam, us, depths, areas, cols, recs); return 0;
  }
  return -1;
}

int surfel_backward(int N, int k3, const float *pws, const float *rots, const float *scales, const float *shs,
                    const float *Rcw, const float *tcw, const float *twc, float fx, float fy, float cx, float cy,
                    const float *rows, float *gpw, float *gsh, float *gs, float *gq) {
  const pg::Cam cam = make_cam(Rcw, tcw, twc, fx, fy, cx, cy);
  switch (k3) {
    case 1: bwd<1>(N, pws, rots, scales, shs, cam, rows, gpw, gsh, gs, gq); return 0;
    case 4: bwd<4>(N, pws, rots, scales, shs, cam, rows, gpw, gsh, gs, gq); return 0;
    case 9: bwd<9>(N, pws, rots, scales, shs, cam, rows, gpw, gsh, gs, gq); return 0;
    case 16: bwd<16>(N, pws, rots, scales, shs, cam, rows, gpw, gsh, gs, gq); return 0;
  }
  return -1;
}

// one pixel: out[4] = (G, z, b3, a), and the gradient of dG G + dz z into gM[9] (dL/du folded in
// through u = (m1z, m2z) / m3z by fold_du) and gd[2] = dL/ddelta
void surfel_pixel(const float *M, const float *u, float x, float y, float dG, float dz, float *out, float *gM,
                  float *gd) {
  sf::PixEval p;
  sf::pixel_eval(M, u, x, y, p);
  out[0] = p.G; out[1] = p.z; out[2] = p.b3 ? 1.f : 0.f; out[3] = p.a;
  for (int k = 0; k < 9; k++) gM[k] = 0.f;
  float gu[2] = {0.f, 0.f};
  gd[0] = gd[1] = 0.f;
  sf::pixel_grad(M, x, y, p, dG, dz, gM, gd, gu);
  sf::fold_du(M, gu, gM);
}

// the record's cull box half-extents; returns the footprint's boundedness at level lv into ext_lv
int surfel_extents(const float *M, const float *u, float alpha, float lv, float *cull, float *ext_lv) {
  sf::cull_extent(M, u, alpha, cull);
  return sf::footprint(M, u, lv, ext_lv) ? 1 : 0;
}

}  // extern "C"
