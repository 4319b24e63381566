// Per-surfel math of 2D Gaussian Splatting (DESIGN 3.15), shared by the surfel kernels
// (surfel.cu) and host builds used only by tests (tests/host_shim/surfel_host.cpp) -- hence
// host+device and no CUDA-only intrinsics.  The stages of pg_fused_math.h (camera_point,
// project_mean, quat_to_R, view_dir, sh_basis) are reused as they are.
//
// A surfel is a flat Gaussian disk: centre pw, tangent axes s0 R e0 and s1 R e1 (R the rotation of
// the normalised quaternion), normal R e2.  In the camera frame
//   tu = s0 Rcw R e0,  tv = s1 Rcw R e1,  pc = Rcw pw + tcw,  n = +-Rcw R e2 (facing the camera)
//   M = K [tu | tv | pc]  (rows m1, m2, m3; m3 = (tu.z, tv.z, pc.z))
// maps the surfel-plane point (a, b, 1) to homogeneous pixel coordinates.  A pixel (x, y) meets the
// plane at (a, b) = (c0, c1) / c2 with c = (x m3 - m1) x (y m3 - m2), G3 = a^2 + b^2; the screen
// filter is G2 = 2 |p - u|^2 with u the projected centre; alpha' = min(0.99, alpha exp(-min(G3, G2)/2)).
#pragma once
#include "pg_fused_math.h"

namespace gsb {
namespace sf {

constexpr float kFilterInvSquare = 2.0f;  // G2 = 2 |p - u|^2 (2DGS's FilterInvSquare)
constexpr float kCutoff2 = 9.0f;          // binning footprint: the 3-sigma disk a^2 + b^2 <= 9
constexpr float kAreaCap = 16777216.0f;   // 2^24: the largest binning half-extent (areas), exact in fp32
constexpr int kRecFloats = 20;            // the rasterizers' 80-byte record
constexpr int kRowFloats = 18;            // the backward rasterizer's per-Gaussian gradient row

struct Surfel {
  float qn[4], qinv;  // normalised quaternion, 1 / |q|
  float R[9];         // R(qn)
  float pc[3];        // camera-frame centre
  float tu[3], tv[3]; // camera-frame tangent axes (scaled)
  float n[3];         // camera-frame unit normal, facing the camera
  float sgn;          // +1, or -1 where Rcw R e2 was flipped
  float M[9];         // K [tu | tv | pc], row-major
  float u[2];         // projected centre
  bool keep;          // pc.z >= 0.2 and the 3-sigma disk lies in front of the camera
};

// The stages of one surfel up to M and u.  keep is also cleared when the binning footprint has no
// bounded projection (footprint below).
GSB_HD void geometry(const float pw[3], const float q[4], const float s[3], const pg::Cam &cam, Surfel &g) {
  g.keep = pg::camera_point(cam.R, cam.t, pw, g.pc);
  const float qq = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  g.qinv = 1.0f / sqrtf(qq);
  for (int k = 0; k < 4; k++) g.qn[k] = q[k] * g.qinv;
  pg::quat_to_R(g.qn, g.R);
  const float *C = cam.R;
  for (int i = 0; i < 3; i++) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int a = 0; a < 3; a++) {
      a0 = fmaf(C[3 * i + a], g.R[3 * a], a0);
      a1 = fmaf(C[3 * i + a], g.R[3 * a + 1], a1);
      a2 = fmaf(C[3 * i + a], g.R[3 * a + 2], a2);
    }
    g.tu[i] = s[0] * a0;
    g.tv[i] = s[1] * a1;
    g.n[i] = a2;
  }
  const float dp = g.n[0] * g.pc[0] + g.n[1] * g.pc[1] + g.n[2] * g.pc[2];
  g.sgn = dp > 0.f ? -1.0f : 1.0f;
  for (int i = 0; i < 3; i++) g.n[i] *= g.sgn;
  const float *cols[3] = {g.tu, g.tv, g.pc};
  for (int j = 0; j < 3; j++) {
    const float *X = cols[j];
    g.M[j] = fmaf(cam.fx, X[0], cam.cx * X[2]);
    g.M[3 + j] = fmaf(cam.fy, X[1], cam.cy * X[2]);
    g.M[6 + j] = X[2];
  }
  const float z = g.keep ? g.pc[2] : 1.0f;
  pg::project_mean(g.pc, 1.0f / z, cam.fx, cam.fy, cam.cx, cam.cy, g.u);
}

// Half-extents around u of the bounding box of {a^2 + b^2 <= lv} (through M) and of the filter disk
// {2 |p - u|^2 <= lv}.  The ellipse's box comes from its dual conic M diag(1, 1, -1/lv) M^T, with
// rows 1 and 2 of M taken relative to u (M[k][j] - u_k M[2][j]):
//   D = m3z^2 - lv (m3x^2 + m3y^2)  (> 0: the disk lies in front of the camera, a bounded ellipse)
//   centre_k = (M[k][2] M[2][2] - lv (M[k][0] M[2][0] + M[k][1] M[2][1])) / D
//   half_k^2 = centre_k^2 - (M[k][2]^2 - lv (M[k][0]^2 + M[k][1]^2)) / D
// Returns false (ext untouched) when D <= 0 (or NaN).
GSB_HD bool footprint(const float M[9], const float u[2], float lv, float ext[2]) {
  const float D = M[8] * M[8] - lv * (M[6] * M[6] + M[7] * M[7]);
  if (!(D > 0.f)) return false;
  const float Di = 1.0f / D;
  const float r = sqrtf(lv / kFilterInvSquare);
  for (int k = 0; k < 2; k++) {
    // row k shifted to u (pixel coordinate p_k - u_k): centre and half^2 are then O(half), not O(u),
    // and half^2 does not cancel two terms of size u^2 (0.4 px of error at u ~ 4000 px otherwise)
    const float m[3] = {fmaf(-u[k], M[6], M[3 * k]), fmaf(-u[k], M[7], M[3 * k + 1]), fmaf(-u[k], M[8], M[3 * k + 2])};
    const float cen = (m[2] * M[8] - lv * (m[0] * M[6] + m[1] * M[7])) * Di;
    const float hh = cen * cen - (m[2] * m[2] - lv * (m[0] * m[0] + m[1] * m[1])) * Di;
    const float h = sqrtf(fmaxf(hh, 0.f));
    ext[k] = fmaxf(fmaxf(fabsf(cen + h), fabsf(cen - h)), r);
  }
  return true;
}

// Level t = 2 ln(alpha / 0.002) of the record's culling box: alpha' >= 0.002 needs min(G3, G2) <= t.
// The box (half-extents around u) is widened by 0.1 % + 0.1 px against fp32 rounding; +inf when the
// t-level ellipse is unbounded (never culled), -inf when alpha < 0.002 (never contributes).
GSB_HD void cull_extent(const float M[9], const float u[2], float alpha, float ext[2]) {
  if (!(alpha >= 0.002f)) {
    ext[0] = ext[1] = -INFINITY;
    return;
  }
  const float t = 2.0f * logf(alpha * 500.0f) + 1e-3f;
  float e[2];
  if (!footprint(M, u, t, e)) {
    ext[0] = ext[1] = INFINITY;
    return;
  }
  ext[0] = fmaf(e[0], 1.001f, 0.1f);
  ext[1] = fmaf(e[1], 1.001f, 0.1f);
}

// One pixel's evaluation of a surfel: the ray-splat point (a, b), which term wins (b3: G3 <= G2) and
// the depth of the hit, z = m3 . (a, b, 1) (pc.z where the filter wins, as in 2DGS).
struct PixEval {
  float hx[3], hy[3];
  float ci, a, b;  // 1 / c2 and the plane point (b3 only)
  float dx, dy;    // p - u
  float G, z;
  bool b3;
};
GSB_HD void pixel_eval(const float M[9], const float u[2], float x, float y, PixEval &p) {
  for (int k = 0; k < 3; k++) {
    p.hx[k] = fmaf(x, M[6 + k], -M[k]);
    p.hy[k] = fmaf(y, M[6 + k], -M[3 + k]);
  }
  const float c0 = p.hx[1] * p.hy[2] - p.hx[2] * p.hy[1];
  const float c1 = p.hx[2] * p.hy[0] - p.hx[0] * p.hy[2];
  const float c2 = p.hx[0] * p.hy[1] - p.hx[1] * p.hy[0];
  float G3 = INFINITY;
  p.ci = 0.f; p.a = 0.f; p.b = 0.f;
  if (c2 != 0.f) {
    p.ci = 1.0f / c2;
    p.a = c0 * p.ci;
    p.b = c1 * p.ci;
    G3 = p.a * p.a + p.b * p.b;
  }
  p.dx = x - u[0];
  p.dy = y - u[1];
  const float G2 = kFilterInvSquare * (p.dx * p.dx + p.dy * p.dy);
  p.b3 = G3 <= G2;
  p.G = p.b3 ? G3 : G2;
  p.z = p.b3 ? fmaf(M[6], p.a, fmaf(M[7], p.b, M[8])) : M[8];
}

// One pixel's terms of a surfel's gradient row, given dL/dG (0 where alpha' is clamped) and dL/dz:
// adds to gM[9] (through the plane point and the depth) and gd[2] = dL/ddelta, and, where the filter
// wins, to gu[2] = dL/du (the caller folds it into dL/dM through u = (m1z, m2z) / m3z).
GSB_HD void pixel_grad(const float M[9], float x, float y, const PixEval &p, float dG, float dz, float gM[9],
                       float gd[2], float gu[2]) {
  gM[8] += dz;
  if (p.b3) {
    const float da = fmaf(dG, 2.0f * p.a, dz * M[6]);
    const float db = fmaf(dG, 2.0f * p.b, dz * M[7]);
    gM[6] = fmaf(dz, p.a, gM[6]);
    gM[7] = fmaf(dz, p.b, gM[7]);
    const float g0 = da * p.ci, g1 = db * p.ci, g2 = -(da * p.a + db * p.b) * p.ci;
    // c = hx x hy:  dL/dhx = hy x gc,  dL/dhy = gc x hx
    const float *hx = p.hx, *hy = p.hy;
    const float ex[3] = {hy[1] * g2 - hy[2] * g1, hy[2] * g0 - hy[0] * g2, hy[0] * g1 - hy[1] * g0};
    const float ey[3] = {g1 * hx[2] - g2 * hx[1], g2 * hx[0] - g0 * hx[2], g0 * hx[1] - g1 * hx[0]};
    for (int k = 0; k < 3; k++) {
      gM[k] -= ex[k];
      gM[3 + k] -= ey[k];
      gM[6 + k] = fmaf(x, ex[k], fmaf(y, ey[k], gM[6 + k]));
    }
    // the whole surfel shifted by delta = evaluated at p - delta: dh/ddelta = -m3
    gd[0] -= ex[0] * M[6] + ex[1] * M[7] + ex[2] * M[8];
    gd[1] -= ey[0] * M[6] + ey[1] * M[7] + ey[2] * M[8];
  } else {
    const float k = -2.0f * kFilterInvSquare * dG;
    gd[0] = fmaf(k, p.dx, gd[0]);
    gd[1] = fmaf(k, p.dy, gd[1]);
    gu[0] = fmaf(k, p.dx, gu[0]);
    gu[1] = fmaf(k, p.dy, gu[1]);
  }
}

// dL/du folded into dL/dM: u = (m1z / m3z, m2z / m3z)
GSB_HD void fold_du(const float M[9], const float gu[2], float gM[9]) {
  const float zi = 1.0f / M[8];
  const float ux = M[2] * zi, uy = M[5] * zi;
  gM[2] = fmaf(gu[0], zi, gM[2]);
  gM[5] = fmaf(gu[1], zi, gM[5]);
  gM[8] -= (gu[0] * ux + gu[1] * uy) * zi;
}

// Forward of one surfel: u, depth (-1 when culled), areas (integer half-extents of the 3-sigma
// footprint, at most 2^24, 0 when culled), colour, and its 80-byte record
//   [M (9), alpha, u (2), cull half-extents (2), colour (3), n (3)]
template <int K3>
GSB_HD void forward_one(const float pw[3], const float q[4], const float s[3], const float *sh /*[K3][3]*/,
                        float alpha, const pg::Cam &cam, float u[2], float *depth, int area[2], float col[3],
                        float rec[kRecFloats]) {
  Surfel g;
  geometry(pw, q, s, cam, g);
  float Y[K3], dY[K3][3];
  float d[3], r[3] = {0.f, 0.f, 0.f};
  if (K3 > 1) pg::view_dir(pw, cam.twc, d, r);
  pg::sh_basis<K3>(r[0], r[1], r[2], Y, dY);
  col[0] = col[1] = col[2] = 0.5f;
  for (int l = 0; l < K3; l++)
    for (int c = 0; c < 3; c++) col[c] = fmaf(Y[l], sh[3 * l + c], col[c]);
  float ext[2] = {0.f, 0.f};
  const bool keep = g.keep && footprint(g.M, g.u, kCutoff2, ext);
  if (keep) {
    // clamped, not culled: a disk whose near edge grazes the camera plane has a finite visible part
    // however large its footprint, and a 2^24 px half-extent still covers every tile of a frame
    area[0] = ext[0] < kAreaCap ? (int)ceilf(ext[0]) : (int)kAreaCap;
    area[1] = ext[1] < kAreaCap ? (int)ceilf(ext[1]) : (int)kAreaCap;
  }
  for (int k = 0; k < kRecFloats; k++) rec[k] = 0.f;
  if (!keep) {
    u[0] = u[1] = 0.f;
    area[0] = area[1] = 0;
    *depth = -1.0f;
    rec[12] = rec[13] = -INFINITY;
    return;
  }
  u[0] = g.u[0];
  u[1] = g.u[1];
  *depth = g.pc[2];
  for (int k = 0; k < 9; k++) rec[k] = g.M[k];
  rec[9] = alpha;
  rec[10] = g.u[0];
  rec[11] = g.u[1];
  cull_extent(g.M, g.u, alpha, rec + 12);
  for (int c = 0; c < 3; c++) {
    rec[14 + c] = col[c];
    rec[17 + c] = g.n[c];
  }
}

// Backward of one surfel from its gradient row [dM (9), dalpha, dcolour (3), dn (3), ddelta (2)]:
// dL/dpw (through M and the view direction), dL/dq (through R e0, R e1, R e2 and the quaternion's
// normalisation; the normal's flip is piecewise constant), dL/ds (s2 gets 0), dL/dsh.  gsh may alias
// sh (row-private in-place update).
template <int K3>
GSB_HD void backward_one(const float pw[3], const float q[4], const float s[3], const float *sh, const pg::Cam &cam,
                         const float row[kRowFloats], float gpw[3], float gq[4], float gs[3], float *gsh) {
  const float *gcol = row + 10;
  float Y[K3], dY[K3][3];
  float d[3], ninv = 1.f, r[3] = {0.f, 0.f, 0.f};
  if (K3 > 1) ninv = pg::view_dir(pw, cam.twc, d, r);
  pg::sh_basis<K3>(r[0], r[1], r[2], Y, dY);
  float gdir[3] = {0.f, 0.f, 0.f};
  for (int l = 0; l < K3; l++) {
    const float t = gcol[0] * sh[3 * l] + gcol[1] * sh[3 * l + 1] + gcol[2] * sh[3 * l + 2];
    if (l > 0) {
      gdir[0] = fmaf(t, dY[l][0], gdir[0]);
      gdir[1] = fmaf(t, dY[l][1], gdir[1]);
      gdir[2] = fmaf(t, dY[l][2], gdir[2]);
    }
    gsh[3 * l] = gcol[0] * Y[l];
    gsh[3 * l + 1] = gcol[1] * Y[l];
    gsh[3 * l + 2] = gcol[2] * Y[l];
  }
  gpw[0] = gpw[1] = gpw[2] = 0.f;
  if (K3 > 1) {
    const float rg = r[0] * gdir[0] + r[1] * gdir[1] + r[2] * gdir[2];
    for (int a = 0; a < 3; a++) gpw[a] = (gdir[a] - r[a] * rg) * ninv;
  }
  gq[0] = gq[1] = gq[2] = gq[3] = 0.f;
  gs[0] = gs[1] = gs[2] = 0.f;
  Surfel g;
  geometry(pw, q, s, cam, g);
  float ext[2];
  if (!g.keep || !footprint(g.M, g.u, kCutoff2, ext)) return;
  // dL/d[tu | tv | pc] = K^T dL/dM, column by column
  float gX[3][3];
  for (int j = 0; j < 3; j++) {
    const float g0 = row[j], g1 = row[3 + j], g2 = row[6 + j];
    gX[j][0] = cam.fx * g0;
    gX[j][1] = cam.fy * g1;
    gX[j][2] = fmaf(cam.cx, g0, fmaf(cam.cy, g1, g2));
  }
  const float *C = cam.R;
  // pc = Rcw pw + tcw
  for (int a = 0; a < 3; a++) gpw[a] += C[a] * gX[2][0] + C[3 + a] * gX[2][1] + C[6 + a] * gX[2][2];
  // world-frame gradients of R e0, R e1, R e2: Rcw^T of the camera-frame ones
  float gw[3][3];
  const float *gcam[3] = {gX[0], gX[1], row + 13};
  const float sc[3] = {s[0], s[1], g.sgn};
  for (int j = 0; j < 3; j++)
    for (int a = 0; a < 3; a++)
      gw[j][a] = sc[j] * (C[a] * gcam[j][0] + C[3 + a] * gcam[j][1] + C[6 + a] * gcam[j][2]);
  // dL/ds_j = dL/dt_j . (Rcw R e_j) = (Rcw^T dL/dt_j) . R e_j
  for (int j = 0; j < 2; j++) {
    float v = 0.f;
    for (int a = 0; a < 3; a++)
      v = fmaf(C[a] * gX[j][0] + C[3 + a] * gX[j][1] + C[6 + a] * gX[j][2], g.R[3 * a + j], v);
    gs[j] = v;
  }
  // dL/dR (row-major): column j is gw[j]
  float dR[9];
  for (int a = 0; a < 3; a++)
    for (int j = 0; j < 3; j++) dR[3 * a + j] = gw[j][a];
  const float w = g.qn[0], x = g.qn[1], y = g.qn[2], z = g.qn[3];
  float gn[4];
  gn[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
  gn[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - w * dR[5] + z * dR[6] + w * dR[7] - 2.f * x * dR[8]);
  gn[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + w * dR[2] + x * dR[3] + z * dR[5] - w * dR[6] + z * dR[7] - 2.f * y * dR[8]);
  gn[3] = 2.f * (-2.f * z * dR[0] - w * dR[1] + x * dR[2] + w * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
  // qn = q / |q|:  dL/dq = (dL/dqn - qn (qn . dL/dqn)) / |q|
  const float dot = w * gn[0] + x * gn[1] + y * gn[2] + z * gn[3];
  for (int k = 0; k < 4; k++) gq[k] = (gn[k] - g.qn[k] * dot) * g.qinv;
}

}  // namespace sf
}  // namespace gsb
