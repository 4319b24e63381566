// Per-Gaussian math, shared by the operator kernels (pergaussian.cu), the fused kernels
// (fused.cu) and host builds used only by tests (tests/host_shim/) -- hence
// host+device, no CUDA-only intrinsics.  Each formula is stated once, as a stage function
// (camera_point, project_mean, cov3d, cov2d, conic, radius, view_dir, sh_basis); the operator
// kernels call the stages one by one and add their Jacobians, the fused path composes them:
//
// forward : (pw, q, s, sh) -> u, conic, colour, depth, radius   == project + computeCov3D +
//           computeCov2D + sh2Color + inverseCov2D of the reference (kernel.cu:274-807) without
//           materialising their Jacobians;
// backward: vector-Jacobian products of the same five stages (docs/backward.md B.1-B.5.3,
//           gsmodel.py:72-85) taken analytically in registers:
//             dL/dcov2d = dL/dconic . dconic/dcov2d
//             G = sym(dL/dcov2d);  dL/dSigma = M^T G M (x2 off-diagonal);  dL/dM = 2 G M Sigma
//             dL/dJ = dL/dM Rcw^T -> dL/dpc through J(x_clamped, y_clamped, z)   (reference
//             quirk kept: derivatives taken as if x,y were unclamped, kernel.cu:527-534)
//             dL/dM3 = 2 sym(dL/dSigma) M3;  dL/ds_j = sum_i R_ij dL/dM3_ij;
//             dL/dq_p = sum_ij dR_ij/dq_p s_j dL/dM3_ij
//             dL/dsh_lc = dL/dcolour_c Y_l;  dL/dpw += (I - r r^T)/|d| sum_l dY_l (dL/dcolour . sh_l)
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define GSB_HD __host__ __device__ __forceinline__
#else
#define GSB_HD inline
#endif

namespace gsb {
namespace pg {

// Camera models (DESIGN 3.14, 3.19).  PINHOLE is the reference's projection; ORTHO, FISHEYE
// (Kannala-Brandt, COLMAP's OPENCV_FISHEYE) and OPENCV (radial-tangential, COLMAP's OPENCV) only
// change the mean u and the Jacobian J of the EWA splat -- everything after cov2d is
// model-independent.  3 is unassigned (the C ABI's GSB_CAMERA_* keep it unknown).
enum CamModel : int { PINHOLE = 0, ORTHO = 1, FISHEYE = 2, OPENCV = 4 };

struct Cam {
  float R[9], t[3], twc[3];
  float fx, fy, cx, cy, tan_fovx, tan_fovy;
  float k[4];  // FISHEYE: theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8)
               // OPENCV: k1, k2, p1, p2 (opencv_delta)
};

constexpr float kMinDepth = 0.2f;  // kernel.cu:10: (float)z < 0.2 (double)  <=>  z < 0.2f
constexpr float kBlur = 0.3f;      // the low-pass filter the reference adds to every cov2d

// camera transform pc = Rcw pw + tcw; false when the Gaussian is nearer than kMinDepth (culled)
GSB_HD bool camera_point(const float R[9], const float t[3], const float pw[3], float pc[3]) {
  pc[0] = fmaf(R[0], pw[0], fmaf(R[1], pw[1], fmaf(R[2], pw[2], t[0])));
  pc[1] = fmaf(R[3], pw[0], fmaf(R[4], pw[1], fmaf(R[5], pw[2], t[1])));
  pc[2] = fmaf(R[6], pw[0], fmaf(R[7], pw[1], fmaf(R[8], pw[2], t[2])));
  return !(pc[2] < kMinDepth);
}

// projected mean u = (fx x/z + cx, fy y/z + cy) of a kept Gaussian; zi = 1/z
GSB_HD void project_mean(const float pc[3], float zi, float fx, float fy, float cx, float cy, float u[2]) {
  u[0] = fmaf(pc[0] * fx, zi, cx);
  u[1] = fmaf(pc[1] * fy, zi, cy);
}

GSB_HD void quat_to_R(const float q[4], float R[9]) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - z * w);       R[2] = 2.f * (x * z + y * w);
  R[3] = 2.f * (x * y + z * w);       R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - x * w);
  R[6] = 2.f * (x * z - y * w);       R[7] = 2.f * (y * z + x * w);       R[8] = 1.f - 2.f * (x * x + y * y);
}

// cov3d: R3 = R(q), M3 = R3 diag(s), S6 = upper triangle of Sigma = M3 M3^T
GSB_HD void cov3d(const float q[4], const float s[3], float R3[9], float M3[9], float S6[6]) {
  quat_to_R(q, R3);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) M3[3 * r + c] = R3[3 * r + c] * s[c];
  int n = 0;
  for (int r = 0; r < 3; r++)
    for (int c = r; c < 3; c++)
      S6[n++] = M3[3 * r] * M3[3 * c] + M3[3 * r + 1] * M3[3 * c + 1] + M3[3 * r + 2] * M3[3 * c + 2];
}

// cov2d = M Sigma M^T + 0.3 I with M = J Rcw.  A culled Gaussian (keep false) is evaluated at
// pc = (0, 0, 1) so that nothing divides by its depth.
struct Cov2d {
  float xc, yc;  // x, y after the 1.3*tan_fov clamp (kernel.cu:458-461)
  float zi;      // 1/z
  float M[6];    // J Rcw (2x3)
  float MS[6];   // M Sigma
  float c2[3];   // cov2d (a, b, c) with the +0.3 blur
  float raw[2];  // its diagonal (a, c) before the blur (antialiasing only; dead code otherwise)
};

GSB_HD void cov2d(const float pc[3], bool keep, const float S6[6], const float R[9], float fx, float fy,
                  float tan_fovx, float tan_fovy, Cov2d &o) {
  const float z = keep ? pc[2] : 1.0f;
  o.zi = 1.0f / z;
  const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
  const float px = keep ? pc[0] : 0.f, py = keep ? pc[1] : 0.f;
  o.xc = fminf(limx, fmaxf(-limx, px / z)) * z;
  o.yc = fminf(limy, fmaxf(-limy, py / z)) * z;
  const float zi2 = o.zi * o.zi;
  const float J00 = fx * o.zi, J11 = fy * o.zi;
  const float J02 = -(fx * o.xc) * zi2, J12 = -(fy * o.yc) * zi2;
  for (int c = 0; c < 3; c++) {
    o.M[c] = fmaf(J00, R[c], J02 * R[6 + c]);
    o.M[3 + c] = fmaf(J11, R[3 + c], J12 * R[6 + c]);
  }
  const float S[9] = {S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5]};
  for (int a = 0; a < 2; a++)
    for (int c = 0; c < 3; c++)
      o.MS[3 * a + c] = o.M[3 * a] * S[c] + o.M[3 * a + 1] * S[3 + c] + o.M[3 * a + 2] * S[6 + c];
  o.c2[0] = o.MS[0] * o.M[0] + o.MS[1] * o.M[1] + o.MS[2] * o.M[2] + kBlur;
  o.c2[1] = o.MS[0] * o.M[3] + o.MS[1] * o.M[4] + o.MS[2] * o.M[5];
  o.c2[2] = o.MS[3] * o.M[3] + o.MS[4] * o.M[4] + o.MS[5] * o.M[5] + kBlur;
  // the same sums without the blur, after c2 so that code which never reads them compiles as before
  o.raw[0] = o.MS[0] * o.M[0] + o.MS[1] * o.M[1] + o.MS[2] * o.M[2];
  o.raw[1] = o.MS[3] * o.M[3] + o.MS[4] * o.M[4] + o.MS[5] * o.M[5];
}

// ---- ORTHO and FISHEYE.  Lens holds the projection of pc and what its derivatives need:
//   ORTHO   u = (fx x + cx, fy y + cy),  J = [[fx, 0, 0], [0, fy, 0]]
//   FISHEYE r = |(x, y)|, theta = atan2(r, z), theta_d = theta P(theta^2), s = theta_d / r,
//           u = (fx s x + cx, fy s y + cy),  g = (1/r) ds/dr,  h = -ds/dz = theta_d' / (r^2 + z^2),
//           J = [[fx (s + x^2 g), fx x y g, -fx x h], [fy x y g, fy (s + y^2 g), -fy y h]]
//   and for the backward's dJ/dpc: G = (1/r) dg/dr, H = (1/r) dh/dr (= -dg/dz), hz = dh/dz.
// s, g and G cancel to nothing as t = r/z -> 0 (0/0 on the axis): below kFishSeries they come
// from their series in t^2,  s = (1 + a1 t^2 + a2 t^4) / z, g = (2 a1 + 4 a2 t^2) / z^3,
// G = 8 a2 / z^5  with a1 = k1 - 1/3, a2 = 1/5 - k1 + k2.  The direct forms lose ~eps/t of dJ/dpc
// and the truncated series ~t^4 (relative), which meet near t = 0.03.
constexpr float kFishSeries = 0.03f;

struct Lens {
  float J[6];           // du/dpc (2x3, row-major); OPENCV: the clamped J of cov2d
  float s, g, h;        // FISHEYE
  float G, H, hz;       // FISHEYE, backward only
  float dlt[2];         // OPENCV: delta(xn, yn)
  float Ju[6];          // OPENCV: du/dpc at the unclamped (xn, yn), backward only
};

// ---- OPENCV (COLMAP's OpenCVCameraModel), on (a, b) = (x, y) / z with rho = a^2 + b^2,
// R = 1 + k1 rho + k2 rho^2, R' = dR/drho = k1 + 2 k2 rho:
//   delta = (a R + 2 p1 a b + p2 (rho + 2 a^2),  b R + p1 (rho + 2 b^2) + 2 p2 a b),
//   u = (fx delta_x(xn, yn) + cx, fy delta_y(xn, yn) + cy)                      (never clamped)
//   J = diag(fx, fy) Ddelta(xh, yh) (1/z) [[1, 0, -xh], [0, 1, -yh]],  (xh, yh) = clamp((xn, yn), +-1.3 tan_fov)
// Ddelta is symmetric:  D00 = R + 2 a^2 R' + 2 p1 b + 6 p2 a,  D01 = D10 = 2 a b R' + 2 p1 a + 2 p2 b,
//   D11 = R + 2 b^2 R' + 6 p1 b + 2 p2 a.  The host stretches tan_fov by the lens (DESIGN 3.19).
// A Gaussian is culled like z < 0.2 where rho >= rho_valid (the radial map r R(r^2) stops
// increasing) or det Ddelta(xn, yn) <= 0: beyond either the polynomial folds back.
GSB_HD void opencv_delta(float a, float b, const float k[4], float dlt[2]) {
  const float rho = fmaf(a, a, b * b), R = fmaf(rho, fmaf(rho, k[1], k[0]), 1.f), ab = a * b;
  dlt[0] = fmaf(a, R, fmaf(2.f * k[2], ab, k[3] * fmaf(2.f * a, a, rho)));
  dlt[1] = fmaf(b, R, fmaf(k[2], fmaf(2.f * b, b, rho), 2.f * k[3] * ab));
}

// Ddelta at (a, b) as (D00, D01, D11)
GSB_HD void opencv_D(float a, float b, const float k[4], float D[3]) {
  const float rho = fmaf(a, a, b * b), R = fmaf(rho, fmaf(rho, k[1], k[0]), 1.f), R1 = fmaf(2.f * k[1], rho, k[0]);
  D[0] = fmaf(2.f * a * a, R1, R) + fmaf(2.f * k[2], b, 6.f * k[3] * a);
  D[1] = fmaf(2.f * a * b, R1, fmaf(2.f * k[2], a, 2.f * k[3] * b));
  D[2] = fmaf(2.f * b * b, R1, R) + fmaf(6.f * k[2], b, 2.f * k[3] * a);
}

// rho_valid: the smallest positive root of d(r R)/dr = 1 + 3 k1 rho + 5 k2 rho^2, +inf if none
GSB_HD float opencv_rho_valid(float k1, float k2) {
  if (k2 == 0.f) return k1 < 0.f ? -1.f / (3.f * k1) : INFINITY;
  const float b = 3.f * k1, a = 5.f * k2, disc = fmaf(b, b, -4.f * a);
  if (disc < 0.f) return INFINITY;
  const float q = -0.5f * (b + copysignf(sqrtf(disc), b));  // roots q / a and 1 / q, q != 0
  const float r1 = q / a, r2 = 1.f / q;
  return fminf(r1 > 0.f ? r1 : INFINITY, r2 > 0.f ? r2 : INFINITY);
}

// J = (1/z) diag(f) [[D0, D1, -(D0 a + D1 b)], [D1, D2, -(D1 a + D2 b)]] with D = Ddelta(a, b)
GSB_HD void opencv_J(float a, float b, float zi, float fx, float fy, const float D[3], float J[6]) {
  const float fxz = fx * zi, fyz = fy * zi;
  J[0] = fxz * D[0]; J[1] = fxz * D[1]; J[2] = -fmaf(J[0], a, J[1] * b);
  J[3] = fyz * D[1]; J[4] = fyz * D[2]; J[5] = -fmaf(J[3], a, J[4] * b);
}

// false when the Gaussian lies beyond the range where the fisheye's theta_d increases
// (theta_d' <= 0), or OPENCV's fold: culled like z < 0.2.  A culled Gaussian (keep false) is
// evaluated at (0, 0, 1).
template <int MODEL>
GSB_HD bool lens(const float pc_in[3], bool keep, const Cam &cam, Lens &L) {
  if constexpr (MODEL == ORTHO) {
    L.J[0] = cam.fx; L.J[1] = 0.f; L.J[2] = 0.f;
    L.J[3] = 0.f; L.J[4] = cam.fy; L.J[5] = 0.f;
    return true;
  } else if constexpr (MODEL == OPENCV) {
    const float x = keep ? pc_in[0] : 0.f, y = keep ? pc_in[1] : 0.f, z = keep ? pc_in[2] : 1.f;
    const float zi = 1.0f / z, xn = x * zi, yn = y * zi;
    const float limx = 1.3f * cam.tan_fovx, limy = 1.3f * cam.tan_fovy;
    const float xh = fminf(limx, fmaxf(-limx, xn)), yh = fminf(limy, fmaxf(-limy, yn));
    opencv_delta(xn, yn, cam.k, L.dlt);
    float Du[3], D[3];
    opencv_D(xn, yn, cam.k, Du);
    opencv_D(xh, yh, cam.k, D);
    opencv_J(xn, yn, zi, cam.fx, cam.fy, Du, L.Ju);
    opencv_J(xh, yh, zi, cam.fx, cam.fy, D, L.J);
    return fmaf(xn, xn, yn * yn) < opencv_rho_valid(cam.k[0], cam.k[1]) && Du[0] * Du[2] - Du[1] * Du[1] > 0.f;
  } else {
    static_assert(MODEL == FISHEYE, "unknown camera model");
    const float x = keep ? pc_in[0] : 0.f, y = keep ? pc_in[1] : 0.f, z = keep ? pc_in[2] : 1.f;
    const float *k = cam.k;
    const float r2 = x * x + y * y, r = sqrtf(r2), q = fmaf(z, z, r2), qi = 1.0f / q, zi = 1.0f / z;
    const float t = r * zi;
    const float th = atan2f(r, z), th2 = th * th;
    // theta_d / theta, theta_d' and theta_d'' / theta, polynomials in theta^2
    const float P = fmaf(th2, fmaf(th2, fmaf(th2, fmaf(th2, k[3], k[2]), k[1]), k[0]), 1.f);
    const float P1 = fmaf(th2, fmaf(th2, fmaf(th2, fmaf(th2, 9.f * k[3], 7.f * k[2]), 5.f * k[1]), 3.f * k[0]), 1.f);
    const float P2 = fmaf(th2, fmaf(th2, fmaf(th2, 72.f * k[3], 42.f * k[2]), 20.f * k[1]), 6.f * k[0]);
    float tht;  // theta / t
    if (t < kFishSeries) {
      const float t2 = t * t, a1 = k[0] - (1.f / 3.f), a2 = 0.2f - k[0] + k[1];
      const float zi2 = zi * zi, zi3 = zi2 * zi;
      L.s = zi * fmaf(t2, fmaf(t2, a2, a1), 1.f);
      L.g = zi3 * fmaf(4.f * a2, t2, 2.f * a1);
      L.G = zi3 * zi2 * (8.f * a2);
      tht = fmaf(t2, -1.f / 3.f, 1.f);
    } else {
      tht = th / t;
      L.s = P * th / r;
      L.g = (P1 * z * qi - L.s) / r2;
      const float A = r * z * qi, sn2 = r2 * qi;       // sin(theta) cos(theta), sin^2(theta)
      const float F = P1 * A - P * th;                   // g r^3
      const float Fp = P2 * th * A - 2.f * P1 * sn2;     // dF/dtheta
      L.G = (A * Fp - 3.f * F) / (r2 * r2 * r);
    }
    L.h = P1 * qi;
    L.H = (P2 * tht - 2.f * P1) * qi * qi;
    L.hz = -(P2 * th * r + 2.f * z * P1) * qi * qi;
    const float fx = cam.fx, fy = cam.fy, xyg = x * y * L.g;
    L.J[0] = fx * fmaf(x * x, L.g, L.s); L.J[1] = fx * xyg; L.J[2] = -fx * x * L.h;
    L.J[3] = fy * xyg; L.J[4] = fy * fmaf(y * y, L.g, L.s); L.J[5] = -fy * y * L.h;
    return P1 > 0.f;
  }
}

// projected mean of a kept Gaussian under ORTHO / FISHEYE / OPENCV (PINHOLE: project_mean)
template <int MODEL>
GSB_HD void lens_mean(const float pc[3], const Cam &cam, const Lens &L, float u[2]) {
  if constexpr (MODEL == ORTHO) {
    u[0] = fmaf(cam.fx, pc[0], cam.cx);
    u[1] = fmaf(cam.fy, pc[1], cam.cy);
  } else if constexpr (MODEL == OPENCV) {
    u[0] = fmaf(cam.fx, L.dlt[0], cam.cx);
    u[1] = fmaf(cam.fy, L.dlt[1], cam.cy);
  } else {
    u[0] = fmaf(cam.fx * L.s, pc[0], cam.cx);
    u[1] = fmaf(cam.fy * L.s, pc[1], cam.cy);
  }
}

// cov2d (Cov2d's M, MS, c2, raw; not xc, yc, zi) under ORTHO / FISHEYE / OPENCV: M = J Rcw with J = L.J
GSB_HD void cov2d_lens(const Lens &L, const float S6[6], const float R[9], Cov2d &o) {
  for (int a = 0; a < 2; a++)
    for (int c = 0; c < 3; c++)
      o.M[3 * a + c] = fmaf(L.J[3 * a], R[c], fmaf(L.J[3 * a + 1], R[3 + c], L.J[3 * a + 2] * R[6 + c]));
  const float S[9] = {S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5]};
  for (int a = 0; a < 2; a++)
    for (int c = 0; c < 3; c++)
      o.MS[3 * a + c] = o.M[3 * a] * S[c] + o.M[3 * a + 1] * S[3 + c] + o.M[3 * a + 2] * S[6 + c];
  o.raw[0] = o.MS[0] * o.M[0] + o.MS[1] * o.M[1] + o.MS[2] * o.M[2];
  o.raw[1] = o.MS[3] * o.M[3] + o.MS[4] * o.M[4] + o.MS[5] * o.M[5];
  o.c2[0] = o.raw[0] + kBlur;
  o.c2[1] = o.MS[0] * o.M[3] + o.MS[1] * o.M[4] + o.MS[2] * o.M[5];
  o.c2[2] = o.raw[1] + kBlur;
}

// dL/dpc of the cov2d term under FISHEYE / OPENCV: sum_ab dL/dJ_ab dJ_ab/dpc (ORTHO: J is constant)
template <int MODEL>
GSB_HD void lens_dJ_dpc(const float pc[3], const Cam &cam, const Lens &L, const float dJ[6], float gpc[3]) {
  if constexpr (MODEL == OPENCV) {
    // J = (1/z) K(xh, yh): 1/z carries dL/dz; a clamped coordinate has no derivative, an unclamped
    // one dxh/dx = 1/z, dxh/dz = -xh/z.  dD/da = (6 a R' + 4 a^3 R'' + 6 p2, 2 b R' + 4 a^2 b R'' + 2 p1,
    // 2 a R' + 4 a b^2 R'' + 2 p2), dD/db = (dD01/da, dD11/da, 6 b R' + 4 b^3 R'' + 6 p1), R'' = 2 k2.
    const float *k = cam.k;
    const float zi = 1.0f / pc[2], xn = pc[0] * zi, yn = pc[1] * zi;
    const float limx = 1.3f * cam.tan_fovx, limy = 1.3f * cam.tan_fovy;
    const float a = fminf(limx, fmaxf(-limx, xn)), b = fminf(limy, fmaxf(-limy, yn));
    const float rho = fmaf(a, a, b * b), R1 = fmaf(2.f * k[1], rho, k[0]), R2 = 2.f * k[1];
    float D[3];
    opencv_D(a, b, k, D);
    const float Da0 = fmaf(6.f * a, R1, fmaf(4.f * a * a * a, R2, 6.f * k[3]));
    const float Da1 = fmaf(2.f * b, R1, fmaf(4.f * a * a * b, R2, 2.f * k[2]));
    const float Da2 = fmaf(2.f * a, R1, fmaf(4.f * a * b * b, R2, 2.f * k[3]));
    const float Db2 = fmaf(6.f * b, R1, fmaf(4.f * b * b * b, R2, 6.f * k[2]));
    const float A0 = dJ[0] * cam.fx, A1 = dJ[1] * cam.fx, A2 = dJ[2] * cam.fx;
    const float B0 = dJ[3] * cam.fy, B1 = dJ[4] * cam.fy, B2 = dJ[5] * cam.fy;
    // dL/da, dL/db of K (row 0: [D0, D1, -(D0 a + D1 b)], row 1: [D1, D2, -(D1 a + D2 b)])
    const float ga = A0 * Da0 + A1 * Da1 - A2 * fmaf(Da0, a, fmaf(Da1, b, D[0])) + B0 * Da1 + B1 * Da2 -
                     B2 * fmaf(Da1, a, fmaf(Da2, b, D[1]));
    const float gb = A0 * Da1 + A1 * Da2 - A2 * fmaf(Da1, a, fmaf(Da2, b, D[1])) + B0 * Da2 + B1 * Db2 -
                     B2 * fmaf(Da2, a, fmaf(Db2, b, D[2]));
    const float gK = A0 * D[0] + A1 * D[1] - A2 * fmaf(D[0], a, D[1] * b) + B0 * D[1] + B1 * D[2] -
                     B2 * fmaf(D[1], a, D[2] * b);
    const float gx = a == xn ? ga : 0.f, gy = b == yn ? gb : 0.f, zi2 = zi * zi;
    gpc[0] = gx * zi2;
    gpc[1] = gy * zi2;
    gpc[2] = -(gK + fmaf(gx, a, gy * b)) * zi2;
  } else {
    static_assert(MODEL == FISHEYE, "dJ/dpc of a camera model without one");
    const float x = pc[0], y = pc[1], fx = cam.fx, fy = cam.fy;
    const float g = L.g, G = L.G, h = L.h, H = L.H, xx = x * x, yy = y * y, xy = x * y;
    // row 0: J00 = fx (s + x^2 g), J01 = fx x y g, J02 = -fx x h
    const float a0 = dJ[0] * fx, a1 = dJ[1] * fx, a2 = dJ[2] * fx;
    const float b0 = dJ[3] * fy, b1 = dJ[4] * fy, b2 = dJ[5] * fy;
    gpc[0] = a0 * x * fmaf(xx, G, 3.f * g) + a1 * y * fmaf(xx, G, g) - a2 * fmaf(xx, H, h) +
             b0 * y * fmaf(xx, G, g) + b1 * x * fmaf(yy, G, g) - b2 * xy * H;
    gpc[1] = a0 * y * fmaf(xx, G, g) + a1 * x * fmaf(yy, G, g) - a2 * xy * H +
             b0 * x * fmaf(yy, G, g) + b1 * y * fmaf(yy, G, 3.f * g) - b2 * fmaf(yy, H, h);
    gpc[2] = -a0 * fmaf(xx, H, h) - a1 * xy * H - a2 * x * L.hz -
             b0 * xy * H - b1 * fmaf(yy, H, h) - b2 * y * L.hz;
  }
}

// The intrinsics gradient of one kept Gaussian under ORTHO / FISHEYE / OPENCV (DESIGN 3.23): gint[8] =
// dL/d(fx, fy, cx, cy, k[4]) = gu . du/dtheta + sum_ab dJ_ab dJ_ab/dtheta, with dJ = dL/dJ as backward_one
// forms it.  Row 0 of J and u - cx are fx times factors free of fx (and row 1, v - cy fy times), so the
// fx, fy terms are those factors; dL/dcx = gu[0], dL/dcy = gu[1].  The clamp bound is a constant (as
// in lens_dJ_dpc): a clamped coordinate contributes dJ/dtheta at the bound.
//   FISHEYE: ds/dk_j = theta^(2j+1) / r, dg/dk_j = ((2j+1) theta^2j z / q - ds/dk_j) / r^2, dh/dk_j =
//   (2j+1) theta^2j / q; below kFishSeries the derivatives of s and g come from their series to O(t^4)
//   relative, ds/dk1 = t^2 (1 - t^2) / z, ds/dk2 = t^4 (1 - 5 t^2 / 3) / z, dg/dk1 = (2 - 4 t^2) / z^3,
//   dg/dk2 = t^2 (4 - 10 t^2) / z^3, and k3's and k4's (O(t^4) and O(t^6) relative to k1's) are taken as 0.
//   OPENCV: ddelta/dk at the unclamped (xn, yn) (in u), dDdelta/dk at the clamped (xh, yh) (in J).
template <int MODEL>
GSB_HD void lens_dintr(const float pc[3], const Cam &cam, const Lens &L, const float dJ[6], const float gu[2],
                       float gint[8]) {
  gint[2] = gu[0];
  gint[3] = gu[1];
  gint[4] = gint[5] = gint[6] = gint[7] = 0.f;
  if constexpr (MODEL == ORTHO) {
    gint[0] = fmaf(gu[0], pc[0], dJ[0]);
    gint[1] = fmaf(gu[1], pc[1], dJ[4]);
  } else if constexpr (MODEL == OPENCV) {
    const float *k = cam.k;
    const float zi = 1.0f / pc[2], xn = pc[0] * zi, yn = pc[1] * zi;
    const float limx = 1.3f * cam.tan_fovx, limy = 1.3f * cam.tan_fovy;
    const float a = fminf(limx, fmaxf(-limx, xn)), b = fminf(limy, fmaxf(-limy, yn));
    float D[3];
    opencv_D(a, b, k, D);
    // dL/dD (J = (1/z) diag(f) [[D0, D1, -(D0 a + D1 b)], [D1, D2, -(D1 a + D2 b)]]) without the f
    const float r0 = zi * fmaf(-dJ[2], a, dJ[0]), r1 = zi * fmaf(-dJ[2], b, dJ[1]);
    const float s1 = zi * fmaf(-dJ[5], a, dJ[3]), s2 = zi * fmaf(-dJ[5], b, dJ[4]);
    gint[0] = fmaf(r0, D[0], fmaf(r1, D[1], gu[0] * L.dlt[0]));
    gint[1] = fmaf(s1, D[1], fmaf(s2, D[2], gu[1] * L.dlt[1]));
    const float g0 = cam.fx * r0, g1 = fmaf(cam.fx, r1, cam.fy * s1), g2 = cam.fy * s2;
    const float A = cam.fx * gu[0], B = cam.fy * gu[1];
    const float rc = fmaf(a, a, b * b), ru = fmaf(xn, xn, yn * yn), ab = a * b, xy = xn * yn;
    const float gd = fmaf(A, xn, B * yn);  // gu . diag(f) (xn, yn)
    gint[4] = fmaf(g0, fmaf(2.f * a, a, rc), fmaf(g1, 2.f * ab, fmaf(g2, fmaf(2.f * b, b, rc), ru * gd)));
    gint[5] = fmaf(rc, fmaf(g0, fmaf(4.f * a, a, rc), fmaf(g1, 4.f * ab, g2 * fmaf(4.f * b, b, rc))), ru * ru * gd);
    gint[6] = fmaf(2.f * g0, b, fmaf(2.f * g1, a, fmaf(6.f * g2, b, fmaf(A, 2.f * xy, B * fmaf(2.f * yn, yn, ru)))));
    gint[7] = fmaf(6.f * g0, a, fmaf(2.f * g1, b, fmaf(2.f * g2, a, fmaf(A, fmaf(2.f * xn, xn, ru), B * 2.f * xy))));
  } else {
    static_assert(MODEL == FISHEYE, "no intrinsics gradient for this camera model");
    const float x = pc[0], y = pc[1], z = pc[2], xx = x * x, yy = y * y, xy = x * y;
    const float a0 = dJ[0], a1 = dJ[1], a2 = dJ[2], b0 = dJ[3], b1 = dJ[4], b2 = dJ[5];
    // row 0: J = fx (s + x^2 g, x y g, -x h), u - cx = fx s x;  row 1 likewise with fy
    gint[0] = fmaf(a0, fmaf(xx, L.g, L.s), fmaf(a1, xy * L.g, fmaf(-a2, x * L.h, gu[0] * L.s * x)));
    gint[1] = fmaf(b0, xy * L.g, fmaf(b1, fmaf(yy, L.g, L.s), fmaf(-b2, y * L.h, gu[1] * L.s * y)));
    const float r2 = xx + yy, r = sqrtf(r2), q = fmaf(z, z, r2), qi = 1.0f / q, zi = 1.0f / z, t = r * zi;
    const float th = atan2f(r, z), th2 = th * th;
    // sum over both rows of dL/d(s, g, h) with the f's: dL/dtheta_k = Ss ds/dk + Sg dg/dk + Sh dh/dk
    const float Ss = cam.fx * fmaf(gu[0], x, a0) + cam.fy * fmaf(gu[1], y, b1);
    const float Sg = cam.fx * fmaf(a0, xx, a1 * xy) + cam.fy * fmaf(b0, xy, b1 * yy);
    const float Sh = -(cam.fx * a2 * x + cam.fy * b2 * y);
    float p = 1.f;  // theta^2j
    for (int j = 0; j < 4; j++) {
      p *= th2;
      const float c = 2.f * j + 3.f;
      float ds, dg;
      if (t < kFishSeries) {
        const float t2 = t * t, zi3 = zi * zi * zi;
        ds = j == 0 ? zi * t2 * fmaf(-t2, 1.f, 1.f) : (j == 1 ? zi * t2 * t2 * fmaf(-5.f / 3.f, t2, 1.f) : 0.f);
        dg = j == 0 ? zi3 * fmaf(-4.f, t2, 2.f) : (j == 1 ? zi3 * t2 * fmaf(-10.f, t2, 4.f) : 0.f);
      } else {
        ds = p * th / r;
        dg = (c * p * z * qi - ds) / r2;
      }
      gint[4 + j] = fmaf(Ss, ds, fmaf(Sg, dg, Sh * (c * p * qi)));
    }
  }
}

// Antialiasing (2D-filter opacity compensation, Mip-Splatting; gsplat's rasterize_mode
// "antialiased"): the blur spreads a Gaussian's mass, so its opacity is scaled by
//   rho = sqrt(max(kAaMinR, r)),  r = det(Sigma) / det(Sigma + kBlur I) = (a c - b^2) di
// with (a, b, c) the pre-blur cov2d and di = 1 / det of the blurred one (conic()).  r is the
// ratio the rasterizers would otherwise over-draw a sub-pixel Gaussian by.
constexpr float kAaMinR = 2.5e-5f;
GSB_HD void aa_scale(float a, float b, float c, float di, float &rho, float &r) {
  r = (a * c - b * b) * di;
  const float x = fmaxf(kAaMinR, r);
#ifdef __CUDA_ARCH__
  rho = x * rsqrtf(x);  // x >= kAaMinR is a normal number: no slow-path call (and no stack frame)
#else
  rho = sqrtf(x);
#endif
}

// conic = cov2d^-1 with di = 1/det; false when di is NaN: such a Gaussian is culled (kernel.cu:301-305)
GSB_HD bool conic(const float c2[3], float &di, float cn[3]) {
  di = 1.0f / (c2[0] * c2[2] - c2[1] * c2[1]);
  cn[0] = di * c2[2];
  cn[1] = -di * c2[1];
  cn[2] = di * c2[0];
  return di == di;
}

// 3-sigma radius in pixels, exactly as the reference (IEEE sqrt, one multiply, ceil, truncate):
// it decides the tile rectangle, so it has to be bit-identical
GSB_HD void radius(const float c2[3], int area[2]) {
  area[0] = (int)ceilf(3.0f * sqrtf(fabsf(c2[0])));
  area[1] = (int)ceilf(3.0f * sqrtf(fabsf(c2[2])));
}

// view direction r = d / |d| with d = pw - twc; returns ninv = 1 / |d|.  FMA_NORM: |d|^2 as
// fma(d2, d2, fma(d0, d0, d1 d1)), the rounding k_sh2color<16> has always had (the compiler
// contracted it there and nowhere else)
template <bool FMA_NORM = false>
GSB_HD float view_dir(const float pw[3], const float twc[3], float d[3], float r[3]) {
  d[0] = pw[0] - twc[0]; d[1] = pw[1] - twc[1]; d[2] = pw[2] - twc[2];
  const float n2 = FMA_NORM ? fmaf(d[2], d[2], fmaf(d[0], d[0], d[1] * d[1]))
                            : d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  const float ninv = 1.0f / sqrtf(n2);
  r[0] = d[0] * ninv; r[1] = d[1] * ninv; r[2] = d[2] * ninv;
  return ninv;
}

// real SH basis up to degree 3 and its partial derivatives wrt the (unit) direction, with
// xx, yy, zz treated as independent monomials exactly as the reference does.
template <int K3>
GSB_HD void sh_basis(float x, float y, float z, float Y[K3], float dY[K3][3]) {
#define GSB_SET(l, v, dx, dy, dz)                        \
  if (l < K3) {                                          \
    Y[l % K3] = (v);                                     \
    dY[l % K3][0] = (dx); dY[l % K3][1] = (dy); dY[l % K3][2] = (dz); \
  }
  const float C1a = -0.4886025119029199f, C1b = 0.4886025119029199f;
  const float C20 = 1.0925484305920792f, C22 = 0.31539156525252005f, C24 = 0.5462742152960396f;
  const float C30 = -0.5900435899266435f, C31 = 2.890611442640554f, C32 = -0.4570457994644658f,
              C33 = 0.3731763325901154f, C35 = 1.445305721320277f;
  GSB_SET(0, 0.28209479177387814f, 0.f, 0.f, 0.f)
  GSB_SET(1, C1a * y, 0.f, C1a, 0.f)
  GSB_SET(2, C1b * z, 0.f, 0.f, C1b)
  GSB_SET(3, C1a * x, C1a, 0.f, 0.f)
  const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
  GSB_SET(4, C20 * xy, C20 * y, C20 * x, 0.f)
  GSB_SET(5, -C20 * yz, 0.f, -C20 * z, -C20 * y)
  GSB_SET(6, C22 * (2.f * zz - xx - yy), -2.f * C22 * x, -2.f * C22 * y, 4.f * C22 * z)
  GSB_SET(7, -C20 * xz, -C20 * z, 0.f, -C20 * x)
  GSB_SET(8, C24 * (xx - yy), 2.f * C24 * x, -2.f * C24 * y, 0.f)
  GSB_SET(9, C30 * y * (3.f * xx - yy), C30 * 6.f * xy, C30 * (3.f * xx - 3.f * yy), 0.f)
  GSB_SET(10, C31 * xy * z, C31 * yz, C31 * xz, C31 * xy)
  GSB_SET(11, C32 * y * (4.f * zz - xx - yy), C32 * (-2.f * xy), C32 * (4.f * zz - xx - 3.f * yy), C32 * 8.f * yz)
  GSB_SET(12, C33 * z * (2.f * zz - 3.f * xx - 3.f * yy), C33 * (-6.f * xz), C33 * (-6.f * yz),
          C33 * (6.f * zz - 3.f * xx - 3.f * yy))
  GSB_SET(13, C32 * x * (4.f * zz - xx - yy), C32 * (4.f * zz - 3.f * xx - yy), C32 * (-2.f * xy), C32 * 8.f * xz)
  GSB_SET(14, C35 * z * (xx - yy), C35 * 2.f * xz, C35 * (-2.f * yz), C35 * (xx - yy))
  GSB_SET(15, C30 * x * (xx - 3.f * yy), C30 * (3.f * xx - 3.f * yy), C30 * (-6.f * xy), 0.f)
#undef GSB_SET
}

// Everything the backward needs again is recomputed from the parameters by this same
// function, so forward and backward see identical intermediates.
struct Geo : Cov2d {
  float pc[3];        // camera-frame position
  float R3[9], M3[9]; // R(q), R(q) diag(s)
  float S6[6];        // cov3d upper triangle
  float di;           // 1 / det(cov2d)
  float cn[3];        // conic
  bool keep;          // z >= 0.2 and 1/det not NaN (FISHEYE: and theta_d' > 0; OPENCV: unfolded)
  Lens L;             // ORTHO / FISHEYE / OPENCV only
};

template <int MODEL = PINHOLE>
GSB_HD void geometry(const float pw[3], const float q[4], const float s[3], const Cam &cam, Geo &g) {
  g.keep = camera_point(cam.R, cam.t, pw, g.pc);
  cov3d(q, s, g.R3, g.M3, g.S6);
  if constexpr (MODEL == PINHOLE) {
    cov2d(g.pc, g.keep, g.S6, cam.R, cam.fx, cam.fy, cam.tan_fovx, cam.tan_fovy, g);
  } else {
    if (!lens<MODEL>(g.pc, g.keep, cam, g.L)) g.keep = false;
    cov2d_lens(g.L, g.S6, cam.R, g);
  }
  if (!conic(g.c2, g.di, g.cn)) g.keep = false;
}

// forward outputs for one Gaussian.  Returns rho (aa_scale) with AA, 1 without or when culled:
// the caller composites rho * alpha.  Every output is the same with and without AA.
template <int K3, bool AA = false, int MODEL = PINHOLE>
GSB_HD float forward_one(const float pw[3], const float q[4], const float s[3], const float *sh /*[K3][3]*/,
                         const Cam &cam, float u[2], float cn[3], float col[3], float *depth, int area[2]) {
  Geo g;
  geometry<MODEL>(pw, q, s, cam, g);
  // colour is not gated by depth in the reference (kernel.cu:619-726)
  float Y[K3], dY[K3][3];
  float d[3], r[3] = {0.f, 0.f, 0.f};
  if (K3 > 1) view_dir(pw, cam.twc, d, r);
  sh_basis<K3>(r[0], r[1], r[2], Y, dY);
  col[0] = col[1] = col[2] = 0.5f;
  for (int l = 0; l < K3; l++)
    for (int c = 0; c < 3; c++) col[c] = fmaf(Y[l], sh[3 * l + c], col[c]);
  if (!g.keep) {
    u[0] = u[1] = 0.f;
    cn[0] = cn[1] = cn[2] = 0.f;
    area[0] = area[1] = 0;
    *depth = -1.0f;
    return 1.f;
  }
  if constexpr (MODEL == PINHOLE)
    project_mean(g.pc, g.zi, cam.fx, cam.fy, cam.cx, cam.cy, u);
  else
    lens_mean<MODEL>(g.pc, cam, g.L, u);
  cn[0] = g.cn[0]; cn[1] = g.cn[1]; cn[2] = g.cn[2];
  radius(g.c2, area);
  *depth = g.pc[2];
  float rho = 1.f;
  if (AA) {
    float r;
    aa_scale(g.raw[0], g.c2[1], g.raw[1], g.di, rho, r);
  }
  return rho;
}

// backward for one Gaussian.  gu[2], gconic[3], gcol[3] are the splatB outputs for it.
// gsh may alias sh (row-private in-place update).  DEPTH: gdepth = dL/dz from the RGB-D
// rasterizer; z = pc[2], so it adds to dL/dpc[2] and reaches dL/dpw through Rcw[2,:].
// POSE: this Gaussian's contribution to the camera gradient, gcam[15] = dL/dRcw (row-major 9),
// dL/dtcw (3), dL/dtwc (3):
//   dL/dtcw = gpc;  dL/dRcw = gpc (x) pw + J^T dL/dM  (pc = Rcw pw + tcw, M = J Rcw);
//   dL/dtwc = -(colour part of dL/dpw)  (the view direction is pw - twc).
// gpc is the vector rotated into dL/dpw (x, y taken as unclamped, as above); a culled Gaussian
// contributes through its colour branch only, as it does to dL/dpw.
// AA: the rasterizers composited alpha_eff = rho alpha (forward_one<K3, true>); galpha =
// dL/dalpha_eff, alpha the raw opacity.  Returns dL/dalpha = rho galpha (galpha without AA) and
// adds alpha galpha drho/d(a, b, c) to dL/dcov2d, from where it reaches every geometry gradient
// (and gcam) like the conic's.  With w = kBlur, D = 1/di = det of the blurred cov2d (a', b, c'):
//   dr/da = w (c c' + b^2) di^2,  dr/db = -2 w b (w + a + c) di^2,  dr/dc = w (a a' + b^2) di^2,
// drho = dr / (2 rho), and 0 where the clamp holds (r <= kAaMinR).  galpha != 0 alone makes the
// Gaussian's geometry gradient non-zero, so it joins the zero-gradient gate.
// INTR (with POSE): gcam[15..22] also receives the intrinsics gradient dL/d(fx, fy, cx, cy, k[4])
// (lens_dintr; PINHOLE: the same with J00 = fx/z, J02 = -fx xc/z^2, u - cx = fx x/z and k's 0), from the
// same dJ and gu, antialiasing's term included; 0 for a culled Gaussian.
template <int K3, bool DEPTH = false, bool POSE = false, bool AA = false, int MODEL = PINHOLE, bool INTR = false>
GSB_HD float backward_one(const float pw[3], const float q[4], const float s[3], const float *sh,
                          const Cam &cam, const float gu[2], const float gconic[3], const float gcol[3],
                          float gpw[3], float gq[4], float gs[3], float *gsh /*[K3][3]*/, float gdepth = 0.f,
                          float *gcam = nullptr /*[15], POSE only; [23] with INTR*/, float galpha = 0.f,
                          float alpha = 0.f) {
  static_assert(!INTR || POSE, "the intrinsics gradient comes with the pose's");
  // ---- colour branch (independent of the depth cull, like sh2Color)
  float Y[K3], dY[K3][3];
  float d[3], ninv = 1.f, r[3] = {0.f, 0.f, 0.f};
  if (K3 > 1) ninv = view_dir(pw, cam.twc, d, r);
  sh_basis<K3>(r[0], r[1], r[2], Y, dY);
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
  if (POSE) {
    for (int e = 0; e < 12; e++) gcam[e] = 0.f;
    for (int a = 0; a < 3; a++) gcam[12 + a] = -gpw[a];
    if (INTR)
      for (int e = 15; e < 23; e++) gcam[e] = 0.f;
  }
  gq[0] = gq[1] = gq[2] = gq[3] = 0.f;
  gs[0] = gs[1] = gs[2] = 0.f;

  // ---- geometry branch
  Geo g;
  geometry<MODEL>(pw, q, s, cam, g);
  const bool any = (gu[0] != 0.f) || (gu[1] != 0.f) || (gconic[0] != 0.f) || (gconic[1] != 0.f) || (gconic[2] != 0.f) ||
                   (DEPTH && gdepth != 0.f) || (AA && galpha != 0.f);
  if (!g.keep || !any) return galpha;  // rho = 1 when culled; rho * 0 otherwise
  const float a = g.c2[0], b = g.c2[1], c = g.c2[2], di = g.di, d2 = di * di;
  // dL/dcov2d = dL/dconic . dconic/dcov2d   (B.5.3)
  float ga = gconic[0] * (-c * c * d2) + gconic[1] * (b * c * d2) + gconic[2] * (di - a * c * d2);
  float gb = gconic[0] * (2.f * b * c * d2) + gconic[1] * (-di - 2.f * b * b * d2) + gconic[2] * (2.f * a * b * d2);
  float gc = gconic[0] * (di - a * c * d2) + gconic[1] * (a * b * d2) + gconic[2] * (-a * a * d2);
  float galpha_raw = galpha;
  if (AA) {
    const float ar = g.raw[0], cr = g.raw[1];
    float rho, r;
    aa_scale(ar, b, cr, di, rho, r);
    galpha_raw = rho * galpha;
    if (r > kAaMinR) {
      // drho/dr = 1 / (2 rho), rho in [0.005, 1]: the fast division is exact to 2 ulp there and
      // adds no slow-path call (whose register saves cost the K3 = 16 kernel a stack frame)
#ifdef __CUDA_ARCH__
      const float k = alpha * galpha * (kBlur * d2) * __fdividef(0.5f, rho);
#else
      const float k = alpha * galpha * (kBlur * d2) * (0.5f / rho);
#endif
      ga += k * (cr * c + b * b);
      gb += k * (-2.f * b * (kBlur + ar + cr));
      gc += k * (ar * a + b * b);
    }
  }
  // G = [[ga, gb/2], [gb/2, gc]]
  const float G00 = ga, G01 = 0.5f * gb, G11 = gc;
  const float *M = g.M;
  // GM (2x3)
  float GM[6];
  for (int k = 0; k < 3; k++) {
    GM[k] = G00 * M[k] + G01 * M[3 + k];
    GM[3 + k] = G01 * M[k] + G11 * M[3 + k];
  }
  // dL/dSigma_ij = (2 - delta_ij) (M^T G M)_ij
  float g3[6];
  {
    int n = 0;
    for (int i = 0; i < 3; i++)
      for (int j = i; j < 3; j++) {
        const float v = M[i] * GM[j] + M[3 + i] * GM[3 + j];
        g3[n++] = (i == j) ? v : 2.f * v;
      }
  }
  // dL/dM = 2 G (M Sigma);  dL/dJ = dL/dM Rcw^T
  float dM[6];
  for (int k = 0; k < 3; k++) {
    dM[k] = 2.f * (G00 * g.MS[k] + G01 * g.MS[3 + k]);
    dM[3 + k] = 2.f * (G01 * g.MS[k] + G11 * g.MS[3 + k]);
  }
  const float *R = cam.R;
  float dJ[6];
  for (int a2 = 0; a2 < 2; a2++)
    for (int k = 0; k < 3; k++)
      dJ[3 * a2 + k] = dM[3 * a2] * R[3 * k] + dM[3 * a2 + 1] * R[3 * k + 1] + dM[3 * a2 + 2] * R[3 * k + 2];
  float gpc[3];
  if constexpr (MODEL == PINHOLE) {
    const float zi = g.zi, zi2 = zi * zi, zi3 = zi2 * zi;
    gpc[0] = dJ[2] * (-cam.fx * zi2);
    gpc[1] = dJ[5] * (-cam.fy * zi2);
    gpc[2] = dJ[0] * (-cam.fx * zi2) + dJ[2] * (2.f * cam.fx * g.xc * zi3) + dJ[4] * (-cam.fy * zi2) +
             dJ[5] * (2.f * cam.fy * g.yc * zi3);
    // projection u = (fx x/z + cx, fy y/z + cy)   (B.1.2, unclamped x, y)
    gpc[0] += gu[0] * (cam.fx * zi);
    gpc[1] += gu[1] * (cam.fy * zi);
    gpc[2] += -(gu[0] * (g.pc[0] * cam.fx) + gu[1] * (g.pc[1] * cam.fy)) * zi2;
    if (DEPTH) gpc[2] += gdepth;  // depth z = pc[2]
    for (int j = 0; j < 3; j++) gpw[j] += gpc[0] * R[j] + gpc[1] * R[3 + j] + gpc[2] * R[6 + j];
    if (POSE) {
      // J = [[J00, 0, J02], [0, J11, J12]] exactly as cov2d() evaluated it
      const float J00 = cam.fx * zi, J11 = cam.fy * zi;
      const float J02 = -(cam.fx * g.xc) * zi2, J12 = -(cam.fy * g.yc) * zi2;
      for (int k = 0; k < 3; k++) {
        gcam[k] = fmaf(gpc[0], pw[k], J00 * dM[k]);
        gcam[3 + k] = fmaf(gpc[1], pw[k], J11 * dM[3 + k]);
        gcam[6 + k] = fmaf(gpc[2], pw[k], fmaf(J02, dM[k], J12 * dM[3 + k]));
        gcam[9 + k] = gpc[k];
      }
    }
    if (INTR) {
      gcam[15] = fmaf(dJ[0], zi, fmaf(-dJ[2], g.xc * zi2, gu[0] * (g.pc[0] * zi)));
      gcam[16] = fmaf(dJ[4], zi, fmaf(-dJ[5], g.yc * zi2, gu[1] * (g.pc[1] * zi)));
      gcam[17] = gu[0];
      gcam[18] = gu[1];
    }
  } else {
    // ORTHO / FISHEYE: u has the exact Jacobian J (no clamp), and the cov2d term goes through dJ/dpc
    // (0 for ORTHO, whose J is constant).  OPENCV: u's Jacobian is the unclamped Ju, cov2d's the clamped J.
    const float *J = g.L.J;
    if constexpr (MODEL == FISHEYE || MODEL == OPENCV) {
      lens_dJ_dpc<MODEL>(g.pc, cam, g.L, dJ, gpc);
    } else {
      gpc[0] = gpc[1] = gpc[2] = 0.f;
    }
    const float *Ju = MODEL == OPENCV ? g.L.Ju : J;
    for (int k = 0; k < 3; k++) gpc[k] = fmaf(gu[0], Ju[k], fmaf(gu[1], Ju[3 + k], gpc[k]));
    if (DEPTH) gpc[2] += gdepth;
    for (int j = 0; j < 3; j++) gpw[j] += gpc[0] * R[j] + gpc[1] * R[3 + j] + gpc[2] * R[6 + j];
    if (POSE) {
      // dL/dRcw = gpc (x) pw + J^T dL/dM
      for (int a2 = 0; a2 < 3; a2++)
        for (int k = 0; k < 3; k++)
          gcam[3 * a2 + k] = fmaf(gpc[a2], pw[k], fmaf(J[a2], dM[k], J[3 + a2] * dM[3 + k]));
      for (int k = 0; k < 3; k++) gcam[9 + k] = gpc[k];
    }
    if (INTR) lens_dintr<MODEL>(g.pc, cam, g.L, dJ, gu, gcam + 15);
  }
  // cov3d: dL/dM3 = 2 sym(g3) M3
  const float G3[9] = {g3[0], 0.5f * g3[1], 0.5f * g3[2], 0.5f * g3[1], g3[3], 0.5f * g3[4],
                       0.5f * g3[2], 0.5f * g3[4], g3[5]};
  float dM3[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      dM3[3 * i + j] = 2.f * (G3[3 * i] * g.M3[j] + G3[3 * i + 1] * g.M3[3 + j] + G3[3 * i + 2] * g.M3[6 + j]);
  for (int j = 0; j < 3; j++) gs[j] = g.R3[j] * dM3[j] + g.R3[3 + j] * dM3[3 + j] + g.R3[6 + j] * dM3[6 + j];
  float dR[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) dR[3 * i + j] = dM3[3 * i + j] * s[j];
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  // dR/dq (halved; the factor 2 is applied at the end)
  gq[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
  gq[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - w * dR[5] + z * dR[6] + w * dR[7] - 2.f * x * dR[8]);
  gq[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + w * dR[2] + x * dR[3] + z * dR[5] - w * dR[6] + z * dR[7] - 2.f * y * dR[8]);
  gq[3] = 2.f * (-2.f * z * dR[0] - w * dR[1] + x * dR[2] + w * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
  return galpha_raw;
}

// ---- Mip-Splatting's 3D smoothing filter (filter3d.cu).  A training camera row is 20 floats:
// Rcw (row-major 9), tcw (3), fx, fy, cx, cy, W, H, 2 pad (kCamRow).  Camera k sees a Gaussian
// when camera_point keeps it (z >= kMinDepth, the rasterizers' cull) and its projected mean lies
// within 15 % of the frame on every side.  Mip-Splatting's compute_3D_filter projects with
// cx = W/2, cy = H/2 and culls z > 0.2; this uses the camera's own cx, cy and the z >= 0.2f cull.
constexpr int kCamRow = 20;
constexpr float kFilterMargin = 0.15f;

// true when the camera `c` (one row) sees pw; z = its camera-frame depth then
GSB_HD bool filter3d_sees(const float *c, const float pw[3], float &z) {
  float pc[3];
  if (!camera_point(c, c + 9, pw, pc)) return false;
  float u[2];
  project_mean(pc, 1.0f / pc[2], c[12], c[13], c[14], c[15], u);
  const float W = c[16], H = c[17];
  z = pc[2];
  return u[0] >= -kFilterMargin * W && u[0] <= (1.0f + kFilterMargin) * W && u[1] >= -kFilterMargin * H &&
         u[1] <= (1.0f + kFilterMargin) * H;
}

// filter3d = sqrt(variance) d / f_max, with d the nearest depth at which a camera sees the Gaussian
GSB_HD float filter3d_value(float d, float fmax, float variance) { return sqrtf(variance) * d / fmax; }

// Apply: s'_j = sqrt(s_j^2 + f^2), t_j = s_j / s'_j, alpha' = c alpha with c = t_0 t_1 t_2 (the
// filtered Gaussian keeps the mass alpha prod s).  f == 0 passes s through and returns c = 1
// exactly (s = f = 0 divides nothing).  t[3] receives t_j (1 when f == 0).
GSB_HD float filter3d_apply(const float s[3], float f, float sf[3], float t[3]) {
  if (f == 0.f) {
    for (int j = 0; j < 3; j++) { sf[j] = s[j]; t[j] = 1.f; }
    return 1.f;
  }
  const float f2 = f * f;
  for (int j = 0; j < 3; j++) {
    sf[j] = sqrtf(fmaf(s[j], s[j], f2));
    t[j] = s[j] / sf[j];
  }
  return t[0] * t[1] * t[2];
}

// Backward of filter3d_apply (f is a constant):
//   dL/ds_j = dL/ds'_j t_j + alpha dL/dalpha' (prod_{k != j} t_k) f^2 / s'_j^3,   dL/dalpha = c dL/dalpha'
// with f^2 / s'^3 evaluated as (f / s')^2 / s' (no underflow of s'^3).  f == 0 passes both through.
// gs may alias gsf (row-private in-place update).  Returns dL/dalpha.
GSB_HD float filter3d_backward(const float s[3], float alpha, float f, const float gsf[3], float galpha_f,
                               float gs[3]) {
  if (f == 0.f) {
    for (int j = 0; j < 3; j++) gs[j] = gsf[j];
    return galpha_f;
  }
  float sf[3], t[3];
  const float c = filter3d_apply(s, f, sf, t);
  const float a = alpha * galpha_f;
  const float other[3] = {t[1] * t[2], t[0] * t[2], t[0] * t[1]};
  for (int j = 0; j < 3; j++) {
    const float q = f / sf[j];
    gs[j] = fmaf(gsf[j], t[j], a * other[j] * (q * q / sf[j]));
  }
  return c * galpha_f;
}

}  // namespace pg
}  // namespace gsb
