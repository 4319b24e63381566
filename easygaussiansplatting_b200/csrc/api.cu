// extern "C" entry points declared in include/gsplat_b200.h.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <initializer_list>
#include <mutex>
#include <vector>

#include "../../include/gsplat_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace gsb {

static thread_local char g_err[512] = "";

int set_cuda_error(cudaError_t e, const char *what, const char *file, int line) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) in %s at %s:%d", (int)e, cudaGetErrorString(e), what,
           file, line);
  return (int)e;
}
int set_arg_error(const char *msg) {
  snprintf(g_err, sizeof(g_err), "argument error: %s", msg);
  return -1;
}

// ---- profiling
static bool g_prof_on = false;
static long long g_launches[K_COUNT] = {0};
struct EvPair { cudaEvent_t a, b; };
static std::vector<EvPair> g_events[K_COUNT];
static std::mutex g_prof_mu;
static const char *const g_names[K_COUNT] = {"project", "computeCov3D", "computeCov2D", "sh2Color",
                                             "inverseCov2D", "rects+scan", "scan(unused)", "keys", "sort",
                                             "ranges", "pack_records", "draw", "draw_backward",
                                             "preprocess_forward", "preprocess_backward",
                                             "finalize_splat_grads", "gau_loss_forward", "gau_loss_backward",
                                             "small_bmm", "density_accumulate", "density_classify",
                                             "density_scan", "density_apply", "reset_alpha",
                                             "ply_rows_to_gs", "gs_to_params", "params_to_gs",
                                             "grad_reduce_broadcast", "sh_grad_expand", "filter3d",
                                             "filter3d_apply", "filter3d_backward", "surfel_forward_batch",
                                             "draw_surfel_batch", "draw_surfel_backward_batch",
                                             "surfel_backward_batch", "draw_2dgs_batch",
                                             "draw_2dgs_backward_batch", "rects+scan_batch",
                                             "preprocess_forward_batch", "preprocess_backward_batch",
                                             "draw_batch", "draw_rgbd_batch", "draw_backward_batch",
                                             "draw_backward_rgbd_batch", "kmeans_assign", "kmeans_update",
                                             "quantize", "dequantize", "density_apply_rows",
                                             "bilagrid_slice", "bilagrid_slice_backward", "bilagrid_tv",
                                             "draw_features", "draw_backward_features", "draw_stats",
                                             "draw_surfel_stats", "mcmc_scan",
                                             "mcmc_sample", "mcmc_relocate", "mcmc_grow", "mcmc_rows",
                                             "mcmc_noise", "tsdf_integrate", "tsdf_plan", "tsdf_emit",
                                             "surfel_forward", "draw_surfel",
                                             "draw_surfel_backward", "surfel_backward", "draw_2dgs",
                                             "draw_2dgs_backward", "draw_backward_abs",
                                             "draw_backward_rgbd_abs",
                                             "adam", "draw_rgbd",
                                             "draw_backward_rgbd"};

ProfScope::ProfScope(int id, cudaStream_t st) : id_(id), st_(st), stop_(nullptr) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_launches[id]++;
  if (g_prof_on) {
    EvPair e;
    if (cudaEventCreate(&e.a) == cudaSuccess && cudaEventCreate(&e.b) == cudaSuccess) {
      cudaEventRecord(e.a, st);
      stop_ = e.b;
      g_events[id].push_back(e);
    }
  }
}
ProfScope::~ProfScope() {
  if (stop_) cudaEventRecord(stop_, st_);
}

}  // namespace gsb

using namespace gsb;

#define GSB_REQUIRE(cond, msg) \
  do {                         \
    if (!(cond)) return set_arg_error(msg); \
  } while (0)

// shs.shape[1] / 3 of SH degrees 0 to 3
static bool sh_dim3_ok(int sh_dim3) { return sh_dim3 == 1 || sh_dim3 == 4 || sh_dim3 == 9 || sh_dim3 == 16; }

extern "C" {

int gsb_abi_version(void) { return GSB_ABI_VERSION; }
const char *gsb_last_error(void) { return g_err; }

int gsb_project(int N, const float *pws, const float *Rcw, const float *tcw, float fx, float fy,
                float cx, float cy, float *us, float *pcs, float *depths, float *du_dpcs,
                gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "project: N < 0");
  GSB_REQUIRE(N == 0 || (pws && Rcw && tcw && us && pcs && depths), "project: null pointer");
  return launch_project(N, pws, Rcw, tcw, fx, fy, cx, cy, us, pcs, depths, du_dpcs, (cudaStream_t)stream);
}

int gsb_compute_cov3d(int N, const float *rots, const float *scales, const float *depths,
                      float *cov3ds, float *dcov3d_drots, float *dcov3d_dscales, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "computeCov3D: N < 0");
  GSB_REQUIRE(N == 0 || (rots && scales && depths && cov3ds), "computeCov3D: null pointer");
  GSB_REQUIRE((dcov3d_drots == nullptr) == (dcov3d_dscales == nullptr),
              "computeCov3D: Jacobian outputs must be both set or both null");
  return launch_cov3d(N, rots, scales, depths, cov3ds, dcov3d_drots, dcov3d_dscales, (cudaStream_t)stream);
}

int gsb_compute_cov2d(int N, const float *cov3ds, const float *pcs, const float *Rcw,
                      const float *depths, float fx, float fy, float width, float height,
                      float *cov2ds, float *dcov2d_dcov3ds, float *dcov2d_dpcs, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "computeCov2D: N < 0");
  GSB_REQUIRE(N == 0 || (cov3ds && pcs && Rcw && depths && cov2ds), "computeCov2D: null pointer");
  GSB_REQUIRE((dcov2d_dcov3ds == nullptr) == (dcov2d_dpcs == nullptr),
              "computeCov2D: Jacobian outputs must be both set or both null");
  return launch_cov2d(N, cov3ds, pcs, Rcw, depths, fx, fy, width, height, cov2ds, dcov2d_dcov3ds,
                      dcov2d_dpcs, (cudaStream_t)stream);
}

int gsb_sh2color(int N, int sh_dim3, const float *shs, const float *pws, const float *twc,
                 float *colors, float *dcolor_dshs, float *dcolor_dpws, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "sh2Color: N < 0");
  GSB_REQUIRE(sh_dim3_ok(sh_dim3), "sh2Color: shs.shape[1]/3 must be 1, 4, 9 or 16");
  GSB_REQUIRE(N == 0 || (shs && pws && twc && colors), "sh2Color: null pointer");
  GSB_REQUIRE((dcolor_dshs == nullptr) == (dcolor_dpws == nullptr),
              "sh2Color: Jacobian outputs must be both set or both null");
  return launch_sh2color(N, sh_dim3, shs, pws, twc, colors, dcolor_dshs, dcolor_dpws, (cudaStream_t)stream);
}

int gsb_inverse_cov2d(int N, const float *cov2ds, float *depths, float *cinv2ds, int32_t *areas,
                      float *dcinv2d_dcov2ds, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "inverseCov2D: N < 0");
  GSB_REQUIRE(N == 0 || (cov2ds && depths && cinv2ds && areas), "inverseCov2D: null pointer");
  return launch_inv_cov2d(N, cov2ds, depths, cinv2ds, areas, dcinv2d_dcov2ds, (cudaStream_t)stream);
}

void gsb_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = on != 0;
}
int gsb_profile_kernels(void) { return (int)K_COUNT; }
const char *gsb_profile_kernel_name(int id) { return (id >= 0 && id < K_COUNT) ? g_names[id] : ""; }
long long gsb_profile_launches(int id) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (id >= 0 && id < K_COUNT) return g_launches[id];
  long long t = 0;
  for (int i = 0; i < K_COUNT; i++) t += g_launches[i];
  return t;
}
int gsb_profile_read(int id, double *ms_total, long long *timed_launches) {
  GSB_REQUIRE(id >= 0 && id < K_COUNT && ms_total && timed_launches, "profile_read: bad arguments");
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double tot = 0.0;
  long long cnt = 0;
  for (auto &e : g_events[id]) {
    float ms = 0.f;
    if (cudaEventSynchronize(e.b) == cudaSuccess && cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) {
      tot += ms;
      cnt++;
    }
    cudaEventDestroy(e.a);
    cudaEventDestroy(e.b);
  }
  g_events[id].clear();
  *ms_total = tot;
  *timed_launches = cnt;
  return 0;
}

static bool aligned(const void *p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// "<who>: <err>" as the argument error
static int arg_error(const char *who, const char *err) {
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", who, err);
  return set_arg_error(msg);
}

// OPENCV's clamp stretch c = r_u / r_d (DESIGN 3.19): r_d is the largest normalised distorted radius
// |((u - cx) / fx, (v - cy) / fy)| of the four image corners, r_u solves r (1 + k1 r^2 + k2 r^4) = r_d
// on [0, sqrt(rho_valid)) by bisection (sqrt(rho_valid) when r_d lies beyond the curve's maximum).
// Exactly 1 without radial terms; the tangential ones are left to the 1.3 margin.
static float opencv_stretch(const float k[4], float fx, float fy, float cx, float cy, float width, float height) {
  const double k1 = k[0], k2 = k[1];
  if (k1 == 0.0 && k2 == 0.0) return 1.f;
  double rd = 0.0;
  for (double u : {0.0, (double)width})
    for (double v : {0.0, (double)height}) rd = std::fmax(rd, std::hypot((u - cx) / fx, (v - cy) / fy));
  if (!(rd > 0.0)) return 1.f;
  const auto dist = [&](double r) { const double r2 = r * r; return r * (1.0 + r2 * (k1 + r2 * k2)); };
  // rho_valid: the smallest positive root of 1 + 3 k1 rho + 5 k2 rho^2
  double rv = INFINITY;
  if (k2 == 0.0) {
    if (k1 < 0.0) rv = -1.0 / (3.0 * k1);
  } else {
    const double b = 3.0 * k1, a = 5.0 * k2, disc = b * b - 4.0 * a;
    if (disc >= 0.0) {
      const double q = -0.5 * (b + std::copysign(std::sqrt(disc), b));
      for (double r : {q / a, 1.0 / q})
        if (r > 0.0) rv = std::fmin(rv, r);
    }
  }
  double lo = 0.0, hi;
  if (std::isfinite(rv)) {
    hi = std::sqrt(rv);
    if (dist(hi) <= rd) return (float)(hi / rd);
  } else {
    hi = rd;
    while (dist(hi) < rd) hi *= 2.0;
  }
  for (int it = 0; it < 200 && hi - lo > 1e-15 * hi; it++) {
    const double m = 0.5 * (lo + hi);
    (dist(m) < rd ? lo : hi) = m;
  }
  return (float)(0.5 * (lo + hi) / rd);
}

// ---- camera models (DESIGN 3.14, 3.19).  NULL or PINHOLE passes no CamLens: the kernels of the
// entry points without a model.  Sets sc.lens.
static int camera_lens(const char *who, const gsb_camera_model *cm, FusedScene &sc, CamLens &out) {
  sc.lens = nullptr;
  if (cm == nullptr) return 0;
  const bool fin = std::isfinite(cm->k[0]) && std::isfinite(cm->k[1]) && std::isfinite(cm->k[2]) &&
                   std::isfinite(cm->k[3]);
  const bool k0 = cm->k[0] == 0.f && cm->k[1] == 0.f && cm->k[2] == 0.f && cm->k[3] == 0.f;
  if (cm->model != GSB_CAMERA_PINHOLE && cm->model != GSB_CAMERA_ORTHO && cm->model != GSB_CAMERA_FISHEYE &&
      cm->model != GSB_CAMERA_OPENCV)
    return arg_error(who, "unknown camera model");
  if (!fin) return arg_error(who, "non-finite radial coefficient");
  if (cm->model != GSB_CAMERA_FISHEYE && cm->model != GSB_CAMERA_OPENCV && !k0)
    return arg_error(who, "radial coefficients are for the fisheye and opencv models only");
  if (cm->model != GSB_CAMERA_PINHOLE && !(sc.fx > 0.f && sc.fy > 0.f)) return arg_error(who, "fx and fy must be > 0");
  if (cm->model == GSB_CAMERA_OPENCV && !(sc.width > 0.f && sc.height > 0.f))
    return arg_error(who, "the opencv model needs width and height > 0");
  if (cm->model == GSB_CAMERA_PINHOLE) return 0;
  out.model = cm->model;
  for (int i = 0; i < 4; i++) out.k[i] = cm->k[i];
  out.stretch = cm->model == GSB_CAMERA_OPENCV
                    ? opencv_stretch(out.k, sc.fx, sc.fy, sc.cx, sc.cy, sc.width, sc.height)
                    : 1.f;
  sc.lens = &out;
  return 0;
}

// The fused forward behind its three entry points.  antialiased: alphas and alphas_eff are
// required; otherwise alphas and records go together.
static int preprocess_forward(const char *who, bool antialiased, const gsb_camera_model *camera_model, FusedScene sc,
                              const FusedFwd &f, gsb_stream_t stream) {
  CamLens cl;
  if (int rc = camera_lens(who, camera_model, sc, cl)) return rc;
  if (sc.N < 0) return arg_error(who, "N < 0");
  if (!antialiased && (f.alphas == nullptr) != (f.recs == nullptr))
    return arg_error(who, "alphas and records go together");
  if (!aligned(f.recs, 16)) return arg_error(who, "records misaligned");
  if (!sh_dim3_ok(sc.k3)) return arg_error(who, "shs.shape[1]/3 must be 1, 4, 9 or 16");
  if (!(sc.N == 0 || (sc.pws && sc.rots && sc.scales && sc.shs && sc.Rcw && sc.tcw && sc.twc && f.us && f.cinv2ds &&
                      f.colors && f.depths && f.areas && (!antialiased || (f.alphas && f.alphas_eff)))))
    return arg_error(who, "null pointer");
  return launch_preprocess_fwd(sc, f, (cudaStream_t)stream);
}

int gsb_preprocess_forward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                           const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                           float fy, float cx, float cy, float width, float height, float *us,
                           float *cinv2ds, float *colors, float *depths, int32_t *areas, const float *alphas,
                           void *records, gsb_stream_t stream) {
  return preprocess_forward("preprocess", false, nullptr,
                            {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                            {us, cinv2ds, colors, depths, areas, alphas, static_cast<Rec *>(records), nullptr}, stream);
}

int gsb_preprocess_forward_aa(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                              const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                              float fy, float cx, float cy, float width, float height, float *us, float *cinv2ds,
                              float *colors, float *depths, int32_t *areas, const float *alphas, void *records,
                              float *alphas_eff, gsb_stream_t stream) {
  return preprocess_forward("preprocess_aa", true, nullptr,
                            {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                            {us, cinv2ds, colors, depths, areas, alphas, static_cast<Rec *>(records), alphas_eff},
                            stream);
}

int gsb_preprocess_forward_model(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, float *us, float *cinv2ds,
                                 float *colors, float *depths, int32_t *areas, const float *alphas, void *records,
                                 float *alphas_eff, const gsb_camera_model *camera_model, gsb_stream_t stream) {
  return preprocess_forward("preprocess_model", alphas_eff != nullptr, camera_model,
                            {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                            {us, cinv2ds, colors, depths, areas, alphas, static_cast<Rec *>(records), alphas_eff},
                            stream);
}

// Which per-Gaussian outputs an entry point of the fused backward writes: dloss_dpws, dloss_dshs,
// dloss_dscales, dloss_drots and, with the moment rows, dloss_dus_out and dloss_dalphas_out.
enum class GradOutputs {
  kAll,        // all of them (plain and RGB-D); with the moment rows dloss_dshs may be NULL (gsb_sh_grad_expand)
  kAllOrNone,  // all of them, or none: the camera gradient only (pose)
  kNone,       // none: the gradients go to the exchange; with the moment rows dloss_dus_out still does (push)
};

// Every check the fused backward's entry points share: N, sh_dim3, the parameter and camera
// pointers, the upstream gradients (the moment rows with the forward's conics, or the plain dL/du,
// dL/dconic and dL/dcolor) and the per-Gaussian outputs `outs` asks for.  `who` prefixes the error
// message.  An entry point checks its own further arguments after this.
static int check_preprocess_backward(const char *who, GradOutputs outs, const FusedScene &sc, const FusedBwd &b) {
  const bool mom = b.mi.moments != nullptr;
  const bool all_but_shs = b.g_pws && b.g_scales && b.g_rots && (!mom || (b.mi.dus_out && b.mi.dalphas_out));
  const bool none = !b.g_pws && !b.g_shs && !b.g_scales && !b.g_rots && (!mom || (!b.mi.dus_out && !b.mi.dalphas_out));
  if (sc.N < 0) return arg_error(who, "N < 0");
  if (!sh_dim3_ok(sc.k3)) return arg_error(who, "shs.shape[1]/3 must be 1, 4, 9 or 16");
  if (sc.N == 0) return 0;
  if (!(sc.pws && sc.rots && sc.scales && sc.shs && sc.Rcw && sc.tcw && sc.twc)) return arg_error(who, "null pointer");
  if (!(mom ? b.mi.cinv2ds != nullptr : (b.g_us && b.g_cinv2ds && b.g_colors)))
    return arg_error(who, "null upstream gradient");
  if (outs == GradOutputs::kAll && !(all_but_shs && (mom || b.g_shs))) return arg_error(who, "null output");
  if (outs == GradOutputs::kAllOrNone && !((all_but_shs && b.g_shs) || none))
    return arg_error(who, "per-Gaussian outputs must be all set or all null");
  if (outs == GradOutputs::kNone && mom && !b.mi.dus_out) return arg_error(who, "null output");
  return 0;
}

// What an entry point of the fused backward requires beyond check_preprocess_backward
enum : unsigned { kNeedDepths = 1, kNeedCamera = 2, kNeedAlphas = 4, kNeedIntrinsics = 8 };

// The fused backward behind its five local entry points.  needs: the kNeed* the entry point
// requires; need_moments: NULL, or why it requires the moment rows (the refusal's text).
// dloss_dcamera (with its workspace): NULL, or also the camera gradient; then the per-Gaussian
// outputs may be all NULL (pose only).  kNeedIntrinsics: dloss_dintrinsics as well (DESIGN 3.23; the
// workspace then holds rows of 24 floats).
static int preprocess_backward(const char *who, unsigned needs, const char *need_moments,
                               const gsb_camera_model *camera_model, FusedScene sc, FusedBwd b, float *dloss_dcamera,
                               void *ws, size_t ws_bytes, gsb_stream_t stream, float *dloss_dintrinsics = nullptr) {
  CamLens cl;
  if (int rc = camera_lens(who, camera_model, sc, cl)) return rc;
  const int N = sc.N;
  if ((needs & kNeedDepths) && N > 0 && b.g_depths == nullptr) return arg_error(who, "null dloss_ddepths");
  const bool pose = dloss_dcamera != nullptr;
  const GradOutputs outs = (needs & kNeedCamera) || pose ? GradOutputs::kAllOrNone : GradOutputs::kAll;
  if (int rc = check_preprocess_backward(who, outs, sc, b)) return rc;
  if ((needs & kNeedCamera) && !pose) return arg_error(who, "null dloss_dcamera");
  if (need_moments && N != 0 && b.mi.moments == nullptr) return arg_error(who, need_moments);
  if ((needs & kNeedAlphas) && N != 0 && b.alphas == nullptr) return arg_error(who, "null alphas");
  const bool intr = needs & kNeedIntrinsics;
  if (intr && dloss_dintrinsics == nullptr) return arg_error(who, "null dloss_dintrinsics");
  const PoseOut po{dloss_dcamera, static_cast<float *>(ws), intr ? dloss_dintrinsics : nullptr};
  if (pose) {
    if (!aligned(ws, 16)) return arg_error(who, "workspace misaligned");
    if (!(ws_bytes >= (intr ? intrinsics_workspace_bytes(N) : pose_workspace_bytes(N)) && (N == 0 || ws != nullptr)))
      return arg_error(who, "workspace too small");
    // (N == 0 launches no per-Gaussian pass: only the camera gradient's zeros)
    b.po = &po;
  }
  return launch_preprocess_bwd(sc, b, (cudaStream_t)stream);
}

int gsb_preprocess_backward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                            const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                            float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                            const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                            float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                            const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                            gsb_stream_t stream) {
  return preprocess_backward("preprocessB", 0, nullptr, nullptr,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}},
                             nullptr, nullptr, 0, stream);
}

int gsb_preprocess_backward_rgbd(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                 const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                 float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                 const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                 const float *dloss_ddepths, gsb_stream_t stream) {
  return preprocess_backward("preprocessB_rgbd", kNeedDepths, nullptr, nullptr,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}, dloss_ddepths},
                             nullptr, nullptr, 0, stream);
}

size_t gsb_preprocess_backward_pose_workspace_bytes(int N) { return pose_workspace_bytes(N); }

int gsb_preprocess_backward_pose(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                 const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                 float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                 const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                 const float *dloss_ddepths, float *dloss_dcamera, void *ws, size_t ws_bytes,
                                 gsb_stream_t stream) {
  return preprocess_backward("preprocessB_pose", kNeedCamera, nullptr, nullptr,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}, dloss_ddepths},
                             dloss_dcamera, ws, ws_bytes, stream);
}

int gsb_preprocess_backward_aa(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                               const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                               float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                               const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                               float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                               const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                               const float *dloss_ddepths, const float *alphas, float *dloss_dcamera, void *ws,
                               size_t ws_bytes, gsb_stream_t stream) {
  return preprocess_backward("preprocessB_aa", kNeedAlphas, "antialiasing takes the moment rows", nullptr,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}, dloss_ddepths, alphas},
                             dloss_dcamera, ws, ws_bytes, stream);
}

int gsb_preprocess_backward_model(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                  const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                  float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                  const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                  float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                  const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                  const float *dloss_ddepths, const float *alphas, float *dloss_dcamera, void *ws,
                                  size_t ws_bytes, const gsb_camera_model *camera_model, gsb_stream_t stream) {
  return preprocess_backward("preprocessB_model", 0, "the camera models take the moment rows", camera_model,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}, dloss_ddepths, alphas},
                             dloss_dcamera, ws, ws_bytes, stream);
}

size_t gsb_preprocess_backward_intrinsics_workspace_bytes(int N) { return intrinsics_workspace_bytes(N); }

int gsb_preprocess_backward_intrinsics(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                       const float *shs, const float *Rcw, const float *tcw, const float *twc,
                                       float fx, float fy, float cx, float cy, float width, float height,
                                       const float *dloss_dus, const float *dloss_dcinv2ds, const float *dloss_dcolors,
                                       float *dloss_dpws, float *dloss_dshs, float *dloss_dscales, float *dloss_drots,
                                       const float *moments, const float *cinv2ds, float *dloss_dus_out,
                                       float *dloss_dalphas_out, const float *dloss_ddepths, const float *alphas,
                                       float *dloss_dcamera, float *dloss_dintrinsics, void *ws, size_t ws_bytes,
                                       const gsb_camera_model *camera_model, gsb_stream_t stream) {
  return preprocess_backward("preprocessB_intrinsics", kNeedCamera | kNeedIntrinsics,
                             "the intrinsics gradient takes the moment rows", camera_model,
                             {N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height},
                             {dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_dpws, dloss_dshs, dloss_dscales,
                              dloss_drots, {moments, cinv2ds, dloss_dus_out, dloss_dalphas_out}, dloss_ddepths, alphas},
                             dloss_dcamera, ws, ws_bytes, stream, dloss_dintrinsics);
}

// ---- Mip-Splatting 3D smoothing filter (filter3d.cu)
static_assert(F3_CHUNK == GSB_FILTER3D_CHUNK, "gsplat_b200.h and kernels.h disagree on the camera chunk");

size_t gsb_filter3d_workspace_bytes(int N, int C) {
  (void)N;
  (void)C;
  return filter3d_workspace_bytes();
}

int gsb_filter3d(int N, const float *pws, int C, const float *cams, float variance, float *filter3d, void *ws,
                 size_t ws_bytes, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && C >= 0, "filter3d: N < 0 or C < 0");
  GSB_REQUIRE(isfinite(variance) && variance >= 0.f, "filter3d: variance must be finite and >= 0");
  if (N == 0) return 0;
  GSB_REQUIRE(pws && filter3d && (C == 0 || cams), "filter3d: null pointer");
  GSB_REQUIRE(aligned(ws, 16), "filter3d: workspace misaligned");
  GSB_REQUIRE(ws != nullptr && ws_bytes >= filter3d_workspace_bytes(), "filter3d: workspace too small");
  return launch_filter3d(N, pws, C, cams, variance, filter3d, static_cast<unsigned int *>(ws), (cudaStream_t)stream);
}

int gsb_filter3d_apply(int N, const float *scales, const float *alphas, const float *filter3d, float *scales_f,
                       float *alphas_f, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "filter3d_apply: N < 0");
  GSB_REQUIRE(N == 0 || (scales && alphas && filter3d && scales_f && alphas_f), "filter3d_apply: null pointer");
  return launch_filter3d_apply(N, scales, alphas, filter3d, scales_f, alphas_f, (cudaStream_t)stream);
}

int gsb_filter3d_backward(int N, const float *scales, const float *alphas, const float *filter3d,
                          const float *dloss_dscales_f, const float *dloss_dalphas_f, float *dloss_dscales,
                          float *dloss_dalphas, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "filter3d_backward: N < 0");
  GSB_REQUIRE(N == 0 || (scales && alphas && filter3d && dloss_dscales_f && dloss_dalphas_f && dloss_dscales &&
                         dloss_dalphas),
              "filter3d_backward: null pointer");
  return launch_filter3d_bwd(N, scales, alphas, filter3d, dloss_dscales_f, dloss_dalphas_f, dloss_dscales,
                             dloss_dalphas, (cudaStream_t)stream);
}

int gsb_sh_grad_expand(int N, int sh_dim3, int V, const float *pws, const float *twcs, const float *dloss_dcolors,
                       float *dloss_dshs, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && V >= 1, "sh_grad_expand: bad N / V");
  GSB_REQUIRE(sh_dim3_ok(sh_dim3), "sh_grad_expand: sh_dim3 must be 1, 4, 9 or 16");
  GSB_REQUIRE(N == 0 || (pws && twcs && dloss_dcolors && dloss_dshs), "sh_grad_expand: null pointer");
  return launch_sh_expand(N, sh_dim3, V, pws, twcs, dloss_dcolors, dloss_dshs, (cudaStream_t)stream);
}

int gsb_small_bmm(long long batch, int m, int k, int n, const float *A, const float *B, int b_shared, float *C,
                  gsb_stream_t stream) {
  GSB_REQUIRE(batch >= 0 && m > 0 && k > 0 && n > 0, "small_bmm: bad shape");
  GSB_REQUIRE(batch == 0 || (A && B && C), "small_bmm: null pointer");
  return launch_small_bmm(batch, m, k, n, A, B, b_shared, C, (cudaStream_t)stream);
}

size_t gsb_gau_loss_workspace_bytes(int H, int W) { return gau_loss_workspace_bytes(H, W); }

int gsb_gau_loss(int H, int W, const float *image, const float *gt_image, float loss_lambda, float *loss_out,
                 float *dloss_dimage, void *ws, size_t ws_bytes, gsb_stream_t stream) {
  GSB_REQUIRE(H > 0 && W > 0, "gau_loss: bad H/W");
  GSB_REQUIRE(image && gt_image && loss_out && ws, "gau_loss: null pointer");
  GSB_REQUIRE(ws_bytes >= gau_loss_workspace_bytes(H, W), "gau_loss: workspace too small");
  return launch_gau_loss(H, W, image, gt_image, loss_lambda, loss_out, dloss_dimage, ws, (cudaStream_t)stream);
}

// The binning packs a Gaussian's tile rectangle into 16-bit fields: x1 == 65536 would wrap to 0
// and put its patches into the wrong tiles.
static bool grid_fits(int H, int W) {
  return ((int64_t)W + GSB_TILE - 1) / GSB_TILE <= GSB_MAX_GRID_TILES &&
         ((int64_t)H + GSB_TILE - 1) / GSB_TILE <= GSB_MAX_GRID_TILES;
}

// The frame cores below take `frames`: 0 for one camera, or the C >= 1 cameras of a batch (DESIGN
// 3.21), binned and drawn as one tall frame of their C N records.  A batch entry point passes its C
// through batch_frames, so that a C < 1 reaches check_frame as -1 and is refused there.
static int batch_frames(int C) { return C >= 1 ? C : -1; }

// the frame a core bins, sorts and draws: the single frame, or the batch's tall frame
struct Tall {
  int H, N;
};
static Tall tall_frame(int frames, int H, int N) {
  return frames > 0 ? Tall{batch_height(frames, H), frames * N} : Tall{H, N};
}

static int launch_bin_frames(int frames, int H, int W, int N, const float *us, float *depths, int32_t *areas,
                             void *bin_ws, const BinLayout &L, cudaStream_t st) {
  return frames > 0 ? launch_bin_batch(frames, H, W, N, us, depths, areas, bin_ws, L, st)
                    : launch_bin(H, W, N, us, depths, areas, bin_ws, L, st);
}

// The checks of a frame every entry point that bins makes; `who` prefixes the error texts.  A batch
// also needs record ids c N + n that fit int32, and a tall frame of C gy tile rows that fits the
// rectangles' 16-bit fields.  bin_ws holds uint2 rectangles and 8-byte look-back descriptors of the
// frame's records (the entry points that do not pass its size pass SIZE_MAX).
static int check_frame(const char *who, int frames, int H, int W, int N, const void *bin_ws, size_t bin_ws_bytes) {
  if (frames < 0) return arg_error(who, "C < 1");
  if (!(N >= 0 && H > 0 && W > 0)) return arg_error(who, "bad N/H/W");
  if ((int64_t)frames * N >= ((int64_t)1 << 31)) return arg_error(who, "C N >= 2^31 records");
  if (!grid_fits(H, W) || (int64_t)frames * ((H + GSB_TILE - 1) / GSB_TILE) > GSB_MAX_GRID_TILES)
    return arg_error(who, frames > 0 ? "more than 65535 tiles in a row or in the C frames' column"
                                     : "more than 65535 tiles in a row or column");
  if (!aligned(bin_ws, 16)) return arg_error(who, "bin_ws misaligned");
  if (bin_ws_bytes < bin_layout(tall_frame(frames, H, N).N).bytes) return arg_error(who, "bin workspace too small");
  return 0;
}

// gsb_splat_bin{,_batch}: the frame's binning, its patch count and largest depth key read back
static int splat_bin(const char *who, int frames, int H, int W, int N, const float *us, float *depths, int32_t *areas,
                     void *bin_ws, size_t bin_ws_bytes, int64_t *P_host, uint32_t *depth_key_max_host,
                     gsb_stream_t stream) {
  if (int rc = check_frame(who, frames, H, W, N, bin_ws, bin_ws_bytes)) return rc;
  if (!(P_host != nullptr && bin_ws != nullptr)) return arg_error(who, "null workspace / P_host");
  if (N > 0 && !(us && depths && areas)) return arg_error(who, "null pointer");
  const BinLayout L = bin_layout(tall_frame(frames, H, N).N);
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = launch_bin_frames(frames, H, W, N, us, depths, areas, bin_ws, L, st)) return rc;
  uint32_t total[3] = {0, 0, 0};  // [patch count, largest depth key, flags]
  GSB_CUDA_TRY(cudaMemcpyAsync(total, static_cast<char *>(bin_ws) + L.total, 3 * sizeof(uint32_t),
                               cudaMemcpyDeviceToHost, st));
  GSB_CUDA_TRY(cudaStreamSynchronize(st));
  if ((total[2] & GSB_STATUS_TOO_MANY_PATCHES) != 0 || total[0] >= (1u << 30))
    return arg_error(who, "more than 2^30 patches");
  *P_host = (int64_t)total[0];
  if (depth_key_max_host) *depth_key_max_host = total[1];
  return 0;
}

size_t gsb_splat_bin_workspace_bytes(int N) { return bin_layout(N).bytes; }

int gsb_splat_bin(int H, int W, int N, const float *us, float *depths, int32_t *areas, void *bin_ws,
                  size_t bin_ws_bytes, int64_t *P_host, uint32_t *depth_key_max_host, gsb_stream_t stream) {
  return splat_bin("splat", 0, H, W, N, us, depths, areas, bin_ws, bin_ws_bytes, P_host, depth_key_max_host, stream);
}

size_t gsb_splat_records_offset(int N, int H, int W, int64_t P) { return sort_layout(N, H, W, P).recs; }

size_t gsb_splat_workspace_bytes(int N, int H, int W, int64_t P) { return sort_layout(N, H, W, P).bytes; }

// The outputs every frame writes: the image planes [3,H,W], contrib and final_tau [H,W], the tile
// ranges [T,2] and the sorted patch list
struct FrameOut {
  float *image;
  int32_t *contrib;
  float *final_tau;
  int32_t *ranges, *gsid;
};

// The draw step of the colour frame and, with both planes, of the RGB-D frame: the records are
// packed_records, or those the sort packed into ws (ws_recs).
struct ColourDraw {
  const void *packed_records;
  float *depth_image, *alpha_image;
  int frames = 0;  // > 0: the planes are [frames, ..., H, W] of a batch (launch_draw)

  int check() const {
    // RGB-D frames (the *_rgbd entry points pass both planes, written like the image planes)
    GSB_REQUIRE((depth_image == nullptr) == (alpha_image == nullptr), "splat: depth_image and alpha_image go together");
    GSB_REQUIRE(aligned(depth_image, 16) && aligned(alpha_image, 16), "splat: misaligned depth_image / alpha_image");
    GSB_REQUIRE(aligned(packed_records, 16), "splat: packed_records misaligned");
    return 0;
  }
  int draw(int H, int W, int, int64_t P, const FrameOut &o, const void *ws_recs, int *work, cudaStream_t st) const {
    const Rec *recs = static_cast<const Rec *>(packed_records ? packed_records : ws_recs);
    // with P == 0 (or N == 0) every tile is empty: the rasterizer only writes zeros
    return launch_draw(H, W, o.ranges, P > 0 ? recs : nullptr, o.gsid, o.image, o.contrib, o.final_tau, depth_image,
                       alpha_image, work, st, frames);
  }
};

extern "C++" {  // (templates)

// A binned frame from the sort to its planes, shared by every way of rendering one: P is the patch
// count (gsb_splat_render, gsb_splat_surfel_render) or its capacity (the *_forward entry points).
// With `sr` (the capacity path) the frame is binned here first, after every argument has been
// checked, and its status is copied to sr->host behind the keys.  `who` prefixes the error texts;
// the sort packs the 48-byte records into ws when `pack`; `draw` checks the planes and records of
// its frame family (draw.check()) and draws them (draw.draw()).
template <class Draw>
static int render_frame(const char *who, int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                        const float *cinv2ds, const float *alphas, float *depths, const float *colors, int32_t *areas,
                        bool pack, void *bin_ws, void *ws, size_t ws_bytes, const FrameOut &o, const Draw &draw,
                        const StatusRead *sr, cudaStream_t st, int frames = 0) {
  if (!(o.image && o.contrib && o.final_tau && o.ranges)) return arg_error(who, "null output");
  // the rasterizers write the image planes with 16-byte stores and the binning writes the tile
  // ranges as 8-byte pairs; these are outputs a caller allocates fresh (gsplat_b200.h)
  if (!(aligned(o.image, 16) && aligned(o.contrib, 16) && aligned(o.final_tau, 16) && aligned(o.ranges, 8)))
    return arg_error(who, "misaligned output");
  if (int rc = draw.check()) return rc;
  // 64-bit keys at ws + 0, records gathered 16 bytes at a time (the layout's offsets are 256-B multiples)
  if (!aligned(ws, 16)) return arg_error(who, "ws misaligned");
  // a batch's sort is the single frame's at the tall frame's height
  const Tall t = tall_frame(frames, H, N);
  const SortLayout SL = sort_layout(t.N, t.H, W, P);
  if (!(ws != nullptr && ws_bytes >= SL.bytes)) return arg_error(who, "workspace too small");
  const BinLayout BL = bin_layout(t.N);
  int rc = sr ? launch_bin_frames(frames, H, W, N, us, depths, areas, bin_ws, BL, st) : 0;
  if (rc) return rc;
  rc = launch_sort_and_pack(t.H, W, t.N, P, depth_key_max, us, cinv2ds, alphas, depths, colors, bin_ws, BL, ws, SL,
                            o.ranges, o.gsid, pack, sr, st);
  if (rc) return rc;
  char *b = static_cast<char *>(ws);
  return draw.draw(H, W, t.N, P, o, b + SL.recs, reinterpret_cast<int *>(b + SL.counters), st);
}

// The status event of the capacity path, one per host thread
static thread_local cudaEvent_t g_status_ready = nullptr;

// The capacity path's wait, shared by gsb_splat_forward{,_rgbd,_enqueue} and gsb_splat_surfel_forward:
// frame(sr) checks and queues the frame (render_frame with `sr`).  With `wait` status_host is zeroed
// first, and then the binning's status is waited for and judged; without it (CUDA graph capture)
// the caller inspects status_host later.  `who` prefixes the verdict's texts.
template <class Frame>
static int capacity_wait(const char *who, int64_t P_cap, uint32_t *status_host, bool wait, const Frame &frame) {
  if (wait && g_status_ready == nullptr)
    GSB_CUDA_TRY(cudaEventCreateWithFlags(&g_status_ready, cudaEventDisableTiming));
  const StatusRead sr{status_host, wait ? g_status_ready : nullptr};
  if (wait) status_host[0] = status_host[1] = status_host[2] = 0;
  const int rc = frame(&sr);
  if (rc || !wait) return rc;
  // the sort and the rasterizer are queued; now look at what the binning found (N == 0: nothing
  // was copied, the zeros stand)
  GSB_CUDA_TRY(cudaEventSynchronize(sr.ready));
  const uint32_t P = status_host[0], flags = status_host[2];
  if ((flags & GSB_STATUS_TOO_MANY_PATCHES) != 0 || P >= (1u << 30)) return arg_error(who, "more than 2^30 patches");
  if ((flags & (GSB_STATUS_P_CAP | GSB_STATUS_DEPTH_KEY)) != 0 || (int64_t)P > P_cap) {
    snprintf(g_err, sizeof(g_err), "%s_forward: capacity exceeded (P = %u of %lld, flags %u)", who, P,
             (long long)P_cap, flags);
    return GSB_CAPACITY_EXCEEDED;
  }
  return 0;
}

}  // extern "C++"

// gsb_splat_render{,_rgbd} and their batch forms: a frame binned by gsb_splat_bin{,_batch}
static int splat_render(const char *who, int frames, int H, int W, int N, int64_t P, uint32_t depth_key_max,
                        const float *us, const float *cinv2ds, const float *alphas, const float *depths,
                        const float *colors, const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes,
                        float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                        int32_t *gsid_per_patch, float *depth_image, float *alpha_image, gsb_stream_t stream) {
  if (int rc = check_frame(who, frames, H, W, N, bin_ws, SIZE_MAX)) return rc;
  if (P < 0) return arg_error(who, "bad P");
  if (P >= ((int64_t)1 << 30)) return arg_error(who, "more than 2^30 patches");
  if (P > 0 && !(us && cinv2ds && alphas && depths && colors && bin_ws && ws && gsid_per_patch))
    return arg_error(who, "null pointer");
  // (without `sr` nothing is binned: depths and bin_ws are only read)
  return render_frame(who, H, W, N, P, depth_key_max, us, cinv2ds, alphas, const_cast<float *>(depths), colors,
                      nullptr, packed_records == nullptr, const_cast<void *>(bin_ws), ws, ws_bytes,
                      {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                      ColourDraw{packed_records, depth_image, alpha_image, frames}, nullptr, (cudaStream_t)stream,
                      frames);
}

int gsb_splat_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                     const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                     const void *packed_records, const void *bin_ws,
                     void *ws, size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                     int32_t *patch_range_per_tile, int32_t *gsid_per_patch, gsb_stream_t stream) {
  return splat_render("splat", 0, H, W, N, P, depth_key_max, us, cinv2ds, alphas, depths, colors, packed_records,
                      bin_ws, ws, ws_bytes, image, contrib, final_tau, patch_range_per_tile, gsid_per_patch, nullptr,
                      nullptr, stream);
}

int gsb_splat_render_rgbd(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                          const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                          const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes, float *image,
                          int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                          float *depth_image, float *alpha_image, gsb_stream_t stream) {
  GSB_REQUIRE(depth_image && alpha_image, "splat_rgbd: null depth_image / alpha_image");
  return splat_render("splat", 0, H, W, N, P, depth_key_max, us, cinv2ds, alphas, depths, colors, packed_records,
                      bin_ws, ws, ws_bytes, image, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                      depth_image, alpha_image, stream);
}

// gsb_splat_forward{,_rgbd,_enqueue} and the batch forms: the capacity path.  `who` prefixes the
// frame's error texts and `fwd` those of the capacity checks; `wait` as capacity_wait's.
static int splat_forward(const char *who, const char *fwd, int frames, int H, int W, int N, const float *us,
                         const float *cinv2ds, const float *alphas, float *depths, const float *colors, int32_t *areas,
                         const void *packed_records, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                         size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                         float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                         uint32_t *status_host, float *depth_image, float *alpha_image, gsb_stream_t stream,
                         bool wait) {
  if (int rc = check_frame(who, frames, H, W, N, bin_ws, bin_ws_bytes)) return rc;
  if (!(P_cap > 0 && P_cap < ((int64_t)1 << 30)))
    return arg_error(fwd, frames > 0 ? "bad P_cap (2^30 patches or more)" : "bad P_cap");
  if (!(gsid_per_patch && status_host && bin_ws)) return arg_error(fwd, "null pointer");
  if (N > 0 && !(us && cinv2ds && alphas && depths && colors && areas)) return arg_error(fwd, "null pointer");
  return capacity_wait(who, P_cap, status_host, wait, [&](const StatusRead *sr) {
    return render_frame(who, H, W, N, P_cap, depth_key_cap, us, cinv2ds, alphas, depths, colors, areas,
                        packed_records == nullptr, bin_ws, ws, ws_bytes,
                        {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                        ColourDraw{packed_records, depth_image, alpha_image, frames}, sr, (cudaStream_t)stream,
                        frames);
  });
}

int gsb_splat_forward(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                      float *depths, const float *colors, int32_t *areas, const void *packed_records,
                      int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                      size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                      int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                      gsb_stream_t stream) {
  return splat_forward("splat", "splat_forward", 0, H, W, N, us, cinv2ds, alphas, depths, colors, areas,
                       packed_records, P_cap, depth_key_cap, bin_ws, bin_ws_bytes, ws, ws_bytes, image, contrib,
                       final_tau, patch_range_per_tile, gsid_per_patch, status_host, nullptr, nullptr, stream, true);
}

int gsb_splat_forward_rgbd(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                           float *depths, const float *colors, int32_t *areas, const void *packed_records,
                           int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                           size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                           int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                           float *depth_image, float *alpha_image, gsb_stream_t stream) {
  GSB_REQUIRE(depth_image && alpha_image, "splat_forward_rgbd: null depth_image / alpha_image");
  return splat_forward("splat", "splat_forward", 0, H, W, N, us, cinv2ds, alphas, depths, colors, areas,
                       packed_records, P_cap, depth_key_cap, bin_ws, bin_ws_bytes, ws, ws_bytes, image, contrib,
                       final_tau, patch_range_per_tile, gsid_per_patch, status_host, depth_image, alpha_image, stream,
                       true);
}

int gsb_splat_forward_enqueue(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                              float *depths, const float *colors, int32_t *areas, const void *packed_records,
                              int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                              size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                              int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                              gsb_stream_t stream) {
  return splat_forward("splat", "splat_forward", 0, H, W, N, us, cinv2ds, alphas, depths, colors, areas,
                       packed_records, P_cap, depth_key_cap, bin_ws, bin_ws_bytes, ws, ws_bytes, image, contrib,
                       final_tau, patch_range_per_tile, gsid_per_patch, status_host, nullptr, nullptr, stream, false);
}

// (a ws at any address: the size is the split from the worst start, 255 bytes short of a 256-B boundary)
size_t gsb_splat_backward_workspace_bytes(int N, int H, int W, int64_t P) { return bwd_layout(N, H, W, P, 1).bytes; }

// gsb_splat_backward, its RGB-D (dg; depths: the re-pack's depth words) and AbsGS forms, and the batch
// forms: the moment rows into moments_out, or (one frame only) with moments_out NULL finalised into
// dloss_dus .. dloss_dcolors.  The records are packed_records or re-packed into ws.
static int splat_backward(const char *who, int frames, int H, int W, int N, int64_t P, const float *us,
                          const float *cinv2ds, const float *alphas, const float *colors, const float *depths,
                          const int32_t *contrib, const float *final_tau, const int32_t *patch_range_per_tile,
                          const int32_t *gsid_per_patch, const float *dloss_dgammas, const DepthGrads *dg,
                          const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus,
                          float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, float *moments_out,
                          float *dloss_dus_abs, gsb_stream_t stream) {
  if (frames != 0) {
    if (int rc = check_frame(who, frames, H, W, N, nullptr, SIZE_MAX)) return rc;
    if (P < 0) return arg_error(who, "bad P");
  } else {
    if (!(N >= 0 && H > 0 && W > 0 && P >= 0)) return arg_error(who, "bad N/H/W/P");
    if (!grid_fits(H, W)) return arg_error(who, "more than 65535 tiles in a row or column");
  }
  if (P >= ((int64_t)1 << 30)) return arg_error(who, "more than 2^30 patches");
  // (a batch has only the moment rows)
  if (N > 0 && !(moments_out || (dloss_dus && dloss_dcinv2ds && dloss_dalphas && dloss_dcolors)))
    return arg_error(who, frames != 0 ? "null pointer" : "null output");
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return 0;
  if (!(cinv2ds && ws)) return arg_error(who, "null pointer");
  // with the forward's records handed in, the workspace only has to hold the moment rows
  const Tall t = tall_frame(frames, H, N);
  const int64_t P_ws = packed_records != nullptr ? 0 : P;
  if (ws_bytes < bwd_layout(t.N, t.H, W, P_ws, 1).bytes) return arg_error(who, "workspace too small");
  char *b = static_cast<char *>(ws);
  const BwdLayout L = bwd_layout(t.N, t.H, W, P_ws, reinterpret_cast<uintptr_t>(ws));
  Rec *recs = reinterpret_cast<Rec *>(b + L.recs);
  float *moments = moments_out != nullptr ? moments_out : reinterpret_cast<float *>(b + L.moments);
  int *work = reinterpret_cast<int *>(b + L.work);
  if (P > 0) {
    if (!(us && alphas && colors && contrib && final_tau && patch_range_per_tile && gsid_per_patch && dloss_dgammas))
      return arg_error(who, "null pointer");
    // (the one-frame RGB-D entry points check dloss_ddepths themselves)
    if (dg != nullptr && !(depths && dg->dloss_ddepth_image && dg->dloss_dalpha_image && dg->ddepths))
      return arg_error(frames != 0 ? who : "splatB_rgbd", "null pointer");
    if (!aligned(packed_records, 16)) return arg_error(who, "packed_records misaligned");
    if (packed_records != nullptr) {  // the forward's record stream is still valid: skip the re-pack
      recs = const_cast<Rec *>(static_cast<const Rec *>(packed_records));
    } else if (int rc = launch_pack_only(t.N, nullptr, us, cinv2ds, alphas, colors, depths, recs, st)) {
      return rc;
    }
  } else if (dg != nullptr && dg->ddepths == nullptr) {
    return arg_error(who, "null pointer");
  }
  // P == 0: nothing was drawn; the zeroed moment rows finalise to all-zero gradients
  return launch_draw_backward(H, W, t.N, patch_range_per_tile, P > 0 ? recs : nullptr, gsid_per_patch, contrib,
                              final_tau, dloss_dgammas, dg, cinv2ds, moments, work, dloss_dus, dloss_dcinv2ds,
                              dloss_dalphas, dloss_dcolors, moments_out == nullptr, dloss_dus_abs, st, frames);
}

int gsb_splat_backward(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                       const float *alphas, const float *colors, const int32_t *contrib,
                       const float *final_tau, const int32_t *patch_range_per_tile,
                       const int32_t *gsid_per_patch, const float *dloss_dgammas,
                       const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus, float *dloss_dcinv2ds, float *dloss_dalphas,
                       float *dloss_dcolors, float *moments_out, gsb_stream_t stream) {
  // (the re-pack leaves the records' depth word 0: k_draw_bwd never reads it)
  return splat_backward("splatB", 0, H, W, N, P, us, cinv2ds, alphas, colors, nullptr, contrib, final_tau,
                        patch_range_per_tile, gsid_per_patch, dloss_dgammas, nullptr, packed_records, ws, ws_bytes,
                        dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors, moments_out, nullptr, stream);
}

int gsb_splat_backward_rgbd(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                            const float *alphas, const float *colors, const float *depths, const int32_t *contrib,
                            const float *final_tau, const int32_t *patch_range_per_tile,
                            const int32_t *gsid_per_patch, const float *dloss_dgammas,
                            const float *dloss_ddepth_image, const float *dloss_dalpha_image,
                            const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus,
                            float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, float *moments_out,
                            float *dloss_ddepths, gsb_stream_t stream) {
  GSB_REQUIRE(N <= 0 || dloss_ddepths != nullptr, "splatB_rgbd: null dloss_ddepths");
  const DepthGrads dg{dloss_ddepth_image, dloss_dalpha_image, dloss_ddepths};
  return splat_backward("splatB", 0, H, W, N, P, us, cinv2ds, alphas, colors, depths, contrib, final_tau,
                        patch_range_per_tile, gsid_per_patch, dloss_dgammas, &dg, packed_records, ws, ws_bytes,
                        dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors, moments_out, nullptr, stream);
}

int gsb_splat_backward_abs(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                           const float *alphas, const float *colors, const int32_t *contrib, const float *final_tau,
                           const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                           const float *dloss_dgammas, const void *packed_records, void *ws, size_t ws_bytes,
                           float *dloss_dus, float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors,
                           float *moments_out, float *dloss_dus_abs, gsb_stream_t stream) {
  GSB_REQUIRE(N <= 0 || dloss_dus_abs != nullptr, "splatB_abs: null dloss_dus_abs");
  return splat_backward("splatB", 0, H, W, N, P, us, cinv2ds, alphas, colors, nullptr, contrib, final_tau,
                        patch_range_per_tile, gsid_per_patch, dloss_dgammas, nullptr, packed_records, ws, ws_bytes,
                        dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors, moments_out, dloss_dus_abs, stream);
}

int gsb_splat_backward_rgbd_abs(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                                const float *alphas, const float *colors, const float *depths, const int32_t *contrib,
                                const float *final_tau, const int32_t *patch_range_per_tile,
                                const int32_t *gsid_per_patch, const float *dloss_dgammas,
                                const float *dloss_ddepth_image, const float *dloss_dalpha_image,
                                const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus,
                                float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, float *moments_out,
                                float *dloss_ddepths, float *dloss_dus_abs, gsb_stream_t stream) {
  GSB_REQUIRE(N <= 0 || dloss_dus_abs != nullptr, "splatB_rgbd_abs: null dloss_dus_abs");
  GSB_REQUIRE(N <= 0 || dloss_ddepths != nullptr, "splatB_rgbd: null dloss_ddepths");
  const DepthGrads dg{dloss_ddepth_image, dloss_dalpha_image, dloss_ddepths};
  return splat_backward("splatB", 0, H, W, N, P, us, cinv2ds, alphas, colors, depths, contrib, final_tau,
                        patch_range_per_tile, gsid_per_patch, dloss_dgammas, &dg, packed_records, ws, ws_bytes,
                        dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors, moments_out, dloss_dus_abs, stream);
}

// ---- batched rendering (DESIGN 3.21): C cameras of one image size and camera model, binned and drawn
// as one tall frame through the frame cores above; the per-Gaussian kernels run the C cameras in one launch.

// The batch call description: the per-camera intrinsics rows (fx, fy, cx, cy, k[4]) checked as
// camera_lens checks one camera, into the kernels' parameter table (tan_fov exactly as the
// single-camera path computes it), and the parameter and pose pointers.
static int batch_scene(const char *who, int C, int N, int sh_dim3, const float *pws, const float *rots,
                       const float *scales, const float *shs, const float *poses, int camera_model,
                       const float *intrinsics, float width, float height, BatchCams &bc, BatchScene &b) {
  if (C < 1) return arg_error(who, "C < 1");
  if (C > BATCH_MAX_CAMERAS) return arg_error(who, "C > GSB_BATCH_MAX_CAMERAS");
  if (N < 0) return arg_error(who, "N < 0");
  if ((int64_t)C * N >= ((int64_t)1 << 31)) return arg_error(who, "C N >= 2^31 records");
  if (!sh_dim3_ok(sh_dim3)) return arg_error(who, "shs.shape[1]/3 must be 1, 4, 9 or 16");
  if (intrinsics == nullptr) return arg_error(who, "null intrinsics");
  for (int c = 0; c < C; c++) {
    const float *r = intrinsics + (size_t)c * GSB_BATCH_INTRINSICS_ROW;
    const gsb_camera_model cm{camera_model, {r[4], r[5], r[6], r[7]}};
    FusedScene sc{N, sh_dim3};
    sc.fx = r[0]; sc.fy = r[1]; sc.cx = r[2]; sc.cy = r[3]; sc.width = width; sc.height = height;
    CamLens cl;
    if (int rc = camera_lens(who, &cm, sc, cl)) return rc;
    const float2 tf = lens_tan_fov(sc);
    bc.f[c] = make_float4(r[0], r[1], r[2], r[3]);
    bc.k[c] = make_float4(r[4], r[5], r[6], r[7]);
    bc.tf[c] = tf;
  }
  b.C = C; b.N = N; b.k3 = sh_dim3; b.model = camera_model; b.cams = &bc;
  b.pws = pws; b.rots = rots; b.scales = scales; b.shs = shs; b.poses = poses;
  return 0;
}

int gsb_preprocess_forward_batch(int C, int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *poses, const float *intrinsics, int camera_model,
                                 float width, float height, float *us, float *cinv2ds, float *colors, float *depths,
                                 int32_t *areas, const float *alphas, void *records, float *alphas_eff,
                                 gsb_stream_t stream) {
  const char *who = "preprocess_batch";
  BatchCams bc;
  BatchScene b{};
  if (int rc = batch_scene(who, C, N, sh_dim3, pws, rots, scales, shs, poses, camera_model, intrinsics, width, height,
                           bc, b))
    return rc;
  if (!aligned(records, 16)) return arg_error(who, "records misaligned");
  if (N > 0 && !(pws && rots && scales && shs && poses && us && cinv2ds && colors && depths && areas && alphas &&
                 records))
    return arg_error(who, "null pointer");
  return launch_preprocess_fwd_batch(b, {us, cinv2ds, colors, depths, areas, alphas, static_cast<Rec *>(records),
                                         alphas_eff},
                                     (cudaStream_t)stream);
}

// gsb_preprocess_backward_batch and, with `pose`, its camera gradients (DESIGN 3.22): then the
// per-Gaussian outputs may be all NULL (pose only).  intr (with pose): dloss_dintrinsics as well
// (DESIGN 3.23; the workspace then holds rows of 24 floats).
static int preprocess_backward_batch(const char *who, bool pose, int C, int N, int sh_dim3, const float *pws,
                                     const float *rots, const float *scales, const float *shs, const float *poses,
                                     const float *intrinsics, int camera_model, float width, float height,
                                     BatchBwd g, float *dloss_dposes, void *ws, size_t ws_bytes,
                                     gsb_stream_t stream, bool intr = false, float *dloss_dintrinsics = nullptr) {
  BatchCams bc;
  BatchScene b{};
  if (int rc = batch_scene(who, C, N, sh_dim3, pws, rots, scales, shs, poses, camera_model, intrinsics, width, height,
                           bc, b))
    return rc;
  if (N > 0 && !(pws && rots && scales && shs && poses && g.moments && g.cinv2ds)) return arg_error(who, "null pointer");
  const bool all = g.g_pws && g.g_shs && g.g_scales && g.g_rots && g.dus_out && g.dalphas_out;
  const bool none = !g.g_pws && !g.g_shs && !g.g_scales && !g.g_rots && !g.dus_out && !g.dalphas_out;
  if (!pose) {
    if (N > 0 && !all) return arg_error(who, "null output");
    return launch_preprocess_bwd_batch(b, g, (cudaStream_t)stream);
  }
  if (N > 0 && !all && !none) return arg_error(who, "per-Gaussian outputs must be all set or all null");
  if (dloss_dposes == nullptr) return arg_error(who, "null dloss_dposes");
  if (intr && dloss_dintrinsics == nullptr) return arg_error(who, "null dloss_dintrinsics");
  if (!aligned(ws, 16)) return arg_error(who, "workspace misaligned");
  const size_t need = intr ? batch_intrinsics_workspace_bytes(C, N) : batch_pose_workspace_bytes(C, N);
  if (!(ws_bytes >= need && (need == 0 || ws != nullptr))) return arg_error(who, "workspace too small");
  const PoseOut po{dloss_dposes, static_cast<float *>(ws), intr ? dloss_dintrinsics : nullptr};
  g.po = &po;
  // (N == 0 launches no per-Gaussian pass: only the C rows of zeros)
  return launch_preprocess_bwd_batch(b, g, (cudaStream_t)stream);
}

int gsb_preprocess_backward_batch(int C, int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                  const float *shs, const float *poses, const float *intrinsics, int camera_model,
                                  float width, float height, const float *moments, const float *cinv2ds,
                                  const float *dloss_ddepths, const float *alphas, float *dloss_dpws,
                                  float *dloss_dshs, float *dloss_dscales, float *dloss_drots, float *dloss_dus_out,
                                  float *dloss_dalphas_out, gsb_stream_t stream) {
  return preprocess_backward_batch("preprocessB_batch", false, C, N, sh_dim3, pws, rots, scales, shs, poses,
                                   intrinsics, camera_model, width, height,
                                   {moments, cinv2ds, dloss_ddepths, alphas, dloss_dus_out, dloss_dalphas_out,
                                    dloss_dpws, dloss_dshs, dloss_dscales, dloss_drots},
                                   nullptr, nullptr, 0, stream);
}

// The batch's workspace queries answer 0 for what its entry points refuse: C < 1, N < 0, C N >= 2^31
static bool batch_records_ok(int C, int N) { return C >= 1 && N >= 0 && (int64_t)C * N < ((int64_t)1 << 31); }

size_t gsb_preprocess_backward_batch_pose_workspace_bytes(int C, int N) {
  return batch_records_ok(C, N) ? batch_pose_workspace_bytes(C, N) : 0;
}

int gsb_preprocess_backward_batch_pose(int C, int N, int sh_dim3, const float *pws, const float *rots,
                                       const float *scales, const float *shs, const float *poses,
                                       const float *intrinsics, int camera_model, float width, float height,
                                       const float *moments, const float *cinv2ds, const float *dloss_ddepths,
                                       const float *alphas, float *dloss_dpws, float *dloss_dshs, float *dloss_dscales,
                                       float *dloss_drots, float *dloss_dus_out, float *dloss_dalphas_out,
                                       float *dloss_dposes, void *ws, size_t ws_bytes, gsb_stream_t stream) {
  return preprocess_backward_batch("preprocessB_batch_pose", true, C, N, sh_dim3, pws, rots, scales, shs, poses,
                                   intrinsics, camera_model, width, height,
                                   {moments, cinv2ds, dloss_ddepths, alphas, dloss_dus_out, dloss_dalphas_out,
                                    dloss_dpws, dloss_dshs, dloss_dscales, dloss_drots},
                                   dloss_dposes, ws, ws_bytes, stream);
}

size_t gsb_preprocess_backward_batch_intrinsics_workspace_bytes(int C, int N) {
  return batch_records_ok(C, N) ? batch_intrinsics_workspace_bytes(C, N) : 0;
}

int gsb_preprocess_backward_batch_intrinsics(int C, int N, int sh_dim3, const float *pws, const float *rots,
                                             const float *scales, const float *shs, const float *poses,
                                             const float *intrinsics, int camera_model, float width, float height,
                                             const float *moments, const float *cinv2ds, const float *dloss_ddepths,
                                             const float *alphas, float *dloss_dpws, float *dloss_dshs,
                                             float *dloss_dscales, float *dloss_drots, float *dloss_dus_out,
                                             float *dloss_dalphas_out, float *dloss_dposes, float *dloss_dintrinsics,
                                             void *ws, size_t ws_bytes, gsb_stream_t stream) {
  return preprocess_backward_batch("preprocessB_batch_intrinsics", true, C, N, sh_dim3, pws, rots, scales, shs, poses,
                                   intrinsics, camera_model, width, height,
                                   {moments, cinv2ds, dloss_ddepths, alphas, dloss_dus_out, dloss_dalphas_out,
                                    dloss_dpws, dloss_dshs, dloss_dscales, dloss_drots},
                                   dloss_dposes, ws, ws_bytes, stream, true, dloss_dintrinsics);
}

size_t gsb_splat_bin_batch_workspace_bytes(int C, int N) { return batch_records_ok(C, N) ? bin_layout(C * N).bytes : 0; }

int gsb_splat_bin_batch(int C, int H, int W, int N, const float *us, float *depths, int32_t *areas, void *bin_ws,
                        size_t bin_ws_bytes, int64_t *P_host, uint32_t *depth_key_max_host, gsb_stream_t stream) {
  return splat_bin("splat_bin_batch", batch_frames(C), H, W, N, us, depths, areas, bin_ws, bin_ws_bytes, P_host,
                   depth_key_max_host, stream);
}

size_t gsb_splat_batch_records_offset(int C, int N, int H, int W, int64_t P) {
  return batch_records_ok(C, N) ? sort_layout(C * N, batch_height(C, H), W, P).recs : 0;
}

size_t gsb_splat_batch_workspace_bytes(int C, int N, int H, int W, int64_t P) {
  return batch_records_ok(C, N) ? sort_layout(C * N, batch_height(C, H), W, P).bytes : 0;
}

int gsb_splat_render_batch(int C, int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                           const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                           const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes, float *image,
                           int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                           int32_t *gsid_per_patch, gsb_stream_t stream) {
  return splat_render("splat_batch", batch_frames(C), H, W, N, P, depth_key_max, us, cinv2ds, alphas, depths, colors,
                      packed_records, bin_ws, ws, ws_bytes, image, contrib, final_tau, patch_range_per_tile,
                      gsid_per_patch, nullptr, nullptr, stream);
}

int gsb_splat_render_batch_rgbd(int C, int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                                const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                                const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes,
                                float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                                int32_t *gsid_per_patch, float *depth_image, float *alpha_image, gsb_stream_t stream) {
  GSB_REQUIRE(depth_image && alpha_image, "splat_batch_rgbd: null depth_image / alpha_image");
  return splat_render("splat_batch_rgbd", batch_frames(C), H, W, N, P, depth_key_max, us, cinv2ds, alphas, depths,
                      colors, packed_records, bin_ws, ws, ws_bytes, image, contrib, final_tau, patch_range_per_tile,
                      gsid_per_patch, depth_image, alpha_image, stream);
}

int gsb_splat_forward_batch(int C, int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                            float *depths, const float *colors, int32_t *areas, const void *packed_records,
                            int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                            size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                            int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                            gsb_stream_t stream) {
  return splat_forward("splat_batch", "splat_batch", batch_frames(C), H, W, N, us, cinv2ds, alphas, depths, colors,
                       areas, packed_records, P_cap, depth_key_cap, bin_ws, bin_ws_bytes, ws, ws_bytes, image, contrib,
                       final_tau, patch_range_per_tile, gsid_per_patch, status_host, nullptr, nullptr, stream, true);
}

int gsb_splat_forward_batch_rgbd(int C, int H, int W, int N, const float *us, const float *cinv2ds,
                                 const float *alphas, float *depths, const float *colors, int32_t *areas,
                                 const void *packed_records, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                                 size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                                 float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                                 uint32_t *status_host, float *depth_image, float *alpha_image, gsb_stream_t stream) {
  GSB_REQUIRE(depth_image && alpha_image, "splat_batch_rgbd: null depth_image / alpha_image");
  return splat_forward("splat_batch_rgbd", "splat_batch_rgbd", batch_frames(C), H, W, N, us, cinv2ds, alphas, depths,
                       colors, areas, packed_records, P_cap, depth_key_cap, bin_ws, bin_ws_bytes, ws, ws_bytes, image,
                       contrib, final_tau, patch_range_per_tile, gsid_per_patch, status_host, depth_image,
                       alpha_image, stream, true);
}

size_t gsb_splat_backward_batch_workspace_bytes(int C, int N, int H, int W, int64_t P) {
  return batch_records_ok(C, N) ? bwd_layout(C * N, batch_height(C, H), W, P, 1).bytes : 0;
}

// the batch's backward rasterizer: the moment rows [C N, 9] (and dL/dz [C N]) for
// gsb_preprocess_backward_batch
int gsb_splat_backward_batch(int C, int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                             const float *alphas, const float *colors, const int32_t *contrib, const float *final_tau,
                             const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                             const float *dloss_dgammas, const void *packed_records, void *ws, size_t ws_bytes,
                             float *moments_out, gsb_stream_t stream) {
  return splat_backward("splatB_batch", batch_frames(C), H, W, N, P, us, cinv2ds, alphas, colors, nullptr, contrib,
                        final_tau, patch_range_per_tile, gsid_per_patch, dloss_dgammas, nullptr, packed_records, ws,
                        ws_bytes, nullptr, nullptr, nullptr, nullptr, moments_out, nullptr, stream);
}

int gsb_splat_backward_batch_rgbd(int C, int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                                  const float *alphas, const float *colors, const float *depths,
                                  const int32_t *contrib, const float *final_tau, const int32_t *patch_range_per_tile,
                                  const int32_t *gsid_per_patch, const float *dloss_dgammas,
                                  const float *dloss_ddepth_image, const float *dloss_dalpha_image,
                                  const void *packed_records, void *ws, size_t ws_bytes, float *moments_out,
                                  float *dloss_ddepths, gsb_stream_t stream) {
  const DepthGrads dg{dloss_ddepth_image, dloss_dalpha_image, dloss_ddepths};
  return splat_backward("splatB_batch_rgbd", batch_frames(C), H, W, N, P, us, cinv2ds, alphas, colors, depths,
                        contrib, final_tau, patch_range_per_tile, gsid_per_patch, dloss_dgammas, &dg, packed_records,
                        ws, ws_bytes, nullptr, nullptr, nullptr, nullptr, moments_out, nullptr, stream);
}

// ---- 2D Gaussian Splatting (surfel.cu, DESIGN 3.15)

static int surfel_scene(const char *who, FusedScene &sc) {
  sc.lens = nullptr;
  if (sc.N < 0) return arg_error(who, "N < 0");
  if (!sh_dim3_ok(sc.k3)) return arg_error(who, "shs.shape[1]/3 must be 1, 4, 9 or 16");
  if (sc.N > 0 && !(sc.pws && sc.rots && sc.scales && sc.shs && sc.Rcw && sc.tcw && sc.twc))
    return arg_error(who, "null pointer");
  return 0;
}

int gsb_surfel_preprocess_forward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                  const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                  float fy, float cx, float cy, float width, float height, const float *alphas,
                                  float *us, float *depths, int32_t *areas, float *colors, float *records,
                                  gsb_stream_t stream) {
  const char *who = "surfel_preprocess";
  FusedScene sc{N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height, nullptr};
  if (int rc = surfel_scene(who, sc)) return rc;
  if (!aligned(records, 16)) return arg_error(who, "records misaligned");
  if (N > 0 && !(alphas && us && depths && areas && colors && records)) return arg_error(who, "null pointer");
  return launch_surfel_fwd(sc, alphas, us, depths, areas, colors, records, (cudaStream_t)stream);
}

int gsb_surfel_preprocess_backward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                   const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                   float fy, float cx, float cy, float width, float height, const float *rows,
                                   float *dloss_dpws, float *dloss_dshs, float *dloss_dalphas, float *dloss_dscales,
                                   float *dloss_drots, float *dloss_dus, gsb_stream_t stream) {
  const char *who = "surfel_preprocessB";
  FusedScene sc{N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height, nullptr};
  if (int rc = surfel_scene(who, sc)) return rc;
  if (N > 0 && !(rows && dloss_dpws && dloss_dshs && dloss_dalphas && dloss_dscales && dloss_drots && dloss_dus))
    return arg_error(who, "null pointer");
  return launch_surfel_bwd(sc, rows, dloss_dpws, dloss_dshs, dloss_dalphas, dloss_dscales, dloss_drots, dloss_dus,
                           (cudaStream_t)stream);
}

size_t gsb_splat_surfel_workspace_bytes(int N, int H, int W, int64_t P) { return sort_layout(N, H, W, P).bytes; }

// The draw step of the surfel frame: its 80-byte records, its three further planes and, for the
// 2DGS geometry frame (gsb_splat_2dgs_*), the geometry planes
struct SurfelDraw {
  const float *records;
  float *depth_image, *alpha_image, *normal_image;
  const GeoPlanes *geo = nullptr;
  int frames = 0;  // > 0: the planes are [frames, ..., H, W] of a batch (launch_draw_surfel)

  int check() const {
    const char *who = geo ? "splat_2dgs" : "splat_surfel";
    if (!(depth_image && alpha_image && normal_image)) return arg_error(who, "null output");
    if (!(aligned(depth_image, 16) && aligned(alpha_image, 16) && aligned(normal_image, 16)))
      return arg_error(who, "misaligned output");
    if (!aligned(records, 16)) return arg_error(who, "records misaligned");
    return 0;
  }
  int draw(int H, int W, int N, int64_t P, const FrameOut &o, const void *, int *work, cudaStream_t st) const {
    return launch_draw_surfel(H, W, o.ranges, P > 0 && N > 0 ? records : nullptr, o.gsid, o.image, o.contrib,
                              o.final_tau, depth_image, alpha_image, normal_image, geo, work, st, frames);
  }
};

// near / far of the geometry planes: 0 < near < far, both finite
static int check_near_far(const char *who, float near, float far) {
  if (!(std::isfinite(near) && std::isfinite(far))) return arg_error(who, "near / far not finite");
  if (!(near > 0.f)) return arg_error(who, "near <= 0");
  if (!(far > near)) return arg_error(who, "far <= near");
  return 0;
}

// The geometry planes of a 2DGS frame, checked (who = "splat_2dgs"): every plane present and 16-byte aligned
static int geo_planes(const char *who, float near, float far, float *distortion, float *moments, float *median_depth,
                      int32_t *median_contrib, GeoPlanes &g) {
  if (int rc = check_near_far(who, near, far)) return rc;
  if (!(distortion && moments && median_depth && median_contrib)) return arg_error(who, "null geometry plane");
  if (!(aligned(distortion, 16) && aligned(moments, 16) && aligned(median_depth, 16) && aligned(median_contrib, 16)))
    return arg_error(who, "misaligned geometry plane");
  g = GeoPlanes{distortion, moments, median_depth, median_contrib, near, (float)((double)far / ((double)far - near))};
  return 0;
}

int gsb_splat_surfel_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                            const float *depths, const float *records, const void *bin_ws, void *ws, size_t ws_bytes,
                            float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                            int32_t *gsid_per_patch, float *depth_image, float *alpha_image, float *normal_image,
                            gsb_stream_t stream) {
  int rc = check_frame("splat", 0, H, W, N, bin_ws, SIZE_MAX);
  if (rc) return rc;
  GSB_REQUIRE(P >= 0, "splat_surfel: bad P");
  GSB_REQUIRE(P == 0 || (us && depths && records && bin_ws && ws && gsid_per_patch), "splat_surfel: null pointer");
  return render_frame("splat_surfel", H, W, N, P, depth_key_max, us, nullptr, nullptr, const_cast<float *>(depths),
                      nullptr, nullptr, false, const_cast<void *>(bin_ws), ws, ws_bytes,
                      {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                      SurfelDraw{records, depth_image, alpha_image, normal_image}, nullptr, (cudaStream_t)stream);
}

int gsb_splat_surfel_forward(int H, int W, int N, const float *us, float *depths, int32_t *areas,
                             const float *records, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                             size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                             float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                             uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                             gsb_stream_t stream) {
  int rc = check_frame("splat", 0, H, W, N, bin_ws, bin_ws_bytes);
  if (rc) return rc;
  GSB_REQUIRE(P_cap > 0 && P_cap < ((int64_t)1 << 30), "splat_surfel_forward: bad P_cap");
  GSB_REQUIRE(gsid_per_patch && status_host && bin_ws, "splat_surfel_forward: null pointer");
  GSB_REQUIRE(N == 0 || (us && depths && areas && records), "splat_surfel_forward: null pointer");
  return capacity_wait("splat_surfel", P_cap, status_host, true, [&](const StatusRead *sr) {
    return render_frame("splat_surfel", H, W, N, P_cap, depth_key_cap, us, nullptr, nullptr, depths, nullptr, areas,
                        false, bin_ws, ws, ws_bytes, {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                        SurfelDraw{records, depth_image, alpha_image, normal_image}, sr, (cudaStream_t)stream);
  });
}

int gsb_splat_surfel_backward(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                              const float *final_tau, const int32_t *patch_range_per_tile,
                              const int32_t *gsid_per_patch, const float *dloss_dimage, const float *dloss_ddepth,
                              const float *dloss_dalpha, const float *dloss_dnormal, void *ws, size_t ws_bytes,
                              float *rows, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && H > 0 && W > 0 && P >= 0, "splatB_surfel: bad N/H/W/P");
  GSB_REQUIRE(grid_fits(H, W), "splatB_surfel: more than 65535 tiles in a row or column");
  if (N == 0) return 0;
  GSB_REQUIRE(rows != nullptr, "splatB_surfel: null output");
  const SortLayout SL = sort_layout(N, H, W, 0);
  GSB_REQUIRE(ws != nullptr && aligned(ws, 16) && ws_bytes >= SL.bytes, "splatB_surfel: workspace too small");
  if (P > 0) {
    GSB_REQUIRE(records && contrib && final_tau && patch_range_per_tile && gsid_per_patch, "splatB_surfel: null pointer");
    GSB_REQUIRE(aligned(records, 16) && aligned(patch_range_per_tile, 8), "splatB_surfel: misaligned input");
  }
  char *b = static_cast<char *>(ws);
  return launch_draw_surfel_backward(H, W, N, patch_range_per_tile, P > 0 ? records : nullptr, gsid_per_patch, contrib,
                                     final_tau, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, nullptr, rows,
                                     reinterpret_cast<int *>(b + SL.counters), (cudaStream_t)stream);
}

// ---- 2DGS geometry frames (surfel.cu k_draw_2dgs / k_draw_2dgs_bwd, DESIGN 3.16): the surfel frame
// through the same render core, with the geometry planes

int gsb_splat_2dgs_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us, const float *depths,
                          const float *records, float near, float far, const void *bin_ws, void *ws, size_t ws_bytes,
                          float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                          int32_t *gsid_per_patch, float *depth_image, float *alpha_image, float *normal_image,
                          float *distortion, float *moments, float *median_depth, int32_t *median_contrib,
                          gsb_stream_t stream) {
  int rc = check_frame("splat", 0, H, W, N, bin_ws, SIZE_MAX);
  if (rc) return rc;
  GSB_REQUIRE(P >= 0, "splat_2dgs: bad P");
  GSB_REQUIRE(P == 0 || (us && depths && records && bin_ws && ws && gsid_per_patch), "splat_2dgs: null pointer");
  GeoPlanes g;
  if ((rc = geo_planes("splat_2dgs", near, far, distortion, moments, median_depth, median_contrib, g))) return rc;
  return render_frame("splat_2dgs", H, W, N, P, depth_key_max, us, nullptr, nullptr, const_cast<float *>(depths),
                      nullptr, nullptr, false, const_cast<void *>(bin_ws), ws, ws_bytes,
                      {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                      SurfelDraw{records, depth_image, alpha_image, normal_image, &g}, nullptr, (cudaStream_t)stream);
}

int gsb_splat_2dgs_forward(int H, int W, int N, const float *us, float *depths, int32_t *areas, const float *records,
                           float near, float far, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                           size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                           float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                           uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                           float *distortion, float *moments, float *median_depth, int32_t *median_contrib,
                           gsb_stream_t stream) {
  int rc = check_frame("splat", 0, H, W, N, bin_ws, bin_ws_bytes);
  if (rc) return rc;
  GSB_REQUIRE(P_cap > 0 && P_cap < ((int64_t)1 << 30), "splat_2dgs_forward: bad P_cap");
  GSB_REQUIRE(gsid_per_patch && status_host && bin_ws, "splat_2dgs_forward: null pointer");
  GSB_REQUIRE(N == 0 || (us && depths && areas && records), "splat_2dgs_forward: null pointer");
  GeoPlanes g;
  if ((rc = geo_planes("splat_2dgs", near, far, distortion, moments, median_depth, median_contrib, g))) return rc;
  return capacity_wait("splat_2dgs", P_cap, status_host, true, [&](const StatusRead *sr) {
    return render_frame("splat_2dgs", H, W, N, P_cap, depth_key_cap, us, nullptr, nullptr, depths, nullptr, areas,
                        false, bin_ws, ws, ws_bytes, {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch},
                        SurfelDraw{records, depth_image, alpha_image, normal_image, &g}, sr, (cudaStream_t)stream);
  });
}

int gsb_splat_2dgs_backward(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                            const float *final_tau, const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                            const float *dloss_dimage, const float *dloss_ddepth, const float *dloss_dalpha,
                            const float *dloss_dnormal, void *ws, size_t ws_bytes, float *rows, float near, float far,
                            const float *alpha_image, const float *moments, const int32_t *median_contrib,
                            const float *dloss_ddistortion, const float *dloss_dmedian, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && H > 0 && W > 0 && P >= 0, "splatB_2dgs: bad N/H/W/P");
  GSB_REQUIRE(grid_fits(H, W), "splatB_2dgs: more than 65535 tiles in a row or column");
  if (int rc = check_near_far("splatB_2dgs", near, far)) return rc;
  if (N == 0) return 0;
  GSB_REQUIRE(rows != nullptr, "splatB_2dgs: null output");
  const SortLayout SL = sort_layout(N, H, W, 0);
  GSB_REQUIRE(ws != nullptr && aligned(ws, 16) && ws_bytes >= SL.bytes, "splatB_2dgs: workspace too small");
  const bool with_geo = dloss_ddistortion != nullptr || dloss_dmedian != nullptr;
  if (P > 0) {
    GSB_REQUIRE(records && contrib && final_tau && patch_range_per_tile && gsid_per_patch, "splatB_2dgs: null pointer");
    GSB_REQUIRE(aligned(records, 16) && aligned(patch_range_per_tile, 8), "splatB_2dgs: misaligned input");
    GSB_REQUIRE(!with_geo || (alpha_image && moments && median_contrib), "splatB_2dgs: null geometry plane");
    // the kernel reads these planes one 4-byte element at a time
    GSB_REQUIRE(!with_geo || (aligned(alpha_image, 4) && aligned(moments, 4) && aligned(median_contrib, 4) &&
                              aligned(dloss_ddistortion, 4) && aligned(dloss_dmedian, 4)),
                "splatB_2dgs: misaligned geometry plane");
  }
  const GeoGrads g{dloss_ddistortion, dloss_dmedian, alpha_image, moments, median_contrib, near,
                   (float)((double)far / ((double)far - near))};
  char *b = static_cast<char *>(ws);
  return launch_draw_surfel_backward(H, W, N, patch_range_per_tile, P > 0 ? records : nullptr, gsid_per_patch, contrib,
                                     final_tau, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, &g, rows,
                                     reinterpret_cast<int *>(b + SL.counters), (cudaStream_t)stream);
}

// ---- batched 2D Gaussian Splatting (surfel.cu, DESIGN 3.25): C pinhole cameras of one image size.
// The per-surfel kernels read each surfel's rows once for all C cameras; the C frames are binned,
// sorted and drawn as one tall frame through the frame core above (render_frame, capacity_wait,
// SurfelDraw with a frame count).  Record c N + n is surfel n seen by camera c.

// the batch call description of the per-surfel entry points: batch_scene's checks and table, pinhole
// cameras only
static int surfel_batch_scene(const char *who, int C, int N, int sh_dim3, const float *pws, const float *rots,
                              const float *scales, const float *shs, const float *poses, const float *intrinsics,
                              int camera_model, float width, float height, BatchCams &bc, BatchScene &b) {
  if (camera_model != GSB_CAMERA_PINHOLE) return arg_error(who, "pinhole cameras only");
  if (int rc = batch_scene(who, C, N, sh_dim3, pws, rots, scales, shs, poses, camera_model, intrinsics, width, height,
                           bc, b))
    return rc;
  if (N > 0 && !(pws && rots && scales && shs && poses)) return arg_error(who, "null pointer");
  return 0;
}

int gsb_2dgs_batch_preprocess_forward(int C, int N, int sh_dim3, const float *pws, const float *rots,
                                      const float *scales, const float *shs, const float *poses,
                                      const float *intrinsics, int camera_model, float width, float height,
                                      const float *alphas, float *us, float *depths, int32_t *areas, float *colors,
                                      float *records, gsb_stream_t stream) {
  const char *who = "2dgs_batch_preprocess";
  BatchCams bc;
  BatchScene b{};
  if (int rc = surfel_batch_scene(who, C, N, sh_dim3, pws, rots, scales, shs, poses, intrinsics, camera_model, width,
                                  height, bc, b))
    return rc;
  if (!aligned(records, 16)) return arg_error(who, "records misaligned");
  if (N > 0 && !(alphas && us && depths && areas && colors && records)) return arg_error(who, "null pointer");
  return launch_surfel_fwd_batch(b, alphas, us, depths, areas, colors, records, (cudaStream_t)stream);
}

int gsb_2dgs_batch_preprocess_backward(int C, int N, int sh_dim3, const float *pws, const float *rots,
                                       const float *scales, const float *shs, const float *poses,
                                       const float *intrinsics, int camera_model, float width, float height,
                                       const float *rows, float *dloss_dpws, float *dloss_dshs, float *dloss_dalphas,
                                       float *dloss_dscales, float *dloss_drots, float *dloss_dus,
                                       gsb_stream_t stream) {
  const char *who = "2dgs_batch_preprocessB";
  BatchCams bc;
  BatchScene b{};
  if (int rc = surfel_batch_scene(who, C, N, sh_dim3, pws, rots, scales, shs, poses, intrinsics, camera_model, width,
                                  height, bc, b))
    return rc;
  if (N > 0 && !(rows && dloss_dpws && dloss_dshs && dloss_dalphas && dloss_dscales && dloss_drots && dloss_dus))
    return arg_error(who, "null pointer");
  return launch_surfel_bwd_batch(b, rows, dloss_dpws, dloss_dshs, dloss_dalphas, dloss_dscales, dloss_drots, dloss_dus,
                                 (cudaStream_t)stream);
}

size_t gsb_2dgs_batch_workspace_bytes(int C, int N, int H, int W, int64_t P) {
  return batch_records_ok(C, N) && C <= BATCH_MAX_CAMERAS ? sort_layout(C * N, batch_height(C, H), W, P).bytes : 0;
}

// The checks every batched surfel frame makes first: check_frame's (C < 1, C N >= 2^31, C gy tile
// rows) and the camera count.  `who` prefixes the error texts.
static int surfel_batch_frame(const char *who, int C, int H, int W, int N, const void *bin_ws, size_t bin_ws_bytes) {
  if (C > BATCH_MAX_CAMERAS) return arg_error(who, "C > GSB_BATCH_MAX_CAMERAS");
  return check_frame(who, batch_frames(C), H, W, N, bin_ws, bin_ws_bytes);
}

// gsb_2dgs_batch_render{,_geometry}: a tall frame binned by gsb_splat_bin_batch (geo: with the geometry planes)
static int surfel_batch_render(const char *who, int C, int H, int W, int N, int64_t P, uint32_t depth_key_max,
                               const float *us, const float *depths, const float *records, const void *bin_ws,
                               void *ws, size_t ws_bytes, const FrameOut &o, float *depth_image, float *alpha_image,
                               float *normal_image, const GeoPlanes *geo, gsb_stream_t stream) {
  if (int rc = surfel_batch_frame(who, C, H, W, N, bin_ws, SIZE_MAX)) return rc;
  if (P < 0) return arg_error(who, "bad P");
  if (P >= ((int64_t)1 << 30)) return arg_error(who, "more than 2^30 patches");
  if (P > 0 && !(us && depths && records && bin_ws && ws && o.gsid)) return arg_error(who, "null pointer");
  return render_frame(who, H, W, N, P, depth_key_max, us, nullptr, nullptr, const_cast<float *>(depths), nullptr,
                      nullptr, false, const_cast<void *>(bin_ws), ws, ws_bytes, o,
                      SurfelDraw{records, depth_image, alpha_image, normal_image, geo, C}, nullptr,
                      (cudaStream_t)stream, C);
}

// gsb_2dgs_batch_forward{,_geometry}: the capacity path
static int surfel_batch_forward(const char *who, int C, int H, int W, int N, const float *us, float *depths,
                                int32_t *areas, const float *records, int64_t P_cap, uint32_t depth_key_cap,
                                void *bin_ws, size_t bin_ws_bytes, void *ws, size_t ws_bytes, const FrameOut &o,
                                uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                                const GeoPlanes *geo, gsb_stream_t stream) {
  if (int rc = surfel_batch_frame(who, C, H, W, N, bin_ws, bin_ws_bytes)) return rc;
  if (!(P_cap > 0 && P_cap < ((int64_t)1 << 30))) return arg_error(who, "bad P_cap (2^30 patches or more)");
  if (!(o.gsid && status_host && bin_ws)) return arg_error(who, "null pointer");
  if (N > 0 && !(us && depths && areas && records)) return arg_error(who, "null pointer");
  return capacity_wait(who, P_cap, status_host, true, [&](const StatusRead *sr) {
    return render_frame(who, H, W, N, P_cap, depth_key_cap, us, nullptr, nullptr, depths, nullptr, areas, false,
                        bin_ws, ws, ws_bytes, o, SurfelDraw{records, depth_image, alpha_image, normal_image, geo, C},
                        sr, (cudaStream_t)stream, C);
  });
}

// gsb_2dgs_batch_backward{,_geometry}: rows [C N, 18] from the tall frame (geo: the geometry terms)
static int surfel_batch_backward(const char *who, int C, int H, int W, int N, int64_t P, const float *records,
                                 const int32_t *contrib, const float *final_tau, const int32_t *ranges,
                                 const int32_t *gsid, const float *dl_image, const float *dl_depth,
                                 const float *dl_alpha, const float *dl_normal, void *ws, size_t ws_bytes, float *rows,
                                 const GeoGrads *geo, gsb_stream_t stream) {
  if (int rc = surfel_batch_frame(who, C, H, W, N, nullptr, SIZE_MAX)) return rc;
  if (P < 0) return arg_error(who, "bad P");
  if (P >= ((int64_t)1 << 30)) return arg_error(who, "more than 2^30 patches");
  if (N == 0) return 0;
  if (rows == nullptr) return arg_error(who, "null output");
  const Tall t = tall_frame(C, H, N);
  const SortLayout SL = sort_layout(t.N, t.H, W, 0);
  if (!(ws != nullptr && aligned(ws, 16) && ws_bytes >= SL.bytes)) return arg_error(who, "workspace too small");
  const bool with_geo = geo != nullptr && (geo->distortion != nullptr || geo->median != nullptr);
  if (P > 0) {
    if (!(records && contrib && final_tau && ranges && gsid)) return arg_error(who, "null pointer");
    if (!(aligned(records, 16) && aligned(ranges, 8))) return arg_error(who, "misaligned input");
    if (with_geo && !(geo->alpha && geo->moments && geo->median_contrib)) return arg_error(who, "null geometry plane");
    // the kernel reads these planes one 4-byte element at a time
    if (with_geo && !(aligned(geo->alpha, 4) && aligned(geo->moments, 4) && aligned(geo->median_contrib, 4) &&
                      aligned(geo->distortion, 4) && aligned(geo->median, 4)))
      return arg_error(who, "misaligned geometry plane");
  }
  char *b = static_cast<char *>(ws);
  return launch_draw_surfel_backward(H, W, t.N, ranges, P > 0 ? records : nullptr, gsid, contrib, final_tau, dl_image,
                                     dl_depth, dl_alpha, dl_normal, geo, rows,
                                     reinterpret_cast<int *>(b + SL.counters), (cudaStream_t)stream, C);
}

int gsb_2dgs_batch_render(int C, int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                          const float *depths, const float *records, const void *bin_ws, void *ws, size_t ws_bytes,
                          float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                          int32_t *gsid_per_patch, float *depth_image, float *alpha_image, float *normal_image,
                          gsb_stream_t stream) {
  return surfel_batch_render("2dgs_batch", C, H, W, N, P, depth_key_max, us, depths, records, bin_ws, ws, ws_bytes,
                             {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch}, depth_image,
                             alpha_image, normal_image, nullptr, stream);
}

int gsb_2dgs_batch_forward(int C, int H, int W, int N, const float *us, float *depths, int32_t *areas,
                           const float *records, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                           size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                           float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                           uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                           gsb_stream_t stream) {
  return surfel_batch_forward("2dgs_batch", C, H, W, N, us, depths, areas, records, P_cap, depth_key_cap, bin_ws,
                              bin_ws_bytes, ws, ws_bytes, {image, contrib, final_tau, patch_range_per_tile,
                                                           gsid_per_patch},
                              status_host, depth_image, alpha_image, normal_image, nullptr, stream);
}

int gsb_2dgs_batch_backward(int C, int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                            const float *final_tau, const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                            const float *dloss_dimage, const float *dloss_ddepth, const float *dloss_dalpha,
                            const float *dloss_dnormal, void *ws, size_t ws_bytes, float *rows, gsb_stream_t stream) {
  return surfel_batch_backward("2dgs_batchB", C, H, W, N, P, records, contrib, final_tau, patch_range_per_tile,
                               gsid_per_patch, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, ws, ws_bytes,
                               rows, nullptr, stream);
}

int gsb_2dgs_batch_render_geometry(int C, int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                                   const float *depths, const float *records, float near, float far,
                                   const void *bin_ws, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                                   float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                                   float *depth_image, float *alpha_image, float *normal_image, float *distortion,
                                   float *moments, float *median_depth, int32_t *median_contrib,
                                   gsb_stream_t stream) {
  GeoPlanes g;
  if (int rc = geo_planes("2dgs_batch", near, far, distortion, moments, median_depth, median_contrib, g)) return rc;
  return surfel_batch_render("2dgs_batch", C, H, W, N, P, depth_key_max, us, depths, records, bin_ws, ws, ws_bytes,
                             {image, contrib, final_tau, patch_range_per_tile, gsid_per_patch}, depth_image,
                             alpha_image, normal_image, &g, stream);
}

int gsb_2dgs_batch_forward_geometry(int C, int H, int W, int N, const float *us, float *depths, int32_t *areas,
                                    const float *records, float near, float far, int64_t P_cap,
                                    uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                                    size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                                    int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                                    float *depth_image, float *alpha_image, float *normal_image, float *distortion,
                                    float *moments, float *median_depth, int32_t *median_contrib,
                                    gsb_stream_t stream) {
  GeoPlanes g;
  if (int rc = geo_planes("2dgs_batch", near, far, distortion, moments, median_depth, median_contrib, g)) return rc;
  return surfel_batch_forward("2dgs_batch", C, H, W, N, us, depths, areas, records, P_cap, depth_key_cap, bin_ws,
                              bin_ws_bytes, ws, ws_bytes, {image, contrib, final_tau, patch_range_per_tile,
                                                           gsid_per_patch},
                              status_host, depth_image, alpha_image, normal_image, &g, stream);
}

int gsb_2dgs_batch_backward_geometry(int C, int H, int W, int N, int64_t P, const float *records,
                                     const int32_t *contrib, const float *final_tau,
                                     const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                                     const float *dloss_dimage, const float *dloss_ddepth, const float *dloss_dalpha,
                                     const float *dloss_dnormal, void *ws, size_t ws_bytes, float *rows, float near,
                                     float far, const float *alpha_image, const float *moments,
                                     const int32_t *median_contrib, const float *dloss_ddistortion,
                                     const float *dloss_dmedian, gsb_stream_t stream) {
  if (int rc = check_near_far("2dgs_batchB", near, far)) return rc;
  const GeoGrads g{dloss_ddistortion, dloss_dmedian, alpha_image, moments, median_contrib, near,
                   (float)((double)far / ((double)far - near))};
  return surfel_batch_backward("2dgs_batchB", C, H, W, N, P, records, contrib, final_tau, patch_range_per_tile,
                               gsid_per_patch, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, ws, ws_bytes,
                               rows, &g, stream);
}

// ---- feature rendering (raster_feat.cu)

size_t gsb_splat_features_workspace_bytes(int N, int H, int W, int64_t P) {
  return feat_layout(N, H, W, P, 1).bytes;  // (a ws at any address: the split from the worst start)
}

// The checks both feature entry points make, and the records they replay: packed_records, or
// those packed into ws from us / cinv2ds / alphas / colors.  -> 0 and *recs (NULL without patches)
static int feature_frame(const char *who, int H, int W, int N, int64_t P, int D, const float *us, const float *cinv2ds,
                         const float *alphas, const float *colors, const float *features, const int32_t *contrib,
                         const int32_t *ranges, const int32_t *gsid, const void *packed_records, void *ws,
                         size_t ws_bytes, const Rec **recs, int **work, cudaStream_t st) {
  char msg[160];
  const char *err = nullptr;
  const int64_t P_ws = packed_records != nullptr ? 0 : P;
  if (N < 0 || H <= 0 || W <= 0 || P < 0)
    err = "bad N/H/W/P";
  else if (D < 1)
    err = "D < 1";
  else if (!grid_fits(H, W))
    err = "more than 65535 tiles in a row or column";
  else if (!aligned(packed_records, 16))
    err = "packed_records misaligned";
  else if (!(contrib && ranges && ws))
    err = "null pointer";
  else if (P > 0 && !(features && gsid && (packed_records || (us && cinv2ds && alphas && colors))))
    err = "null pointer";
  else if (ws_bytes < feat_layout(N, H, W, P_ws, 1).bytes)
    err = "workspace too small";
  if (err) {
    snprintf(msg, sizeof(msg), "%s: %s", who, err);
    return set_arg_error(msg);
  }
  char *b = static_cast<char *>(ws);
  const FeatLayout L = feat_layout(N, H, W, P_ws, reinterpret_cast<uintptr_t>(ws));
  *work = reinterpret_cast<int *>(b + L.work);
  *recs = nullptr;
  if (P == 0 || N == 0) return 0;
  if (packed_records != nullptr) {
    *recs = static_cast<const Rec *>(packed_records);
    return 0;
  }
  Rec *r = reinterpret_cast<Rec *>(b + L.recs);
  *recs = r;
  return launch_pack_only(N, nullptr, us, cinv2ds, alphas, colors, nullptr, r, st);
}

int gsb_splat_features(int H, int W, int N, int64_t P, int D, const float *us, const float *cinv2ds,
                       const float *alphas, const float *colors, const float *features, const void *packed_records,
                       const int32_t *contrib, const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                       void *ws, size_t ws_bytes, float *feature_image, gsb_stream_t stream) {
  GSB_REQUIRE(feature_image != nullptr, "splat_features: null feature_image");
  GSB_REQUIRE(aligned(feature_image, 16), "splat_features: misaligned feature_image");
  cudaStream_t st = (cudaStream_t)stream;
  const Rec *recs = nullptr;
  int *work = nullptr;
  if (int rc = feature_frame("splat_features", H, W, N, P, D, us, cinv2ds, alphas, colors, features, contrib,
                             patch_range_per_tile, gsid_per_patch, packed_records, ws, ws_bytes, &recs, &work, st))
    return rc;
  return launch_draw_features(H, W, D, patch_range_per_tile, recs, gsid_per_patch, contrib, features, feature_image,
                              work, st);
}

int gsb_splat_features_backward(int H, int W, int N, int64_t P, int D, const float *us, const float *cinv2ds,
                                const float *alphas, const float *colors, const float *features,
                                const void *packed_records, const int32_t *contrib, const float *final_tau,
                                const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                                const float *dloss_dfeature_image, void *ws, size_t ws_bytes, float *moments,
                                float *dloss_dfeatures, gsb_stream_t stream) {
  GSB_REQUIRE(N == 0 || (moments && dloss_dfeatures), "splat_features_backward: null output");
  GSB_REQUIRE(P == 0 || (final_tau && dloss_dfeature_image), "splat_features_backward: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const Rec *recs = nullptr;
  int *work = nullptr;
  if (int rc = feature_frame("splat_features_backward", H, W, N, P, D, us, cinv2ds, alphas, colors, features, contrib,
                             patch_range_per_tile, gsid_per_patch, packed_records, ws, ws_bytes, &recs, &work, st))
    return rc;
  return launch_draw_features_backward(H, W, N, D, patch_range_per_tile, recs, gsid_per_patch, contrib, final_tau,
                                       features, dloss_dfeature_image, moments, dloss_dfeatures, work, st);
}

// ---- contribution statistics (raster_stats.cu, surfel.cu k_draw_stats_2dgs; DESIGN 3.18)

size_t gsb_splat_stats_workspace_bytes(int N, int H, int W, int64_t P) {
  return feat_layout(N, H, W, P, 1).bytes;  // the feature replay's records and work area
}

// the outputs both statistics entry points accumulate into
static int stats_outputs(const char *who, int N, const float *weight_sum, const float *weight_max,
                         const int64_t *hit_count) {
  if (N > 0 && !(weight_sum && weight_max && hit_count)) return arg_error(who, "null output");
  // 4-byte atomics on the two float arrays, 8-byte atomics on the counts
  if (!aligned(weight_sum, 4) || !aligned(weight_max, 4) || !aligned(hit_count, 8))
    return arg_error(who, "misaligned output");
  return 0;
}

int gsb_splat_stats(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds, const float *alphas,
                    const float *colors, const void *packed_records, const int32_t *contrib,
                    const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch, void *ws, size_t ws_bytes,
                    float *weight_sum, float *weight_max, int64_t *hit_count, gsb_stream_t stream) {
  if (int rc = stats_outputs("splat_stats", N, weight_sum, weight_max, hit_count)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const Rec *recs = nullptr;
  int *work = nullptr;
  // feature_frame's checks and records with one "feature" channel: the statistics read no features,
  // so any non-null pointer stands in for them
  if (int rc = feature_frame("splat_stats", H, W, N, P, 1, us, cinv2ds, alphas, colors, weight_sum, contrib,
                             patch_range_per_tile, gsid_per_patch, packed_records, ws, ws_bytes, &recs, &work, st))
    return rc;
  return launch_draw_stats(H, W, patch_range_per_tile, recs, gsid_per_patch, contrib, weight_sum, weight_max,
                           hit_count, work, st);
}

int gsb_splat_stats_2dgs(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                           const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch, float *weight_sum,
                           float *weight_max, int64_t *hit_count, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && H > 0 && W > 0 && P >= 0, "splat_stats_2dgs: bad N/H/W/P");
  GSB_REQUIRE(grid_fits(H, W), "splat_stats_2dgs: more than 65535 tiles in a row or column");
  if (int rc = stats_outputs("splat_stats_2dgs", N, weight_sum, weight_max, hit_count)) return rc;
  if (N == 0 || P == 0) return 0;
  GSB_REQUIRE(records && contrib && patch_range_per_tile && gsid_per_patch, "splat_stats_2dgs: null pointer");
  GSB_REQUIRE(aligned(records, 16) && aligned(patch_range_per_tile, 8), "splat_stats_2dgs: misaligned input");
  return launch_draw_surfel_stats(H, W, patch_range_per_tile, records, gsid_per_patch, contrib, weight_sum, weight_max,
                                  hit_count, (cudaStream_t)stream);
}

// ---- density control + record conversion (density.cu)

static bool gau_complete(const gsb_gaussians *g) {
  return g && g->pws && g->low_shs && g->high_shs && g->alphas_raw && g->scales_raw && g->rots_raw;
}
static float *const *gau_ptrs(const gsb_gaussians *g) {
  // six consecutive float* members: the struct IS the pointer table the launchers index
  static_assert(sizeof(gsb_gaussians) == 6 * sizeof(float *), "gsb_gaussians layout");
  return reinterpret_cast<float *const *>(g);
}
// the Adam moments of a call: all of `m` given or all NULL.  tables: `m` are gsb_gaussians, and a
// given one must also hold all six tensors
static bool moments_ok(std::initializer_list<const void *> m, bool tables = false) {
  bool any = false, all = true;
  for (const void *p : m)
    any |= p != nullptr, all &= tables ? gau_complete(static_cast<const gsb_gaussians *>(p)) : p != nullptr;
  return all || !any;
}

int gsb_density_accumulate(int64_t N, const float *dloss_dus, const uint8_t *mask, float *grad_accum,
                           int32_t *cunt, int first, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "density_accumulate: N < 0");
  GSB_REQUIRE(N == 0 || (dloss_dus && mask && grad_accum && cunt), "density_accumulate: null pointer");
  return launch_density_accumulate(N, dloss_dus, mask, grad_accum, cunt, first, (cudaStream_t)stream);
}

size_t gsb_density_workspace_bytes(int64_t N) { return density_workspace_bytes(N); }

int gsb_density_plan(int64_t N, const float *alphas_raw, const float *scales_raw, const float *grad_accum,
                     const int32_t *cunt, float alpha_raw_min, float scale_raw_max, float grad_min,
                     float scale_clone_max, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                     int64_t *counts_host, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < ((int64_t)1 << 31), "density_plan: N out of range");
  GSB_REQUIRE(counts_host != nullptr, "density_plan: counts_host is null");
  GSB_REQUIRE(N == 0 || (alphas_raw && scales_raw && grad_accum && cunt && ws && cls && slots),
              "density_plan: null pointer");
  GSB_REQUIRE(N == 0 || ws_bytes >= density_workspace_bytes(N), "density_plan: workspace too small");
  return launch_density_plan(N, alphas_raw, scales_raw, grad_accum, cunt, alpha_raw_min, scale_raw_max, grad_min,
                             scale_clone_max, ws, ws_bytes, cls, slots, counts_host, (cudaStream_t)stream);
}

int gsb_density_plan_keep(int64_t N, const uint8_t *keep, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                          int64_t *counts_host, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < ((int64_t)1 << 31), "density_plan_keep: N out of range");
  GSB_REQUIRE(counts_host != nullptr, "density_plan_keep: counts_host is null");
  GSB_REQUIRE(N == 0 || (keep && ws && cls && slots), "density_plan_keep: null pointer");
  GSB_REQUIRE(N == 0 || ws_bytes >= density_workspace_bytes(N), "density_plan_keep: workspace too small");
  return launch_density_plan_keep(N, keep, ws, cls, slots, counts_host, (cudaStream_t)stream);
}

int gsb_density_apply(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int64_t S,
                      const gsb_gaussians *src, const gsb_gaussians *src_m, const gsb_gaussians *src_v,
                      const float *z, const gsb_gaussians *dst, const gsb_gaussians *dst_m,
                      const gsb_gaussians *dst_v, gsb_stream_t stream) {
  // N < 2^30: the rebuild's row table packs the class into bits 30-31 of the survivor slot
  GSB_REQUIRE(N >= 0 && N < ((int64_t)1 << 30) && K >= 0 && C >= 0 && S >= 0 && K <= N && C + S <= K,
              "density_apply: bad counts");
  if (N == 0) return 0;
  GSB_REQUIRE(cls && slots, "density_apply: null plan");
  GSB_REQUIRE(gau_complete(src), "density_apply: src has a null tensor");
  GSB_REQUIRE(K + C + S == 0 || gau_complete(dst), "density_apply: dst has a null tensor");
  const bool state = src_m != nullptr;
  GSB_REQUIRE(moments_ok({src_m, src_v, dst_m, dst_v}), "density_apply: Adam moments must be all given or all NULL");
  if (state)
    GSB_REQUIRE(gau_complete(src_m) && gau_complete(src_v) && (K + C + S == 0 || (gau_complete(dst_m) && gau_complete(dst_v))),
                "density_apply: a moment tensor is null");
  GSB_REQUIRE(S == 0 || z != nullptr, "density_apply: z is null");
  if (K + C + S == 0) return 0;
  return launch_density_apply(N, cls, slots, K, C, gau_ptrs(src), state ? gau_ptrs(src_m) : nullptr,
                              state ? gau_ptrs(src_v) : nullptr, z, gau_ptrs(dst), state ? gau_ptrs(dst_m) : nullptr,
                              state ? gau_ptrs(dst_v) : nullptr, (cudaStream_t)stream);
}

int gsb_density_apply_rows(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int64_t S,
                           int D, const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                           float *dst_v, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && K >= 0 && C >= 0 && S >= 0 && K <= N && C + S <= K && D >= 1, "density_apply_rows: bad counts");
  if (N == 0 || K + C + S == 0) return 0;
  GSB_REQUIRE(cls && slots && src && dst, "density_apply_rows: null pointer");
  GSB_REQUIRE(moments_ok({src_m, src_v, dst_m, dst_v}),
              "density_apply_rows: Adam moments must be all given or all NULL");
  return launch_density_apply_rows(N, cls, slots, K, C, D, src, src_m, src_v, dst, dst_m, dst_v, (cudaStream_t)stream);
}

int gsb_reset_alpha(int64_t N, float *alphas_raw, float *exp_avg, float *exp_avg_sq, float reset_raw,
                    gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "reset_alpha: N < 0");
  GSB_REQUIRE(N == 0 || alphas_raw, "reset_alpha: null pointer");
  return launch_reset_alpha(N, alphas_raw, exp_avg, exp_avg_sq, reset_raw, (cudaStream_t)stream);
}

// ---- MCMC densification (density.cu)

static const int64_t kMcmcMaxN = (int64_t)1 << 31;  // row ids are int32

size_t gsb_mcmc_workspace_bytes(int64_t N, int64_t n) {
  return mcmc_workspace_bytes(N < 0 ? 0 : N, n < 0 ? 0 : n);
}

#define GSB_MCMC_WS(ws, ws_bytes, N, n, what)                                                   \
  do {                                                                                          \
    GSB_REQUIRE(ws != nullptr && aligned(ws, 16), what ": workspace null or misaligned");      \
    GSB_REQUIRE(ws_bytes >= mcmc_workspace_bytes(N, n), what ": workspace too small");          \
  } while (0)

int gsb_mcmc_plan(int64_t N, const float *alphas_raw, float alpha_raw_min, int mode, void *ws, size_t ws_bytes,
                  int64_t *counts_host, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < kMcmcMaxN, "mcmc_plan: N out of range");
  GSB_REQUIRE(mode == 0 || mode == 1, "mcmc_plan: mode must be 0 (relocate) or 1 (grow)");
  GSB_REQUIRE(counts_host != nullptr, "mcmc_plan: counts_host is null");
  if (N == 0) return counts_host[0] = counts_host[1] = 0, 0;
  GSB_REQUIRE(alphas_raw != nullptr, "mcmc_plan: null pointer");
  GSB_MCMC_WS(ws, ws_bytes, N, 0, "mcmc_plan");
  return launch_mcmc_plan(N, alphas_raw, alpha_raw_min, mode, ws, counts_host, (cudaStream_t)stream);
}

int gsb_mcmc_sample(int64_t N, int64_t n, const double *u, void *ws, size_t ws_bytes, int32_t *sampled,
                    gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < kMcmcMaxN && n >= 0, "mcmc_sample: bad counts");
  GSB_REQUIRE(n == 0 || N > 0, "mcmc_sample: draws from no rows");
  if (n == 0) return 0;
  GSB_REQUIRE(u && sampled, "mcmc_sample: null pointer");
  GSB_MCMC_WS(ws, ws_bytes, N, 0, "mcmc_sample");
  return launch_mcmc_sample(N, n, u, ws, sampled, (cudaStream_t)stream);
}

int gsb_mcmc_relocate(int64_t N, int64_t n, const int32_t *sampled, void *ws, size_t ws_bytes, double min_opacity,
                      int n_max, const gsb_gaussians *params, const gsb_gaussians *exp_avg,
                      const gsb_gaussians *exp_avg_sq, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < kMcmcMaxN && n >= 0 && n <= N, "mcmc_relocate: bad counts");
  GSB_REQUIRE(n_max >= 1 && n_max <= 51, "mcmc_relocate: n_max must be in [1, 51]");
  GSB_REQUIRE(min_opacity > 0.0 && min_opacity < 1.0, "mcmc_relocate: min_opacity must be in (0, 1)");
  if (n == 0) return 0;
  GSB_REQUIRE(sampled && gau_complete(params), "mcmc_relocate: null pointer");
  GSB_REQUIRE(moments_ok({exp_avg, exp_avg_sq}, true), "mcmc_relocate: Adam moments must be both given or both NULL");
  GSB_MCMC_WS(ws, ws_bytes, N, n, "mcmc_relocate");
  return launch_mcmc_relocate(N, n, sampled, ws, min_opacity, n_max, gau_ptrs(params),
                              exp_avg ? gau_ptrs(exp_avg) : nullptr, exp_avg_sq ? gau_ptrs(exp_avg_sq) : nullptr,
                              (cudaStream_t)stream);
}

int gsb_mcmc_relocate_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, size_t ws_bytes, int D,
                           float *x, float *exp_avg, float *exp_avg_sq, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && N < kMcmcMaxN && n >= 0 && n <= N && D >= 1, "mcmc_relocate_rows: bad counts");
  if (n == 0) return 0;
  GSB_REQUIRE(sampled && x, "mcmc_relocate_rows: null pointer");
  GSB_REQUIRE(moments_ok({exp_avg, exp_avg_sq}), "mcmc_relocate_rows: Adam moments must be both given or both NULL");
  GSB_MCMC_WS(ws, ws_bytes, N, 0, "mcmc_relocate_rows");
  return launch_mcmc_relocate_rows(N, n, sampled, ws, D, x, exp_avg, exp_avg_sq, (cudaStream_t)stream);
}

int gsb_mcmc_grow(int64_t N, int64_t n, const int32_t *sampled, void *ws, size_t ws_bytes, double min_opacity,
                  int n_max, const gsb_gaussians *src, const gsb_gaussians *src_m, const gsb_gaussians *src_v,
                  const gsb_gaussians *dst, const gsb_gaussians *dst_m, const gsb_gaussians *dst_v,
                  gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && n >= 0 && N + n < kMcmcMaxN, "mcmc_grow: bad counts");
  GSB_REQUIRE(n_max >= 1 && n_max <= 51, "mcmc_grow: n_max must be in [1, 51]");
  GSB_REQUIRE(min_opacity > 0.0 && min_opacity < 1.0, "mcmc_grow: min_opacity must be in (0, 1)");
  GSB_REQUIRE(n == 0 || N > 0, "mcmc_grow: draws from no rows");
  if (N == 0) return 0;
  GSB_REQUIRE(gau_complete(src) && gau_complete(dst) && (n == 0 || sampled), "mcmc_grow: null pointer");
  const bool state = src_m != nullptr;
  GSB_REQUIRE(moments_ok({src_m, src_v, dst_m, dst_v}, true), "mcmc_grow: Adam moments must be all given or all NULL");
  GSB_MCMC_WS(ws, ws_bytes, N, n, "mcmc_grow");
  return launch_mcmc_grow(N, n, sampled, ws, min_opacity, n_max, gau_ptrs(src), state ? gau_ptrs(src_m) : nullptr,
                          state ? gau_ptrs(src_v) : nullptr, gau_ptrs(dst), state ? gau_ptrs(dst_m) : nullptr,
                          state ? gau_ptrs(dst_v) : nullptr, (cudaStream_t)stream);
}

int gsb_mcmc_grow_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, size_t ws_bytes, int D,
                       const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                       float *dst_v, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && n >= 0 && N + n < kMcmcMaxN && D >= 1, "mcmc_grow_rows: bad counts");
  GSB_REQUIRE(n == 0 || N > 0, "mcmc_grow_rows: draws from no rows");
  if (N == 0) return 0;
  GSB_REQUIRE(src && dst && (n == 0 || sampled), "mcmc_grow_rows: null pointer");
  GSB_REQUIRE(moments_ok({src_m, src_v, dst_m, dst_v}), "mcmc_grow_rows: Adam moments must be all given or all NULL");
  GSB_MCMC_WS(ws, ws_bytes, N, 0, "mcmc_grow_rows");
  return launch_mcmc_grow_rows(N, n, sampled, ws, D, src, src_m, src_v, dst, dst_m, dst_v, (cudaStream_t)stream);
}

int gsb_mcmc_noise(int64_t N, float *pws, const float *alphas_raw, const float *scales_raw, const float *rots_raw,
                   const float *z, float scale, float k, float x0, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "mcmc_noise: N < 0");
  GSB_REQUIRE(N == 0 || (pws && alphas_raw && scales_raw && rots_raw && z), "mcmc_noise: null pointer");
  return launch_mcmc_noise(N, pws, alphas_raw, scales_raw, rots_raw, z, scale, k, x0, (cudaStream_t)stream);
}

int gsb_adam_step(int n_tensors, const gsb_adam_tensor *table, int64_t N, const uint8_t *visibility, double beta1,
                  double beta2, double eps, gsb_stream_t stream) {
  GSB_REQUIRE(n_tensors >= 0 && N >= 0, "adam_step: negative count");
  GSB_REQUIRE(n_tensors == 0 || table != nullptr, "adam_step: null table");
  GSB_REQUIRE(visibility != nullptr || N == 0, "adam_step: N > 0 without a visibility mask");
  GSB_REQUIRE(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0, "adam_step: betas must be in [0, 1)");
  GSB_REQUIRE(eps >= 0.0 && isfinite(eps), "adam_step: eps must be finite and >= 0");
  bool work = false;
  for (int i = 0; i < n_tensors; i++) {
    const gsb_adam_tensor &a = table[i];
    GSB_REQUIRE(a.numel >= 0, "adam_step: negative numel");
    if (visibility) {
      GSB_REQUIRE(a.D >= 1 && a.numel == N * (int64_t)a.D, "adam_step: a tensor's numel is not N * D");
    }
    if (a.numel == 0) continue;
    GSB_REQUIRE(a.param && a.grad && a.exp_avg && a.exp_avg_sq, "adam_step: null pointer");
    GSB_REQUIRE(aligned(a.param, 4) && aligned(a.grad, 4) && aligned(a.exp_avg, 4) && aligned(a.exp_avg_sq, 4),
                "adam_step: misaligned tensor");
    work = true;
  }
  if (!work) return 0;
  return launch_adam(n_tensors, table, visibility, beta1, beta2, eps, (cudaStream_t)stream);
}

static bool sh_dim_ok(int d) { return d == 3 || d == 12 || d == 27 || d == 48; }

int gsb_ply_rows_to_gs(int64_t N, int stride, int sh_dim, const float *rows, const int32_t *colmap,
                       float *gs_rows, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && sh_dim_ok(sh_dim), "ply_rows_to_gs: sh_dim must be 3, 12, 27 or 48");
  GSB_REQUIRE(stride >= 11 + sh_dim, "ply_rows_to_gs: row stride smaller than 11 + sh_dim");
  GSB_REQUIRE(N == 0 || (rows && colmap && gs_rows), "ply_rows_to_gs: null pointer");
  return launch_ply_rows_to_gs(N, stride, sh_dim, rows, colmap, gs_rows, (cudaStream_t)stream);
}

int gsb_gs_to_params(int64_t N, int sh_dim, const float *gs_rows, const gsb_gaussians *dst, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && sh_dim_ok(sh_dim), "gs_to_params: sh_dim must be 3, 12, 27 or 48");
  GSB_REQUIRE(N == 0 || (gs_rows && gau_complete(dst)), "gs_to_params: null pointer");
  if (N == 0) return 0;
  return launch_gs_to_params(N, sh_dim, gs_rows, gau_ptrs(dst), (cudaStream_t)stream);
}

int gsb_params_to_gs(int64_t N, const gsb_gaussians *src, float *gs_rows, gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0, "params_to_gs: N < 0");
  GSB_REQUIRE(N == 0 || (gs_rows && gau_complete(src)), "params_to_gs: null pointer");
  if (N == 0) return 0;
  return launch_params_to_gs(N, gau_ptrs(src), gs_rows, (cudaStream_t)stream);
}

// ---- multi-GPU gradient exchange (comm.cu, fused.cu PUSH variant)

size_t gsb_exchange_region_bytes(int N, int sh_dim3, int world) {
  if (N < 0 || world < 1 || world > kMaxWorld) return 0;
  return exchange_geom(N, sh_dim3, world).bytes;
}

size_t gsb_exchange_result_offset(int N, int sh_dim3, int world, int segment) {
  if (segment < 0 || segment > 4 || world < 1 || world > kMaxWorld) return 0;
  const ExchangeGeom G = exchange_geom(N, sh_dim3, world);
  return G.result_base + (size_t)G.result_off[segment] * sizeof(float);
}

int gsb_comm_alloc(size_t bytes, void **ptr, void *handle_out) {
  GSB_REQUIRE(ptr && handle_out && bytes > 0, "comm_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == GSB_COMM_HANDLE_BYTES, "IPC handle size");
  GSB_CUDA_TRY(cudaMalloc(ptr, bytes));
  GSB_CUDA_TRY(cudaMemset(*ptr, 0, bytes));
  GSB_CUDA_TRY(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  GSB_CUDA_TRY(cudaIpcGetMemHandle(&h, *ptr));
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int gsb_comm_open(const void *handle, void **peer_ptr) {
  GSB_REQUIRE(handle && peer_ptr, "comm_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  GSB_CUDA_TRY(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

int gsb_comm_close(void *peer_ptr) {
  if (peer_ptr) GSB_CUDA_TRY(cudaIpcCloseMemHandle(peer_ptr));
  return 0;
}

int gsb_comm_free(void *ptr) {
  if (ptr) GSB_CUDA_TRY(cudaFree(ptr));
  return 0;
}

int gsb_exchange_status(const void *region, int *status_host) {
  GSB_REQUIRE(region && status_host, "exchange_status: bad arguments");
  uint32_t v = 0;
  GSB_CUDA_TRY(cudaMemcpy(&v, static_cast<const char *>(region) + 136, sizeof(v), cudaMemcpyDeviceToHost));
  *status_host = (int)v;
  return 0;
}

int gsb_preprocess_backward_push(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc,
                                 float fx, float fy, float cx, float cy, float width, float height,
                                 const float *dloss_dus, const float *dloss_dcinv2ds, const float *dloss_dcolors,
                                 const float *dloss_dalphas, const float *moments, const float *cinv2ds,
                                 float *dloss_dus_out, int world, int rank, void *const *regions_host,
                                 uint32_t epoch, gsb_stream_t stream) {
  const FusedScene sc{N, sh_dim3, pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height};
  FusedBwd b{dloss_dus, dloss_dcinv2ds, dloss_dcolors};
  b.mi = {moments, cinv2ds, dloss_dus_out, nullptr};
  if (int rc = check_preprocess_backward("preprocess_backward_push", GradOutputs::kNone, sc, b)) return rc;
  GSB_REQUIRE(N == 0 || moments || dloss_dalphas, "preprocess_backward_push: null upstream gradient");
  GSB_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world && regions_host && epoch != 0,
              "preprocess_backward_push: bad world / rank / regions / epoch");
  const ExchangeGeom G = exchange_geom(N, sh_dim3, world);
  GradPush gp{};
  for (int p = 0; p < world; p++) {
    GSB_REQUIRE(regions_host[p] != nullptr, "preprocess_backward_push: null region");
    char *r = static_cast<char *>(regions_host[p]);
    gp.slot[p] = reinterpret_cast<float *>(r + G.staging_off) + (size_t)rank * G.slot_floats;
    gp.flags[p] = reinterpret_cast<uint32_t *>(r);
  }
  gp.counter = reinterpret_cast<uint32_t *>(static_cast<char *>(regions_host[rank]) + 128);
  gp.g_alphas = dloss_dalphas;
  gp.off_rots = G.slot_off[1];
  gp.off_pws = G.slot_off[2];
  gp.off_scales = G.slot_off[3];
  gp.off_alphas = G.slot_off[4];
  gp.world = world;
  gp.rank = rank;
  gp.epoch = epoch;
  b.gp = &gp;
  return launch_preprocess_bwd(sc, b, (cudaStream_t)stream);
}

int gsb_grad_reduce_broadcast(int N, int sh_dim3, int world, int rank, void *const *regions_host, uint32_t epoch,
                              gsb_stream_t stream) {
  GSB_REQUIRE(N >= 0 && world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world && regions_host && epoch != 0,
              "grad_reduce_broadcast: bad arguments");
  for (int p = 0; p < world; p++) GSB_REQUIRE(regions_host[p] != nullptr, "grad_reduce_broadcast: null region");
  const ExchangeGeom G = exchange_geom(N, sh_dim3, world);
  return launch_grad_reduce_bcast(G, rank, regions_host, epoch, (cudaStream_t)stream);
}

// ---- mesh extraction (tsdf.cu, DESIGN 3.17)
// the grid checks every TSDF entry point makes; 0 or the argument error "<who>: <reason>"
static int tsdf_grid_check(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const char *who) {
  if (nx < 1 || ny < 1 || nz < 1) return arg_error(who, "bad grid dimension");
  if ((int64_t)nx * ny * nz >= ((int64_t)1 << 31)) return arg_error(who, "2^31 or more voxels");
  if (!(std::isfinite(voxel) && voxel > 0.f)) return arg_error(who, "voxel must be finite and > 0");
  if (!(std::isfinite(ox) && std::isfinite(oy) && std::isfinite(oz))) return arg_error(who, "origin not finite");
  return 0;
}

int gsb_tsdf_integrate(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc,
                       float depth_trunc, int V, int H, int W, const float *cams, const float *depth,
                       const float *color, float *tsdf, float *weight, float *color_grid, gsb_stream_t stream) {
  if (int rc = tsdf_grid_check(nx, ny, nz, ox, oy, oz, voxel, "tsdf_integrate")) return rc;
  GSB_REQUIRE(std::isfinite(trunc) && trunc > 0.f, "tsdf_integrate: trunc must be finite and > 0");
  GSB_REQUIRE(depth_trunc > 0.f, "tsdf_integrate: depth_trunc must be > 0");
  GSB_REQUIRE(V >= 1 && H >= 1 && W >= 1, "tsdf_integrate: V, H and W must be >= 1");
  GSB_REQUIRE((color == nullptr) == (color_grid == nullptr), "tsdf_integrate: colour given to one side only");
  GSB_REQUIRE(cams && depth && tsdf && weight, "tsdf_integrate: null pointer");
  for (const void *p : {(const void *)cams, (const void *)depth, (const void *)color, (const void *)tsdf,
                        (const void *)weight, (const void *)color_grid})
    GSB_REQUIRE(aligned(p, 4), "tsdf_integrate: misaligned array");
  const TsdfGrid g{nx, ny, nz, ox, oy, oz, voxel};
  return launch_tsdf_integrate(g, trunc, depth_trunc, V, H, W, cams, depth, color, tsdf, weight, color_grid,
                               (cudaStream_t)stream);
}

size_t gsb_tsdf_extract_workspace_bytes(int nx, int ny, int nz) {
  if (nx < 1 || ny < 1 || nz < 1 || (int64_t)nx * ny * nz >= ((int64_t)1 << 31)) return 0;
  return tsdf_extract_workspace_bytes((int64_t)nx * ny * nz);
}

// the volume and workspace checks of the plan and the emit
static int tsdf_extract_args(int nx, int ny, int nz, const float *tsdf, const float *weight, const void *ws,
                             size_t ws_bytes, const char *who) {
  if (!(tsdf && weight && ws)) return arg_error(who, "null pointer");
  if (!(aligned(tsdf, 4) && aligned(weight, 4) && aligned(ws, 256)))
    return arg_error(who, "misaligned array or workspace");
  if (ws_bytes < gsb_tsdf_extract_workspace_bytes(nx, ny, nz)) return arg_error(who, "workspace too small");
  return 0;
}

int gsb_tsdf_extract_plan(int nx, int ny, int nz, const float *tsdf, const float *weight, void *ws, size_t ws_bytes,
                          int64_t *counts_host, gsb_stream_t stream) {
  if (int rc = tsdf_grid_check(nx, ny, nz, 0.f, 0.f, 0.f, 1.f, "tsdf_extract_plan")) return rc;  // no geometry
  GSB_REQUIRE(counts_host != nullptr, "tsdf_extract_plan: counts_host is null");
  if (int rc = tsdf_extract_args(nx, ny, nz, tsdf, weight, ws, ws_bytes, "tsdf_extract_plan")) return rc;
  const TsdfGrid g{nx, ny, nz, 0.f, 0.f, 0.f, 1.f};
  if (int rc = launch_tsdf_extract_plan(g, tsdf, weight, ws, counts_host, (cudaStream_t)stream)) return rc;
  GSB_REQUIRE(counts_host[0] <= INT32_MAX && counts_host[1] <= INT32_MAX,
              "tsdf_extract_plan: 2^31 or more vertices or faces");
  return 0;
}

int gsb_tsdf_extract_emit(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float *tsdf,
                          const float *weight, const float *color_grid, const void *ws, size_t ws_bytes,
                          int64_t n_verts, int64_t n_faces, float *verts, float *vcolors, int32_t *faces,
                          gsb_stream_t stream) {
  if (int rc = tsdf_grid_check(nx, ny, nz, ox, oy, oz, voxel, "tsdf_extract_emit")) return rc;
  if (int rc = tsdf_extract_args(nx, ny, nz, tsdf, weight, ws, ws_bytes, "tsdf_extract_emit")) return rc;
  GSB_REQUIRE(n_verts >= 0 && n_faces >= 0 && n_verts <= INT32_MAX && n_faces <= INT32_MAX,
              "tsdf_extract_emit: vertex or face count out of range");
  GSB_REQUIRE(vcolors == nullptr || color_grid != nullptr, "tsdf_extract_emit: vertex colours without a colour grid");
  GSB_REQUIRE((n_verts == 0 || verts) && (n_faces == 0 || faces), "tsdf_extract_emit: null pointer");
  GSB_REQUIRE(aligned(verts, 4) && aligned(vcolors, 4) && aligned(faces, 4) && aligned(color_grid, 4),
              "tsdf_extract_emit: misaligned array");
  if (n_verts == 0 && n_faces == 0) return 0;
  const TsdfGrid g{nx, ny, nz, ox, oy, oz, voxel};
  return launch_tsdf_extract_emit(g, tsdf, weight, color_grid, ws, (int)n_verts, (int)n_faces, verts, vcolors, faces,
                                  (cudaStream_t)stream);
}

// ---- bilateral-grid colour correction (bilagrid.cu, DESIGN 3.20)
static_assert(BILAGRID_MAX_DIM == GSB_BILAGRID_MAX_DIM && BILAGRID_MAX_BATCH == GSB_BILAGRID_MAX_BATCH,
              "gsplat_b200.h and kernels.h disagree on the bilateral-grid limits");

static int bilagrid_shape(int M, int L, int Y, int X, const char *who) {
  if (M < 1) return arg_error(who, "M < 1");
  if (L < 1 || Y < 1 || X < 1 || L > GSB_BILAGRID_MAX_DIM || Y > GSB_BILAGRID_MAX_DIM || X > GSB_BILAGRID_MAX_DIM)
    return arg_error(who, "grid size out of [1, 64]");
  return 0;
}

// the checks of the slice and its backward; 0 or the argument error "<who>: <reason>"
static int bilagrid_slice_args(int M, int L, int Y, int X, const float *grids, int B, const int32_t *image_ids,
                               int H, int W, std::initializer_list<const void *> images, const char *who) {
  if (int rc = bilagrid_shape(M, L, Y, X, who)) return rc;
  if (B < 1 || B > GSB_BILAGRID_MAX_BATCH) return arg_error(who, "batch out of [1, 64]");
  if (H < 1 || W < 1) return arg_error(who, "bad H/W");
  if ((int64_t)H * W >= ((int64_t)1 << 31)) return arg_error(who, "2^31 or more pixels");
  if (image_ids == nullptr) return arg_error(who, "image_ids is null");
  for (int b = 0; b < B; b++)
    if (image_ids[b] < 0 || image_ids[b] >= M) return arg_error(who, "image id out of [0, M)");
  if (grids == nullptr) return arg_error(who, "null pointer");
  if (!aligned(grids, 4)) return arg_error(who, "misaligned array");
  for (const void *p : images) {
    if (p == nullptr) return arg_error(who, "null pointer");
    if (!aligned(p, 4)) return arg_error(who, "misaligned array");
  }
  return 0;
}

int gsb_bilagrid_slice(int M, int L, int Y, int X, const float *grids, int B, const int32_t *image_ids, int H, int W,
                       const float *rgb, float *out, gsb_stream_t stream) {
  if (int rc = bilagrid_slice_args(M, L, Y, X, grids, B, image_ids, H, W, {rgb, out}, "bilagrid_slice")) return rc;
  return launch_bilagrid_slice({M, L, Y, X}, grids, B, image_ids, H, W, rgb, out, (cudaStream_t)stream);
}

int gsb_bilagrid_slice_backward(int M, int L, int Y, int X, const float *grids, int B, const int32_t *image_ids,
                                int H, int W, const float *rgb, const float *dloss_dout, float *dloss_drgb,
                                float *dloss_dgrids, gsb_stream_t stream) {
  if (int rc = bilagrid_slice_args(M, L, Y, X, grids, B, image_ids, H, W, {rgb, dloss_dout, dloss_drgb, dloss_dgrids},
                                   "bilagrid_slice_backward"))
    return rc;
  return launch_bilagrid_slice_bwd({M, L, Y, X}, grids, B, image_ids, H, W, rgb, dloss_dout, dloss_drgb, dloss_dgrids,
                                   (cudaStream_t)stream);
}

size_t gsb_bilagrid_tv_workspace_bytes(int M, int L, int Y, int X) {
  if (bilagrid_shape(M, L, Y, X, "bilagrid_tv_workspace_bytes")) return 0;
  return bilagrid_tv_workspace_bytes({M, L, Y, X});
}

int gsb_bilagrid_tv(int M, int L, int Y, int X, const float *grids, float *tv_out, float *dloss_dgrids, void *ws,
                    size_t ws_bytes, gsb_stream_t stream) {
  if (int rc = bilagrid_shape(M, L, Y, X, "bilagrid_tv")) return rc;
  GSB_REQUIRE(grids && tv_out && ws, "bilagrid_tv: null pointer");
  GSB_REQUIRE(aligned(grids, 4) && aligned(tv_out, 4) && aligned(dloss_dgrids, 4) && aligned(ws, 8),
              "bilagrid_tv: misaligned array");
  GSB_REQUIRE(ws_bytes >= bilagrid_tv_workspace_bytes({M, L, Y, X}), "bilagrid_tv: workspace too small");
  return launch_bilagrid_tv({M, L, Y, X}, grids, tv_out, dloss_dgrids, ws, (cudaStream_t)stream);
}

// ---- compressed export (compress.cu, DESIGN 3.24)
static_assert(KMEANS_MAX_DIM == GSB_KMEANS_MAX_DIM, "gsplat_b200.h and kernels.h disagree on the k-means width");

// the shape checks of the k-means entry points; 0 or the argument error "<who>: <reason>"
static int kmeans_shape(int N, int K, int D, int64_t ldx, const char *who) {
  if (N < 0) return arg_error(who, "N < 0");
  if (K < 1) return arg_error(who, "K < 1");
  if (D < 1 || D > GSB_KMEANS_MAX_DIM) return arg_error(who, "D out of [1, 64]");
  if (K > INT32_MAX - 127) return arg_error(who, "K overflows the centroid index");
  if (ldx < D) return arg_error(who, "ldx < D");
  if (N > 0 && ldx > INT64_MAX / N) return arg_error(who, "N ldx overflows the row offset");
  return 0;
}

size_t gsb_kmeans_assign_workspace_bytes(int K, int D) {
  if (kmeans_shape(0, K, D, D, "kmeans_assign_workspace_bytes")) return 0;
  return kmeans_assign_workspace_bytes(K, D);
}

int gsb_kmeans_assign(int N, int K, int D, const float *x, int64_t ldx, const float *centroids, int32_t *labels,
                      float *dist, void *ws, size_t ws_bytes, gsb_stream_t stream) {
  if (int rc = kmeans_shape(N, K, D, ldx, "kmeans_assign")) return rc;
  GSB_REQUIRE(centroids && ws, "kmeans_assign: null pointer");
  GSB_REQUIRE(N == 0 || (x && labels && dist), "kmeans_assign: null pointer");
  GSB_REQUIRE(aligned(x, 4) && aligned(centroids, 4) && aligned(labels, 4) && aligned(dist, 4) && aligned(ws, 16),
              "kmeans_assign: misaligned array or workspace");
  GSB_REQUIRE(ws_bytes >= kmeans_assign_workspace_bytes(K, D), "kmeans_assign: workspace too small");
  return launch_kmeans_assign(N, K, D, x, ldx, centroids, labels, dist, ws, (cudaStream_t)stream);
}

int gsb_kmeans_update(int N, int K, int D, const float *x, int64_t ldx, const int32_t *labels, const int32_t *perm,
                      const float *centroids, float *centroids_out, int32_t *counts, gsb_stream_t stream) {
  if (int rc = kmeans_shape(N, K, D, ldx, "kmeans_update")) return rc;
  GSB_REQUIRE(centroids && centroids_out && counts, "kmeans_update: null pointer");
  GSB_REQUIRE(N == 0 || (x && labels && perm), "kmeans_update: null pointer");
  GSB_REQUIRE(aligned(x, 4) && aligned(labels, 4) && aligned(perm, 4) && aligned(centroids, 4) &&
                  aligned(centroids_out, 4) && aligned(counts, 4),
              "kmeans_update: misaligned array");
  return launch_kmeans_update(N, K, D, x, ldx, labels, perm, centroids, centroids_out, counts, (cudaStream_t)stream);
}

// the checks of the quantiser and its inverse
static int quant_shape(int N, int D, int bits, const char *who) {
  if (N < 0) return arg_error(who, "N < 0");
  if (D < 1 || D > GSB_KMEANS_MAX_DIM) return arg_error(who, "D out of [1, 64]");
  if (bits != 8 && bits != 16) return arg_error(who, "bits must be 8 or 16");
  return 0;
}

int gsb_quantize(int N, int D, const float *x, int64_t ldx, int bits, int log_transform, int fit_range, float *range,
                 void *codes, gsb_stream_t stream) {
  if (int rc = quant_shape(N, D, bits, "quantize")) return rc;
  GSB_REQUIRE(ldx >= D, "quantize: ldx < D");
  GSB_REQUIRE(N == 0 || ldx <= INT64_MAX / N, "quantize: N ldx overflows the row offset");
  GSB_REQUIRE(range != nullptr && (N == 0 || (x && codes)), "quantize: null pointer");
  GSB_REQUIRE(aligned(x, 4) && aligned(range, 4) && aligned(codes, bits / 8), "quantize: misaligned array");
  return launch_quantize(N, D, x, ldx, bits, log_transform != 0, fit_range != 0, range, codes, (cudaStream_t)stream);
}

int gsb_dequantize(int N, int D, const void *codes, int bits, const float *range, int log_transform, float *out,
                   gsb_stream_t stream) {
  if (int rc = quant_shape(N, D, bits, "dequantize")) return rc;
  GSB_REQUIRE(N == 0 || (codes && range && out), "dequantize: null pointer");
  GSB_REQUIRE(aligned(codes, bits / 8) && aligned(range, 4) && aligned(out, 4), "dequantize: misaligned array");
  return launch_dequantize(N, D, codes, bits, range, log_transform != 0, out, (cudaStream_t)stream);
}

}  // extern "C"
