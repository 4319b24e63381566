// Internal launcher prototypes (host side, C++).  The public surface is include/gsplat_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

struct gsb_adam_tensor;

namespace gsb {

struct Rec;

// ---- launch accounting / optional per-kernel CUDA-event timing (api.cu).  Every launcher
// opens a ProfScope; the launch counter always runs, events are recorded only while
// gsb_profile_enable(1) is in effect (bench.py's roofline leg).
enum KernelId {
  K_PROJECT = 0, K_COV3D, K_COV2D, K_SH2COLOR, K_INVCOV, K_RECTS, K_SCAN, K_KEYS, K_SORT, K_RANGES,
  K_PACK, K_DRAW, K_DRAW_BWD, K_PRE_FWD, K_PRE_BWD, K_FINALIZE, K_LOSS_FWD, K_LOSS_BWD, K_BMM,
  K_DENSITY_ACC, K_DENSITY_CLASSIFY, K_DENSITY_SCAN, K_DENSITY_APPLY, K_RESET_ALPHA, K_GS_DECODE,
  K_GS_TO_PARAMS, K_PARAMS_TO_GS, K_GRAD_EXCHANGE, K_SH_EXPAND, K_FILTER3D, K_FILTER3D_APPLY, K_FILTER3D_BWD,
  K_SURFEL_FWD_BATCH, K_DRAW_SURFEL_BATCH, K_DRAW_SURFEL_BWD_BATCH, K_SURFEL_BWD_BATCH, K_DRAW_2DGS_BATCH,
  K_DRAW_2DGS_BWD_BATCH, K_RECTS_BATCH, K_PRE_FWD_BATCH, K_PRE_BWD_BATCH, K_DRAW_BATCH, K_DRAW_RGBD_BATCH, K_DRAW_BWD_BATCH,
  K_DRAW_BWD_RGBD_BATCH, K_KMEANS_ASSIGN, K_KMEANS_UPDATE, K_QUANTIZE, K_DEQUANTIZE, K_DENSITY_ROWS, K_BILAGRID_SLICE, K_BILAGRID_SLICE_BWD, K_BILAGRID_TV, K_DRAW_FEAT, K_DRAW_FEAT_BWD, K_DRAW_STATS, K_DRAW_SURFEL_STATS, K_MCMC_SCAN, K_MCMC_SAMPLE, K_MCMC_RELOCATE, K_MCMC_GROW,
  K_MCMC_ROWS, K_MCMC_NOISE, K_TSDF_INTEGRATE, K_TSDF_PLAN, K_TSDF_EMIT,
  K_SURFEL_FWD, K_DRAW_SURFEL, K_DRAW_SURFEL_BWD, K_SURFEL_BWD, K_DRAW_2DGS, K_DRAW_2DGS_BWD,
  K_DRAW_BWD_ABS, K_DRAW_BWD_RGBD_ABS, K_ADAM, K_DRAW_RGBD, K_DRAW_BWD_RGBD, K_COUNT
};
struct ProfScope {
  ProfScope(int id, cudaStream_t st);
  ~ProfScope();
  int id_;
  cudaStream_t st_;
  cudaEvent_t stop_;
};

int launch_project(int N, const float *pws, const float *Rcw, const float *tcw, float fx, float fy,
                   float cx, float cy, float *us, float *pcs, float *depths, float *du_dpcs,
                   cudaStream_t st);
int launch_cov3d(int N, const float *rots, const float *scales, const float *depths, float *cov3ds,
                 float *Jr, float *Js, cudaStream_t st);
int launch_cov2d(int N, const float *cov3ds, const float *pcs, const float *Rcw, const float *depths,
                 float fx, float fy, float width, float height, float *cov2ds, float *Jc, float *Jp,
                 cudaStream_t st);
int launch_sh2color(int N, int k3, const float *shs, const float *pws, const float *twc, float *colors,
                    float *Js, float *Jp, cudaStream_t st);
int launch_inv_cov2d(int N, const float *cov2ds, float *depths, float *cinv2ds, int32_t *areas,
                     float *J, cudaStream_t st);

// ---- fused per-Gaussian path (fused.cu)
// camera model of the fused per-Gaussian kernels (gsb_camera_model)
struct CamLens {
  int model;      // pg::CamModel
  float k[4];     // FISHEYE's k1..k4, OPENCV's k1, k2, p1, p2
  float stretch;  // OPENCV: the clamp limits' factor r_u / r_d (DESIGN 3.19); 1 otherwise
};
// the Gaussians and the view: what every fused call is about
struct FusedScene {
  int N, k3;  // k3 = shs.shape[1] / 3
  const float *pws, *rots, *scales, *shs, *Rcw, *tcw, *twc;
  float fx, fy, cx, cy, width, height;
  // NULL or PINHOLE (the reference's projection), or ORTHO / FISHEYE / OPENCV with their k
  // (pg_fused_math.h; the backward's non-pinhole forms take the moment rows and no exchange)
  const CamLens *lens;
};
// the forward's outputs and the opacities it may read.  alphas with recs: also the rasterizers'
// records.  alphas_eff: NULL, or antialiasing (alphas required): alphas_eff[N] = rho alpha, also in
// recs.  (The fields of FusedFwd and FusedBwd follow the entry points' argument order.)
struct FusedFwd {
  float *us, *cinv2ds, *colors, *depths;
  int32_t *areas;
  const float *alphas;
  Rec *recs;
  float *alphas_eff;
};
int launch_preprocess_fwd(const FusedScene &sc, const FusedFwd &f, cudaStream_t st);
// upstream gradients given as the rasterizer backward's moment rows (fused.cu, MOM variants)
struct MomentsIn {
  const float *moments;  // [N,9]
  const float *cinv2ds;  // [N,3]
  float *dus_out;        // [N,2]  dL/du, still needed by the caller
  float *dalphas_out;    // [N]    dL/dalpha (nullable: the push variant forwards it instead)
};
struct GradPush;
// the camera gradient (fused.cu, POSE variants): gcam[15] = dL/dRcw (9), dL/dtcw (3), dL/dtwc (3);
// part = ceil(N/128) partial rows of 16 floats (16-byte aligned), one per CTA.  gint: NULL, or also the
// intrinsics gradient gint[8] = dL/d(fx, fy, cx, cy, k[4]) (DESIGN 3.23, k_preprocess_bwd_intrinsics;
// moment rows required); then the rows are 24 floats wide.
struct PoseOut {
  float *gcam;
  float *part;
  float *gint;
};
constexpr size_t pose_workspace_bytes(int N) { return N > 0 ? (size_t)((N + 127) / 128) * 16 * sizeof(float) : 0; }
constexpr size_t intrinsics_workspace_bytes(int N) {
  return N > 0 ? (size_t)((N + 127) / 128) * 24 * sizeof(float) : 0;
}
// The backward's gradients in and out.  gp == nullptr: the gradients go to g_pws, g_shs, g_scales,
// g_rots; otherwise into the exchange staging slots gp describes (the g_* outputs are unused).
// mi.moments == nullptr: the upstream gradients are g_us, g_cinv2ds, g_colors; otherwise the moment
// rows of mi.  g_depths: NULL, or dL/dz[N] of the RGB-D rasterizer (not with gp).  po: NULL, or also
// the camera gradient (not with gp; a pass of its own); then g_pws == NULL (with g_shs, g_scales,
// g_rots and mi's outputs NULL) writes only that.  alphas: NULL, or antialiasing (the raw
// opacities; only with mi, not with gp): the moment rows' dL/dalpha is dL/dalpha_eff.  The fields
// are checked by the entry points (api.cu check_preprocess_backward).
struct FusedBwd {
  const float *g_us, *g_cinv2ds, *g_colors;
  float *g_pws, *g_shs, *g_scales, *g_rots;
  MomentsIn mi;
  const float *g_depths;
  const float *alphas;
  const PoseOut *po;
  const GradPush *gp;
};
int launch_preprocess_bwd(const FusedScene &sc, const FusedBwd &b, cudaStream_t st);

// the kernels' tan_fovx, tan_fovy of a scene whose lens camera_lens (api.cu) has set
float2 lens_tan_fov(const FusedScene &sc);

// ---- batched per-Gaussian path (fused.cu, DESIGN 3.21).  The intrinsics of the C cameras travel
// in kernel parameter memory (nothing to copy to the device, nothing to wait for): C <= 64.
constexpr int BATCH_MAX_CAMERAS = 64;
struct BatchCams {
  float4 f[BATCH_MAX_CAMERAS];   // fx, fy, cx, cy
  float4 k[BATCH_MAX_CAMERAS];   // the lens's k (FISHEYE, OPENCV)
  float2 tf[BATCH_MAX_CAMERAS];  // tan_fovx, tan_fovy (lens_tan_fov)
};
// the Gaussians and C cameras of one model and image size: poses [C,15] = Rcw (9), tcw (3), twc (3)
// per camera in device memory, cams on the host
struct BatchScene {
  int C, N, k3;
  const float *pws, *rots, *scales, *shs, *poses;
  int model;  // pg::CamModel
  const BatchCams *cams;
};
// f: the [C, N, ...] outputs (alphas [N] and recs [C N] required; alphas_eff [C, N]: antialiasing)
int launch_preprocess_fwd_batch(const BatchScene &b, const FusedFwd &f, cudaStream_t st);
// moments [C N, 9], cinv2ds [C N, 3], g_depths NULL or [C N] (RGB-D), alphas NULL or the raw
// opacities [N] (antialiasing); outputs dus_out [C N, 2], dalphas_out [N] and the four gradients.
// po: NULL, or also the camera gradients (DESIGN 3.22): gcam [C, 15], part C ceil(N/128) rows of 16
// floats (16-byte aligned), in a pass of its own; then g_pws == NULL (with the other per-Gaussian
// outputs NULL) writes only those.
struct BatchBwd {
  const float *moments, *cinv2ds, *g_depths, *alphas;
  float *dus_out, *dalphas_out, *g_pws, *g_shs, *g_scales, *g_rots;
  const PoseOut *po;
};
constexpr size_t batch_pose_workspace_bytes(int C, int N) { return (size_t)C * pose_workspace_bytes(N); }
constexpr size_t batch_intrinsics_workspace_bytes(int C, int N) { return (size_t)C * intrinsics_workspace_bytes(N); }
int launch_preprocess_bwd_batch(const BatchScene &b, const BatchBwd &g, cudaStream_t st);

// dL/dsh[N,3k] = sum over V views of Y(dir_v) (x) dL/dcolor_v  (fused.cu k_sh_expand)
int launch_sh_expand(int N, int k3, int V, const float *pws, const float *twcs, const float *gcols, float *g_shs,
                     cudaStream_t st);

// ---- Mip-Splatting 3D smoothing filter (filter3d.cu; the math is pg_fused_math.h filter3d_*).
// cams: the [C][20] training-camera table (pg::kCamRow); ws: 2 words, zeroed here.  C == 0 gives
// zeros.  The backward's outputs may alias dscales_f / dalphas_f.
constexpr int F3_CHUNK = 64;  // cameras k_filter3d_depth stages in shared memory at once (GSB_FILTER3D_CHUNK)
constexpr size_t filter3d_workspace_bytes() { return 16; }
int launch_filter3d(int N, const float *pws, int C, const float *cams, float variance, float *filter3d,
                    unsigned int *ws, cudaStream_t st);
int launch_filter3d_apply(int N, const float *scales, const float *alphas, const float *filter3d, float *scales_f,
                          float *alphas_f, cudaStream_t st);
int launch_filter3d_bwd(int N, const float *scales, const float *alphas, const float *filter3d,
                        const float *dscales_f, const float *dalphas_f, float *dscales, float *dalphas,
                        cudaStream_t st);

// ---- multi-GPU gradient exchange (comm.cu; the producer is the PUSH variant in fused.cu).
// Every rank owns one region of peer-mapped memory:
//   [control 4 KiB: arrive[8] u32 @0, done[8] u32 @64, counters @128/@132, status @136]
//   [staging: world slots x (rpr rows x (ks+11) floats), slot s = what rank s pushed here]
//   [result:  world*rpr rows x (ks+11) floats, the summed gradients, identical on every rank]
// Tiles of 128 Gaussians are dealt round-robin: rank r owns global tiles r, r + world, ...
// (local tile lt <-> global tile lt * world + r), rpr = tiles_per_rank * 128 rows per rank;
// slot and result keep the SoA segment order shs | rots | pws | scales | alphas.
constexpr int kMaxWorld = 8;
constexpr size_t kCtrlBytes = 4096;
struct ExchangeGeom {
  int world, ks, tiles_per_rank;
  long long rpr, rows_total, slot_floats;
  long long slot_off[5], result_off[5];  // float offsets of the 5 segments inside a slot / the result
  int seg_k[5];
  size_t staging_off, result_base, bytes;  // byte offsets inside the region
};
ExchangeGeom exchange_geom(int N, int k3, int world);
struct GradPush {
  float *slot[kMaxWorld];      // staging slot `rank` on each owner
  uint32_t *flags[kMaxWorld];  // arrive[] array of each rank
  uint32_t *counter;
  const float *g_alphas;       // dL/dalpha of this view (unused when the moment rows are given)
  long long off_rots, off_pws, off_scales, off_alphas;  // float offsets of the segments inside a slot
  int world, rank;
  uint32_t epoch;
};
int launch_grad_reduce_bcast(const ExchangeGeom &G, int rank, void *const *regions, uint32_t epoch,
                             cudaStream_t st);

// ---- batched tiny matmul for the reference's Jacobian chain (smallbmm.cu)
int launch_small_bmm(long long batch, int M, int K, int NN, const float *A, const float *B, int b_shared,
                     float *C, cudaStream_t st);

// ---- fused training loss (loss.cu)
size_t gau_loss_workspace_bytes(int H, int W);
int launch_gau_loss(int H, int W, const float *img, const float *gt, float lambda, float *loss_out,
                    float *grad, void *ws, cudaStream_t st);

// ---- density control + Gaussian record conversion (density.cu).  Tensor order everywhere:
// pws, low_shs, high_shs, alphas_raw, scales_raw, rots_raw (widths 3, 3, 45, 1, 3, 4).
size_t density_workspace_bytes(int64_t N);
int launch_density_accumulate(int64_t N, const float *dloss_dus, const uint8_t *mask, float *grad_accum,
                              int32_t *cunt, int init, cudaStream_t st);
int launch_density_plan(int64_t N, const float *alphas_raw, const float *scales_raw, const float *grad_accum,
                        const int32_t *cunt, float alpha_raw_min, float scale_raw_max, float grad_min,
                        float scale_clone_max, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                        int64_t *counts_host, cudaStream_t st);
// the plan of a prune by mask: cls = CLS_KEEP where keep[i] != 0, else CLS_PRUNE, the same slots
// scan; counts_host <- (K, 0, 0)
int launch_density_plan_keep(int64_t N, const uint8_t *keep, void *ws, uint8_t *cls, int32_t *slots,
                             int64_t *counts_host, cudaStream_t st);
int launch_density_apply(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C,
                         float *const *src, float *const *src_m, float *const *src_v, const float *z,
                         float *const *dst, float *const *dst_m, float *const *dst_v, cudaStream_t st);
// the same plan applied to one more [N, D] tensor and its Adam moments (src_m .. dst_v: all NULL or
// all set): survivors, then clones, then splits, each new row a copy of its source (moments: 0)
int launch_density_apply_rows(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int D,
                              const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                              float *dst_v, cudaStream_t st);
int launch_reset_alpha(int64_t N, float *alphas_raw, float *m, float *v, float val, cudaStream_t st);
// MCMC densification (density.cu, DESIGN 3.11).  ws: mcmc_workspace_bytes(N, n) bytes, 256-B
// aligned, shared by the calls of one relocate / grow; mode 0 samples alive rows (relocate) and
// lists the dead ones, mode 1 samples every non-NaN row (grow).  counts_host <- (W_total, dead count).
size_t mcmc_workspace_bytes(int64_t N, int64_t n);
int launch_mcmc_plan(int64_t N, const float *alphas_raw, float alpha_raw_min, int mode, void *ws,
                     int64_t *counts_host, cudaStream_t st);
int launch_mcmc_sample(int64_t N, int64_t n, const double *u, void *ws, int32_t *sampled, cudaStream_t st);
int launch_mcmc_relocate(int64_t N, int64_t n, const int32_t *sampled, void *ws, double min_opacity, int n_max,
                         float *const *p, float *const *m, float *const *v, cudaStream_t st);
int launch_mcmc_relocate_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, int D, float *x,
                              float *m, float *v, cudaStream_t st);
int launch_mcmc_grow(int64_t N, int64_t n, const int32_t *sampled, void *ws, double min_opacity, int n_max,
                     float *const *src, float *const *src_m, float *const *src_v, float *const *dst,
                     float *const *dst_m, float *const *dst_v, cudaStream_t st);
int launch_mcmc_grow_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, int D, const float *src,
                          const float *src_m, const float *src_v, float *dst, float *dst_m, float *dst_v,
                          cudaStream_t st);
int launch_mcmc_noise(int64_t N, float *pws, const float *alphas_raw, const float *scales_raw, const float *rots_raw,
                      const float *z, float scale, float k, float x0, cudaStream_t st);
int launch_ply_rows_to_gs(int64_t N, int stride, int sh_dim, const float *rows, const int32_t *colmap, float *gs,
                          cudaStream_t st);
int launch_gs_to_params(int64_t N, int sh_dim, const float *gs, float *const *dst, cudaStream_t st);
int launch_params_to_gs(int64_t N, float *const *src, float *gs, cudaStream_t st);

// ---- fused Adam step (adam.cu, DESIGN 3.12): the table of gsb_adam_step, checked by the entry
// point; visibility NULL is dense Adam
int launch_adam(int n_tensors, const gsb_adam_tensor *table, const uint8_t *visibility, double beta1, double beta2,
                double eps, cudaStream_t st);

// ---- binning (binning.cu)
struct BinLayout {  // carve-up of the phase-1 workspace
  size_t rects, offsets, total, scan_desc, bytes;  // total: [P, max depth key, flags, scan claim] u32
};
BinLayout bin_layout(int N);
int launch_bin(int H, int W, int N, const float *us, float *depths, int32_t *areas, void *ws,
               const BinLayout &L, cudaStream_t st);
// phase 1 of a batch of C frames binned as one tall frame (DESIGN 3.21): us / depths / areas hold
// the C N records (record c N + n: Gaussian n in camera c), L = bin_layout(C N); record c N + n's
// rectangle is the single frame's, clamped to frame c's gy tile rows and moved down by c gy rows.
int launch_bin_batch(int C, int H, int W, int N, const float *us, float *depths, int32_t *areas, void *ws,
                     const BinLayout &L, cudaStream_t st);
// the tall frame's height in pixels: C whole-tile frames (its phase 2 is the single frame's at this height)
constexpr int batch_height(int C, int H) { return C * ((H + 15) / 16) * 16; }

struct SortLayout {  // carve-up of the phase-2 workspace
  size_t keys_a, keys_b, vals_a, vals_b, recs, counters;
  size_t sort_state, desc;  // radix-sort scan: claim counter, look-back descriptors (reset per pass)
  size_t counts;            // [digit][sort tile] counts, then scatter bases
  size_t bytes;
};
SortLayout sort_layout(int N, int H, int W, int64_t P);
// carve-up of splatB's workspace, as offsets from `base`, the address it starts at (any byte):
// [records, only when they are rebuilt (P > 0), 256-B aligned] [N x 9 moment rows] [rasterizer
// work area].  bytes covers the split from that start.
struct BwdLayout {
  size_t recs, moments, work, bytes;
};
BwdLayout bwd_layout(int N, int H, int W, int64_t P, uintptr_t base);
// capacity-based path: where to copy [P, max depth key, flags] for the host, and the event that
// tells it the copy has landed (recorded right after the key kernel)
struct StatusRead {
  uint32_t *host;
  cudaEvent_t ready;
};
int launch_sort_and_pack(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                         const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                         const void *bin_ws, const BinLayout &BL, void *ws, const SortLayout &SL,
                         int32_t *ranges, int32_t *gsid_per_patch, bool pack, const StatusRead *sr,
                         cudaStream_t st);
// depths: nullable; the records' depth word (q2.w) is 0 without them
int launch_pack_only(int64_t P, const int32_t *gsid_per_patch, const float *us, const float *cinv2ds,
                     const float *alphas, const float *colors, const float *depths, Rec *recs, cudaStream_t st);

// ---- rasterizer (raster_fwd.cu, raster_bwd.cu).  recs: one 48-byte record per Gaussian; gsid: the
// sorted patch list -- the kernels gather records through it.  work = [item counter, #entries,
// entries ...] (2 + 4 * tiles ints, see k_tile_list); with outputs given the empty tiles are
// zero-filled there.
// depth_image / alpha_image: both NULL (colour frame), or the RGB-D frame's D and A planes [H,W]
// (k_draw_rgbd; the records' depth word must hold z).
// frames > 0: the tall frame of a batch of `frames` H x W frames (DESIGN 3.21): ranges of its
// frames * gx * gy tiles, planes [frames, ..., H, W] (k_tile_list_batch, k_draw_batch, k_draw_rgbd_batch)
int launch_tile_list(int H, int W, const int32_t *ranges, float *image, int32_t *contrib, float *final_tau,
                     float *depth_image, float *alpha_image, int *work, cudaStream_t st, int frames = 0);
int launch_draw(int H, int W, const int32_t *ranges, const Rec *recs, const int32_t *gsid, float *image,
                int32_t *contrib, float *final_tau, float *depth_image, float *alpha_image, int *work,
                cudaStream_t st, int frames = 0);
// the RGB-D backward's extra upstream planes [H,W] and its dL/dz output [N] (zeroed here)
struct DepthGrads {
  const float *dloss_ddepth_image;
  const float *dloss_dalpha_image;
  float *ddepths;
};
// dg == nullptr: k_draw_bwd; otherwise k_draw_bwd_rgbd.  dus_abs: NULL, or [N,2] (any 4-byte
// alignment, zeroed here) for the per-pixel absolute sums of dL/du: then k_draw_bwd_abs /
// k_draw_bwd_rgbd_abs.  frames > 0: as for launch_draw (N = all records of the batch; no dus_abs):
// k_draw_bwd_batch / k_draw_bwd_rgbd_batch
int launch_draw_backward(int H, int W, int N, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                         const int32_t *contrib, const float *final_tau, const float *dloss_dgammas,
                         const DepthGrads *dg, const float *cinv2ds, float *moments, int *work, float *dloss_dus,
                         float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, bool finalize,
                         float *dus_abs, cudaStream_t st, int frames = 0);

// ---- feature rasterizers (raster_feat.cu): replays of the colour forward's binning that composite
// features[N,D] (row stride D, any 4-byte alignment) with the image's weights.  ranges: any
// alignment; work: the 2 + 4 * tiles ints of launch_tile_list.  recs == nullptr: no patches.
// The forward writes every element of feature_image[D,H,W] (16-byte aligned).  The backward ADDS
// its terms to moment rows 0-5 of moments[N,9] and writes every element of dloss_dfeatures[N,D].
int launch_draw_features(int H, int W, int D, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                         const int32_t *contrib, const float *features, float *feature_image, int *work,
                         cudaStream_t st);
int launch_draw_features_backward(int H, int W, int N, int D, const int32_t *ranges, const Rec *recs,
                                  const int32_t *gsid, const int32_t *contrib, const float *final_tau,
                                  const float *features, const float *dloss_dfeature_image, float *moments,
                                  float *dloss_dfeatures, int *work, cudaStream_t st);
// carve-up of the feature passes' workspace from `base` (any byte): [records, only when they are
// rebuilt (P > 0), 256-B aligned] [rasterizer work area]
struct FeatLayout {
  size_t recs, work, bytes;
};
FeatLayout feat_layout(int N, int H, int W, int64_t P, uintptr_t base);

// ---- contribution statistics (raster_stats.cu, surfel.cu; DESIGN 3.18): replays of a drawn frame
// that ADD per-Gaussian sums of the blending weights w, their maximum (weight_max[N] updated as the
// uint bits of w >= 0) and the count of pixels with w > 0.  weight_sum / weight_max: any 4-byte
// alignment, hit_count 8-byte aligned.  recs == nullptr: no patches, nothing added.  The colour
// replay takes feat_layout's records and work area (launch_tile_list's); the surfel replay launches
// one CTA per tile and needs no work area.
int launch_draw_stats(int H, int W, const int32_t *ranges, const Rec *recs, const int32_t *gsid,
                      const int32_t *contrib, float *weight_sum, float *weight_max, int64_t *hit_count, int *work,
                      cudaStream_t st);
int launch_draw_surfel_stats(int H, int W, const int32_t *ranges, const float *recs, const int32_t *gsid,
                             const int32_t *contrib, float *weight_sum, float *weight_max, int64_t *hit_count,
                             cudaStream_t st);

// ---- 2D Gaussian Splatting (surfel.cu, DESIGN 3.15; the math is surfel_math.h).  recs: one 80-byte
// record per surfel ([N,20] floats, 16-byte aligned); rows: the backward rasterizer's [N,18]
// gradient rows [dM (9), dalpha, dcolour (3), dn (3), ddelta (2)], zeroed by its launcher.
int launch_surfel_fwd(const FusedScene &sc, const float *alphas, float *us, float *depths, int32_t *areas, float *colors,
                      float *recs, cudaStream_t st);
int launch_surfel_bwd(const FusedScene &sc, const float *rows, float *g_pws, float *g_shs, float *g_alphas,
                      float *g_scales, float *g_rots, float *g_us, cudaStream_t st);
// their batch forms (DESIGN 3.25): C pinhole cameras (b.model unused), us / depths / areas / colors
// [C, N, ...] and recs [C N, 20]; rows [C N, 18] -> the summed per-surfel gradients and g_us [C, N, 2]
int launch_surfel_fwd_batch(const BatchScene &b, const float *alphas, float *us, float *depths, int32_t *areas,
                            float *colors, float *recs, cudaStream_t st);
int launch_surfel_bwd_batch(const BatchScene &b, const float *rows, float *g_pws, float *g_shs, float *g_alphas,
                            float *g_scales, float *g_rots, float *g_us, cudaStream_t st);
// The 2DGS geometry planes (DESIGN 3.16) of one frame, on the NDC-mapped hit depth
// m(z) = mscale (1 - near / max(z, near)), mscale = far / (far - near):
// distortion[H,W] = sum_{j<i} w_i w_j (m_i - m_j)^2, moments[2,H,W] = (sum w m, sum w m^2),
// median_depth[H,W] = z of the last contributing record whose incoming tau > 0.5 (0: none) and
// median_contrib[H,W] = its patch index in the tile + 1 (0: none).
struct GeoPlanes {
  float *distortion, *moments, *median_depth;
  int32_t *median_contrib;
  float near, mscale;
};
// Their backward: the upstream dL/d(distortion), dL/d(median_depth) (NULL reads as zero) and the
// forward's alpha plane (the final sum w), moments and median_contrib.
struct GeoGrads {
  const float *distortion, *median, *alpha, *moments;
  const int32_t *median_contrib;
  float near, mscale;
};
// work: launch_tile_list's work area; recs == nullptr: no patches (zeros only).  The normal plane
// [3,H,W] is written like the image planes.  geo: also the geometry planes (k_draw_2dgs), or NULL
// (k_draw_surfel).  frames > 0: the tall frame of a batch of `frames` H x W frames (DESIGN 3.25):
// ranges of its frames gx gy tiles, every plane [frames, ..., H, W] (k_draw_disk_batch, k_draw_2dgs_batch).
int launch_draw_surfel(int H, int W, const int32_t *ranges, const float *recs, const int32_t *gsid, float *image,
                       int32_t *contrib, float *final_tau, float *depth_image, float *alpha_image, float *normal_image,
                       const GeoPlanes *geo, int *work, cudaStream_t st, int frames = 0);
// the upstream planes dl_*: NULL reads as zero (all NULL: the rows stay 0).  geo with an upstream
// geometry plane: k_draw_2dgs_bwd adds the geometry terms; otherwise k_draw_surfel_bwd runs.
// frames > 0: as for launch_draw_surfel, N = all records of the batch (k_draw_disk_bwd_batch,
// k_draw_2dgs_bwd_batch).
int launch_draw_surfel_backward(int H, int W, int N, const int32_t *ranges, const float *recs, const int32_t *gsid,
                                const int32_t *contrib, const float *final_tau, const float *dl_image,
                                const float *dl_depth, const float *dl_alpha, const float *dl_normal,
                                const GeoGrads *geo, float *rows, int *work, cudaStream_t st, int frames = 0);

// ---- mesh extraction (tsdf.cu, DESIGN 3.17; the fp64 model is oracle/tsdf_oracle.py).  The grid:
// nx x ny x nz points, point (i, j, k) at origin + voxel (i, j, k), arrays [nz, ny, nx] (x fastest),
// colour [3, nz, ny, nx]; N = nx ny nz < 2^31, checked by the entry points.
struct TsdfGrid {
  int nx, ny, nz;
  float ox, oy, oz, voxel;
};
// cams: V rows of the [V, 20] camera table (ops.camera_table); depth [V, H, W]; color [V, 3, H, W]
// and color_grid: both NULL or both set
int launch_tsdf_integrate(const TsdfGrid &g, float trunc, float depth_trunc, int V, int H, int W, const float *cams,
                          const float *depth, const float *color, float *tsdf, float *weight, float *color_grid,
                          cudaStream_t st);
// ws: tsdf_extract_workspace_bytes(N) bytes, 256-B aligned, carried from the plan to the emit;
// counts_host <- (vertices, faces) after a host synchronisation
size_t tsdf_extract_workspace_bytes(int64_t N);
int launch_tsdf_extract_plan(const TsdfGrid &g, const float *tsdf, const float *weight, void *ws,
                             int64_t *counts_host, cudaStream_t st);
// writes vertex ids < n_verts and face slots < n_faces only, whatever the workspace holds
int launch_tsdf_extract_emit(const TsdfGrid &g, const float *tsdf, const float *weight, const float *color_grid,
                             const void *ws, int n_verts, int n_faces, float *verts, float *vcolors, int32_t *faces,
                             cudaStream_t st);

// ---- bilateral-grid colour correction (bilagrid.cu, DESIGN 3.20).  grids[M, 12, L, Y, X]; the shape
// and the ids are checked by the entry points.  rgb, out, dout, drgb: B planar [3, H, W] images; item
// b reads grid ids[b].  The backward writes drgb and ADDS into dgrids.  The TV writes dgrids (when
// not NULL) and the value to tv[0] through bilagrid_tv_workspace_bytes of per-CTA partial sums.
constexpr int BILAGRID_MAX_DIM = 64, BILAGRID_MAX_BATCH = 64;
struct BilagridShape {
  int M, L, Y, X;
};
int launch_bilagrid_slice(const BilagridShape &s, const float *grids, int B, const int32_t *ids, int H, int W,
                          const float *rgb, float *out, cudaStream_t st);
int launch_bilagrid_slice_bwd(const BilagridShape &s, const float *grids, int B, const int32_t *ids, int H, int W,
                              const float *rgb, const float *dout, float *drgb, float *dgrids, cudaStream_t st);
size_t bilagrid_tv_workspace_bytes(const BilagridShape &s);
int launch_bilagrid_tv(const BilagridShape &s, const float *grids, float *tv, float *dgrids, void *ws,
                       cudaStream_t st);

// ---- compressed export (compress.cu, DESIGN 3.24).  x[N, D] rows ldx floats apart (any 4-byte
// alignment), 1 <= D <= KMEANS_MAX_DIM; centroids [K, D] contiguous.  The arguments are checked by the
// entry points.
constexpr int KMEANS_MAX_DIM = 64;
// K rounded up to the 128-centroid tile; ws of the assignment: the transposed codebook and its norms
int kmeans_padded(int K);
size_t kmeans_assign_workspace_bytes(int K, int D);
int launch_kmeans_assign(int N, int K, int D, const float *x, int64_t ldx, const float *centroids, int32_t *labels,
                         float *dist, void *ws, cudaStream_t st);
// perm: a stable ascending sort of labels (member lists in ascending point index)
int launch_kmeans_update(int N, int K, int D, const float *x, int64_t ldx, const int32_t *labels, const int32_t *perm,
                         const float *centroids, float *centroids_out, int32_t *counts, cudaStream_t st);
// range[2, D] (lo row, hi row): fit_range: reduced here, else read; codes [N, D] uint8 (bits 8) or uint16
int launch_quantize(int N, int D, const float *x, int64_t ldx, int bits, int log_t, int fit_range, float *range,
                    void *codes, cudaStream_t st);
int launch_dequantize(int N, int D, const void *codes, int bits, const float *range, int log_t, float *out,
                      cudaStream_t st);

}  // namespace gsb
