/*
 * gsplat_b200.h -- C ABI of the H100-native differentiable 3DGS rasterizer.
 *
 * This is the drop-in boundary for the hot path of scomup/EasyGaussianSplatting: the seven
 * operators its pybind11 module `gsplatcu` exports (reference gsplatcu/ext.cpp:68-76, host
 * launchers gsplatcu/gausplat.cu).  The reference has no C ABI of its own -- its boundary
 * is `std::vector<torch::Tensor> f(torch::Tensor...)` -- so each entry point below is what
 * a maintainer would call from those launchers instead of the `<<<>>>` launches
 * (INTEGRATION.md shows the binding).  The Python package `gsplatcu/` in this repository
 * binds them with ctypes and reproduces the reference's Python operator surface.
 *
 * Conventions (all entry points):
 *   - plain C, no torch / C++ types; every pointer is a DEVICE pointer unless the name ends
 *     in `_host`; tensors are dense row-major float32 (int32 where stated);
 *   - caller owns every buffer, including workspaces (sizes from the *_workspace_bytes
 *     queries); nothing is allocated or freed inside;
 *   - stream-ordered on `stream` (a cudaStream_t passed as void*); no device-wide sync.
 *     The only host synchronisation is gsb_splat_bin's wait for the patch count P;
 *   - return 0 on success, non-zero (a cudaError_t value, or -1 for argument errors)
 *     otherwise; gsb_last_error() returns a thread-local description;
 *   - N == 0 / P == 0 are valid and produce empty / zero outputs (the reference reads out
 *     of bounds for N == 0, gausplat.cu:67, and drops the image for P == 1,
 *     kernel.cu:140-143; both are handled here).
 *   - "culled" Gaussians (depths[i] < 0.2) get all-zero outputs, exactly what the
 *     reference's zero-filled tensors hold for them.
 *   - any float32 / int32 array may start at any 4-byte boundary (e.g. a slice of one flat
 *     buffer at an odd offset): row-wise vector loads and stores are only used when the base
 *     pointer is aligned for them.  The exceptions are buffers the caller allocates for the
 *     call: packed_records must be 16-byte aligned, and so must gsb_splat_render's /
 *     gsb_splat_forward's image, contrib and final_tau, the sort workspace `ws` of those and of
 *     gsb_splat_forward_enqueue, and the binning workspace `bin_ws` of those and of
 *     gsb_splat_bin; their patch_range_per_tile must be 8-byte aligned.  A misaligned one is
 *     an argument error.  (gsb_splat_backward's `ws` may start anywhere.)
 */
#ifndef GSPLAT_B200_H_
#define GSPLAT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_ABI_VERSION 1
#define GSB_TILE 16            /* reference common.cuh:13 BLOCK */
#define GSB_MAX_GRID_TILES 65535 /* tiles per row and per column the binning entry points accept:
                                  * W, H <= 1 048 560 pixels; larger frames are refused */
#define GSB_RECORD_BYTES 48    /* packed per-Gaussian record, see DESIGN.md "data layout" */

typedef void *gsb_stream_t; /* cudaStream_t */

int gsb_abi_version(void);
const char *gsb_last_error(void);

/* F.1.1/F.1.2/B.1.2.  Replaces `project` (ext.cpp:54-61, gausplat.cu:253-296, kernel.cu:553-617).
 * pws[N,3], Rcw[3,3], tcw[3] -> us[N,2], pcs[N,3], depths[N] (-1 where z < 0.2),
 * du_dpcs[N,2,3] (nullable = calc_J false). */
int gsb_project(int N, const float *pws, const float *Rcw, const float *tcw, float fx, float fy,
                float cx, float cy, float *us, float *pcs, float *depths, float *du_dpcs,
                gsb_stream_t stream);

/* F.2/B.2.  Replaces `computeCov3D` (ext.cpp:39-42, gausplat.cu:162-199, kernel.cu:326-423).
 * rots[N,4] (w,x,y,z; used un-normalised), scales[N,3], depths[N] -> cov3ds[N,6] (upper
 * triangle), dcov3d_drots[N,6,4], dcov3d_dscales[N,6,3] (both nullable together). */
int gsb_compute_cov3d(int N, const float *rots, const float *scales, const float *depths,
                      float *cov3ds, float *dcov3d_drots, float *dcov3d_dscales,
                      gsb_stream_t stream);

/* F.3/B.3.  Replaces `computeCov2D` (ext.cpp:44-52, gausplat.cu:201-251, kernel.cu:425-551).
 * width/height only feed the +-1.3*tan_fov clamp.  -> cov2ds[N,3], dcov2d_dcov3ds[N,3,6],
 * dcov2d_dpcs[N,3,3] (nullable together). */
int gsb_compute_cov2d(int N, const float *cov3ds, const float *pcs, const float *Rcw,
                      const float *depths, float fx, float fy, float width, float height,
                      float *cov2ds, float *dcov2d_dcov3ds, float *dcov2d_dpcs,
                      gsb_stream_t stream);

/* F.4.  Replaces `sh2Color` (ext.cpp:63-66, gausplat.cu:298-338, kernel.cu:619-807).
 * shs[N,3*k] laid out [coef][rgb], k = sh_dim3 in {1,4,9,16}; not gated by depth.
 * -> colors[N,3], dcolor_dshs[N,1,k], dcolor_dpws[N,3,3] (nullable together). */
int gsb_sh2color(int N, int sh_dim3, const float *shs, const float *pws, const float *twc,
                 float *colors, float *dcolor_dshs, float *dcolor_dpws, gsb_stream_t stream);

/* F.5.3/B.5.3.  Replaces `inverseCov2D` (ext.cpp:34-36, gausplat.cu:340-373, kernel.cu:274-324).
 * depths is READ-WRITE: a NaN 1/det sets depths[i] = -1.  -> cinv2ds[N,3], areas[N,2] int32,
 * dcinv2d_dcov2ds[N,3,3] (nullable). */
int gsb_inverse_cov2d(int N, const float *cov2ds, float *depths, float *cinv2ds, int32_t *areas,
                      float *dcinv2d_dcov2ds, gsb_stream_t stream);

/* ---- fused per-Gaussian path (extension; SURVEY 8f row N1).  No single reference entry point:
 * gsb_preprocess_forward == project + computeCov3D + computeCov2D + sh2Color + inverseCov2D
 * with calc_J = false (gsmodel.py:21-36 without the Jacobian outputs) in one kernel, and
 * gsb_preprocess_backward == the Jacobian chain of gsmodel.py:72-85 (torch.bmm over the saved
 * Jacobians) as analytic vector-Jacobian products recomputed from the parameters.
 * width/height feed the fov clamp exactly as in gsb_compute_cov2d.  Outputs of the forward
 * feed gsb_splat_bin / gsb_splat_render unchanged; the backward consumes gsb_splat_backward's
 * dloss_dus / dloss_dcinv2ds / dloss_dcolors (dloss_dalphas passes through untouched) and
 * writes dloss_dpws[N,3], dloss_dshs[N,3k], dloss_dscales[N,3], dloss_drots[N,4].
 * Two optional short cuts around passes that only re-format data:
 *   forward:  alphas[N] + records (both or neither) -- also writes the N packed 48-byte
 *             per-Gaussian records the rasterizers gather from; hand them to gsb_splat_render /
 *             gsb_splat_backward as `packed_records` and the separate pack pass is skipped;
 *   backward: moments[N,9] + cinv2ds[N,3] + dloss_dus_out[N,2] + dloss_dalphas_out[N] (all or
 *             none) -- the upstream gradients are taken as the raw moment rows
 *             gsb_splat_backward leaves in `moments_out`; the three dloss_d* inputs are then
 *             ignored (may be NULL) and dL/du, dL/dalpha are written to the two outputs. */
int gsb_preprocess_forward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                           const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                           float fy, float cx, float cy, float width, float height, float *us,
                           float *cinv2ds, float *colors, float *depths, int32_t *areas, const float *alphas,
                           void *records, gsb_stream_t stream);
int gsb_preprocess_backward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                            const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                            float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                            const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                            float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                            const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                            gsb_stream_t stream);
/* RGB-D form (extension): the same, plus dloss_ddepths[N] = dL/dz from gsb_splat_backward_rgbd.
 * z = (Rcw pw + tcw)[2], so dL/dpws gains dloss_ddepths Rcw[2,:]; a culled Gaussian (z < 0.2)
 * gets 0, as for every other gradient. */
int gsb_preprocess_backward_rgbd(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                 const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                 float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                 const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                 const float *dloss_ddepths, gsb_stream_t stream);

/* Camera gradient (extension; pose refinement and RGB-D tracking).  The arguments of
 * gsb_preprocess_backward_rgbd, where dloss_ddepths may be NULL (colour only), plus
 * dloss_dcamera[15] = dL/dRcw (row-major 3x3), dL/dtcw (3), dL/dtwc (3), summed over the N
 * Gaussians:  dL/dtcw = sum dL/dpc,  dL/dRcw = sum dL/dpc (x) pw + J^T dL/d(J Rcw),
 * dL/dtwc = -sum (colour part of dL/dpw) (0 at SH degree 0).  dL/dpc is the vector the backward
 * rotates into dloss_dpws (x, y differentiated as if unclamped, as there); a culled Gaussian
 * contributes through its colour only.  Intrinsics are not differentiated, and Rcw, tcw, twc
 * are independent inputs (twc = -Rcw^T tcw is the caller's relation to chain).
 * dloss_dpws, dloss_dshs, dloss_dscales, dloss_drots (and with moments dloss_dus_out,
 * dloss_dalphas_out) are all set -- the same per-Gaussian outputs as gsb_preprocess_backward,
 * bit for bit (they come from the same kernel, after a pass that computes the camera gradient)
 * -- or all NULL: pose only, for a frozen map; one pass, nothing per Gaussian is written.
 * ws: caller-owned, 16-byte aligned, at least gsb_preprocess_backward_pose_workspace_bytes(N)
 * bytes.  The CTAs' partial sums are added in a fixed order in fp64 (no atomics): the same
 * inputs give the same bits on every run.  N = 0 writes zeros. */
size_t gsb_preprocess_backward_pose_workspace_bytes(int N);
int gsb_preprocess_backward_pose(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                 const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                 float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                 const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                 const float *dloss_ddepths, float *dloss_dcamera, void *ws, size_t ws_bytes,
                                 gsb_stream_t stream);

/* Antialiasing (extension; the 2D-filter opacity compensation of Mip-Splatting, gsplat's
 * rasterize_mode="antialiased").  The rasterizers keep drawing cov2d + 0.3 I, and each Gaussian's
 * opacity is scaled by how much that blur spread it:
 *     r = det(cov2d) / det(cov2d + 0.3 I)  (pre-blur over blurred),  rho = sqrt(max(2.5e-5, r)),
 *     alpha_eff = rho * alpha               (rho = 1 for a culled Gaussian).
 * gsb_preprocess_forward_aa: gsb_preprocess_forward's arguments with alphas required, plus
 * alphas_eff[N] (output).  The records (optional) carry alpha_eff; every other output is
 * bit-identical to gsb_preprocess_forward's.  Render with alphas_eff.
 * gsb_preprocess_backward_aa: gsb_preprocess_backward_pose's arguments plus the raw alphas[N];
 * the moment rows are required (they come from a splat backward run on alphas_eff, so their
 * dL/dalpha is dL/dalpha_eff).  dloss_dalphas_out = rho dL/dalpha_eff, and alpha dL/dalpha_eff
 * drho/dcov2d joins the geometry gradients (0 where the 2.5e-5 clamp holds).  dloss_ddepths
 * may be NULL (colour only); dloss_dcamera NULL (ws ignored) is the plain or (dloss_dshs NULL)
 * compact call, otherwise the camera gradient as in gsb_preprocess_backward_pose, with the
 * per-Gaussian outputs all set or all NULL (pose only). */
int gsb_preprocess_forward_aa(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                              const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                              float fy, float cx, float cy, float width, float height, float *us, float *cinv2ds,
                              float *colors, float *depths, int32_t *areas, const float *alphas, void *records,
                              float *alphas_eff, gsb_stream_t stream);
int gsb_preprocess_backward_aa(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                               const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                               float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                               const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                               float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                               const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                               const float *dloss_ddepths, const float *alphas, float *dloss_dcamera, void *ws,
                               size_t ws_bytes, gsb_stream_t stream);

/* Camera models (extension; gsplat's camera_model="pinhole" | "ortho" | "fisheye", and "opencv").  Only the
 * projected mean u and the Jacobian J of the EWA splat change; everything after cov2d (conic,
 * radius, records, the rasterizers) is the same.  Depth stays the camera-frame z, and every model
 * culls z < 0.2.
 *   PINHOLE  u = (fx x/z + cx, fy y/z + cy), J with the +-1.3 tan_fov clamp: the entry points above.
 *   ORTHO    u = (fx x + cx, fy y + cy),  J = [[fx, 0, 0], [0, fy, 0]];  no clamp.
 *   FISHEYE  Kannala-Brandt (COLMAP's OPENCV_FISHEYE; k = 0 is the equidistant lens):
 *            theta = atan2(|(x, y)|, z),  theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6
 *            + k4 theta^8),  u = (fx theta_d x / r + cx, fy theta_d y / r + cy), J its exact
 *            Jacobian; no clamp.  A Gaussian where d theta_d / d theta <= 0 is culled like z < 0.2.
 *   OPENCV   radial-tangential (COLMAP's OPENCV; RADIAL is p1 = p2 = 0, SIMPLE_RADIAL also k2 = 0 and
 *            fx = fy), k = (k1, k2, p1, p2).  With (a, b) = (x/z, y/z), rho = a^2 + b^2 and
 *            R = 1 + k1 rho + k2 rho^2:  u = (fx (a R + 2 p1 a b + p2 (rho + 2 a^2)) + cx,
 *            fy (b R + p1 (rho + 2 b^2) + 2 p2 a b) + cy), never clamped.  J is the distortion's
 *            Jacobian times pinhole's at (a, b) clamped to +-1.3 W / (2 fx) c, +-1.3 H / (2 fy) c, where
 *            c is how far the radial terms move the image corners (1 when k1 = k2 = 0).  A Gaussian
 *            beyond the first maximum of r (1 + k1 r^2 + k2 r^4), or where the distortion's Jacobian
 *            has det <= 0, is culled like z < 0.2.  Needs width, height > 0.
 * k must be 0 for PINHOLE and ORTHO and finite for all; fx, fy > 0 for every model but PINHOLE.
 * The ids skip 3, which stays an unknown model: callers built against an earlier header that
 * passed 3 as an invalid id still get an argument error.
 * gsb_preprocess_forward_model: gsb_preprocess_forward_aa's arguments with alphas_eff nullable
 * (NULL: no antialiasing, and then alphas and records go together as in gsb_preprocess_forward).
 * gsb_preprocess_backward_model: gsb_preprocess_backward_aa's arguments with alphas nullable (NULL:
 * no antialiasing) and the moment rows required.  A NULL camera_model, or PINHOLE, runs the
 * kernels the entry points above run.  width/height feed only PINHOLE's and OPENCV's clamp. */
#define GSB_CAMERA_PINHOLE 0
#define GSB_CAMERA_ORTHO 1
#define GSB_CAMERA_FISHEYE 2
#define GSB_CAMERA_OPENCV 4
typedef struct gsb_camera_model {
  int32_t model; /* GSB_CAMERA_* */
  float k[4];    /* FISHEYE: k1..k4;  OPENCV: k1, k2, p1, p2 */
} gsb_camera_model;
int gsb_preprocess_forward_model(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                 float fy, float cx, float cy, float width, float height, float *us, float *cinv2ds,
                                 float *colors, float *depths, int32_t *areas, const float *alphas, void *records,
                                 float *alphas_eff, const gsb_camera_model *camera_model, gsb_stream_t stream);
int gsb_preprocess_backward_model(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                  const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                  float fy, float cx, float cy, float width, float height, const float *dloss_dus,
                                  const float *dloss_dcinv2ds, const float *dloss_dcolors, float *dloss_dpws,
                                  float *dloss_dshs, float *dloss_dscales, float *dloss_drots, const float *moments,
                                  const float *cinv2ds, float *dloss_dus_out, float *dloss_dalphas_out,
                                  const float *dloss_ddepths, const float *alphas, float *dloss_dcamera, void *ws,
                                  size_t ws_bytes, const gsb_camera_model *camera_model, gsb_stream_t stream);

/* dL/dsh from per-view dL/dcolor (extension; multi-view data parallelism, SURVEY 8e).
 * colour = 0.5 + sum_l Y_l(dir) sh_l is linear in sh and never clamped (kernel.cu:735-774), so
 * dloss_dshs[n, l, c] = sum_v Y_l((pws[n] - twcs[v]) / |.|) * dloss_dcolors[v, n, c].
 * gsb_preprocess_backward may then be called with dloss_dshs = NULL (it skips the 192-byte row),
 * the V views of a step exchange 12 B per Gaussian and view instead of one 192-byte row, and every
 * rank expands here.  twcs[V,3], dloss_dcolors[V,N,3] -> dloss_dshs[N,3*sh_dim3] (overwritten;
 * views summed in index order; V = 1 reproduces gsb_preprocess_backward's row to rounding). */
int gsb_sh_grad_expand(int N, int sh_dim3, int V, const float *pws, const float *twcs, const float *dloss_dcolors,
                       float *dloss_dshs, gsb_stream_t stream);

/* Mip-Splatting 3D smoothing filter (extension).  Bounds each Gaussian's size from below by the
 * sampling rate of the training views, so that a scene rendered closer or at a higher resolution
 * than it was trained at shows no high-frequency erosion.  scales and alphas are the ACTIVATED
 * values (exp of the raw scales, sigmoid of the raw opacities), as the fused path takes them.
 * gsb_filter3d: pws[N,3] and the training cameras cams[C,20] (row: Rcw row-major 9, tcw 3, fx,
 * fy, cx, cy, W, H, 2 unused) -> filter3d[N]:
 *     camera k sees Gaussian i  iff  z = (Rcw pw + tcw)[2] >= 0.2f (the rasterizers' cull) and the
 *       projected mean u = (fx x/z + cx, fy y/z + cy) lies in [-0.15 W, 1.15 W] x [-0.15 H, 1.15 H];
 *     d_i = min z over the cameras that see i, or the largest d of the seen Gaussians if none does;
 *     filter3d_i = sqrt(variance) d_i / max_k fx_k (the largest POSITIVE fx; the table is not
 *       checked on the host, so a camera with fx <= 0 or NaN only drops out of that maximum);
 *     all 0 when no Gaussian is seen, when C == 0, or when no camera has fx > 0.
 * (Mip-Splatting's compute_3D_filter with the camera's own cx, cy instead of W/2, H/2, and the
 * z >= 0.2f cull instead of z > 0.2.)  The cameras are staged GSB_FILTER3D_CHUNK at a time; any
 * C works.  ws: 16-byte aligned, gsb_filter3d_workspace_bytes(N, C) bytes.  Deterministic.
 * gsb_filter3d_apply: (scales[N,3], alphas[N]) -> scales_f[N,3], alphas_f[N] with
 *     s'_j = sqrt(s_j^2 + f^2),  alpha' = alpha prod_j s_j / s'_j    (f = filter3d_i);
 *     f == 0 copies both exactly.  Render (and run the fused backward) with s', alpha'.
 * gsb_filter3d_backward: dL/ds' (dloss_dscales_f[N,3]) and dL/dalpha' (dloss_dalphas_f[N]) ->
 *     dL/ds = dL/ds'_j s_j/s'_j + alpha dL/dalpha' prod_{k!=j}(s_k/s'_k) f^2/s'_j^3,
 *     dL/dalpha = prod_j (s_j/s'_j) dL/dalpha'   (f is a constant; f == 0 passes both through).
 *     The outputs may be the inputs (in place). */
#define GSB_FILTER3D_CHUNK 64
size_t gsb_filter3d_workspace_bytes(int N, int C);
int gsb_filter3d(int N, const float *pws, int C, const float *cams, float variance, float *filter3d, void *ws,
                 size_t ws_bytes, gsb_stream_t stream);
int gsb_filter3d_apply(int N, const float *scales, const float *alphas, const float *filter3d, float *scales_f,
                       float *alphas_f, gsb_stream_t stream);
int gsb_filter3d_backward(int N, const float *scales, const float *alphas, const float *filter3d,
                          const float *dloss_dscales_f, const float *dloss_dalphas_f, float *dloss_dscales,
                          float *dloss_dalphas, gsb_stream_t stream);

/* ---- splat, phase 1: tile rectangles + patch count.
 * Replaces getRects + thrust::inclusive_scan + the D2H read of the total
 * (gausplat.cu:54-67, kernel.cu:82-122).  depths and areas are READ-WRITE (Gaussians that
 * touch no tile get depths = -1, areas = 0).  Leaves rects/offsets in `bin_ws` for phase 2.
 * Writes the patch count to *P_host and the largest depth key (uint32)(depth*1000) of a
 * binned Gaussian to *depth_key_max_host (nullable) after synchronising `stream` (the one
 * host sync; the reference has the same read-back, gausplat.cu:67).
 * This and every other entry point that bins (gsb_splat_render, gsb_splat_forward,
 * gsb_splat_forward_enqueue) return an argument error when ceil(W/16) or ceil(H/16) exceeds
 * GSB_MAX_GRID_TILES, and when a frame has 2^30 patches or more. */
size_t gsb_splat_bin_workspace_bytes(int N);
int gsb_splat_bin(int H, int W, int N, const float *us, float *depths, int32_t *areas,
                  void *bin_ws, size_t bin_ws_bytes, int64_t *P_host, uint32_t *depth_key_max_host,
                  gsb_stream_t stream);

/* ---- splat, phase 2: keys, duplicate-key radix sort, tile ranges, record packing, draw.
 * Replaces createKeys + thrust::sort_by_key + getRanges + draw (gausplat.cu:69-105,
 * kernel.cu:46-80,125-271).  `alphas` is [N] (or [N,1]).  Outputs: image[3,H,W] planar,
 * contrib[H,W] int32, final_tau[H,W], patch_range_per_tile[T,2] int32 (T = tiles),
 * gsid_per_patch[P] int32 (Gaussian id of every patch in (tile, depth-mm, id) order).
 * Every output element is written (no pre-zeroing needed).
 * depth_key_max: the value phase 1 returned (bounds the sort width; keys are packed into 32
 * bits when tile and depth bits fit), or 0xFFFFFFFF for the reference's full 64-bit layout --
 * the resulting order is the same.  packed_records: NULL, or the per-Gaussian records
 * gsb_preprocess_forward wrote.  With NULL they are built here, sit at
 * ws + gsb_splat_records_offset(...) after the call and may be handed to gsb_splat_backward as
 * `packed_records` while `ws` and the inputs are unchanged. */
size_t gsb_splat_workspace_bytes(int N, int H, int W, int64_t P);
size_t gsb_splat_records_offset(int N, int H, int W, int64_t P);
int gsb_splat_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                     const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                     const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes, float *image,
                     int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                     int32_t *gsid_per_patch, gsb_stream_t stream);

/* ---- RGB-D rendering (extension).  The *_rgbd forms of gsb_splat_render / gsb_splat_forward also
 * write two more [H,W] planes, 16-byte aligned like `image` (a misaligned one is an argument error):
 *   depth_image D[p] = sum_i w_i(p) z_i,   alpha_image A[p] = sum_i w_i(p),
 * with the image's compositing weights w_i = tau_i alpha'_i (same clamp, skip and stop rules) and
 * z_i the Gaussian's camera-frame depth, i.e. its `depths` value.  Pixels of tiles without patches
 * get D = A = 0.  D is not normalised: the expected depth is D / A.  Every other output is
 * bit-identical to the colour entry point's.
 * The packed records carry z in their last word (q2.w): those gsb_preprocess_forward writes and
 * those the render entry points pack (from `depths`) both do, and only the RGB-D rasterizers
 * read it. */
int gsb_splat_render_rgbd(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                          const float *cinv2ds, const float *alphas, const float *depths, const float *colors,
                          const void *packed_records, const void *bin_ws, void *ws, size_t ws_bytes, float *image,
                          int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                          float *depth_image, float *alpha_image, gsb_stream_t stream);

/* ---- splat, both phases without the mid-way host round trip (extension).
 * gsb_splat_bin + gsb_splat_render stall the GPU while the host reads P back to size the sort
 * workspace (the reference does the same, gausplat.cu:64-67).  Here the caller provides CAPACITIES
 * instead -- an upper bound P_cap on the patch count (e.g. 1.25 x the previous frame's P) and on the
 * depth keys (depth_key_cap >= every (uint32)(depth*1000); it fixes the key width and the depth
 * bits the sort orders; a key needing more bits is reported, never sorted by its low bits) -- all kernels
 * read the actual P from device memory, and the host looks at [P, max depth key, flags] only
 * after the sort and the rasterizer have been enqueued behind the copy: no GPU bubble.
 * Workspaces: bin_ws as for gsb_splat_bin; ws >= gsb_splat_workspace_bytes(N, H, W, P_cap);
 * gsid_per_patch[P_cap] (the first P entries are valid).  status_host[3] (pinned memory for a truly
 * asynchronous copy) receives P, the largest depth key and the flags (GSB_STATUS_*).
 * Returns 0, or GSB_CAPACITY_EXCEEDED when a bound was too small: the outputs are then undefined and
 * the caller repeats the frame with gsb_splat_bin / gsb_splat_render (or larger capacities);
 * depths / areas have been culled in place exactly as gsb_splat_bin does, which is idempotent. */
#define GSB_CAPACITY_EXCEEDED 2
#define GSB_STATUS_TOO_MANY_PATCHES 1u /* flags bit 0: 2^32 patches or more (P saturated) */
#define GSB_STATUS_P_CAP 2u            /* flags bit 1: the patches did not fit P_cap */
#define GSB_STATUS_DEPTH_KEY 4u        /* flags bit 2: a depth key wider than depth_key_cap plans */
int gsb_splat_forward(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                      float *depths, const float *colors, int32_t *areas, const void *packed_records,
                      int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                      size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                      int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                      gsb_stream_t stream);
/* RGB-D form: the same, plus depth_image / alpha_image as for gsb_splat_render_rgbd. */
int gsb_splat_forward_rgbd(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                           float *depths, const float *colors, int32_t *areas, const void *packed_records,
                           int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                           size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                           int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                           float *depth_image, float *alpha_image, gsb_stream_t stream);

/* Same, but only ENQUEUES (no host wait, no event): for capture into a CUDA graph.  status_host is
 * written by a stream-ordered copy; the caller reads it after the work has completed (any
 * GSB_STATUS_* flag, or P > P_cap -> the frame's outputs are invalid). */
int gsb_splat_forward_enqueue(int H, int W, int N, const float *us, const float *cinv2ds, const float *alphas,
                              float *depths, const float *colors, int32_t *areas, const void *packed_records,
                              int64_t P_cap, uint32_t depth_key_cap, void *bin_ws, size_t bin_ws_bytes, void *ws,
                              size_t ws_bytes, float *image, int32_t *contrib, float *final_tau,
                              int32_t *patch_range_per_tile, int32_t *gsid_per_patch, uint32_t *status_host,
                              gsb_stream_t stream);

/* ---- splatB.  Replaces `splatB` (ext.cpp:20-32, gausplat.cu:114-159, kernel.cu:809-950).
 * Consumes the forward's contrib / final_tau / patch_range_per_tile / gsid_per_patch.
 * -> dloss_dus[N,1,2], dloss_dcinv2ds[N,1,3], dloss_dalphas[N,1,1], dloss_dcolors[N,1,3]
 * (every element written).  packed_records: NULL (the per-Gaussian records are rebuilt from the
 * four attribute arrays into `ws`) or the forward's record array.
 * moments_out: NULL, or [N,9] -- the raw per-Gaussian moment rows are left there and the
 * conversion to the four gradient tensors is skipped (they may then be NULL): the caller feeds
 * the rows to gsb_preprocess_backward, which does the conversion in registers. */
size_t gsb_splat_backward_workspace_bytes(int N, int H, int W, int64_t P);
int gsb_splat_backward(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                       const float *alphas, const float *colors, const int32_t *contrib,
                       const float *final_tau, const int32_t *patch_range_per_tile,
                       const int32_t *gsid_per_patch, const float *dloss_dgammas,
                       const void *packed_records, void *ws,
                       size_t ws_bytes, float *dloss_dus, float *dloss_dcinv2ds,
                       float *dloss_dalphas, float *dloss_dcolors, float *moments_out, gsb_stream_t stream);
/* RGB-D form (extension): the backward of gsb_splat_render_rgbd / gsb_splat_forward_rgbd.  Extra inputs:
 * depths[N] (the depth words of the records it re-packs when packed_records is NULL),
 * dloss_ddepth_image[H,W] and dloss_dalpha_image[H,W] (any 4-byte alignment, like dloss_dgammas);
 * extra output dloss_ddepths[N] = dL/dz (every element written; 0 for Gaussians no pixel replays).
 * packed_records, when given, must carry z (gsb_preprocess_forward's, or the forward's own). */
int gsb_splat_backward_rgbd(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                            const float *alphas, const float *colors, const float *depths, const int32_t *contrib,
                            const float *final_tau, const int32_t *patch_range_per_tile,
                            const int32_t *gsid_per_patch, const float *dloss_dgammas,
                            const float *dloss_ddepth_image, const float *dloss_dalpha_image,
                            const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus,
                            float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, float *moments_out,
                            float *dloss_ddepths, gsb_stream_t stream);

/* Absolute-gradient densification (extension; AbsGS, gsplat's absgrad=True).  The arguments of
 * gsb_splat_backward / gsb_splat_backward_rgbd, plus one output dloss_dus_abs[N,2] (any 4-byte
 * alignment; every element written, 0 for Gaussians no pixel replays):
 *     dloss_dus_abs[i] = ( sum_p |g_ip.x| , sum_p |g_ip.y| ),   dloss_dus[i] = sum_p g_ip,
 *     g_ip = -w_ip (A dx + B dy, B dx + C dy),  w_ip = dL/dalpha'_ip alpha'_ip,  (dx, dy) = u_i - p,
 * with (A, B, C) = cinv2ds[i] and dL/dalpha' that of the colour (RGB-D form: colour, depth and
 * alpha) planes -- the per-pixel terms whose sum is dL/du.  Per-pixel gradients of opposite sign
 * cancel in dL/du but not here, so a Gaussian that covers a large, textured region gets a large
 * statistic to densify on.  Every other output (moments_out included) is that of the plain call.
 * A NULL dloss_dus_abs is an argument error (unless N == 0). */
int gsb_splat_backward_abs(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                           const float *alphas, const float *colors, const int32_t *contrib, const float *final_tau,
                           const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                           const float *dloss_dgammas, const void *packed_records, void *ws, size_t ws_bytes,
                           float *dloss_dus, float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors,
                           float *moments_out, float *dloss_dus_abs, gsb_stream_t stream);
int gsb_splat_backward_rgbd_abs(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds,
                                const float *alphas, const float *colors, const float *depths, const int32_t *contrib,
                                const float *final_tau, const int32_t *patch_range_per_tile,
                                const int32_t *gsid_per_patch, const float *dloss_dgammas,
                                const float *dloss_ddepth_image, const float *dloss_dalpha_image,
                                const void *packed_records, void *ws, size_t ws_bytes, float *dloss_dus,
                                float *dloss_dcinv2ds, float *dloss_dalphas, float *dloss_dcolors, float *moments_out,
                                float *dloss_ddepths, float *dloss_dus_abs, gsb_stream_t stream);

/* ---- feature rendering (extension).  Composites per-Gaussian feature vectors features[N,D]
 * (row-major, row stride D, any 4-byte alignment; D >= 1) with the image's weights:
 *   feature_image[c, p] = sum_i w_i(p) features[i, c],   w_i = tau_i alpha'_i
 * (the same clamp, skip and stop rules and the same fp32 operations as the colour image: a feature
 * column equal to a colour channel composites to that image plane's bits).  Both calls replay a
 * frame the colour forward binned and drew: its contrib, patch_range_per_tile (any alignment) and
 * gsid_per_patch (P entries), and final_tau for the backward; the colour entry points are not
 * involved.  packed_records: the forward's record array, or NULL -- the records are then packed
 * into `ws` from us, cinv2ds, alphas and colors, as gsb_splat_backward does.  With P == 0 (or
 * N == 0) nothing was drawn.  ws: gsb_splat_features_workspace_bytes(N, H, W, P) bytes, any
 * alignment (P = 0 when packed_records is given); one workspace serves both calls.
 * gsb_splat_features: -> feature_image[D,H,W] planar, 16-byte aligned like `image` (a misaligned
 *   one is an argument error); every element written, 0 on tiles without patches.
 * gsb_splat_features_backward: dloss_dfeature_image[D,H,W] (any 4-byte alignment) ->
 *   moments[N,9] READ-MODIFY-WRITE: rows 0-5 (the geometry and opacity moments gsb_splat_backward
 *     leaves with moments_out) are ADDED to, rows 6-8 are left alone, so the conversion of
 *     gsb_splat_backward / gsb_preprocess_backward* yields the gradients of the sum of both losses;
 *   dloss_dfeatures[N,D] = sum_p tau alpha' dL/dF(p) (every element written; 0 for Gaussians no
 *     pixel replays, culled ones included; summed with float atomics).
 * Argument errors: D < 1, a misaligned feature_image, and the tile-grid limit of the splat entry
 * points (GSB_MAX_GRID_TILES). */
size_t gsb_splat_features_workspace_bytes(int N, int H, int W, int64_t P);
int gsb_splat_features(int H, int W, int N, int64_t P, int D, const float *us, const float *cinv2ds,
                       const float *alphas, const float *colors, const float *features, const void *packed_records,
                       const int32_t *contrib, const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                       void *ws, size_t ws_bytes, float *feature_image, gsb_stream_t stream);
int gsb_splat_features_backward(int H, int W, int N, int64_t P, int D, const float *us, const float *cinv2ds,
                                const float *alphas, const float *colors, const float *features,
                                const void *packed_records, const int32_t *contrib, const float *final_tau,
                                const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                                const float *dloss_dfeature_image, void *ws, size_t ws_bytes, float *moments,
                                float *dloss_dfeatures, gsb_stream_t stream);

/* ---- contribution statistics (extension; DESIGN 3.18).  Per Gaussian, over the pixels of one
 * drawn frame, with the blending weights w = tau alpha' the frame composited (same clamp, skip and
 * stop rules, same fp32 operations: every w is the bit pattern the image used):
 *   weight_sum[i] += sum_p w_i(p)            (fp32 atomics: the order of the additions varies)
 *   weight_max[i]  = max(weight_max[i], max_p w_i(p))   (exact; updated through its uint bits,
 *                    so it must hold values >= 0, e.g. zeros, before the first frame)
 *   hit_count[i]  += #{p : w_i(p) > 0}       (exact)
 * All three are READ-MODIFY-WRITE: zero them once, then call once per view to accumulate.
 * weight_sum, weight_max: any 4-byte alignment; hit_count: 8-byte aligned.  N == 0 or P == 0:
 * nothing is added.
 * gsb_splat_stats replays a frame gsb_splat_render / _forward (colour or RGB-D) drew: its contrib,
 *   patch_range_per_tile, gsid_per_patch and records, given as packed_records or packed into `ws`
 *   from us, cinv2ds, alphas and colors, as gsb_splat_features does.  ws:
 *   gsb_splat_stats_workspace_bytes(N, H, W, P) bytes, any alignment (P = 0 when packed_records is
 *   given).
 * gsb_splat_stats_2dgs replays a surfel frame (2D Gaussian Splatting) that gsb_splat_surfel_* or
 *   gsb_splat_2dgs_* drew, from its 80-byte records (16-byte aligned); no workspace. */
size_t gsb_splat_stats_workspace_bytes(int N, int H, int W, int64_t P);
int gsb_splat_stats(int H, int W, int N, int64_t P, const float *us, const float *cinv2ds, const float *alphas,
                    const float *colors, const void *packed_records, const int32_t *contrib,
                    const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch, void *ws, size_t ws_bytes,
                    float *weight_sum, float *weight_max, int64_t *hit_count, gsb_stream_t stream);
int gsb_splat_stats_2dgs(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                           const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch, float *weight_sum,
                           float *weight_max, int64_t *hit_count, gsb_stream_t stream);

/* ---- batched tiny matmul (extension).  C[b] = A[b] (m x k) . B[b] (k x n), or B shared by all
 * batches when b_shared != 0; dense row-major f32.  This is the product the reference's
 * GSFunction.backward applies ~12 times over the per-Gaussian Jacobians (gsmodel.py:72-85);
 * ops.py routes torch.matmul on the Jacobian tensors it returns to this entry point so the
 * unmodified reference chain runs at HBM speed instead of through batched-GEMV library calls. */
int gsb_small_bmm(long long batch, int m, int k, int n, const float *A, const float *B, int b_shared, float *C,
                  gsb_stream_t stream);

/* ---- training loss (extension; SURVEY 8f row N2).  Replaces `gau_loss`
 * (gsplat/pytorch_ssim.py:64-67, called at train.py:52) and its autograd backward:
 *   loss = (1 - lambda) mean|image - gt| + lambda (1 - mean SSIM), 11x11 Gaussian window
 *   (sigma 1.5), zero padding, C1 = 0.01^2, C2 = 0.03^2, image/gt [3,H,W] planar f32.
 * Writes the scalar loss to *loss_out (device) and, if dloss_dimage != NULL, dloss/dimage
 * [3,H,W] -- the tensor loss.backward() would hand to splatB. */
size_t gsb_gau_loss_workspace_bytes(int H, int W);
int gsb_gau_loss(int H, int W, const float *image, const float *gt_image, float loss_lambda, float *loss_out,
                 float *dloss_dimage, void *ws, size_t ws_bytes, gsb_stream_t stream);

/* ---- density control (extension; SURVEY 8f row N3).  Replaces GSModel.update_density_info,
 * update_gaussian_density and reset_alpha with prune_params / update_params
 * (gsplat/gsmodel.py:132-166, 219-331): one classify pass, one scan, one pass that moves every
 * surviving row of the 6 parameter tensors and their Adam moments exactly once and appends the
 * clones and splits, instead of 18 boolean-index + torch.cat rebuilds.
 *
 * gsb_gaussians: the reference's six training tensors (gsmodel.py:114-127), device pointers
 * to dense row-major f32.  For the Adam moments pass two more of these (exp_avg, exp_avg_sq);
 * a NULL struct pointer means "the optimizer has no state yet" (update_params' else branch). */
typedef struct gsb_gaussians {
  float *pws;        /* [N,3]  */
  float *low_shs;    /* [N,3]  */
  float *high_shs;   /* [N,45] */
  float *alphas_raw; /* [N,1]  logit of opacity */
  float *scales_raw; /* [N,3]  log of scale     */
  float *rots_raw;   /* [N,4]  (w,x,y,z), un-normalised */
} gsb_gaussians;

/* update_density_info (:219-234): grad_accum[i] += |dloss_dus[i]|, cunt[i] += 1 where mask[i]
 * (uint8 0/1).  first != 0 reproduces the first call after a density update: grad_accum is
 * overwritten with the norm of EVERY Gaussian and cunt with the mask (:228-229). */
int gsb_density_accumulate(int64_t N, const float *dloss_dus, const uint8_t *mask, float *grad_accum,
                           int32_t *cunt, int first, gsb_stream_t stream);

/* Classification + output slots (:238-262).  Class per Gaussian into cls[N] (0 keep, 1 keep +
 * clone, 2 keep + split, 3 prune): prune if alphas_raw < alpha_raw_min or max(scales_raw) >
 * scale_raw_max; else g = grad_accum / cunt (0/0 -> 0); g >= grad_min selects it, and
 * max(exp(scales_raw)) <= scale_clone_max decides clone vs split.  slots[N,3] int32 = the
 * exclusive counts of survivors / clones / splits before each Gaussian.
 * counts_host[3] <- (K survivors, C clones, S splits).  HOST SYNCHRONISATION: waits for the
 * counts, like the reference's int(torch.sum(...)) reads -- the caller sizes the outputs
 * (K + C + S rows) and draws the S x 3 unit normals from them. */
size_t gsb_density_workspace_bytes(int64_t N);
int gsb_density_plan(int64_t N, const float *alphas_raw, const float *scales_raw, const float *grad_accum,
                     const int32_t *cunt, float alpha_raw_min, float scale_raw_max, float grad_min,
                     float scale_clone_max, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                     int64_t *counts_host, gsb_stream_t stream);

/* The plan of a prune by mask: cls[i] = 0 (keep) where keep[i] != 0, else 3 (prune), and slots
 * as gsb_density_plan writes them; counts_host[3] <- (K survivors, 0, 0), so gsb_density_apply /
 * gsb_density_apply_rows with C = S = 0 keep the survivors in order with their Adam moments.
 * Workspace: gsb_density_workspace_bytes(N).  HOST SYNCHRONISATION: one read of K, as
 * gsb_density_plan. */
int gsb_density_plan_keep(int64_t N, const uint8_t *keep, void *ws, size_t ws_bytes, uint8_t *cls, int32_t *slots,
                          int64_t *counts_host, gsb_stream_t stream);

/* The rebuild (:236-318 + :132-166).  dst rows: survivors in order, then clones, then splits.
 * A clone row is (pws, shs, logit(sigmoid(alphas_raw)), log(exp(scales_raw)),
 * normalize(rots_raw)); a split row moves pws by R(q) (z * exp(scales_raw)) with z[S,3] the
 * caller's unit normals (the reference draws torch.normal(0, std=scales) = z * std, :276-277)
 * and shrinks the NEW Gaussian's scale by 0.6 (the original keeps its size, :281-282).  New
 * rows get zero Adam moments.  src_m/src_v/dst_m/dst_v: NULL, or all four set.  N < 2^30
 * (253 GB of parameters): a larger N is refused as bad counts. */
int gsb_density_apply(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int64_t S,
                      const gsb_gaussians *src, const gsb_gaussians *src_m, const gsb_gaussians *src_v,
                      const float *z, const gsb_gaussians *dst, const gsb_gaussians *dst_m,
                      const gsb_gaussians *dst_v, gsb_stream_t stream);

/* The same plan applied to one more per-Gaussian tensor of any width D >= 1 (features[N,D],
 * row-major f32): dst[K + C + S, D] gets the survivors in order, then the clones, then the
 * splits, each new row a copy of its source row; src_m/src_v (Adam moments, same shape) -> dst_m/
 * dst_v with zero rows for the new Gaussians.  src_m/src_v/dst_m/dst_v: NULL, or all four set. */
int gsb_density_apply_rows(int64_t N, const uint8_t *cls, const int32_t *slots, int64_t K, int64_t C, int64_t S,
                           int D, const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                           float *dst_v, gsb_stream_t stream);

/* reset_alpha (:320-331): alphas_raw = min(alphas_raw, reset_raw); the alpha group's Adam
 * moments (nullable) are zeroed. */
int gsb_reset_alpha(int64_t N, float *alphas_raw, float *exp_avg, float *exp_avg_sq, float reset_raw,
                    gsb_stream_t stream);

/* ---- MCMC densification (extension; Kheradmand et al., "3D Gaussian Splatting as Markov Chain
 * Monte Carlo", 2024; DESIGN 3.11).  A fixed Gaussian budget: dead Gaussians are moved onto live
 * ones instead of pruned, growth samples existing Gaussians, and positions get noise shaped by each
 * Gaussian's covariance.  o = sigmoid(alphas_raw), N < 2^31.
 *
 * Sampler: row i weighs q_i = floor(o_i 2^32) (o_i in fp64 from the fp32 raw value; 0 for rows
 * the mode excludes), W = its uint64 inclusive prefix sum, and a draw u in [0, 1) picks the first i
 * with W_i > min(floor(u W_total), W_total - 1).  Integer sums do not depend on the order of
 * summation, so the ids are reproducible.  mode 0 (relocate): a row is dead when
 * !(alphas_raw > alpha_raw_min) (NaN included); only alive rows are sampled, and the dead rows are
 * listed in ascending order.  mode 1 (grow): every row but NaN ones is sampled.
 *
 * ws: gsb_mcmc_workspace_bytes(N, n) bytes, 16-byte aligned, for n draws; one workspace carries a
 * plan through its sample and relocate / grow calls.  gsb_mcmc_plan -> counts_host[2] =
 * (W_total, dead count).  HOST SYNCHRONISATION: waits for the two counts; the caller sizes the draws
 * (relocate: n = dead count) and skips a call with W_total == 0 (nothing can be sampled).
 * gsb_mcmc_sample: u[n] fp64 uniforms -> sampled[n] int32 row ids (plus the per-row hit counts c,
 * kept in ws).
 *
 * Relocation value of a source hit c times, in fp64: r = min(c + 1, n_max),
 *   o' = clamp(1 - (1 - o)^(1/r), min_opacity, 1 - 2^-23),
 *   denom = sum_{m=1..r} C(r,m) (-1)^(m+1) o'^m / sqrt(m),
 *   alphas_raw' = (float) logit(o'),  scales_raw' = (float)((double) scales_raw + log(o / denom)).
 * gsb_mcmc_relocate (in place, mode 0 plan): every source gets its relocation value, dead row j of
 *   the list becomes a copy of the updated source sampled[j]; the Adam moments (exp_avg /
 *   exp_avg_sq: NULL, or both set) of every source and destination row are zeroed.
 * gsb_mcmc_grow (mode 1 plan): dst [N + n rows] = the src rows with the sources updated, then
 *   row N + j = a copy of the updated source sampled[j]; moments carried, except zero for the
 *   sources and the new rows.  src_m/src_v/dst_m/dst_v: NULL, or all four set.
 * The _rows variants do the same to one more per-Gaussian tensor [N, D] (features): a plain copy.
 * gsb_mcmc_noise: pws += Sigma(q, s) z * scale / (1 + exp(-k ((1 - o) - x0))) with Sigma = R S^2
 *   R^T of q = normalize(rots_raw), s = exp(scales_raw), z[N,3] the caller's unit normals and
 *   scale = lr * noise_lr; in place. */
size_t gsb_mcmc_workspace_bytes(int64_t N, int64_t n);
int gsb_mcmc_plan(int64_t N, const float *alphas_raw, float alpha_raw_min, int mode, void *ws, size_t ws_bytes,
                  int64_t *counts_host, gsb_stream_t stream);
int gsb_mcmc_sample(int64_t N, int64_t n, const double *u, void *ws, size_t ws_bytes, int32_t *sampled,
                    gsb_stream_t stream);
int gsb_mcmc_relocate(int64_t N, int64_t n, const int32_t *sampled, void *ws, size_t ws_bytes, double min_opacity,
                      int n_max, const gsb_gaussians *params, const gsb_gaussians *exp_avg,
                      const gsb_gaussians *exp_avg_sq, gsb_stream_t stream);
int gsb_mcmc_relocate_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, size_t ws_bytes, int D,
                           float *x, float *exp_avg, float *exp_avg_sq, gsb_stream_t stream);
int gsb_mcmc_grow(int64_t N, int64_t n, const int32_t *sampled, void *ws, size_t ws_bytes, double min_opacity,
                  int n_max, const gsb_gaussians *src, const gsb_gaussians *src_m, const gsb_gaussians *src_v,
                  const gsb_gaussians *dst, const gsb_gaussians *dst_m, const gsb_gaussians *dst_v,
                  gsb_stream_t stream);
int gsb_mcmc_grow_rows(int64_t N, int64_t n, const int32_t *sampled, const void *ws, size_t ws_bytes, int D,
                       const float *src, const float *src_m, const float *src_v, float *dst, float *dst_m,
                       float *dst_v, gsb_stream_t stream);
int gsb_mcmc_noise(int64_t N, float *pws, const float *alphas_raw, const float *scales_raw, const float *rots_raw,
                   const float *z, float scale, float k, float x0, gsb_stream_t stream);

/* ---- fused Adam step (extension; DESIGN 3.12).  One launch updates every tensor of the table in
 * place, with torch.optim.Adam's foreach arithmetic in fp32 and in its order:
 *   m = lerp(m, g, 1 - beta1);  v = v * beta2 + (1 - beta2) * g * g;
 *   denom = sqrt(v) / bc2_sqrt + eps;  p = p - step_size * m / denom.
 * step_size = lr / (1 - beta1^t) and bc2_sqrt = sqrt(1 - beta2^t) are per tensor (the caller
 * forms them in double and rounds once).  beta1, beta2 and eps come as doubles so that 1 - beta1
 * and 1 - beta2 are formed in double and rounded once, as torch does.  numel == 0 rows are skipped.
 * Any 4-byte alignment; tensors whose four pointers share their offset mod 16 use 16-byte accesses.
 * Selective mode (visibility != NULL, uint8 [N]): every tensor has numel == N * D (D >= 1) and row
 * r = element / D is updated only where visibility[r] != 0; other rows' p, g, m and v are neither
 * read (beyond the 16-byte quads a visible row shares) nor written.  Dense mode: visibility NULL,
 * N = 0.  An empty table, or N = 0 in selective mode, is a no-op. */
typedef struct gsb_adam_tensor {
  float *param;
  const float *grad;
  float *exp_avg;
  float *exp_avg_sq;
  int64_t numel;
  int32_t D;       /* row width (selective mode) */
  float step_size; /* lr / (1 - beta1^t) */
  float bc2_sqrt;  /* sqrt(1 - beta2^t) */
} gsb_adam_tensor;
int gsb_adam_step(int n_tensors, const gsb_adam_tensor *table, int64_t N, const uint8_t *visibility, double beta1,
                  double beta2, double eps, gsb_stream_t stream);

/* ---- Gaussian record conversion (extension; SURVEY 8f row N3, gsplat/gau_io.py).  A "gs row"
 * is the reference's .npy record (gau_io.py:7-12): pw[3] rot[4] scale[3] alpha sh[sh_dim],
 * 11 + sh_dim floats, activated values.
 * gsb_ply_rows_to_gs: load_ply's arithmetic (:60-107) on the PLY vertex block rows[N,stride]:
 *   colmap[11 + sh_dim] (device, int32) = source column of each output column (the host folds
 *   the f_rest channel-major -> coefficient-major transpose of :91 into it); rot / |rot|,
 *   exp(scale), sigmoid(opacity).
 * gsb_gs_to_params: get_training_params (gsmodel.py:95-113): gs rows -> the six raw tensors,
 *   high_shs padded with 0.001 up to 45 columns.   sh_dim in {3, 12, 27, 48}.
 * gsb_params_to_gs: save_training_params (gau_io.py:138-153): -> gs rows with sh_dim = 48. */
int gsb_ply_rows_to_gs(int64_t N, int stride, int sh_dim, const float *rows, const int32_t *colmap,
                       float *gs_rows, gsb_stream_t stream);
int gsb_gs_to_params(int64_t N, int sh_dim, const float *gs_rows, const gsb_gaussians *dst, gsb_stream_t stream);
int gsb_params_to_gs(int64_t N, const gsb_gaussians *src, float *gs_rows, gsb_stream_t stream);

/* ---- multi-GPU gradient exchange (extension; SURVEY 8e -- the reference is single-GPU).
 * Multi-view data parallelism: one process per GPU, Gaussians replicated, one camera per rank;
 * the parameter gradients (dshs, drots, dpws, dscales, dalphas = 3k + 11 floats per Gaussian)
 * must be summed over ranks.  Instead of an all-reduce after the backward, the fused
 * per-Gaussian backward PUSHES each gradient tile into peer memory while it computes
 * (gsb_preprocess_backward_push), and one kernel sums and broadcasts
 * (gsb_grad_reduce_broadcast).  Protocol, per step, on every rank, same `epoch` (1, 2, 3, ...):
 *     gsb_preprocess_backward_push(...);  gsb_grad_reduce_broadcast(...);
 * after which the summed gradients sit in the rank's own region at
 * gsb_exchange_result_offset(..., segment), segment 0..4 = dshs [R,3k], drots [R,4], dpws [R,3],
 * dscales [R,3], dalphas [R,1] with R = world * rows-per-rank >= N (rows >= N are padding).
 *
 * A "region" is device memory of gsb_exchange_region_bytes(N, sh_dim3, world) bytes obtained
 * from gsb_comm_alloc (cudaMalloc + zero fill + CUDA IPC handle, GSB_COMM_HANDLE_BYTES bytes);
 * the handles are exchanged between the processes by the caller (any transport) and opened
 * with gsb_comm_open.  regions_host[world]: HOST array of device pointers, entry r = rank r's
 * region as seen from this process (own pointer for r == rank).  world in {1, 2, 4, 8}.
 * gsb_preprocess_backward_push takes the upstream gradients either as the four dloss_d* tensors
 * or, like gsb_preprocess_backward, as moments[N,9] + cinv2ds[N,3] (+ dloss_dus_out[N,2]).
 * The kernels spin on flags in peer memory with a 5 s timeout; gsb_exchange_status returns 1
 * if a wait ever timed out (a peer missing) -- the results are then invalid. */
#define GSB_COMM_HANDLE_BYTES 64
size_t gsb_exchange_region_bytes(int N, int sh_dim3, int world);
size_t gsb_exchange_result_offset(int N, int sh_dim3, int world, int segment);
int gsb_comm_alloc(size_t bytes, void **ptr, void *handle_out);
int gsb_comm_open(const void *handle, void **peer_ptr);
int gsb_comm_close(void *peer_ptr);
int gsb_comm_free(void *ptr);
int gsb_exchange_status(const void *region, int *status_host);
int gsb_preprocess_backward_push(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                 const float *shs, const float *Rcw, const float *tcw, const float *twc,
                                 float fx, float fy, float cx, float cy, float width, float height,
                                 const float *dloss_dus, const float *dloss_dcinv2ds, const float *dloss_dcolors,
                                 const float *dloss_dalphas, const float *moments, const float *cinv2ds,
                                 float *dloss_dus_out, int world, int rank, void *const *regions_host,
                                 uint32_t epoch, gsb_stream_t stream);
int gsb_grad_reduce_broadcast(int N, int sh_dim3, int world, int rank, void *const *regions_host, uint32_t epoch,
                              gsb_stream_t stream);

/* ---- 2D Gaussian Splatting (extension; DESIGN 3.15): each Gaussian is a flat disk (surfel) with
 * axes scales[:,0] R e0 and scales[:,1] R e1 (scales[:,2] is not read), drawn where the pixel's ray
 * meets it; pinhole cameras only.
 * gsb_surfel_preprocess_forward: us[N,2], depths[N] (-1 = culled), areas[N,2] (integer half-extents
 * of the 3-sigma footprint), colors[N,3] (the SH colour of gsb_preprocess_forward) and records
 * [N,20] floats (16-byte aligned), the rasterizers' per-surfel input.  alphas[N] is read into the
 * records.  N == 0 does nothing. */
int gsb_surfel_preprocess_forward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                  const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                  float fy, float cx, float cy, float width, float height, const float *alphas,
                                  float *us, float *depths, int32_t *areas, float *colors, float *records,
                                  gsb_stream_t stream);
/* rows[N,18]: the gradient rows gsb_splat_surfel_backward wrote.  Writes dloss_dpws[N,3],
 * dloss_dshs[N,3k], dloss_dalphas[N], dloss_dscales[N,3] (column 2: 0), dloss_drots[N,4] and
 * dloss_dus[N,2] (dL/d of a screen-space shift of the whole surfel: the densification statistic). */
int gsb_surfel_preprocess_backward(int N, int sh_dim3, const float *pws, const float *rots, const float *scales,
                                   const float *shs, const float *Rcw, const float *tcw, const float *twc, float fx,
                                   float fy, float cx, float cy, float width, float height, const float *rows,
                                   float *dloss_dpws, float *dloss_dshs, float *dloss_dalphas, float *dloss_dscales,
                                   float *dloss_drots, float *dloss_dus, gsb_stream_t stream);
/* Workspace of gsb_splat_surfel_render / _forward for P patches (P_cap), and of
 * gsb_splat_surfel_backward with P = 0.  The binning is gsb_splat_bin's (its bin_ws). */
size_t gsb_splat_surfel_workspace_bytes(int N, int H, int W, int64_t P);
/* The frame binned by gsb_splat_bin (P patches, largest depth key depth_key_max), drawn from the
 * records: image[3,H,W], contrib, final_tau, patch_range_per_tile, gsid_per_patch as gsb_splat_render,
 * depth_image[H,W] = sum w z(p) (the camera-frame depth of each ray-splat hit, not normalised),
 * alpha_image[H,W] = sum w and normal_image[3,H,W] = sum w n (camera frame).  Every plane and
 * records 16-byte aligned, patch_range_per_tile 8-byte aligned. */
int gsb_splat_surfel_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us,
                            const float *depths, const float *records, const void *bin_ws, void *ws, size_t ws_bytes,
                            float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                            int32_t *gsid_per_patch, float *depth_image, float *alpha_image, float *normal_image,
                            gsb_stream_t stream);
/* The capacity form (as gsb_splat_forward): bins here, sorts into P_cap slots, and returns
 * GSB_CAPACITY_EXCEEDED when the frame outgrew P_cap or depth_key_cap (status_host as there). */
int gsb_splat_surfel_forward(int H, int W, int N, const float *us, float *depths, int32_t *areas,
                             const float *records, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                             size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                             float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                             uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                             gsb_stream_t stream);
/* Backward of the surfel frame: upstream planes dloss_dimage[3,H,W], dloss_ddepth[H,W],
 * dloss_dalpha[H,W], dloss_dnormal[3,H,W], each nullable (NULL = zero; a frame with none of them
 * costs one memset).  rows[N,18] (written in full): [dL/dM (9), dL/dalpha, dL/dcolour (3), dL/dn (3),
 * dL/ddelta (2)] per surfel, for gsb_surfel_preprocess_backward. */
int gsb_splat_surfel_backward(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                              const float *final_tau, const int32_t *patch_range_per_tile,
                              const int32_t *gsid_per_patch, const float *dloss_dimage, const float *dloss_ddepth,
                              const float *dloss_dalpha, const float *dloss_dnormal, void *ws, size_t ws_bytes,
                              float *rows, gsb_stream_t stream);

/* ---- 2D Gaussian Splatting geometry terms (extension; DESIGN 3.16): the surfel frame of
 * gsb_splat_surfel_render / _forward / _backward (same arguments, same workspace:
 * gsb_splat_surfel_workspace_bytes, same planes bit for bit) with 2DGS's depth-distortion and
 * median-depth planes.  Per pixel, over the contributing records in compositing order (w = tau alpha'):
 *   m(z) = far / (far - near) (1 - near / max(z, near))   (z: the record's hit depth; 0 < near < far)
 *   distortion[H,W] = sum_{j<i} w_i w_j (m_i - m_j)^2,  moments[2,H,W] = (sum w m, sum w m^2),
 *   median_depth[H,W] = z of the last record whose incoming tau > 0.5 (0 where none contributes),
 *   median_contrib[H,W] (int32) = that record's patch index in its tile + 1 (0: none), as contrib.
 * Every geometry plane is 16-byte aligned; all are written in full. */
int gsb_splat_2dgs_render(int H, int W, int N, int64_t P, uint32_t depth_key_max, const float *us, const float *depths,
                          const float *records, float near, float far, const void *bin_ws, void *ws, size_t ws_bytes,
                          float *image, int32_t *contrib, float *final_tau, int32_t *patch_range_per_tile,
                          int32_t *gsid_per_patch, float *depth_image, float *alpha_image, float *normal_image,
                          float *distortion, float *moments, float *median_depth, int32_t *median_contrib,
                          gsb_stream_t stream);
/* The capacity form (as gsb_splat_surfel_forward). */
int gsb_splat_2dgs_forward(int H, int W, int N, const float *us, float *depths, int32_t *areas, const float *records,
                           float near, float far, int64_t P_cap, uint32_t depth_key_cap, void *bin_ws,
                           size_t bin_ws_bytes, void *ws, size_t ws_bytes, float *image, int32_t *contrib,
                           float *final_tau, int32_t *patch_range_per_tile, int32_t *gsid_per_patch,
                           uint32_t *status_host, float *depth_image, float *alpha_image, float *normal_image,
                           float *distortion, float *moments, float *median_depth, int32_t *median_contrib,
                           gsb_stream_t stream);
/* Backward of the geometry frame: gsb_splat_surfel_backward's arguments, plus the forward's
 * alpha_image, moments and median_contrib and the upstream dloss_ddistortion[H,W] and
 * dloss_dmedian[H,W] (each nullable; with both NULL this is gsb_splat_surfel_backward and the three
 * forward planes are not read).  Those five planes are 4-byte aligned.  rows[N,18] as there. */
int gsb_splat_2dgs_backward(int H, int W, int N, int64_t P, const float *records, const int32_t *contrib,
                            const float *final_tau, const int32_t *patch_range_per_tile, const int32_t *gsid_per_patch,
                            const float *dloss_dimage, const float *dloss_ddepth, const float *dloss_dalpha,
                            const float *dloss_dnormal, void *ws, size_t ws_bytes, float *rows, float near, float far,
                            const float *alpha_image, const float *moments, const int32_t *median_contrib,
                            const float *dloss_ddistortion, const float *dloss_dmedian, gsb_stream_t stream);

/* ---- mesh extraction (extension; DESIGN 3.17): projective TSDF fusion of depth maps into a
 * dense grid and marching cubes over it, the step that turns a trained 2D Gaussian Splatting
 * model into a mesh.
 *
 * The grid has nx x ny x nz sample points; point (i, j, k) sits at (ox, oy, oz) + voxel (i, j, k).
 * Arrays are [nz, ny, nx] float32 with x fastest: tsdf, weight, and the optional color_grid
 * [3, nz, ny, nx].  A new volume is tsdf 1, weight 0, colour 0 (the caller fills it).  Every
 * dimension >= 1 and nx ny nz < 2^31.  Device arrays are 4-byte aligned.
 *
 * gsb_tsdf_integrate fuses V views in one launch, in view order.  cams: V rows of the [V, 20]
 * camera table (Rcw row-major 9, tcw 3, fx, fy, cx, cy, W, H, 2 unused; pinhole), depth[V, H, W],
 * color[V, 3, H, W] (NULL with color_grid NULL).  For every point p and view:
 *   pc = Rcw p + tcw, skipped unless pc.z > 0;  u = fx pc.x / pc.z + cx, v = fy pc.y / pc.z + cy;
 *   skipped unless 0 <= u + 1/2 < W and 0 <= v + 1/2 < H;  pixel (floor(u + 1/2), floor(v + 1/2));
 *   D = depth there, skipped unless finite and 0 < D <= depth_trunc;  sdf = D - pc.z, skipped if
 *   sdf < -trunc;  t = min(1, sdf / trunc);
 *   tsdf <- (tsdf w + t) / (w + 1), colour <- (colour w + c) / (w + 1), w <- w + 1.
 * One launch of V views and V launches of one view give bit-identical grids.  Refused: a bad
 * dimension or voxel count, voxel or trunc not finite and > 0, depth_trunc not > 0 (inf allowed),
 * an origin not finite, V, H or W < 1, colour on one side only.
 *
 * Extraction: a point is observed when w > 0 and inside when tsdf < 0; a cell (8 points, lowest
 * corner g) is valid when all 8 are observed.  Edge (g, axis a) has a vertex when its ends differ
 * in insideness and a valid cell contains it, at p_g + voxel e_a f, f = T_g / (T_g - T_{g+e_a}),
 * colour C_g + f (C_{g+e_a} - C_g); vertices in order of (linear index of g, a).  Faces: valid
 * cells in linear order, each cell's triangles in table order (mc_table.h), oriented from inside to
 * outside; int32 indices into the vertices.  The output is deterministic.
 * gsb_tsdf_extract_plan -> counts_host[2] = (vertices, faces).  HOST SYNCHRONISATION: it waits for
 * the counts; the caller sizes verts[V, 3], vcolors[V, 3] and faces[F, 3] from them and passes the
 * same workspace, grid and counts to gsb_tsdf_extract_emit.  n_verts and n_faces must be exactly the
 * plan's counts: the emit writes no vertex id >= n_verts and no face slot >= n_faces, so smaller
 * counts, or a workspace planned for another grid, give a wrong mesh but no write past the
 * buffers.  A count of 2^31 or more is refused
 * (by the plan, after writing the counts).  A grid with a dimension of 1 has no cells: 0, 0.
 * vcolors: NULL, or with color_grid. */
int gsb_tsdf_integrate(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc,
                       float depth_trunc, int V, int H, int W, const float *cams, const float *depth,
                       const float *color, float *tsdf, float *weight, float *color_grid, gsb_stream_t stream);
size_t gsb_tsdf_extract_workspace_bytes(int nx, int ny, int nz);
int gsb_tsdf_extract_plan(int nx, int ny, int nz, const float *tsdf, const float *weight, void *ws, size_t ws_bytes,
                          int64_t *counts_host, gsb_stream_t stream);
int gsb_tsdf_extract_emit(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float *tsdf,
                          const float *weight, const float *color_grid, const void *ws, size_t ws_bytes,
                          int64_t n_verts, int64_t n_faces, float *verts, float *vcolors, int32_t *faces,
                          gsb_stream_t stream);

/* ---- bilateral-grid colour correction (extension; DESIGN 3.20; Wang et al., "Bilateral Guided
 * Radiance Field Processing", SIGGRAPH 2024).  One learnable grid of 3 x 4 affine colour matrices per
 * training image, sliced on the rendered image before the loss.
 *
 * grids[M, 12, L, Y, X] float32 (gsplat's layout): channel c = 4 r + k holds A[r][k]; identity is
 * A = [I | 0].  1 <= X, Y, L <= GSB_BILAGRID_MAX_DIM, M >= 1.  rgb, out, dloss_dout, dloss_drgb:
 * B planar images [B, 3, H, W], 1 <= B <= GSB_BILAGRID_MAX_BATCH, H, W >= 1, H W < 2^31.
 * image_ids: a HOST array of B grid indices in [0, M), read by the call (no device read, no
 * synchronisation); two items may name the same grid.  Device arrays are 4-byte aligned.
 * For pixel (px, py) of item b, with G = grids[image_ids[b]]:
 *   g  = 0.299 r + 0.587 g + 0.114 b                      (guidance: the luminance of the input)
 *   gx = (px + 1/2) / W (X - 1),  gy = (py + 1/2) / H (Y - 1),  gz = clamp(g, 0, 1) (L - 1)
 *   A  = trilinear interpolation of G at (gx, gy, gz)     (an axis of size 1 is constant along it)
 *   out[:, p] = A[:, :3] rgb[:, p] + A[:, 3]
 * i.e. F.grid_sample(G[None], 2 xyz - 1, bilinear, padding "border", align_corners=True) at
 * xyz = ((px + 1/2) / W, (py + 1/2) / H, g).
 * gsb_bilagrid_slice_backward writes dloss_drgb = A[:, :3]^T dL/dout + (dL/dout . dA/dgz [rgb; 1])
 * (L - 1) (0.299, 0.587, 0.114), the last term only where 0 < g < 1, and ADDS
 * w_corner dL/dout_r [rgb, 1]_k into dloss_dgrids[M, 12, L, Y, X] (the caller zeroes it).  The grid
 * gradient is summed with one float atomicAdd per CTA and window element, so it is not
 * bit-reproducible from run to run; dloss_drgb is.
 * gsb_bilagrid_tv: TV = sum over the axes a in {L, Y, X} of mean((G shifted by one along a - G)^2)
 * over all M grids (an axis of size 1 adds 0); writes *tv_out (device) and, when dloss_dgrids is not
 * NULL, dTV/dgrids (written, not added).  ws: gsb_bilagrid_tv_workspace_bytes bytes, 8-byte aligned.
 * The value is bit-reproducible. */
#define GSB_BILAGRID_MAX_DIM 64
#define GSB_BILAGRID_MAX_BATCH 64
int gsb_bilagrid_slice(int M, int L, int Y, int X, const float *grids, int B, const int32_t *image_ids, int H, int W,
                       const float *rgb, float *out, gsb_stream_t stream);
int gsb_bilagrid_slice_backward(int M, int L, int Y, int X, const float *grids, int B, const int32_t *image_ids,
                                int H, int W, const float *rgb, const float *dloss_dout, float *dloss_drgb,
                                float *dloss_dgrids, gsb_stream_t stream);
size_t gsb_bilagrid_tv_workspace_bytes(int M, int L, int Y, int X);
int gsb_bilagrid_tv(int M, int L, int Y, int X, const float *grids, float *tv_out, float *dloss_dgrids, void *ws,
                    size_t ws_bytes, gsb_stream_t stream);

/* ---- launch accounting and optional per-kernel timing (no reference counterpart; used by
 * bench.py for `gpu_launches` and the roofline's live CUDA-event kernel durations).
 * Kernel ids 0..gsb_profile_kernels()-1, names from gsb_profile_kernel_name().
 * gsb_profile_launches(id) counts launches since load (id < 0: all kernels).
 * While enabled, every kernel launch is bracketed by two events on its stream;
 * gsb_profile_read() waits for them, returns the summed duration and clears the list. */
void gsb_profile_enable(int on);
int gsb_profile_kernels(void);
const char *gsb_profile_kernel_name(int id);
long long gsb_profile_launches(int id);
int gsb_profile_read(int id, double *ms_total, long long *timed_launches);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H_ */
