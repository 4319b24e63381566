/* Absolute-gradient oracle (test infrastructure only): fp64 per-pixel absolute sums of dL/du.
 *
 * An extension of gs_oracle.c and rgbd_oracle.c, compiled together with them (the #include below)
 * so that it shares orc_drawB's alpha'(), skip, clamp and ambiguity rules by construction rather
 * than by copy.  Built into its own library by oracle/absgrad_oracle.py; the other oracle sources
 * and their libraries are unchanged.
 *
 * orc_drawB (and orc_drawB_rgbd) sum, per Gaussian g, one term per replayed (pixel, record) pair
 *   g_ip = w_ip (-A dx - B dy, -B dx - C dy),   w_ip = dL/dalpha'_ip alpha'_ip
 * into dloss_dus.  AbsGS densifies on the sums of their absolute values instead,
 *   dloss_dus_abs[g] = ( sum_p |g_ip.x| , sum_p |g_ip.y| ),
 * which per-pixel terms of opposite sign cannot cancel.  Both functions return the signed sums
 * (equal to orc_drawB's / orc_drawB_rgbd's dloss_dus) next to the absolute ones. */
#include "rgbd_oracle.c"

/* nch = 3: the colour frame (dl = dL/dimage); nch = 5: the RGB-D frame (also dL/dD, dL/dA with
 * values z, 1), as orc_drawB_rgbd. */
static void drawB_abs(int nch, int H, int W, int N, const int32_t *ranges, const int32_t *gsid, const float *us,
                      const float *cinv2ds, const float *alphas, const float *colors, const float *depths,
                      const double *final_tau, const int32_t *contrib, const float *dloss_dgammas,
                      const float *dloss_ddepth_image, const float *dloss_dalpha_image, double *dloss_dus,
                      double *dloss_dus_abs, uint8_t *amb_gs, double margin) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
  if (amb_gs) memset(amb_gs, 0, (size_t)N);
  memset(dloss_dus, 0, sizeof(double) * 2 * N);
  memset(dloss_dus_abs, 0, sizeof(double) * 2 * N);
#pragma omp parallel for schedule(dynamic, 4)
  for (int t = 0; t < gx * gy; t++) {
    int start = ranges[2 * t], end = ranges[2 * t + 1];
    if (end - start == 0) continue;
    int tx = t % gx, ty = t / gx;
    for (int py = ty * TILE; py < imin(H, ty * TILE + TILE); py++)
      for (int px = tx * TILE; px < imin(W, tx * TILE + TILE); px++) {
        size_t pix = (size_t)py * W + px;
        double dl[5] = {dloss_dgammas[pix], dloss_dgammas[HW + pix], dloss_dgammas[2 * HW + pix], 0, 0};
        if (nch == 5) {
          dl[3] = dloss_ddepth_image[pix];
          dl[4] = dloss_dalpha_image[pix];
        }
        double tau = final_tau[pix];
        double gn[5] = {0, 0, 0, 0, 0};
        for (int p = start + contrib[pix] - 1; p >= start; p--) {
          int g = gsid[p];
          double A = cinv2ds[3 * g], B = cinv2ds[3 * g + 1], C = cinv2ds[3 * g + 2];
          double dx = (double)us[2 * g] - px, dy = (double)us[2 * g + 1] - py;
          double ap = alpha_prime(alphas[g], A, B, C, dx, dy, NULL);
          if (amb_gs && fabs(ap - ALPHA_SKIP) <= margin * ALPHA_SKIP) amb_gs[g] = 1;
          if (ap < ALPHA_SKIP) continue;
          tau = tau / (1.0 - ap);
          const double val[5] = {colors[3 * g], colors[3 * g + 1], colors[3 * g + 2], nch == 5 ? depths[g] : 0.0,
                                 1.0};
          double dl_dap = 0;
          for (int c = 0; c < nch; c++) dl_dap += dl[c] * tau * (val[c] - gn[c]);
          const double v[4] = {dl_dap * ap * (-A * dx - B * dy), dl_dap * ap * (-B * dx - C * dy), 0, 0};
          double *dst[4] = {&dloss_dus[2 * g], &dloss_dus[2 * g + 1], &dloss_dus_abs[2 * g], &dloss_dus_abs[2 * g + 1]};
          const double add[4] = {v[0], v[1], fabs(v[0]), fabs(v[1])};
          for (int k = 0; k < 4; k++) {
#pragma omp atomic
            *dst[k] += add[k];
          }
          for (int c = 0; c < nch; c++) gn[c] = ap * val[c] + (1.0 - ap) * gn[c];
        }
      }
  }
}

/* The colour frame: orc_drawB's arguments (its dloss_dus) plus dloss_dus_abs[N,2]. */
void orc_drawB_abs(int H, int W, int N, const int32_t *ranges, const int32_t *gsid, const float *us,
                   const float *cinv2ds, const float *alphas, const float *colors, const double *final_tau,
                   const int32_t *contrib, const float *dloss_dgammas, double *dloss_dus, double *dloss_dus_abs,
                   uint8_t *amb_gs, double margin) {
  drawB_abs(3, H, W, N, ranges, gsid, us, cinv2ds, alphas, colors, NULL, final_tau, contrib, dloss_dgammas, NULL,
            NULL, dloss_dus, dloss_dus_abs, amb_gs, margin);
}

/* The RGB-D frame: orc_drawB_rgbd's arguments (its dloss_dus) plus dloss_dus_abs[N,2]. */
void orc_drawB_rgbd_abs(int H, int W, int N, const int32_t *ranges, const int32_t *gsid, const float *us,
                        const float *cinv2ds, const float *alphas, const float *colors, const float *depths,
                        const double *final_tau, const int32_t *contrib, const float *dloss_dgammas,
                        const float *dloss_ddepth_image, const float *dloss_dalpha_image, double *dloss_dus,
                        double *dloss_dus_abs, uint8_t *amb_gs, double margin) {
  drawB_abs(5, H, W, N, ranges, gsid, us, cinv2ds, alphas, colors, depths, final_tau, contrib, dloss_dgammas,
            dloss_ddepth_image, dloss_dalpha_image, dloss_dus, dloss_dus_abs, amb_gs, margin);
}
