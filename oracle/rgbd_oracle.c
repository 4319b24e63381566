/* RGB-D oracle (test infrastructure only): fp64 depth and opacity compositing and its backward.
 *
 * An extension of gs_oracle.c, not a separate model: it is compiled together with it (the
 * #include below) so that it shares orc_draw's alpha'(), thresholds, tile size and ambiguity
 * rules by construction rather than by copy.  Built into its own library by
 * oracle/rgbd_oracle.py; gs_oracle.c and its library are unchanged.
 * The reference renders colour only, so there is no golden fixture for these functions:
 * tests/test_rgbd_cpu.py pins them against orc_draw / orc_drawB and against central
 * differences of the whole chain. */
#include "gs_oracle.c"

/* ------------------------------------------------------------------------------------
 * RGB-D compositing (an extension; the reference renders colour only).  Depth and opacity
 * composite like two more colour channels whose per-Gaussian values are z = depths[g] and 1:
 *   D[p] = sum_i w_i z_i,  A[p] = sum_i w_i,  w_i = tau_i alpha'_i
 * with exactly orc_draw's rules (same clamp, skip, stop, contrib and ambiguity flags); pixels of
 * empty tiles get D = A = 0.  image / contrib / final_tau equal orc_draw's.
 * ---------------------------------------------------------------------------------- */
void orc_draw_rgbd(int H, int W, const int32_t *ranges, const int32_t *gsid, const float *us,
                   const float *cinv2ds, const float *alphas, const float *colors, const float *depths,
                   double *image, double *depth_image, double *alpha_image, int32_t *contrib,
                   double *final_tau, uint8_t *ambiguous, double margin) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
  memset(image, 0, sizeof(double) * 3 * HW);
  memset(depth_image, 0, sizeof(double) * HW);
  memset(alpha_image, 0, sizeof(double) * HW);
  memset(contrib, 0, sizeof(int32_t) * HW);
  memset(final_tau, 0, sizeof(double) * HW);
  if (ambiguous) memset(ambiguous, 0, HW);
#pragma omp parallel for schedule(dynamic, 4)
  for (int t = 0; t < gx * gy; t++) {
    int start = ranges[2 * t], end = ranges[2 * t + 1];
    if (end - start == 0) continue;
    int tx = t % gx, ty = t / gx;
    for (int py = ty * TILE; py < imin(H, ty * TILE + TILE); py++)
      for (int px = tx * TILE; px < imin(W, tx * TILE + TILE); px++) {
        double tau = 1.0, col[5] = {0, 0, 0, 0, 0};
        int cont = 0, amb = 0;
        for (int p = start; p < end; p++) {
          int g = gsid[p];
          double dx = (double)us[2 * g] - px, dy = (double)us[2 * g + 1] - py;
          double ap = alpha_prime(alphas[g], cinv2ds[3 * g], cinv2ds[3 * g + 1],
                                  cinv2ds[3 * g + 2], dx, dy, NULL);
          if (fabs(ap - ALPHA_SKIP) <= margin * ALPHA_SKIP) amb = 1;
          if (ap < ALPHA_SKIP) continue;
          const double val[5] = {colors[3 * g], colors[3 * g + 1], colors[3 * g + 2], depths[g], 1.0};
          for (int c = 0; c < 5; c++) col[c] += tau * ap * val[c];
          cont = p - start + 1;
          tau *= (1.0 - ap);
          if (fabs(tau - TAU_STOP) <= 10 * margin * TAU_STOP) amb = 1;
          if (tau < TAU_STOP) break;
        }
        size_t pix = (size_t)py * W + px;
        image[pix] = col[0];
        image[HW + pix] = col[1];
        image[2 * HW + pix] = col[2];
        depth_image[pix] = col[3];
        alpha_image[pix] = col[4];
        contrib[pix] = cont;
        final_tau[pix] = tau;
        if (ambiguous) ambiguous[pix] = (uint8_t)amb;
      }
  }
}

/* Backward of orc_draw_rgbd: orc_drawB with the five-channel upstream gradient
 * (dL/dimage[3,H,W], dL/dD[H,W], dL/dA[H,W]) and values (colour, z, 1), so
 *   dL/dalpha' = tau sum_c dl_c (val_c - next_c)  over the five channels,
 *   dL/dz_g   = sum over the pixels it reaches of dl_D alpha' tau   -> dloss_ddepths[N].
 * With dL/dD = dL/dA = 0 it equals orc_drawB (and dloss_ddepths = 0). */
void orc_drawB_rgbd(int H, int W, int N, const int32_t *ranges, const int32_t *gsid,
                    const float *us, const float *cinv2ds, const float *alphas,
                    const float *colors, const float *depths, const double *final_tau,
                    const int32_t *contrib, const float *dloss_dgammas, const float *dloss_ddepth_image,
                    const float *dloss_dalpha_image, double *dloss_dus, double *dloss_dcinv2ds,
                    double *dloss_dalphas, double *dloss_dcolors, double *dloss_ddepths, uint8_t *amb_gs,
                    double margin) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
  if (amb_gs) memset(amb_gs, 0, (size_t)N);
  memset(dloss_dus, 0, sizeof(double) * 2 * N);
  memset(dloss_dcinv2ds, 0, sizeof(double) * 3 * N);
  memset(dloss_dalphas, 0, sizeof(double) * N);
  memset(dloss_dcolors, 0, sizeof(double) * 3 * N);
  memset(dloss_ddepths, 0, sizeof(double) * N);
#pragma omp parallel for schedule(dynamic, 4)
  for (int t = 0; t < gx * gy; t++) {
    int start = ranges[2 * t], end = ranges[2 * t + 1];
    if (end - start == 0) continue;
    int tx = t % gx, ty = t / gx;
    for (int py = ty * TILE; py < imin(H, ty * TILE + TILE); py++)
      for (int px = tx * TILE; px < imin(W, tx * TILE + TILE); px++) {
        size_t pix = (size_t)py * W + px;
        double dl[5] = {dloss_dgammas[pix], dloss_dgammas[HW + pix], dloss_dgammas[2 * HW + pix],
                        dloss_ddepth_image[pix], dloss_dalpha_image[pix]};
        double tau = final_tau[pix];
        double gn[5] = {0, 0, 0, 0, 0};
        for (int p = start + contrib[pix] - 1; p >= start; p--) {
          int g = gsid[p];
          double A = cinv2ds[3 * g], B = cinv2ds[3 * g + 1], C = cinv2ds[3 * g + 2];
          double dx = (double)us[2 * g] - px, dy = (double)us[2 * g + 1] - py;
          double gg;
          double ap = alpha_prime(alphas[g], A, B, C, dx, dy, &gg);
          if (amb_gs && fabs(ap - ALPHA_SKIP) <= margin * ALPHA_SKIP) amb_gs[g] = 1;
          if (ap < ALPHA_SKIP) continue;
          tau = tau / (1.0 - ap);
          const double val[5] = {colors[3 * g], colors[3 * g + 1], colors[3 * g + 2], depths[g], 1.0};
          double dl_dap = 0;
          for (int c = 0; c < 5; c++) dl_dap += dl[c] * tau * (val[c] - gn[c]);
          double v[10];
          v[0] = dl_dap * ap * (-A * dx - B * dy);
          v[1] = dl_dap * ap * (-B * dx - C * dy);
          v[2] = dl_dap * (-0.5 * ap * dx * dx);
          v[3] = dl_dap * (-1.0 * ap * dx * dy);
          v[4] = dl_dap * (-0.5 * ap * dy * dy);
          v[5] = dl_dap * gg;
          for (int c = 0; c < 3; c++) v[6 + c] = dl[c] * ap * tau;
          v[9] = dl[3] * ap * tau;
          double *dst[10] = {&dloss_dus[2 * g],      &dloss_dus[2 * g + 1],
                             &dloss_dcinv2ds[3 * g], &dloss_dcinv2ds[3 * g + 1],
                             &dloss_dcinv2ds[3 * g + 2], &dloss_dalphas[g],
                             &dloss_dcolors[3 * g],  &dloss_dcolors[3 * g + 1],
                             &dloss_dcolors[3 * g + 2], &dloss_ddepths[g]};
          for (int k = 0; k < 10; k++) {
#pragma omp atomic
            *dst[k] += v[k];
          }
          for (int c = 0; c < 5; c++) gn[c] = ap * val[c] + (1.0 - ap) * gn[c];
        }
      }
  }
}

