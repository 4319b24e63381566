/* Contribution-statistics oracle (test infrastructure only): fp64 per-Gaussian sums, maxima and
 * counts of the blending weights w = tau alpha' of one colour frame.
 *
 * An extension of gs_oracle.c, compiled together with it (the #include below) so that alpha'(),
 * the 0.002 skip, the 1e-4 stop and the 0.99 clamp are orc_draw's by construction rather than by
 * copy.  Built into its own library by oracle/stats_oracle.py; gs_oracle.c and its library are
 * unchanged.
 *
 * orc_draw_stats walks every pixel front to back exactly as orc_draw does and adds, for each record
 * the pixel composites (alpha' >= 0.002, before the stop),
 *   weight_sum[g] += w,  weight_max[g] = max(weight_max[g], w),  hit_count[g] += 1.
 * amb_gs[N] (optional): 1 for a Gaussian an fp32 kernel may score differently because a decision
 * came within `margin` (relative) of its threshold: its own alpha' near 0.002 or alpha g near the
 * 0.99 clamp; a tau near 1e-4 (the record after the stop, or the one the stop was taken at); and a
 * record a pixel reaches after such a decision with a weight near the Gaussian's maximum (the
 * other side of the decision moves tau, and so that weight). */
#include "gs_oracle.c"

/* One walk of every pixel.  pass 0 adds the statistics and flags the Gaussians of the decisions
 * near a threshold; pass 1 (weight_max known) flags the Gaussians whose weight after such a decision
 * at the pixel comes within LATE_REL of their maximum: the other side of the decision moves tau,
 * and so those weights, by up to ~0.2 % (1 - 0.002, or 1 - 0.99 against 1 - 0.99 (1 + margin)).
 * After a near decision the stop is judged near within STOP_REL. */
#define LATE_REL 5e-3
#define STOP_REL 5e-3
static void draw_stats_pass(int pass, int H, int W, const int32_t *ranges, const int32_t *gsid, const float *us,
                            const float *cinv2ds, const float *alphas, double *weight_sum, double *weight_max,
                            int64_t *hit_count, uint8_t *amb_gs, double margin) {
  const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
#pragma omp parallel for schedule(dynamic, 4)
  for (int t = 0; t < gx * gy; t++) {
    int start = ranges[2 * t], end = ranges[2 * t + 1];
    if (end - start == 0) continue;
    int tx = t % gx, ty = t / gx;
    for (int py = ty * TILE; py < imin(H, ty * TILE + TILE); py++)
      for (int px = tx * TILE; px < imin(W, tx * TILE + TILE); px++) {
        double tau = 1.0;
        int amb = 0, stopped = 0;
        for (int p = start; p < end; p++) {
          int g = gsid[p];
          double dx = (double)us[2 * g] - px, dy = (double)us[2 * g + 1] - py, gg;
          double ap = alpha_prime(alphas[g], cinv2ds[3 * g], cinv2ds[3 * g + 1], cinv2ds[3 * g + 2], dx, dy, &gg);
          const double ag = alphas[g] * gg;
          const int reach = ap >= ALPHA_SKIP * (1.0 - margin);  /* composited on one side of the skip */
          const int near = fabs(ap - ALPHA_SKIP) <= margin * ALPHA_SKIP || fabs(ag - ALPHA_CLAMP) <= margin * ALPHA_CLAMP;
          if (stopped) {  /* the record after a near stop */
            if (reach) {
              if (pass == 0 && amb_gs) {
#pragma omp atomic write
                amb_gs[g] = 1;
              }
              break;
            }
            continue;
          }
          if (pass == 0 && near && amb_gs) {
#pragma omp atomic write
            amb_gs[g] = 1;
          }
          if (ap < ALPHA_SKIP) {
            amb |= near;
            continue;
          }
          const double w = tau * ap;
          if (pass == 0) {
#pragma omp atomic
            weight_sum[g] += w;
#pragma omp atomic
            hit_count[g] += 1;
            double cur;
#pragma omp atomic read
            cur = weight_max[g];
            if (w > cur) {
#pragma omp critical(stats_max)
              if (w > weight_max[g]) weight_max[g] = w;
            }
          } else if (amb && amb_gs && w >= (1.0 - LATE_REL) * weight_max[g]) {
#pragma omp atomic write
            amb_gs[g] = 1;
          }
          amb |= near;
          tau *= (1.0 - ap);
          const int near_stop = fabs(tau - TAU_STOP) <= (amb ? STOP_REL : 10 * margin) * TAU_STOP;
          if (near_stop) {
            amb = 1;
            if (pass == 0 && amb_gs) {
#pragma omp atomic write
              amb_gs[g] = 1;
            }
          }
          if (tau < TAU_STOP) {
            if (!near_stop) break;
            stopped = 1;
          }
        }
      }
  }
}

void orc_draw_stats(int H, int W, int N, const int32_t *ranges, const int32_t *gsid, const float *us,
                    const float *cinv2ds, const float *alphas, double *weight_sum, double *weight_max,
                    int64_t *hit_count, uint8_t *amb_gs, double margin) {
  memset(weight_sum, 0, sizeof(double) * N);
  memset(weight_max, 0, sizeof(double) * N);
  memset(hit_count, 0, sizeof(int64_t) * N);
  if (amb_gs) memset(amb_gs, 0, (size_t)N);
  for (int pass = 0; pass < 2; pass++)
    draw_stats_pass(pass, H, W, ranges, gsid, us, cinv2ds, alphas, weight_sum, weight_max, hit_count, amb_gs, margin);
}
