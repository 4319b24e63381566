// TEST-ONLY host build of the binning's rectangle arithmetic (easygaussiansplatting_b200/csrc/rect_math.h
// tile_rect), as k_rects_scan (batch = 0) and k_rects_scan_batch (batch = 1) call it for record i of
// n_total: frame i / nc's rows in the tall frame.  Never part of the product library.
#include <stdint.h>

#include "../../easygaussiansplatting_b200/csrc/rect_math.h"

extern "C" void tile_rects(int n_total, int nc, int batch, const float *us, const int32_t *areas, int gx, int gy,
                           int32_t *out) {
  for (int i = 0; i < n_total; i++) {
    int x0, x1, y0, y1;
    gsb::tile_rect(us[2 * i], us[2 * i + 1], (float)areas[2 * i], (float)areas[2 * i + 1], gx, gy,
                   batch ? (i / nc) * gy : 0, x0, x1, y0, y1);
    out[4 * i] = x0; out[4 * i + 1] = x1; out[4 * i + 2] = y0; out[4 * i + 3] = y1;
  }
}
