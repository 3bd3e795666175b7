// imgmetricssim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The thread bodies of the image-metric kernels (lidar4d_b200/csrc/l4d_imgmetrics.cuh) compiled for the CPU and driven
// serially, as k_im_columns / k_im_rows / k_im_ssim drive them on the device, for tests/test_image_metrics_hostsim.py.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_imgmetrics.cuh"

// pred, gt [H, W] -> clamped cp, cg, absd [H, W], the five filtered maps maps[5][H, W] (x, y, x*x, y*y, x*y: both axes),
// the per-column sums of squares sq[W] and gt's min / max gmin[W], gmax[W]
extern "C" void ims_maps(const float* pred, const float* gt, int H, int W, float lo, float hi, float* cp, float* cg,
                         float* absd, float* maps, double* sq, float* gmin, float* gmax) {
  const size_t hw = (size_t)H * W;
  float* m0 = (float*)malloc(sizeof(float) * 5 * hw);
  for (int j = 0; j < W; ++j) l4d_im_column(pred, gt, H, W, j, lo, hi, cp, cg, absd, m0, sq + j, gmin + j, gmax + j);
  for (int t = 0; t < 5 * H; ++t) {
    const size_t off = (size_t)(t % 5) * hw + (size_t)(t / 5) * W;
    l4d_im_line(m0 + off, W, maps + off);
  }
  free(m0);
}

// one line of uniform_filter1d(., 7, mode='reflect')
extern "C" void ims_line(const float* in, int n, float* out) { l4d_im_line(in, n, out); }

// (C1, C2) from gt's min and max, and the S map of five filtered maps [5][n] given C1, C2
extern "C" void ims_consts(float gmin, float gmax, float* c) { l4d_im_consts(gmin, gmax, c, c + 1); }

extern "C" void ims_smap(const float* maps, size_t n, float C1, float C2, float* S) {
  for (size_t k = 0; k < n; ++k)
    S[k] = l4d_im_ssim(maps[k], maps[n + k], maps[2 * n + k], maps[3 * n + k], maps[4 * n + k], C1, C2);
}
