// refinesim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The element math of the ray-drop refinement ops (lidar4d_b200/csrc/l4d_refine.cuh) compiled for the CPU, for
// tests/test_refine_hostsim.py: the box mask of k_box_mask and the BCE element and gradient of k_bce / k_bce_bwd.
#include <stdint.h>
#include <stdlib.h>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_refine.cuh"

// k_box_mask's rule over x[planes, H, W]; boxes[n, 4] = (y0, x0, h, w)
extern "C" void rfs_box_mask(const float* x, float* out, uint32_t planes, uint32_t H, uint32_t W, const int32_t* boxes,
                             uint32_t n) {
  L4DBoxes b;
  b.n = n;
  for (uint32_t k = 0; k < n; ++k) {
    b.y0[k] = boxes[4 * k]; b.x0[k] = boxes[4 * k + 1]; b.h[k] = boxes[4 * k + 2]; b.w[k] = boxes[4 * k + 3];
  }
  for (uint32_t c = 0; c < planes; ++c)
    for (uint32_t y = 0; y < H; ++y)
      for (uint32_t xx = 0; xx < W; ++xx) {
        const size_t i = ((size_t)c * H + y) * W + xx;
        out[i] = l4d_box_apply(x[i], l4d_box_value(b, (int32_t)y, (int32_t)xx));
      }
}

// per-element BCE (reduction='none') and its mean-reduction gradient for the incoming gradient g
extern "C" void rfs_bce(const float* x, const float* t, size_t n, float* loss) {
  for (size_t i = 0; i < n; ++i) loss[i] = l4d_bce_elem(x[i], t[i]);
}
extern "C" void rfs_bce_grad(const float* x, const float* t, size_t n, float g, float* grad) {
  for (size_t i = 0; i < n; ++i) grad[i] = l4d_bce_grad(x[i], t[i], g, (float)n);
}
