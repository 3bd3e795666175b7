// losssim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The per-patch and per-sample math of the train-step losses (lidar4d_b200/csrc/l4d_losses.cuh) compiled for the CPU and
// driven serially, as k_patch_loss and k_los_partial / k_los_finalize / k_los_backward drive it on the device, for
// tests/test_losses_hostsim.py.
#include <math.h>
#include <stdint.h>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_losses.cuh"

extern "C" void ls_patch(const float* depth, const float* gt, uint32_t n, uint32_t px, uint32_t py, float scale, uint32_t crit,
                         uint32_t flags, float a_grad, float a_gn, float a_sp, float a_tv, float* loss, float* g) {
  const L4DPatchArgs a = l4d_patch_args(n, px, py, scale, crit, flags, a_grad, a_gn, a_sp, a_tv);
  double s[L4D_PS_N] = {0, 0, 0, 0, 0, 0, 0};
  if (px <= 1) {
    for (uint32_t i = 0; i < n; ++i) g[i] = 0.f;
    *loss = 0.f;
    return;
  }
  for (uint32_t p = 0; p < n / (px * py); ++p) l4d_patch_eval(depth, gt, a, p, s, g);
  *loss = l4d_patch_value(s, a);
}

// loss and d loss / d w for an incoming gradient g_in
extern "C" void ls_los(const float* w, const float* z, const float* gt, uint32_t n, uint32_t S, double eps, float g_in,
                       float* loss, float* g_w) {
  const L4DLosArgs a = l4d_los_args(eps);
  double se = 0, sn = 0;
  float mn = INFINITY;
  uint32_t cnt = 0;
  for (uint32_t r = 0; r < n; ++r) {
    const float gd = gt[3 * r + 2] * gt[3 * r];
    cnt += gd > 0.f;
    for (uint32_t k = 0; k < S; ++k) {
      const L4DLosSample s = l4d_los_sample(z[(size_t)r * S + k], gd, a);
      float e2, n2;
      l4d_los_terms(w[(size_t)r * S + k], s, a.peak, &e2, &n2);
      se += e2; sn += n2;
      mn = fminf(mn, s.d2);
    }
  }
  const float maxv = l4d_los_max(mn, a);
  if (maxv != a.peak) {
    sn = 0;
    for (size_t i = 0; i < (size_t)n * S; ++i) {
      const L4DLosSample s = l4d_los_sample(z[i], gt[3 * (i / S) + 2] * gt[3 * (i / S)], a);
      float e2, n2;
      l4d_los_terms(w[i], s, maxv, &e2, &n2);
      sn += n2;
    }
  }
  *loss = l4d_los_value(se, sn, (float)cnt);
  const float gs = (g_in * 0.1f) / (float)cnt;
  for (size_t i = 0; i < (size_t)n * S; ++i) {
    const L4DLosSample s = l4d_los_sample(z[i], gt[3 * (i / S) + 2] * gt[3 * (i / S)], a);
    g_w[i] = l4d_los_grad(w[i], s, maxv, gs);
  }
}
