// mainlosssim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The per-element, cosine and fold math of the main LiDAR loss (lidar4d_b200/csrc/l4d_losses.cuh) compiled for the CPU
// and driven serially in the order k_main_loss / k_main_finish / k_main_eval drive it, for
// tests/test_main_loss_hostsim.py.  The chamfer search itself is not here: the test runs the chamfer oracle on the
// clouds this writes and hands its gradient back to ms_fold.
#include <math.h>
#include <stdint.h>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_losses.cuh"

// k_main_loss: the criteria's sum (double), d loss / d (pred_d, image) and, if rays_d != nullptr, the two clouds
extern "C" void ms_train(const float* depth, const float* image, const float* gt, const float* rays_d, uint32_t n,
                         const uint32_t* crit, const float* alpha, double smooth, float scale, float delta, double* crit_sum,
                         float* g_pd, float* g_image, float* pred, float* gtc) {
  const L4DMainArgs A = l4d_main_args(n, crit, alpha, smooth, scale, delta);
  L4DCos cs[L4D_MT_N];
  float cosv[L4D_MT_N] = {0.f, 0.f, 0.f};
  for (int k = 0; k < L4D_MT_N; ++k) cs[k] = l4d_cos_norms(0.0, 0.0);
  if (A.any_cos) {
    double v[6] = {0, 0, 0, 0, 0, 0}, c[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t r = 0; r < n; ++r) {
      const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
      for (int k = 0; k < L4D_MT_N; ++k) { v[2 * k] += (double)e.a[k] * e.a[k]; v[2 * k + 1] += (double)e.b[k] * e.b[k]; }
    }
    for (int k = 0; k < L4D_MT_N; ++k) cs[k] = l4d_cos_norms(v[2 * k], v[2 * k + 1]);
    for (uint32_t r = 0; r < n; ++r) {
      const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
      for (int k = 0; k < L4D_MT_N; ++k) {
        c[2 * k] += (double)l4d_cos_term(e.a[k], e.b[k], cs[k]);
        c[2 * k + 1] += l4d_cos_dot_term(e.a[k], e.b[k], cs[k]);
      }
    }
    for (int k = 0; k < L4D_MT_N; ++k) { cosv[k] = (float)c[2 * k]; cs[k].dot = (float)c[2 * k + 1]; }
  }
  double s = 0;
  for (uint32_t r = 0; r < n; ++r) {
    const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
    float da[L4D_MT_N];
    const float v = l4d_main_value(e, A, cosv, da);
    if (!A.all_cos || r == 0) s += v;
    l4d_main_grad(e, A, da, cs, &g_pd[r], &g_image[2 * r], &g_image[2 * r + 1]);
    if (rays_d)
      for (int c = 0; c < 3; ++c) {
        pred[3 * r + c] = l4d_main_point(rays_d[3 * r + c], e.a[L4D_MT_D], A);
        gtc[3 * r + c] = l4d_main_point(rays_d[3 * r + c], e.b[L4D_MT_D], A);
      }
  }
  *crit_sum = s;
}

// k_main_finish: the loss, and d loss / d depth = (g_pd + fold of the chamfer gradient gx1) * m (gx1 == nullptr: no
// chamfer term, g_pd * m)
extern "C" float ms_finish(const float* gt, const float* rays_d, uint32_t n, float scale, double crit_sum, const float* d1,
                           const float* d2, const float* gx1, const float* g_pd, float* g_depth) {
  const uint32_t crit[L4D_MT_N] = {0, 0, 0};
  const float alpha[L4D_MT_N] = {0, 0, 0};
  const L4DMainArgs A = l4d_main_args(n, crit, alpha, 0.0, scale, 0.f);
  double s = 0;
  for (uint32_t r = 0; r < n; ++r) {
    if (gx1) {
      s += (double)(d1[r] + d2[r]);
      g_depth[r] = (g_pd[r] + l4d_main_fold(gx1 + 3 * r, rays_d + 3 * r, A)) * gt[3 * r];
    } else {
      g_depth[r] = g_pd[r] * gt[3 * r];
    }
  }
  return l4d_main_total(crit_sum, s, n, gx1 != nullptr);
}

// k_main_eval with a float32 ray-drop prediction (nullptr: image_0 or its sigmoid)
extern "C" float ms_eval(const float* depth, const float* image, const float* gt, const float* raydrop, uint32_t B, uint32_t H,
                         uint32_t W, const uint32_t* crit, const float* alpha, float delta) {
  const size_t n = (size_t)B * H * W;
  const L4DMainArgs A = l4d_main_args((uint32_t)n, crit, alpha, 0.0, 0.f, delta);
  auto pred_r = [&](size_t i) {
    if (raydrop) return raydrop[i];
    return A.crit[L4D_MT_R] == L4D_GRAD_BCE ? l4d_logistic(image[2 * i]) : image[2 * i];
  };
  double v[L4D_MT_N] = {0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, i, pred_r(i));
    for (int k = 0; k < L4D_MT_N; ++k) {
      float da;
      if (A.crit[k] != L4D_GRAD_COS) v[k] += l4d_grad_crit(A.crit[k], e.a[k], e.b[k], A.delta, &da);
    }
  }
  for (uint32_t col = 0; col < B * W; ++col) {
    const size_t base = (size_t)(col / W) * H * W + col % W;
    double sq[6] = {0, 0, 0, 0, 0, 0}, c[L4D_MT_N] = {0, 0, 0};
    for (uint32_t h = 0; h < H; ++h) {
      const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, base + (size_t)h * W, pred_r(base + (size_t)h * W));
      for (int k = 0; k < L4D_MT_N; ++k) { sq[2 * k] += (double)e.a[k] * e.a[k]; sq[2 * k + 1] += (double)e.b[k] * e.b[k]; }
    }
    L4DCos cs[L4D_MT_N];
    for (int k = 0; k < L4D_MT_N; ++k) cs[k] = l4d_cos_norms(sq[2 * k], sq[2 * k + 1]);
    for (uint32_t h = 0; h < H; ++h) {
      const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, base + (size_t)h * W, pred_r(base + (size_t)h * W));
      for (int k = 0; k < L4D_MT_N; ++k) c[k] += (double)l4d_cos_term(e.a[k], e.b[k], cs[k]);
    }
    for (int k = 0; k < L4D_MT_N; ++k)
      if (A.crit[k] == L4D_GRAD_COS) v[k] += (double)(float)c[k];
  }
  double cnt[L4D_MT_N];
  for (int k = 0; k < L4D_MT_N; ++k) cnt[k] = A.crit[k] == L4D_GRAD_COS ? (double)B * W : (double)n;
  return l4d_main_eval_total(v, cnt, A);
}
