// l4d_losses.cuh - the rest of the reference's train_step after the flow loss, value and gradient in CUDA:
//   k_patch_loss      model/runner.py:278-369: the depth-gradient loss of patch batches (finite differences or Sobel,
//                     criteria l1 / mse / huber / bce / cos) and the grad_norm_smooth / spatial_smooth / tv_loss terms
//   k_los_partial     model/runner.py:255-276: URF's line-of-sight loss over weights / z_vals [n, S]
//   k_los_finalize      (+ its fixed-order reduction, and the degenerate case of the global distr maximum)
//   k_los_backward    d loss / d weights
//   k_loss_scale      d loss / d depth of the patch loss times the incoming gradient, read from device memory
//   k_main_loss       model/runner.py:193-220: the main LiDAR loss (criteria l1 / mse / huber / bce / cos for depth, ray
//                     drop and intensity) with d loss / d (depth, image), and the chamfer term's two point clouds
//   k_main_finish       (+ the chamfer term's mean, its gradient folded into d loss / d depth)
//   k_main_scale      both saved gradients times the incoming gradient, read from device memory
//   k_main_eval       model/runner.py:409-421: eval_step's loss (means, ray-drop mask taken from the prediction)
// The per-element and per-patch math is in __host__ __device__ functions, so tests/hostsim/losssim.cu runs it on the CPU.
// Sums are accumulated in double in a fixed order: the same inputs give the same bits.
#pragma once
#include <math.h>
#include <stdint.h>

// ------------------------------------------------------------------------------------------------------------------
// patch loss
// ------------------------------------------------------------------------------------------------------------------
struct L4DPatchArgs {
  uint32_t px, py;          // patch rows (the y direction) x columns (the x direction), get_lidar_rays' order
  uint32_t crit, flags;     // L4D_GRAD_* criterion, L4D_PATCH_* flags
  float inv_scale;          // 1 / opt.scale: `tensor / scale` as ATen evaluates it, times the fp32 reciprocal
  float delta;              // huber delta = 0.2 * scale
  float a_grad, a_gn, a_sp, a_tv;
  double nx, ny;            // element counts of dx and dy over all patches (the smoothness means' denominators)
};

inline L4DPatchArgs l4d_patch_args(uint32_t n, uint32_t px, uint32_t py, float scale, uint32_t crit, uint32_t flags,
                                   float a_grad, float a_gn, float a_sp, float a_tv) {
  L4DPatchArgs a;
  a.px = px; a.py = py; a.crit = crit; a.flags = flags;
  a.inv_scale = 1.0f / scale;
  a.delta = (float)(0.2 * (double)scale);
  a.a_grad = a_grad; a.a_gn = a_gn; a.a_sp = a_sp; a.a_tv = a_tv;
  const double np = px * py ? (double)(n / (px * py)) : 0.0;
  const bool sobel = flags & L4D_PATCH_SOBEL;
  a.nx = np * px * (sobel ? py : py - 1.0);
  a.ny = np * (sobel ? px : px - 1.0) * py;
  return a;
}

// sums[]: the grad criterion summed, then sum exp(-d), sum d^2, sum d, each for dx and dy
enum { L4D_PS_GRAD = 0, L4D_PS_EXP_X, L4D_PS_EXP_Y, L4D_PS_SQ_X, L4D_PS_SQ_Y, L4D_PS_ABS_X, L4D_PS_ABS_Y, L4D_PS_N };

__host__ __device__ inline float l4d_sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// one element of a torch criterion with reduction='none' (main_lidar4d.py:183-188) and its derivative in `a`
__host__ __device__ inline float l4d_grad_crit(uint32_t crit, float a, float b, float delta, float* da) {
  const float x = a - b;
  switch (crit) {
    case L4D_GRAD_MSE: *da = 2.f * x; return x * x;
    case L4D_GRAD_HUBER: {
      const float z = fabsf(x);
      *da = x < -delta ? -delta : (x > delta ? delta : x);
      return z < delta ? 0.5f * z * z : delta * (z - 0.5f * delta);
    }
    case L4D_GRAD_BCE: {     // BCEWithLogits: (1 - t) a - log_sigmoid(a); d/da = sigmoid(a) - t
      const float ls = fminf(a, 0.f) - log1pf(expf(-fabsf(a)));
      *da = 1.f / (1.f + expf(-a)) - b;
      return (1.f - b) * a - ls;
    }
    default: *da = l4d_sgn(x); return fabsf(x);   // l1 (cos is per patch, see l4d_patch_eval)
  }
}

// ATen's cosine_similarity over one vector, in the order ATen evaluates it: each side divided by max(|v|, eps), then
// the dot product.  Squared norms and sums are accumulated in double by the caller; these are the per-element pieces.
struct L4DCos {
  float na, nb;             // max(|a|, 1e-8), max(|b|, 1e-8)
  float norm_a;             // |a|
  float dot;                // sum a * (b / nb), for the gradient
};

__host__ __device__ inline L4DCos l4d_cos_norms(double sa2, double sb2) {
  L4DCos c;
  c.norm_a = sqrtf((float)sa2);
  c.na = fmaxf(c.norm_a, 1e-8f);
  c.nb = fmaxf(sqrtf((float)sb2), 1e-8f);
  c.dot = 0.f;
  return c;
}
// one term of the cosine (summed: the cosine) and of the gradient's dot product (summed: L4DCos::dot)
__host__ __device__ inline float l4d_cos_term(float a, float b, const L4DCos& c) { return (a / c.na) * (b / c.nb); }
__host__ __device__ inline double l4d_cos_dot_term(float a, float b, const L4DCos& c) { return (double)a * (b / c.nb); }
// d cos / d a for one element (the clamp of |a| at eps has no gradient)
__host__ __device__ inline float l4d_cos_grad(float a, float b, const L4DCos& c) {
  float d = b / c.nb / c.na;
  if (c.norm_a >= 1e-8f) d -= a / c.norm_a * c.dot / (c.na * c.na);
  return d;
}

// patch p: adds its terms to sums[] and, if g != nullptr, writes d(branch loss)/d depth for its px*py rays
__host__ __device__ inline void l4d_patch_eval(const float* __restrict__ depth, const float* __restrict__ gt,
                                               const L4DPatchArgs& a, uint32_t p, double* sums, float* __restrict__ g) {
  const int px = (int)a.px, py = (int)a.py;
  const size_t base = (size_t)p * a.px * a.py;
  const bool sobel = a.flags & L4D_PATCH_SOBEL, want_grad = a.flags & L4D_PATCH_GRAD;
  const bool smooth = a.flags & (L4D_PATCH_GRAD_NORM | L4D_PATCH_SPATIAL | L4D_PATCH_TV);
  const bool use_cos = a.crit == L4D_GRAD_COS;
  // pred = depth * m / scale and gt_d = gt_depth * m / scale; zero outside the patch (conv2d's padding=1)
  auto in = [&](int i, int j) { return i >= 0 && j >= 0 && i < px && j < py; };
  auto P = [&](int i, int j) {
    if (!in(i, j)) return 0.f;
    const size_t k = base + (size_t)i * py + j;
    return depth[k] * gt[3 * k] * a.inv_scale;
  };
  auto G = [&](int i, int j) {
    if (!in(i, j)) return 0.f;
    const size_t k = base + (size_t)i * py + j;
    return gt[3 * k + 2] * gt[3 * k] * a.inv_scale;
  };
  auto M = [&](int i, int j) { return gt[3 * (base + (size_t)i * py + j)]; };
  // x difference at (i, j): Sobel_x (signed) or |P(i,j) - P(i,j+1)|; `s` = d value / d P(i,j) for the finite difference
  auto dxv = [&](auto F, int i, int j, bool absval, float* s) {
    if (sobel) return ((F(i - 1, j + 1) - F(i - 1, j - 1)) + 2.f * (F(i, j + 1) - F(i, j - 1))) + (F(i + 1, j + 1) - F(i + 1, j - 1));
    const float d = F(i, j) - F(i, j + 1);
    if (s) *s = l4d_sgn(d);
    return absval ? fabsf(d) : d;
  };
  auto dyv = [&](auto F, int i, int j, float* s) {
    if (sobel) return ((F(i + 1, j - 1) + 2.f * F(i + 1, j)) + F(i + 1, j + 1)) - ((F(i - 1, j - 1) + 2.f * F(i - 1, j)) + F(i - 1, j + 1));
    const float d = F(i, j) - F(i + 1, j);
    if (s) *s = l4d_sgn(d);
    return fabsf(d);
  };
  const int xr = px, xc = sobel ? py : py - 1;            // x-difference grid
  const int yr = sobel ? px : px - 1, yc = py;            // y-difference grid
  if (g)
    for (int k = 0; k < px * py; ++k) g[base + k] = 0.f;
  // dv = d loss / d (difference value): scatter it onto the patch through the stencil
  auto scatter_x = [&](int i, int j, float dv, float s) {
    if (!sobel) { g[base + (size_t)i * py + j] += dv * s; g[base + (size_t)i * py + j + 1] -= dv * s; return; }
    for (int r = -1; r <= 1; ++r) {
      const float w = r == 0 ? 2.f : 1.f;
      if (in(i + r, j + 1)) g[base + (size_t)(i + r) * py + j + 1] += w * dv;
      if (in(i + r, j - 1)) g[base + (size_t)(i + r) * py + j - 1] -= w * dv;
    }
  };
  auto scatter_y = [&](int i, int j, float dv, float s) {
    if (!sobel) { g[base + (size_t)i * py + j] += dv * s; g[base + (size_t)(i + 1) * py + j] -= dv * s; return; }
    for (int c = -1; c <= 1; ++c) {
      const float w = c == 0 ? 2.f : 1.f;
      if (in(i + 1, j + c)) g[base + (size_t)(i + 1) * py + j + c] += w * dv;
      if (in(i - 1, j + c)) g[base + (size_t)(i - 1) * py + j + c] -= w * dv;
    }
  };
  // the smoothness terms of one |difference| d and their derivative in d
  auto smooth_term = [&](float d, double n, double* se, double* ss, double* sa) {
    float dd = 0.f;
    if (a.flags & L4D_PATCH_GRAD_NORM) { const float e = expf(-d); *se += e; dd += -a.a_gn * e / (float)n; }
    if (a.flags & L4D_PATCH_SPATIAL) { *ss += (double)d * d; dd += a.a_sp * 2.f * d / (float)n; }
    if (a.flags & L4D_PATCH_TV) { *sa += d; dd += a.a_tv / (float)n; }
    return dd;
  };
  // cosine similarity per patch
  L4DCos cs = l4d_cos_norms(0.0, 0.0);
  if (want_grad && use_cos) {
    double sa2 = 0, sb2 = 0;
    for (int i = 0; i < xr; ++i)
      for (int j = 0; j < xc; ++j) {
        const float gv = dxv(G, i, j, false, nullptr);
        const float mk = M(i, j) * (fabsf(gv) < 0.01f ? 1.f : 0.f);
        const float av = dxv(P, i, j, true, nullptr) * mk, bv = gv * mk;
        sa2 += (double)av * av; sb2 += (double)bv * bv;
      }
    cs = l4d_cos_norms(sa2, sb2);
    double c = 0, d = 0;
    for (int i = 0; i < xr; ++i)
      for (int j = 0; j < xc; ++j) {
        const float gv = dxv(G, i, j, false, nullptr);
        const float mk = M(i, j) * (fabsf(gv) < 0.01f ? 1.f : 0.f);
        const float av = dxv(P, i, j, true, nullptr) * mk, bv = gv * mk;
        c += (double)l4d_cos_term(av, bv, cs);
        d += l4d_cos_dot_term(av, bv, cs);
      }
    cs.dot = (float)d;
    sums[L4D_PS_GRAD] += 1.0 - (double)(float)c;
  }
  if (want_grad || smooth)
    for (int i = 0; i < xr; ++i)
      for (int j = 0; j < xc; ++j) {
        float s = 0.f;
        const float v = dxv(P, i, j, true, &s);
        float dv = 0.f;
        if (smooth) dv = l4d_sgn(v) * smooth_term(fabsf(v), a.nx, &sums[L4D_PS_EXP_X], &sums[L4D_PS_SQ_X], &sums[L4D_PS_ABS_X]);
        if (want_grad) {
          const float gv = dxv(G, i, j, false, nullptr);
          const float mk = M(i, j) * (fabsf(gv) < 0.01f ? 1.f : 0.f);
          float da;
          if (use_cos) {
            da = -l4d_cos_grad(v * mk, gv * mk, cs);
          } else {
            sums[L4D_PS_GRAD] += l4d_grad_crit(a.crit, v * mk, gv * mk, a.delta, &da);
          }
          dv += a.a_grad * da * mk;
        }
        if (g) scatter_x(i, j, dv, s);
      }
  if (smooth)
    for (int i = 0; i < yr; ++i)
      for (int j = 0; j < yc; ++j) {
        float s = 0.f;
        const float v = dyv(P, i, j, &s);
        const float dv = l4d_sgn(v) * smooth_term(fabsf(v), a.ny, &sums[L4D_PS_EXP_Y], &sums[L4D_PS_SQ_Y], &sums[L4D_PS_ABS_Y]);
        if (g) scatter_y(i, j, dv, s);
      }
  if (g)
    for (int k = 0; k < px * py; ++k) g[base + k] *= a.inv_scale * gt[3 * (base + k)];
}

// the branch's loss from the summed terms, added in the reference's order (grad_norm, spatial, tv, grad)
__host__ __device__ inline float l4d_patch_value(const double* s, const L4DPatchArgs& a) {
  float loss = 0.f;
  if (a.flags & L4D_PATCH_GRAD_NORM) loss += a.a_gn * ((float)(s[L4D_PS_EXP_X] / a.nx) + (float)(s[L4D_PS_EXP_Y] / a.ny));
  if (a.flags & L4D_PATCH_SPATIAL) loss += a.a_sp * ((float)(s[L4D_PS_SQ_X] / a.nx) + (float)(s[L4D_PS_SQ_Y] / a.ny));
  if (a.flags & L4D_PATCH_TV) loss += a.a_tv * ((float)(s[L4D_PS_ABS_X] / a.nx) + (float)(s[L4D_PS_ABS_Y] / a.ny));
  if (a.flags & L4D_PATCH_GRAD) loss += a.a_grad * (float)s[L4D_PS_GRAD];
  return loss;
}

// ------------------------------------------------------------------------------------------------------------------
// line-of-sight loss
// ------------------------------------------------------------------------------------------------------------------
struct L4DLosArgs {
  float eps;                // (float) eps
  float peak;               // (float) 1 / (sigma sqrt(2 pi)), sigma = eps / 3 in double as the reference's Python floats
  float inv_2s2;            // 1 / (float)(2 sigma^2): ATen's `tensor / python_scalar`
};

struct L4DLosSample {
  float me, mn;             // mask_empty, mask_near as 0 / 1
  float d2;                 // (mask_near * (z - gt_d))^2
  float distr;              // peak * exp(-(d2 / (2 sigma^2))), before the division by its global maximum
};

// the reference's Python-double scalars, rounded to fp32 where its tensor ops take them
inline L4DLosArgs l4d_los_args(double eps) {
  const double sigma = eps / 3.;
  L4DLosArgs a;
  a.eps = (float)eps;
  a.peak = (float)(1.0 / (sigma * sqrt(2 * 3.14159265358979323846)));
  a.inv_2s2 = 1.0f / (float)(2 * (sigma * sigma));
  return a;
}

__host__ __device__ inline L4DLosSample l4d_los_sample(float z, float gd, const L4DLosArgs& a) {
  const float lo = gd - a.eps, hi = gd + a.eps;
  L4DLosSample s;
  s.me = (z < lo || z > hi) ? 1.f : 0.f;
  s.mn = (z > lo && z < hi) ? 1.f : 0.f;
  const float dist = s.mn * (z - gd);
  s.d2 = dist * dist;
  s.distr = a.peak * expf(-(s.d2 * a.inv_2s2));
  return s;
}

// the global maximum of distr: every fp32 step of peak * exp(-d2 / (2 sigma^2)) is monotone in d2, so it is f(min d2)
__host__ __device__ inline float l4d_los_max(float min_d2, const L4DLosArgs& a) {
  return a.peak * expf(-(min_d2 * a.inv_2s2));
}

// (mask_empty * w)^2 and (mask_near * w - distr / max * mask_near)^2
__host__ __device__ inline void l4d_los_terms(float w, const L4DLosSample& s, float maxv, float* e2, float* n2) {
  const float q = s.me * w, r = s.mn * w - (s.distr / maxv) * s.mn;
  *e2 = q * q;
  *n2 = r * r;
}

// d loss / d w with gs = 0.1 * g / count
__host__ __device__ inline float l4d_los_grad(float w, const L4DLosSample& s, float maxv, float gs) {
  const float q = s.me * w, r = s.mn * w - (s.distr / maxv) * s.mn;
  return gs * (2.f * q) * s.me + gs * (2.f * r) * s.mn;
}

__host__ __device__ inline float l4d_los_value(double se, double sn, float cnt) {
  return 0.1f * ((float)se / cnt) + 0.1f * ((float)sn / cnt);
}

// ------------------------------------------------------------------------------------------------------------------
// main LiDAR loss (train_step and eval_step)
// ------------------------------------------------------------------------------------------------------------------
enum { L4D_MT_D = 0, L4D_MT_R, L4D_MT_I, L4D_MT_N };      // the depth, ray-drop and intensity terms, in the sum's order

struct L4DMainArgs {
  uint32_t crit[L4D_MT_N];  // L4D_GRAD_* of each term
  float alpha[L4D_MT_N];    // alpha_d, alpha_r, alpha_i
  float lo, hi;             // train: the label smoothing clamp(m, s, 1 - s) as ATen takes its Python bounds, (float) each
  float delta;              // huber delta: (float)(0.2 * opt.scale), the product in double
  float inv_scale;          // 1 / (float) opt.scale: `tensor / scale` as ATen evaluates it on CUDA (see L4DPatchArgs)
  float kcos;               // train: times each cos term counts in the sum, n (broadcast over the elementwise terms) or 1
  uint32_t any_cos;         // some term is cos
  uint32_t all_cos;         // every term is cos: lidar_loss is [1], not [1, n], and its sum counts one element
};

inline L4DMainArgs l4d_main_args(uint32_t n, const uint32_t* crit, const float* alpha, double smooth, float scale,
                                 float delta) {
  L4DMainArgs a;
  uint32_t ncos = 0;
  for (int k = 0; k < L4D_MT_N; ++k) {
    a.crit[k] = crit[k];
    a.alpha[k] = alpha[k];
    ncos += crit[k] == L4D_GRAD_COS;
  }
  a.lo = (float)smooth;
  a.hi = (float)(1.0 - smooth);
  a.delta = delta;
  a.inv_scale = scale != 0.f ? 1.0f / scale : 0.f;
  a.kcos = ncos == L4D_MT_N ? 1.f : (float)n;
  a.any_cos = ncos != 0;
  a.all_cos = ncos == L4D_MT_N;
  return a;
}

// a * b and a + b rounded on their own: the reference evaluates each of them as a separate tensor op
__host__ __device__ inline float l4d_mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float l4d_add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// torch.sigmoid's element (ATen: 1 / (1 + exp(-x))); the same expression as l4d_core.cuh's, which host builds do not include
__host__ __device__ inline float l4d_logistic(float x) { return 1.f / (1.f + expf(-x)); }

// one ray's three (prediction, target) pairs
struct L4DMainElem {
  float a[L4D_MT_N], b[L4D_MT_N];
  float m;                  // the ground-truth ray-drop mask
};

// train_step (runner.py:193-213): pred_d = depth m, pred_r = image_0 (its sigmoid for bce), pred_i = image_1 m against
// gt_d = gt_2 m, clamp(m, s, 1 - s), gt_i = gt_1 m
__host__ __device__ inline L4DMainElem l4d_main_train_elem(const float* depth, const float* image, const float* gt, size_t r,
                                                           const L4DMainArgs& A) {
  L4DMainElem e;
  e.m = gt[3 * r];
  e.a[L4D_MT_D] = l4d_mul_rn(depth[r], e.m);
  e.b[L4D_MT_D] = l4d_mul_rn(gt[3 * r + 2], e.m);
  const float x = image[2 * r];
  e.a[L4D_MT_R] = A.crit[L4D_MT_R] == L4D_GRAD_BCE ? l4d_logistic(x) : x;
  e.b[L4D_MT_R] = fminf(fmaxf(e.m, A.lo), A.hi);
  e.a[L4D_MT_I] = l4d_mul_rn(image[2 * r + 1], e.m);
  e.b[L4D_MT_I] = l4d_mul_rn(gt[3 * r + 1], e.m);
  return e;
}

// eval_step (runner.py:409-421): mask = pred_r > 0.5 (0 for NaN), depth * mask, pred_r, intensity * mask against gt_d,
// m (no smoothing), gt_i; pred_r is the ray-drop prediction as the caller took it (sigmoid or U-Net output)
__host__ __device__ inline L4DMainElem l4d_main_eval_elem(const float* depth, const float* image, const float* gt, size_t r,
                                                          float pred_r) {
  L4DMainElem e;
  e.m = gt[3 * r];
  const float mask = pred_r > 0.5f ? 1.f : 0.f;
  e.a[L4D_MT_D] = l4d_mul_rn(depth[r], mask);
  e.b[L4D_MT_D] = l4d_mul_rn(gt[3 * r + 2], e.m);
  e.a[L4D_MT_R] = pred_r;
  e.b[L4D_MT_R] = e.m;
  e.a[L4D_MT_I] = l4d_mul_rn(image[2 * r + 1], mask);
  e.b[L4D_MT_I] = l4d_mul_rn(gt[3 * r + 1], e.m);
  return e;
}

// train: the ray's element of lidar_loss, (a_d C_d + a_r C_r) + a_i C_i, with each cos term's value cosv[k] broadcast;
// da[k] = d C_k / d a_k of the elementwise terms
__host__ __device__ inline float l4d_main_value(const L4DMainElem& e, const L4DMainArgs& A, const float* cosv, float* da) {
  float t[L4D_MT_N];
  for (int k = 0; k < L4D_MT_N; ++k) {
    da[k] = 0.f;
    t[k] = A.crit[k] == L4D_GRAD_COS ? cosv[k] : l4d_grad_crit(A.crit[k], e.a[k], e.b[k], A.delta, &da[k]);
  }
  return l4d_add_rn(l4d_add_rn(l4d_mul_rn(A.alpha[0], t[0]), l4d_mul_rn(A.alpha[1], t[1])), l4d_mul_rn(A.alpha[2], t[2]));
}

// train: d loss / d (pred_d, image_0, image_1) of the criteria for a unit upstream gradient (pred_d before its `* m`)
__host__ __device__ inline void l4d_main_grad(const L4DMainElem& e, const L4DMainArgs& A, const float* da, const L4DCos* cs,
                                              float* g_pd, float* g_r, float* g_i) {
  float g[L4D_MT_N];
  for (int k = 0; k < L4D_MT_N; ++k)
    g[k] = A.crit[k] == L4D_GRAD_COS ? A.alpha[k] * (A.kcos * l4d_cos_grad(e.a[k], e.b[k], cs[k])) : A.alpha[k] * da[k];
  *g_pd = g[L4D_MT_D];
  // bce: the sigmoid taken before BCEWithLogits, ATen's sigmoid_backward g (1 - y) y
  *g_r = A.crit[L4D_MT_R] == L4D_GRAD_BCE ? (g[L4D_MT_R] * (1.f - e.a[L4D_MT_R])) * e.a[L4D_MT_R] : g[L4D_MT_R];
  *g_i = g[L4D_MT_I] * e.m;
}

// the chamfer term's points: rays_d * pred_depth.unsqueeze(-1) / scale, each product rounded as ATen rounds it
__host__ __device__ inline float l4d_main_point(float rd, float d, const L4DMainArgs& A) {
  return l4d_mul_rn(l4d_mul_rn(rd, d), A.inv_scale);
}

// the chamfer gradient of one predicted point folded into d loss / d pred_d: sum_c (g_c / scale) rd_c
__host__ __device__ inline float l4d_main_fold(const float* gp, const float* rd, const L4DMainArgs& A) {
  return l4d_add_rn(l4d_add_rn(l4d_mul_rn(l4d_mul_rn(gp[0], A.inv_scale), rd[0]), l4d_mul_rn(l4d_mul_rn(gp[1], A.inv_scale), rd[1])),
                    l4d_mul_rn(l4d_mul_rn(gp[2], A.inv_scale), rd[2]));
}

// train: the loss from the criteria's double sum and the chamfer distances' double sum over n rays
__host__ __device__ inline float l4d_main_total(double crit_sum, double cham_sum, uint32_t n, bool chamfer) {
  const float l = (float)crit_sum;
  return chamfer ? l + (float)(cham_sum / n) * 0.5f : l;
}

// eval: a_d mean C_d + a_r mean C_r + a_i mean C_i from each term's double sum over `cnt[k]` elements (columns for cos)
__host__ __device__ inline float l4d_main_eval_total(const double* s, const double* cnt, const L4DMainArgs& A) {
  float m[L4D_MT_N];
  for (int k = 0; k < L4D_MT_N; ++k) m[k] = (float)(s[k] / cnt[k]);
  return l4d_add_rn(l4d_add_rn(l4d_mul_rn(A.alpha[0], m[0]), l4d_mul_rn(A.alpha[1], m[1])), l4d_mul_rn(A.alpha[2], m[2]));
}

// the train loss's work buffer (float offsets; used only with the chamfer term)
struct L4DMainLayout {
  size_t pred, gtc, d1, d2, i1, i2, gdist, gx1, gx2, keys, hdr, total;   // bytes
};
inline L4DMainLayout l4d_main_layout(uint32_t n) {
  L4DMainLayout L;
  const size_t f = (size_t)n * sizeof(float);
  L.pred = 0; L.gtc = 3 * f; L.d1 = 6 * f; L.d2 = 7 * f; L.i1 = 8 * f; L.i2 = 9 * f; L.gdist = 10 * f;
  L.gx1 = 12 * f; L.gx2 = 15 * f;
  L.keys = (18 * f + 15) & ~(size_t)15;
  L.hdr = L.keys + 2 * (size_t)n * sizeof(unsigned long long);
  L.total = L.hdr + 16;
  return L;
}

#ifdef __CUDACC__
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#define L4D_LOS_BLOCKS 1024     // fixed partial count: the summation order does not depend on the device
#define L4D_LOS_THREADS 256
#define L4D_PATCH_THREADS 512

struct L4DLosPartial {
  double se, sn;
  float min_d2;
  uint32_t cnt;
};
struct L4DLosWork {          // the work buffer: header (read by the backward), then one partial per CTA
  float cnt, maxv;
  uint32_t pad[2];
  L4DLosPartial part[L4D_LOS_BLOCKS];
};

template <int NT, int K>
__device__ inline void l4d_block_sum(double (&v)[K], double (*s)[NT / 32]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) s[k][warp] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k < K; ++k) {
      double t = 0;
      for (int w = 0; w < NT / 32; ++w) t += s[k][w];
      v[k] = t;
    }
}

// one CTA: thread t takes patches t, t + NT, ...; the patches of a thread and the tree are fixed, so is the sum
__global__ void __launch_bounds__(L4D_PATCH_THREADS) k_patch_loss(const float* __restrict__ depth, const float* __restrict__ gt,
                                                                  uint32_t n, L4DPatchArgs a, float* __restrict__ loss,
                                                                  float* __restrict__ g_depth) {
  __shared__ double s_red[L4D_PS_N][L4D_PATCH_THREADS / 32];
  double v[L4D_PS_N] = {0, 0, 0, 0, 0, 0, 0};
  if (a.px <= 1) {        // model/runner.py:286: no patch loss unless patch_size_x > 1
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) g_depth[i] = 0.f;
    if (threadIdx.x == 0) *loss = 0.f;
    return;
  }
  const uint32_t n_patch = n / (a.px * a.py);
  for (uint32_t p = threadIdx.x; p < n_patch; p += blockDim.x) l4d_patch_eval(depth, gt, a, p, v, g_depth);
  l4d_block_sum<L4D_PATCH_THREADS, L4D_PS_N>(v, s_red);
  if (threadIdx.x == 0) *loss = l4d_patch_value(v, a);
}

__global__ void __launch_bounds__(256) k_loss_scale(const float* __restrict__ g_saved, const float* __restrict__ g_loss,
                                                    uint32_t n, float* __restrict__ out) {
  const float g = *g_loss;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = g_saved[i] * g;
}

__global__ void __launch_bounds__(L4D_LOS_THREADS) k_los_partial(const float* __restrict__ w, const float* __restrict__ z,
                                                                 const float* __restrict__ gt, uint32_t n, uint32_t S,
                                                                 L4DLosArgs a, L4DLosWork* __restrict__ work) {
  __shared__ double s_red[2][L4D_LOS_THREADS / 32];
  __shared__ float s_min[L4D_LOS_THREADS / 32];
  __shared__ uint32_t s_cnt[L4D_LOS_THREADS / 32];
  double v[2] = {0, 0};
  float mn = INFINITY;
  uint32_t cnt = 0;
  const uint32_t total = n * S, stride = gridDim.x * blockDim.x;       // n * S < 2^32 (l4d_los_loss)
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const uint32_t r = i / S;
    const float gd = gt[3 * (size_t)r + 2] * gt[3 * (size_t)r];
    if (i - r * S == 0) cnt += gd > 0.f;
    const L4DLosSample s = l4d_los_sample(z[i], gd, a);
    float e2, n2;
    l4d_los_terms(w[i], s, a.peak, &e2, &n2);      // the normal case: some sample lies outside its window, max = peak
    v[0] += e2; v[1] += n2;
    mn = fminf(mn, s.d2);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) { s_min[warp] = mn; s_cnt[warp] = cnt; }
  l4d_block_sum<L4D_LOS_THREADS, 2>(v, s_red);
  if (threadIdx.x == 0) {
    for (int k = 1; k < L4D_LOS_THREADS / 32; ++k) { mn = fminf(mn, s_min[k]); cnt += s_cnt[k]; }
    work->part[blockIdx.x] = L4DLosPartial{v[0], v[1], mn, cnt};
  }
}

// one CTA: the partials in a fixed order; if no sample lies outside its window (max < peak), loss_near again with the
// true maximum over all n*S samples - slow, and never the case for a real ray's samples
__global__ void __launch_bounds__(1024) k_los_finalize(const float* __restrict__ w, const float* __restrict__ z,
                                                       const float* __restrict__ gt, uint32_t n, uint32_t S, uint32_t parts,
                                                       L4DLosArgs a, L4DLosWork* __restrict__ work, float* __restrict__ loss) {
  __shared__ double s_red[2][32];
  __shared__ float s_min[32], s_maxv;
  __shared__ uint32_t s_cnt[32];
  double v[2] = {0, 0};
  float mn = INFINITY;
  uint32_t cnt = 0;
  for (uint32_t b = threadIdx.x; b < parts; b += blockDim.x) {
    const L4DLosPartial p = work->part[b];
    v[0] += p.se; v[1] += p.sn; mn = fminf(mn, p.min_d2); cnt += p.cnt;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) { s_min[warp] = mn; s_cnt[warp] = cnt; }
  l4d_block_sum<1024, 2>(v, s_red);
  if (threadIdx.x == 0) {
    for (int k = 1; k < 32; ++k) { mn = fminf(mn, s_min[k]); cnt += s_cnt[k]; }
    s_maxv = l4d_los_max(mn, a);
    work->cnt = (float)cnt;
    work->maxv = s_maxv;
  }
  __syncthreads();
  const float maxv = s_maxv;
  if (maxv == a.peak) {
    if (threadIdx.x == 0) *loss = l4d_los_value(v[0], v[1], work->cnt);
    return;
  }
  double sn[1] = {0};
  const uint32_t total = n * S;
  for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
    const uint32_t r = i / S;
    const L4DLosSample s = l4d_los_sample(z[i], gt[3 * (size_t)r + 2] * gt[3 * (size_t)r], a);
    float e2, n2;
    l4d_los_terms(w[i], s, maxv, &e2, &n2);
    sn[0] += n2;
  }
  __syncthreads();
  l4d_block_sum<1024, 1>(sn, s_red);
  if (threadIdx.x == 0) *loss = l4d_los_value(v[0], sn[0], work->cnt);
}

__global__ void __launch_bounds__(256) k_los_backward(const float* __restrict__ w, const float* __restrict__ z,
                                                      const float* __restrict__ gt, uint32_t n, uint32_t S, L4DLosArgs a,
                                                      const L4DLosWork* __restrict__ work, const float* __restrict__ g_loss,
                                                      float* __restrict__ g_w) {
  const float maxv = work->maxv, gs = (*g_loss * 0.1f) / work->cnt;
  const uint32_t total = n * S, stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const uint32_t r = i / S;
    const L4DLosSample s = l4d_los_sample(z[i], gt[3 * (size_t)r + 2] * gt[3 * (size_t)r], a);
    g_w[i] = l4d_los_grad(w[i], s, maxv, gs);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// main LiDAR loss kernels: one CTA each for the reductions, so the sums have one fixed order for every n
// ------------------------------------------------------------------------------------------------------------------
#define L4D_MAIN_THREADS 1024

struct L4DMainPtrs {        // the chamfer term's buffers (l4d_main_layout), all null without it
  float *pred, *gtc, *d1, *d2, *gdist, *gx1, *gx2;
  double* crit_sum;
};

// cos terms first (squared norms, then the cosine and the gradient's dot product, ATen's order), then one pass that
// sums the elements, writes the criteria's gradient and, with the chamfer term, its point clouds and zeroed sinks.
// Without the chamfer term the loss is final here: written, or added to *loss when `accumulate`.
__global__ void __launch_bounds__(L4D_MAIN_THREADS) k_main_loss(const float* __restrict__ depth, const float* __restrict__ image,
                                                                const float* __restrict__ gt, const float* __restrict__ rays_d,
                                                                uint32_t n, L4DMainArgs A, L4DMainPtrs P, uint32_t accumulate,
                                                                float* __restrict__ loss, float* __restrict__ g_depth,
                                                                float* __restrict__ g_image) {
  __shared__ double s_red[6][L4D_MAIN_THREADS / 32];
  __shared__ L4DCos s_cos[L4D_MT_N];
  __shared__ float s_cosv[L4D_MT_N];
  if (A.any_cos) {
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
      const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
      for (int k = 0; k < L4D_MT_N; ++k)
        if (A.crit[k] == L4D_GRAD_COS) { v[2 * k] += (double)e.a[k] * e.a[k]; v[2 * k + 1] += (double)e.b[k] * e.b[k]; }
    }
    l4d_block_sum<L4D_MAIN_THREADS, 6>(v, s_red);
    if (threadIdx.x == 0)
      for (int k = 0; k < L4D_MT_N; ++k) s_cos[k] = l4d_cos_norms(v[2 * k], v[2 * k + 1]);
    __syncthreads();
    double c[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
      const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
      for (int k = 0; k < L4D_MT_N; ++k)
        if (A.crit[k] == L4D_GRAD_COS) {
          c[2 * k] += (double)l4d_cos_term(e.a[k], e.b[k], s_cos[k]);
          c[2 * k + 1] += l4d_cos_dot_term(e.a[k], e.b[k], s_cos[k]);
        }
    }
    l4d_block_sum<L4D_MAIN_THREADS, 6>(c, s_red);
    if (threadIdx.x == 0)
      for (int k = 0; k < L4D_MT_N; ++k) { s_cosv[k] = (float)c[2 * k]; s_cos[k].dot = (float)c[2 * k + 1]; }
    __syncthreads();
  } else if (threadIdx.x < L4D_MT_N) {
    s_cosv[threadIdx.x] = 0.f;
    s_cos[threadIdx.x] = l4d_cos_norms(0.0, 0.0);
  }
  __syncthreads();
  const bool chamfer = rays_d != nullptr;
  const float gdist = 0.5f / (float)n;        // d (0.5 mean(dist1 + dist2)) / d dist, ATen's mean backward
  double sum[1] = {0};
  for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
    const L4DMainElem e = l4d_main_train_elem(depth, image, gt, r, A);
    float da[L4D_MT_N], g_pd, g_r, g_i;
    const float v = l4d_main_value(e, A, s_cosv, da);
    if (!A.all_cos || r == 0) sum[0] += v;
    l4d_main_grad(e, A, da, s_cos, &g_pd, &g_r, &g_i);
    g_depth[r] = chamfer ? g_pd : g_pd * e.m;    // with the chamfer term, k_main_finish adds its part and applies m
    g_image[2 * (size_t)r] = g_r;
    g_image[2 * (size_t)r + 1] = g_i;
    if (chamfer) {
      for (int c = 0; c < 3; ++c) {
        const float rd = rays_d[3 * (size_t)r + c];
        P.pred[3 * (size_t)r + c] = l4d_main_point(rd, e.a[L4D_MT_D], A);
        P.gtc[3 * (size_t)r + c] = l4d_main_point(rd, e.b[L4D_MT_D], A);
        P.gx1[3 * (size_t)r + c] = 0.f;
        P.gx2[3 * (size_t)r + c] = 0.f;
      }
      P.gdist[r] = gdist;
      P.gdist[n + r] = gdist;
    }
  }
  __syncthreads();
  l4d_block_sum<L4D_MAIN_THREADS, 1>(sum, s_red);
  if (threadIdx.x == 0) {
    if (chamfer) {
      *P.crit_sum = sum[0];
    } else {
      const float l = l4d_main_total(sum[0], 0.0, n, false);
      *loss = accumulate ? *loss + l : l;
    }
  }
}

// after l4d_chamfer_forward / _backward: 0.5 mean(dist1 + dist2) added to the criteria, and the chamfer gradient of the
// predicted cloud folded into d loss / d depth = (d criteria / d pred_d + sum_c g_c rd_c / scale) * m
__global__ void __launch_bounds__(L4D_MAIN_THREADS) k_main_finish(const float* __restrict__ gt, const float* __restrict__ rays_d,
                                                                  uint32_t n, L4DMainArgs A, L4DMainPtrs P, uint32_t accumulate,
                                                                  float* __restrict__ loss, float* __restrict__ g_depth) {
  __shared__ double s_red[1][L4D_MAIN_THREADS / 32];
  double s[1] = {0};
  for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
    s[0] += (double)(P.d1[r] + P.d2[r]);
    const float gc = l4d_main_fold(P.gx1 + 3 * (size_t)r, rays_d + 3 * (size_t)r, A);
    g_depth[r] = (g_depth[r] + gc) * gt[3 * (size_t)r];
  }
  l4d_block_sum<L4D_MAIN_THREADS, 1>(s, s_red);
  if (threadIdx.x == 0) {
    const float l = l4d_main_total(*P.crit_sum, s[0], n, true);
    *loss = accumulate ? *loss + l : l;
  }
}

__global__ void __launch_bounds__(256) k_main_scale(const float* __restrict__ gs_depth, const float* __restrict__ gs_image,
                                                    const float* __restrict__ g_loss, uint32_t n, float* __restrict__ g_depth,
                                                    float* __restrict__ g_image) {
  const float g = *g_loss;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 3 * (size_t)n; i += (size_t)gridDim.x * blockDim.x) {
    if (i < n) g_depth[i] = gs_depth[i] * g;
    else g_image[i - n] = gs_image[i - n] * g;
  }
}

__device__ inline float l4d_load_pred(const void* p, uint32_t dtype, size_t i) {
  if (dtype == L4D_DTYPE_F16) return __half2float(static_cast<const __half*>(p)[i]);
  if (dtype == L4D_DTYPE_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  return static_cast<const float*>(p)[i];
}

// eval: the ray-drop prediction is `raydrop` (dtype L4D_DTYPE_*) when given, else image_0 (its sigmoid for bce).
// Elementwise terms: one sum over the B*H*W pixels; cos terms: one cosine per (b, w) column over H, thread = column.
__global__ void __launch_bounds__(L4D_MAIN_THREADS) k_main_eval(const float* __restrict__ depth, const float* __restrict__ image,
                                                                const float* __restrict__ gt, const void* __restrict__ raydrop,
                                                                uint32_t dtype, uint32_t B, uint32_t H, uint32_t W, L4DMainArgs A,
                                                                float* __restrict__ loss) {
  __shared__ double s_red[L4D_MT_N][L4D_MAIN_THREADS / 32];
  const size_t n = (size_t)B * H * W;
  auto pred_r = [&](size_t i) {
    if (raydrop) return l4d_load_pred(raydrop, dtype, i);
    const float x = image[2 * i];
    return A.crit[L4D_MT_R] == L4D_GRAD_BCE ? l4d_logistic(x) : x;
  };
  double v[L4D_MT_N] = {0, 0, 0};
  bool elementwise = false;
  for (int k = 0; k < L4D_MT_N; ++k) elementwise |= A.crit[k] != L4D_GRAD_COS;
  if (elementwise)
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
      const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, i, pred_r(i));
      for (int k = 0; k < L4D_MT_N; ++k) {
        float da;
        if (A.crit[k] != L4D_GRAD_COS) v[k] += l4d_grad_crit(A.crit[k], e.a[k], e.b[k], A.delta, &da);
      }
    }
  if (A.any_cos)
    for (uint32_t col = threadIdx.x; col < B * W; col += blockDim.x) {
      const size_t base = (size_t)(col / W) * H * W + col % W;
      double sq[2 * L4D_MT_N] = {0, 0, 0, 0, 0, 0}, c[L4D_MT_N] = {0, 0, 0};
      for (uint32_t h = 0; h < H; ++h) {
        const size_t i = base + (size_t)h * W;
        const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, i, pred_r(i));
        for (int k = 0; k < L4D_MT_N; ++k) { sq[2 * k] += (double)e.a[k] * e.a[k]; sq[2 * k + 1] += (double)e.b[k] * e.b[k]; }
      }
      L4DCos cs[L4D_MT_N];
      for (int k = 0; k < L4D_MT_N; ++k) cs[k] = l4d_cos_norms(sq[2 * k], sq[2 * k + 1]);
      for (uint32_t h = 0; h < H; ++h) {
        const size_t i = base + (size_t)h * W;
        const L4DMainElem e = l4d_main_eval_elem(depth, image, gt, i, pred_r(i));
        for (int k = 0; k < L4D_MT_N; ++k) c[k] += (double)l4d_cos_term(e.a[k], e.b[k], cs[k]);
      }
      for (int k = 0; k < L4D_MT_N; ++k)
        if (A.crit[k] == L4D_GRAD_COS) v[k] += (double)(float)c[k];
    }
  l4d_block_sum<L4D_MAIN_THREADS, L4D_MT_N>(v, s_red);
  if (threadIdx.x == 0) {
    double cnt[L4D_MT_N];
    for (int k = 0; k < L4D_MT_N; ++k) cnt[k] = A.crit[k] == L4D_GRAD_COS ? (double)B * W : (double)n;
    *loss = l4d_main_eval_total(v, cnt, A);
  }
}
#endif
