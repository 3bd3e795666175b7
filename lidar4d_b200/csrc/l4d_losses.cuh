// l4d_losses.cuh - the rest of the reference's train_step after the flow loss, value and gradient in CUDA:
//   k_patch_loss      model/runner.py:278-369: the depth-gradient loss of patch batches (finite differences or Sobel,
//                     criteria l1 / mse / huber / bce / cos) and the grad_norm_smooth / spatial_smooth / tv_loss terms
//   k_los_partial     model/runner.py:255-276: URF's line-of-sight loss over weights / z_vals [n, S]
//   k_los_finalize      (+ its fixed-order reduction, and the degenerate case of the global distr maximum)
//   k_los_backward    d loss / d weights
//   k_loss_scale      d loss / d depth of the patch loss times the incoming gradient, read from device memory
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
  // cosine similarity per patch (ATen's cosine_similarity: each side divided by max(|v|, eps), then the dot product)
  float na = 0.f, nb = 0.f, dot_ab = 0.f, norm_a = 0.f;
  if (want_grad && use_cos) {
    double sa2 = 0, sb2 = 0;
    for (int i = 0; i < xr; ++i)
      for (int j = 0; j < xc; ++j) {
        const float gv = dxv(G, i, j, false, nullptr);
        const float mk = M(i, j) * (fabsf(gv) < 0.01f ? 1.f : 0.f);
        const float av = dxv(P, i, j, true, nullptr) * mk, bv = gv * mk;
        sa2 += (double)av * av; sb2 += (double)bv * bv;
      }
    norm_a = sqrtf((float)sa2);
    na = fmaxf(norm_a, 1e-8f); nb = fmaxf(sqrtf((float)sb2), 1e-8f);
    double c = 0, d = 0;
    for (int i = 0; i < xr; ++i)
      for (int j = 0; j < xc; ++j) {
        const float gv = dxv(G, i, j, false, nullptr);
        const float mk = M(i, j) * (fabsf(gv) < 0.01f ? 1.f : 0.f);
        const float av = dxv(P, i, j, true, nullptr) * mk, bv = gv * mk;
        c += (double)((av / na) * (bv / nb));
        d += (double)av * (bv / nb);
      }
    dot_ab = (float)d;
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
            const float av = v * mk, bv = gv * mk;
            da = bv / nb / na;
            if (norm_a >= 1e-8f) da -= av / norm_a * dot_ab / (na * na);
            da = -da;
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

#ifdef __CUDACC__
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
#endif
