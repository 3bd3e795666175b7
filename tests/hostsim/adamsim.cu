// adamsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The per-element Adam update of k_adam_flat (l4d_adam_elem, lidar4d_b200/csrc/l4d_optim.cuh) compiled for the CPU, next to
// two independent restatements that tests/test_adam_hostsim.py holds it against:
//   as_torch:  torch 2.11's fused Adam, ATen/native/cuda/fused_adam_utils.cuh adam_math (no weight decay, no amsgrad,
//              not maximising), written from that source with std::fma, sqrtf and '/';
//   as_former: the update k_adam_flat computed before l4d_adam_elem existed (lerp form of the first moment, an unfused second
//              moment, power-of-two scaling of every sqrtf / division operand, bias corrections in double on the host), kept
//              to show which of its differences the test detects.
// Built with -ffp-contract=off, so every operation rounds where the source says it does.  Arrays are updated in place.
#include <math.h>
#include <stdint.h>
#include <cmath>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_optim.cuh"

extern "C" void as_kernel(int64_t n, float* p, float* m, float* v, const float* g, float inv_scale, float beta1, float beta2,
                          float eps, float lr, float bc1, float bc2_sqrt) {
  const float step_size = lr / bc1;
  for (int64_t i = 0; i < n; ++i) l4d_adam_elem(p[i], m[i], v[i], g[i], inv_scale, beta1, beta2, eps, step_size, bc2_sqrt);
}

extern "C" void as_torch(int64_t n, float* p, float* m, float* v, const float* g, float grad_scale, float beta1, float beta2,
                         float eps, float lr, float bc1, float bc2_sqrt) {
  for (int64_t i = 0; i < n; ++i) {
    float param = p[i], grad = g[i], exp_avg = m[i], exp_avg_sq = v[i];
    grad /= grad_scale;
    exp_avg = std::fma(beta1, exp_avg, std::fma(-beta1, grad, grad));
    exp_avg_sq = std::fma(beta2, exp_avg_sq, std::fma(-beta2, grad * grad, grad * grad));
    const float step_size = lr / bc1;
    const float denom = (std::sqrt(exp_avg_sq) / bc2_sqrt) + eps;
    param -= step_size * exp_avg / denom;
    p[i] = param; m[i] = exp_avg; v[i] = exp_avg_sq;
  }
}

extern "C" void as_former(int64_t n, float* p, float* m, float* v, const float* g, float inv_scale, float beta1, float beta2,
                          float eps, float lr, uint32_t step) {
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  const float w = 1.0f - beta1, w2 = 1.0f - beta2;
  const float st = lr / bc1;
  for (int64_t i = 0; i < n; ++i) {
    const float gg = g[i] * inv_scale;
    m[i] = fmaf(w, gg - m[i], m[i]);
    v[i] = beta2 * v[i] + w2 * gg * gg;
    const float den = (sqrtf(v[i] * 1.8446744073709552e19f) * 2.3283064365386963e-10f) / bc2_sqrt + eps;
    p[i] = p[i] - ((st * m[i]) * 1.8446744073709552e19f) / den * 5.421010862427522e-20f;
  }
}
