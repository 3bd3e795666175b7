// l4d_refine.cuh - the array work of the reference's ray-drop refinement loop (model/runner.py Trainer.refine:865-913):
//   k_box_mask      runner.py:888-898: input * mask, mask = 0 inside up to L4D_MAX_BOXES random boxes (the same for
//                   every frame and channel) and 1 elsewhere - one launch, boxes passed by value
//   k_bce           runner.py:901: torch.nn.BCELoss() (mean), per-CTA double partial sums of the element losses
//   k_bce_finish      (+ one CTA summing the partials in a fixed order: the same inputs give the same bits)
//   k_bce_bwd       d loss / d pred times the incoming gradient, read from device memory
// The element math is in __host__ __device__ functions, so tests/hostsim/refinesim.cu runs it on the CPU.
#pragma once
#include <math.h>
#include <stdint.h>

#include "l4d_losses.cuh"       // l4d_block_sum

struct L4DBoxes {           // kernel argument: (y0, x0, h, w) of each box, h, w >= 1, inside the image
  uint32_t n;
  int32_t y0[L4D_MAX_BOXES], x0[L4D_MAX_BOXES], h[L4D_MAX_BOXES], w[L4D_MAX_BOXES];
};

// the mask value of pixel (y, x): 0 inside any box, else 1
__host__ __device__ inline float l4d_box_value(const L4DBoxes& b, int32_t y, int32_t x) {
  for (uint32_t k = 0; k < b.n; ++k)
    if ((uint32_t)(y - b.y0[k]) < (uint32_t)b.h[k] && (uint32_t)(x - b.x0[k]) < (uint32_t)b.w[k]) return 0.f;
  return 1.f;
}

// `input * mask` as ATen evaluates it: a multiplication, so -0.0 for x < 0 in a box and NaN for inf / NaN in a box
__host__ __device__ inline float l4d_box_apply(float x, float m) { return x * m; }

// torch's binary_cross_entropy element (ATen Loss.cu): each log term clamped at -100.  Torch asserts on a prediction
// outside [0, 1]; here that element is NaN.
__host__ __device__ inline float l4d_bce_elem(float x, float t) {
  if (!(x >= 0.f && x <= 1.f)) return NAN;
  const float li = fmaxf(logf(x), -100.f);
  const float l1 = fmaxf(log1pf(-x), -100.f);
  return ((t - 1.f) * l1) - (t * li);
}

// torch's binary_cross_entropy_backward element, then the mean's division: ((g (x - t)) / max((1 - x) x, 1e-12)) / n
__host__ __device__ inline float l4d_bce_grad(float x, float t, float g, float n) {
  if (!(x >= 0.f && x <= 1.f)) return NAN;
  const float den = fmaxf((1.f - x) * x, 1e-12f);
  return g * (x - t) / den / n;
}

#ifdef __CUDACC__
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#define L4D_BOX_NT 256
#define L4D_BOX_PLANES 16       // planes ([H, W] images) per thread: the mask of a pixel is found once for all of them
#define L4D_BCE_NT 256
#define L4D_BCE_PER_THREAD 8    // elements per thread before the grid caps at L4D_BCE_BLOCKS
#define L4D_BCE_BLOCKS 1024     // fixed partial count: the partition depends on n only, not on the device

struct L4DBceWork {
  double part[L4D_BCE_BLOCKS];
};

__device__ inline float l4d_to_float(float v) { return v; }
__device__ inline float l4d_to_float(__half v) { return __half2float(v); }
__device__ inline float l4d_to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ inline void l4d_from_float(float v, float* o) { *o = v; }
__device__ inline void l4d_from_float(float v, __half* o) { *o = __float2half_rn(v); }
__device__ inline void l4d_from_float(float v, __nv_bfloat16* o) { *o = __float2bfloat16_rn(v); }

// grid (pixel blocks, plane groups): thread = one pixel of HW, L4D_BOX_PLANES planes of the B*C
__global__ void __launch_bounds__(L4D_BOX_NT) k_box_mask(const float* x, float* out, uint32_t planes, uint32_t H,
                                                         uint32_t W, L4DBoxes boxes) {
  const uint32_t hw = H * W;
  const uint32_t p = blockIdx.x * L4D_BOX_NT + threadIdx.x;
  if (p >= hw) return;
  const int32_t y = (int32_t)(p / W), xx = (int32_t)(p - (uint32_t)y * W);
  const float m = l4d_box_value(boxes, y, xx);
  const uint32_t c0 = blockIdx.y * L4D_BOX_PLANES;
  const uint32_t c1 = c0 + L4D_BOX_PLANES < planes ? c0 + L4D_BOX_PLANES : planes;
  float v[L4D_BOX_PLANES];
#pragma unroll
  for (int k = 0; k < L4D_BOX_PLANES; ++k)
    if (c0 + k < c1) v[k] = x[(size_t)(c0 + k) * hw + p];
#pragma unroll
  for (int k = 0; k < L4D_BOX_PLANES; ++k)
    if (c0 + k < c1) out[(size_t)(c0 + k) * hw + p] = l4d_box_apply(v[k], m);
}

template <typename T>
__global__ void __launch_bounds__(L4D_BCE_NT) k_bce(const T* __restrict__ pred, const float* __restrict__ target, uint32_t n,
                                                    L4DBceWork* __restrict__ work) {
  __shared__ double s_red[1][L4D_BCE_NT / 32];
  double v[1] = {0};
  for (uint32_t i = blockIdx.x * L4D_BCE_NT + threadIdx.x; i < n; i += gridDim.x * L4D_BCE_NT)
    v[0] += (double)l4d_bce_elem(l4d_to_float(pred[i]), target[i]);
  l4d_block_sum<L4D_BCE_NT, 1>(v, s_red);
  if (threadIdx.x == 0) work->part[blockIdx.x] = v[0];
}

__global__ void __launch_bounds__(1024) k_bce_finish(const L4DBceWork* __restrict__ work, uint32_t parts, uint32_t n,
                                                     float* __restrict__ loss) {
  __shared__ double s_red[1][32];
  double v[1] = {0};
  for (uint32_t b = threadIdx.x; b < parts; b += 1024) v[0] += work->part[b];
  l4d_block_sum<1024, 1>(v, s_red);
  if (threadIdx.x == 0) *loss = (float)(v[0] / (double)n);
}

template <typename T>
__global__ void __launch_bounds__(256) k_bce_bwd(const T* __restrict__ pred, const float* __restrict__ target, uint32_t n,
                                                 const float* __restrict__ g_loss, T* __restrict__ g_pred) {
  const float g = *g_loss, fn = (float)n;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    l4d_from_float(l4d_bce_grad(l4d_to_float(pred[i]), target[i], g, fn), g_pred + i);
}
#endif
