// l4d_rays.cuh - SURVEY.md 8(f) #2: the thin layer in front of the render kernels, one launch instead of the
// reference's chain of elementwise torch ops (the main loss behind them is in l4d_losses.cuh):
//   k_lidar_rays   data/base_dataset.py:15-102 get_lidar_rays (pixel -> azimuth / elevation -> direction @ R^T, origin)
//                  + the ground-truth gather of data/kitti360_dataset.py:170-178 (images_lidar[inds])
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// pose: device [4][4] row-major cam2world; inds: flat pixel ids i_row*W + i_col (nullptr = all H*W pixels in order)
__global__ void __launch_bounds__(256) k_lidar_rays(const float* __restrict__ pose, float fov_up, float fov, uint32_t H, uint32_t W,
                                                    const long long* __restrict__ inds, uint32_t n, const float* __restrict__ image,
                                                    uint32_t C, float* __restrict__ rays_o, float* __restrict__ rays_d,
                                                    float* __restrict__ gt) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const long long pix = inds ? inds[r] : (long long)r;
  // meshgrid of base_dataset.py:31-36: i = column (0..W-1), j = row (0..H-1), flattened row-major
  const float i = (float)(pix % W), j = (float)(pix / W);
  // beta = -(i - W/2) / W * 2 * pi ; alpha = (fov_up - j / H * fov) / 180 * pi, fp32 op by op like the torch chain on CUDA,
  // where `tensor / python_scalar` is evaluated as tensor * (1.0f / scalar) (ATen BinaryDivTrueKernel.cu)
  const float inv_w = 1.0f / (float)W, inv_h = 1.0f / (float)H, inv_180 = 1.0f / 180.0f, pi = 3.14159265358979323846f;
  const float beta = __fmul_rn(__fmul_rn(__fmul_rn(-__fsub_rn(i, (float)W / 2.0f), inv_w), 2.0f), pi);
  const float alpha = __fmul_rn(__fmul_rn(__fsub_rn(fov_up, __fmul_rn(__fmul_rn(j, inv_h), fov)), inv_180), pi);
  const float ca = cosf(alpha), sa = sinf(alpha), cb = cosf(beta), sb = sinf(beta);
  const float d0 = __fmul_rn(ca, cb), d1 = __fmul_rn(ca, sb), d2 = sa;
  // rays_d = directions @ R^T : d_k = sum_m dir_m * R[k][m]
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float v = fmaf(d2, pose[4 * k + 2], fmaf(d1, pose[4 * k + 1], __fmul_rn(d0, pose[4 * k])));
    rays_d[3 * (size_t)r + k] = v;
    rays_o[3 * (size_t)r + k] = pose[4 * k + 3];
  }
  if (gt && image)
    for (uint32_t c = 0; c < C; ++c) gt[(size_t)r * C + c] = image[(size_t)pix * C + c];
}
