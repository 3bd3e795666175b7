// l4d_sweep.cuh - the per-pixel step between a rendered LiDAR frame and the files the reference writes from it:
// ray-drop thresholding, masking, the depth / scale division and the 8-bit colour-mapped images of
//   SIM   model/simulator.py:124-171          Simulator.render
//   TEST  model/runner.py:462-469, 755-793    Trainer.test_step + Trainer.test
//   EVAL  model/runner.py:611-634             Trainer.evaluate_one_epoch's validation panel
// k_sweep_images is one launch, a thread a pixel.  The numerics are the NumPy / torch ones the reference relies on, and
// they live in the __host__ __device__ functions below, so tests/hostsim/sweepsim.cu runs them on the CPU:
//   * float -> uint8 is NumPy's C cast as x86-64 compiles it: truncation to int32 (cvtt*2si), then the low byte; NaN, inf
//     and anything outside the int32 range come out as INT32_MIN, i.e. 0.  CUDA's cvt.rzi.s32 saturates instead, hence
//     the explicit range test.  300.7 -> 44, -1 -> 255.
//   * r * 255 is computed in r's dtype.  A float16 ray drop (the U-Net under fp16 autocast) is multiplied as NumPy's
//     half ufunc does it, in float32 and rounded once to half (the float32 product of a half and 255 is exact).
//   * m = r > 0.5 in r's dtype.  x * m is torch's float32 * int64: x * 1.0f or x * 0.0f (NaN * 0 stays NaN).
//   * EVAL rows 5-6 are NumPy's float32 * int64 mask, which promotes to float64: the product with 255 is taken in double.
//   * The cloud input is x / f32(scale) (NumPy 2 promotes the Python float weakly), an IEEE division.
// Every float operation is an explicit round-to-nearest intrinsic on the device, so nothing contracts into an FMA.
#pragma once
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

constexpr int L4D_SWEEP_NT = 256;
constexpr int L4D_SWEEP_CODES = 6;     // 8-bit values per pixel (EVAL uses all six)

__host__ __device__ inline float l4d_sw_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double l4d_sw_dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float l4d_sw_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// NumPy's float32 / float64 -> uint8 cast (see the header)
__host__ __device__ inline uint8_t l4d_u8_f32(float x) {
  if (!(x >= -2147483648.0f && x < 2147483648.0f)) return 0;
  return (uint8_t)(uint32_t)(int32_t)x;
}
__host__ __device__ inline uint8_t l4d_u8_f64(double x) {
  if (!(x > -2147483649.0 && x < 2147483648.0)) return 0;
  return (uint8_t)(uint32_t)(int32_t)x;
}

// r * 255 rounded to r's dtype, then cast; r16 is the half's bit pattern
__host__ __device__ inline uint8_t l4d_sw_r255_f32(float r) { return l4d_u8_f32(l4d_sw_mul(r, 255.0f)); }
__host__ __device__ inline uint8_t l4d_sw_r255_f16(uint16_t r16) {
  __half_raw hr;
  hr.x = r16;
  const float p = l4d_sw_mul(__half2float(__half(hr)), 255.0f);
  return l4d_u8_f32(__half2float(__float2half_rn(p)));
}
__host__ __device__ inline bool l4d_sw_keep_f16(uint16_t r16) {
  __half_raw hr;
  hr.x = r16;
  return __half2float(__half(hr)) > 0.5f;
}

// One pixel: r (r32, or the half r16 when is_f16), intensity I, depth D ->
//   codes[]  SIM:  u8(r 255), u8(f32(I m) 255), u8(f32(D m) 255)
//            TEST: u8(m 255), u8(I' 255), u8(D' 255)                   (I', D' = I m, D m when test_mask, else I, D)
//            EVAL: u8(r 255), u8(I 255), u8(D 255), u8(m 255), u8(f64(I m) 255), u8(f64(D m) 255)
//   *pano    SIM: D m / f32(scale), TEST: D' / f32(scale)
//   *inten   SIM: I m
__host__ __device__ inline void l4d_sweep_pixel(uint32_t layout, bool is_f16, float r32, uint16_t r16, float I, float D,
                                                float scale, bool test_mask, uint8_t* codes, float* pano, float* inten) {
  const bool keep = is_f16 ? l4d_sw_keep_f16(r16) : (r32 > 0.5f);
  const uint8_t r255 = is_f16 ? l4d_sw_r255_f16(r16) : l4d_sw_r255_f32(r32);
  const float mf = keep ? 1.0f : 0.0f;
  const float Im = l4d_sw_mul(I, mf), Dm = l4d_sw_mul(D, mf);
  const uint8_t m255 = keep ? 255 : 0;
  if (layout == L4D_SWEEP_SIM) {
    codes[0] = r255;
    codes[1] = l4d_u8_f32(l4d_sw_mul(Im, 255.0f));
    codes[2] = l4d_u8_f32(l4d_sw_mul(Dm, 255.0f));
    *pano = l4d_sw_div(Dm, scale);
    *inten = Im;
  } else if (layout == L4D_SWEEP_TEST) {
    const float Ix = test_mask ? Im : I, Dx = test_mask ? Dm : D;
    codes[0] = m255;
    codes[1] = l4d_u8_f32(l4d_sw_mul(Ix, 255.0f));
    codes[2] = l4d_u8_f32(l4d_sw_mul(Dx, 255.0f));
    *pano = l4d_sw_div(Dx, scale);
  } else {
    const double md = keep ? 1.0 : 0.0;
    codes[0] = r255;
    codes[1] = l4d_u8_f32(l4d_sw_mul(I, 255.0f));
    codes[2] = l4d_u8_f32(l4d_sw_mul(D, 255.0f));
    codes[3] = m255;
    codes[4] = l4d_u8_f64(l4d_sw_dmul(l4d_sw_dmul((double)I, md), 255.0));
    codes[5] = l4d_u8_f64(l4d_sw_dmul(l4d_sw_dmul((double)D, md), 255.0));
  }
}

// Which panel row gets which code and how it is coloured: 0 = grey (cv2 GRAY2BGR: the byte three times, or once in the
// TEST layout's single-channel ray-drop image), 1 = the intensity table (COLORMAP_BONE), 2 = the depth table (TURBO).
__host__ __device__ inline int l4d_sweep_rows(uint32_t layout) {
  return layout == L4D_SWEEP_EVAL ? 6 : 3;
}
__host__ __device__ inline int l4d_sweep_row_kind(int row) { return row % 3; }

struct L4DSweepArgs {
  const float* depth;         // [H*W]
  const float* image;         // [H*W, 2]: channel 0 ray drop, channel 1 intensity
  const void* raydrop;        // [H*W] float or half, or null (then image channel 0)
  const uint8_t* lut[2];      // [256, 3] BGR: intensity, depth
  uint8_t* panel;
  float* pano;
  float* inten;
  uint32_t hw, layout, is_f16, test_mask;
  float scale;
};

__global__ void __launch_bounds__(L4D_SWEEP_NT) k_sweep_images(const L4DSweepArgs A) {
  const uint32_t p = blockIdx.x * L4D_SWEEP_NT + threadIdx.x;
  if (p >= A.hw) return;
  float r32 = 0.0f;
  uint16_t r16 = 0;
  if (!A.raydrop) r32 = __ldg(A.image + 2 * (size_t)p);
  else if (A.is_f16) r16 = __ldg((const unsigned short*)A.raydrop + p);
  else r32 = __ldg((const float*)A.raydrop + p);
  const float I = __ldg(A.image + 2 * (size_t)p + 1), D = __ldg(A.depth + p);
  uint8_t c[L4D_SWEEP_CODES];
  float pano = 0.0f, inten = 0.0f;
  l4d_sweep_pixel(A.layout, A.is_f16 != 0, r32, r16, I, D, A.scale, A.test_mask != 0, c, &pano, &inten);
  if (A.layout != L4D_SWEEP_EVAL) A.pano[p] = pano;
  if (A.layout == L4D_SWEEP_SIM) A.inten[p] = inten;
  const size_t plane = (size_t)A.hw * 3;
  if (A.layout == L4D_SWEEP_TEST) {   // [H, W] ray drop, then [H, W, 3] intensity and [H, W, 3] depth
    A.panel[p] = c[0];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint8_t* lut = k == 0 ? A.lut[0] : A.lut[1];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) A.panel[A.hw + k * plane + 3 * (size_t)p + ch] = __ldg(lut + 3 * c[k + 1] + ch);
    }
    return;
  }
  const int rows = l4d_sweep_rows(A.layout);   // [rows * H, W, 3], row blocks stacked as cv2.vconcat stacks them
#pragma unroll
  for (int r = 0; r < L4D_SWEEP_CODES; ++r) {
    if (r >= rows) break;
    const int kind = l4d_sweep_row_kind(r);
    const uint8_t* lut = kind == 1 ? A.lut[0] : A.lut[1];
    uint8_t* o = A.panel + r * plane + 3 * (size_t)p;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch] = kind == 0 ? c[r] : __ldg(lut + 3 * c[r] + ch);
  }
}
