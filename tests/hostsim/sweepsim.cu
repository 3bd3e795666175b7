// sweepsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The per-pixel rule of k_sweep_images (lidar4d_b200/csrc/l4d_sweep.cuh) compiled for the CPU, for
// tests/test_sweep_hostsim.py: the three casts (float16, float32, float64 products) and the whole pixel function.
#include <stdint.h>
#include <stdlib.h>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_sweep.cuh"

// u8(r * 255) with the product rounded to half, for half bit patterns h[n]
extern "C" void sws_r255_f16(const uint16_t* h, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; ++k) out[k] = l4d_sw_r255_f16(h[k]);
}
// u8(f32(x * 255))
extern "C" void sws_x255_f32(const float* x, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; ++k) out[k] = l4d_sw_r255_f32(x[k]);
}
// u8(f64(x) * f64(m) * 255), m in {0, 1}
extern "C" void sws_x255_f64(const float* x, const uint8_t* m, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; ++k) out[k] = l4d_u8_f64(l4d_sw_dmul(l4d_sw_dmul((double)x[k], m[k] ? 1.0 : 0.0), 255.0));
}
// the raw casts
extern "C" void sws_u8_f32(const float* x, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; ++k) out[k] = l4d_u8_f32(x[k]);
}
extern "C" void sws_u8_f64(const double* x, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; ++k) out[k] = l4d_u8_f64(x[k]);
}
// k_sweep_images' pixel function over n pixels: r (float, or half bits when is_f16), I, D -> codes[n, 6], pano[n],
// inten[n] (codes a layout does not produce are left as they are)
extern "C" void sws_pixels(uint32_t layout, int is_f16, const void* r, const float* I, const float* D, size_t n,
                           float scale, int test_mask, uint8_t* codes, float* pano, float* inten) {
  for (size_t k = 0; k < n; ++k) {
    const float r32 = is_f16 ? 0.0f : ((const float*)r)[k];
    const uint16_t r16 = is_f16 ? ((const uint16_t*)r)[k] : 0;
    l4d_sweep_pixel(layout, is_f16 != 0, r32, r16, I[k], D[k], scale, test_mask != 0, codes + 6 * k, pano + k, inten + k);
  }
}
