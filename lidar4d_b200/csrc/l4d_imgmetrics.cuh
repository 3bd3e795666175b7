// l4d_imgmetrics.cuh - the reference's depth / intensity / ray-drop evaluation meters (utils/metrics.py) in CUDA:
//   k_im_columns      compute_*_errors' clamp, |gt - pred|, the per-column sum of (gt - pred)^2 and min / max of gt, and
//                     the axis-0 pass of uniform_filter(., 7) over pred, gt, pred*pred, gt*gt, pred*gt (a thread a column)
//   k_im_rows         the axis-1 pass of those five maps (a thread a (row, map) pair)
//   k_im_ssim         skimage's SSIM map and the per-CTA sums of its cropped mean
//   k_im_finish       the exact median of |gt - pred| (radix select), RMSE, SSIM and PSNR (one CTA)
//   k_raydrop         RaydropMeter.update's RMSE, accuracy and F1 (one CTA)
// The line recurrences and the SSIM element math are __host__ __device__ functions, so tests/hostsim/imgmetricssim.cu
// runs them on the CPU.  Sums are taken in double in a fixed order and no float atomics reach a result: the same inputs
// give the same bits.
//
// [skimage-ext] structural_similarity (scikit-image >= 0.19) at the reference's arguments - a 2-D float32 image,
// win_size 7, uniform filter, use_sample_covariance=True, K1 = 0.01, K2 = 0.03, data_range R = f32(max(gt) - min(gt)):
//   ux, uy, uxx, uyy, uxy = U(x), U(y), U(x*x), U(y*y), U(x*y)               (U = scipy.ndimage.uniform_filter(., 7))
//   vx = c (uxx - ux ux), vy = c (uyy - uy uy), vxy = c (uxy - ux uy),        c = f32(49 / 48)
//   S = ((2 ux) uy + C1)(2 vxy + C2) / ((ux ux + uy uy + C1)(vx + vy + C2)),  C1 = (0.01 R)^2, C2 = (0.03 R)^2
//   ssim = float64 mean of S[3:H-3, 3:W-3]
// all in float32 NumPy ufuncs, so every element operation here is an explicit round-to-nearest intrinsic that nvcc
// cannot contract into an FMA.  skimage squares C1 / C2 with libm powf; here they are x * x (at most an ulp apart).
//
// SciPy's uniform_filter(x, 7) on float32: axis 0 first, its result stored as float32, then axis 1 on that; mode
// 'reflect' (... c b a | a b c ...).  Along a line, in double: t = the left-to-right sum of the first 7 extended values,
// out[0] = f32(t / 7); then t = t + (x[i+3] - x[i-4]) (the difference first) and out[i] = f32(t / 7).
#pragma once
#include <math.h>
#include <stdint.h>

constexpr int L4D_IM_WIN = 7;
constexpr int L4D_IM_R = 3;                    // (win - 1) / 2: the filter radius and the SSIM crop
constexpr int L4D_IM_COL_NT = 128;             // threads per CTA of k_im_columns
constexpr int L4D_IM_ROW_NT = 32;              // ... of k_im_rows (few, long threads: spread them over SMs)
constexpr int L4D_IM_SSIM_NT = 256;            // ... of k_im_ssim
constexpr int L4D_IM_PARTS = 1024;             // most CTAs of k_im_ssim (one double partial each)
constexpr int L4D_IM_FIN_NT = 1024;            // threads of the one-CTA kernels

// float32 operations as NumPy performs them, each rounded once
__host__ __device__ inline float l4d_im_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float l4d_im_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline float l4d_im_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ inline float l4d_im_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// `x[x < lo] = lo; x[x > hi] = hi` (NaN stays NaN)
__host__ __device__ inline float l4d_im_clamp(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

// mode='reflect' index of extended position p of a line of n >= 3 values
__host__ __device__ inline int l4d_im_reflect(int p, int n) { return p < 0 ? -p - 1 : (p >= n ? 2 * n - p - 1 : p); }

// NaN-propagating min / max, as np.min / np.max
__host__ __device__ inline float l4d_im_min(float a, float b) { return (a != a) ? a : ((b != b || b < a) ? b : a); }
__host__ __device__ inline float l4d_im_max(float a, float b) { return (a != a) ? a : ((b != b || b > a) ? b : a); }

// work buffer: clamped pred / gt first (the images the meters measure), then |gt - pred|, the axis-0 and the final
// filtered maps (five each, map-major), the per-column statistics and the SSIM partials; every segment 256-byte aligned
struct L4DImLayout {
  size_t pred, gt, absd, m0, m1, col_sq, col_min, col_max, parts, total;
};

__host__ __device__ inline L4DImLayout l4d_im_layout(uint32_t H, uint32_t W) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t hw = (size_t)H * W;
  L4DImLayout L;
  L.pred = 0;
  L.gt = L.pred + al(4 * hw);
  L.absd = L.gt + al(4 * hw);
  L.m0 = L.absd + al(4 * hw);
  L.m1 = L.m0 + al(4 * 5 * hw);
  L.col_sq = L.m1 + al(4 * 5 * hw);
  L.col_min = L.col_sq + al(8 * (size_t)W);
  L.col_max = L.col_min + al(4 * (size_t)W);
  L.parts = L.col_max + al(4 * (size_t)W);
  L.total = L.parts + al(8 * (size_t)L4D_IM_PARTS);
  return L;
}

// the five products of one clamped pixel pair, in map order (x, y, x*x, y*y, x*y)
__host__ __device__ inline void l4d_im_products(float x, float y, double v[5]) {
  v[0] = (double)x; v[1] = (double)y;
  v[2] = (double)l4d_im_mul(x, x); v[3] = (double)l4d_im_mul(y, y); v[4] = (double)l4d_im_mul(x, y);
}

// k_im_columns' thread body, column j: clamps the column into cp / cg, writes |gt - pred| to absd, returns the column's
// sum of f32((gt - pred)^2) in double (rows in order) and its NaN-propagating min / max of gt, and writes the axis-0 pass of
// the five maps to m0 (map c at m0 + c*H*W)
__host__ __device__ inline void l4d_im_column(const float* __restrict__ pred, const float* __restrict__ gt, int H, int W, int j,
                                              float lo, float hi, float* __restrict__ cp, float* __restrict__ cg,
                                              float* __restrict__ absd, float* __restrict__ m0, double* sq, float* gmin,
                                              float* gmax) {
  const size_t hw = (size_t)H * W;
  double s = 0.0;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = 0; i < H; ++i) {
    const size_t k = (size_t)i * W + j;
    const float p = l4d_im_clamp(pred[k], lo, hi), g = l4d_im_clamp(gt[k], lo, hi);
    cp[k] = p;
    cg[k] = g;
    const float d = l4d_im_sub(g, p);
    absd[k] = fabsf(d);
    s += (double)l4d_im_mul(d, d);
    mn = l4d_im_min(mn, g);
    mx = l4d_im_max(mx, g);
  }
  *sq = s; *gmin = mn; *gmax = mx;
  double t[5] = {0.0, 0.0, 0.0, 0.0, 0.0}, a[5], b[5];
  for (int p = -L4D_IM_R; p <= L4D_IM_R; ++p) {
    const size_t k = (size_t)l4d_im_reflect(p, H) * W + j;
    l4d_im_products(cp[k], cg[k], a);
    for (int c = 0; c < 5; ++c) t[c] += a[c];
  }
  for (int c = 0; c < 5; ++c) m0[c * hw + j] = (float)(t[c] / 7.0);
  for (int i = 1; i < H; ++i) {
    const size_t ka = (size_t)l4d_im_reflect(i + L4D_IM_R, H) * W + j, kb = (size_t)l4d_im_reflect(i - L4D_IM_R - 1, H) * W + j;
    l4d_im_products(cp[ka], cg[ka], a);
    l4d_im_products(cp[kb], cg[kb], b);
    for (int c = 0; c < 5; ++c) {
      t[c] = t[c] + (a[c] - b[c]);
      m0[c * hw + (size_t)i * W + j] = (float)(t[c] / 7.0);
    }
  }
}

// k_im_rows' thread body: uniform_filter1d(., 7, mode='reflect') of one contiguous float32 line of n values
__host__ __device__ inline void l4d_im_line(const float* __restrict__ in, int n, float* __restrict__ out) {
  double t = 0.0;
  for (int p = -L4D_IM_R; p <= L4D_IM_R; ++p) t += (double)in[l4d_im_reflect(p, n)];
  out[0] = (float)(t / 7.0);
  for (int i = 1; i < n; ++i) {
    t = t + ((double)in[l4d_im_reflect(i + L4D_IM_R, n)] - (double)in[l4d_im_reflect(i - L4D_IM_R - 1, n)]);
    out[i] = (float)(t / 7.0);
  }
}

// (C1, C2) = ((0.01 R)^2, (0.03 R)^2) from R = f32(max(gt) - min(gt)), squared as x * x
__host__ __device__ inline void l4d_im_consts(float gmin, float gmax, float* C1, float* C2) {
  const float R = l4d_im_sub(gmax, gmin);
  const float k1 = l4d_im_mul(0.01f, R), k2 = l4d_im_mul(0.03f, R);
  *C1 = l4d_im_mul(k1, k1);
  *C2 = l4d_im_mul(k2, k2);
}

// one element of skimage's S map, in its float32 order
__host__ __device__ inline float l4d_im_ssim(float ux, float uy, float uxx, float uyy, float uxy, float C1, float C2) {
  const float c = (float)(49.0 / 48.0);
  const float vx = l4d_im_mul(c, l4d_im_sub(uxx, l4d_im_mul(ux, ux)));
  const float vy = l4d_im_mul(c, l4d_im_sub(uyy, l4d_im_mul(uy, uy)));
  const float vxy = l4d_im_mul(c, l4d_im_sub(uxy, l4d_im_mul(ux, uy)));
  const float A1 = l4d_im_add(l4d_im_mul(l4d_im_mul(2.f, ux), uy), C1);
  const float A2 = l4d_im_add(l4d_im_mul(2.f, vxy), C2);
  const float B1 = l4d_im_add(l4d_im_add(l4d_im_mul(ux, ux), l4d_im_mul(uy, uy)), C1);
  const float B2 = l4d_im_add(l4d_im_add(vx, vy), C2);
  const float D = l4d_im_mul(B1, B2);
  return l4d_im_div(l4d_im_mul(A1, A2), D);
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------------
// block-wide fold of v in a fixed order (a shuffle tree per warp, then the warps in order); the result is in thread 0
template <typename T, typename Op>
__device__ inline T l4d_im_block_fold(T v, Op op, T* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_down_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();                                  // sh may still be read from a previous fold
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < nw; ++w) v = op(v, sh[w]);
  return v;
}

struct L4DImAddD { __device__ double operator()(double a, double b) const { return a + b; } };
struct L4DImAddU { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };
struct L4DImMinF { __device__ float operator()(float a, float b) const { return l4d_im_min(a, b); } };
struct L4DImMaxF { __device__ float operator()(float a, float b) const { return l4d_im_max(a, b); } };
struct L4DImMinU { __device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a < b ? a : b; } };

__global__ void __launch_bounds__(L4D_IM_COL_NT) k_im_columns(const float* __restrict__ pred, const float* __restrict__ gt,
                                                               uint32_t H, uint32_t W, float lo, float hi, char* __restrict__ work) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= W) return;
  const L4DImLayout L = l4d_im_layout(H, W);
  l4d_im_column(pred, gt, (int)H, (int)W, (int)j, lo, hi, (float*)(work + L.pred), (float*)(work + L.gt),
                (float*)(work + L.absd), (float*)(work + L.m0), (double*)(work + L.col_sq) + j, (float*)(work + L.col_min) + j,
                (float*)(work + L.col_max) + j);
}

__global__ void __launch_bounds__(L4D_IM_ROW_NT) k_im_rows(uint32_t H, uint32_t W, char* __restrict__ work) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 5 * H) return;
  const L4DImLayout L = l4d_im_layout(H, W);
  const size_t off = (size_t)(t % 5) * H * W + (size_t)(t / 5) * W;   // map t % 5, row t / 5
  l4d_im_line((const float*)(work + L.m0) + off, (int)W, (float*)(work + L.m1) + off);
}

__global__ void __launch_bounds__(L4D_IM_SSIM_NT) k_im_ssim(uint32_t H, uint32_t W, char* __restrict__ work) {
  __shared__ float s_f[L4D_IM_SSIM_NT / 32];
  __shared__ double s_d[L4D_IM_SSIM_NT / 32];
  __shared__ float s_c[2];
  const L4DImLayout L = l4d_im_layout(H, W);
  // every CTA folds the column minima / maxima of gt itself (W values), so that no launch is spent on R
  const float* cmin = (const float*)(work + L.col_min);
  const float* cmax = (const float*)(work + L.col_max);
  float mn = INFINITY, mx = -INFINITY;
  for (uint32_t j = threadIdx.x; j < W; j += blockDim.x) { mn = l4d_im_min(mn, cmin[j]); mx = l4d_im_max(mx, cmax[j]); }
  mn = l4d_im_block_fold(mn, L4DImMinF(), s_f);
  mx = l4d_im_block_fold(mx, L4DImMaxF(), s_f);
  if (threadIdx.x == 0) l4d_im_consts(mn, mx, &s_c[0], &s_c[1]);
  __syncthreads();
  const float C1 = s_c[0], C2 = s_c[1];
  const size_t hw = (size_t)H * W;
  const float* m1 = (const float*)(work + L.m1);
  const uint32_t cw = W - 2 * L4D_IM_R, n = (H - 2 * L4D_IM_R) * cw;
  double s = 0.0;
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
    const size_t k = (size_t)(q / cw + L4D_IM_R) * W + (q % cw + L4D_IM_R);
    s += (double)l4d_im_ssim(m1[k], m1[hw + k], m1[2 * hw + k], m1[3 * hw + k], m1[4 * hw + k], C1, C2);
  }
  s = l4d_im_block_fold(s, L4DImAddD(), s_d);
  if (threadIdx.x == 0) ((double*)(work + L.parts))[blockIdx.x] = s;
}

// the r-th smallest (0-based) of n float32 keys >= 0 (|gt - pred|, NaN above +inf) by bit pattern: four 8-bit radix
// passes, each a shared histogram of the keys that match the digits chosen so far.  Returns the key in every thread and
// sets *n_eq (thread 0) to the number of keys equal to it and *rank_in_eq to r's position among them.
__device__ inline uint32_t l4d_im_select(const uint32_t* __restrict__ key, uint32_t n, uint32_t r, uint32_t* hist,
                                         uint32_t* s_sel, uint32_t* n_eq, uint32_t* rank_in_eq) {
  uint32_t prefix = 0, mask = 0;
  const int lane = threadIdx.x & 31;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += blockDim.x) {
      const uint32_t i = base + threadIdx.x;
      uint32_t bin = 256;                                   // no bin: past the end or not a candidate
      if (i < n) {
        const uint32_t k = key[i];
        if ((k & mask) == prefix) bin = (k >> shift) & 255u;
      }
      const uint32_t peers = __match_any_sync(0xffffffffu, bin);
      if (bin < 256 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 32) {                                 // warp 0 finds the bin holding rank r: 8 bins a lane
      uint32_t c[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { c[q] = hist[8 * lane + q]; sum += c[q]; }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const uint32_t hit = __ballot_sync(0xffffffffu, incl > r);
      if (lane == __ffs(hit) - 1) {
        uint32_t before = incl - sum, sel = 0, cnt = 0;
        bool found = false;
#pragma unroll
        for (int q = 0; q < 8; ++q) {                       // unrolled, so that c[] stays in registers
          if (found) continue;
          if (before + c[q] > r) { found = true; sel = q; cnt = c[q]; }
          else before += c[q];
        }
        s_sel[0] = 8 * lane + sel;
        s_sel[1] = r - before;
        s_sel[2] = cnt;
      }
    }
    __syncthreads();
    prefix |= s_sel[0] << shift;
    mask |= 255u << shift;
    r = s_sel[1];
    __syncthreads();
  }
  *n_eq = s_sel[2];
  *rank_in_eq = r;
  return prefix;
}

__global__ void __launch_bounds__(L4D_IM_FIN_NT) k_im_finish(uint32_t H, uint32_t W, uint32_t n_parts, float peak,
                                                             const char* __restrict__ work, double* __restrict__ out) {
  __shared__ uint32_t hist[256], s_sel[3], s_u[L4D_IM_FIN_NT / 32];
  __shared__ double s_d[L4D_IM_FIN_NT / 32];
  const L4DImLayout L = l4d_im_layout(H, W);
  const uint32_t n = H * W;
  const uint32_t* key = (const uint32_t*)(work + L.absd);
  // median of |gt - pred|: np.median takes the middle value, or f32(f32(a + b) / 2) of the two middle values
  uint32_t n_eq, rank;
  const uint32_t lo_key = l4d_im_select(key, n, (n - 1) / 2, hist, s_sel, &n_eq, &rank);
  uint32_t hi_key = lo_key;
  if (!(n & 1u)) {
    uint32_t nxt = 0xffffffffu;                              // the smallest key above lo_key, when lo_key is its last copy
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint32_t k = key[i];
      if (k > lo_key && k < nxt) nxt = k;
    }
    nxt = l4d_im_block_fold(nxt, L4DImMinU(), s_u);
    if (threadIdx.x == 0 && rank + 1 >= n_eq) hi_key = nxt;
  }
  double sq = 0.0, ss = 0.0;
  for (uint32_t j = threadIdx.x; j < W; j += blockDim.x) sq += ((const double*)(work + L.col_sq))[j];
  sq = l4d_im_block_fold(sq, L4DImAddD(), s_d);
  for (uint32_t b = threadIdx.x; b < n_parts; b += blockDim.x) ss += ((const double*)(work + L.parts))[b];
  ss = l4d_im_block_fold(ss, L4DImAddD(), s_d);
  if (threadIdx.x != 0) return;
  const float mse = (float)(sq / (double)n);                 // NumPy's float32 mean (its sum order aside)
  const float a = __uint_as_float(lo_key), b = __uint_as_float(hi_key);
  const float medae = sq != sq ? NAN : ((n & 1u) ? a : l4d_im_div(l4d_im_add(a, b), 2.f));
  out[0] = (double)sqrtf(mse);
  out[1] = (double)medae;
  out[2] = NAN;                                              // LPIPS: not computed here
  out[3] = ss / (double)((H - 2 * L4D_IM_R) * (W - 2 * L4D_IM_R));
  out[4] = (double)l4d_im_mul(10.f, log10f(l4d_im_div(peak, mse)));
}

// RaydropMeter.update: rmse = sqrt(mean(f32((gt - pred)^2))), mask = pred > ratio, acc = mean(mask == gt),
// f1 = 2 p r / (p + r) with p = TP / (TP + FP), r = TP / (TP + FN), in double; counts are 64-bit
__global__ void __launch_bounds__(L4D_IM_FIN_NT) k_raydrop(const float* __restrict__ pred, const float* __restrict__ gt, uint32_t n,
                                                           float ratio, double* __restrict__ out) {
  __shared__ double s_d[L4D_IM_FIN_NT / 32];
  __shared__ unsigned long long s_u[L4D_IM_FIN_NT / 32];
  double sq = 0.0;
  unsigned long long acc = 0, tp = 0, fp = 0, fn = 0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float p = pred[i], t = gt[i];
    const float d = l4d_im_sub(t, p);
    sq += (double)l4d_im_mul(d, d);
    const bool m = p > ratio;
    acc += (m ? 1.f : 0.f) == t;
    tp += m && t == 1.f;
    fp += m && t == 0.f;
    fn += !m && t == 1.f;
  }
  sq = l4d_im_block_fold(sq, L4DImAddD(), s_d);
  acc = l4d_im_block_fold(acc, L4DImAddU(), s_u);
  tp = l4d_im_block_fold(tp, L4DImAddU(), s_u);
  fp = l4d_im_block_fold(fp, L4DImAddU(), s_u);
  fn = l4d_im_block_fold(fn, L4DImAddU(), s_u);
  if (threadIdx.x != 0) return;
  const double pr = (double)tp / (double)(tp + fp), rc = (double)tp / (double)(tp + fn);
  out[0] = (double)sqrtf((float)(sq / (double)n));
  out[1] = (double)acc / (double)n;
  out[2] = (2.0 * (pr * rc)) / (pr + rc);
}
#endif  // __CUDACC__
