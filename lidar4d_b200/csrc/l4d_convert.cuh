// l4d_convert.cuh - range image <-> point cloud conversions of utils/convert.py and the reduction after the chamfer op
// in PointsMeter.update (utils/metrics.py:249-270), one sm_90a kernel family each:
//   k_pano_project<PASS>    lidar_to_pano_with_intensities (convert.py:4-65): point cloud -> range image + intensities
//   k_pano_unproject<PASS>  pano_to_lidar_with_intensities (convert.py:99-138): range image -> points, np.where order
//   k_point_metrics         Chamfer distance, precisions and F-score from the two squared-distance vectors (metrics.py:13-27)
// (included at the end of l4d_kernels.cu: one translation unit, one shared library)
//
// Projection arithmetic.  The reference runs its loop on NumPy float32 scalars; under NEP 50 promotion a Python float
// does not widen them, so every step is float32 (the constants are rounded once from double, as Python computes them):
//   dist  = sqrt((x*x + y*y) + z*z)                          (np.linalg.norm, no contraction)
//   beta  = fl(pi) - atan2(y, x)
//   alpha = atan2(z, sqrt(x*x + y*y)) + fl(fov_down/180*pi)
//   c = rint(beta / fl(2*pi/W)),  r = rint(H - alpha / fl(fov/180*pi/H))      (Python round: half to even)
// Every operation is spelled with an explicit IEEE rounding so that no FMA contraction changes it.  atan2f is the
// device's, not NumPy's (neither is correctly rounded), and the reference's `x**2` is libm powf, which is 1 ulp off
// x*x for some inputs: both can move a point across a .5 rounding boundary, nothing else.
//
// Z-buffer.  The reference folds the points in order with `if pano == 0: set; elif pano > dist: set`.  So a point at
// distance 0 resets its pixel to empty (keeping its own intensity) and later points refill it, and among the points
// after the last such reset the smallest distance wins, the earliest on ties.  Three passes reproduce that fold:
//   PASS 0: per pixel, atomicMax of 1 + the index of every zero-distance point (0 = none);
//   PASS 1: per pixel, a 64-bit atomicMin of (dist bits << 32 | index) over the positive-distance points whose index is
//           past that reset (for non-negative floats the integer order is the float order, and ties go to the smaller
//           index - the trick of k_chamfer_nn);
//   PASS 2: per pixel, resolve the key (or the reset, or nothing) into pano and intensities.
#pragma once

namespace l4d_convert {

constexpr int CV_NT = 128;                    // threads per CTA of the grid-stride kernels
constexpr int CV_PIX = 8;                     // pixels per thread of an unprojection tile
constexpr int CV_TILE = CV_NT * CV_PIX;       // pixels per unprojection tile (one count per tile)
constexpr int CV_RED_NT = 1024;               // threads of the single-CTA metric reduction
constexpr uint64_t CV_MAX_PIXELS = 1ull << 31;

struct ProjectArgs {
  const float* pts;           // [n, stride]
  uint32_t n, stride;
  uint32_t H, W;
  float pi, alpha_off, c_scale, r_scale, Hf, max_depth;
  uint32_t* zlast;            // [H*W] 1 + index of the last zero-distance point, 0 = none
  unsigned long long* keys;   // [H*W] (dist bits << 32 | index), ~0 = none
  float* pano;                // [H*W]
  float* inten;               // [H*W] or nullptr
};

__device__ __forceinline__ float cv_dist(float x, float y, float z) {
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// flat pixel of a point, or -1 when it falls outside the image (NaN angles fail every comparison and are dropped too)
__device__ __forceinline__ long long cv_pixel(const ProjectArgs& A, float x, float y, float z) {
  const float beta = __fsub_rn(A.pi, atan2f(y, x));
  const float rho = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
  const float alpha = __fadd_rn(atan2f(z, rho), A.alpha_off);
  const float cf = rintf(__fdiv_rn(beta, A.c_scale));
  const float rf = rintf(__fsub_rn(A.Hf, __fdiv_rn(alpha, A.r_scale)));
  if (!(cf >= 0.f && rf >= 0.f && cf < 4294967296.f && rf < 4294967296.f)) return -1;
  const uint32_t c = (uint32_t)cf, r = (uint32_t)rf;
  if (r >= A.H || c >= A.W) return -1;         // convert.py:54: c == W is dropped, not wrapped
  return (long long)r * A.W + c;
}

template <int PASS>
__global__ void __launch_bounds__(CV_NT) k_pano_project(const ProjectArgs A) {
  const size_t stride = (size_t)gridDim.x * CV_NT;
  if constexpr (PASS == 2) {
    const size_t hw = (size_t)A.H * A.W;
    for (size_t p = (size_t)blockIdx.x * CV_NT + threadIdx.x; p < hw; p += stride) {
      const unsigned long long k = A.keys[p];
      const uint32_t z = A.zlast[p];
      float d = 0.f, it = 0.f;
      if (k != ~0ull) {
        d = __uint_as_float((uint32_t)(k >> 32));
        if (A.stride == 4) it = A.pts[(size_t)(uint32_t)k * 4 + 3];
      } else if (z && A.stride == 4) {
        it = A.pts[(size_t)(z - 1) * 4 + 3];        // emptied by a zero-distance point: its intensity stays
      }
      A.pano[p] = d;
      if (A.inten) A.inten[p] = it;
    }
  } else {
    for (size_t i = (size_t)blockIdx.x * CV_NT + threadIdx.x; i < A.n; i += stride) {
      const float* p = A.pts + i * A.stride;
      const float x = p[0], y = p[1], z = p[2];
      const float d = cv_dist(x, y, z);
      if (!(d < A.max_depth)) continue;          // convert.py:44 (a NaN distance is dropped: the reference raises on it)
      if (PASS == 0) {
        if (d != 0.f) continue;
        const long long px = cv_pixel(A, x, y, z);
        if (px >= 0) atomicMax(A.zlast + px, (uint32_t)i + 1u);
      } else {
        if (d == 0.f) continue;
        const long long px = cv_pixel(A, x, y, z);
        if (px < 0 || (uint32_t)i < A.zlast[px]) continue;    // before the pixel's last reset: folded away
        atomicMin(A.keys + px, ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)i);
      }
    }
  }
}

// Order-preserving compaction of elements [0, size) in tiles of CV_TILE, shared by k_pano_unproject and the ground-removal
// kernels (l4d_ground.cuh).  Op supplies `bool keep(size_t q) const` and `void emit(size_t q, uint32_t pos) const`.
// PASS 0: kept elements per tile; PASS 1 (one CTA): exclusive scan of the tile counts and the total to *count;
// PASS 2: every tile scatters its kept elements to its offset in element order (an atomic counter would not keep it)
template <class Op, int PASS>
__device__ __forceinline__ void cv_compact(const Op& op, size_t size, uint32_t n_tiles, uint32_t* offsets, uint32_t* count) {
  __shared__ uint32_t s_warp[CV_NT / 32];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (PASS == 1) {
    uint32_t carry = 0;
    for (uint32_t t0 = 0; t0 < n_tiles; t0 += CV_NT) {
      const uint32_t t = t0 + threadIdx.x;
      const uint32_t v = t < n_tiles ? offsets[t] : 0u;
      uint32_t inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (uint32_t)o) inc += u;
      }
      if (lane == 31) s_warp[warp] = inc;
      __syncthreads();
      uint32_t before = carry;
      for (uint32_t w = 0; w < warp; ++w) before += s_warp[w];
      if (t < n_tiles) offsets[t] = before + inc - v;
      uint32_t total = 0;
      for (int w = 0; w < CV_NT / 32; ++w) total += s_warp[w];
      carry += total;
      __syncthreads();
    }
    if (threadIdx.x == 0) *count = carry;
    return;
  }
  for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const size_t base = (size_t)t * CV_TILE;
    if (PASS == 0) {
      uint32_t c = 0;
#pragma unroll
      for (int j = 0; j < CV_PIX; ++j) {
        const size_t q = base + (size_t)j * CV_NT + threadIdx.x;
        c += (q < size && op.keep(q)) ? 1u : 0u;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) s_warp[warp] = c;
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < CV_NT / 32; ++w) s += s_warp[w];
        offsets[t] = s;
      }
      __syncthreads();
      continue;
    }
    uint32_t off = offsets[t];
    for (int j = 0; j < CV_PIX; ++j) {          // row j of the tile = CV_NT consecutive elements, in element order
      const size_t q = base + (size_t)j * CV_NT + threadIdx.x;
      const bool keep = q < size && op.keep(q);
      const uint32_t ballot = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_warp[warp] = __popc(ballot);
      __syncthreads();
      uint32_t pos = off + __popc(ballot & ((1u << lane) - 1u));
      uint32_t row_total = 0;
      for (uint32_t w = 0; w < CV_NT / 32; ++w) {
        if (w < warp) pos += s_warp[w];
        row_total += s_warp[w];
      }
      if (keep) op.emit(q, pos);
      off += row_total;
      __syncthreads();
    }
  }
}

// pano != 0 as NumPy tests it: NaN is kept, +-0 is not
__device__ __forceinline__ bool cv_kept(float v) { return v != 0.f; }

struct UnprojectArgs {
  const float* pano;          // [H*W]
  const float* inten;         // [H*W] or nullptr
  uint32_t H, W;
  float fov_up, fov, pi;
  uint32_t n_tiles;
  uint32_t* offsets;          // [n_tiles]: kept pixels per tile (PASS 0), then their exclusive prefix sum (PASS 1)
  float* out;                 // [H*W, 3 | 4]
  uint32_t* count;            // device scalar

  __device__ __forceinline__ bool keep(size_t q) const { return cv_kept(pano[q]); }
  __device__ __forceinline__ void emit(size_t q, uint32_t pos) const {
    // beta = -(i - W/2)/W*2*pi, alpha = (fov_up - j/H*fov)/180*pi: convert.py:112-116 in float32, op by op
    const float v = pano[q];
    const float ci = (float)(q % W), rj = (float)(q / W);
    const float beta = __fmul_rn(__fmul_rn(__fdiv_rn(-__fsub_rn(ci, (float)W * 0.5f), (float)W), 2.0f), pi);
    const float alpha = __fmul_rn(__fdiv_rn(__fsub_rn(fov_up, __fmul_rn(__fdiv_rn(rj, (float)H), fov)), 180.0f), pi);
    const float ca = cosf(alpha);
    float* o = out + (size_t)pos * (inten ? 4 : 3);
    o[0] = __fmul_rn(__fmul_rn(ca, cosf(beta)), v);
    o[1] = __fmul_rn(__fmul_rn(ca, sinf(beta)), v);
    o[2] = __fmul_rn(sinf(alpha), v);
    if (inten) o[3] = inten[q];
  }
};

// every pixel with pano != 0 becomes a row, in row-major pixel order: cv_compact over the H*W pixels
template <int PASS>
__global__ void __launch_bounds__(CV_NT) k_pano_unproject(const UnprojectArgs A) {
  cv_compact<UnprojectArgs, PASS>(A, (size_t)A.H * A.W, A.n_tiles, A.offsets, A.count);
}

// PointsMeter.update after the chamfer op, dist1 / dist2 = squared distances: out = {cd, fscore, p1, p2, 0} with
// cd = mean(dist1) + mean(dist2), p = count(dist < thr) / size (exact integer counts), fscore = 2 p1 p2 / (p1 + p2) or 0
// where that is NaN.  One CTA: each thread sums a fixed strided subset in double, then a fixed tree - the same inputs
// give the same bits, with no atomics and no second launch.  The op reads 4 (n + m) bytes, well under a megabyte for
// the clouds of one range image, so one SM streams it in microseconds.
__global__ void __launch_bounds__(CV_RED_NT) k_point_metrics(const float* __restrict__ d1, uint32_t n, const float* __restrict__ d2,
                                                             uint32_t m, float thr, float* __restrict__ out) {
  __shared__ double s_sum[2][CV_RED_NT / 32];
  __shared__ uint32_t s_cnt[2][CV_RED_NT / 32];
  double s1 = 0.0, s2 = 0.0;
  uint32_t c1 = 0, c2 = 0;
  for (uint32_t i = threadIdx.x; i < n; i += CV_RED_NT) {
    const float v = d1[i];
    s1 += (double)v;
    c1 += v < thr ? 1u : 0u;
  }
  for (uint32_t i = threadIdx.x; i < m; i += CV_RED_NT) {
    const float v = d2[i];
    s2 += (double)v;
    c2 += v < thr ? 1u : 0u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_down_sync(0xffffffffu, s1, o);
    s2 += __shfl_down_sync(0xffffffffu, s2, o);
    c1 += __shfl_down_sync(0xffffffffu, c1, o);
    c2 += __shfl_down_sync(0xffffffffu, c2, o);
  }
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_sum[0][warp] = s1; s_sum[1][warp] = s2;
    s_cnt[0][warp] = c1; s_cnt[1][warp] = c2;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double t1 = 0.0, t2 = 0.0;
  uint32_t k1 = 0, k2 = 0;
  for (int w = 0; w < CV_RED_NT / 32; ++w) {
    t1 += s_sum[0][w]; t2 += s_sum[1][w];
    k1 += s_cnt[0][w]; k2 += s_cnt[1][w];
  }
  const float p1 = __fdiv_rn((float)k1, (float)n), p2 = __fdiv_rn((float)k2, (float)m);
  float f = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, p1), p2), __fadd_rn(p1, p2));
  if (f != f) f = 0.f;                           // metrics.py:26
  out[0] = (float)(t1 / (double)n + t2 / (double)m);
  out[1] = f;
  out[2] = p1;
  out[3] = p2;
  out[4] = 0.f;
}

static int check_image(uint32_t H, uint32_t W, const char* who) {
  if (H == 0 || W == 0 || (uint64_t)H * W > CV_MAX_PIXELS) return l4d_fail(L4D_EINVAL, "%s: H and W must be >= 1 with H*W <= 2^31", who);
  return L4D_OK;
}

static int cv_grid(size_t work) {
  size_t g = (work + CV_NT - 1) / CV_NT;
  const size_t cap = (size_t)16 * sm_count();       // a full SM of 128-thread CTAs; the loops stride over the rest
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

}  // namespace l4d_convert
using namespace l4d_convert;

extern "C" size_t l4d_pano_project_work_bytes(uint32_t H, uint32_t W) {
  return (size_t)H * W * (sizeof(unsigned long long) + sizeof(uint32_t));
}

extern "C" int l4d_pano_project(const float* points, uint32_t n, uint32_t stride, double fov_up, double fov, uint32_t H, uint32_t W,
                                float max_depth, float* pano, float* intensities_or_null, void* work, size_t work_bytes, void* stream) {
  if (check_image(H, W, "l4d_pano_project") != L4D_OK) return L4D_EINVAL;
  if (stride != 3 && stride != 4) return l4d_fail(L4D_EINVAL, "l4d_pano_project: stride must be 3 or 4");
  if (!pano || (n && !points)) return l4d_fail(L4D_EINVAL, "l4d_pano_project: null pointer");
  if (!work || work_bytes < l4d_pano_project_work_bytes(H, W)) return l4d_fail(L4D_ESIZE, "l4d_pano_project: work buffer too small");
  const size_t hw = (size_t)H * W;
  ProjectArgs A;
  A.pts = points; A.n = n; A.stride = stride; A.H = H; A.W = W;
  // the reference's constants, evaluated in double as Python does and rounded once to float32 where they meet a float32
  A.pi = (float)M_PI;
  A.alpha_off = (float)((fov - fov_up) / 180.0 * M_PI);
  A.c_scale = (float)(2.0 * M_PI / W);
  A.r_scale = (float)(fov / 180.0 * M_PI / H);
  A.Hf = (float)H;
  A.max_depth = max_depth;
  A.keys = reinterpret_cast<unsigned long long*>(work);
  A.zlast = reinterpret_cast<uint32_t*>(A.keys + hw);
  A.pano = pano; A.inten = intensities_or_null;
  cudaStream_t st = (cudaStream_t)stream;
  L4D_CUDA(cudaMemsetAsync(A.keys, 0xff, hw * sizeof(unsigned long long), st));
  L4D_CUDA(cudaMemsetAsync(A.zlast, 0, hw * sizeof(uint32_t), st));
  if (n) {
    ++g_launches; k_pano_project<0><<<cv_grid(n), CV_NT, 0, st>>>(A);
    ++g_launches; k_pano_project<1><<<cv_grid(n), CV_NT, 0, st>>>(A);
  }
  ++g_launches; k_pano_project<2><<<cv_grid(hw), CV_NT, 0, st>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_pano_unproject_work_bytes(uint32_t H, uint32_t W) {
  return ((size_t)H * W + CV_TILE - 1) / CV_TILE * sizeof(uint32_t);
}

extern "C" int l4d_pano_unproject(const float* pano, const float* intensities_or_null, uint32_t H, uint32_t W, float fov_up, float fov,
                                  float* out, uint32_t* count, void* work, size_t work_bytes, void* stream) {
  if (check_image(H, W, "l4d_pano_unproject") != L4D_OK) return L4D_EINVAL;
  if (!pano || !out || !count) return l4d_fail(L4D_EINVAL, "l4d_pano_unproject: null pointer");
  if (!work || work_bytes < l4d_pano_unproject_work_bytes(H, W)) return l4d_fail(L4D_ESIZE, "l4d_pano_unproject: work buffer too small");
  UnprojectArgs A;
  A.pano = pano; A.inten = intensities_or_null; A.H = H; A.W = W;
  A.fov_up = fov_up; A.fov = fov; A.pi = (float)M_PI;
  A.n_tiles = (uint32_t)(((size_t)H * W + CV_TILE - 1) / CV_TILE);
  A.offsets = reinterpret_cast<uint32_t*>(work);
  A.out = out; A.count = count;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = cv_grid((size_t)A.n_tiles * CV_NT);
  ++g_launches; k_pano_unproject<0><<<grid, CV_NT, 0, st>>>(A);
  ++g_launches; k_pano_unproject<1><<<1, CV_NT, 0, st>>>(A);
  ++g_launches; k_pano_unproject<2><<<grid, CV_NT, 0, st>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_point_metrics(const float* dist1, uint32_t n, const float* dist2, uint32_t m, float thr, float* out, void* stream) {
  if (!dist1 || !dist2 || !out) return l4d_fail(L4D_EINVAL, "l4d_point_metrics: null pointer");
  if (n == 0 || m == 0) return l4d_fail(L4D_EINVAL, "l4d_point_metrics: empty point cloud");
  ++g_launches; k_point_metrics<<<1, CV_RED_NT, 0, (cudaStream_t)stream>>>(dist1, n, dist2, m, thr, out);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}
