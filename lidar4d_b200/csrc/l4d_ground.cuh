// l4d_ground.cuh - the flow loss's point-cloud preparation (utils/misc.py point_removal, model/runner.py
// process_pointcloud) as sm_90a kernels:
//   k_range_filter_*     range_filter (misc.py:116-125): cv_compact over the points, float32 mask op by op
//   k_knn_mean_dist      the mean distance to the k <= 64 nearest points (the point itself included), exact, float64:
//                        the first half of Open3D's PointCloud::RemoveStatisticalOutliers
//   k_outlier_stats      one CTA: cloud mean and standard deviation of those means, fixed-order float64 reduction
//   k_outlier_select_*   the other half: keep avg > 0 && avg < mean + ratio * std, cv_compact
//   k_plane_scores       inlier counts of a batch of RANSAC plane hypotheses (misc.py:90-93)
//   k_plane_mask         OR the inlier mask of one hypothesis into a byte mask (the union of the six my_ransac calls)
//   k_ground_split_*     ground = mask && z < z_max, the rest, each in index order (cv_compact twice)
//   k_pose_transform     (pose @ [scale * p, 1]^T)^T[:, :3] in float64 (runner.py:940-946)
// (included at the end of l4d_kernels.cu, after l4d_convert.cuh whose cv_compact and cv_grid it uses)
//
// k-NN design.  Brute force, 128 queries per CTA (one per thread), candidates streamed through shared memory in tiles
// of GR_TILE points as float32.  Each thread keeps a max-heap of its k smallest float64 squared distances in shared
// memory; a candidate is screened in float32 against the heap's top widened by a margin that covers every float32
// rounding (see gr_bound), and only a candidate that passes is recomputed in float64 from global memory, in nanoflann's
// L2_Adaptor order ((dx*dx) + dy*dy) + dz*dz, and pushed if it beats the top.  So the selection is exact: the heap ends
// holding the k smallest float64 squared distances (which of several equal k-th distances is kept does not change the
// sum).  The scan of a query block starts at the tile that holds it and wraps around: scan order follows the sensor's
// row-major order, so the nearby points come first, the bound tightens at once and few later candidates pass the screen.
// A uniform grid would do less arithmetic on even clouds, but a LiDAR sweep's density spans orders of magnitude
// from 1 m to 50 m and the duplicate clusters of real scans defeat any fixed cell size; the brute-force scan has no
// worst case beyond its n^2 float32 screens (4.6e9 for a 67,980-point sweep).
#pragma once

namespace l4d_ground {

constexpr int GR_KNN_NT = 128;                // queries per k-NN CTA
constexpr int GR_MAXK = 64;
constexpr int GR_TILE = 512;                  // candidates per shared-memory tile
constexpr size_t GR_KNN_SMEM = (size_t)GR_MAXK * GR_KNN_NT * sizeof(double) + (size_t)GR_TILE * sizeof(float4);
constexpr uint32_t GR_MAX_POINTS = 0x7fffffffu;

// --- range filter -------------------------------------------------------------------------------------------------
struct RangeFilterOp {
  const float* pts;           // [n, stride]
  uint32_t stride;
  float dist_min, dist_max, z_lo, z_hi;
  float* out;                 // [n, stride]

  __device__ __forceinline__ bool keep(size_t q) const {
    const float* p = pts + q * stride;
    const float x = p[0], y = p[1], z = p[2];
    // np.sqrt(np.sum(p**2, axis=1)): the array square is x*x, the 3-term row sum runs left to right
    const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    const bool ego = x > -2.f && x < 2.f && y > -1.f && y < 1.f && z > -2.f && z < 2.f;
    return d >= dist_min && d <= dist_max && z > z_lo && z < z_hi && !ego;
  }
  __device__ __forceinline__ void emit(size_t q, uint32_t pos) const {
    for (uint32_t c = 0; c < stride; ++c) out[(size_t)pos * stride + c] = pts[q * stride + c];
  }
};

template <int PASS>
__global__ void __launch_bounds__(CV_NT) k_range_filter(const RangeFilterOp op, uint32_t n, uint32_t n_tiles, uint32_t* offsets,
                                                         uint32_t* count) {
  cv_compact<RangeFilterOp, PASS>(op, n, n_tiles, offsets, count);
}

// --- exact k-NN mean distance ---------------------------------------------------------------------------------------
// The float32 screen admits a candidate iff fl32(|c - q|^2) <= gr_bound(top, M), where top is the heap's largest float64
// squared distance and M bounds |coordinate| of the query and the tile.  With u = 2^-24, rounding the coordinates to
// float32 and subtracting moves the difference vector by at most 3.5 u M + u |d|, and the FMA sum of squares adds a
// relative 3.01 u; so every candidate with |d| <= t = sqrt(top) has fl32(|d|^2) <= (t (1 + u) + 3.5 u M)^2 (1 + 3.01 u).
// The bound uses 2^-20 = 16 u in place of each of those factors and rounds up to float32.
__device__ __forceinline__ float gr_bound(double top, float M) {
  if (!(top < INFINITY)) return INFINITY;
  const double e = 0x1p-20;
  const double t = sqrt(top) * (1.0 + e) + e * (double)M;
  return __double2float_ru(t * t * (1.0 + e));
}

__global__ void __launch_bounds__(GR_KNN_NT) k_knn_mean_dist(const double* __restrict__ pts, uint32_t n, uint32_t k,
                                                             double* __restrict__ avg) {
  extern __shared__ __align__(16) unsigned char gr_smem[];
  double* heap = reinterpret_cast<double*>(gr_smem);                     // heap[s * GR_KNN_NT + tid]
  float4* tile = reinterpret_cast<float4*>(heap + GR_MAXK * GR_KNN_NT);   // x, y, z, max |coordinate| of the point
  __shared__ float s_tmax[GR_KNN_NT / 32];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t K = k < n ? k : n;
  const uint32_t n_blocks = (n + GR_KNN_NT - 1) / GR_KNN_NT, n_tiles = (n + GR_TILE - 1) / GR_TILE;
  double* H = heap + tid;
#define GR_H(s) H[(size_t)(s) * GR_KNN_NT]
  for (uint32_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const uint32_t i = blk * GR_KNN_NT + tid;
    const bool active = i < n;
    double qx = 0.0, qy = 0.0, qz = 0.0;
    if (active) { qx = pts[(size_t)i * 3]; qy = pts[(size_t)i * 3 + 1]; qz = pts[(size_t)i * 3 + 2]; }
    const float fx = (float)qx, fy = (float)qy, fz = (float)qz;
    const float Mq = fmaxf(fabsf(fx), fmaxf(fabsf(fy), fabsf(fz)));
    for (uint32_t s = 0; s < K; ++s) GR_H(s) = INFINITY;
    double top = INFINITY;
    const uint32_t t0 = (blk * GR_KNN_NT) / GR_TILE;
    for (uint32_t tt = 0; tt < n_tiles; ++tt) {
      uint32_t t = t0 + tt;
      if (t >= n_tiles) t -= n_tiles;
      const uint32_t base = t * GR_TILE;
      const uint32_t cnt = n - base < (uint32_t)GR_TILE ? n - base : (uint32_t)GR_TILE;
      __syncthreads();                                   // the previous tile is no longer read
      float m = 0.f;
      for (uint32_t j = tid; j < cnt; j += GR_KNN_NT) {
        const double* p = pts + (size_t)(base + j) * 3;
        const float x = (float)p[0], y = (float)p[1], z = (float)p[2];
        const float a = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
        tile[j] = make_float4(x, y, z, a);
        m = fmaxf(m, a);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) s_tmax[warp] = m;
      __syncthreads();
      float M = Mq;
      for (int w = 0; w < GR_KNN_NT / 32; ++w) M = fmaxf(M, s_tmax[w]);
      if (!active) continue;
      float T = gr_bound(top, M);
      for (uint32_t j = 0; j < cnt; ++j) {
        const float4 c = tile[j];
        const float dx = c.x - fx, dy = c.y - fy, dz = c.z - fz;
        const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        if (!(d2 <= T)) continue;                        // NaN never passes
        const double* p = pts + (size_t)(base + j) * 3;
        const double ex = __dsub_rn(p[0], qx), ey = __dsub_rn(p[1], qy), ez = __dsub_rn(p[2], qz);
        const double e2 = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
        if (!(e2 < top)) continue;
        uint32_t pos = 0;                                // replace the root, sift down
        for (;;) {
          uint32_t ch = 2 * pos + 1;
          if (ch >= K) break;
          double cv = GR_H(ch);
          if (ch + 1 < K) {
            const double c2 = GR_H(ch + 1);
            if (c2 > cv) { ++ch; cv = c2; }
          }
          if (!(cv > e2)) break;
          GR_H(pos) = cv;
          pos = ch;
        }
        GR_H(pos) = e2;
        top = GR_H(0);
        T = gr_bound(top, M);
      }
    }
    if (active) {
      for (uint32_t end = K - 1; end > 0; --end) {      // heapsort: the K distances in ascending order
        const double v = GR_H(end);
        GR_H(end) = GR_H(0);
        uint32_t pos = 0;
        for (;;) {
          uint32_t ch = 2 * pos + 1;
          if (ch >= end) break;
          double cv = GR_H(ch);
          if (ch + 1 < end) {
            const double c2 = GR_H(ch + 1);
            if (c2 > cv) { ++ch; cv = c2; }
          }
          if (!(cv > v)) break;
          GR_H(pos) = cv;
          pos = ch;
        }
        GR_H(pos) = v;
      }
      double s = 0.0;                                    // std::accumulate(sqrt(d), 0.0) / k, ascending
      for (uint32_t j = 0; j < K; ++j) s = __dadd_rn(s, __dsqrt_rn(GR_H(j)));
      avg[i] = __ddiv_rn(s, (double)K);
    }
  }
#undef GR_H
}

// --- outlier statistics and selection -------------------------------------------------------------------------------
// Open3D: n_valid counts every point whose neighbour search returned anything - all n of them; a point with avg = 0
// (all its neighbours are duplicates of it) adds nothing to either sum but still counts.
//   mean = sum_{avg > 0} avg / n_valid,  std = sqrt(sum_{avg > 0} (avg - mean)^2 / (n_valid - 1))
//   stats = {mean + ratio * std, mean, std}
// Each thread sums a fixed strided subset in order, then a fixed shuffle tree and a sequential sum over the warps: the
// same inputs give the same bits.
__device__ __forceinline__ double gr_block_sum(double v, double* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31u) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < CV_RED_NT / 32; ++w) t = __dadd_rn(t, s_red[w]);
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(CV_RED_NT) k_outlier_stats(const double* __restrict__ avg, uint32_t n, double ratio,
                                                             double* __restrict__ stats) {
  __shared__ double s_red[CV_RED_NT / 32];
  double s = 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += CV_RED_NT) {
    const double a = avg[i];
    if (a > 0.0) s = __dadd_rn(s, a);
  }
  const double mean = __ddiv_rn(gr_block_sum(s, s_red), (double)n);
  double q = 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += CV_RED_NT) {
    const double a = avg[i];
    if (a > 0.0) {
      const double d = __dsub_rn(a, mean);
      q = __dadd_rn(q, __dmul_rn(d, d));
    }
  }
  const double sq = gr_block_sum(q, s_red);
  if (threadIdx.x == 0) {
    const double sd = __dsqrt_rn(__ddiv_rn(sq, (double)n - 1.0));
    stats[0] = __dadd_rn(mean, __dmul_rn(ratio, sd));
    stats[1] = mean;
    stats[2] = sd;
  }
}

struct SelectOp {
  const double* pts;          // [n, 3]
  const double* avg;          // [n]
  const double* thr;          // device scalar (k_outlier_stats)
  double* out;                // [n, 3]
  int32_t* idx;               // [n] or nullptr

  __device__ __forceinline__ bool keep(size_t q) const {
    const double a = avg[q];
    return a > 0.0 && a < *thr;
  }
  __device__ __forceinline__ void emit(size_t q, uint32_t pos) const {
    for (int c = 0; c < 3; ++c) out[(size_t)pos * 3 + c] = pts[q * 3 + c];
    if (idx) idx[pos] = (int32_t)q;
  }
};

template <int PASS>
__global__ void __launch_bounds__(CV_NT) k_outlier_select(const SelectOp op, uint32_t n, uint32_t n_tiles, uint32_t* offsets,
                                                           uint32_t* count) {
  cv_compact<SelectOp, PASS>(op, n, n_tiles, offsets, count);
}

// --- RANSAC plane scoring -------------------------------------------------------------------------------------------
// |((a x + b y) + c z) + d| / r < thr in float64, every operation rounded on its own (no FMA), as NumPy evaluates
// np.abs(np.matmul(coeffs[:3], data.T) + coeffs[3]) / r < thr term by term
__device__ __forceinline__ bool gr_inlier(const double* h, double x, double y, double z, double thr) {
  const double e = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(h[0], x), __dmul_rn(h[1], y)), __dmul_rn(h[2], z)), h[3]);
  return __ddiv_rn(fabs(e), h[4]) < thr;
}

// counts[h] += inliers of hypothesis h (a, b, c, d, r) among this CTA's points: one warp sum and one atomic per warp and
// hypothesis (integer sums: the order does not matter)
__global__ void __launch_bounds__(CV_NT) k_plane_scores(const double* __restrict__ pts, uint32_t n, const double* __restrict__ hyp,
                                                        uint32_t M, double thr, uint32_t* __restrict__ counts) {
  const uint32_t lane = threadIdx.x & 31u;
  for (size_t base = (size_t)blockIdx.x * CV_NT; base < n; base += (size_t)gridDim.x * CV_NT) {
    const size_t i = base + threadIdx.x;
    const bool in = i < n;
    double x = 0.0, y = 0.0, z = 0.0;
    if (in) { x = pts[i * 3]; y = pts[i * 3 + 1]; z = pts[i * 3 + 2]; }
    for (uint32_t h = 0; h < M; ++h) {
      const bool hit = in && gr_inlier(hyp + (size_t)h * 5, x, y, z, thr);
      const uint32_t c = __popc(__ballot_sync(0xffffffffu, hit));
      if (lane == 0 && c) atomicAdd(counts + h, c);
    }
  }
}

struct PlaneArgs { double h[5]; };

__global__ void __launch_bounds__(CV_NT) k_plane_mask(const double* __restrict__ pts, uint32_t n, const PlaneArgs P, double thr,
                                                      uint8_t* __restrict__ mask) {
  for (size_t i = (size_t)blockIdx.x * CV_NT + threadIdx.x; i < n; i += (size_t)gridDim.x * CV_NT)
    if (gr_inlier(P.h, pts[i * 3], pts[i * 3 + 1], pts[i * 3 + 2], thr)) mask[i] = 1;
}

// --- ground split and pose ------------------------------------------------------------------------------------------
struct SplitOp {
  const double* pts;          // [n, 3]
  const uint8_t* mask;        // [n]
  double z_max;
  bool ground;                // true: mask && z < z_max; false: the complement
  double* out;                // [n, 3]
  int32_t* idx;               // [n] or nullptr

  __device__ __forceinline__ bool keep(size_t q) const {
    return (mask[q] != 0 && pts[q * 3 + 2] < z_max) == ground;
  }
  __device__ __forceinline__ void emit(size_t q, uint32_t pos) const {
    for (int c = 0; c < 3; ++c) out[(size_t)pos * 3 + c] = pts[q * 3 + c];
    if (idx) idx[pos] = (int32_t)q;
  }
};

template <int PASS>
__global__ void __launch_bounds__(CV_NT) k_ground_split(const SplitOp op, uint32_t n, uint32_t n_tiles, uint32_t* offsets,
                                                        uint32_t* count) {
  cv_compact<SplitOp, PASS>(op, n, n_tiles, offsets, count);
}

struct PoseArgs { double pose[12]; double scale; };   // the top 3 rows of a float32 4x4 pose, widened

// out_r = ((p_r0 X + p_r1 Y) + p_r2 Z) + p_r3 with (X, Y, Z) = scale * p: NumPy's float64 (pose @ [X, 1]^T)^T
__global__ void __launch_bounds__(CV_NT) k_pose_transform(const double* __restrict__ pts, uint32_t n, const PoseArgs P,
                                                          double* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * CV_NT + threadIdx.x; i < n; i += (size_t)gridDim.x * CV_NT) {
    const double X = __dmul_rn(pts[i * 3], P.scale), Y = __dmul_rn(pts[i * 3 + 1], P.scale), Z = __dmul_rn(pts[i * 3 + 2], P.scale);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const double* p = P.pose + 4 * r;
      out[i * 3 + r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], X), __dmul_rn(p[1], Y)), __dmul_rn(p[2], Z)), p[3]);
    }
  }
}

static int gr_check_n(uint32_t n, const char* who) {
  if (n == 0 || n > GR_MAX_POINTS) return l4d_fail(L4D_EINVAL, "%s: n must be in [1, 2^31)", who);
  return L4D_OK;
}

static uint32_t gr_tiles(uint32_t n) { return (uint32_t)(((size_t)n + CV_TILE - 1) / CV_TILE); }

}  // namespace l4d_ground
using namespace l4d_ground;

// the three launches of one cv_compact over N elements
#define GR_COMPACT(KERNEL, OP, N, OFFSETS, COUNT, ST)                                                               \
  do {                                                                                                              \
    const uint32_t nt_ = gr_tiles(N);                                                                               \
    const int g_ = cv_grid((size_t)nt_ * CV_NT);                                                                    \
    ++g_launches; KERNEL<0><<<g_, CV_NT, 0, ST>>>(OP, N, nt_, OFFSETS, COUNT);                                      \
    ++g_launches; KERNEL<1><<<1, CV_NT, 0, ST>>>(OP, N, nt_, OFFSETS, COUNT);                                       \
    ++g_launches; KERNEL<2><<<g_, CV_NT, 0, ST>>>(OP, N, nt_, OFFSETS, COUNT);                                      \
  } while (0)

static size_t gr_compact_bytes(uint32_t n) { return (size_t)gr_tiles(n) * sizeof(uint32_t); }

extern "C" size_t l4d_range_filter_work_bytes(uint32_t n) { return gr_compact_bytes(n); }

extern "C" int l4d_range_filter(const float* points, uint32_t n, uint32_t stride, float dist_min, float dist_max, float z_lo,
                                float z_hi, float* out, uint32_t* count, void* work, size_t work_bytes, void* stream) {
  if (gr_check_n(n, "l4d_range_filter") != L4D_OK) return L4D_EINVAL;
  if (stride < 3) return l4d_fail(L4D_EINVAL, "l4d_range_filter: stride must be >= 3");
  if (!points || !out || !count) return l4d_fail(L4D_EINVAL, "l4d_range_filter: null pointer");
  if (!work || work_bytes < l4d_range_filter_work_bytes(n)) return l4d_fail(L4D_ESIZE, "l4d_range_filter: work buffer too small");
  RangeFilterOp op{points, stride, dist_min, dist_max, z_lo, z_hi, out};
  GR_COMPACT(k_range_filter, op, n, reinterpret_cast<uint32_t*>(work), count, (cudaStream_t)stream);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_knn_mean_dist(const double* points, uint32_t n, uint32_t k, double* avg, void* stream) {
  if (gr_check_n(n, "l4d_knn_mean_dist") != L4D_OK) return L4D_EINVAL;
  if (k == 0 || k > GR_MAXK) return l4d_fail(L4D_EINVAL, "l4d_knn_mean_dist: k must be in [1, 64]");
  if (!points || !avg) return l4d_fail(L4D_EINVAL, "l4d_knn_mean_dist: null pointer");
  L4D_CUDA(cudaFuncSetAttribute(k_knn_mean_dist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GR_KNN_SMEM));
  int per_sm = 0;
  L4D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_knn_mean_dist, GR_KNN_NT, GR_KNN_SMEM));
  const size_t blocks = ((size_t)n + GR_KNN_NT - 1) / GR_KNN_NT;
  size_t grid = (size_t)(per_sm > 0 ? per_sm : 1) * sm_count();
  if (grid > blocks) grid = blocks;
  ++g_launches; k_knn_mean_dist<<<(int)grid, GR_KNN_NT, GR_KNN_SMEM, (cudaStream_t)stream>>>(points, n, k, avg);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_outlier_select_work_bytes(uint32_t n) { return 4 * sizeof(double) + gr_compact_bytes(n); }

extern "C" int l4d_outlier_select(const double* points, uint32_t n, const double* avg, double std_ratio, double* out,
                                  int32_t* index_or_null, uint32_t* count, double* stats_or_null, void* work, size_t work_bytes,
                                  void* stream) {
  if (gr_check_n(n, "l4d_outlier_select") != L4D_OK) return L4D_EINVAL;
  if (!points || !avg || !out || !count) return l4d_fail(L4D_EINVAL, "l4d_outlier_select: null pointer");
  if (!work || work_bytes < l4d_outlier_select_work_bytes(n)) return l4d_fail(L4D_ESIZE, "l4d_outlier_select: work buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  double* stats = stats_or_null ? stats_or_null : reinterpret_cast<double*>(work);
  uint32_t* offsets = reinterpret_cast<uint32_t*>(reinterpret_cast<double*>(work) + 4);
  ++g_launches; k_outlier_stats<<<1, CV_RED_NT, 0, st>>>(avg, n, std_ratio, stats);
  SelectOp op{points, avg, stats, out, index_or_null};
  GR_COMPACT(k_outlier_select, op, n, offsets, count, st);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_plane_scores(const double* points, uint32_t n, const double* hypotheses, uint32_t m, double threshold,
                                uint32_t* counts, void* stream) {
  if (gr_check_n(n, "l4d_plane_scores") != L4D_OK) return L4D_EINVAL;
  if (m == 0) return l4d_fail(L4D_EINVAL, "l4d_plane_scores: no hypotheses");
  if (!points || !hypotheses || !counts) return l4d_fail(L4D_EINVAL, "l4d_plane_scores: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  L4D_CUDA(cudaMemsetAsync(counts, 0, (size_t)m * sizeof(uint32_t), st));
  ++g_launches; k_plane_scores<<<cv_grid(n), CV_NT, 0, st>>>(points, n, hypotheses, m, threshold, counts);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_plane_mask(const double* points, uint32_t n, double a, double b, double c, double d, double r, double threshold,
                              uint8_t* mask, void* stream) {
  if (gr_check_n(n, "l4d_plane_mask") != L4D_OK) return L4D_EINVAL;
  if (!points || !mask) return l4d_fail(L4D_EINVAL, "l4d_plane_mask: null pointer");
  PlaneArgs P{{a, b, c, d, r}};
  ++g_launches; k_plane_mask<<<cv_grid(n), CV_NT, 0, (cudaStream_t)stream>>>(points, n, P, threshold, mask);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_ground_split_work_bytes(uint32_t n) { return gr_compact_bytes(n); }

extern "C" int l4d_ground_split(const double* points, uint32_t n, const uint8_t* mask, double z_max, double* ground,
                                int32_t* ground_index_or_null, double* rest, int32_t* rest_index_or_null, uint32_t* counts,
                                void* work, size_t work_bytes, void* stream) {
  if (gr_check_n(n, "l4d_ground_split") != L4D_OK) return L4D_EINVAL;
  if (!points || !mask || !ground || !rest || !counts) return l4d_fail(L4D_EINVAL, "l4d_ground_split: null pointer");
  if (!work || work_bytes < l4d_ground_split_work_bytes(n)) return l4d_fail(L4D_ESIZE, "l4d_ground_split: work buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint32_t* offsets = reinterpret_cast<uint32_t*>(work);
  const SplitOp g{points, mask, z_max, true, ground, ground_index_or_null};
  GR_COMPACT(k_ground_split, g, n, offsets, counts, st);
  const SplitOp r{points, mask, z_max, false, rest, rest_index_or_null};
  GR_COMPACT(k_ground_split, r, n, offsets, counts + 1, st);    // stream order: the offsets are free again
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_pose_transform(const double* points, uint32_t n, double scale, const float* pose, double* out, void* stream) {
  if (gr_check_n(n, "l4d_pose_transform") != L4D_OK) return L4D_EINVAL;
  if (!points || !pose || !out) return l4d_fail(L4D_EINVAL, "l4d_pose_transform: null pointer");
  PoseArgs P;
  for (int j = 0; j < 12; ++j) P.pose[j] = (double)pose[j];
  P.scale = scale;
  ++g_launches; k_pose_transform<<<cv_grid(n), CV_NT, 0, (cudaStream_t)stream>>>(points, n, P, out);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}
