// l4d_nngrid.cuh - exact nearest-neighbour search through a uniform grid, and the flow loss of train_step
// (model/runner.py:222-253) on top of it.
//
// The brute-force op (l4d_chamfer.cuh) is the right tool for the 1,024-point chamfer term and one-off metrics.  The flow
// loss searches, every optimiser step, clouds of 1e4..1e5 points that never change: they are indexed once.
//
// Index (l4d_nn_grid_build, five launches, no device-to-host read: every buffer size is a function of n alone):
//   k_nng_bbox      bounding box of the points whose three coordinates are finite, per-CTA partials; zeroes the counters
//   k_nng_geometry  one CTA: reduces the partials and picks the grid (nng_geometry): cubic cells of edge 1/ih, the finest
//                   of a fixed ladder whose cell count fits the budget l4d_nng_budget(n); writes the device header
//   k_nng_count     cell of every point (0xffffffff = left out: a non-finite point can never win a strict '<'), histogram
//   k_nng_scan      one CTA: exclusive scan of the histogram -> cell_start[cells + 1], and the scatter cursors
//   k_nng_scatter   points cell-sorted as 16-byte (x, y, z, original index) records through an atomic cursor
// Query (k_nng_query, thread == query): the shells of cells around the query's own (clamped) cell, outwards.  A row of a
// shell along x is one contiguous range of records.  Candidates are reduced on (distance, original index) - the
// brute-force op's 64-bit key order - so the result does not depend on the order of the records inside a cell.
//
// CONTRACT: dist and idx equal l4d_chamfer_forward's bit for bit.  The distance is the same chain,
// fma(dz,dz, fma(dx,dx, dy*dy)) with d = target - query, every operation rounded to nearest.
//
// Why the stopping rule is safe under rounding.  Write fl() for rounding to nearest; it is monotone.  Along one axis
//   u(x) = fl(fl(x - lo) * ih),   cell(x) = clamp(floor(u(x)), 0, dim - 1)
// for points and queries alike (nng_u, nng_cell); the cell edge is the real number 1/ih, so ih carries no error.
//  (1) An indexed point p with cell(p) >= k, 1 <= k <= dim-1, has u(p) >= k (the clamp from below yields 0 < k, the clamp
//      from above only lowers).  With tp = fl(p - lo) >= 0:  tp*ih*(1+d1) >= k and p - lo = tp/(1+d2), |d| <= 2^-24
//      (k >= 1: no underflow), hence p - lo >= (k/ih)(1 - 2^-22).
//      A point with cell(p) <= k, k <= dim-2, has u(p) < k+1 and likewise p - lo <= ((k+1)/ih)(1 + 2^-22)
//      (a product that underflows errs by 2^-150 at most, far inside the slack below).
//  (2) The query: tq = fl(q - lo) is finite (otherwise the whole cloud is scanned), so |(q - lo) - tq| <= 2^-23 |tq|.
//  (3) So for every point on the far side of the face k of shell r,
//        p - q >= k/ih - tq - 2^-22 (k/ih + |tq|)            (+ side, k = cq + r + 1)
//        q - p >= tq - (k+1)/ih - 2^-22 ((k+1)/ih + |tq|)    (- side, k = cq - r - 1)
//      nng_axis_gap evaluates the right-hand side in fp32 with k/ih as fl(k * h), h = fl(1/ih) (relative error 2^-23 of
//      k/ih, and 2^-24 of the difference), subtracts 2^-20 (k/ih + |tq|) and scales by 1 - 2^-20: more than twice the
//      error it has to absorb.  The result b >= 0 is an fp32 number below the real |p - q|, so the computed difference
//      fl(p - q) has |.| >= b, by monotonicity.
//  (4) In the chain every addend is >= 0 and fl is monotone: d >= fl(dx*dx), d >= fl(dy*dy), d >= fl(dz*dz), and
//      |dx| >= b gives fl(dx*dx) >= fl(b*b).
//  (5) A cell outside shells 0..r differs from the query's cell by more than r along at least one axis, so it lies
//      beyond one of the (at most six) faces: the minimum of fl(b*b) over the faces that exist is <= the computed
//      distance of every point in every unvisited cell.  No face left means no cell left.
// The walk goes on while bound <= best: an equal distance with a smaller index may lie outside.  After
// L4D_NNG_MAX_SHELLS shells the whole cloud is scanned (a far outlier is slow but right).  A query with a non-finite
// coordinate returns (+inf, 0), a cloud with no finite point returns that for every query: '<' on NaN / +inf in the
// brute-force op.  Every loop is bounded by the grid dimensions or the shell limit; every cell index is clamped.
//
// The geometry, the bound, the shell walk and the candidate loop are __host__ __device__: tests/hostsim/nngridsim.cu
// runs them on the CPU.  (included by l4d_kernels.cu: one translation unit, one shared library)
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "l4d_losses.cuh"     // l4d_block_sum, l4d_sgn

#define L4D_NNG_MAX_SHELLS 16
#define L4D_NNG_QT 64              // threads of a query CTA
#define L4D_NNG_BBOX_BLOCKS 256
#define L4D_NNG_LADDER 80          // cell edges tried: extent / 1024 * 1.1^i

struct __align__(16) L4DNNGHeader {
  float lo[3], ih;                 // box corner, 1 / cell edge
  float hi[3];
  uint32_t n_valid;                // points indexed (all three coordinates finite)
  uint32_t dim[3], cells;          // cells = dim[0] * dim[1] * dim[2] <= budget; x runs fastest
  float h;                         // fl(1 / ih), for the stopping bound only (a division per face would cost a call)
  uint32_t pad[3];
};

// cells the index of an n-point cloud may use: about four per point (a LiDAR sweep is far denser near the sensor than
// its box average, DESIGN.md 7)
inline uint32_t l4d_nng_budget(uint32_t n) {
  const uint64_t c = 4ull * n;
  return (uint32_t)(c < 64 ? 64 : (c > (1ull << 22) ? (1ull << 22) : c));
}
struct L4DNNGLayout { size_t start, pts, total; uint32_t budget; };       // the index: header | cell_start | records
struct L4DNNGWork { size_t bbox, cell_of, cursor, total; };               // build scratch
inline size_t l4d_nng_align(size_t v) { return (v + 255) / 256 * 256; }
inline L4DNNGLayout l4d_nng_layout(uint32_t n) {
  L4DNNGLayout L;
  L.budget = l4d_nng_budget(n);
  L.start = 256;
  L.pts = L.start + l4d_nng_align(((size_t)L.budget + 1) * sizeof(uint32_t));
  L.total = L.pts + l4d_nng_align((size_t)n * 16);
  return L;
}
inline L4DNNGWork l4d_nng_work(uint32_t n) {
  L4DNNGWork W;
  W.bbox = 0;
  W.cell_of = l4d_nng_align(L4D_NNG_BBOX_BLOCKS * 6 * sizeof(float));
  W.cursor = W.cell_of + l4d_nng_align((size_t)n * sizeof(uint32_t));
  W.total = W.cursor + l4d_nng_align((size_t)l4d_nng_budget(n) * sizeof(uint32_t));
  return W;
}

// fp32 operations rounded to nearest, one rounding each, whatever the compiler would like to contract
#ifdef __CUDA_ARCH__
__device__ __forceinline__ float nng_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float nng_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float nng_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float nng_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float nng_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ uint32_t nng_bits(float v) { return __float_as_uint(v); }
__device__ __forceinline__ float4 nng_load(const float4* p) { return __ldg(p); }
#else
inline float nng_add(float a, float b) { volatile float r = a + b; return r; }
inline float nng_sub(float a, float b) { volatile float r = a - b; return r; }
inline float nng_mul(float a, float b) { volatile float r = a * b; return r; }
inline float nng_div(float a, float b) { volatile float r = a / b; return r; }
inline float nng_fma(float a, float b, float c) { return fmaf(a, b, c); }
inline uint32_t nng_bits(float v) { uint32_t u; memcpy(&u, &v, 4); return u; }
inline float4 nng_load(const float4* p) { return *p; }
#endif
__host__ __device__ inline float nng_from_bits(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float v; memcpy(&v, &u, 4); return v;
#endif
}
__host__ __device__ inline bool nng_finite(float v) { return fabsf(v) <= 3.402823466e38f; }

__host__ __device__ inline float nng_u(float x, float lo, float ih) { return nng_mul(nng_sub(x, lo), ih); }
__host__ __device__ inline int nng_cell(float u, uint32_t dim) {        // NaN -> 0
  return (int)fminf(fmaxf(floorf(u), 0.f), (float)(dim - 1));
}

// the grid of a box lo..hi (of the finite points; lo > hi when there is none): one cell when the box is a point, is
// empty or its extent is outside [1e-30, 1e30]; otherwise the first edge of the ladder whose grid fits the budget.  The
// last edge is about twice the extent, which gives one cell: the loop always returns.
__host__ __device__ inline void nng_geometry(const float* lo, const float* hi, uint32_t budget, L4DNNGHeader* H) {
  const bool any = lo[0] <= hi[0] && lo[1] <= hi[1] && lo[2] <= hi[2];
  float E = 0.f;
  for (int a = 0; a < 3; ++a) {
    H->lo[a] = any ? lo[a] : 0.f;
    H->hi[a] = any ? hi[a] : 0.f;
    H->dim[a] = 1;
    E = fmaxf(E, nng_sub(H->hi[a], H->lo[a]));
  }
  H->ih = 1.f;
  H->h = 1.f;
  H->cells = 1;
  H->n_valid = 0;
  H->pad[0] = H->pad[1] = H->pad[2] = 0;
  if (!(E > 1e-30f && E < 1e30f)) return;
  float ih = nng_div(1024.f, E);
  for (int it = 0; it < L4D_NNG_LADDER; ++it) {
    uint32_t d[3];
    for (int a = 0; a < 3; ++a) d[a] = (uint32_t)nng_cell(nng_u(H->hi[a], H->lo[a], ih), 2048u) + 1u;
    const uint64_t cells = (uint64_t)d[0] * d[1] * d[2];
    if (cells <= budget) {
      H->ih = ih;
      H->h = nng_div(1.f, ih);
      H->cells = (uint32_t)cells;
      for (int a = 0; a < 3; ++a) H->dim[a] = d[a];
      return;
    }
    ih = nng_mul(ih, 0.90909088f);
  }
}

// the cell of a point, or 0xffffffff for a point that is left out
__host__ __device__ inline uint32_t nng_point_cell(const L4DNNGHeader& H, float x, float y, float z) {
  if (!(nng_finite(x) && nng_finite(y) && nng_finite(z))) return 0xffffffffu;
  const uint32_t cx = (uint32_t)nng_cell(nng_u(x, H.lo[0], H.ih), H.dim[0]);
  const uint32_t cy = (uint32_t)nng_cell(nng_u(y, H.lo[1], H.ih), H.dim[1]);
  const uint32_t cz = (uint32_t)nng_cell(nng_u(z, H.lo[2], H.ih), H.dim[2]);
  return (cz * H.dim[1] + cy) * H.dim[0] + cx;
}

// (3) of the header: a lower bound of |fl(p - q)| along one axis over the indexed points p with cell >= k (side > 0) or
// cell <= k (side < 0), for a query with tq = fl(q - lo)
__host__ __device__ __forceinline__ float nng_axis_gap(float tq, float h, int k, int side) {
  const float A = nng_mul((float)(side > 0 ? k : k + 1), h);
  const float g = side > 0 ? nng_sub(A, tq) : nng_sub(tq, A);
  const float slack = nng_mul(nng_add(A, fabsf(tq)), 9.5367431640625e-7f);          // 2^-20
  const float b = nng_mul(nng_sub(g, slack), 0.99999904632568359375f);              // 1 - 2^-20
  return b > 0.f ? b : 0.f;                                                          // NaN -> 0: keep searching
}

// (5): false when no cell lies outside shells 0..r; else *bound <= the computed distance of every point out there
__host__ __device__ __forceinline__ bool nng_shell_bound(const L4DNNGHeader& H, const float* tq, const int* cq, int r, float* bound) {
  float b2 = INFINITY;
  bool any = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int kp = cq[a] + r + 1, km = cq[a] - r - 1;
    if (kp <= (int)H.dim[a] - 1) {
      const float g = nng_axis_gap(tq[a], H.h, kp, +1);
      b2 = fminf(b2, nng_mul(g, g));
      any = true;
    }
    if (km >= 0) {
      const float g = nng_axis_gap(tq[a], H.h, km, -1);
      b2 = fminf(b2, nng_mul(g, g));
      any = true;
    }
  }
  *bound = b2;
  return any;
}

// records s..e against one query; returns the number examined
__host__ __device__ __forceinline__ uint32_t nng_scan(const float4* __restrict__ pts, uint32_t s, uint32_t e, float qx, float qy, float qz,
                                             float& best, uint32_t& bi) {
  for (uint32_t i = s; i < e; ++i) {
    const float4 p = nng_load(pts + i);
    const float dx = nng_sub(p.x, qx), dy = nng_sub(p.y, qy), dz = nng_sub(p.z, qz);
    const float d = nng_fma(dz, dz, nng_fma(dx, dx, nng_mul(dy, dy)));      // l4d_chamfer.cuh:87-93
    const uint32_t k = nng_bits(p.w);
    if (d < best || (d == best && k < bi)) { best = d; bi = k; }            // the order of (distance bits << 32 | index)
  }
  return e - s;
}

// shell r of the cells around cq, clipped to the grid: rows along x are contiguous ranges of records
__host__ __device__ __forceinline__ uint32_t nng_visit_shell(const L4DNNGHeader& H, const uint32_t* __restrict__ cs, const float4* __restrict__ pts,
                                                    const int* cq, int r, float qx, float qy, float qz, float& best, uint32_t& bi) {
  const int dx = (int)H.dim[0], dy = (int)H.dim[1], dz = (int)H.dim[2];
  const int z0 = cq[2] - r < 0 ? 0 : cq[2] - r, z1 = cq[2] + r > dz - 1 ? dz - 1 : cq[2] + r;
  const int y0 = cq[1] - r < 0 ? 0 : cq[1] - r, y1 = cq[1] + r > dy - 1 ? dy - 1 : cq[1] + r;
  const int x0 = cq[0] - r < 0 ? 0 : cq[0] - r, x1 = cq[0] + r > dx - 1 ? dx - 1 : cq[0] + r;
  uint32_t cand = 0;
  for (int z = z0; z <= z1; ++z)
    for (int y = y0; y <= y1; ++y) {
      const uint32_t base = (uint32_t)(z * dy + y) * (uint32_t)dx;
      const int az = z - cq[2], ay = y - cq[1];
      if (az == r || az == -r || ay == r || ay == -r) {
        cand += nng_scan(pts, cs[base + x0], cs[base + x1 + 1], qx, qy, qz, best, bi);
      } else {
        if (cq[0] - r >= 0) cand += nng_scan(pts, cs[base + cq[0] - r], cs[base + cq[0] - r + 1], qx, qy, qz, best, bi);
        if (cq[0] + r <= dx - 1) cand += nng_scan(pts, cs[base + cq[0] + r], cs[base + cq[0] + r + 1], qx, qy, qz, best, bi);
      }
    }
  return cand;
}

// one query: nearest indexed point as (distance, original index); returns the number of records examined
__host__ __device__ __forceinline__ uint32_t nng_query_one(const L4DNNGHeader& H, const uint32_t* __restrict__ cs, const float4* __restrict__ pts,
                                                  float qx, float qy, float qz, float* dist, uint32_t* idx) {
  float best = INFINITY;
  uint32_t bi = 0, cand = 0;
  const float q[3] = {qx, qy, qz};
  float tq[3];
  int cq[3];
  bool q_ok = true, t_ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    tq[a] = nng_sub(q[a], H.lo[a]);
    q_ok = q_ok && nng_finite(q[a]);
    t_ok = t_ok && nng_finite(tq[a]);
    cq[a] = nng_cell(nng_mul(tq[a], H.ih), H.dim[a]);
  }
  if (q_ok && H.n_valid) {
    bool done = false;
    for (int r = 0; t_ok && r <= L4D_NNG_MAX_SHELLS; ++r) {
      cand += nng_visit_shell(H, cs, pts, cq, r, qx, qy, qz, best, bi);
      float bound;
      if (!nng_shell_bound(H, tq, cq, r, &bound) || !(bound <= best)) { done = true; break; }
    }
    if (!done) cand += nng_scan(pts, 0, H.n_valid, qx, qy, qz, best, bi);
  }
  *dist = best;
  *idx = bi;
  return cand;
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------------------------
// index build
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_nng_bbox(const float* __restrict__ xyz, uint32_t n, float* __restrict__ part,
                                                  uint32_t* __restrict__ counts, uint32_t n_counts) {
  __shared__ float s[6][8];
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t i = t0; i < n_counts; i += stride) counts[i] = 0;
  float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (uint32_t i = t0; i < n; i += stride) {
    const float x = __ldg(xyz + 3 * (size_t)i), y = __ldg(xyz + 3 * (size_t)i + 1), z = __ldg(xyz + 3 * (size_t)i + 2);
    if (!(nng_finite(x) && nng_finite(y) && nng_finite(z))) continue;
    v[0] = fminf(v[0], x); v[1] = fminf(v[1], y); v[2] = fminf(v[2], z);
    v[3] = fmaxf(v[3], x); v[4] = fmaxf(v[4], y); v[5] = fmaxf(v[5], z);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, v[k], o);
      v[k] = k < 3 ? fminf(v[k], w) : fmaxf(v[k], w);
    }
    if (lane == 0) s[k][warp] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    const int k = threadIdx.x;
    float r = s[k][0];
    for (int w = 1; w < 8; ++w) r = k < 3 ? fminf(r, s[k][w]) : fmaxf(r, s[k][w]);
    part[6 * blockIdx.x + k] = r;
  }
}

__global__ void __launch_bounds__(32) k_nng_geometry(const float* __restrict__ part, uint32_t n_part, uint32_t budget,
                                                     L4DNNGHeader* __restrict__ H) {
  float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (uint32_t b = threadIdx.x; b < n_part; b += 32)
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = k < 3 ? fminf(v[k], part[6 * b + k]) : fmaxf(v[k], part[6 * b + k]);
#pragma unroll
  for (int k = 0; k < 6; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, v[k], o);
      v[k] = k < 3 ? fminf(v[k], w) : fmaxf(v[k], w);
    }
  if (threadIdx.x == 0) {
    L4DNNGHeader h;
    nng_geometry(v, v + 3, budget, &h);
    h.n_valid = 0;                       // k_nng_scan writes it
    *H = h;
  }
}

__global__ void __launch_bounds__(256) k_nng_count(const float* __restrict__ xyz, uint32_t n, const L4DNNGHeader* __restrict__ Hp,
                                                   uint32_t* __restrict__ cell_of, uint32_t* __restrict__ counts) {
  const L4DNNGHeader H = *Hp;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c = nng_point_cell(H, __ldg(xyz + 3 * (size_t)i), __ldg(xyz + 3 * (size_t)i + 1), __ldg(xyz + 3 * (size_t)i + 2));
    cell_of[i] = c;
    if (c != 0xffffffffu) atomicAdd(counts + c, 1u);
  }
}

// one CTA of 1024 threads, a contiguous chunk of cells per thread: counts -> exclusive starts in place, start[cells] =
// the number of indexed points, cursor = a copy for the scatter
__global__ void __launch_bounds__(1024) k_nng_scan(L4DNNGHeader* __restrict__ H, uint32_t* __restrict__ start, uint32_t* __restrict__ cursor) {
  __shared__ uint32_t s_warp[32];
  const uint32_t cells = H->cells;
  const uint32_t chunk = (cells + 1023u) / 1024u;
  const uint32_t a = min(cells, threadIdx.x * chunk), b = min(cells, a + chunk);
  uint32_t sum = 0;
  for (uint32_t i = a; i < b; ++i) sum += start[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t w = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += w;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  uint32_t run = inc - sum + (warp ? s_warp[warp - 1] : 0u);
  for (uint32_t i = a; i < b; ++i) {
    const uint32_t c = start[i];
    start[i] = run;
    cursor[i] = run;
    run += c;
  }
  if (threadIdx.x == 1023) {
    start[cells] = s_warp[31];
    H->n_valid = s_warp[31];
  }
}

__global__ void __launch_bounds__(256) k_nng_scatter(const float* __restrict__ xyz, uint32_t n, const uint32_t* __restrict__ cell_of,
                                                     uint32_t* __restrict__ cursor, float4* __restrict__ pts) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c = cell_of[i];
    if (c == 0xffffffffu) continue;
    const uint32_t pos = atomicAdd(cursor + c, 1u);
    pts[pos] = make_float4(__ldg(xyz + 3 * (size_t)i), __ldg(xyz + 3 * (size_t)i + 1), __ldg(xyz + 3 * (size_t)i + 2), __uint_as_float(i));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// query.  WARP: the query is pc[j] + flow6[j, col..col+2] * step, written to warped[j] (one flow-loss term's forward).
// parts != nullptr: the CTA's sum of distances, in double and in a fixed order, goes to parts[blockIdx.x].
// ------------------------------------------------------------------------------------------------------------------
template <bool WARP>
__global__ void __launch_bounds__(L4D_NNG_QT, 1) k_nng_query(const unsigned char* __restrict__ grid, L4DNNGLayout L, const float* __restrict__ q,
                                                          const float* __restrict__ flow6, uint32_t col, float step,
                                                          float* __restrict__ warped, uint32_t nq, float* __restrict__ dist,
                                                          int* __restrict__ idx, double* __restrict__ parts) {
  __shared__ double s_red[1][L4D_NNG_QT / 32];
  const L4DNNGHeader H = *reinterpret_cast<const L4DNNGHeader*>(grid);
  const uint32_t* cs = reinterpret_cast<const uint32_t*>(grid + L.start);
  const float4* pts = reinterpret_cast<const float4*>(grid + L.pts);
  double acc = 0;
  for (uint32_t j = blockIdx.x * L4D_NNG_QT + threadIdx.x; j < nq; j += gridDim.x * L4D_NNG_QT) {
    float x = __ldg(q + 3 * (size_t)j), y = __ldg(q + 3 * (size_t)j + 1), z = __ldg(q + 3 * (size_t)j + 2);
    if (WARP) {       // pc + flow * step as ATen evaluates it: the product, then the sum
      const float* f = flow6 + 6 * (size_t)j + col;
      x = nng_add(x, nng_mul(__ldg(f), step));
      y = nng_add(y, nng_mul(__ldg(f + 1), step));
      z = nng_add(z, nng_mul(__ldg(f + 2), step));
      warped[3 * (size_t)j] = x; warped[3 * (size_t)j + 1] = y; warped[3 * (size_t)j + 2] = z;
    }
    float d;
    uint32_t k;
    nng_query_one(H, cs, pts, x, y, z, &d, &k);
    if (dist) dist[j] = d;
    idx[j] = (int)k;
    acc += d;
  }
  if (parts) {
    double v[1] = {acc};
    l4d_block_sum<L4D_NNG_QT, 1>(v, s_red);
    if (threadIdx.x == 0) parts[blockIdx.x] = v[0];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// flow loss: the zero-flow term of the ground points, the final sum, and the backward launches
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_flow_ground(const float* __restrict__ f, uint32_t total, double* __restrict__ parts) {
  __shared__ double s_red[1][8];
  double v[1] = {0};
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) v[0] += fabsf(f[i]);
  l4d_block_sum<256, 1>(v, s_red);
  if (threadIdx.x == 0) parts[blockIdx.x] = v[0];
}

// loss = 0.5 * (sum of the chamfer partials) + 0.001 * (sum of the ground partials), one CTA, fixed order
__global__ void __launch_bounds__(1024) k_flow_finish(const double* __restrict__ parts, uint32_t n_chamfer, uint32_t n_ground,
                                                      float* __restrict__ loss) {
  __shared__ double s_red[2][32];
  double v[2] = {0, 0};
  for (uint32_t i = threadIdx.x; i < n_chamfer; i += 1024) v[0] += parts[i];
  for (uint32_t i = threadIdx.x; i < n_ground; i += 1024) v[1] += parts[n_chamfer + i];
  l4d_block_sum<1024, 2>(v, s_red);
  if (threadIdx.x == 0) *loss = (float)(0.5 * v[0] + 0.001 * v[1]);
}

// one term's backward: d (0.5 (sum dist1 + sum dist2)) / d flow[:, col..col+2] with w = pc + flow * step:
// row j gets step g (w_j - t_idx1[j]); row idx2[k] gets -step g (t_k - w_idx2[k]) from every target k.  Rows are shared
// with the other step of the same direction and with other threads of this launch: atomics.
__global__ void __launch_bounds__(256) k_flow_term_bwd(const float* __restrict__ w, uint32_t n, const float* __restrict__ t, uint32_t m,
                                                       const int* __restrict__ idx1, const int* __restrict__ idx2, uint32_t col,
                                                       float step, const float* __restrict__ g_loss, float* __restrict__ g_flow6) {
  const float g = *g_loss * step;
  const uint32_t top = n > m ? n : m;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < top; i += gridDim.x * blockDim.x) {
    if (i < n) {
      const size_t k = (size_t)idx1[i];
#pragma unroll
      for (int c = 0; c < 3; ++c) atomicAdd(g_flow6 + 6 * (size_t)i + col + c, g * (w[3 * (size_t)i + c] - t[3 * k + c]));
    }
    if (i < m) {
      const size_t k = (size_t)idx2[i];
#pragma unroll
      for (int c = 0; c < 3; ++c) atomicAdd(g_flow6 + 6 * k + col + c, -(g * (t[3 * (size_t)i + c] - w[3 * k + c])));
    }
  }
}

__global__ void __launch_bounds__(256) k_flow_ground_bwd(const float* __restrict__ f, uint32_t total, const float* __restrict__ g_loss,
                                                         float* __restrict__ g_f) {
  const float g = *g_loss * 0.001f;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) g_f[i] = l4d_sgn(f[i]) * g;
}
#endif
