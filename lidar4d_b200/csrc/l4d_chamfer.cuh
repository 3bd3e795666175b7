// l4d_chamfer.cuh - nearest-neighbour ("chamfer") distance op, SURVEY.md 8(f) rank 1.
//
// Replaces utils/chamfer3D/chamfer3D.cu (NmDistanceKernel :11-133, NmDistanceGradKernel :154-174) behind the
// interface of utils/chamfer3D/dist_chamfer_3D.py:31-73.  Semantics restated from those lines:
//   dist1[b,j] = min_k |xyz1[b,j] - xyz2[b,k]|^2   (fp32, d = dx*dx + dy*dy + dz*dz with dx = x2 - x1, left to right)
//   idx1[b,j]  = the smallest k attaining it        (strict '<' while scanning k upwards, '>' across 512-chunks)
//   and the same with the roles of the clouds swapped; backward: d dist / d point = 2 (p1 - p2) on both ends.
//
// Design.  The reference launches a fixed 32 x 16 grid whose x-dimension strides over the batch: with b = 1
// (every call in runner.py:216-251) 16 CTAs are busy.  Here the query cloud is cut into blocks of 256 threads x Q
// queries and, when that does not fill the SMs twice, the target cloud is split across gridDim.y as well; partial
// results meet in a 64-bit atomicMin on (distance bits << 32 | index): for non-negative floats the integer order is
// the float order and ties resolve to the smaller index, i.e. exactly the reference's rule.  Targets are staged in
// shared memory as coordinate-wise pairs of consecutive points, so one broadcast LDS.64 per coordinate serves two
// targets: the distance of one query to two targets costs 6 FADD + 2 FMUL + 4 FFMA, four
// targets are screened with one min/compare against the running best, and the (rare) update is resolved in scan
// order - FP32-pipe bound, no tensor cores (K = 3 is not a GEMM, and the reference's rounding is part of the result).
// (included at the end of l4d_kernels.cu: one translation unit, one shared library)
#pragma once

namespace l4d_chamfer {

constexpr int CH_NT = 256;      // threads per CTA
constexpr int CH_Q = 4;         // queries per thread
constexpr int CH_TILE = 2048;   // target points per shared-memory tile (24 KB as packed pairs)

__device__ __forceinline__ unsigned long long pack_key(float d, uint32_t idx) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned long long)idx;
}
// coordinate-wise pairs of fp32 (two targets per operand), IEEE round-to-nearest per lane: sm_90 has no packed fp32
// instructions, so each pair operation is two FADD / FMUL / FFMA with the rounding of the packed form
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk2(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// two consecutive targets (k, k+1), coordinate-wise: one LDS.64 per coordinate yields a packed operand
struct __align__(8) TargetPair { float2 x, y, z; };

// one direction: for every query point of `q` the nearest target of `t`.  grid = (query blocks, target splits, batch)
// DIRECT: gridDim.y == 1 -> write dist / idx straight away; otherwise combine through keys[b, nq]
template <bool DIRECT>
__global__ void __launch_bounds__(CH_NT) k_chamfer_nn(const float* __restrict__ q, uint32_t nq, const float* __restrict__ t, uint32_t nt,
                                                      float* __restrict__ dist, int* __restrict__ idx, unsigned long long* __restrict__ keys) {
  __shared__ TargetPair s_t[CH_TILE / 2];
  const uint32_t b = blockIdx.z;
  q += (size_t)b * nq * 3;
  t += (size_t)b * nt * 3;
  // this CTA's slice of the targets
  const uint32_t per = (nt + gridDim.y - 1) / gridDim.y;
  const uint32_t t0 = blockIdx.y * per;
  const uint32_t t1 = min(nt, t0 + per);
  f32x2 QX[CH_Q], QY[CH_Q], QZ[CH_Q];
  float best[CH_Q];
  uint32_t bi[CH_Q];
  const uint32_t j0 = (blockIdx.x * CH_NT + threadIdx.x) * CH_Q;
#pragma unroll
  for (int u = 0; u < CH_Q; ++u) {
    const uint32_t j = min(j0 + u, nq - 1);
    const float x = __ldg(q + 3 * (size_t)j), y = __ldg(q + 3 * (size_t)j + 1), z = __ldg(q + 3 * (size_t)j + 2);
    QX[u] = pk2(x, x); QY[u] = pk2(y, y); QZ[u] = pk2(z, z);
    best[u] = __int_as_float(0x7f800000);      // +inf: the first candidate always wins (the reference's k == 0 case)
    bi[u] = t0;
  }
  const float inf = __int_as_float(0x7f800000);
  for (uint32_t k0 = t0; k0 < t1; k0 += CH_TILE) {
    const uint32_t cnt = min((uint32_t)CH_TILE, t1 - k0);
    const uint32_t cnt4 = (cnt + 3u) & ~3u;                // padded with points at infinity: d = +inf never wins
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < cnt4; i += CH_NT) {
      const float* p = t + 3 * (size_t)(k0 + i);
      const bool ok = i < cnt;
      const float x = ok ? __ldg(p) : inf, y = ok ? __ldg(p + 1) : inf, z = ok ? __ldg(p + 2) : inf;
      float* dst = reinterpret_cast<float*>(&s_t[i >> 1]) + (i & 1u);
      dst[0] = x; dst[2] = y; dst[4] = z;
    }
    __syncthreads();
#pragma unroll 2
    for (uint32_t k = 0; k < cnt4; k += 4) {
      const TargetPair a = s_t[k >> 1], c = s_t[(k >> 1) + 1];
      const f32x2 ax = pk2(a.x.x, a.x.y), ay = pk2(a.y.x, a.y.y), az = pk2(a.z.x, a.z.y);
      const f32x2 cx = pk2(c.x.x, c.x.y), cy = pk2(c.y.x, c.y.y), cz = pk2(c.z.x, c.z.y);
#pragma unroll
      for (int u = 0; u < CH_Q; ++u) {
        // chamfer3D.cu:29-32 `x2*x2+y2*y2+z2*z2` with x2 = target - query: nvcc (12.9, default -fmad) contracts it to
        // fma(dz,dz, fma(dx,dx, dy*dy)); spelled out so the rounding never depends on the compiler's choice (the
        // oracle emulates exactly this chain), two targets per instruction
        f32x2 dx = sub2(ax, QX[u]), dy = sub2(ay, QY[u]), dz = sub2(az, QZ[u]);
        const f32x2 d01 = fma2(dz, dz, fma2(dx, dx, mul2(dy, dy)));
        dx = sub2(cx, QX[u]); dy = sub2(cy, QY[u]); dz = sub2(cz, QZ[u]);
        const f32x2 d23 = fma2(dz, dz, fma2(dx, dx, mul2(dy, dy)));
        float d0, d1, d2, d3;
        upk2(d01, d0, d1);
        upk2(d23, d2, d3);
        if (__builtin_expect(fminf(fminf(d0, d1), fminf(d2, d3)) < best[u], 0)) {   // rare after the first tiles: resolve in scan order
          if (d0 < best[u]) { best[u] = d0; bi[u] = k0 + k; }
          if (d1 < best[u]) { best[u] = d1; bi[u] = k0 + k + 1; }
          if (d2 < best[u]) { best[u] = d2; bi[u] = k0 + k + 2; }
          if (d3 < best[u]) { best[u] = d3; bi[u] = k0 + k + 3; }
        }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < CH_Q; ++u) {
    const uint32_t j = j0 + u;
    if (j >= nq || t1 <= t0) continue;
    if (DIRECT) {
      dist[(size_t)b * nq + j] = best[u];
      idx[(size_t)b * nq + j] = (int)bi[u];
    } else {
      atomicMin(keys + (size_t)b * nq + j, pack_key(best[u], bi[u]));
    }
  }
}

__global__ void k_chamfer_fill(unsigned long long* keys, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = ~0ull;
}
__global__ void k_chamfer_unpack(const unsigned long long* __restrict__ keys, size_t n, float* __restrict__ dist, int* __restrict__ idx) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  dist[i] = __uint_as_float((uint32_t)(k >> 32));
  idx[i] = (int)(uint32_t)k;
}

// backward of one direction (semantics of chamfer3D.cu:154-174): with v = 2 * dL/ddist[j] * (q_j - t_nn(j)),
// the query point receives +v and its nearest target -v.  One thread per query; the query's own gradient row is
// touched by this thread only in this launch but shared with the other direction's launch, hence atomics on both.
__global__ void k_chamfer_grad(uint32_t nq, const float* __restrict__ q, uint32_t nt, const float* __restrict__ t, const float* __restrict__ gdist,
                               const int* __restrict__ idx, float* __restrict__ gq, float* __restrict__ gt) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nq) return;
  const size_t qrow = (size_t)blockIdx.y * nq + j;
  const size_t trow = (size_t)blockIdx.y * nt + (size_t)idx[qrow];
  const float scale = gdist[qrow] * 2;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = scale * (q[3 * qrow + c] - t[3 * trow + c]);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    atomicAdd(gq + 3 * qrow + c, v[c]);
    atomicAdd(gt + 3 * trow + c, -v[c]);
  }
}

// target splits so that every SM gets about eight CTAs (four are resident at a time): with only two per SM the last,
// partial wave leaves most of the SMs idle
static uint32_t splits_for(uint32_t b, uint32_t nq, uint32_t nt) {
  const uint32_t qblocks = (nq + CH_NT * CH_Q - 1) / (CH_NT * CH_Q);
  const uint32_t want = 8u * (uint32_t)sm_count();
  uint32_t s = (want + qblocks * b - 1) / (qblocks * b);
  const uint32_t max_s = (nt + 255) / 256;        // at least 256 targets per split
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  if (s > 65535u) s = 65535u;
  return s;
}

static int nn_one_direction(const float* q, uint32_t nq, const float* t, uint32_t nt, uint32_t b, float* dist, int* idx,
                     unsigned long long* keys, cudaStream_t st) {
  const uint32_t qblocks = (nq + CH_NT * CH_Q - 1) / (CH_NT * CH_Q);
  const uint32_t s = splits_for(b, nq, nt);
  const dim3 grid(qblocks, s, b);
  if (s == 1) {
    ++g_launches; k_chamfer_nn<true><<<grid, CH_NT, 0, st>>>(q, nq, t, nt, dist, idx, nullptr);
  } else {
    const size_t n = (size_t)b * nq;
    ++g_launches; k_chamfer_fill<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n);
    ++g_launches; k_chamfer_nn<false><<<grid, CH_NT, 0, st>>>(q, nq, t, nt, nullptr, nullptr, keys);
    ++g_launches; k_chamfer_unpack<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n, dist, idx);
  }
  return 0;
}

}  // namespace l4d_chamfer
using namespace l4d_chamfer;

extern "C" size_t l4d_chamfer_work_bytes(uint32_t b, uint32_t n, uint32_t m) {
  return ((size_t)b * n + (size_t)b * m) * sizeof(unsigned long long);
}

extern "C" int l4d_chamfer_forward(const float* xyz1, const float* xyz2, uint32_t b, uint32_t n, uint32_t m, float* dist1,
                                   float* dist2, int32_t* idx1, int32_t* idx2, void* work, size_t work_bytes, void* stream) {
  if (!xyz1 || !xyz2 || !dist1 || !dist2 || !idx1 || !idx2) return l4d_fail(L4D_EINVAL, "null pointer");
  if (b == 0) return L4D_OK;
  if (n == 0 || m == 0) return l4d_fail(L4D_EINVAL, "chamfer: empty point cloud");
  if (b > 65535u) return l4d_fail(L4D_EINVAL, "chamfer: batch too large");
  if (!work || work_bytes < l4d_chamfer_work_bytes(b, n, m)) return l4d_fail(L4D_ESIZE, "chamfer work buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(work);
  nn_one_direction(xyz1, n, xyz2, m, b, dist1, idx1, keys, st);
  nn_one_direction(xyz2, m, xyz1, n, b, dist2, idx2, keys + (size_t)b * n, st);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return l4d_fail(L4D_ECUDA, "chamfer forward: %s", cudaGetErrorString(e));
  return L4D_OK;
}

extern "C" int l4d_chamfer_backward(const float* xyz1, const float* xyz2, uint32_t b, uint32_t n, uint32_t m, const float* g_dist1,
                                    const float* g_dist2, const int32_t* idx1, const int32_t* idx2, float* g_xyz1, float* g_xyz2,
                                    void* stream) {
  if (!xyz1 || !xyz2 || !g_dist1 || !g_dist2 || !idx1 || !idx2 || !g_xyz1 || !g_xyz2) return l4d_fail(L4D_EINVAL, "null pointer");
  if (b == 0) return L4D_OK;
  if (n == 0 || m == 0) return l4d_fail(L4D_EINVAL, "chamfer: empty point cloud");
  if (b > 65535u) return l4d_fail(L4D_EINVAL, "chamfer: batch too large");
  cudaStream_t st = (cudaStream_t)stream;
  ++g_launches; k_chamfer_grad<<<dim3((n + 255) / 256, b), 256, 0, st>>>(n, xyz1, m, xyz2, g_dist1, idx1, g_xyz1, g_xyz2);
  ++g_launches; k_chamfer_grad<<<dim3((m + 255) / 256, b), 256, 0, st>>>(m, xyz2, n, xyz1, g_dist2, idx2, g_xyz2, g_xyz1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return l4d_fail(L4D_ECUDA, "chamfer backward: %s", cudaGetErrorString(e));
  return L4D_OK;
}
