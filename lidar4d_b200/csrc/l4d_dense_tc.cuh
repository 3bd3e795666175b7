// l4d_dense_tc.cuh - tensor-core (wgmma) versions of the dense kernels of the split pipeline.
// Requires mlp_fp16 (MLP weights are fp16 working copies, as tiny-cuda-nn keeps them).
//
// Tile = 128 samples; warpgroup w owns rows [64w, 64w + 64) of every product.
// Operands live in shared memory as fp16 in the K-major interleaved layout of l4d_tc.cuh
// ([k/8][row][8 halves], 16-byte chunks).  Activations are carried as hi + lo fp16 pairs
// (x = hi + lo to ~2^-22 relative), i.e. every product with an fp16 weight is exact and the fp32
// accumulation reproduces the fp32-FMA kernels to ~1e-6: the 1e-4 parity bar holds on the
// tensor-core path too.  Every warpgroup issues the wgmma of its 64-row block and runs the epilogues
// on the accumulator fragments in its registers; weight gradients are flushed with fp32 atomics
// straight from there.
#pragma once
#include "l4d_core.cuh"
#include "l4d_tc.cuh"

namespace l4dtc {

// ---- tile helpers ----------------------------------------------------------------------------
// 16-byte chunk (row r, k-chunk c) of a 128-row tile
__device__ __forceinline__ unsigned char* tile_chunk(unsigned char* tile, int r, int c) { return tile + ((size_t)c * 128 + r) * 16; }

// write 8 consecutive k-values of row r as hi and lo fp16 chunks
__device__ __forceinline__ void tile_put8(unsigned char* hi, unsigned char* lo, int r, int c, const float* v) {
  float res[8];
  __half2 h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    const float2 f = __half22float2(h[i]);
    res[2 * i] = v[2 * i] - f.x;
    res[2 * i + 1] = v[2 * i + 1] - f.y;
  }
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&h[0]); o.y = *reinterpret_cast<uint32_t*>(&h[1]);
  o.z = *reinterpret_cast<uint32_t*>(&h[2]); o.w = *reinterpret_cast<uint32_t*>(&h[3]);
  *reinterpret_cast<uint4*>(tile_chunk(hi, r, c)) = o;
  *reinterpret_cast<uint4*>(tile_chunk(lo, r, c)) = pack8_half(res);
}

// all threads: make generic-proxy tile writes visible to the tensor cores, then barrier
__device__ __forceinline__ void publish() {
  fence_proxy_async();
  __syncthreads();
}

// warpgroup-wide: make this warpgroup's generic-proxy tile writes visible to its own next wgmma
__device__ __forceinline__ void wg_publish() {
  fence_proxy_async();
  wg_bar();
}

// The products below are warpgroup-wide and cover the 64-row block [m0, m0 + 64) of a 128-row tile; the result stays
// in the caller's registers (fragment layout of l4d_tc.cuh).
//
// D[64 x N] = (Ah + Al) * B^T over n_chunks 16-byte k-chunks (n_chunks even): A = 128-row tiles (chunk stride 2048),
// B = K-major [k/8][b_rows][8] (b points at its first used row)
template <int N>
__device__ __forceinline__ void mma_rows(float (&d)[N / 2], int m0, uint32_t a_hi, uint32_t a_lo, uint32_t b, uint32_t b_rows, int n_chunks) {
  const Opnd a{{a_hi + (uint32_t)m0 * 16u, a_lo + (uint32_t)m0 * 16u, 0u}, 4096u, 2048u, 128u};
  const Opnd w{{b, b, 0u}, 2u * b_rows * 16u, b_rows * 16u, 128u};
  wg_gemm<N, 0, 0>(d, a, w, 2, n_chunks / 2);
}
// D[64 x N] = (Ah + Al) * W: W stored [k_in/8][w_rows][8] (forward layout) and read as B(n = k_in, k = row), i.e.
// MN-major; w points at the chunk of the first k_in column used.  Issued as one wgmma group; the caller waits.
template <int N>
__device__ __forceinline__ void mma_prop_issue(float (&d)[N / 2], int m0, uint32_t a_hi, uint32_t a_lo, int n_chunks, uint32_t w, uint32_t w_rows) {
  const Opnd a{{a_hi + (uint32_t)m0 * 16u, a_lo + (uint32_t)m0 * 16u, 0u}, 4096u, 2048u, 128u};
  const Opnd b{{w, w, 0u}, 256u, 128u, w_rows * 16u};
  wg_gemm_issue<N, 0, 1>(d, a, b, 2, n_chunks / 2);
}
template <int N>
__device__ __forceinline__ void mma_prop(float (&d)[N / 2], int m0, uint32_t a_hi, uint32_t a_lo, int n_chunks, uint32_t w, uint32_t w_rows) {
  mma_prop_issue<N>(d, m0, a_hi, a_lo, n_chunks, w, w_rows);
  wg_wait<0>();
}
// v = relu(d); bit i of the result = element d[i] was positive.  The epilogues of the dense kernels write their results
// to a separate array: a non-wgmma write to an accumulator makes ptxas serialize every wgmma of the kernel.
template <int N>
__device__ __forceinline__ uint32_t frag_relu(const float (&d)[N / 2], float (&v)[N / 2]) {
  uint32_t m = 0u;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const bool on = d[i] > 0.f;
    v[i] = on ? d[i] : 0.f;
    m |= on ? (1u << i) : 0u;
  }
  return m;
}
// column c of a 64 x 16 fragment (rows [m0, m0 + 64)) -> column c + SHIFT of a 16-wide 128-row hi|lo tile; columns that
// land outside [0, 16) are dropped.  Rounding as tile_put8.
template <int SHIFT>
__device__ __forceinline__ void frag_put16_shift(unsigned char* hi, unsigned char* lo, int m0, const float (&d)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = 8 * (i >> 2) + frag_col() + (i & 1) + SHIFT, r = m0 + frag_row() + 8 * ((i >> 1) & 1);
    if (c < 0 || c > 15) continue;
    const __half x = __float2half_rn(d[i]);
    const __half y = __float2half_rn(d[i] - __half2float(x));
    const size_t off = ((size_t)(c >> 3) * 128 + r) * 16 + (c & 7) * 2;
    *reinterpret_cast<__half*>(hi + off) = x;
    *reinterpret_cast<__half*>(lo + off) = y;
  }
}
// one fp16 element (row r, column c) of a 128-row hi|lo tile
__device__ __forceinline__ void tile_put1(unsigned char* hi, unsigned char* lo, int r, int c, float v) {
  const __half x = __float2half_rn(v);
  const size_t off = ((size_t)(c >> 3) * 128 + r) * 16 + (c & 7) * 2;
  *reinterpret_cast<__half*>(hi + off) = x;
  *reinterpret_cast<__half*>(lo + off) = __float2half_rn(v - __half2float(x));
}

}  // namespace l4dtc

// smem carve-up of the dense forward kernel (bytes)
struct DenseFwdSmem {
  uint32_t w1, w2, wa1, wa2[2];     // weights
  uint32_t xh, xl;                  // feature tile (later reused for the 128-wide attribute hidden tile)
  uint32_t hh, hl;                  // 64-wide hidden tile
  uint32_t gh, gl;                  // 16-wide tile (geo)
  uint32_t misc;                    // enc[80] cdir[128] w[32] sig[128] att[2][128] floats
  uint32_t total;
};
__host__ __device__ inline DenseFwdSmem dense_fwd_smem(uint32_t in_pad) {
  DenseFwdSmem L;
  uint32_t o = 0;
  auto take = [&](uint32_t b) { uint32_t r = o; o += (b + 127u) & ~127u; return r; };
  L.w1 = take(in_pad * 64 * 2); L.w2 = take(64 * 16 * 2); L.wa1 = take(16 * 128 * 2);
  L.wa2[0] = take(64 * 64 * 2); L.wa2[1] = take(64 * 64 * 2);
  const uint32_t xbytes = (in_pad > 128 ? in_pad : 128) * 128 * 2;
  L.xh = take(xbytes); L.xl = take(xbytes);
  L.hh = take(64 * 128 * 2); L.hl = take(64 * 128 * 2);
  L.gh = take(16 * 128 * 2); L.gl = take(16 * 128 * 2);
  L.misc = take((80 + 128 + 32 + 128 + 256) * 4);
  L.total = o;
  return L;
}

// =============================================================================================
// backward 1/3 on tensor cores.
//
// Every GEMM of the dense backward runs as wgmma on 128-sample tiles:
//   forward recompute   Y = A * W^T            A K-major tile (hi+lo), W K-major weights
//   delta propagation   dA = dY * W            dY K-major tile (hi+lo), W read as an MN-major operand
//   weight gradients    dW^T = A^T * dY        both sample-major tiles read as MN-major operands
//                                              (3 terms: Ah*dh + Al*dh + Ah*dl)
// Gradient tiles are stored as fp16 hi/lo pairs after a per-tile power-of-two scale (block amax), so
// loss-scaled or tiny upstream gradients neither overflow nor flush; the scale is undone when the
// fp32 accumulators are read back.  Weight-gradient accumulators are flushed from the registers with fp32
// atomics once per tile (same count as the FMA kernel's tile_outer_accum).
// Shared memory at sigma_in_pad = 176 (L = 16): 217 KB; one CTA per SM.
// =============================================================================================
struct DenseBwdSmem {
  uint32_t w1, w2, wa1[2], wa2[2];
  uint32_t R;            // 96 KB: X hi|lo (24 chunks each) or T1,T2,T3 (hi|lo, 8 chunks each)
  uint32_t RH;           // 32 KB: sigma hidden hi|lo, later its delta
  uint32_t g16, do16, do8;   // small tiles, hi|lo
  uint32_t slab2, slab1;     // attribute weight-gradient partials of warpgroup 1 (fp32, fragment order): dW2 + dw3, dW1g
  uint32_t misc;
  uint32_t total;
};
__host__ __device__ inline DenseBwdSmem dense_bwd_smem(uint32_t in_pad) {
  DenseBwdSmem L;
  uint32_t o = 0;
  auto take = [&](uint32_t b) { uint32_t r = o; o += (b + 127u) & ~127u; return r; };
  L.w1 = take(in_pad * 64 * 2); L.w2 = take(64 * 16 * 2);
  L.wa1[0] = take(16 * 64 * 2); L.wa1[1] = take(16 * 64 * 2);
  L.wa2[0] = take(64 * 64 * 2); L.wa2[1] = take(64 * 64 * 2);
  L.R = take(96 * 1024); L.RH = take(32 * 1024);
  L.g16 = take(2 * 4096); L.do16 = take(2 * 4096); L.do8 = take(2 * 2048);
  L.slab2 = take((32 + 2) * 128 * 4); L.slab1 = take(8 * 128 * 4);
  L.misc = take((80 + 128 + 128 + 128 + 32 + 128 + 256 + 128) * 4);
  L.total = o;
  return L;
}

namespace l4dtc {
// dW^T[64 x N] = Ah^T * Bh + Al^T * Bh + Ah^T * Bl over the 128 samples of sample-major tiles read as MN-major operands;
// a / b = shared address of the first 16-byte feature chunk used.  Warpgroup-wide; f(row, col, v[col], v[col + 1]).
template <int N, class F>
__device__ __forceinline__ void mma_tt(uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, F&& f) {
  const Opnd a{{a_hi, a_lo, a_hi}, 256u, 128u, 2048u};
  const Opnd b{{b_hi, b_hi, b_lo}, 256u, 128u, 2048u};
  float d[N / 2];
  wg_gemm<N, 1, 1>(d, a, b, 3, 8);
  frag_foreach<N>(d, f);
}
// the same product over the 64 samples [m0, m0 + 64) only, issued as one wgmma group; the caller waits
template <int N>
__device__ __forceinline__ void mma_tt64_issue(float (&d)[N / 2], int m0, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  const uint32_t o = (uint32_t)m0 * 16u;
  const Opnd a{{a_hi + o, a_lo + o, a_hi + o}, 256u, 128u, 2048u};
  const Opnd b{{b_hi + o, b_hi + o, b_lo + o}, 256u, 128u, 2048u};
  wg_gemm_issue<N, 1, 1>(d, a, b, 3, 4);
}
__device__ __forceinline__ void red2(float* p, float a, float b) { atomicAdd(reinterpret_cast<float2*>(p), make_float2(a, b)); }
__device__ __forceinline__ float block_amax128(float v, float* s_w) {
  v = fabsf(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  const float r = fmaxf(fmaxf(s_w[0], s_w[1]), fmaxf(s_w[2], s_w[3]));
  __syncthreads();
  return r;
}
// power-of-two factor r that maps amax into [2^5, 2^6): fp16 hi+lo then resolve the tile to ~2^-30 of its
// largest element while leaving 2^10 of headroom below the fp16 maximum
__device__ __forceinline__ float pow2_factor(float amax) {
  int e;
  frexpf(amax, &e);
  // capped at 2^126: a tile whose amax is below 2^-120 (surface-like rays, transmittance ~1e-30 behind the surface)
  // would otherwise get an infinite scale, and inf * 0 turns the whole tile's gradients into NaN
  return ldexpf(1.0f, min(6 - e, 126));
}
}  // namespace l4dtc

namespace l4dtc {
// 256-thread CTA with two threads per row: warps 0-3 and 4-7 run the same 128-wide scans redundantly
__device__ __forceinline__ float half_excl_prod(float v, float* s_w, float& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, base = warp & 4, wq = warp & 3;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= t;
  }
  if (lane == 31) s_w[warp] = inc;
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) ex = 1.f;
  __syncthreads();
  float pre = 1.f, tot = 1.f;
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const float t = s_w[base + w];
    if (w < wq) pre *= t;
    tot *= t;
  }
  total = tot;
  __syncthreads();
  return pre * ex;
}
__device__ __forceinline__ float half_excl_suffix_sum(float v, float* s_w, float& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, base = warp & 4, wq = warp & 3;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_down_sync(0xffffffffu, inc, o);
    if (lane + o < 32) inc += t;
  }
  if (lane == 0) s_w[warp] = inc;
  float ex = __shfl_down_sync(0xffffffffu, inc, 1);
  if (lane == 31) ex = 0.f;
  __syncthreads();
  float post = 0.f, tot = 0.f;
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const float t = s_w[base + w];
    if (w > wq) post += t;
    tot += t;
  }
  total = tot;
  __syncthreads();
  return post + ex;
}
// max |v| over the 128 threads of this thread's warpgroup (s_w[4 wg .. 4 wg + 3])
__device__ __forceinline__ float wg_amax(float v, float* s_w) {
  const int warp = threadIdx.x >> 5, base = warp & 4;
  v = fabsf(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) s_w[warp] = v;
  wg_bar();
  const float r = fmaxf(fmaxf(s_w[base], s_w[base + 1]), fmaxf(s_w[base + 2], s_w[base + 3]));
  wg_bar();
  return r;
}
// producer / consumer handshake between the two warpgroups of a 256-thread CTA on named barrier id: one warpgroup
// arrives (does not wait), the other waits for it
__device__ __forceinline__ void pair_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void pair_wait(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ float block_amax256(float v, float* s_w) {
  v = fabsf(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = s_w[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = fmaxf(r, s_w[w]);
  __syncthreads();
  return r;
}
}  // namespace l4dtc

// -------------------------------------------------------------------------------------------
// forward 2/2 on tensor cores: sigma MLP, compositing, attribute heads.  One CTA per ray, 256 threads: warpgroup w
// computes rows [64w, 64w + 64) of every product and runs its epilogues on the accumulator fragments; the compositing
// scans run in row order (two threads per row, thread half h accumulates head h) and exchange per-row values with the
// fragments through small per-row arrays.
// -------------------------------------------------------------------------------------------
namespace l4dtc {
// sum over the 128 rows of one thread half (warps 0-3 / 4-7) of a 256-thread CTA; every thread of the half gets it
__device__ __forceinline__ float half_sum(float v, float* s_w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, base = warp & 4;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) s_w[warp] = v;
  __syncthreads();
  const float r = (s_w[base] + s_w[base + 1]) + (s_w[base + 2] + s_w[base + 3]);
  __syncthreads();
  return r;
}
}  // namespace l4dtc

__global__ void __launch_bounds__(256) k_fwd_dense_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  __shared__ __align__(8) uint64_t s_xbar;
  const DevModel& M = A.M;
  const int tid = threadIdx.x;
  const int row = tid & 127, half = tid >> 7;
  const uint32_t in_pad = M.sigma_in_pad;
  const DenseFwdSmem L = dense_fwd_smem(in_pad);
  unsigned char *xh = dsm + L.xh, *xl = dsm + L.xl, *hh = dsm + L.hh, *hl = dsm + L.hl, *gh = dsm + L.gh, *gl = dsm + L.gl;
  float* s_enc = reinterpret_cast<float*>(dsm + L.misc);
  float* s_cdir = s_enc + 80;
  float* s_w = s_cdir + 128;
  float* s_sig = s_w + 32;         // per row: sigma pre-activation (output column 0)
  float* s_att = s_sig + 128;      // per head and row: attribute logit
  const int m0 = 64 * half;        // rows of this warpgroup
  const uint32_t sb = smem_u32(dsm);

  if (tid == 0) { mbar_init(&s_xbar, 1); fence_mbar_init(); }
  // weights -> shared memory (already in operand layout in global memory)
  {
    auto cp = [&](uint32_t off, const __half* src, uint32_t bytes) {
      for (uint32_t i = tid * 16; i < bytes; i += 256 * 16)
        *reinterpret_cast<uint4*>(dsm + off + i) = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(src) + i));
    };
    cp(L.w1, M.tc_sig_w1, in_pad * 64 * 2);
    cp(L.w2, M.tc_sig_w2, 64 * 16 * 2);
    cp(L.wa1, M.tc_att_w1g, 16 * 128 * 2);
    cp(L.wa2[0], M.tc_att_w2[0], 64 * 64 * 2);
    cp(L.wa2[1], M.tc_att_w2[1], 64 * 64 * 2);
  }
  publish();
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t n_steps = A.S;
  const int n_xchunks = (int)in_pad / 8;
  // feature tiles arrive as fp16 hi|lo operand tiles (written by k_fwd_gather) with one bulk copy per half; the copy of
  // the next tile is issued as soon as the last MMA that reads the X buffer has completed
  const uint32_t xbytes = A.sv.x_chunks * 2048u;
  const uint32_t n_tiles = A.sv.n_tiles;
  uint32_t xphase = 0u;
  auto x_issue = [&](uint32_t r, uint32_t t) {
    if (half == 0) {       // tcnn's ones-padding chunks are not stored in global memory
      for (int c = (int)A.sv.x_chunks; c < n_xchunks; ++c) {
        *reinterpret_cast<uint4*>(tile_chunk(xh, row, c)) = make_uint4(0x3C003C00u, 0x3C003C00u, 0x3C003C00u, 0x3C003C00u);
        *reinterpret_cast<uint4*>(tile_chunk(xl, row, c)) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    if (tid == 0) {
      const unsigned char* src = A.sv.feat_tc + ((size_t)r * n_tiles + t) * (size_t)(2u * xbytes);
      mbar_expect_tx(&s_xbar, 2u * xbytes);
      bulk_g2s(sb + L.xh, src, xbytes, &s_xbar);
      bulk_g2s(sb + L.xl, src + xbytes, xbytes, &s_xbar);
    }
  };
  auto x_issue_next = [&](uint32_t r, uint32_t t) {
    if (t + 1 < n_tiles) x_issue(r, t + 1);
    else if (r + gridDim.x < A.n_rays) x_issue(r + gridDim.x, 0u);
  };
  if (blockIdx.x < A.n_rays) x_issue(blockIdx.x, 0u);

  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
    const float dx = __ldg(A.rays_d + 3 * ray), dy = __ldg(A.rays_d + 3 * ray + 1), dz = __ldg(A.rays_d + 3 * ray + 2);
    __syncthreads();
    for (int i = tid; i < L4D_ENC; i += 256) {
      const int dim = i / 24, k = (i % 24) >> 1, ph = i & 1;
      s_enc[i] = l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), k, ph);
    }
    __syncthreads();
    if (tid < 128) s_cdir[tid] = l4d_attr_cdir(M, tid >> 6, tid & 63, s_enc);
    __syncthreads();
    // per-thread partial sums over this thread's row: half 0 carries depth, weight sum and head 0, half 1 carries head 1
    float carry = 1.f, pd = 0.f, pa = 0.f, pw = 0.f;
    const uint64_t rg = A.ray_offset + ray;
    for (uint32_t j0 = 0; j0 < n_steps; j0 += 128) {
      const uint32_t j = j0 + row;
      const bool valid = j < n_steps;
      const size_t p = (size_t)ray * n_steps + (valid ? j : 0);
      if (tid == 0 && A.train) A.sv.tstart[(size_t)ray * n_tiles + (j0 >> 7)] = carry;     // the backward starts every tile from here
      mbar_wait(&s_xbar, xphase);      // this tile's features have landed
      xphase ^= 1u;
      publish();
      // ---- warpgroup wg: rows [m0, m0 + 64).  hidden = relu(X W1^T) -> hi/lo tile, then the output layer ----
      {
        float d[32];
        mma_rows<64>(d, m0, sb + L.xh, sb + L.xl, sb + L.w1, 64, n_xchunks);
        float v[32];
        frag_relu<64>(d, v);
        frag_put<64>(hh, hl, 128, m0, 0, v);
      }
      wg_publish();
      {
        float o[8];
        mma_rows<16>(o, m0, sb + L.hh, sb + L.hl, sb + L.w2, 16, 8);
        if ((tid & 3) == 0) { s_sig[m0 + frag_row()] = o[0]; s_sig[m0 + frag_row() + 8] = o[2]; }
        frag_put16_shift<-1>(gh, gl, m0, o);          // geo -> attribute input columns 0..14 (rows outside the mask: below)
      }
      __syncthreads();
      float zj = 0.f, alpha = 0.f, sigma = 0.f;
      if (valid) {
        sigma = expf(s_sig[row]);
        zj = l4d_z(rs, rg, j);
        const float delta = (j + 1 < n_steps) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
        alpha = l4d_alpha(M, delta, sigma);
      }
      const float vv = valid ? (1.0f - alpha) + 1e-15f : 1.f;
      float total;
      const float T = carry * half_excl_prod(vv, s_w, total);      // both halves run the same 128-row scan
      carry *= total;
      const float w = alpha * T;
      const bool masked = valid && w > 1e-4f;
      float a = 0.f;                     // this half's attribute head
      const bool any_masked = __syncthreads_or(masked ? 1 : 0) != 0;
      if (!any_masked) x_issue_next(ray, j0 >> 7);       // the X buffer is free already
      if (any_masked) {
        // ---- attribute heads: [geo,0] (K=16) -> 2x64 -> relu -> 64 -> relu -> dot w3 -> sigmoid ----
        if (half == 0) {
          if (masked) tile_put1(gh, gl, row, 15, 0.f);
          else {
            *reinterpret_cast<uint4*>(tile_chunk(gh, row, 0)) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(tile_chunk(gh, row, 1)) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(tile_chunk(gl, row, 0)) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(tile_chunk(gl, row, 1)) = make_uint4(0u, 0u, 0u, 0u);
          }
        }
        publish();
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {    // 128 columns: net0 hidden | net1 hidden -> chunks 0..15 of the x tile
          float d[32];
          mma_rows<64>(d, m0, sb + L.gh, sb + L.gl, sb + L.wa1 + (uint32_t)net * 64u * 16u, 128, 2);
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = fmaxf(d[i] + s_cdir[net * 64 + 8 * (i >> 2) + frag_col() + (i & 1)], 0.f);
          frag_put<64>(xh, xl, 128, m0, 8 * net, v);
        }
        wg_publish();
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {
          float d[32];
          mma_rows<64>(d, m0, sb + L.xh + (uint32_t)net * 8u * 2048u, sb + L.xl + (uint32_t)net * 8u * 2048u, sb + L.wa2[net], 64, 8);
          float o[2] = {0.f, 0.f};
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int h = (i >> 1) & 1;
            o[h] = fmaf(fmaxf(d[i], 0.f), l4d_ld1(M.att_w3[net] + 8 * (i >> 2) + frag_col() + (i & 1)), o[h]);
          }
          o[0] = quad_sum(o[0]);
          o[1] = quad_sum(o[1]);
          if ((tid & 3) == 0) { s_att[net * 128 + m0 + frag_row()] = o[0]; s_att[net * 128 + m0 + frag_row() + 8] = o[1]; }
        }
        __syncthreads();
        x_issue_next(ray, j0 >> 7);                    // the attribute hidden tile (in the X buffer) has been consumed
        if (masked) a = l4d_sigmoid(s_att[half * 128 + row]);
      }
      pa = fmaf(w, a, pa);
      if (half == 0) { pd = fmaf(w, zj, pd); pw += w; }
      if (valid) {
        if (A.train) {
          if (half == 0) A.sv.sigma[p] = sigma;
          A.sv.attr[(size_t)half * A.sv.P + p] = a;
        }
        if (half == 0) {
          if (A.weights) A.weights[p] = w;
          if (A.zvals) A.zvals[p] = zj;
        }
      }
      __syncthreads();          // the operand tiles and the per-row arrays are reused by the next tile
    }
    pd = half_sum(pd, s_w); pa = half_sum(pa, s_w); pw = half_sum(pw, s_w);
    if (tid == 0) { A.depth[ray] = pd; A.image[2 * ray] = pa; A.wsum[ray] = pw; }
    if (tid == 128) A.image[2 * ray + 1] = pa;
  }
}

#ifdef L4D_PHASE_CLOCKS
__device__ unsigned long long g_phase_clk[32];
#define L4D_PH(i) do { if (tid == 0) { const long long t_ = clock64(); s_clk[i] += (unsigned long long)(t_ - t_last); t_last = t_; } } while (0)
#else
#define L4D_PH(i) do { } while (0)
#endif

// backward 0/3: the compositing backward of the tensor-core pipeline.  One 128-thread CTA per ray (thread == row of a
// tile) walks the tiles back to front with the carried suffix sum and leaves {dL/dsigma, dL/da0, dL/da1, attribute mask
// (0 / 1)} of every sample in quad 0 of the sample's row of the dL/dfeature tile.  k_bwd_dense_tc reads them at the
// start of the tile and overwrites them with dL/dfeature at its end.  The scans are the forward's (half_excl_prod over
// four warps from the saved transmittance at the tile start), the per-sample arithmetic that of the FMA kernels.
__global__ void __launch_bounds__(128) k_bwd_composite(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  __shared__ float s_w[8];
  const DevModel& M = A.M;
  const int row = threadIdx.x;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t n_steps = A.S;
  const int n_tiles = (int)A.sv.n_tiles;
  const float kk = M.active_sensor ? 2.0f : 1.0f;
  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
    const float gd = __ldg(A.g_depth + ray), gi0 = __ldg(A.g_image + 2 * ray), gi1 = __ldg(A.g_image + 2 * ray + 1);
    const float gws = A.g_wsum ? __ldg(A.g_wsum + ray) : 0.f;
    const uint64_t rg = A.ray_offset + ray;
    float suffix = 0.f;
    for (int t = n_tiles - 1; t >= 0; --t) {
      const uint32_t j = (uint32_t)t * 128 + row;
      const bool active = j < n_steps;
      const size_t p = (size_t)ray * n_steps + (active ? j : 0);
      float v = 1.f, alpha = 0.f, gw = 0.f, delta = 0.f;
      if (active) {
        const float zj = l4d_z(rs, rg, j);
        delta = (j + 1 < n_steps) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
        alpha = l4d_alpha(M, delta, A.sv.sigma[p]);
        v = (1.0f - alpha) + 1e-15f;
        gw = gd * zj + gi0 * A.sv.attr[p] + gi1 * A.sv.attr[A.sv.P + p] + gws;
        if (A.g_weights) gw += __ldg(A.g_weights + p);
      }
      float total, qtot;
      const float T = __ldg(A.sv.tstart + (size_t)ray * n_tiles + t) * half_excl_prod(v, s_w, total);
      const float w = alpha * T;
      const float suf = suffix + half_excl_suffix_sum(gw * w, s_w, qtot);
      suffix += qtot;
      if (active) {
        const float dsigma = (gw * T - suf / v) * (kk * delta * M.density_scale) * (1.0f - alpha);
        const bool masked = w > 1e-4f;
        *reinterpret_cast<float4*>(A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j)) =
            masked ? make_float4(dsigma, w * gi0, w * gi1, 1.f) : make_float4(dsigma, 0.f, 0.f, 0.f);
      }
    }
  }
}

// backward 1/3 on tensor cores.  256 threads: warpgroup w owns rows [64w, 64w + 64) of every tile and computes them in
// every row-wise product, running its epilogues on the fragments.  In the attribute heads the warpgroups run apart:
// each skips a head whose rows carry no gradient, scales its delta tiles by its own 64-row amax and forms the weight
// gradients of its own 64 samples; where both ran a head, warpgroup 1 hands its (unscaled) partials to warpgroup 0
// through a shared-memory slab and warpgroup 0 issues the reductions, so every weight gradient is still reduced once per
// 128-sample tile.  The sigma-MLP phases (P1, P3, P4) synchronise the CTA as before.
__global__ void __launch_bounds__(256) k_bwd_dense_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  __shared__ __align__(8) uint64_t s_xbar;
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  const int row = tid & 127, half = tid >> 7;     // row-order work: two threads per row
  const int wg = half;                            // warpgroup
  const uint32_t in_pad = M.sigma_in_pad;
  const DenseBwdSmem L = dense_bwd_smem(in_pad);
  const uint32_t sb = smem_u32(dsm);
  // tile views
  unsigned char* xh = dsm + L.R;                 // X hi: 24 chunks
  unsigned char* xl = dsm + L.R + 48 * 1024;     // X lo
  unsigned char* t1h = dsm + L.R, *t1l = t1h + 16384;              // T1
  unsigned char* t2h = dsm + L.R + 32768, *t2l = t2h + 16384;      // T2
  unsigned char* t3h = dsm + L.R + 65536, *t3l = t3h + 16384;      // T3
  unsigned char* hh = dsm + L.RH, *hl = hh + 16384;
  unsigned char* g16h = dsm + L.g16, *g16l = g16h + 4096;
  unsigned char* o16h = dsm + L.do16, *o16l = o16h + 4096;
  unsigned char* o8h = dsm + L.do8, *o8l = o8h + 2048;
  const uint32_t aXh = sb + L.R, aXl = aXh + 48 * 1024;
  const uint32_t aT1h = sb + L.R, aT1l = aT1h + 16384, aT2h = aT1h + 32768, aT2l = aT2h + 16384, aT3h = aT1h + 65536, aT3l = aT3h + 16384;
  const uint32_t aHh = sb + L.RH, aHl = aHh + 16384;
  const uint32_t aG16h = sb + L.g16, aG16l = aG16h + 4096, aO16h = sb + L.do16, aO16l = aO16h + 4096, aO8h = sb + L.do8, aO8l = aO8h + 2048;
  float* s_enc = reinterpret_cast<float*>(dsm + L.misc);
  float* s_cdir = s_enc + 80;      // full per-ray first-layer term (as the forward uses it)
  float* s_cdir2 = s_cdir + 128;   // same minus the first ones-row (the tile's column 15 carries that 1)
  float* s_csum = s_cdir2 + 128;
  float* s_w = s_csum + 128;
  float* s_dsig = s_w + 32;        // per row: dL/dsigma, attribute deltas of both heads, attribute mask (0 / 1)
  float* s_da = s_dsig + 128;
  float* s_mk = s_da + 256;
  float* slab2 = reinterpret_cast<float*>(dsm + L.slab2);
  float* slab1 = reinterpret_cast<float*>(dsm + L.slab1);
  const int m0 = 64 * wg;          // rows of this warpgroup
  const int lt = tid & 127;        // thread within the warpgroup (slab index)
  __shared__ float s_w3max[2];
  // per tile (two slots, by the parity of the CTA's tile count): bit 2 w + net = rows of warpgroup w carry a gradient
  // for attribute head net
  __shared__ uint32_t s_heads[2];
  uint32_t tile_no = 0;
  // warpgroup 1: a slab holds partials warpgroup 0 has not consumed yet (named barriers 3 / 4: slab2 full / free,
  // 5 / 6: slab1 full / free)
  bool slab2_busy = false, slab1_busy = false;
#ifdef L4D_PHASE_CLOCKS
  __shared__ unsigned long long s_clk[32];
  long long t_last = clock64();
  if (tid < 32) s_clk[tid] = 0ull;
  __syncthreads();
#endif

  if (tid == 0) { mbar_init(&s_xbar, 1); fence_mbar_init(); }
  if (tid < 2) {
    float m = 1.0f;
    for (int k = 0; k < 64; ++k) m = fmaxf(m, fabsf(l4d_ld1(M.att_w3[tid] + k)));
    s_w3max[tid] = m;
  }
  {
    auto cp = [&](uint32_t off, const __half* src, uint32_t bytes) {
      for (uint32_t i = tid * 16; i < bytes; i += 256 * 16)
        *reinterpret_cast<uint4*>(dsm + off + i) = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(src) + i));
    };
    cp(L.w1, M.tc_sig_w1, in_pad * 64 * 2);
    cp(L.w2, M.tc_sig_w2, 64 * 16 * 2);
    cp(L.wa1[0], M.tc_att_w1g_net[0], 16 * 64 * 2);
    cp(L.wa1[1], M.tc_att_w1g_net[1], 16 * 64 * 2);
    cp(L.wa2[0], M.tc_att_w2[0], 64 * 64 * 2);
    cp(L.wa2[1], M.tc_att_w2[1], 64 * 64 * 2);
  }
  if (tid < 2) s_heads[tid] = 0u;
  publish();
  const uint32_t n_steps = A.S;
  const int n_tiles = (int)((n_steps + 127) / 128);
  const int n_xchunks = (int)in_pad / 8;

  // The X tile (fp16 hi|lo operand tile written by k_fwd_gather) arrives by bulk copy.  It is needed twice per tile
  // (forward recompute, first-layer weight gradient) and the attribute phase reuses its buffer in between, so:
  //   - the copy for the NEXT tile is issued as soon as this tile's last MMAs have completed (hidden behind the epilogue)
  //   - the re-load for P4 is issued only if the attribute phase ran, and overlaps with P3
  const uint32_t xbytes = A.sv.x_chunks * 2048u;
  uint32_t xphase = 0u;
  bool x_inflight = false;
  auto x_issue = [&](uint32_t r, int t) {
    if (half == 0) {       // tcnn's ones-padding chunks are not stored in global memory
      for (int c = (int)A.sv.x_chunks; c < 24; ++c) {
        const bool one = c < n_xchunks;
        *reinterpret_cast<uint4*>(tile_chunk(xh, row, c)) = one ? make_uint4(0x3C003C00u, 0x3C003C00u, 0x3C003C00u, 0x3C003C00u) : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(tile_chunk(xl, row, c)) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    if (tid == 0) {
      const unsigned char* src = A.sv.feat_tc + ((size_t)r * A.sv.n_tiles + (uint32_t)t) * (size_t)(2u * xbytes);
      mbar_expect_tx(&s_xbar, 2u * xbytes);
      bulk_g2s(aXh, src, xbytes, &s_xbar);
      bulk_g2s(aXl, src + xbytes, xbytes, &s_xbar);
    }
    x_inflight = true;
  };
  auto x_wait = [&]() {
    if (x_inflight) { mbar_wait(&s_xbar, xphase); xphase ^= 1u; x_inflight = false; }
  };
  auto x_issue_next = [&](uint32_t r, int t) {       // tiles of a ray are walked back to front
    if (t > 0) x_issue(r, t - 1);
    else if (r + gridDim.x < A.n_rays) x_issue(r + gridDim.x, n_tiles - 1);
  };
  if (blockIdx.x < A.n_rays) x_issue(blockIdx.x, n_tiles - 1);

  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
    const float dx = __ldg(A.rays_d + 3 * ray), dy = __ldg(A.rays_d + 3 * ray + 1), dz = __ldg(A.rays_d + 3 * ray + 2);
    __syncthreads();
    for (int i = tid; i < L4D_ENC; i += 256) {
      const int dim = i / 24, k = (i % 24) >> 1, ph = i & 1;
      s_enc[i] = l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), k, ph);
    }
    if (tid < 128) s_csum[tid] = 0.f;
    __syncthreads();
    if (tid < 128) {
      const float c = l4d_attr_cdir(M, tid >> 6, tid & 63, s_enc);
      s_cdir[tid] = c;
      s_cdir2[tid] = c - l4d_ld1(M.att_w1t[tid >> 6] + (size_t)M.attr_in_dim * L4D_H + (tid & 63));
    }
    L4D_PH(0);
    for (int t = n_tiles - 1; t >= 0; --t) {
      const uint32_t j = (uint32_t)t * 128 + row;
      const bool active = j < n_steps;
      float* dq = A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j);     // this row in the dfeat tile (float4 per 4 features)
      const uint32_t slot = tile_no & 1u;
      if (tid == 0) s_heads[slot ^ 1u] = 0u;     // the previous tile's flags: read by every thread before its last barrier
      ++tile_no;
      if (half == 0) {      // per-row values for the fragment epilogues (visible after the barrier in publish below)
        const float4 c = active ? *reinterpret_cast<const float4*>(dq) : make_float4(0.f, 0.f, 0.f, 0.f);   // k_bwd_composite
        s_dsig[row] = c.x;
        s_da[row] = c.y;
        s_da[128 + row] = c.z;
        s_mk[row] = c.w;
        const uint32_t b = (__ballot_sync(0xffffffffu, c.y != 0.f) ? 1u : 0u) | (__ballot_sync(0xffffffffu, c.z != 0.f) ? 2u : 0u);
        if ((tid & 31) == 0 && b) atomicOr(&s_heads[slot], b << (2 * (row >> 6)));
      }
      // this thread's fragment rows: m0 + frag_row() + 8h
      const int fr = m0 + frag_row();

      L4D_PH(1);
      // ---------------- P1: sigma MLP forward (rows [m0, m0 + 64) on this warpgroup) ----------------
      x_wait();
      publish();
      L4D_PH(2);
      uint32_t msk;                            // relu pattern of the hidden fragment
      {
        float d[32];
        mma_rows<64>(d, m0, aXh, aXl, sb + L.w1, 64, n_xchunks);
        float v[32];
        msk = frag_relu<64>(d, v);
        frag_put<64>(hh, hl, 128, m0, 0, v);
      }
      wg_publish();
      float out[8], dgeo[8];                   // output-layer fragment; dG fragment (geo columns 0..14)
      mma_rows<16>(out, m0, aHh, aHl, sb + L.w2, 16, 8);
#pragma unroll
      for (int i = 0; i < 8; ++i) dgeo[i] = 0.f;

      L4D_PH(3);
      // ---------------- P2: attribute heads (each warpgroup on its own rows) ----------------
      const uint32_t heads = s_heads[slot];
      const uint32_t mine = (heads >> (2 * wg)) & 3u, theirs = (heads >> (2 * (wg ^ 1))) & 3u;
      const bool x_dirty = heads != 0u;        // the attribute phase reuses the X buffer for its tiles
      if (mine) {
        // [geo, 1] tile rows of this warpgroup; zero rows for samples outside the attribute mask
        const bool mk[2] = {s_mk[fr] != 0.f, s_mk[fr + 8] != 0.f};
        {
          float gv[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) gv[i] = mk[(i >> 1) & 1] ? out[i] : 0.f;
          frag_put16_shift<-1>(g16h, g16l, m0, gv);
          if ((tid & 3) == 0) {
            tile_put1(g16h, g16l, fr, 15, mk[0] ? 1.0f : 0.f);
            tile_put1(g16h, g16l, fr + 8, 15, mk[1] ? 1.0f : 0.f);
          }
        }
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {
          if (!((mine >> net) & 1u)) continue;       // no gradient reaches this head on this warpgroup's rows
          const bool pair = (theirs >> net) & 1u;    // the other warpgroup forms partials of this head's weight gradients too
          wg_publish();
          float d[32], v[32];
          mma_rows<64>(d, m0, aG16h, aG16l, sb + L.wa1[net], 64, 2);
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = d[i] + s_cdir2[net * 64 + 8 * (i >> 2) + frag_col() + (i & 1)];
          const uint32_t m1 = frag_relu<64>(v, v);
          frag_put<64>(t1h, t1l, 128, m0, 0, v);
          wg_publish();
          mma_rows<64>(d, m0, aT1h, aT1l, sb + L.wa2[net], 64, 8);
          const uint32_t m2 = frag_relu<64>(d, v);
          float cs = 1.0f;
          float d_o[2];
          {   // output layer (fp32), sigmoid backward, delta of the second hidden layer
            float o[2] = {0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 32; ++i)
              o[(i >> 1) & 1] = fmaf(v[i], l4d_ld1(M.att_w3[net] + 8 * (i >> 2) + frag_col() + (i & 1)), o[(i >> 1) & 1]);
            frag_put<64>(t2h, t2l, 128, m0, 0, v);
            float d_raw[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float a = l4d_sigmoid(quad_sum(o[h]));
              d_raw[h] = mk[h] ? s_da[net * 128 + fr + 8 * h] * a * (1.0f - a) : 0.f;
            }
            // power-of-two scale of this warpgroup's rows of the delta tiles (|w3| <= w3max bounds the second tile too)
            const float am = wg_amax(fmaxf(fabsf(d_raw[0]), fabsf(d_raw[1])) * s_w3max[net], s_w);
            cs = am > 0.f ? pow2_factor(am) : 1.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              d_o[h] = d_raw[h] * cs;
              if ((tid & 3) == 0) {
                const float d8[8] = {d_o[h], 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                tile_put8(o8h, o8l, fr + 8 * h, 0, d8);
              }
            }
#pragma unroll
            for (int i = 0; i < 32; ++i)
              v[i] = ((m2 >> i) & 1u) ? l4d_ld1(M.att_w3[net] + 8 * (i >> 2) + frag_col() + (i & 1)) * d_o[(i >> 1) & 1] : 0.f;
            frag_put<64>(t3h, t3l, 128, m0, 0, v);
          }
          wg_publish();
          const float inv = 1.0f / cs;
          {   // dw3^T[64 x 8] = H2^T * dO (column 0 carries dO) and dW2^T[64 x 64] = H1^T * dH2 over this warpgroup's samples
            float p3[4], p2[32];
            mma_tt64_issue<8>(p3, m0, aT2h, aT2l, aO8h, aO8l);
            mma_tt64_issue<64>(p2, m0, aT1h, aT1l, aT3h, aT3l);
            wg_wait<0>();
            if (pair && wg == 1) {           // hand the partials to warpgroup 0
              if (slab2_busy) pair_wait(4);
#pragma unroll
              for (int i = 0; i < 32; ++i) slab2[i * 128 + lt] = p2[i] * inv;
              slab2[32 * 128 + lt] = p3[0] * inv;
              slab2[33 * 128 + lt] = p3[2] * inv;
              pair_arrive(3);
              slab2_busy = true;
            } else {
              if (pair) pair_wait(3);
              frag_foreach<8>(p3, [&](int r, int c, float x, float) {
                if (c == 0) atomicAdd(G.att_w3[net] + r, pair ? x * inv + slab2[(32 + (r & 8) / 8) * 128 + lt] : x * inv);
              });
              int k = 0;
              frag_foreach<64>(p2, [&](int r, int c, float x, float y) {
                float a = x * inv, b = y * inv;
                if (pair) { a += slab2[k * 128 + lt]; b += slab2[(k + 1) * 128 + lt]; }
                k += 2;
                red2(G.att_w2t[net] + (size_t)r * 64 + c, a, b);
              });
              if (pair) pair_arrive(4);
            }
          }
          // dH1[64 x 64] = dH2 * W2 on this warpgroup's rows
          mma_prop<64>(d, m0, aT3h, aT3l, 8, sb + L.wa2[net], 64);
          float inv2;      // (1 / cs) / r: cs r can pass 2^128, where 1 / (cs r) is 0 rather than a subnormal
          {   // re-scale the propagated delta with its own amax, then dH1 * relu1 -> T2 (H2 is dead: its products have completed)
            float am = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              v[i] = ((m1 >> i) & 1u) ? d[i] : 0.f;
              am = fmaxf(am, fabsf(v[i]));
            }
            am = wg_amax(am, s_w);
            const float r = am > 0.f ? pow2_factor(am) : 1.0f;
            inv2 = (1.0f / cs) / r;
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] *= r;
            frag_put<64>(t2h, t2l, 128, m0, 0, v);
          }
          L4D_PH(4);
          wg_publish();
          {   // dW1g[64 x 16] = dH1^T * [geo,1] over this warpgroup's samples (column 15 is the ones column) and
              // dG[64 x 16] = dH1 * W1g on its rows
            float p1[8], g[8];
            mma_tt64_issue<16>(p1, m0, aT2h, aT2l, aG16h, aG16l);
            mma_prop_issue<16>(g, m0, aT2h, aT2l, 8, sb + L.wa1[net], 64);
            wg_wait<0>();
#pragma unroll
            for (int i = 0; i < 8; ++i) dgeo[i] = fmaf(g[i], inv2, dgeo[i]);
            if (pair && wg == 1) {
              if (slab1_busy) pair_wait(6);
#pragma unroll
              for (int i = 0; i < 8; ++i) slab1[i * 128 + lt] = p1[i] * inv2;
              pair_arrive(5);
              slab1_busy = true;
            } else {
              if (pair) pair_wait(5);
              int k = 0;
              frag_foreach<16>(p1, [&](int r, int c, float x, float y) {
                float a = x * inv2, b = y * inv2;
                if (pair) { a += slab1[k * 128 + lt]; b += slab1[(k + 1) * 128 + lt]; }
                k += 2;
                atomicAdd(G.att_w1t[net] + (size_t)(L4D_ENC + c) * 64 + r, a);
                if (c + 1 < 15) atomicAdd(G.att_w1t[net] + (size_t)(L4D_ENC + c + 1) * 64 + r, b);
                else s_csum[net * 64 + r] += b;
              });
              if (pair) pair_arrive(6);
            }
          }
          L4D_PH(6);
        }
      }

      // ---------------- P3: sigma MLP backward ----------------
      // dO fragment: column 0 = dsigma * d(sigma)/d(out0) (lanes with frag_col() == 0), columns 1..15 = dG
      float ds[2], am = 0.f;
      bool fact[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        fact[h] = (uint32_t)t * 128 + (uint32_t)(fr + 8 * h) < n_steps;
        ds[h] = fact[h] ? s_dsig[fr + 8 * h] * expf(fminf(fmaxf(out[2 * h], -15.f), 15.f)) : 0.f;
        if ((tid & 3) == 0) am = fmaxf(am, fabsf(ds[h]));
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        dgeo[i] = (fact[(i >> 1) & 1] && 8 * (i >> 2) + frag_col() + (i & 1) < 15) ? dgeo[i] : 0.f;
        am = fmaxf(am, fabsf(dgeo[i]));
      }
      const float amax = block_amax256(am, s_w);
      if (amax == 0.f) {           // nothing flows back through this tile
        if (active) for (int kq = half; kq < (int)A.sv.d_quads; kq += 2) *reinterpret_cast<float4*>(dq + (size_t)kq * 512) = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        x_issue_next(ray, t);
        continue;
      }
      if (x_dirty) x_issue(ray, t);      // bring X back for P4 while P3 runs
      const float sc = pow2_factor(amax);
      float inv = 1.0f / sc;
#pragma unroll
      for (int i = 0; i < 8; ++i) dgeo[i] *= sc;
      frag_put16_shift<1>(o16h, o16l, m0, dgeo);
      if ((tid & 3) == 0) {
        tile_put1(o16h, o16l, fr, 0, ds[0] * sc);
        tile_put1(o16h, o16l, fr + 8, 0, ds[1] * sc);
      }
      publish();
      float e[32];
      // dHs[64 x 64] = dO * W2 on this warpgroup's rows  (W2 stored [k/8][16 rows][8])
      mma_prop<64>(e, m0, aO16h, aO16l, 2, sb + L.w2, 16);
      // dW2s^T[64 x 16] = Hs^T * dO (warpgroup w: columns [8w, 8w + 8))
      mma_tt<8>(aHh, aHl, aO16h + (uint32_t)wg * 2048u, aO16l + (uint32_t)wg * 2048u, [&](int r, int c, float x, float y) {
        atomicAdd(G.sig_w2 + (size_t)(8 * wg + c) * 64 + r, x * inv);
        atomicAdd(G.sig_w2 + (size_t)(8 * wg + c + 1) * 64 + r, y * inv);
      });
      {   // re-scale the propagated delta with its own amax, then dHs * relu -> RH (hidden is dead past the barrier)
        float am2 = 0.f, v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          v[i] = ((msk >> i) & 1u) ? e[i] : 0.f;
          am2 = fmaxf(am2, fabsf(v[i]));
        }
        am2 = block_amax256(am2, s_w);
        const float r = am2 > 0.f ? pow2_factor(am2) : 1.0f;
        inv = (1.0f / sc) / r;            // not 1 / (sc r): that is 0 once sc r passes 2^128, (1/sc)/r a subnormal to 2^149
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] *= r;
        frag_put<64>(hh, hl, 128, m0, 0, v);
      }
      L4D_PH(7);
      // ---------------- P4: input gradients and first-layer weight gradient ----------------
      x_wait();
      publish();
      L4D_PH(8);
      {
        // dW1^T[in x 64] = X^T * dHs: feature rows [0,64) on warpgroup 0, [64,128) on warpgroup 1, [128,192) split by columns
        auto flush = [&](int r, int c, float x, float y) {
          if (r < (int)in_pad) red2(G.sig_w1t + (size_t)r * 64 + c, x * inv, y * inv);
        };
        mma_tt<64>(aXh + (uint32_t)wg * 8u * 2048u, aXl + (uint32_t)wg * 8u * 2048u, aHh, aHl,
                   [&](int r, int c, float x, float y) { flush(64 * wg + r, c, x, y); });
        if (in_pad > 128)
          mma_tt<32>(aXh + 16u * 2048u, aXl + 16u * 2048u, aHh + (uint32_t)wg * 4u * 2048u, aHl + (uint32_t)wg * 4u * 2048u,
                     [&](int r, int c, float x, float y) { flush(128 + r, 32 * wg + c, x, y); });
      }
      __syncthreads();
      x_issue_next(ray, t);              // X is free: fetch the next tile behind the input gradients
      L4D_PH(9);
      {
        // dX[64 x in_pad] = dHs * W1 (W1 stored [k/8][64 rows][8]) on this warpgroup's rows -> dfeat, in column blocks of
        // 64 straight from the registers: blocks 0 and 1 in flight together, then block 2.  Every block is waited for
        // before any of its registers is read: storing one block while another is in flight makes ptxas serialize
        // every wgmma of the kernel (C7514).  The last block may read past W1 into the weights that follow it: those
        // columns are not stored.
        const int ncols = (int)A.sv.d_quads * 4;
        auto issue = [&](float (&d)[32], int n0) {
          mma_prop_issue<64>(d, m0, aHh, aHl, 8, sb + L.w1 + (uint32_t)(n0 / 8) * 64u * 16u, 64);
        };
        auto store = [&](const float (&d)[32], int n0) {
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const uint32_t jr = (uint32_t)t * 128 + (uint32_t)(fr + 8 * ((i >> 1) & 1));
            const int col = n0 + 8 * (i >> 2) + frag_col();
            if (jr < n_steps && col < ncols)
              *reinterpret_cast<float2*>(A.sv.dfeat + l4d_dfeat_off(A.sv, ray, jr) + (size_t)(col >> 2) * 512 + (col & 3)) =
                  make_float2(d[i] * inv, d[i + 1] * inv);
          }
        };
        {
          float d0[32], d1[32];
          issue(d0, 0);
          if (ncols > 64) issue(d1, 64);
          wg_wait<0>();
          store(d0, 0);
          if (ncols > 64) store(d1, 64);
        }
        if (ncols > 128) {
          float d[32];
          issue(d, 128);
          wg_wait<0>();
          store(d, 128);
        }
      }
      __syncthreads();
      L4D_PH(11);
    }
    // direction / ones rows of the first attribute layer: dW1t[k][j] += enc[k] * sum_samples dh1[j]
    __syncthreads();
    for (int i = tid; i < 2 * (L4D_ENC + 9) * 64; i += 256) {
      const int net = i / ((L4D_ENC + 9) * 64);
      const int r = (i / 64) % (L4D_ENC + 9), jx = i & 63;
      const float cs = s_csum[net * 64 + jx];
      if (r < L4D_ENC) atomicAdd(G.att_w1t[net] + (size_t)r * 64 + jx, s_enc[r] * cs);
      else atomicAdd(G.att_w1t[net] + (size_t)(M.attr_in_dim + (r - L4D_ENC)) * 64 + jx, cs);
    }
  }
  if (wg == 1) {          // warpgroup 0 has read the last partials handed to it
    if (slab2_busy) pair_wait(4);
    if (slab1_busy) pair_wait(6);
  }
#ifdef L4D_PHASE_CLOCKS
  __syncthreads();
  L4D_PH(12);
  if (tid < 32) atomicAdd(&g_phase_clk[tid], s_clk[tid]);
#endif
}

// =============================================================================================
// flow MLP (16 -> 64 -> 64 -> 6) on tensor cores.  One warpgroup per CTA computes both 64-row blocks of a tile.
// =============================================================================================
struct FlowTcSmem {
  uint32_t w0, w1, w2;       // weights
  uint32_t fin;              // 16-wide tile hi|lo (2 x 4 KB)
  uint32_t t1, t2;           // 64-wide tiles hi|lo (32 KB each); the forward uses t1 only
  uint32_t do16;             // 16-wide delta tile hi|lo
  uint32_t total_fwd, total;
};
__host__ __device__ inline FlowTcSmem flow_tc_smem() {
  FlowTcSmem L;
  uint32_t o = 0;
  auto take = [&](uint32_t b) { uint32_t r = o; o += (b + 127u) & ~127u; return r; };
  L.w0 = take(16 * 64 * 2); L.w1 = take(64 * 64 * 2); L.w2 = take(64 * 16 * 2);
  L.fin = take(2 * 4096);
  L.t1 = take(32 * 1024);
  L.total_fwd = o;
  L.t2 = take(32 * 1024);
  L.do16 = take(2 * 4096);
  L.total = o;
  return L;
}

namespace l4dtc {
__device__ __forceinline__ void flow_copy_weights(unsigned char* dsm, const FlowTcSmem& L, const DevModel& M) {
  auto cp = [&](uint32_t off, const __half* src, uint32_t bytes) {
    for (uint32_t i = threadIdx.x * 16; i < bytes; i += 128 * 16)
      *reinterpret_cast<uint4*>(dsm + off + i) = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(src) + i));
  };
  cp(L.w0, M.tc_flo_w0, 16 * 64 * 2);
  cp(L.w1, M.tc_flo_w1, 64 * 64 * 2);
  cp(L.w2, M.tc_flo_w2, 64 * 16 * 2);
}

// flow MLP forward for the 128 samples of the CTA.  fin[16] per thread (thread == row) in; out: per 64-row block mb the
// first 8 columns of the output fragment, flow[mb][2h + e] = flow[row 64 mb + frag_row() + 8h][frag_col() + e] (6 used),
// and the relu patterns of both hidden layers (frag_relu bits per block).  Leaves relu(layer 2) in tile t1 and, when
// H1_OUT, relu(layer 1) in tile h1.
template <bool H1_OUT>
__device__ __forceinline__ void flow_forward_tc(unsigned char* dsm, uint32_t sb, const FlowTcSmem& L, const float (&fin)[16],
                                                float (&flow)[2][4], uint32_t (&m1)[2], uint32_t (&m2)[2], unsigned char* h1_hi,
                                                unsigned char* h1_lo, uint32_t a_h1_hi, uint32_t a_h1_lo) {
  const int tid = threadIdx.x;
  unsigned char *fh = dsm + L.fin, *fl = fh + 4096, *t1h = dsm + L.t1, *t1l = t1h + 16384;
  unsigned char *y1h = H1_OUT ? h1_hi : t1h, *y1l = H1_OUT ? h1_lo : t1l;
  const uint32_t a_y1h = H1_OUT ? a_h1_hi : sb + L.t1, a_y1l = H1_OUT ? a_h1_lo : sb + L.t1 + 16384u;
  tile_put8(fh, fl, tid, 0, fin);
  tile_put8(fh, fl, tid, 1, fin + 8);
  publish();
#pragma unroll
  for (int mb = 0; mb < 2; ++mb) {
    float d[32];
    mma_rows<64>(d, 64 * mb, sb + L.fin, sb + L.fin + 4096u, sb + L.w0, 64, 2);
    m1[mb] = frag_relu<64>(d, d);
    frag_put<64>(y1h, y1l, 128, 64 * mb, 0, d);
  }
  publish();
#pragma unroll
  for (int mb = 0; mb < 2; ++mb) {
    float d[32];
    mma_rows<64>(d, 64 * mb, a_y1h, a_y1l, sb + L.w1, 64, 8);
    m2[mb] = frag_relu<64>(d, d);
    if (!H1_OUT) __syncthreads();        // layer 2 overwrites its own input rows
    frag_put<64>(t1h, t1l, 128, 64 * mb, 0, d);
  }
  publish();
#pragma unroll
  for (int mb = 0; mb < 2; ++mb) {
    float o[8];
    mma_rows<16>(o, 64 * mb, sb + L.t1, sb + L.t1 + 16384u, sb + L.w2, 16, 8);
#pragma unroll
    for (int i = 0; i < 4; ++i) flow[mb][i] = o[i];
  }
}
}  // namespace l4dtc

// -------------------------------------------------------------------------------------------
// forward 0/2: flow field on tensor cores (flow-grid gather + 16->64->64->6 MLP), tiles of 128 consecutive
// samples; writes the flow-MLP inputs and the flow.  Kept apart from the feature gather on purpose: the MMA
// round trips need block-wide barriers, and barriers around the long, irregular feature gathers stall warps
// that would otherwise run free (measured: fusing them doubled the forward at L=16).
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 4) k_fwd_flow_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  const DevModel& M = A.M;
  const int tid = threadIdx.x;
  const FlowTcSmem L = flow_tc_smem();
  const uint32_t sb = smem_u32(dsm);
  flow_copy_weights(dsm, L, M);
  publish();
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  for (size_t base = (size_t)blockIdx.x * 128; base < P; base += (size_t)gridDim.x * 128) {
    const size_t pp = base + tid;
    const bool active = pp < P;
    const size_t p = active ? pp : P - 1;
    const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
    const float zj = l4d_z(rs, A.ray_offset + ray, j);
    const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
    const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
    const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
    const float* b = A.FT.frames[l4d_frame_of(A.FT, ray)].flow_basis;
    float fin[16];
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      float e[8];
      l4d_encode3_f8(M.gf, M.hf, l, x, y, z, e);
      fin[2 * l] = ((b[0] * e[0] + b[1] * e[2]) + b[2] * e[4]) + b[3] * e[6];
      fin[2 * l + 1] = ((b[0] * e[1] + b[1] * e[3]) + b[2] * e[5]) + b[3] * e[7];
    }
    if (active) {
#pragma unroll
      for (int k = 0; k < 16; ++k) A.sv.flow_in[(size_t)k * P + p] = fin[k];
    }
    float flow[2][4];
    uint32_t m1[2], m2[2];
    flow_forward_tc<false>(dsm, sb, L, fin, flow, m1, m2, nullptr, nullptr, 0u, 0u);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const size_t q = base + 64 * mb + frag_row() + 8 * (i >> 1);
        const int k = frag_col() + (i & 1);
        if (k < 6 && q < P) A.sv.flow[(size_t)k * P + q] = flow[mb][i];
      }
    __syncthreads();
  }
}

// -------------------------------------------------------------------------------------------
// backward 3/4 on tensor cores: flow MLP backprop + weight gradients; dL/d(flow-MLP input) -> flow_in planes
// Two 64-wide tiles are enough (each delta tile overwrites the activation tile that has just been consumed).
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 2) k_bwd_flow_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  __shared__ float s_w[32];
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  const FlowTcSmem L = flow_tc_smem();
  const uint32_t sb = smem_u32(dsm);
  unsigned char *t1h = dsm + L.t1, *t1l = t1h + 16384, *t2h = dsm + L.t2, *t2l = t2h + 16384;
  unsigned char *o16h = dsm + L.do16, *o16l = o16h + 4096;
  const uint32_t aFinH = sb + L.fin, aFinL = aFinH + 4096u;
  const uint32_t aT1h = sb + L.t1, aT1l = aT1h + 16384u, aT2h = sb + L.t2, aT2l = aT2h + 16384u;
  const uint32_t aO16h = sb + L.do16, aO16l = aO16h + 4096u;
  flow_copy_weights(dsm, L, M);
  publish();
  const size_t P = A.sv.P;
  for (size_t base = (size_t)blockIdx.x * 128; base < P; base += (size_t)gridDim.x * 128) {
    const size_t pp = base + tid;
    const bool active = pp < P;
    const size_t p = active ? pp : P - 1;
    float fin[16], g[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) fin[k] = active ? __ldg(A.sv.flow_in + (size_t)k * P + p) : 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) g[k] = (active && k < 6) ? __ldg(A.sv.dflow + (size_t)k * P + p) : 0.f;
    float am = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) am = fmaxf(am, fabsf(g[k]));
    am = block_amax128(am, s_w);
    if (am == 0.f) {                               // no gradient reaches the flow field from this tile
      if (active) {
#pragma unroll
        for (int k = 0; k < 16; ++k) A.sv.flow_in[(size_t)k * P + p] = 0.f;
      }
      continue;
    }
    // forward recompute: relu(layer 1) -> T2, relu(layer 2) -> T1, relu patterns
    float flow[2][4];
    uint32_t m1[2], m2[2];
    flow_forward_tc<true>(dsm, sb, L, fin, flow, m1, m2, t2h, t2l, aT2h, aT2l);
    const float sc = pow2_factor(am);
    float inv = 1.0f / sc;
#pragma unroll
    for (int k = 0; k < 16; ++k) g[k] *= sc;
    tile_put8(o16h, o16l, tid, 0, g);
    tile_put8(o16h, o16l, tid, 1, g + 8);
    publish();
    float d[2][32];
    // dH2[128 x 64] = dO * W2 (W2 stored [k/8][16 rows][8]) ; dW2^T[64 x 16] = H2^T * dO
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) mma_prop<64>(d[mb], 64 * mb, aO16h, aO16l, 2, sb + L.w2, 16);
    mma_tt<16>(aT1h, aT1l, aO16h, aO16l, [&](int r, int c, float x, float y) {
      if (c < 6) atomicAdd(G.flo_w2 + (size_t)c * 64 + r, x * inv);
      if (c + 1 < 6) atomicAdd(G.flo_w2 + (size_t)(c + 1) * 64 + r, y * inv);
    });
    // dH2 * relu2, re-scaled -> T1 (H2 is dead once every thread is past the barrier in block_amax128)
    float a2 = 0.f;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        d[mb][i] = ((m2[mb] >> i) & 1u) ? d[mb][i] : 0.f;
        a2 = fmaxf(a2, fabsf(d[mb][i]));
      }
    a2 = block_amax128(a2, s_w);
    float r = a2 > 0.f ? pow2_factor(a2) : 1.0f;
    const float inv2 = (1.0f / sc) / r;      // not 1 / (sc r): that is 0 once sc r passes 2^128
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
      for (int i = 0; i < 32; ++i) d[mb][i] *= r;
      frag_put<64>(t1h, t1l, 128, 64 * mb, 0, d[mb]);
    }
    inv = inv2;
    publish();
    // dH1[128 x 64] = dH2 * W1 ; dW1^T[64 x 64] = H1^T * dH2
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) mma_prop<64>(d[mb], 64 * mb, aT1h, aT1l, 8, sb + L.w1, 64);
    mma_tt<64>(aT2h, aT2l, aT1h, aT1l, [&](int r, int c, float x, float y) {
      red2(G.flo_w1t + (size_t)r * 64 + c, x * inv, y * inv);
    });
    // dH1 * relu1, re-scaled -> T2 (H1 is dead once every thread is past the barrier in block_amax128)
    float a3 = 0.f;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        d[mb][i] = ((m1[mb] >> i) & 1u) ? d[mb][i] : 0.f;
        a3 = fmaxf(a3, fabsf(d[mb][i]));
      }
    a3 = block_amax128(a3, s_w);
    r = a3 > 0.f ? pow2_factor(a3) : 1.0f;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
      for (int i = 0; i < 32; ++i) d[mb][i] *= r;
      frag_put<64>(t2h, t2l, 128, 64 * mb, 0, d[mb]);
    }
    inv = inv2 / r;
    publish();
    // dFin[128 x 16] = dH1 * W0 ; dW0[64 x 16] = dH1^T * Fin
    // dL/d(flow-MLP input) replaces the saved input in place (every thread read its row above); k_bwd_flowgrid turns it
    // into flow-grid reductions at full occupancy
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      float o[8];
      mma_prop<16>(o, 64 * mb, aT2h, aT2l, 8, sb + L.w0, 64);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const size_t q = base + 64 * mb + frag_row() + 8 * ((i >> 1) & 1);
        const int k = 8 * (i >> 2) + frag_col() + (i & 1);
        if (q < P) A.sv.flow_in[(size_t)k * P + q] = o[i] * inv;
      }
    }
    mma_tt<16>(aT2h, aT2l, aFinH, aFinL, [&](int r, int c, float x, float y) {
      atomicAdd(G.flo_w0t + (size_t)c * 64 + r, x * inv);
      atomicAdd(G.flo_w0t + (size_t)(c + 1) * 64 + r, y * inv);
    });
    __syncthreads();
  }
}
