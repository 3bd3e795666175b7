// l4d_dense_tc.cuh - tensor-core (wgmma) versions of the dense kernels of the split pipeline.
// Requires mlp_fp16 (MLP weights are fp16 working copies, as tiny-cuda-nn keeps them).
//
// Tile = 128 samples; in the epilogues thread (threadIdx.x % 128) owns sample row.
// Operands live in shared memory as fp16 in the K-major interleaved layout of l4d_tc.cuh
// ([k/8][row][8 halves], 16-byte chunks).  Activations are carried as hi + lo fp16 pairs
// (x = hi + lo to ~2^-22 relative), i.e. every product with an fp16 weight is exact and the fp32
// accumulation reproduces the fp32-FMA kernels to ~1e-6: the 1e-4 parity bar holds on the
// tensor-core path too.  Every warpgroup issues the wgmma of its 64-row block; activation products
// go through the fp32 staging tile (one row per thread), weight gradients are flushed with fp32
// atomics straight from the accumulator registers.
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

// The products below are called by every thread of the CTA; the warpgroups split the two 64-row blocks of a
// 128-sample product.  A thread may read the staging tile only after the __syncthreads() that follows.
//
// D[128 x N] = (Ah + Al) * B^T over n_chunks 16-byte k-chunks (n_chunks even): A = 128-row tiles (chunk stride 2048),
// B = K-major [k/8][b_rows][8] (b points at its first used row) -> staging columns [c0, c0 + N)
template <int N>
__device__ __forceinline__ void mma_rows(float* S, int c0, uint32_t a_hi, uint32_t a_lo, uint32_t b, uint32_t b_rows, int n_chunks) {
  for (int mb = threadIdx.x >> 7; mb < 2; mb += blockDim.x >> 7) {
    const Opnd a{{a_hi + (uint32_t)mb * 1024u, a_lo + (uint32_t)mb * 1024u, 0u}, 4096u, 2048u, 128u};
    const Opnd w{{b, b, 0u}, 2u * b_rows * 16u, b_rows * 16u, 128u};
    float d[N / 2];
    wg_gemm<N, 0, 0>(d, a, w, 2, n_chunks / 2);
    acc_store<N>(S, d, 64 * mb, c0);
  }
}
// D[128 x N] = (Ah + Al) * W: W stored [k_in/8][w_rows][8] (forward layout) and read as B(n = k_in, k = row), i.e.
// MN-major; w points at the chunk of the first k_in column used.  f(row, col, v[col], v[col + 1]) per element pair.
template <int N, class F>
__device__ __forceinline__ void mma_prop_frag(uint32_t a_hi, uint32_t a_lo, int n_chunks, uint32_t w, uint32_t w_rows, F&& f) {
  for (int mb = threadIdx.x >> 7; mb < 2; mb += blockDim.x >> 7) {
    const Opnd a{{a_hi + (uint32_t)mb * 1024u, a_lo + (uint32_t)mb * 1024u, 0u}, 4096u, 2048u, 128u};
    const Opnd b{{w, w, 0u}, 256u, 128u, w_rows * 16u};
    float d[N / 2];
    wg_gemm<N, 0, 1>(d, a, b, 2, n_chunks / 2);
    frag_foreach<N>(d, [&](int r, int c, float x, float y) { f(64 * mb + r, c, x, y); });
  }
}
template <int N>
__device__ __forceinline__ void mma_prop(float* S, int c0, uint32_t a_hi, uint32_t a_lo, int n_chunks, uint32_t w, uint32_t w_rows) {
  mma_prop_frag<N>(a_hi, a_lo, n_chunks, w, w_rows, [&](int r, int c, float x, float y) {
    *reinterpret_cast<float2*>(S + acc_idx(r, c0 + c)) = make_float2(x, y);
  });
}

}  // namespace l4dtc

// smem carve-up of the dense forward kernel (bytes)
struct DenseFwdSmem {
  uint32_t w1, w2, wa1, wa2[2];     // weights
  uint32_t xh, xl;                  // feature tile (later reused for the 128-wide attribute hidden tile)
  uint32_t hh, hl;                  // 64-wide hidden tile
  uint32_t gh, gl;                  // 16-wide tile (geo)
  uint32_t misc;                    // enc[80] cdir[128] w[32] floats
  uint32_t acc;                     // fp32 staging tile
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
  L.misc = take((80 + 128 + 32) * 4);
  L.acc = take(l4dtc::acc_tile_bytes());
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
// Shared memory at sigma_in_pad = 176 (L = 16): 226 KB, within the 227 KB an sm_90 CTA may use; one CTA per SM.
// =============================================================================================
struct DenseBwdSmem {
  uint32_t w1, w2, wa1[2], wa2[2];
  uint32_t R;            // 96 KB: X hi|lo (24 chunks each) or T1,T2,T3 (hi|lo, 8 chunks each)
  uint32_t RH;           // 32 KB: sigma hidden hi|lo, later its delta
  uint32_t g16, do16, do8;   // small tiles, hi|lo
  uint32_t misc;
  uint32_t acc;          // 32 KB fp32 staging tile
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
  L.misc = take((80 + 128 + 128 + 128 + 32 + 64) * 4);
  L.acc = take(l4dtc::acc_tile_bytes());
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
  return ldexpf(1.0f, 6 - e);
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
// forward 2/2 on tensor cores: sigma MLP, compositing, attribute heads.  One CTA per ray, 256 threads: two threads per
// row (sample) split the columns of every epilogue; in the attribute phase thread half h owns head h, and the heads'
// products pass through the 64-column staging tile one after the other.
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
  float* S = reinterpret_cast<float*>(dsm + L.acc);
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
      mma_rows<64>(S, 0, sb + L.xh, sb + L.xl, sb + L.w1, 64, n_xchunks);
      __syncthreads();
      // ---- hidden = relu(.) -> hi/lo tile (each half its 32 columns) ----
#pragma unroll
      for (int qq = 0; qq < 2; ++qq) {
        const int q = 2 * half + qq;
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
        tile_put8(hh, hl, row, 2 * q, v);
        tile_put8(hh, hl, row, 2 * q + 1, v + 8);
      }
      publish();
      mma_rows<16>(S, 0, sb + L.hh, sb + L.hl, sb + L.w2, 16, 8);
      __syncthreads();
      float out[16];
      acc_ld16(S, 0, out);
      float zj = 0.f, alpha = 0.f, sigma = 0.f;
      if (valid) {
        sigma = expf(out[0]);
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
        {
          float g8[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float gv = half ? (i < 7 ? out[9 + i] : 0.f) : out[1 + i];      // geo[0..7] | geo[8..14], 0
            g8[i] = masked ? gv : 0.f;
          }
          tile_put8(gh, gl, row, half, g8);
        }
        publish();
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {    // 128 columns: net0 hidden | net1 hidden -> chunks 0..15 of the x tile
          mma_rows<64>(S, 0, sb + L.gh, sb + L.gl, sb + L.wa1 + (uint32_t)net * 64u * 16u, 128, 2);
          __syncthreads();
          if (half == net) {
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              const int q = 4 * half + qq;
              float v[16];
              acc_ld16(S, qq * 16, v);
#pragma unroll
              for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i] + s_cdir[q * 16 + i], 0.f);
              tile_put8(xh, xl, row, 2 * q, v);
              tile_put8(xh, xl, row, 2 * q + 1, v + 8);
            }
          }
          publish();
        }
        float o = 0.f;
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {
          mma_rows<64>(S, 0, sb + L.xh + (uint32_t)net * 8u * 2048u, sb + L.xl + (uint32_t)net * 8u * 2048u, sb + L.wa2[net], 64, 8);
          __syncthreads();
          if (half == net) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float v[16];
              acc_ld16(S, q * 16, v);
#pragma unroll
              for (int i = 0; i < 16; ++i) o = fmaf(fmaxf(v[i], 0.f), l4d_ld1(M.att_w3[half] + q * 16 + i), o);
            }
          }
          __syncthreads();
        }
        x_issue_next(ray, j0 >> 7);                    // the attribute hidden tile (in the X buffer) has been consumed
        if (masked) a = l4d_sigmoid(o);
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
      __syncthreads();          // the staging tile and the operand tiles are reused by the next tile
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

// 256 threads, two threads per row that split the columns of every epilogue: twice the warps to hide latency, and one
// warpgroup per 64-row block of every 128-sample product.
__global__ void __launch_bounds__(256) k_bwd_dense_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  __shared__ __align__(8) uint64_t s_xbar;
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  const int row = tid & 127, half = tid >> 7;     // two threads per row: `half` owns columns [32*half, 32*half+32) of every 64-wide block
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
  float* s_tstart = s_w + 32;
  float* S = reinterpret_cast<float*>(dsm + L.acc);
  // the attribute phase's per-row dot-product exchange lives in the dO8 tile, which is dead while it is used
  float* s_part = reinterpret_cast<float*>(o8h);
  __shared__ float s_w3max[2];
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
  publish();
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t n_steps = A.S;
  const int n_tiles = (int)((n_steps + 127) / 128);
  const float kk = M.active_sensor ? 2.0f : 1.0f;
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
    const float gd = __ldg(A.g_depth + ray), gi0 = __ldg(A.g_image + 2 * ray), gi1 = __ldg(A.g_image + 2 * ray + 1);
    const float gws = A.g_wsum ? __ldg(A.g_wsum + ray) : 0.f;
    const uint64_t rg = A.ray_offset + ray;
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
    __syncthreads();
    // transmittance at the start of every tile: saved by k_fwd_dense_tc
    for (int t = tid; t < n_tiles; t += 256) s_tstart[t] = __ldg(A.sv.tstart + (size_t)ray * A.sv.n_tiles + t);
    __syncthreads();
    L4D_PH(0);
    float suffix = 0.f;
    for (int t = n_tiles - 1; t >= 0; --t) {
      const uint32_t j = (uint32_t)t * 128 + row;
      const bool active = j < n_steps;
      const size_t p = (size_t)ray * n_steps + (active ? j : 0);
      bool masked = false;
      float dsigma = 0.f, da[2] = {0.f, 0.f};
      {
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
        const float T = s_tstart[t] * half_excl_prod(v, s_w, total);
        const float w = alpha * T;
        const float suf = suffix + half_excl_suffix_sum(gw * w, s_w, qtot);
        suffix += qtot;
        if (active) {
          dsigma = (gw * T - suf / v) * (kk * delta * M.density_scale) * (1.0f - alpha);
          masked = w > 1e-4f;
          if (masked) { da[0] = w * gi0; da[1] = w * gi1; }
        }
      }

      L4D_PH(1);
      // ---------------- P1: sigma MLP forward ----------------
      x_wait();
      publish();
      L4D_PH(2);
      mma_rows<64>(S, 0, aXh, aXl, sb + L.w1, 64, n_xchunks);
      __syncthreads();
      uint32_t msk = 0u;                       // relu pattern of this half's 32 hidden units
#pragma unroll
      for (int qq = 0; qq < 2; ++qq) {
        const int q = 2 * half + qq;
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const bool on = v[i] > 0.f;
          v[i] = on ? v[i] : 0.f;
          msk |= on ? (1u << (qq * 16 + i)) : 0u;
        }
        tile_put8(hh, hl, row, 2 * q, v);
        tile_put8(hh, hl, row, 2 * q + 1, v + 8);
      }
      publish();
      mma_rows<16>(S, 0, aHh, aHl, sb + L.w2, 16, 8);
      __syncthreads();
      float out[16], dgeo[16];
      acc_ld16(S, 0, out);
#pragma unroll
      for (int i = 0; i < 16; ++i) dgeo[i] = 0.f;

      L4D_PH(3);
      // ---------------- P2: attribute heads ----------------
      bool x_dirty = false;          // the attribute phase reuses the X buffer for its tiles
      if (__syncthreads_or(masked ? 1 : 0)) {
        {   // [geo, 1] tile (zero rows for samples outside the attribute mask)
          float g[16];
#pragma unroll
          for (int i = 0; i < 15; ++i) g[i] = masked ? out[1 + i] : 0.f;
          g[15] = masked ? 1.0f : 0.f;
          float g8[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) g8[i] = half ? g[8 + i] : g[i];
          tile_put8(g16h, g16l, row, half, g8);
        }
#pragma unroll 1
        for (int net = 0; net < 2; ++net) {
          if (block_amax256(da[net], s_w) == 0.f) continue;       // no gradient reaches this head in this tile
          x_dirty = true;
          publish();
          mma_rows<64>(S, 0, aG16h, aG16l, sb + L.wa1[net], 64, 2);
          __syncthreads();
          uint32_t m1 = 0u;
#pragma unroll
          for (int qq = 0; qq < 2; ++qq) {
            const int q = 2 * half + qq;
            float v[16];
            acc_ld16(S, q * 16, v);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float y = v[i] + s_cdir2[net * 64 + q * 16 + i];
              const bool on = y > 0.f;
              v[i] = on ? y : 0.f;
              m1 |= on ? (1u << (qq * 16 + i)) : 0u;
            }
            tile_put8(t1h, t1l, row, 2 * q, v);
            tile_put8(t1h, t1l, row, 2 * q + 1, v + 8);
          }
          publish();
          mma_rows<64>(S, 0, aT1h, aT1l, sb + L.wa2[net], 64, 8);
          __syncthreads();
          float cs = 1.0f;
          {   // output layer (fp32), sigmoid backward, delta of the second hidden layer
            float o = 0.f;
            uint32_t m2 = 0u;
#pragma unroll
            for (int qq = 0; qq < 2; ++qq) {
              const int q = 2 * half + qq;
              float v[16];
              acc_ld16(S, q * 16, v);
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const bool on = v[i] > 0.f;
                v[i] = on ? v[i] : 0.f;
                m2 |= on ? (1u << (qq * 16 + i)) : 0u;
                o = fmaf(v[i], l4d_ld1(M.att_w3[net] + q * 16 + i), o);
              }
              tile_put8(t2h, t2l, row, 2 * q, v);
              tile_put8(t2h, t2l, row, 2 * q + 1, v + 8);
            }
            s_part[half * 128 + row] = o;           // the two halves of the row exchange their partial dot products
            __syncthreads();
            o = s_part[row] + s_part[128 + row];
            const float a = l4d_sigmoid(o);
            const float d_raw = masked ? da[net] * a * (1.0f - a) : 0.f;
            // per-tile power-of-two scale of the delta tiles (|w3| <= w3max bounds the second tile too)
            const float am = block_amax256(d_raw * s_w3max[net], s_w);
            cs = am > 0.f ? pow2_factor(am) : 1.0f;
            const float d_o = d_raw * cs;
            if (half == 0) {
              float d8[8] = {d_o, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
              tile_put8(o8h, o8l, row, 0, d8);
            }
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              const int q = 4 * half + qq;
              float v[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) v[i] = ((m2 >> (qq * 8 + i)) & 1u) ? l4d_ld1(M.att_w3[net] + q * 8 + i) * d_o : 0.f;
              tile_put8(t3h, t3l, row, q, v);
            }
          }
          publish();
          const float inv = 1.0f / cs;
          // dw3^T[64 x 8] = H2^T * dO (column 0 carries dO; warpgroup 0)
          if (wg == 0)
            mma_tt<8>(aT2h, aT2l, aO8h, aO8l, [&](int r, int c, float x, float) {
              if (c == 0) atomicAdd(G.att_w3[net] + r, x * inv);
            });
          // dW2^T[64 x 64] = H1^T * dH2 (warpgroup w: columns [32w, 32w + 32))
          mma_tt<32>(aT1h, aT1l, aT3h + (uint32_t)wg * 4u * 2048u, aT3l + (uint32_t)wg * 4u * 2048u, [&](int r, int c, float x, float y) {
            red2(G.att_w2t[net] + (size_t)r * 64 + 32 * wg + c, x * inv, y * inv);
          });
          // dH1[128 x 64] = dH2 * W2
          mma_prop<64>(S, 0, aT3h, aT3l, 8, sb + L.wa2[net], 64);
          __syncthreads();
          float cs2;
          {   // re-scale the propagated delta with its own amax, then dH1 * relu1 -> T2 (H2 is dead)
            float am = 0.f;
            float vv[2][16];
#pragma unroll
            for (int qq = 0; qq < 2; ++qq) {
              acc_ld16(S, (2 * half + qq) * 16, vv[qq]);
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                vv[qq][i] = ((m1 >> (qq * 16 + i)) & 1u) ? vv[qq][i] : 0.f;
                am = fmaxf(am, fabsf(vv[qq][i]));
              }
            }
            am = block_amax256(am, s_w);
            const float r = am > 0.f ? pow2_factor(am) : 1.0f;
            cs2 = cs * r;
#pragma unroll
            for (int qq = 0; qq < 2; ++qq) {
              const int q = 2 * half + qq;
#pragma unroll
              for (int i = 0; i < 16; ++i) vv[qq][i] *= r;
              tile_put8(t2h, t2l, row, 2 * q, vv[qq]);
              tile_put8(t2h, t2l, row, 2 * q + 1, vv[qq] + 8);
            }
          }
          const float inv2 = 1.0f / cs2;
          L4D_PH(4);
          L4D_PH(5);
          publish();
          // dW1g[64 x 16] = dH1^T * [geo,1] (warpgroup w: columns [8w, 8w + 8); column 15 is the ones column)
          mma_tt<8>(aT2h, aT2l, aG16h + (uint32_t)wg * 2048u, aG16l + (uint32_t)wg * 2048u, [&](int r, int c, float x, float y) {
            const int ii = 8 * wg + c;
            atomicAdd(G.att_w1t[net] + (size_t)(L4D_ENC + ii) * 64 + r, x * inv2);
            if (ii + 1 < 15) atomicAdd(G.att_w1t[net] + (size_t)(L4D_ENC + ii + 1) * 64 + r, y * inv2);
            else s_csum[net * 64 + r] += y * inv2;
          });
          // dG[128 x 16] = dH1 * W1g
          mma_prop<16>(S, 0, aT2h, aT2l, 8, sb + L.wa1[net], 64);
          __syncthreads();
          {
            float v[16];
            acc_ld16(S, 0, v);
#pragma unroll
            for (int i = 0; i < 15; ++i) dgeo[i] = fmaf(v[i], inv2, dgeo[i]);
          }
          __syncthreads();
          L4D_PH(6);
        }
      }

      // ---------------- P3: sigma MLP backward ----------------
      float d16[16];
      d16[0] = active ? dsigma * expf(fminf(fmaxf(out[0], -15.f), 15.f)) : 0.f;
#pragma unroll
      for (int i = 0; i < 15; ++i) d16[1 + i] = active ? dgeo[i] : 0.f;
      float am = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) am = fmaxf(am, fabsf(d16[i]));
      const float amax = block_amax256(am, s_w);
      float* dq = A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j);     // this row in the dfeat tile (float4 per 4 features)
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
      for (int i = 0; i < 16; ++i) d16[i] *= sc;
      {
        float d8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d8[i] = half ? d16[8 + i] : d16[i];
        tile_put8(o16h, o16l, row, half, d8);
      }
      publish();
      // dHs[128 x 64] = dO * W2   (W2 stored [k/8][16 rows][8])
      mma_prop<64>(S, 0, aO16h, aO16l, 2, sb + L.w2, 16);
      // dW2s^T[64 x 16] = Hs^T * dO (warpgroup w: columns [8w, 8w + 8))
      mma_tt<8>(aHh, aHl, aO16h + (uint32_t)wg * 2048u, aO16l + (uint32_t)wg * 2048u, [&](int r, int c, float x, float y) {
        atomicAdd(G.sig_w2 + (size_t)(8 * wg + c) * 64 + r, x * inv);
        atomicAdd(G.sig_w2 + (size_t)(8 * wg + c + 1) * 64 + r, y * inv);
      });
      __syncthreads();
      {   // re-scale the propagated delta with its own amax, then dHs * relu -> RH (hidden is dead)
        float am2 = 0.f;
        float vv[2][16];
#pragma unroll
        for (int qq = 0; qq < 2; ++qq) {
          acc_ld16(S, (2 * half + qq) * 16, vv[qq]);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            vv[qq][i] = ((msk >> (qq * 16 + i)) & 1u) ? vv[qq][i] : 0.f;
            am2 = fmaxf(am2, fabsf(vv[qq][i]));
          }
        }
        am2 = block_amax256(am2, s_w);
        const float r = am2 > 0.f ? pow2_factor(am2) : 1.0f;
        inv = 1.0f / (sc * r);
#pragma unroll
        for (int qq = 0; qq < 2; ++qq) {
          const int q = 2 * half + qq;
#pragma unroll
          for (int i = 0; i < 16; ++i) vv[qq][i] *= r;
          tile_put8(hh, hl, row, 2 * q, vv[qq]);
          tile_put8(hh, hl, row, 2 * q + 1, vv[qq] + 8);
        }
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
      // dX[128 x in_pad] = dHs * W1 (W1 stored [k/8][64 rows][8]) -> dfeat, 16 columns at a time straight from the registers
      for (int n0 = 0; n0 < (int)A.sv.d_quads * 4; n0 += 16) {
        mma_prop_frag<16>(aHh, aHl, 8, sb + L.w1 + (uint32_t)(n0 / 8) * 64u * 16u, 64, [&](int r, int c, float x, float y) {
          const uint32_t jr = (uint32_t)t * 128 + (uint32_t)r;
          const int col = n0 + c;
          if (jr < n_steps && col < (int)A.sv.d_quads * 4)
            *reinterpret_cast<float2*>(A.sv.dfeat + l4d_dfeat_off(A.sv, ray, jr) + (size_t)(col >> 2) * 512 + (col & 3)) =
                make_float2(x * inv, y * inv);
        });
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
#ifdef L4D_PHASE_CLOCKS
  __syncthreads();
  L4D_PH(12);
  if (tid < 32) atomicAdd(&g_phase_clk[tid], s_clk[tid]);
#endif
}

// =============================================================================================
// flow MLP (16 -> 64 -> 64 -> 6) on tensor cores
// =============================================================================================
struct FlowTcSmem {
  uint32_t w0, w1, w2;       // weights
  uint32_t fin;              // 16-wide tile hi|lo (2 x 4 KB)
  uint32_t t1, t2;           // 64-wide tiles hi|lo (32 KB each); the forward uses t1 only
  uint32_t acc;              // fp32 staging tile
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
  L.acc = take(l4dtc::acc_tile_bytes());
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

// flow MLP forward for the 128 samples of the CTA.  fin[16] per thread in, flow[8] out (6 used).
// Optionally returns the relu patterns and leaves relu(layer-2) in tile t1 and (when H1_OUT) relu(layer-1) in tile h1_out.
template <bool H1_OUT>
__device__ __forceinline__ void flow_forward_tc(unsigned char* dsm, uint32_t sb, const FlowTcSmem& L, float* S,
                                                const float (&fin)[16], float (&flow)[8], uint32_t& m1a,
                                                uint32_t& m1b, uint32_t& m2a, uint32_t& m2b, unsigned char* h1_hi,
                                                unsigned char* h1_lo, uint32_t a_h1_hi, uint32_t a_h1_lo) {
  const int tid = threadIdx.x;
  unsigned char *fh = dsm + L.fin, *fl = fh + 4096, *t1h = dsm + L.t1, *t1l = t1h + 16384;
  unsigned char *y1h = H1_OUT ? h1_hi : t1h, *y1l = H1_OUT ? h1_lo : t1l;
  const uint32_t a_y1h = H1_OUT ? a_h1_hi : sb + L.t1, a_y1l = H1_OUT ? a_h1_lo : sb + L.t1 + 16384u;
  tile_put8(fh, fl, tid, 0, fin);
  tile_put8(fh, fl, tid, 1, fin + 8);
  publish();
  mma_rows<64>(S, 0, sb + L.fin, sb + L.fin + 4096u, sb + L.w0, 64, 2);
  __syncthreads();
  m1a = m1b = m2a = m2b = 0u;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float v[16];
    acc_ld16(S, q * 16, v);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int k = q * 16 + i;
      const bool on = v[i] > 0.f;
      v[i] = on ? v[i] : 0.f;
      if (k < 32) m1a |= on ? (1u << k) : 0u; else m1b |= on ? (1u << (k - 32)) : 0u;
    }
    tile_put8(y1h, y1l, tid, 2 * q, v);
    tile_put8(y1h, y1l, tid, 2 * q + 1, v + 8);
  }
  publish();
  mma_rows<64>(S, 0, a_y1h, a_y1l, sb + L.w1, 64, 8);
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float v[16];
    acc_ld16(S, q * 16, v);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int k = q * 16 + i;
      const bool on = v[i] > 0.f;
      v[i] = on ? v[i] : 0.f;
      if (k < 32) m2a |= on ? (1u << k) : 0u; else m2b |= on ? (1u << (k - 32)) : 0u;
    }
    tile_put8(t1h, t1l, tid, 2 * q, v);
    tile_put8(t1h, t1l, tid, 2 * q + 1, v + 8);
  }
  publish();
  mma_rows<16>(S, 0, sb + L.t1, sb + L.t1 + 16384u, sb + L.w2, 16, 8);
  __syncthreads();
  float o[16];
  acc_ld16(S, 0, o);
#pragma unroll
  for (int k = 0; k < 8; ++k) flow[k] = o[k];
}
}  // namespace l4dtc

// -------------------------------------------------------------------------------------------
// forward 0/2: flow field on tensor cores (flow-grid gather + 16->64->64->6 MLP), tiles of 128 consecutive
// samples; writes the flow-MLP inputs and the flow.  Kept apart from the feature gather on purpose: the MMA
// round trips need block-wide barriers, and barriers around the long, irregular feature gathers stall warps
// that would otherwise run free (measured: fusing them doubled the forward at L=16).
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 2) k_fwd_flow_tc(const __grid_constant__ SplitArgs A) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char dsm[];
  const DevModel& M = A.M;
  const int tid = threadIdx.x;
  const FlowTcSmem L = flow_tc_smem();
  const uint32_t sb = smem_u32(dsm);
  float* S = reinterpret_cast<float*>(dsm + L.acc);
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
    float fin[16];
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      float e[8];
      l4d_encode3_f8(M.gf, M.hf, l, x, y, z, e);
      const float* b = A.F.flow_basis;
      fin[2 * l] = ((b[0] * e[0] + b[1] * e[2]) + b[2] * e[4]) + b[3] * e[6];
      fin[2 * l + 1] = ((b[0] * e[1] + b[1] * e[3]) + b[2] * e[5]) + b[3] * e[7];
    }
    if (active) {
#pragma unroll
      for (int k = 0; k < 16; ++k) A.sv.flow_in[(size_t)k * P + p] = fin[k];
    }
    float flow[8];
    uint32_t a, b, c, d;
    flow_forward_tc<false>(dsm, sb, L, S, fin, flow, a, b, c, d, nullptr, nullptr, 0u, 0u);
    if (active) {
#pragma unroll
      for (int k = 0; k < 6; ++k) A.sv.flow[(size_t)k * P + p] = flow[k];
    }
    __syncthreads();
  }
}

// -------------------------------------------------------------------------------------------
// backward 3/4 on tensor cores: flow MLP backprop + weight gradients; dL/d(flow-MLP input) -> flow_in planes
// Two 64-wide tiles are enough (each delta tile overwrites the activation tile that has just been consumed).
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_bwd_flow_tc(const __grid_constant__ SplitArgs A) {
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
  float* S = reinterpret_cast<float*>(dsm + L.acc);
  flow_copy_weights(dsm, L, M);
  publish();
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
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
    float flow[8];
    uint32_t m1a, m1b, m2a, m2b;
    flow_forward_tc<true>(dsm, sb, L, S, fin, flow, m1a, m1b, m2a, m2b, t2h, t2l, aT2h, aT2l);
    const float sc = pow2_factor(am);
    float inv = 1.0f / sc;
#pragma unroll
    for (int k = 0; k < 16; ++k) g[k] *= sc;
    tile_put8(o16h, o16l, tid, 0, g);
    tile_put8(o16h, o16l, tid, 1, g + 8);
    publish();
    // dH2[128 x 64] = dO * W2 (W2 stored [k/8][16 rows][8]) ; dW2^T[64 x 16] = H2^T * dO
    mma_prop<64>(S, 0, aO16h, aO16l, 2, sb + L.w2, 16);
    mma_tt<16>(aT1h, aT1l, aO16h, aO16l, [&](int r, int c, float x, float y) {
      if (c < 6) atomicAdd(G.flo_w2 + (size_t)c * 64 + r, x * inv);
      if (c + 1 < 6) atomicAdd(G.flo_w2 + (size_t)(c + 1) * 64 + r, y * inv);
    });
    __syncthreads();
    float cs2;
    {   // dH2 * relu2, re-scaled -> T1 (H2 is dead: dW2^T has been computed)
      float a2 = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) if (l4d_bit(m2a, m2b, q * 16 + i)) a2 = fmaxf(a2, fabsf(v[i]));
      }
      a2 = block_amax128(a2, s_w);
      const float r = a2 > 0.f ? pow2_factor(a2) : 1.0f;
      cs2 = sc * r;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = l4d_bit(m2a, m2b, q * 16 + i) ? v[i] * r : 0.f;
        tile_put8(t1h, t1l, tid, 2 * q, v);
        tile_put8(t1h, t1l, tid, 2 * q + 1, v + 8);
      }
    }
    inv = 1.0f / cs2;
    publish();
    // dH1[128 x 64] = dH2 * W1 ; dW1^T[64 x 64] = H1^T * dH2
    mma_prop<64>(S, 0, aT1h, aT1l, 8, sb + L.w1, 64);
    mma_tt<64>(aT2h, aT2l, aT1h, aT1l, [&](int r, int c, float x, float y) {
      red2(G.flo_w1t + (size_t)r * 64 + c, x * inv, y * inv);
    });
    __syncthreads();
    float cs3;
    {   // dH1 * relu1, re-scaled -> T2 (H1 is dead: dW1^T has been computed)
      float a3 = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) if (l4d_bit(m1a, m1b, q * 16 + i)) a3 = fmaxf(a3, fabsf(v[i]));
      }
      a3 = block_amax128(a3, s_w);
      const float r = a3 > 0.f ? pow2_factor(a3) : 1.0f;
      cs3 = cs2 * r;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[16];
        acc_ld16(S, q * 16, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = l4d_bit(m1a, m1b, q * 16 + i) ? v[i] * r : 0.f;
        tile_put8(t2h, t2l, tid, 2 * q, v);
        tile_put8(t2h, t2l, tid, 2 * q + 1, v + 8);
      }
    }
    inv = 1.0f / cs3;
    publish();
    // dFin[128 x 16] = dH1 * W0 ; dW0[64 x 16] = dH1^T * Fin
    mma_prop<16>(S, 0, aT2h, aT2l, 8, sb + L.w0, 64);
    mma_tt<16>(aT2h, aT2l, aFinH, aFinL, [&](int r, int c, float x, float y) {
      atomicAdd(G.flo_w0t + (size_t)c * 64 + r, x * inv);
      atomicAdd(G.flo_w0t + (size_t)(c + 1) * 64 + r, y * inv);
    });
    __syncthreads();
    float dfin[16];
    acc_ld16(S, 0, dfin);
    if (active) {
      // dL/d(flow-MLP input) replaces the saved input in place (same thread, same addresses); k_bwd_flowgrid
      // turns it into flow-grid reductions at full occupancy
#pragma unroll
      for (int k = 0; k < 16; ++k) A.sv.flow_in[(size_t)k * P + p] = dfin[k] * inv;
    }
    __syncthreads();
  }
}
