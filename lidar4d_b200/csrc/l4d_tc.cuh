// l4d_tc.cuh - wgmma / mbarrier / bulk-copy building blocks for sm_90a (inline PTX).
//
// Tile convention used by the MLP engine: M = 128 samples, operands fp16 in shared memory in the canonical
// *interleaved* (no-swizzle) layout: 16-byte chunks of 8 halves along K, [chunk][row] order:
//     byte(row, k) = (k/8) * (ROWS*16) + row*16 + (k%8)*2
// => core matrix = 8 rows x 16 B contiguous; K-major: LBO (next K chunk) = ROWS*16 B, SBO (next 8 rows) = 128 B.
// A thread that owns a row writes one 16-byte chunk per store: conflict-free.
//
// MMAs are warpgroup-wide (wgmma.mma_async, m64nNk16, fp32 accumulators in registers).  A 128-row product is two
// 64-row blocks; in a 256-thread CTA each warpgroup computes one.  Epilogues work on the accumulator fragments in the
// registers: activations go back to operand tiles with frag_put, per-row reductions are quad shuffles, weight-gradient
// products are flushed straight from the registers.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace l4dtc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// bulk copy global -> shared (TMA engine, no tensor map): completion is counted in bytes on an mbarrier
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_saddr, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_saddr),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- descriptors ---------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, no swizzle.  K-major: LBO = stride of the next 8-wide K chunk, SBO = stride of
// the next 8 rows.  MN-major: LBO = stride of the next 8 K rows, SBO = stride of the next 8-wide MN chunk.
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// ---- wgmma ---------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N]; TA / TB = 1 selects an MN-major operand.  acc == 0 overwrites D.
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(N == 8 || N == 16 || N == 32 || N == 64, "wgmma_f16: N in {8, 16, 32, 64}");
  if constexpr (N == 8) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0,%1,%2,%3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
  } else if constexpr (N == 16) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
  } else if constexpr (N == 32) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
  } else {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
  }
}

// One operand of a product: start address of each term, byte step per K=16 step, LBO / SBO of its descriptor.
struct Opnd {
  uint32_t addr[3];
  uint32_t kstep, lbo, sbo;
};
// issue D[64 x N] = sum over terms t of A_t * B_t over ksteps K=16 steps as one wgmma group; warpgroup-wide.
// D must not be touched before a wg_wait that covers the group.
template <int N, int TA, int TB>
__device__ __forceinline__ void wg_gemm_issue(float (&d)[N / 2], const Opnd& A, const Opnd& B, int nterms, int ksteps) {
  wg_fence();
  for (int t = 0; t < nterms; ++t)
    for (int k = 0; k < ksteps; ++k)
      wgmma_f16<N, TA, TB>(d, smem_desc(A.addr[t] + (uint32_t)k * A.kstep, A.lbo, A.sbo),
                           smem_desc(B.addr[t] + (uint32_t)k * B.kstep, B.lbo, B.sbo), (t | k) ? 1u : 0u);
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// wait until at most PENDING of this warpgroup's wgmma groups are still in flight
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// D[64 x N] = sum over terms t of A_t * B_t; returns with D in registers
template <int N, int TA, int TB>
__device__ __forceinline__ void wg_gemm(float (&d)[N / 2], const Opnd& A, const Opnd& B, int nterms, int ksteps) {
  wg_gemm_issue<N, TA, TB>(d, A, B, nterms, ksteps);
  wg_wait<0>();
}
// visit the accumulator fragment of a 64 x N product: f(row, col, v[col], v[col + 1]) for the thread's element pairs
template <int N, class F>
__device__ __forceinline__ void frag_foreach(const float (&d)[N / 2], F&& f) {
  const int t = threadIdx.x & 127, r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    f(r, 8 * j + c, d[4 * j], d[4 * j + 1]);
    f(r + 8, 8 * j + c, d[4 * j + 2], d[4 * j + 3]);
  }
}

// ---- epilogues in the fragment layout ------------------------------------------------------
// Thread t of a warpgroup holds rows frag_row() and frag_row() + 8 of the 64-row block and, per 8-column group j,
// columns 8j + frag_col() + {0, 1}:  d[4j + 2h + e] = D[frag_row() + 8h][8j + frag_col() + e].
__device__ __forceinline__ int frag_row() { const int t = threadIdx.x & 127; return 16 * (t >> 5) + ((t & 31) >> 2); }
__device__ __forceinline__ int frag_col() { return 2 * (threadIdx.x & 3); }

// fragment (rows [m0, m0 + 64)) -> fp16 hi|lo operand tile [k/8][rows][8], k-chunks [c0, c0 + N/8); hi = rn(v),
// lo = rn(v - hi).  One 4-byte store per half2: a warp covers 8 consecutive 16-byte rows of a chunk, conflict-free.
template <int N>
__device__ __forceinline__ void frag_put(unsigned char* hi, unsigned char* lo, uint32_t rows, int m0, int c0, const float (&d)[N / 2]) {
  const int r = m0 + frag_row(), q = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float a = d[4 * j + 2 * h], b = d[4 * j + 2 * h + 1];
      const __half2 x = __floats2half2_rn(a, b);
      const float2 f = __half22float2(x);
      const __half2 y = __floats2half2_rn(a - f.x, b - f.y);
      const size_t off = ((size_t)(c0 + j) * rows + r + 8 * h) * 16 + q * 4;
      *reinterpret_cast<__half2*>(hi + off) = x;
      *reinterpret_cast<__half2*>(lo + off) = y;
    }
}
// sum over the four lanes that share a fragment row
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// barrier over the 128 threads of this thread's warpgroup (named barrier 1 + warpgroup; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar() { asm volatile("bar.sync %0, 128;" ::"r"(1 + (int)(threadIdx.x >> 7)) : "memory"); }

// pack 8 floats into one 16-byte chunk of fp16 (round to nearest)
__device__ __forceinline__ uint4 pack8_half(const float* f) {
  __half2 a = __floats2half2_rn(f[0], f[1]), b = __floats2half2_rn(f[2], f[3]);
  __half2 c = __floats2half2_rn(f[4], f[5]), d = __floats2half2_rn(f[6], f[7]);
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
  o.z = *reinterpret_cast<uint32_t*>(&c); o.w = *reinterpret_cast<uint32_t*>(&d);
  return o;
}

}  // namespace l4dtc

// =============================================================================================
// self-test: C[128][N] = A[128][K] * B[N][K]^T with fp16 operands, fp32 accumulate, one CTA (one warpgroup).
// Exercises the descriptor encoding and the accumulator fragment layout exactly as the MLP engine uses them.
// =============================================================================================
__global__ void __launch_bounds__(128) k_tc_selftest(const __half* __restrict__ A, const __half* __restrict__ B,
                                                     float* __restrict__ C, int N, int K) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char tc_smem[];
  const int tid = threadIdx.x;
  unsigned char* sA = tc_smem;                         // [K/8][128][16 B]
  unsigned char* sB = tc_smem + (size_t)(K / 8) * 128 * 16;   // [K/8][N][16 B]
  for (int c = 0; c < K / 8; ++c)
    *reinterpret_cast<uint4*>(sA + ((size_t)c * 128 + tid) * 16) = *reinterpret_cast<const uint4*>(A + (size_t)tid * K + c * 8);
  for (int i = tid; i < (K / 8) * N; i += 128) {
    const int c = i / N, n = i % N;
    *reinterpret_cast<uint4*>(sB + ((size_t)c * N + n) * 16) = *reinterpret_cast<const uint4*>(B + (size_t)n * K + c * 8);
  }
  fence_proxy_async();
  __syncthreads();
  for (int mb = 0; mb < 2; ++mb)
    for (int n0 = 0; n0 < N; n0 += 8) {
      const Opnd a{{smem_u32(sA) + (uint32_t)mb * 1024u, 0u, 0u}, 2u * 128u * 16u, 128u * 16u, 128u};
      const Opnd b{{smem_u32(sB) + (uint32_t)n0 * 16u, 0u, 0u}, 2u * (uint32_t)N * 16u, (uint32_t)N * 16u, 128u};
      float d[4];
      wg_gemm<8, 0, 0>(d, a, b, 1, K / 16);
      frag_foreach<8>(d, [&](int r, int c, float x, float y) {
        C[(size_t)(64 * mb + r) * N + n0 + c] = x;
        C[(size_t)(64 * mb + r) * N + n0 + c + 1] = y;
      });
    }
}

// =============================================================================================
// self-test 2: operands arrive already in tile format (prepared on the host), any major-ness, M = 64 or 128.
//   K-major operand  X[rows][K]      : byte((k/8)*rows*16 + r*16 + (k%8)*2)           LBO = rows*16, SBO = 128
//   MN-major operand X[rows=mn][K=k] : byte((mn/8)*K*16  + k*16 + (mn%8)*2)           LBO = 128,     SBO = K*16
// =============================================================================================
template <int TA, int TB>
__device__ __forceinline__ void tc_selftest2_body(const unsigned char* sA, const unsigned char* sB, float* __restrict__ C, int M,
                                                  int N, int K) {
  using namespace l4dtc;
  for (int mb = 0; mb < M / 64; ++mb)
    for (int n0 = 0; n0 < N; n0 += 8) {
      const Opnd a = TA ? Opnd{{smem_u32(sA) + (uint32_t)mb * 8u * (uint32_t)K * 16u, 0u, 0u}, 256u, 128u, (uint32_t)K * 16u}
                        : Opnd{{smem_u32(sA) + (uint32_t)mb * 1024u, 0u, 0u}, 2u * (uint32_t)M * 16u, (uint32_t)M * 16u, 128u};
      const Opnd b = TB ? Opnd{{smem_u32(sB) + (uint32_t)(n0 / 8) * (uint32_t)K * 16u, 0u, 0u}, 256u, 128u, (uint32_t)K * 16u}
                        : Opnd{{smem_u32(sB) + (uint32_t)n0 * 16u, 0u, 0u}, 2u * (uint32_t)N * 16u, (uint32_t)N * 16u, 128u};
      float d[4];
      wg_gemm<8, TA, TB>(d, a, b, 1, K / 16);
      frag_foreach<8>(d, [&](int r, int c, float x, float y) {
        C[(size_t)(64 * mb + r) * N + n0 + c] = x;
        C[(size_t)(64 * mb + r) * N + n0 + c + 1] = y;
      });
    }
}
__global__ void __launch_bounds__(128) k_tc_selftest2(const unsigned char* __restrict__ A, const unsigned char* __restrict__ B,
                                                      float* __restrict__ C, int M, int N, int K, int a_mn, int b_mn) {
  using namespace l4dtc;
  extern __shared__ __align__(128) unsigned char tc_smem[];
  const int tid = threadIdx.x;
  const int a_bytes = M * K * 2, b_bytes = N * K * 2;
  unsigned char* sA = tc_smem;
  unsigned char* sB = tc_smem + ((a_bytes + 1023) & ~1023);
  for (int i = tid * 16; i < a_bytes; i += 128 * 16) *reinterpret_cast<uint4*>(sA + i) = *reinterpret_cast<const uint4*>(A + i);
  for (int i = tid * 16; i < b_bytes; i += 128 * 16) *reinterpret_cast<uint4*>(sB + i) = *reinterpret_cast<const uint4*>(B + i);
  fence_proxy_async();
  __syncthreads();
  if (a_mn && b_mn) tc_selftest2_body<1, 1>(sA, sB, C, M, N, K);
  else if (a_mn) tc_selftest2_body<1, 0>(sA, sB, C, M, N, K);
  else if (b_mn) tc_selftest2_body<0, 1>(sA, sB, C, M, N, K);
  else tc_selftest2_body<0, 0>(sA, sB, C, M, N, K);
}
