// micro-benchmark for the "stage plane slices into shared memory with TMA" design question (VERDICT r1 #9, north_star):
// the plane reads of k_fwd_gather are 32-byte texel fetches (2 x LDG.128) at ray-coherent addresses from small,
// L1-resident fp32 tables.  Variant A reads the [32][32][8] plane from global memory (L1 hits after warm-up); variant B
// first stages the same plane into shared memory with ONE cp.async.bulk.tensor.2d (a CUtensorMap: UTMALDG in SASS) and
// reads it with LDS.128.  Same index stream, same arithmetic, same occupancy.  Both go through the L1TEX data pipe.
#include <cstdio>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

#define PW 32
#define PH 32
#define PC 8
__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
// texel index of (thread, iteration): COHERENT = lanes of a warp walk a short line (a ray segment: ~1 texel per 8 lanes at this
// resolution), else every lane its own random texel
template <bool COHERENT>
__device__ __forceinline__ uint32_t texel(uint32_t tid, uint32_t it) {
  if (COHERENT) {
    const uint32_t w = hash32((tid >> 5) * 2654435761u + it * 40503u);
    const uint32_t x = ((w & 1023u) + ((tid & 31u) << 2)) >> 5, y = (w >> 10) & 31u;     // x advances 1 texel per 8 lanes
    return (y * PW + (x & 31u));
  }
  return hash32(tid * 2654435761u + it * 40503u) & (PW * PH - 1);
}
template <bool COHERENT>
__global__ void __launch_bounds__(128) k_global(const float* __restrict__ plane, int iters, float* out) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4* p = reinterpret_cast<const float4*>(plane + (size_t)texel<COHERENT>(tid, it * 4 + u) * PC);
      const float4 a = __ldg(p), b = __ldg(p + 1);
      acc += a.x * b.w + a.z;
    }
  }
  if (acc == 123.456f) out[0] = acc;
}
template <bool COHERENT>
__global__ void __launch_bounds__(128) k_tma(const __grid_constant__ CUtensorMap tmap, int iters, float* out) {
  extern __shared__ __align__(128) float s_plane[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar), d = (uint32_t)__cvta_generic_to_shared(s_plane);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((uint32_t)(PW * PH * PC * 4)));
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(d), "l"(&tmap), "r"(0), "r"(0), "r"(b) : "memory");
  }
  {
    const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar);
    uint32_t done = 0;
    while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(b));
  }
  float acc = 0.f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4* p = reinterpret_cast<const float4*>(s_plane + (size_t)texel<COHERENT>(tid, it * 4 + u) * PC);
      const float4 a = p[0], b = p[1];
      acc += a.x * b.w + a.z;
    }
  }
  if (acc == 123.456f) out[0] = acc;
}
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
template <bool COH>
static void run(const float* plane, const CUtensorMap& tm, float* out, int per_sm, const char* name, bool first) {
  const int blocks = 132 * per_sm, threads = 128, iters = 512;
  const size_t smem = PW * PH * PC * 4;
  cudaFuncSetAttribute(k_tma<COH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  float ms_g, ms_t;
  k_global<COH><<<blocks, threads>>>(plane, 8, out); cudaDeviceSynchronize();
  cudaEventRecord(a); k_global<COH><<<blocks, threads>>>(plane, iters, out); cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms_g, a, b);
  k_tma<COH><<<blocks, threads, smem>>>(tm, 8, out); cudaDeviceSynchronize();
  cudaEventRecord(a); k_tma<COH><<<blocks, threads, smem>>>(tm, iters, out); cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms_t, a, b);
  const double texels = (double)blocks * threads * iters * 4;
  printf("%s{\"pattern\": \"%s\", \"ctas_per_sm\": %d, \"global_L1_gtexels_s\": %.1f, \"tma_smem_gtexels_s\": %.1f, \"err\": \"%s\"}", first ? "" : ", ", name, per_sm,
         texels / ms_g / 1e6, texels / ms_t / 1e6, cudaGetErrorString(cudaGetLastError()));
}
int main() {
  float *plane, *out;
  cudaMalloc(&plane, PW * PH * PC * 4); cudaMemset(plane, 0, PW * PH * PC * 4); cudaMalloc(&out, 4);
  EncodeFn enc = nullptr;
  cudaDriverEntryPointQueryResult qr;
  cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &qr);
  CUtensorMap tm;
  const cuuint64_t dims[2] = {PW * PC, PH};                  // innermost: 256 floats (one plane row, channels-last), 32 rows
  const cuuint64_t strides[1] = {PW * PC * 4};
  const cuuint32_t box[2] = {PW * PC, PH}, estr[2] = {1, 1};
  const CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, plane, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  printf("{\"what\": \"32-byte texel reads of one [32][32][8] fp32 plane: global (L1-resident) vs staged into shared memory by one cp.async.bulk.tensor.2d\", "
         "\"encode_rc\": %d, \"results\": [", (int)r);
  bool first = true;
  for (int per_sm : {2, 4, 6}) {
    run<true>(plane, tm, out, per_sm, "ray-coherent (1 texel per 8 lanes)", first); first = false;
    run<false>(plane, tm, out, per_sm, "divergent (random texel per lane)", first);
  }
  printf("]}\n");
  return 0;
}
