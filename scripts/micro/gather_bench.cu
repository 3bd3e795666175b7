// micro-benchmark: ceiling of divergent gathers from an L2-resident table - the access pattern of k_fwd_gather
// (every lane of a warp reads its own random sector; 8 B = static-hash corner, 16 B = dynamic-hash pair / flow corner,
// 32 B = plane texel).  Reports G sectors/s and the equivalent GB/s of 32-byte sectors: the roofline unit bench.py
// quotes for the gather kernel (the working set is L2-resident, so HBM is not the bound).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
template <int BYTES>
__global__ void __launch_bounds__(128) k(const unsigned char* __restrict__ table, uint32_t n_sectors, int iters, float* out) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t s = hash32(tid * 2654435761u + 12345u);
  float acc = 0.f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {          // 8 independent loads in flight per thread, like the unrolled corner loops
      s = hash32(s + u);
      const unsigned char* p = table + (size_t)(s % n_sectors) * 32;
      if (BYTES == 8) { const float2 v = __ldg(reinterpret_cast<const float2*>(p)); acc += v.x + v.y; }
      else if (BYTES == 16) { const float4 v = __ldg(reinterpret_cast<const float4*>(p)); acc += v.x + v.w; }
      else { const float4 v = __ldg(reinterpret_cast<const float4*>(p)), w = __ldg(reinterpret_cast<const float4*>(p) + 1); acc += v.x + w.w; }
    }
  }
  if (acc == 123.456f) out[0] = acc;
}
template <int BYTES>
static double run(const unsigned char* t, uint32_t n_sectors, float* out, int per_sm) {
  const int blocks = 132 * per_sm, threads = 128, iters = 64;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<BYTES><<<blocks, threads>>>(t, n_sectors, 4, out);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k<BYTES><<<blocks, threads>>>(t, n_sectors, iters, out);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  return (double)blocks * threads * iters * 8 / (ms * 1e-3) / 1e9;     // G sectors / s
}
int main() {
  printf("{\"what\": \"divergent gathers, one random 32-byte sector per lane\", \"results\": [");
  bool first = true;
  for (uint32_t mb : {24u, 96u, 320u}) {
    const uint32_t n_sectors = mb * 1024u * 1024u / 32u;
    unsigned char* t; float* out;
    cudaMalloc(&t, (size_t)n_sectors * 32); cudaMemset(t, 1, (size_t)n_sectors * 32); cudaMalloc(&out, 4);
    for (int per_sm : {8, 16}) {
      const double g8 = run<8>(t, n_sectors, out, per_sm), g16 = run<16>(t, n_sectors, out, per_sm), g32 = run<32>(t, n_sectors, out, per_sm);
      printf("%s{\"table_mb\": %u, \"ctas_per_sm\": %d, \"gsectors_s_8B\": %.1f, \"gsectors_s_16B\": %.1f, \"gsectors_s_32B\": %.1f}", first ? "" : ", ",
             mb, per_sm, g8, g16, g32);
      first = false;
    }
    cudaFree(t); cudaFree(out);
  }
  printf("]}\n");
  return 0;
}
