// micro-benchmark: throughput of fp32 vector reductions (RED.E.ADD.F32x4) to an L2-resident table
//   mode 0: every lane hits its own random 32-byte sector (16 of its 32 bytes)
//   mode 1: lane pairs (2i, 2i+1) hit the two 16-byte halves of one random sector
//   mode 2: as 0 but scalar fp32 REDs (4 per lane, consecutive addresses)
//   mode 3: lane quads share one 64-byte region (4 x 16 B)
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ void red4(float* p, float a, float b, float c, float d) {
  atomicAdd(reinterpret_cast<float4*>(p), make_float4(a, b, c, d));
}
__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
template <int MODE>
__global__ void k(float* table, uint32_t n_sectors, int iters) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t s = hash32(tid * 2654435761u + 12345u);
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      s = hash32(s + u);
      if (MODE == 0) {
        red4(table + (size_t)(s % n_sectors) * 8 + ((s >> 31) ? 4 : 0), 1.f, 2.f, 3.f, 4.f);
      } else if (MODE == 1) {
        const uint32_t sp = __shfl_sync(0xffffffffu, s, threadIdx.x & ~1u);
        red4(table + (size_t)(sp % n_sectors) * 8 + (threadIdx.x & 1u) * 4, 1.f, 2.f, 3.f, 4.f);
      } else if (MODE == 2) {
        float* q = table + (size_t)(s % n_sectors) * 8;
        atomicAdd(q, 1.f); atomicAdd(q + 1, 2.f); atomicAdd(q + 2, 3.f); atomicAdd(q + 3, 4.f);
      } else {
        const uint32_t sp = __shfl_sync(0xffffffffu, s, threadIdx.x & ~3u);
        red4(table + (size_t)(sp % (n_sectors / 2)) * 16 + (threadIdx.x & 3u) * 4, 1.f, 2.f, 3.f, 4.f);
      }
    }
  }
}
template <int MODE>
static void run(float* table, uint32_t n_sectors, const char* name) {
  const int blocks = 132 * 8, threads = 128, iters = 64;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<blocks, threads>>>(table, n_sectors, 4);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k<MODE><<<blocks, threads>>>(table, n_sectors, iters);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  const double lane_ops = (double)blocks * threads * iters * 8;
  printf("[red] %-34s table %6.1f MB: %7.3f ms  %8.1f G lane-ops/s  %6.2f cycles/lane-op/SM (1.98 GHz)\n", name,
         n_sectors * 32.0 / 1e6, ms, lane_ops / ms / 1e6, ms * 1e-3 * 1.98e9 * 132 / lane_ops);
}
int main() {
  for (uint32_t mb : {8u, 24u, 96u, 320u}) {
    const uint32_t n_sectors = mb * 1024u * 1024u / 32u;
    float* t; cudaMalloc(&t, (size_t)n_sectors * 32); cudaMemset(t, 0, (size_t)n_sectors * 32);
    run<0>(t, n_sectors, "RED.128, 32 distinct sectors");
    run<1>(t, n_sectors, "RED.128, lane pairs share a sector");
    run<3>(t, n_sectors, "RED.128, lane quads share 64 B");
    run<2>(t, n_sectors, "4 x RED.32 (lane-op = 4 REDs)");
    cudaFree(t);
  }
  return 0;
}
