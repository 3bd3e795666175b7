// l4d_optim.cuh - the optimiser-step tail of the hot path (SURVEY.md 8(f) #4), included by l4d_kernels.cu:
//   * k_adam_flat: one launch of Adam over the flat fp32 parameter / gradient / moment arenas (per-segment learning
//     rate = the reference's param groups, lidar4d.py:226-237; recipe main_lidar4d.py:298-300: betas (0.9, 0.99),
//     eps 1e-15) that ALSO writes the fp16 working copies of the hash tables the render kernels gather from
//     (static / flow: straight casts; dynamic: the two slice-pair records an entry lives in), so the 300 MB of
//     tables are read once per step instead of three times;
//   * k_stage_jobs / k_unstage_jobs: every small staging op (planes -> channels-last, MLP transposes, tensor-core operand
//     packing) and every gradient fold-back in ONE launch each, driven by a job table in kernel-parameter space
//     (they were ~55 and ~35 separate launches: ~0.4 ms of pure launch latency at the reference's 1,024-ray step).
#pragma once
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

// ---------------------------------------------------------------------------------------------------------------
// Adam
// ---------------------------------------------------------------------------------------------------------------
// L4D_ADAM_CHUNK (include/lidar4d_b200.h) floats: arena segments start on multiples of it, so a chunk has one segment
struct AdamSeg {
  unsigned long long begin, end;       // [begin, end) in floats; begin % L4D_ADAM_CHUNK == 0
  float lr;
  uint32_t stride0, off0, stride1, off1;   // fp16 emission: byte stride per float4 and byte offset, per destination
  uint32_t pad;
  unsigned char* dst0;                 // nullptr = no emission
  unsigned char* dst1;
};
struct AdamArgs {
  float* p;
  const float* g;
  float* m;
  float* v;
  unsigned long long n_chunks;
  float beta1, beta2, eps, step, inv_scale;   // step as a float, like torch's state_steps
  int n_seg;
  uint32_t zero_grad;                  // 1: clear the gradient arena in the same pass (saves the next step's memset)
  float* g_rw;
  AdamSeg seg[L4D_ADAM_MAX_SEGMENTS];
};

// One element of Adam (no weight decay, no amsgrad, not maximising) in the operation order of torch 2.11's fused Adam,
// ATen/native/cuda/fused_adam_utils.cuh adam_math, with its fused multiply-adds written out so that contraction cannot
// change a bit.  step_size = lr / bc1 and bc2_sqrt = sqrtf(bc2), with bc = 1 - powf(beta, (float)step) in fp32 as torch
// computes them.  The gradient is MULTIPLIED by inv_scale; for a power-of-two loss scale (all GradScaler produces) that
// is exactly torch's g / grad_scale.  Compiles for the host too (tests/hostsim/adamsim.cu).
//
// IEEE sqrtf and division take a slow path on subnormal operands or quotients, and the second moments of rarely touched
// entries are subnormal (g ~ 1e-20 => g^2 ~ 1e-40).  Both are evaluated on operands scaled by powers of two, but only
// where the scaled result is provably the unscaled one, so the result equals the plain IEEE formula for EVERY input:
//   sqrtf(v) = sqrtf(v * 2^64) * 2^-32 for v < 2^64 (the root of a subnormal is normal; v >= 2^64 is left unscaled);
//   a / den = ((a * 2^64) / den) * 2^-64 when that scaled quotient is 0 or a finite normal >= 2^-62: then a * 2^64 did not
//   overflow and a / den is normal too (or rounds to 0), so scaling commutes with rounding.  Otherwise (a subnormal or
//   overflowing quotient, inf, NaN) it is recomputed unscaled.
// Every product that can meet an addition (q * 2^-64 before p - u) is exact, so contraction cannot change those either.
__host__ __device__ __forceinline__ void l4d_adam_elem(float& p, float& m, float& v, float g, float inv_scale, float beta1,
                                                     float beta2, float eps, float step_size, float bc2_sqrt) {
  g = g * inv_scale;
  m = fmaf(beta1, m, fmaf(-beta1, g, g));
  const float gsq = g * g;
  v = fmaf(beta2, v, fmaf(-beta2, gsq, gsq));
  const bool v_small = v < 0x1p64f;
  const float root = sqrtf(v * (v_small ? 0x1p64f : 1.0f)) * (v_small ? 0x1p-32f : 1.0f);
  const float den = root / bc2_sqrt + eps;
  const float a = step_size * m;
  const float q = (a * 0x1p64f) / den;
  const float aq = fabsf(q);
  float u = q * 0x1p-64f;
  if (!((aq >= 0x1p-62f || aq == 0.0f) && aq <= 0x1.fffffep127f)) u = a / den;
  p = p - u;
}

__global__ void __launch_bounds__(256) k_adam_flat(const __grid_constant__ AdamArgs A) {
  const float bc1 = 1.0f - powf(A.beta1, A.step);
  const float bc2_sqrt = sqrtf(1.0f - powf(A.beta2, A.step));
  for (unsigned long long c = blockIdx.x; c < A.n_chunks; c += gridDim.x) {
    const unsigned long long base = c * L4D_ADAM_CHUNK;
    int lo = 0, hi = A.n_seg - 1;                       // last segment with begin <= base (uniform per block)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (A.seg[mid].begin <= base) lo = mid; else hi = mid - 1;
    }
    const AdamSeg& s = A.seg[lo];
    if (base < s.begin) continue;                       // chunk before the first segment: not covered
    const unsigned long long i = base + 4ull * threadIdx.x;
    if (i >= s.end) continue;                           // alignment padding behind a tensor, or a gap
    float4 p = *reinterpret_cast<const float4*>(A.p + i);
    float4 g = __ldcs(reinterpret_cast<const float4*>(A.g + i));
    float4 m = *reinterpret_cast<const float4*>(A.m + i);
    float4 v = *reinterpret_cast<const float4*>(A.v + i);
    const float step_size = s.lr / bc1;
    l4d_adam_elem(p.x, m.x, v.x, g.x, A.inv_scale, A.beta1, A.beta2, A.eps, step_size, bc2_sqrt);
    l4d_adam_elem(p.y, m.y, v.y, g.y, A.inv_scale, A.beta1, A.beta2, A.eps, step_size, bc2_sqrt);
    l4d_adam_elem(p.z, m.z, v.z, g.z, A.inv_scale, A.beta1, A.beta2, A.eps, step_size, bc2_sqrt);
    l4d_adam_elem(p.w, m.w, v.w, g.w, A.inv_scale, A.beta1, A.beta2, A.eps, step_size, bc2_sqrt);
    *reinterpret_cast<float4*>(A.p + i) = p;
    *reinterpret_cast<float4*>(A.m + i) = m;
    *reinterpret_cast<float4*>(A.v + i) = v;
    if (A.zero_grad) *reinterpret_cast<float4*>(A.g_rw + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s.dst0 || s.dst1) {
      const __half2 a = __floats2half2_rn(p.x, p.y), b = __floats2half2_rn(p.z, p.w);
      uint2 o;
      o.x = *reinterpret_cast<const uint32_t*>(&a);
      o.y = *reinterpret_cast<const uint32_t*>(&b);
      const unsigned long long r4 = (i - s.begin) >> 2;
      if (s.dst0) *reinterpret_cast<uint2*>(s.dst0 + r4 * s.stride0 + s.off0) = o;
      if (s.dst1) *reinterpret_cast<uint2*>(s.dst1 + r4 * s.stride1 + s.off1) = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// job tables
// ---------------------------------------------------------------------------------------------------------------
enum { L4D_JOB_PLANE_TO_CL = 0, L4D_JOB_TRANSPOSE = 1, L4D_JOB_COPY = 2, L4D_JOB_PACK_UMMA = 3,
       L4D_JOB_PLANE_FROM_CL = 4, L4D_JOB_ADD_TRANSPOSED = 5, L4D_JOB_ADD = 6 };
struct StageJob {
  const float* src;
  void* dst;
  int type, n, a, b, c, d, e, round16;     // n = elements of the job's index space
};
#define L4D_MAX_JOBS 72
struct JobArgs {
  int n_jobs;
  StageJob job[L4D_MAX_JOBS];
};

__device__ __forceinline__ float l4d_r16(float x, int on) { return on ? __half2float(__float2half_rn(x)) : x; }

// blockIdx.y = job; blocks stride over the job's elements
__global__ void __launch_bounds__(256) k_stage_jobs(const __grid_constant__ JobArgs A) {
  const StageJob& J = A.job[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < J.n; i += gridDim.x * blockDim.x) {
    switch (J.type) {
      case L4D_JOB_PLANE_TO_CL: {            // NCHW [8][hw] -> [hw][8];  a = hw
        const int c = i & 7, px = i >> 3;
        reinterpret_cast<float*>(J.dst)[i] = __ldg(J.src + (size_t)c * J.a + px);
      } break;
      case L4D_JOB_TRANSPOSE: {              // dst[r][c] = src[c][r]; a = src_ld, b = dst_cols, c = valid_rows, d = valid_cols
        const int r = i / J.b, c = i % J.b;
        reinterpret_cast<float*>(J.dst)[i] = (r < J.c && c < J.d) ? l4d_r16(__ldg(J.src + (size_t)c * J.a + r), J.round16) : 0.f;
      } break;
      case L4D_JOB_COPY: {                   // a = n_valid
        reinterpret_cast<float*>(J.dst)[i] = i < J.a ? l4d_r16(__ldg(J.src + i), J.round16) : 0.f;
      } break;
      case L4D_JOB_PACK_UMMA: {              // W[n][k0+k] (ld a) -> fp16 [k/8][row_off + n][8]; b = K, c = k0, d = rows_total, e = row_off
        const int n = i / J.b, k = i % J.b;
        reinterpret_cast<__half*>(J.dst)[((size_t)(k >> 3) * J.d + J.e + n) * 8 + (k & 7)] =
            __float2half_rn(__ldg(J.src + (size_t)n * J.a + J.c + k));
      } break;
      default: break;
    }
  }
}

// gradient fold-back: dst (master layout) += src (working layout); src is cleared so the work buffer stays zero
__global__ void __launch_bounds__(256) k_unstage_jobs(const __grid_constant__ JobArgs A) {
  const StageJob& J = A.job[blockIdx.y];
  float* src = const_cast<float*>(J.src);
  float* dst = reinterpret_cast<float*>(J.dst);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < J.n; i += gridDim.x * blockDim.x) {
    size_t si;
    switch (J.type) {
      case L4D_JOB_PLANE_FROM_CL: { const int px = i % J.a, c = i / J.a; si = (size_t)px * 8 + c; } break;     // a = hw
      case L4D_JOB_ADD_TRANSPOSED: { const int r = i / J.b, c = i % J.b; si = (size_t)c * J.a + r; } break;   // a = src_cols, b = dst_cols
      default: si = (size_t)i; break;
    }
    const float s = src[si];
    if (s != 0.f) { dst[i] += s; src[si] = 0.f; }
  }
}
