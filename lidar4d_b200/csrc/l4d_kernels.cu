// l4d_kernels.cu - sm_90a kernels and the C-ABI of liblidar4d_b200.so
// (include/lidar4d_b200.h).  Thread == sample; one CTA walks one ray tile by
// tile and carries the transmittance; persistent grid over rays.
//
// Reference path replaced: model/renderer.py:44-140 (LiDAR_Renderer.run),
// model/lidar4d.py:124-223 (flow/density/attribute) and the encoders under it.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "l4d_bwd.cuh"
#include "l4d_core.cuh"
#include "l4d_host.h"
#include "l4d_tc.cuh"
#include "l4d_optim.cuh"
#include "l4d_losses.cuh"
#include "l4d_nngrid.cuh"
#include "l4d_imgmetrics.cuh"
#include "l4d_sweep.cuh"
#include "l4d_refine.cuh"

// =============================================================================
// error plumbing
// =============================================================================
static thread_local char g_err[512] = "";
static unsigned long long g_launches = 0;
int l4d_fail(int code, const char* fmt, const char* a, const char* b) {
  snprintf(g_err, sizeof(g_err), fmt, a, b);
  return code;
}
#define L4D_CUDA(call)                                                                     \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess) return l4d_fail(L4D_ECUDA, "%s failed: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

// -----------------------------------------------------------------------------
// optional per-kernel timing (profiling aid, not thread-safe): CUDA events recorded on the launch
// stream around every kernel of the render pipeline while enabled
// -----------------------------------------------------------------------------
#define L4D_PROF_MAX 256
static bool g_prof = false;
static int g_prof_n = 0;
static cudaEvent_t g_prof_ev[L4D_PROF_MAX];
static const char* g_prof_name[L4D_PROF_MAX];
static void prof_mark(cudaStream_t st, const char* name) {
  if (!g_prof || g_prof_n >= L4D_PROF_MAX) return;
  if (!g_prof_ev[g_prof_n]) cudaEventCreate(&g_prof_ev[g_prof_n]);
  cudaEventRecord(g_prof_ev[g_prof_n], st);
  g_prof_name[g_prof_n++] = name;
}
extern "C" int l4d_profile_start(void) { g_prof = true; g_prof_n = 0; return L4D_OK; }
// stops recording, synchronises the recorded events and writes up to `cap` (name, milliseconds) pairs: the time
// from the previous mark to the mark called `name`; marks called "begin" open a new call and are skipped
extern "C" int l4d_profile_stop(const char** names, float* ms, int cap) {
  g_prof = false;
  int n = 0;
  for (int i = 1; i < g_prof_n && n < cap; ++i) {
    if (!strcmp(g_prof_name[i], "begin")) continue;
    if (cudaEventSynchronize(g_prof_ev[i]) != cudaSuccess) return l4d_fail(L4D_ECUDA, "cudaEventSynchronize failed");
    float t = 0.f;
    if (cudaEventElapsedTime(&t, g_prof_ev[i - 1], g_prof_ev[i]) != cudaSuccess) return l4d_fail(L4D_ECUDA, "cudaEventElapsedTime failed");
    names[n] = g_prof_name[i];
    ms[n++] = t;
  }
  g_prof_n = 0;
  return n;
}

// kernels launched by this library in this process (bench "gpu_launches"; counted where they are launched)
extern "C" unsigned long long l4d_launch_count(void) { return g_launches; }

extern "C" int l4d_abi_version(void) { return L4D_ABI_VERSION; }
extern "C" const char* l4d_last_error(void) { return g_err; }

// =============================================================================
// staging kernels (once per optimiser step; pure HBM streaming)
// =============================================================================
__global__ void k_cast_half(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i * 4 + 3 < n; i += stride) {
    float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
    __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&a);
    o.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(dst)[i] = o;
  }
}
// two fp32 time slices -> one fp16 pair record per entry {lo.f0..3, hi.f0..3}
__global__ void k_pack_pair(const float* __restrict__ lo, const float* __restrict__ hi, uint4* __restrict__ dst, size_t n_entries) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n_entries; i += stride) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(lo) + i), b = __ldg(reinterpret_cast<const float4*>(hi) + i);
    __half2 a0 = __floats2half2_rn(a.x, a.y), a1 = __floats2half2_rn(a.z, a.w);
    __half2 b0 = __floats2half2_rn(b.x, b.y), b1 = __floats2half2_rn(b.z, b.w);
    uint4 o;
    o.x = *reinterpret_cast<uint32_t*>(&a0); o.y = *reinterpret_cast<uint32_t*>(&a1);
    o.z = *reinterpret_cast<uint32_t*>(&b0); o.w = *reinterpret_cast<uint32_t*>(&b1);
    dst[i] = o;
  }
}
// NCHW [8][H*W] -> channels-last [H*W][8]
__global__ void k_plane_to_cl(const float* __restrict__ src, float* __restrict__ dst, int hw) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hw * 8) return;
  int c = i & 7, px = i >> 3;
  dst[i] = __ldg(src + (size_t)c * hw + px);
}
// channels-last grad -> += NCHW grad
__global__ void k_plane_from_cl(const float* __restrict__ src, float* __restrict__ dst, int hw) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hw * 8) return;
  int px = i % hw, c = i / hw;
  dst[i] += src[(size_t)px * 8 + c];
}
// dst[c][r] = src[r][c] (src rows x cols); rows_valid/cols_valid select a sub-block, rest zero
__global__ void k_transpose(const float* __restrict__ src, int src_ld, float* __restrict__ dst, int dst_rows,
                            int dst_cols, int valid_rows, int valid_cols) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dst_rows * dst_cols) return;
  int r = i / dst_cols, c = i % dst_cols;       // dst[r][c] = src[c][r]
  dst[i] = (r < valid_rows && c < valid_cols) ? __ldg(src + (size_t)c * src_ld + r) : 0.f;
}
__global__ void k_copy_block(const float* __restrict__ src, float* __restrict__ dst, int n_valid, int n_total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_total) return;
  dst[i] = i < n_valid ? __ldg(src + i) : 0.f;
}
// dst[r][c] += src[c][r]   (fold an in-major work gradient into a native-layout master gradient)
__global__ void k_add_transposed(const float* __restrict__ src, int src_cols, float* __restrict__ dst, int dst_rows,
                                 int dst_cols) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dst_rows * dst_cols) return;
  int r = i / dst_cols, c = i % dst_cols;
  dst[i] += src[(size_t)c * src_cols + r];
}
__global__ void k_add(const float* __restrict__ src, float* __restrict__ dst, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}

// distribute the slice-independent dynamic-hash gradient (DevGrads::hd_comb: one float per entry = sum of w_corner * d)
// over the four time-basis features of the entry and the two live time slices, and clear it
__global__ void k_fold_dynamic(float* __restrict__ comb, float4* __restrict__ glo, float4* __restrict__ ghi, size_t n,
                               float w_lo, float w_hi, float b0, float b1, float b2, float b3) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float c = comb[i];
  if (c == 0.f) return;
  const float e0 = c * b0, e1 = c * b1, e2 = c * b2, e3 = c * b3;
  float4 a = glo[i];
  a.x = fmaf(w_lo, e0, a.x); a.y = fmaf(w_lo, e1, a.y); a.z = fmaf(w_lo, e2, a.z); a.w = fmaf(w_lo, e3, a.w);
  glo[i] = a;
  if (ghi) {
    float4 b = ghi[i];
    b.x = fmaf(w_hi, e0, b.x); b.y = fmaf(w_hi, e1, b.y); b.z = fmaf(w_hi, e2, b.z); b.w = fmaf(w_hi, e3, b.w);
    ghi[i] = b;
  }
  comb[i] = 0.f;
}
// DevModel::hd_con: contract the pair records of one dynamic table with the time constants of the frame's queries
// (l4d_contract_entry), one thread per entry.  786 k entries at L = 16: 12.6 MB of pair records read per query, 3 x 3.1 MB written - microseconds, once per launch.
struct ContractArgs {
  const uint4* table[3];      // [pair][entries] records of plane p
  float* con[3][3];           // [plane][query]
  uint32_t entries[3];
  uint32_t n_slices, n_queries_mask;      // bit q set: query q (cur, fwd, bwd) is live
  L4DTimeQuery q[3];
};
__global__ void k_contract_dynamic(const __grid_constant__ ContractArgs A) {
  const uint32_t p = blockIdx.y;
  const uint32_t n = A.entries[p];
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
#pragma unroll
    for (int qi = 0; qi < 3; ++qi) {
      if (!((A.n_queries_mask >> qi) & 1u)) continue;
      const uint32_t pair = l4d_time_pair(A.q[qi], A.n_slices);
      const uint4 rec = __ldg(A.table[p] + (size_t)pair * n + e);
      A.con[p][qi][e] = l4d_contract_entry(rec, A.q[qi], A.n_slices);
    }
  }
}
// DevModel::pl_con / DevGrads::pl_rows: the time (y) half of the bilinear blend of the three time planes of every scale is a
// launch constant per query.  k_contract_planes blends the two live rows of a plane into one row per query before the gather;
// k_fold_planes distributes the gradient rows over the two plane rows after the scatter, and clears them.
struct TimeRowArgs {
  float* plane[L4D_MAX_PLANE_SCALES][3];          // channels-last [T][R][8] plane (contract: read; fold: gradient, +=)
  float* row[L4D_MAX_PLANE_SCALES][3][3];         // [scale][plane][query] rows [R][8]
  uint32_t res[L4D_MAX_PLANE_SCALES];
  uint32_t qmask;                                 // bit q: query q (cur, fwd, bwd) is live
  int y0[3], y1[3];
  float wy0[3], wy1[3];
};
static void fill_time_rows(TimeRowArgs& T, const L4DConfig* cfg, const L4DFrame* frame) {
  memset(&T, 0, sizeof(T));
  const L4DTimeQuery* qs[3] = {&frame->cur, &frame->fwd, &frame->bwd};
  T.qmask = 1u | (frame->has_fwd ? 2u : 0u) | (frame->has_bwd ? 4u : 0u);
  for (int q = 0; q < 3; ++q) {
    const Bilerp b = l4d_bilerp(0.f, 2, qs[q]->tau, (int)cfg->time_resolution);
    T.y0[q] = b.y0; T.y1[q] = b.y1; T.wy0[q] = b.wy0; T.wy1[q] = b.wy1;
  }
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s) T.res[s] = cfg->plane_res[s];
}
__global__ void k_contract_planes(const __grid_constant__ TimeRowArgs A) {
  const uint32_t s = blockIdx.y / 3u, t = blockIdx.y % 3u;
  const uint32_t R = A.res[s], n = R * 8u;
  const float* P = A.plane[s][t];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      if (!((A.qmask >> q) & 1u)) continue;
      A.row[s][t][q][i] = __ldg(P + (size_t)A.y0[q] * n + i) * A.wy0[q] + __ldg(P + (size_t)A.y1[q] * n + i) * A.wy1[q];
    }
  }
}
__global__ void k_fold_planes(const __grid_constant__ TimeRowArgs A) {
  const uint32_t s = blockIdx.y / 3u, t = blockIdx.y % 3u;
  const uint32_t R = A.res[s], n = R * 8u;
  float* G = A.plane[s][t];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {       // one thread owns element i of all three queries: plain adds, no race
      if (!((A.qmask >> q) & 1u)) continue;
      const float v = A.row[s][t][q][i];
      if (v == 0.f) continue;
      G[(size_t)A.y0[q] * n + i] = fmaf(A.wy0[q], v, G[(size_t)A.y0[q] * n + i]);
      if (A.wy1[q] != 0.f) G[(size_t)A.y1[q] * n + i] = fmaf(A.wy1[q], v, G[(size_t)A.y1[q] * n + i]);
      A.row[s][t][q][i] = 0.f;
    }
  }
}
// flow grid: feature (2i + c) of an entry gets basis[i] * comb[entry][c] (DevGrads::hf_comb), then clear
__global__ void k_fold_flow(float2* __restrict__ comb, float4* __restrict__ g, size_t n, float b0, float b1, float b2, float b3) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float2 c = comb[i];
  if (c.x == 0.f && c.y == 0.f) return;
  float4 lo = g[2 * i], hi = g[2 * i + 1];
  lo.x = fmaf(b0, c.x, lo.x); lo.y = fmaf(b0, c.y, lo.y); lo.z = fmaf(b1, c.x, lo.z); lo.w = fmaf(b1, c.y, lo.w);
  hi.x = fmaf(b2, c.x, hi.x); hi.y = fmaf(b2, c.y, hi.y); hi.z = fmaf(b3, c.x, hi.z); hi.w = fmaf(b3, c.y, hi.w);
  g[2 * i] = lo; g[2 * i + 1] = hi;
  comb[i] = make_float2(0.f, 0.f);
}

// round fp32 values to the nearest fp16-representable value (MLP weights in mlp_fp16 mode)
__global__ void k_round_fp16(float* __restrict__ w, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) w[i] = __half2float(__float2half_rn(w[i]));
}
// native W[n][k0 + k] (row stride ld) -> fp16 wgmma K-major interleaved layout [k/8][row_off + n][8], rows_total rows
__global__ void k_pack_umma(const float* __restrict__ W, int ld, int n_rows, int k0, int K, __half* __restrict__ dst,
                            int rows_total, int row_off) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows * K) return;
  int n = i / K, k = i % K;
  dst[((size_t)(k >> 3) * rows_total + row_off + n) * 8 + (k & 7)] = __float2half_rn(__ldg(W + (size_t)n * ld + k0 + k));
}

static int sm_count();
static inline int nblk(size_t n, int t = 256) { return (int)((n + t - 1) / t); }

extern "C" size_t l4d_staged_bytes(const L4DConfig* cfg) {
  if (check_config(cfg) != L4D_OK) return 0;
  return staged_layout(cfg).total;
}

static inline StageJob make_job(int type, const float* src, void* dst, int n, int a = 0, int b = 0, int c = 0, int d = 0, int e = 0, int round16 = 0) {
  StageJob j;
  j.src = src; j.dst = dst; j.type = type; j.n = n; j.a = a; j.b = b; j.c = c; j.d = d; j.e = e; j.round16 = round16;
  return j;
}

extern "C" int l4d_stage_params_ex(const L4DConfig* cfg, const L4DMasterParams* m, void* staged, size_t staged_bytes,
                                   uint32_t what, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!m || !staged) return l4d_fail(L4D_EINVAL, "null pointer");
  StagedLayout L = staged_layout(cfg);
  if (staged_bytes < L.total) return l4d_fail(L4D_ESIZE, "staged buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  char* b = reinterpret_cast<char*>(staged);
  auto H = [&](size_t off) { return reinterpret_cast<__half*>(b + off); };
  auto F = [&](size_t off) { return reinterpret_cast<float*>(b + off); };
  if (what & L4D_STAGE_TABLES) {
    {
      size_t n = (size_t)cfg->hash_static.offset[cfg->hash_static.n_levels] * 4;
      ++g_launches; k_cast_half<<<2048, 256, 0, st>>>(m->hash_static, H(L.hs), n);
    }
    for (int p = 0; p < 3; ++p) {
      const size_t ne = (size_t)cfg->hash_dynamic[p].offset[cfg->hash_dynamic[p].n_levels];
      for (uint32_t s = 0; s < cfg->time_resolution; ++s)
        if (!m->hash_dynamic[p][s]) return l4d_fail(L4D_EINVAL, "null hash_dynamic slice");
      for (uint32_t s = 0; s + 1 < cfg->time_resolution; ++s) {
        ++g_launches;
        k_pack_pair<<<512, 256, 0, st>>>(m->hash_dynamic[p][s], m->hash_dynamic[p][s + 1],
                                          reinterpret_cast<uint4*>(b + L.hd[p]) + (size_t)s * ne, ne);
      }
    }
    {
      size_t n = (size_t)cfg->flow.offset[cfg->flow.n_levels] * 8;
      ++g_launches; k_cast_half<<<2048, 256, 0, st>>>(m->flow_grid, H(L.hf), n);
    }
  }
  if (what & L4D_STAGE_SMALL) {
    // planes, MLP working copies (both orientations) and tensor-core operand copies: one launch, one job each
    JobArgs J;
    int nj = 0;
    auto add = [&](const StageJob& j) { if (nj < L4D_MAX_JOBS) J.job[nj] = j; ++nj; };
    int maxn = 0;
    for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
      for (int ci = 0; ci < 6; ++ci) {
        int Hh, W;
        plane_hw(cfg, s, ci, Hh, W);
        add(make_job(L4D_JOB_PLANE_TO_CL, m->planes[s][ci], F(L.planes[s][ci]), Hh * W * 8, Hh * W));
      }
    const int r16 = cfg->mlp_fp16 ? 1 : 0;   // fp32 working copies become fp16-representable (as tcnn holds its weights)
    auto T = [&](const float* src, int src_ld, size_t dst, int dst_rows, int dst_cols, int vr, int vc) {
      add(make_job(L4D_JOB_TRANSPOSE, src, F(dst), dst_rows * dst_cols, src_ld, dst_cols, vr, vc, 0, r16));
    };
    auto Cp = [&](const float* src, size_t dst, int n_valid, int n_total) {
      add(make_job(L4D_JOB_COPY, src, F(dst), n_total, n_valid, 0, 0, 0, 0, r16));
    };
    auto U = [&](const float* W, int ld, int n_rows, int k0, int K, size_t dst, int rows_total, int row_off) {
      add(make_job(L4D_JOB_PACK_UMMA, W, H(dst), n_rows * K, ld, K, k0, rows_total, row_off));
    };
    // sigma net: params = [64][in_pad] | [16][64]
    const int ip = (int)cfg->sigma_in_pad;
    T(m->sigma_net, ip, L.sig_w1t, ip, 64, ip, 64);
    T(m->sigma_net + 64 * ip, 64, L.sig_w2t, 64, 16, 64, 16);
    Cp(m->sigma_net + 64 * ip, L.sig_w2, 16 * 64, 16 * 64);
    // attribute nets: [64][96] | [64][64] | [16][64]; image channel 0 = raydrop, 1 = intensity (lidar4d.py:216)
    const float* att[2] = {m->raydrop_net, m->intensity_net};
    const int ap = (int)cfg->attr_in_pad;
    for (int n = 0; n < 2; ++n) {
      T(att[n], ap, L.att_w1t[n], ap, 64, ap, 64);
      T(att[n] + 64 * ap, 64, L.att_w2t[n], 64, 64, 64, 64);
      Cp(att[n] + 64 * ap, L.att_w2[n], 64 * 64, 64 * 64);
      Cp(att[n] + 64 * ap + 64 * 64, L.att_w3[n], 64, 64);
    }
    // flow MLP: [64][16], [64][64], [6][64]
    T(m->flow_mlp[0], 16, L.flo_w0t, 16, 64, 16, 64);
    T(m->flow_mlp[1], 64, L.flo_w1t, 64, 64, 64, 64);
    Cp(m->flow_mlp[1], L.flo_w1, 64 * 64, 64 * 64);
    T(m->flow_mlp[2], 64, L.flo_w2t, 64, 8, 64, 6);
    Cp(m->flow_mlp[2], L.flo_w2, 6 * 64, 8 * 64);
    // tensor-core operand copies (fp16, no-swizzle K-major layout).  Rows / columns these jobs never write
    // (tc_att_w1g column 15, tc_flo_w2 rows 6..15) must be zero: the caller zero-fills `staged` once at allocation.
    U(m->sigma_net, ip, 64, 0, ip, L.tc_sig_w1, 64, 0);
    U(m->sigma_net + 64 * ip, 64, 16, 0, 64, L.tc_sig_w2, 16, 0);
    for (int n = 0; n < 2; ++n) {
      U(att[n], ap, 64, L4D_ENC, 15, L.tc_att_w1g, 128, n * 64);
      U(att[n] + 64 * ap, 64, 64, 0, 64, L.tc_att_w2[n], 64, 0);
      U(att[n], ap, 64, L4D_ENC, 16, L.tc_att_w1g_net[n], 64, 0);
    }
    U(m->flow_mlp[0], 16, 64, 0, 16, L.tc_flo_w0, 64, 0);
    U(m->flow_mlp[1], 64, 64, 0, 64, L.tc_flo_w1, 64, 0);
    U(m->flow_mlp[2], 64, 6, 0, 64, L.tc_flo_w2, 16, 0);
    if (nj > L4D_MAX_JOBS) return l4d_fail(L4D_EINVAL, "too many staging jobs");
    J.n_jobs = nj;
    for (int i = 0; i < nj; ++i) maxn = J.job[i].n > maxn ? J.job[i].n : maxn;
    int gx = (maxn + 256 * 8 - 1) / (256 * 8);
    if (gx < 1) gx = 1;
    ++g_launches; k_stage_jobs<<<dim3(gx, nj), 256, 0, st>>>(J);
  }
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_stage_params(const L4DConfig* cfg, const L4DMasterParams* m, void* staged, size_t staged_bytes,
                                void* stream) {
  // the operand-copy padding must be zero; callers of the _ex variant zero-fill once, this entry point does it per call
  if (cfg && staged && check_config(cfg) == L4D_OK) {
    StagedLayout L = staged_layout(cfg);
    if (staged_bytes >= L.total) {
      char* b = reinterpret_cast<char*>(staged);
      cudaMemsetAsync(b + L.tc_att_w1g, 0, 16 * 128 * 2, (cudaStream_t)stream);
      cudaMemsetAsync(b + L.tc_flo_w2, 0, 64 * 16 * 2, (cudaStream_t)stream);
    }
  }
  return l4d_stage_params_ex(cfg, m, staged, staged_bytes, L4D_STAGE_TABLES | L4D_STAGE_SMALL, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// Adam over the flat arenas, fused with the fp16 refresh of the hash tables (l4d_optim.cuh)
// ---------------------------------------------------------------------------------------------------------------
extern "C" int l4d_adam_step(const L4DConfig* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                             uint64_t n_floats, const L4DAdamGroup* groups, uint32_t n_groups, float beta1, float beta2,
                             float eps, uint32_t step, float inv_scale, uint32_t zero_grad, const L4DMasterParams* master,
                             void* staged, size_t staged_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!params || !grads || !exp_avg || !exp_avg_sq || !groups) return l4d_fail(L4D_EINVAL, "null pointer");
  if (n_groups < 1 || n_groups > L4D_ADAM_MAX_SEGMENTS) return l4d_fail(L4D_EINVAL, "1..64 Adam groups");
  if (n_floats % L4D_ADAM_CHUNK || step < 1) return l4d_fail(L4D_EINVAL, "arena size must be a multiple of 1024 floats, step >= 1");
  if ((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15)) return l4d_fail(L4D_EINVAL, "arenas must be 16-byte aligned");
  AdamArgs A;
  memset(&A, 0, sizeof(A));
  A.p = params; A.g = grads; A.g_rw = grads; A.m = exp_avg; A.v = exp_avg_sq;
  A.n_chunks = n_floats / L4D_ADAM_CHUNK;
  A.beta1 = beta1; A.beta2 = beta2; A.eps = eps; A.inv_scale = inv_scale; A.zero_grad = zero_grad;
  A.step = (float)step;                 // bias corrections: in fp32 on the device, as torch's fused Adam computes them
  A.n_seg = (int)n_groups;
  StagedLayout L;
  char* sb = reinterpret_cast<char*>(staged);
  if (master) {
    if (!staged) return l4d_fail(L4D_EINVAL, "master given without a staged buffer");
    L = staged_layout(cfg);
    if (staged_bytes < L.total) return l4d_fail(L4D_ESIZE, "staged buffer too small");
  }
  unsigned long long prev_end = 0;
  for (uint32_t i = 0; i < n_groups; ++i) {
    AdamSeg& s = A.seg[i];
    s.begin = groups[i].begin; s.end = groups[i].end; s.lr = groups[i].lr;
    if (s.begin % L4D_ADAM_CHUNK || s.end <= s.begin || s.end > n_floats || s.begin < prev_end || (s.end & 3))
      return l4d_fail(L4D_EINVAL, "Adam groups must be sorted, disjoint, start on multiples of 1024 floats and end on multiples of 4");
    prev_end = s.end;
    if (!master) continue;
    const float* gp = params + s.begin;
    const unsigned long long len = s.end - s.begin;
    if (gp == master->hash_static && len == (unsigned long long)cfg->hash_static.offset[cfg->hash_static.n_levels] * 4) {
      s.dst0 = reinterpret_cast<unsigned char*>(sb + L.hs); s.stride0 = 8;
    } else if (gp == master->flow_grid && len == (unsigned long long)cfg->flow.offset[cfg->flow.n_levels] * 8) {
      s.dst0 = reinterpret_cast<unsigned char*>(sb + L.hf); s.stride0 = 8;
    } else {
      for (int p = 0; p < 3; ++p) {
        const unsigned long long ne = cfg->hash_dynamic[p].offset[cfg->hash_dynamic[p].n_levels];
        for (uint32_t t = 0; t < cfg->time_resolution; ++t) {
          if (gp != master->hash_dynamic[p][t] || len != ne * 4) continue;
          unsigned char* base = reinterpret_cast<unsigned char*>(sb + L.hd[p]);        // pair k = slices k, k+1: {lo 4 halves | hi 4 halves}
          if (t + 1 < cfg->time_resolution) { s.dst0 = base + (size_t)t * ne * 16; s.stride0 = 16; s.off0 = 0; }
          if (t > 0) { s.dst1 = base + (size_t)(t - 1) * ne * 16; s.stride1 = 16; s.off1 = 8; }
        }
      }
    }
  }
  unsigned long long blocks = A.n_chunks;
  const unsigned long long cap = (unsigned long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  ++g_launches; k_adam_flat<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_grad_work_bytes(const L4DConfig* cfg) {
  if (check_config(cfg) != L4D_OK) return 0;
  return grad_work_layout(cfg).total;
}

extern "C" int l4d_unstage_grads(const L4DConfig* cfg, const void* grad_work, size_t grad_work_bytes,
                                 const L4DMasterGrads* g, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!grad_work || !g) return l4d_fail(L4D_EINVAL, "null pointer");
  GradWorkLayout L = grad_work_layout(cfg);
  if (grad_work_bytes < L.total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  const char* b = reinterpret_cast<const char*>(grad_work);
  auto F = [&](size_t off) { return reinterpret_cast<const float*>(b + off); };
  JobArgs J;
  int nj = 0, maxn = 0;
  auto add = [&](int type, size_t src, float* dst, int n, int a = 0, int bb = 0) {
    if (!dst) return;
    if (nj < L4D_MAX_JOBS) J.job[nj] = make_job(type, F(src), dst, n, a, bb);
    ++nj;
    maxn = n > maxn ? n : maxn;
  };
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) {
      int Hh, W;
      plane_hw(cfg, s, ci, Hh, W);
      add(L4D_JOB_PLANE_FROM_CL, L.planes[s][ci], g->planes[s][ci], Hh * W * 8, Hh * W);
    }
  const int ip = (int)cfg->sigma_in_pad, ap = (int)cfg->attr_in_pad;
  add(L4D_JOB_ADD_TRANSPOSED, L.sig_w1t, g->sigma_net, 64 * ip, 64, ip);
  add(L4D_JOB_ADD, L.sig_w2, g->sigma_net ? g->sigma_net + 64 * ip : nullptr, 16 * 64);
  float* att[2] = {g->raydrop_net, g->intensity_net};
  for (int n = 0; n < 2; ++n) {
    if (!att[n]) continue;
    add(L4D_JOB_ADD_TRANSPOSED, L.att_w1t[n], att[n], 64 * ap, 64, ap);
    add(L4D_JOB_ADD_TRANSPOSED, L.att_w2t[n], att[n] + 64 * ap, 64 * 64, 64, 64);
    add(L4D_JOB_ADD, L.att_w3[n], att[n] + 64 * ap + 64 * 64, 64);       // row 0 of the [16][64] output layer
  }
  add(L4D_JOB_ADD_TRANSPOSED, L.flo_w0t, g->flow_mlp[0], 64 * 16, 64, 16);
  add(L4D_JOB_ADD_TRANSPOSED, L.flo_w1t, g->flow_mlp[1], 64 * 64, 64, 64);
  add(L4D_JOB_ADD, L.flo_w2, g->flow_mlp[2], 6 * 64);
  if (nj > L4D_MAX_JOBS) return l4d_fail(L4D_EINVAL, "too many unstaging jobs");
  if (nj == 0) return L4D_OK;
  J.n_jobs = nj;
  int gx = (maxn + 256 * 8 - 1) / (256 * 8);
  ++g_launches; k_unstage_jobs<<<dim3(gx < 1 ? 1 : gx, nj), 256, 0, st>>>(J);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// block-level primitives
// =============================================================================
template <int NT>
__device__ __forceinline__ float block_excl_prod(float v, float* s_w, float& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= t;
  }
  if (lane == 31) s_w[warp] = inc;
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) ex = 1.f;
  __syncthreads();
  float pre = 1.f, tot = 1.f;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) {
    float t = s_w[w];
    if (w < warp) pre *= t;
    tot *= t;
  }
  total = tot;
  __syncthreads();
  return pre * ex;
}

// exclusive suffix sum: result_j = sum_{k>j} v_k within the block; total = sum of all
template <int NT>
__device__ __forceinline__ float block_excl_suffix_sum(float v, float* s_w, float& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_down_sync(0xffffffffu, inc, o);
    if (lane + o < 32) inc += t;
  }
  if (lane == 0) s_w[warp] = inc;
  float ex = __shfl_down_sync(0xffffffffu, inc, 1);
  if (lane == 31) ex = 0.f;
  __syncthreads();
  float post = 0.f, tot = 0.f;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) {
    float t = s_w[w];
    if (w > warp) post += t;
    tot += t;
  }
  total = tot;
  __syncthreads();
  return post + ex;
}

template <int NT>
__device__ __forceinline__ float block_sum(float v, float* s_w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) s_w[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) t += s_w[w];
  __syncthreads();
  return t;
}

// dW[k][0..64) += sum_m TA[m][k] * TB[m][0..64) for k < K (K multiple of 8, <= 64); all NT threads.
// Work items = 16-row blocks of k x m-ranges, one per warp; lanes own columns j and j+32.
template <int NT>
__device__ __forceinline__ void tile_outer_accum(const float* __restrict__ TA, const float* __restrict__ TB, int K,
                                                 float* __restrict__ dW) {
  constexpr int NW = NT / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nkb = (K + 15) / 16;
  const int ms = nkb >= NW ? 1 : NW / nkb;
  const int items = nkb * ms;
  const int mlen = NT / ms;
  for (int it = warp; it < items; it += NW) {
    const int kb = it / ms, k0 = kb * 16;
    const int m0 = (it % ms) * mlen;
    float a0[16], a1[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { a0[k] = 0.f; a1[k] = 0.f; }
    for (int m = m0; m < m0 + mlen; ++m) {
      const float4* ar = reinterpret_cast<const float4*>(TA + (size_t)m * L4D_TILE_LD + k0);
      const float b0 = TB[(size_t)m * L4D_TILE_LD + lane];
      const float b1 = TB[(size_t)m * L4D_TILE_LD + lane + 32];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 a = ar[q];
        a0[4 * q + 0] = fmaf(a.x, b0, a0[4 * q + 0]); a1[4 * q + 0] = fmaf(a.x, b1, a1[4 * q + 0]);
        a0[4 * q + 1] = fmaf(a.y, b0, a0[4 * q + 1]); a1[4 * q + 1] = fmaf(a.y, b1, a1[4 * q + 1]);
        a0[4 * q + 2] = fmaf(a.z, b0, a0[4 * q + 2]); a1[4 * q + 2] = fmaf(a.z, b1, a1[4 * q + 2]);
        a0[4 * q + 3] = fmaf(a.w, b0, a0[4 * q + 3]); a1[4 * q + 3] = fmaf(a.w, b1, a1[4 * q + 3]);
      }
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (k0 + k < K) {
        atomicAdd(dW + (size_t)(k0 + k) * 64 + lane, a0[k]);
        atomicAdd(dW + (size_t)(k0 + k) * 64 + lane + 32, a1[k]);
      }
    }
  }
}

// column sums of a tile: out[j] = sum_m T[m][j], j<64.  threads 0..63 return their column's sum
template <int NT>
__device__ __forceinline__ float tile_colsum(const float* __restrict__ T) {
  float s = 0.f;
  if (threadIdx.x < 64) {
    for (int m = 0; m < NT; ++m) s += T[(size_t)m * L4D_TILE_LD + threadIdx.x];
  }
  return s;
}

#include "l4d_split.cuh"
#include "l4d_dense_tc.cuh"

// =============================================================================
// forward render kernel
// =============================================================================
struct FwdArgs {
  DevModel M;
  L4DFrameTable FT;
  const float* rays_o;
  const float* rays_d;
  uint32_t n_rays, S, perturb;
  uint64_t seed, ray_offset;
  float *depth, *image, *wsum, *weights, *zvals;
  SavedView sv;
  uint32_t train;
};

template <int NT, bool MF>
__global__ void __launch_bounds__(NT) k_render_fwd(const __grid_constant__ FwdArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;                 // [64][NT]
  float* s_enc = xbuf + 64 * NT;      // [80]
  float* s_cdir = s_enc + 80;         // [128]
  float* s_w = s_cdir + 128;          // [32]
  const DevModel& M = A.M;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t S = A.S;

  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
    const L4DFrame& F = A.FT.frames[l4d_frame_of<MF>(A.FT, ray)];
    const float ox = __ldg(A.rays_o + 3 * ray), oy = __ldg(A.rays_o + 3 * ray + 1), oz = __ldg(A.rays_o + 3 * ray + 2);
    const float dx = __ldg(A.rays_d + 3 * ray), dy = __ldg(A.rays_d + 3 * ray + 1), dz = __ldg(A.rays_d + 3 * ray + 2);
    __syncthreads();
    for (int i = tid; i < L4D_ENC; i += NT) {
      const int dim = i / 24, k = (i % 24) >> 1, ph = i & 1;
      s_enc[i] = l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), k, ph);
    }
    __syncthreads();
    for (int i = tid; i < 128; i += NT) s_cdir[i] = l4d_attr_cdir(M, i >> 6, i & 63, s_enc);
    __syncthreads();

    float carry = 1.f, pd = 0.f, p0 = 0.f, p1 = 0.f, pw = 0.f;
    const uint64_t rg = A.ray_offset + ray;
    for (uint32_t j0 = 0; j0 < S; j0 += NT) {
      const uint32_t j = j0 + tid;
      const bool valid = j < S;
      const size_t p = (size_t)ray * S + j;
      float zj = 0.f, alpha = 0.f, sigma = 0.f, geo[L4D_GEO];
      if (valid) {
        zj = l4d_z(rs, rg, j);
        const float delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
        const float x = l4d_x01(ox, dx, zj, M.bound), y = l4d_x01(oy, dy, zj, M.bound), z = l4d_x01(oz, dz, zj, M.bound);
        FeatSink sink;
        sink.feat = A.train ? A.sv.feat : nullptr;
        sink.P = A.sv.P;
        sink.p = p;
        sink.dense = nullptr;
        float h0, fl[6];
        l4d_density_sample(M, F, x, y, z, xb, NT, sink, A.train ? A.sv.flow_in + p : nullptr, A.sv.P, sigma, h0, geo, fl);
        alpha = l4d_alpha(M, delta, sigma);
      }
      const float v = valid ? (1.0f - alpha) + 1e-15f : 1.f;
      float total;
      const float T = carry * block_excl_prod<NT>(v, s_w, total);
      carry *= total;
      const float w = alpha * T;
      float a0 = 0.f, a1 = 0.f;
      if (valid && w > 1e-4f) {
        a0 = l4d_attr_net(M, 0, s_cdir, geo, xb, NT);
        a1 = l4d_attr_net(M, 1, s_cdir, geo, xb, NT);
      }
      pd = fmaf(w, zj, pd); p0 = fmaf(w, a0, p0); p1 = fmaf(w, a1, p1); pw += w;
      if (valid) {
        if (A.train) { A.sv.sigma[p] = sigma; A.sv.attr[p] = a0; A.sv.attr[A.sv.P + p] = a1; }
        if (A.weights) A.weights[p] = w;
        if (A.zvals) A.zvals[p] = zj;
      }
    }
    pd = block_sum<NT>(pd, s_w); p0 = block_sum<NT>(p0, s_w); p1 = block_sum<NT>(p1, s_w); pw = block_sum<NT>(pw, s_w);
    if (tid == 0) {
      A.depth[ray] = pd; A.image[2 * ray] = p0; A.image[2 * ray + 1] = p1; A.wsum[ray] = pw;
    }
  }
}

// =============================================================================
// backward render kernel
// =============================================================================
#define L4D_MAX_TILES 64
struct BwdArgs {
  DevModel M;
  L4DFrameTable FT;
  DevGrads G;
  const float* rays_o;
  const float* rays_d;
  uint32_t n_rays, S, perturb;
  uint64_t seed, ray_offset;
  const float *g_depth, *g_image, *g_wsum, *g_weights;
  SavedView sv;
};

template <int NT>
__global__ void __launch_bounds__(NT) k_render_bwd(const __grid_constant__ BwdArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;                             // [64][NT]
  float* TA = xbuf + 64 * NT;                     // [NT][LD]
  float* TB = TA + NT * L4D_TILE_LD;              // [NT][LD]
  float* s_enc = TB + NT * L4D_TILE_LD;           // [80]
  float* s_cdir = s_enc + 80;                     // [128]
  float* s_csum = s_cdir + 128;                   // [128]
  float* s_w = s_csum + 128;                      // [32]
  float* s_tstart = s_w + 32;                     // [L4D_MAX_TILES]
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  float* ta_row = TA + (size_t)tid * L4D_TILE_LD;
  float* tb_row = TB + (size_t)tid * L4D_TILE_LD;
  float* hid = A.sv.hidden + (size_t)blockIdx.x * 64 * NT + tid;   // per-CTA scratch column, stride NT
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t S = A.S;
  const int n_tiles = (int)((S + NT - 1) / NT);
  const float kk = M.active_sensor ? 2.0f : 1.0f;
  const int n_chunks = (int)(M.sigma_in_pad + 63) / 64;

  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
    const L4DFrame& F = A.FT.frames[l4d_frame_of(A.FT, ray)];
    const float ox = __ldg(A.rays_o + 3 * ray), oy = __ldg(A.rays_o + 3 * ray + 1), oz = __ldg(A.rays_o + 3 * ray + 2);
    const float dx = __ldg(A.rays_d + 3 * ray), dy = __ldg(A.rays_d + 3 * ray + 1), dz = __ldg(A.rays_d + 3 * ray + 2);
    const float gd = __ldg(A.g_depth + ray), gi0 = __ldg(A.g_image + 2 * ray), gi1 = __ldg(A.g_image + 2 * ray + 1);
    const float gws = A.g_wsum ? __ldg(A.g_wsum + ray) : 0.f;
    const uint64_t rg = A.ray_offset + ray;
    __syncthreads();
    for (int i = tid; i < L4D_ENC; i += NT) {
      const int dim = i / 24, k = (i % 24) >> 1, ph = i & 1;
      s_enc[i] = l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), k, ph);
    }
    for (int i = tid; i < 128; i += NT) s_csum[i] = 0.f;
    __syncthreads();
    for (int i = tid; i < 128; i += NT) s_cdir[i] = l4d_attr_cdir(M, i >> 6, i & 63, s_enc);
    __syncthreads();

    // ---- pass 1: transmittance at the start of every tile ----
    {
      float carry = 1.f;
      for (int t = 0; t < n_tiles; ++t) {
        const uint32_t j = (uint32_t)t * NT + tid;
        const bool valid = j < S;
        float v = 1.f;
        if (valid) {
          const float zj = l4d_z(rs, rg, j);
          const float delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
          const float alpha = l4d_alpha(M, delta, A.sv.sigma[(size_t)ray * S + j]);
          v = (1.0f - alpha) + 1e-15f;
        }
        if (tid == 0) s_tstart[t] = carry;
        float total;
        block_excl_prod<NT>(v, s_w, total);
        carry *= total;
      }
    }
    __syncthreads();

    // ---- pass 2: tiles in reverse, carrying the suffix sum of dL/dw * w ----
    float suffix = 0.f;
    for (int t = n_tiles - 1; t >= 0; --t) {
      const uint32_t j = (uint32_t)t * NT + tid;
      const size_t p = (size_t)ray * S + j;
      BwSample s;
      s.active = j < S;
      s.masked = false;
      s.dsigma = 0.f; s.da[0] = 0.f; s.da[1] = 0.f;
      s.x = s.y = s.z = 0.f;
      float v = 1.f, q = 0.f, alpha = 0.f, gw = 0.f, delta = 0.f;
      if (s.active) {
        const float zj = l4d_z(rs, rg, j);
        delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
        s.x = l4d_x01(ox, dx, zj, M.bound); s.y = l4d_x01(oy, dy, zj, M.bound); s.z = l4d_x01(oz, dz, zj, M.bound);
        alpha = l4d_alpha(M, delta, A.sv.sigma[p]);
        v = (1.0f - alpha) + 1e-15f;
        gw = gd * zj + gi0 * A.sv.attr[p] + gi1 * A.sv.attr[A.sv.P + p] + gws;
        if (A.g_weights) gw += __ldg(A.g_weights + p);
      }
      float total;
      const float T = s_tstart[t] * block_excl_prod<NT>(v, s_w, total);
      const float w = alpha * T;
      q = gw * w;
      float qtot;
      const float suf = suffix + block_excl_suffix_sum<NT>(q, s_w, qtot);
      suffix += qtot;
      if (s.active) {
        const float dalpha = gw * T - suf / v;
        s.dsigma = dalpha * (kk * delta * M.density_scale) * (1.0f - alpha);
        s.masked = w > 1e-4f;
        if (s.masked) { s.da[0] = w * gi0; s.da[1] = w * gi1; }
      }

      // B0 / B1: recompute flow + sigma MLP forward
      l4d_bw_flow_fwd(M, s, A.sv.flow_in + p, A.sv.P, xb, NT);
      l4d_bw_sigma_fwd(M, s, A.sv.feat + p, A.sv.P, xb, NT, hid, NT);

      // B2: attribute heads
#pragma unroll 1
      for (int net = 0; net < 2; ++net) {
        uint32_t m1a, m1b;
        l4d_bw_attr_a(M, net, s, s_cdir, xb, NT, ta_row, tb_row, m1a, m1b);
        __syncthreads();
        {
          const float cs = tile_colsum<NT>(TB);
          if (tid < 64) atomicAdd(G.att_w3[net] + tid, cs);
        }
        __syncthreads();
        l4d_bw_attr_b(xb, NT, tb_row);
        __syncthreads();
        tile_outer_accum<NT>(TA, TB, 64, G.att_w2t[net]);
        __syncthreads();
        l4d_bw_attr_c(M, net, s, xb, NT, ta_row, tb_row, m1a, m1b);
        __syncthreads();
        tile_outer_accum<NT>(TA, TB, 16, G.att_w1t[net] + (size_t)L4D_ENC * 64);
        {
          const float cs = tile_colsum<NT>(TB);
          if (tid < 64) s_csum[net * 64 + tid] += cs;
        }
        __syncthreads();
      }

      // B3: sigma MLP backprop
      l4d_bw_sigma_a(M, s, hid, NT, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 16, G.sig_w2);
      __syncthreads();
      l4d_bw_sigma_b(M, s, xb, NT, tb_row);
#pragma unroll 1
      for (int c = 0; c < n_chunks; ++c) {
        l4d_bw_sigma_c(M, s, A.sv.feat + p, A.sv.P, c, ta_row);
        __syncthreads();
        const int rows = min(64, (int)M.sigma_in_pad - c * 64);
        tile_outer_accum<NT>(TA, TB, rows, G.sig_w1t + (size_t)c * 64 * 64);
        __syncthreads();
      }

      // B4: encoders
      l4d_bw_scatter<false>(M, F, G, s);

      // B5: flow MLP backprop + flow grid
      l4d_bw_flow_a(M, s, A.sv.flow_in + p, A.sv.P, s.dflow, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 8, G.flo_w2);
      __syncthreads();
      l4d_bw_flow_b(M, s, s.dflow, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 64, G.flo_w1t);
      __syncthreads();
      l4d_bw_flow_c(M, F, G, s, A.sv.flow_in + p, A.sv.P, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 16, G.flo_w0t);
      __syncthreads();
    }

    // direction / ones rows of the first attribute layer: dW1t[k][j] += enc[k] * sum_samples dh1[j]
    for (int i = tid; i < 2 * (L4D_ENC + 9) * 64; i += NT) {
      const int net = i / ((L4D_ENC + 9) * 64);
      const int r = (i / 64) % (L4D_ENC + 9), jx = i & 63;
      const float cs = s_csum[net * 64 + jx];
      if (r < L4D_ENC) atomicAdd(G.att_w1t[net] + (size_t)r * 64 + jx, s_enc[r] * cs);
      else atomicAdd(G.att_w1t[net] + (size_t)(M.attr_in_dim + (r - L4D_ENC)) * 64 + jx, cs);
    }
  }
}

// =============================================================================
// flow-only kernels (LiDAR4D.flow, lidar4d.py:124-137)
// =============================================================================
struct FlowArgs {
  DevModel M;
  L4DFrame F;
  DevGrads G;
  const float* x;
  uint32_t n;
  float* flow;
  float* saved;         // [16][n] or null
  const float* g_flow;  // [n][6]
};

template <int NT>
__global__ void __launch_bounds__(NT) k_flow_fwd(const __grid_constant__ FlowArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;
  const DevModel& M = A.M;
  for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
    const uint32_t i = base + threadIdx.x;
    if (i < A.n) {
      const float b2 = L4D_MUL(2.0f, M.bound);
      const float x = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i), M.bound), b2);
      const float y = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i + 1), M.bound), b2);
      const float z = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i + 2), M.bound), b2);
      l4d_flow_inputs(M, A.F.flow_basis, x, y, z, xb, NT, A.saved ? A.saved + i : nullptr, A.n);
      float fl[8];
      uint32_t a, b, c, d;
      l4d_flow_mlp(M, xb, NT, fl, a, b, c, d);
#pragma unroll
      for (int k = 0; k < 6; ++k) A.flow[(size_t)i * 6 + k] = fl[k];
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(NT) k_flow_bwd(const __grid_constant__ FlowArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;
  float* TA = xbuf + 64 * NT;
  float* TB = TA + NT * L4D_TILE_LD;
  float* xb = xbuf + threadIdx.x;
  float* ta_row = TA + (size_t)threadIdx.x * L4D_TILE_LD;
  float* tb_row = TB + (size_t)threadIdx.x * L4D_TILE_LD;
  const DevModel& M = A.M;
  for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
    const uint32_t i = base + threadIdx.x;
    BwSample s;
    s.active = i < A.n;
    s.masked = false;
    s.x = s.y = s.z = 0.f;
    float g[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const size_t ii = s.active ? i : 0;
    if (s.active) {
      const float b2 = L4D_MUL(2.0f, M.bound);
      s.x = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i), M.bound), b2);
      s.y = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i + 1), M.bound), b2);
      s.z = L4D_DIV(L4D_ADD(__ldg(A.x + 3 * i + 2), M.bound), b2);
#pragma unroll
      for (int k = 0; k < 6; ++k) g[k] = __ldg(A.g_flow + (size_t)i * 6 + k);
    }
    __syncthreads();
    l4d_bw_flow_fwd(M, s, A.saved + ii, A.n, xb, NT);
    l4d_bw_flow_a(M, s, A.saved + ii, A.n, g, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 8, A.G.flo_w2);
    __syncthreads();
    l4d_bw_flow_b(M, s, g, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 64, A.G.flo_w1t);
    __syncthreads();
    l4d_bw_flow_c(M, A.F, A.G, s, A.saved + ii, A.n, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 16, A.G.flo_w0t);
  }
}

// =============================================================================
// debug kernels
// =============================================================================
__global__ void k_hash_indices(DevGrid g, int D, int level, const float* x, uint32_t n, uint32_t* idx, float* w) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (D == 3) {
    uint32_t id[8]; float ww[8];
    l4d_corners3(g, level, x[3 * i], x[3 * i + 1], x[3 * i + 2], id, ww);
    for (int c = 0; c < 8; ++c) { idx[8 * i + c] = id[c]; w[8 * i + c] = ww[c]; }
  } else {
    uint32_t id[4]; float ww[4];
    l4d_corners2(g, level, x[2 * i], x[2 * i + 1], id, ww);
    for (int c = 0; c < 4; ++c) { idx[4 * i + c] = id[c]; w[4 * i + c] = ww[c]; }
  }
}

struct DensityArgs {
  DevModel M;
  L4DFrame F;
  const float* x;
  uint32_t n;
  float *sigma, *geo, *features, *flow;
};
template <int NT>
__global__ void __launch_bounds__(NT) k_density(const __grid_constant__ DensityArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;
  const DevModel& M = A.M;
  const uint32_t i = blockIdx.x * NT + threadIdx.x;
  if (i >= A.n) return;
  const float b2 = L4D_MUL(2.0f, M.bound);
  const float x = L4D_DIV(L4D_ADD(A.x[3 * i], M.bound), b2);
  const float y = L4D_DIV(L4D_ADD(A.x[3 * i + 1], M.bound), b2);
  const float z = L4D_DIV(L4D_ADD(A.x[3 * i + 2], M.bound), b2);
  FeatSink sink;
  sink.feat = nullptr; sink.P = 0; sink.p = 0;
  sink.dense = A.features ? A.features + (size_t)i * M.sigma_in_dim : nullptr;
  float sigma, h0, geo[L4D_GEO], fl[6];
  l4d_density_sample(M, A.F, x, y, z, xb, NT, sink, nullptr, 0, sigma, h0, geo, fl);
  A.sigma[i] = sigma;
  for (int k = 0; k < L4D_GEO; ++k) A.geo[(size_t)i * L4D_GEO + k] = geo[k];
  if (A.flow) for (int k = 0; k < 6; ++k) A.flow[(size_t)i * 6 + k] = fl[k];
}

// LiDAR4D.attribute on explicit points (parity / API completeness; render() has the heads fused in)
struct AttributeArgs {
  DevModel M;
  const float* d;
  const float* geo;
  const unsigned char* mask;
  uint32_t n;
  float* out;
};
template <int NT>
__global__ void __launch_bounds__(NT) k_attribute(const __grid_constant__ AttributeArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;                    // exchange column, stride NT
  float* enc = smem + 64 * NT + threadIdx.x * 81;    // this point's direction encoding (odd stride: conflict-free)
  float* cdir = smem + 64 * NT + 81 * NT + threadIdx.x * 129;
  const DevModel& M = A.M;
  const uint32_t i = blockIdx.x * NT + threadIdx.x;
  if (i >= A.n) return;
  float o0 = 0.f, o1 = 0.f;
  if (!A.mask || A.mask[i]) {
    const float dx = A.d[3 * i], dy = A.d[3 * i + 1], dz = A.d[3 * i + 2];
    for (int k = 0; k < L4D_ENC; ++k) {
      const int dim = k / 24, f = (k % 24) >> 1, ph = k & 1;
      enc[k] = l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), f, ph);
    }
    for (int k = 0; k < 128; ++k) cdir[k] = l4d_attr_cdir(M, k >> 6, k & 63, enc);
    float geo[L4D_GEO];
    for (int k = 0; k < L4D_GEO; ++k) geo[k] = A.geo[(size_t)i * L4D_GEO + k];
    o0 = l4d_attr_net(M, 0, cdir, geo, xb, NT);
    o1 = l4d_attr_net(M, 1, cdir, geo, xb, NT);
  }
  A.out[2 * i] = o0;
  A.out[2 * i + 1] = o1;
}

#include "l4d_points.cuh"
#include "l4d_modules.cuh"

// =============================================================================
// C-ABI launchers
// =============================================================================

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// n_steps = 1 is refused: the reference's deltas z[1:] - z[:-1] are empty there, so its weights are [N, 0] and depth,
// image and weight sum are 0 - an artefact of broadcasting an empty tensor, not a render
static int check_n_steps(uint32_t n_steps) {
  if (n_steps < 2 || n_steps > L4D_MAX_TILES * L4D_NT) return l4d_fail(L4D_EINVAL, "n_steps out of range [2, 8192]");
  return L4D_OK;
}

extern "C" size_t l4d_saved_bytes(const L4DConfig* cfg, uint32_t n_rays, uint32_t n_steps) {
  return l4d_saved_bytes_frames(cfg, n_rays, n_steps, 1);
}

static int check_n_frames(uint32_t n_frames) {
  if (n_frames == 0 || n_frames > L4D_MAX_FRAMES) return l4d_fail(L4D_EINVAL, "n_frames out of range [1, L4D_MAX_FRAMES]");
  return L4D_OK;
}
extern "C" size_t l4d_saved_bytes_frames(const L4DConfig* cfg, uint32_t n_rays, uint32_t n_steps, uint32_t n_frames) {
  if (check_config(cfg) != L4D_OK || check_n_steps(n_steps) != L4D_OK || check_n_frames(n_frames) != L4D_OK) return 0;
  return saved_layout(cfg, n_rays, n_steps, n_frames).total;
}
extern "C" size_t l4d_grad_work_bytes_frames(const L4DConfig* cfg, uint32_t n_frames) {
  if (check_config(cfg) != L4D_OK || check_n_frames(n_frames) != L4D_OK) return 0;
  return grad_work_layout(cfg, n_frames).total;
}

// a frame table must name a frame for every ray of the launch
static int check_frames(const L4DFrameTable* T, uint32_t n_rays) {
  if (!T) return l4d_fail(L4D_EINVAL, "null frame table");
  int rc = check_n_frames(T->n_frames);
  if (rc != L4D_OK) return rc;
  if (T->rays_per_frame == 0) return l4d_fail(L4D_EINVAL, "rays_per_frame is 0");
  if (T->first_ray_phase >= T->rays_per_frame) return l4d_fail(L4D_EINVAL, "first_ray_phase >= rays_per_frame");
  if ((uint64_t)T->first_ray_phase + n_rays > (uint64_t)T->n_frames * T->rays_per_frame)
    return l4d_fail(L4D_EINVAL, "the frame table does not cover n_rays");
  return L4D_OK;
}
// the one-frame table of the single-frame entry points
static L4DFrameTable one_frame(const L4DFrame* frame, uint32_t n_rays) {
  L4DFrameTable T;
  memset(&T, 0, sizeof(T));
  T.n_frames = 1;
  T.rays_per_frame = n_rays > 0 ? n_rays : 1;
  T.frames[0] = *frame;
  return T;
}

static int check_rays(const L4DRays* r) {
  if (!r || !r->rays_o || !r->rays_d) return l4d_fail(L4D_EINVAL, "null rays");
  return check_n_steps(r->n_steps);
}

template <typename K>
static int grid_for(K kernel, int nt, size_t smem, uint32_t work, int& grid, int force_per_sm = 0) {
  // the attribute / occupancy calls cost ~10 us of host time each: remember the answer per (kernel, smem, threads) -
  // at the reference's 1,024-ray step the 15 launches of a step are otherwise host-bound
  struct Memo { const void* k; size_t smem; int nt, force, per_sm; };
  struct SmemSet { const void* k; size_t max_set; };
  static thread_local Memo memo[64];
  static thread_local SmemSet smem_set[32];
  static thread_local int n_memo = 0, n_set = 0;
  int per_sm = 0;
  const void* key = reinterpret_cast<const void*>(kernel);
  // the opt-in dynamic shared-memory limit is a sticky per-function attribute: only ever RAISE it (configurations with
  // different tile sizes alternate in one process, and lowering it would make the larger one's next launch invalid)
  {
    SmemSet* e = nullptr;
    for (int i = 0; i < n_set; ++i) if (smem_set[i].k == key) { e = &smem_set[i]; break; }
    if (!e || smem > e->max_set) {
      cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (err != cudaSuccess) return l4d_fail(L4D_ECUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(err));
      if (e) e->max_set = smem;
      else if (n_set < 32) smem_set[n_set++] = SmemSet{key, smem};
    }
  }
  for (int i = 0; i < n_memo; ++i)
    if (memo[i].k == key && memo[i].smem == smem && memo[i].nt == nt && memo[i].force == force_per_sm) { per_sm = memo[i].per_sm; break; }
  if (per_sm == 0) {
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, nt, smem);
    if (e != cudaSuccess) return l4d_fail(L4D_ECUDA, "occupancy query: %s", cudaGetErrorString(e));
    if (per_sm < 1) per_sm = 1;
    if (force_per_sm > 0) per_sm = force_per_sm;
    // small-shared-memory kernels: ask for just the carve-out the resident CTAs need, the rest stays L1 (the driver's
    // default for k_fwd_gather was 132 KB of shared memory for 55 KB of use, i.e. half of the L1 given away)
    if (smem <= 16 * 1024) {
      const size_t need = (size_t)per_sm * (smem + 1024);
      int pct = (int)((need * 100 + 233471) / 233472);
      if (pct > 100) pct = 100;
      cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    }
    if (n_memo < 64) memo[n_memo++] = Memo{key, smem, nt, force_per_sm, per_sm};
  }
  long g = (long)per_sm * sm_count();
  if ((long)work < g) g = work;
  if (g < 1) g = 1;
  grid = (int)g;
  return L4D_OK;
}

// the frame table travels in the kernel parameter block (no copy, no sync): it needs the large parameter space of CUDA 12.1+
static_assert(sizeof(SplitArgs) <= 32764 && sizeof(FwdArgs) <= 32764 && sizeof(BwdArgs) <= 32764, "kernel parameter limit");

static void fill_split(SplitArgs& A, const L4DConfig* cfg, const void* staged, const L4DFrameTable* frames, const L4DRays* rays,
                       void* saved) {
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.FT = *frames;
  A.con_fstride = saved_layout(cfg, rays->n_rays, rays->n_steps).con_frame / sizeof(float);
  A.comb_fstride = grad_work_layout(cfg).comb_frame / sizeof(float);
  A.rays_o = rays->rays_o; A.rays_d = rays->rays_d;
  A.n_rays = rays->n_rays; A.S = rays->n_steps; A.perturb = rays->perturb;
  A.seed = rays->seed; A.ray_offset = rays->ray_offset;
  A.sv = saved_view(cfg, saved, rays->n_rays, rays->n_steps);
}

#define L4D_FLAG_FUSED 1u   /* L4DRays.reserved bit 0: single-kernel path */

// Dynamic shared memory of the tensor-core kernels: the carve-up plus the 128-byte alignment of its base
static size_t tc_dyn_smem(uint32_t bytes) { return (size_t)bytes + 128; }
// the tensor-core dense kernels hold a 128 x sigma_in_pad fp16 hi|lo tile in shared memory; on sm_90 (227 KB per CTA)
// the backward's carve-up (217 KB) fits the largest input a valid configuration has (176: 16 hash levels, 4 plane scales)
static bool use_tc_dense(const L4DConfig* cfg) {
  static int optin = 0;
  if (!optin) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  }
  return cfg->mlp_fp16 && cfg->sigma_in_pad <= 192 && tc_dyn_smem(dense_bwd_smem(cfg->sigma_in_pad).total) + 128 <= (size_t)optin;
}

// compositing backward of the tensor-core pipeline: per-sample dL/dsigma, attribute deltas and mask into quad 0 of the
// dL/dfeature tiles, where k_bwd_dense_tc picks them up
static int launch_bwd_composite(const SplitArgs& A, cudaStream_t st) {
  int grid;
  const int rc = grid_for(k_bwd_composite, 128, 0, A.n_rays, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_bwd_composite<<<grid, 128, 0, st>>>(A);
  prof_mark(st, "k_bwd_composite");
  return L4D_OK;
}

// k_bwd_composite alone, on the saved buffer of a training forward: afterwards feature columns 0..3 of the saved
// dL/dfeature hold {dL/dsigma, dL/da0, dL/da1, attribute mask} of every sample
extern "C" int l4d_composite_backward(const L4DConfig* cfg, const L4DRays* rays, void* saved, size_t saved_bytes,
                                      const float* g_depth, const float* g_image, const float* g_wsum, const float* g_weights,
                                      void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  rc = check_rays(rays);
  if (rc != L4D_OK) return rc;
  if (!saved || !g_depth || !g_image) return l4d_fail(L4D_EINVAL, "null pointer");
  if (!use_tc_dense(cfg)) return l4d_fail(L4D_EINVAL, "l4d_composite_backward: tensor-core configurations only");
  if (saved_bytes < saved_layout(cfg, rays->n_rays, rays->n_steps).total) return l4d_fail(L4D_ESIZE, "saved buffer too small");
  if (rays->n_rays == 0) return L4D_OK;
  SplitArgs A;
  memset(&A, 0, sizeof(A));
  A.M.near_lidar = cfg->near_lidar; A.M.far_lidar = cfg->far_lidar;
  A.M.active_sensor = cfg->active_sensor; A.M.density_scale = cfg->density_scale;
  A.n_rays = rays->n_rays; A.S = rays->n_steps; A.perturb = rays->perturb;
  A.seed = rays->seed; A.ray_offset = rays->ray_offset;
  A.g_depth = g_depth; A.g_image = g_image; A.g_wsum = g_wsum; A.g_weights = g_weights;
  A.sv = saved_view(cfg, saved, rays->n_rays, rays->n_steps);
  rc = launch_bwd_composite(A, (cudaStream_t)stream);
  if (rc != L4D_OK) return rc;
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_render_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                  float* depth, float* image, float* wsum, float* weights, float* zvals, void* saved,
                                  size_t saved_bytes, void* stream) {
  L4DFrameTable T;
  const bool ok = frame && rays;
  if (ok) T = one_frame(frame, rays->n_rays);
  return l4d_render_forward_frames(cfg, staged, ok ? &T : nullptr, rays, depth, image, wsum, weights, zvals, saved, saved_bytes, stream);
}

extern "C" int l4d_render_forward_frames(const L4DConfig* cfg, const void* staged, const L4DFrameTable* frames,
                                         const L4DRays* rays, float* depth, float* image, float* wsum, float* weights,
                                         float* zvals, void* saved, size_t saved_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  rc = check_rays(rays);
  if (rc != L4D_OK) return rc;
  if (!staged || !frames || !depth || !image || !wsum) return l4d_fail(L4D_EINVAL, "null pointer");
  rc = check_frames(frames, rays->n_rays);
  if (rc != L4D_OK) return rc;
  if (rays->n_rays == 0) return L4D_OK;
  if (saved && saved_bytes < saved_layout(cfg, rays->n_rays, rays->n_steps, frames->n_frames).total)
    return l4d_fail(L4D_ESIZE, "saved buffer too small");
  const bool fused = (rays->reserved & L4D_FLAG_FUSED) || !saved;
  const bool mf = frames->n_frames > 1;
  cudaStream_t st = (cudaStream_t)stream;
  prof_mark(st, "begin");
  if (fused) {
    FwdArgs A;
    memset(&A, 0, sizeof(A));
    build_model(cfg, staged, A.M);
    A.FT = *frames;
    A.rays_o = rays->rays_o; A.rays_d = rays->rays_d;
    A.n_rays = rays->n_rays; A.S = rays->n_steps; A.perturb = rays->perturb;
    A.seed = rays->seed; A.ray_offset = rays->ray_offset;
    A.depth = depth; A.image = image; A.wsum = wsum; A.weights = weights; A.zvals = zvals;
    A.train = saved ? 1u : 0u;
    if (saved) A.sv = saved_view(cfg, saved, rays->n_rays, rays->n_steps);
    const size_t smem = (64 * L4D_NT + 80 + 128 + 32) * sizeof(float);
    int grid;
    auto kernel = mf ? k_render_fwd<L4D_NT, true> : k_render_fwd<L4D_NT, false>;
    rc = grid_for(kernel, L4D_NT, smem, rays->n_rays, grid);
    if (rc != L4D_OK) return rc;
    ++g_launches; kernel<<<grid, L4D_NT, smem, st>>>(A);
    prof_mark(st, "k_render_fwd");
    L4D_CUDA(cudaGetLastError());
    return L4D_OK;
  }
  SplitArgs A;
  fill_split(A, cfg, staged, frames, rays, saved);
  A.depth = depth; A.image = image; A.wsum = wsum; A.weights = weights; A.zvals = zvals;
  A.train = 1u;
  const size_t P = (size_t)rays->n_rays * rays->n_steps;
  // contraction of the time-dependent encoders with each frame's constants, into that frame's dynamic-hash tables
  // (DevModel::hd_con) and time-plane rows (DevModel::pl_con)
  point_contracted(cfg, saved, rays->n_rays, rays->n_steps, A.M);
  for (uint32_t f = 0; f < frames->n_frames; ++f) {
    const L4DFrame* frame = &frames->frames[f];
    const size_t off = f * A.con_fstride;
    {
      ContractArgs C;
      memset(&C, 0, sizeof(C));
      uint32_t nmax = 0;
      for (int p = 0; p < 3; ++p) {
        C.table[p] = reinterpret_cast<const uint4*>(A.M.hd[p]);
        C.entries[p] = A.M.hd_slice_entries[p];
        nmax = C.entries[p] > nmax ? C.entries[p] : nmax;
        for (int q = 0; q < 3; ++q) C.con[p][q] = const_cast<float*>(A.M.hd_con[p][q]) + off;
      }
      C.n_slices = cfg->time_resolution;
      C.n_queries_mask = 1u | (frame->has_fwd ? 2u : 0u) | (frame->has_bwd ? 4u : 0u);
      C.q[0] = frame->cur; C.q[1] = frame->fwd; C.q[2] = frame->bwd;
      ++g_launches; k_contract_dynamic<<<dim3((unsigned)nblk(nmax), 3), 256, 0, st>>>(C);
    }
    {
      TimeRowArgs T;
      fill_time_rows(T, cfg, frame);
      uint32_t rmax = 0;
      for (uint32_t s2 = 0; s2 < cfg->n_plane_scales; ++s2) {
        rmax = cfg->plane_res[s2] > rmax ? cfg->plane_res[s2] : rmax;
        for (int t = 0; t < 3; ++t) {
          T.plane[s2][t] = const_cast<float*>(A.M.planes[s2][t == 0 ? 2 : (t == 1 ? 4 : 5)]);
          for (int q = 0; q < 3; ++q) T.row[s2][t][q] = const_cast<float*>(A.M.pl_con[s2][t][q]) + off;
        }
      }
      ++g_launches; k_contract_planes<<<dim3((unsigned)nblk((size_t)rmax * 8), 3 * cfg->n_plane_scales), 256, 0, st>>>(T);
    }
  }
  prof_mark(st, "k_contract");
  if (cfg->mlp_fp16) {
    {
      const size_t smem = tc_dyn_smem(flow_tc_smem().total_fwd);
      int grid;
      rc = grid_for(k_fwd_flow_tc, 128, smem, (uint32_t)((P + 127) / 128), grid);
      if (rc != L4D_OK) return rc;
      ++g_launches; k_fwd_flow_tc<<<grid, 128, smem, st>>>(A);
      prof_mark(st, "k_fwd_flow_tc");
    }
    const size_t smem = 16 * L4D_NT * sizeof(float);
    int grid;
    if (use_tc_dense(cfg)) {
      const uint32_t work = rays->n_rays * A.sv.n_tiles;       // whole 128-row tiles
      auto kernel = mf ? k_fwd_gather<L4D_NT, true, true, true> : k_fwd_gather<L4D_NT, true, true, false>;
      rc = grid_for(kernel, L4D_NT, smem, work, grid);
      if (rc != L4D_OK) return rc;
      ++g_launches; kernel<<<grid, L4D_NT, smem, st>>>(A);
    } else {
      auto kernel = mf ? k_fwd_gather<L4D_NT, true, false, true> : k_fwd_gather<L4D_NT, true, false, false>;
      rc = grid_for(kernel, L4D_NT, smem, (uint32_t)((P + L4D_NT - 1) / L4D_NT), grid);
      if (rc != L4D_OK) return rc;
      ++g_launches; kernel<<<grid, L4D_NT, smem, st>>>(A);
    }
    prof_mark(st, "k_fwd_gather");
  } else {
    const size_t smem = 64 * L4D_NT * sizeof(float);
    int grid;
    auto kernel = mf ? k_fwd_gather<L4D_NT, false, false, true> : k_fwd_gather<L4D_NT, false, false, false>;
    rc = grid_for(kernel, L4D_NT, smem, (uint32_t)((P + L4D_NT - 1) / L4D_NT), grid);
    if (rc != L4D_OK) return rc;
    ++g_launches; kernel<<<grid, L4D_NT, smem, st>>>(A);
    prof_mark(st, "k_fwd_gather");
  }
  if (use_tc_dense(cfg)) {
    const size_t smem = tc_dyn_smem(dense_fwd_smem(cfg->sigma_in_pad).total);
    int grid;
    rc = grid_for(k_fwd_dense_tc, 256, smem, rays->n_rays, grid);
    if (rc != L4D_OK) return rc;
    ++g_launches; k_fwd_dense_tc<<<grid, 256, smem, st>>>(A);
    prof_mark(st, "k_fwd_dense_tc");
  } else {
    const size_t smem = (64 * L4D_NT + 80 + 128 + 32) * sizeof(float);
    int grid;
    rc = grid_for(k_fwd_dense<L4D_NT>, L4D_NT, smem, rays->n_rays, grid);
    if (rc != L4D_OK) return rc;
    ++g_launches; k_fwd_dense<L4D_NT><<<grid, L4D_NT, smem, st>>>(A);
    prof_mark(st, "k_fwd_dense");
  }
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_render_backward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                      const void* saved, size_t saved_bytes, const float* g_depth, const float* g_image,
                                      const float* g_wsum, const float* g_weights, const L4DMasterGrads* grads,
                                      void* grad_work, size_t grad_work_bytes, void* ev_hash_done, void* stream);
extern "C" int l4d_render_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                   const void* saved, size_t saved_bytes, const float* g_depth, const float* g_image,
                                   const float* g_wsum, const float* g_weights, const L4DMasterGrads* grads,
                                   void* grad_work, size_t grad_work_bytes, void* stream) {
  return l4d_render_backward_ex(cfg, staged, frame, rays, saved, saved_bytes, g_depth, g_image, g_wsum, g_weights, grads, grad_work,
                                grad_work_bytes, nullptr, stream);
}
extern "C" int l4d_render_backward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                      const void* saved, size_t saved_bytes, const float* g_depth, const float* g_image,
                                      const float* g_wsum, const float* g_weights, const L4DMasterGrads* grads,
                                      void* grad_work, size_t grad_work_bytes, void* ev_hash_done, void* stream) {
  L4DFrameTable T;
  const bool ok = frame && rays;
  if (ok) T = one_frame(frame, rays->n_rays);
  return l4d_render_backward_frames(cfg, staged, ok ? &T : nullptr, rays, saved, saved_bytes, g_depth, g_image, g_wsum, g_weights, grads,
                                    grad_work, grad_work_bytes, ev_hash_done, stream);
}

extern "C" int l4d_render_backward_frames(const L4DConfig* cfg, const void* staged, const L4DFrameTable* frames,
                                          const L4DRays* rays, const void* saved, size_t saved_bytes, const float* g_depth,
                                          const float* g_image, const float* g_wsum, const float* g_weights,
                                          const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes,
                                          void* ev_hash_done, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  rc = check_rays(rays);
  if (rc != L4D_OK) return rc;
  if (!staged || !frames || !saved || !g_depth || !g_image || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  rc = check_frames(frames, rays->n_rays);
  if (rc != L4D_OK) return rc;
  const bool fused = (rays->reserved & L4D_FLAG_FUSED) != 0;
  const bool mf = frames->n_frames > 1;
  if (saved_bytes < saved_layout(cfg, rays->n_rays, rays->n_steps, frames->n_frames).total)
    return l4d_fail(L4D_ESIZE, "saved buffer too small");
  // the single kernel accumulates straight into the slices: only the split pipeline has per-frame accumulators
  if (grad_work_bytes < grad_work_layout(cfg, fused ? 1u : frames->n_frames).total)
    return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  if (!grads->hash_static || !grads->flow_grid) return l4d_fail(L4D_EINVAL, "null hash gradient buffer");
  for (int p = 0; p < 3; ++p)
    for (uint32_t s = 0; s < cfg->time_resolution; ++s)
      if (!grads->hash_dynamic[p][s]) return l4d_fail(L4D_EINVAL, "null hash_dynamic gradient buffer");
  if (rays->n_rays == 0) return L4D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  prof_mark(st, "begin");
  if (!fused) {
    SplitArgs A;
    fill_split(A, cfg, staged, frames, rays, const_cast<void*>(saved));
    build_grads(cfg, grads, grad_work, A.G, true);
    point_contracted(cfg, const_cast<void*>(saved), rays->n_rays, rays->n_steps, A.M);   // what the forward left in `saved`
    A.g_depth = g_depth; A.g_image = g_image; A.g_wsum = g_wsum; A.g_weights = g_weights;
    A.train = 1u;
    const size_t P = (size_t)rays->n_rays * rays->n_steps;
    const uint32_t tiles = (uint32_t)((P + L4D_NT - 1) / L4D_NT);
    if (use_tc_dense(cfg)) {
      rc = launch_bwd_composite(A, st);
      if (rc != L4D_OK) return rc;
      const size_t smem = tc_dyn_smem(dense_bwd_smem(cfg->sigma_in_pad).total);
      int grid;
      rc = grid_for(k_bwd_dense_tc, 256, smem, rays->n_rays, grid);
      if (rc != L4D_OK) return rc;
      ++g_launches; k_bwd_dense_tc<<<grid, 256, smem, st>>>(A);
      prof_mark(st, "k_bwd_dense_tc");
    } else {
      const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD + 80 + 128 + 128 + 32 + L4D_MAX_TILES) * sizeof(float);
      int grid;
      rc = grid_for(k_bwd_dense<L4D_NT>, L4D_NT, smem, rays->n_rays, grid);
      if (rc != L4D_OK) return rc;
      if (grid > L4D_BWD_SCRATCH_CTAS) grid = L4D_BWD_SCRATCH_CTAS;
      ++g_launches; k_bwd_dense<L4D_NT><<<grid, L4D_NT, smem, st>>>(A);
      prof_mark(st, "k_bwd_dense");
    }
    {
      int grid;
      auto scatter = mf ? k_bwd_encoders<L4D_NT, true> : k_bwd_encoders<L4D_NT, false>;
      rc = grid_for(scatter, L4D_NT, 0, tiles * (1u + cfg->hash_static.n_levels), grid);
      if (rc != L4D_OK) return rc;
      // the static-hash CTAs: L4D_SCATTER_STATIC_PER_SM of every L4D_SCATTER_MIN_CTAS, the first ones dispatched
      const uint32_t n_static = ((uint32_t)grid * L4D_SCATTER_STATIC_PER_SM + L4D_SCATTER_MIN_CTAS - 1) / L4D_SCATTER_MIN_CTAS;
      A.scatter_tickets = reinterpret_cast<uint32_t*>(static_cast<char*>(grad_work) + grad_work_layout(cfg).scatter_tickets);
      ++g_launches; scatter<<<grid, L4D_NT, 0, st>>>(A, n_static);
      prof_mark(st, "k_bwd_encoders");
      for (uint32_t f = 0; f < frames->n_frames; ++f) {       // gradient rows -> the two live time rows of every time plane
        TimeRowArgs T;
        fill_time_rows(T, cfg, &frames->frames[f]);
        uint32_t rmax = 0;
        for (uint32_t s2 = 0; s2 < cfg->n_plane_scales; ++s2) {
          rmax = cfg->plane_res[s2] > rmax ? cfg->plane_res[s2] : rmax;
          for (int t = 0; t < 3; ++t) {
            T.plane[s2][t] = A.G.planes_cl[s2][t == 0 ? 2 : (t == 1 ? 4 : 5)];
            for (int q = 0; q < 3; ++q) T.row[s2][t][q] = A.G.pl_rows[s2][t][q] + f * A.comb_fstride;
          }
        }
        ++g_launches; k_fold_planes<<<dim3((unsigned)nblk((size_t)rmax * 8), 3 * cfg->n_plane_scales), 256, 0, st>>>(T);
      }
      prof_mark(st, "k_fold_planes");
      for (uint32_t f = 0; f < frames->n_frames; ++f) {
        const L4DFrame* frame = &frames->frames[f];
        for (int p = 0; p < 3; ++p) {
          const size_t n = cfg->hash_dynamic[p].offset[cfg->hash_dynamic[p].n_levels];
          const bool single = frame->cur.single != 0;
          const float* tb = frame->cur.basis;
          ++g_launches; k_fold_dynamic<<<nblk(n), 256, 0, st>>>(A.G.hd_comb[p] + f * A.comb_fstride,
                                                 reinterpret_cast<float4*>(A.G.hd[p][frame->cur.slice_lo]),
                                                 single ? nullptr : reinterpret_cast<float4*>(A.G.hd[p][frame->cur.slice_hi]), n,
                                                 single ? 1.0f : frame->cur.w_lo, frame->cur.w_hi, tb[0], tb[1], tb[2], tb[3]);
        }
      }
      prof_mark(st, "k_fold_dynamic");
      // hash_static and hash_dynamic gradients are final from here on (the flow backward below only touches the flow net)
      if (ev_hash_done) L4D_CUDA(cudaEventRecord((cudaEvent_t)ev_hash_done, st));
    }
    bool any_neighbour = false;
    for (uint32_t f = 0; f < frames->n_frames; ++f) any_neighbour |= frames->frames[f].has_fwd || frames->frames[f].has_bwd;
    if (any_neighbour) {     // with no neighbour frame nothing reaches the flow field (samples of such frames give dL/dflow = 0)
      if (cfg->mlp_fp16) {
        const size_t smem = tc_dyn_smem(flow_tc_smem().total);
        int grid;
        rc = grid_for(k_bwd_flow_tc, 128, smem, tiles, grid);
        if (rc != L4D_OK) return rc;
        ++g_launches; k_bwd_flow_tc<<<grid, 128, smem, st>>>(A);
        prof_mark(st, "k_bwd_flow_tc");
        auto flowgrid = mf ? k_bwd_flowgrid<L4D_NT, true> : k_bwd_flowgrid<L4D_NT, false>;
        rc = grid_for(flowgrid, L4D_NT, 0, tiles, grid);
        if (rc != L4D_OK) return rc;
        ++g_launches; flowgrid<<<grid, L4D_NT, 0, st>>>(A);
        const size_t n = cfg->flow.offset[cfg->flow.n_levels];
        for (uint32_t f = 0; f < frames->n_frames; ++f) {
          const L4DFrame* frame = &frames->frames[f];
          if (!frame->has_fwd && !frame->has_bwd) continue;       // its accumulator received zeros only
          const float* fb = frame->flow_basis;
          ++g_launches; k_fold_flow<<<nblk(n), 256, 0, st>>>(reinterpret_cast<float2*>(A.G.hf_comb + f * A.comb_fstride),
                                                             reinterpret_cast<float4*>(A.G.hf), n, fb[0], fb[1], fb[2], fb[3]);
        }
        prof_mark(st, "k_bwd_flowgrid");
      } else {
        const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD) * sizeof(float);
        int grid;
        rc = grid_for(k_bwd_flow<L4D_NT>, L4D_NT, smem, tiles, grid);
        if (rc != L4D_OK) return rc;
        ++g_launches; k_bwd_flow<L4D_NT><<<grid, L4D_NT, smem, st>>>(A);
        prof_mark(st, "k_bwd_flow");
      }
    }
    L4D_CUDA(cudaGetLastError());
    return L4D_OK;
  }
  BwdArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  build_grads(cfg, grads, grad_work, A.G);
  A.FT = *frames;
  A.rays_o = rays->rays_o; A.rays_d = rays->rays_d;
  A.n_rays = rays->n_rays; A.S = rays->n_steps; A.perturb = rays->perturb;
  A.seed = rays->seed; A.ray_offset = rays->ray_offset;
  A.g_depth = g_depth; A.g_image = g_image; A.g_wsum = g_wsum; A.g_weights = g_weights;
  A.sv = saved_view(cfg, const_cast<void*>(saved), rays->n_rays, rays->n_steps);
  const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD + 80 + 128 + 128 + 32 + L4D_MAX_TILES) * sizeof(float);
  int grid;
  rc = grid_for(k_render_bwd<L4D_NT>, L4D_NT, smem, rays->n_rays, grid);
  if (rc != L4D_OK) return rc;
  if (grid > L4D_BWD_SCRATCH_CTAS) grid = L4D_BWD_SCRATCH_CTAS;
  ++g_launches; k_render_bwd<L4D_NT><<<grid, L4D_NT, smem, st>>>(A);
  prof_mark(st, "k_render_bwd");
  if (ev_hash_done) L4D_CUDA(cudaEventRecord((cudaEvent_t)ev_hash_done, st));
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x,
                                uint32_t n, float* flow, float* flow_saved, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !frame || !x || !flow) return l4d_fail(L4D_EINVAL, "null pointer");
  if (n == 0) return L4D_OK;
  FlowArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.F = *frame; A.x = x; A.n = n; A.flow = flow; A.saved = flow_saved;
  const size_t smem = 64 * L4D_NT * sizeof(float);
  int grid;
  rc = grid_for(k_flow_fwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_flow_fwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x,
                                 uint32_t n, const float* flow_saved, const float* g_flow, const L4DMasterGrads* grads,
                                 void* grad_work, size_t grad_work_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !frame || !x || !flow_saved || !g_flow || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  if (grad_work_bytes < grad_work_layout(cfg).total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  if (!grads->flow_grid) return l4d_fail(L4D_EINVAL, "null flow_grid gradient buffer");
  if (n == 0) return L4D_OK;
  FlowArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  {
    // only the flow sinks are touched; hash_static/dynamic may be null here
    GradWorkLayout L = grad_work_layout(cfg);
    char* b = reinterpret_cast<char*>(grad_work);
    A.G.hf = grads->flow_grid;
    A.G.flo_w0t = reinterpret_cast<float*>(b + L.flo_w0t);
    A.G.flo_w1t = reinterpret_cast<float*>(b + L.flo_w1t);
    A.G.flo_w2 = reinterpret_cast<float*>(b + L.flo_w2);
  }
  A.F = *frame; A.x = x; A.n = n; A.saved = const_cast<float*>(flow_saved); A.g_flow = g_flow;
  const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD) * sizeof(float);
  int grid;
  rc = grid_for(k_flow_bwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_flow_bwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_hash_indices(const L4DConfig* cfg, uint32_t grid_id, uint32_t level, const float* x, uint32_t n,
                                uint32_t* idx, float* w, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (grid_id > 4 || !x || !idx || !w) return l4d_fail(L4D_EINVAL, "bad argument");
  const L4DGrid& g = grid_id == 0 ? cfg->hash_static : (grid_id == 4 ? cfg->flow : cfg->hash_dynamic[grid_id - 1]);
  if (level >= g.n_levels) return l4d_fail(L4D_EINVAL, "level out of range");
  if (n == 0) return L4D_OK;
  DevGrid d;
  fill_grid(d, g);
  ++g_launches; k_hash_indices<<<nblk(n), 256, 0, (cudaStream_t)stream>>>(d, (int)g.n_dims, (int)level, x, n, idx, w);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_density_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x,
                                   uint32_t n, float* sigma, float* geo, float* features, float* flow, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !frame || !x || !sigma || !geo) return l4d_fail(L4D_EINVAL, "null pointer");
  if (n == 0) return L4D_OK;
  DensityArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.F = *frame; A.x = x; A.n = n; A.sigma = sigma; A.geo = geo; A.features = features; A.flow = flow;
  const size_t smem = 64 * L4D_NT * sizeof(float);
  L4D_CUDA(cudaFuncSetAttribute(k_density<L4D_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ++g_launches; k_density<L4D_NT><<<nblk(n, L4D_NT), L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_attribute_forward(const L4DConfig* cfg, const void* staged, const float* d, const float* geo,
                                     const unsigned char* mask, uint32_t n, float* out, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !d || !geo || !out) return l4d_fail(L4D_EINVAL, "null pointer");
  if (n == 0) return L4D_OK;
  AttributeArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.d = d; A.geo = geo; A.mask = mask; A.n = n; A.out = out;
  constexpr int NT = 64;
  const size_t smem = (size_t)(64 + 81 + 129) * NT * sizeof(float);
  L4D_CUDA(cudaFuncSetAttribute(k_attribute<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ++g_launches; k_attribute<NT><<<nblk(n, NT), NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// ---- LiDAR4D.density / .attribute on explicit points with a backward (l4d_points.cuh) ----------------------------
extern "C" size_t l4d_density_saved_bytes(const L4DConfig* cfg, uint32_t n) {
  if (check_config(cfg) != L4D_OK) return 0;
  return density_saved_layout(cfg, n).total;
}

extern "C" int l4d_density_forward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x,
                                      uint32_t n, float* sigma, float* geo, float* features, float* flow, void* saved,
                                      size_t saved_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !frame || !x || !sigma || !geo) return l4d_fail(L4D_EINVAL, "null pointer");
  if (!saved) return l4d_density_forward(cfg, staged, frame, x, n, sigma, geo, features, flow, stream);
  const DensitySavedLayout L = density_saved_layout(cfg, n);
  if (saved_bytes < L.total) return l4d_fail(L4D_ESIZE, "saved buffer too small");
  if (n == 0) return L4D_OK;
  DensityTrainArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.F = *frame; A.x = x; A.n = n; A.sigma = sigma; A.geo = geo; A.features = features; A.flow = flow;
  char* b = reinterpret_cast<char*>(saved);
  A.flow_in = reinterpret_cast<float*>(b + L.flow_in);
  A.feat = reinterpret_cast<float*>(b + L.feat);
  const size_t smem = 64 * L4D_NT * sizeof(float);
  L4D_CUDA(cudaFuncSetAttribute(k_density_train<L4D_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ++g_launches; k_density_train<L4D_NT><<<nblk(n, L4D_NT), L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// every gradient sink the point backwards write must be present: l4d_unstage_grads only clears the grad_work regions it
// folds into a non-null master, and grad_work has to be all zero again after it
static int check_point_grads(const L4DConfig* cfg, const L4DMasterGrads* g, bool density) {
  if (!g->intensity_net && !density) return l4d_fail(L4D_EINVAL, "null intensity_net gradient buffer");
  if (!g->raydrop_net && !density) return l4d_fail(L4D_EINVAL, "null raydrop_net gradient buffer");
  if (!density) return L4D_OK;
  if (!g->hash_static || !g->flow_grid || !g->sigma_net) return l4d_fail(L4D_EINVAL, "null gradient buffer");
  for (int k = 0; k < 3; ++k)
    if (!g->flow_mlp[k]) return l4d_fail(L4D_EINVAL, "null flow_mlp gradient buffer");
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci)
      if (!g->planes[s][ci]) return l4d_fail(L4D_EINVAL, "null plane gradient buffer");
  for (int p = 0; p < 3; ++p)
    for (uint32_t s = 0; s < cfg->time_resolution; ++s)
      if (!g->hash_dynamic[p][s]) return l4d_fail(L4D_EINVAL, "null hash_dynamic gradient buffer");
  return L4D_OK;
}

extern "C" int l4d_density_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x,
                                    uint32_t n, const void* saved, size_t saved_bytes, const float* g_sigma,
                                    const float* g_geo, const L4DMasterGrads* grads, void* grad_work,
                                    size_t grad_work_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !frame || !x || !saved || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  const DensitySavedLayout L = density_saved_layout(cfg, n);
  if (saved_bytes < L.total) return l4d_fail(L4D_ESIZE, "saved buffer too small");
  if (grad_work_bytes < grad_work_layout(cfg).total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  rc = check_point_grads(cfg, grads, true);
  if (rc != L4D_OK) return rc;
  if (n == 0 || (!g_sigma && !g_geo)) return L4D_OK;
  DensityBwdArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  build_grads(cfg, grads, grad_work, A.G);
  A.F = *frame; A.x = x; A.n = n; A.g_sigma = g_sigma; A.g_geo = g_geo;
  const char* b = reinterpret_cast<const char*>(saved);
  A.flow_in = reinterpret_cast<const float*>(b + L.flow_in);
  A.feat = reinterpret_cast<const float*>(b + L.feat);
  A.hidden = const_cast<float*>(reinterpret_cast<const float*>(b + L.hidden));
  const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD) * sizeof(float);
  int grid;
  rc = grid_for(k_density_bwd<L4D_NT>, L4D_NT, smem, L.ctas, grid);
  if (rc != L4D_OK) return rc;
  if (grid > (int)L.ctas) grid = (int)L.ctas;          // one hidden-scratch block per CTA
  ++g_launches; k_density_bwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_attribute_backward(const L4DConfig* cfg, const void* staged, const float* d, const float* geo,
                                      const unsigned char* mask, uint32_t n, const float* g_out, float* g_geo,
                                      const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes, void* stream) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !d || !geo || !g_out || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  if (grad_work_bytes < grad_work_layout(cfg).total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  rc = check_point_grads(cfg, grads, false);
  if (rc != L4D_OK) return rc;
  if (n == 0) return L4D_OK;
  AttributeBwdArgs A;
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  {
    // only the attribute-head sinks are touched; the other master gradients may be null here
    GradWorkLayout GL = grad_work_layout(cfg);
    char* b = reinterpret_cast<char*>(grad_work);
    for (int k = 0; k < 2; ++k) {
      A.G.att_w1t[k] = reinterpret_cast<float*>(b + GL.att_w1t[k]);
      A.G.att_w2t[k] = reinterpret_cast<float*>(b + GL.att_w2t[k]);
      A.G.att_w3[k] = reinterpret_cast<float*>(b + GL.att_w3[k]);
    }
  }
  A.d = d; A.geo = geo; A.mask = mask; A.n = n; A.g_out = g_out; A.g_geo = g_geo;
  const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD + L4D_ENC * L4D_NT) * sizeof(float);
  int grid;
  rc = grid_for(k_attribute_bwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_attribute_bwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// ---- LiDAR4D's submodules on their own (l4d_modules.cuh) -----------------------------------------------------------
static bool misaligned4(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 3u); }

// input / output widths of an encoder module; false for an unknown id
static bool module_dims(const L4DConfig* cfg, uint32_t module, uint32_t& in, uint32_t& out) {
  const uint32_t L = cfg->hash_static.n_levels;
  switch (module) {
    case L4D_MOD_HASH_STATIC: in = 3; out = 4 * L; return true;
    case L4D_MOD_HASH_T0: case L4D_MOD_HASH_T0 + 1: case L4D_MOD_HASH_T0 + 2: in = 2; out = L; return true;
    case L4D_MOD_HASH_DYNAMIC: in = 3; out = 3 * L; return true;
    case L4D_MOD_HASH_SLICE0: case L4D_MOD_HASH_SLICE0 + 1: case L4D_MOD_HASH_SLICE0 + 2: in = 2; out = 4 * L; return true;
    case L4D_MOD_PLANES_STATIC: case L4D_MOD_PLANES_DYNAMIC: in = 4; out = 8 * cfg->n_plane_scales; return true;
    case L4D_MOD_FLOW_GRID: in = 3; out = 8 * cfg->flow.n_levels; return true;
    case L4D_MOD_FLOW: in = 4; out = 6; return true;
    case L4D_MOD_FREQ: in = 3; out = L4D_ENC; return true;
  }
  return false;
}

static int module_check(const L4DConfig* cfg, const void* staged, uint32_t module, const L4DTimeQuery* q, uint32_t slice,
                        const float* x, uint32_t n, ModuleArgs& A) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !x) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(x)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  if (n > (1u << 31)) return l4d_fail(L4D_EINVAL, "n > 2^31");
  memset(&A, 0, sizeof(A));
  if (!module_dims(cfg, module, A.in_dim, A.out_dim)) return l4d_fail(L4D_EINVAL, "unknown module id");
  const bool timed = (module >= L4D_MOD_HASH_T0 && module <= L4D_MOD_HASH_T0 + 2) || module == L4D_MOD_HASH_DYNAMIC;
  if (timed) {
    if (!q) return l4d_fail(L4D_EINVAL, "null time query");
    if (q->slice_lo >= cfg->time_resolution || q->slice_hi >= cfg->time_resolution)
      return l4d_fail(L4D_EINVAL, "time query slice out of range");
    A.q = *q;
  }
  if (module >= L4D_MOD_HASH_SLICE0 && module <= L4D_MOD_HASH_SLICE0 + 2 && slice >= cfg->time_resolution)
    return l4d_fail(L4D_EINVAL, "slice out of range");
  build_model(cfg, staged, A.M);
  A.module = module; A.slice = slice; A.x = x; A.n = n;
  return L4D_OK;
}

extern "C" int l4d_encoder_forward(const L4DConfig* cfg, const void* staged, uint32_t module, const L4DTimeQuery* q,
                                   uint32_t slice, const float* x, uint32_t n, float* out, void* stream) {
  ModuleArgs A;
  int rc = module_check(cfg, staged, module, q, slice, x, n, A);
  if (rc != L4D_OK) return rc;
  if (!out) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(out)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  if (n == 0) return L4D_OK;
  A.out = out;
  const size_t smem = 64 * L4D_NT * sizeof(float);
  int grid;
  rc = grid_for(k_module_fwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_module_fwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_encoder_backward(const L4DConfig* cfg, const void* staged, uint32_t module, const L4DTimeQuery* q,
                                    uint32_t slice, const float* x, uint32_t n, const float* g_out, float* g_x,
                                    const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes, void* stream) {
  ModuleArgs A;
  int rc = module_check(cfg, staged, module, q, slice, x, n, A);
  if (rc != L4D_OK) return rc;
  if (module == L4D_MOD_FREQ) return l4d_fail(L4D_EINVAL, "the frequency encoding has no parameters");
  if (!g_out || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(g_out) || misaligned4(g_x) || misaligned4(grad_work)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  const bool planes = module == L4D_MOD_PLANES_STATIC || module == L4D_MOD_PLANES_DYNAMIC;
  if (g_x && !planes) return l4d_fail(L4D_EINVAL, "only the planes give an input gradient");
  if (grad_work_bytes < grad_work_layout(cfg).total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  // the module's gradient buffers
  switch (module) {
    case L4D_MOD_HASH_STATIC:
      if (!grads->hash_static) return l4d_fail(L4D_EINVAL, "null hash_static gradient buffer");
      break;
    case L4D_MOD_FLOW_GRID:
    case L4D_MOD_FLOW:
      if (!grads->flow_grid) return l4d_fail(L4D_EINVAL, "null flow_grid gradient buffer");
      if (module == L4D_MOD_FLOW)
        for (int k = 0; k < 3; ++k)
          if (!grads->flow_mlp[k]) return l4d_fail(L4D_EINVAL, "null flow_mlp gradient buffer");
      break;
    case L4D_MOD_PLANES_STATIC: case L4D_MOD_PLANES_DYNAMIC:
      for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
        for (int ci = 0; ci < 6; ++ci)
          if (!grads->planes[s][ci]) return l4d_fail(L4D_EINVAL, "null plane gradient buffer");
      break;
    default: {       // dynamic hash: the slices the call reaches
      const bool all = module == L4D_MOD_HASH_DYNAMIC;
      for (uint32_t p = 0; p < 3; ++p) {
        const bool used = all || module == L4D_MOD_HASH_T0 + p || module == L4D_MOD_HASH_SLICE0 + p;
        if (!used) continue;
        const bool slice_mod = module >= L4D_MOD_HASH_SLICE0;
        if (!grads->hash_dynamic[p][slice_mod ? slice : A.q.slice_lo] || (!slice_mod && !grads->hash_dynamic[p][A.q.slice_hi]))
          return l4d_fail(L4D_EINVAL, "null hash_dynamic gradient buffer");
      }
    }
  }
  if (n == 0) return L4D_OK;
  build_grads(cfg, grads, grad_work, A.G);
  A.g_out = g_out; A.g_x = g_x;
  const bool flow = module == L4D_MOD_FLOW;
  const size_t smem = flow ? (80 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD) * sizeof(float) : 0;
  int grid;
  rc = grid_for(k_module_bwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_module_bwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

static int mlp_check(const L4DConfig* cfg, const void* staged, uint32_t net, const float* in, uint32_t n, MlpArgs& A) {
  int rc = check_config(cfg);
  if (rc != L4D_OK) return rc;
  if (!staged || !in) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(in)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  if (n > (1u << 31)) return l4d_fail(L4D_EINVAL, "n > 2^31");
  if (net > L4D_NET_INTENSITY) return l4d_fail(L4D_EINVAL, "unknown net id");
  memset(&A, 0, sizeof(A));
  build_model(cfg, staged, A.M);
  A.net = net; A.in = in; A.n = n;
  A.n_in = net == L4D_NET_SIGMA ? cfg->sigma_in_dim : cfg->attr_in_dim;
  A.n_out = net == L4D_NET_SIGMA ? 16 : 1;
  return L4D_OK;
}

extern "C" int l4d_mlp_forward(const L4DConfig* cfg, const void* staged, uint32_t net, const float* in, uint32_t n,
                               float* out, void* stream) {
  MlpArgs A;
  int rc = mlp_check(cfg, staged, net, in, n, A);
  if (rc != L4D_OK) return rc;
  if (!out) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(out)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  if (n == 0) return L4D_OK;
  A.out = out;
  const size_t smem = 64 * L4D_NT * sizeof(float);
  int grid;
  rc = grid_for(k_mlp_fwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_mlp_fwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_mlp_backward(const L4DConfig* cfg, const void* staged, uint32_t net, const float* in, uint32_t n,
                                const float* g_out, float* g_in, const L4DMasterGrads* grads, void* grad_work,
                                size_t grad_work_bytes, void* stream) {
  MlpArgs A;
  int rc = mlp_check(cfg, staged, net, in, n, A);
  if (rc != L4D_OK) return rc;
  if (!g_out || !grads || !grad_work) return l4d_fail(L4D_EINVAL, "null pointer");
  if (misaligned4(g_out) || misaligned4(g_in) || misaligned4(grad_work)) return l4d_fail(L4D_EINVAL, "misaligned pointer");
  if (grad_work_bytes < grad_work_layout(cfg).total) return l4d_fail(L4D_ESIZE, "grad_work buffer too small");
  const float* master = net == L4D_NET_SIGMA ? grads->sigma_net : (net == L4D_NET_RAYDROP ? grads->raydrop_net : grads->intensity_net);
  if (!master) return l4d_fail(L4D_EINVAL, "null network gradient buffer");
  if (n == 0) return L4D_OK;
  build_grads(cfg, grads, grad_work, A.G);
  A.g_out = g_out; A.g_in = g_in;
  const size_t smem = (64 * L4D_NT + 2 * L4D_NT * L4D_TILE_LD) * sizeof(float);
  int grid;
  rc = grid_for(k_mlp_bwd<L4D_NT>, L4D_NT, smem, (n + L4D_NT - 1) / L4D_NT, grid);
  if (rc != L4D_OK) return rc;
  ++g_launches; k_mlp_bwd<L4D_NT><<<grid, L4D_NT, smem, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// wgmma self-test: C[128][N] = A[128][K] (fp16) * B[N][K]^T (fp16), fp32 accumulate
extern "C" int l4d_tc_selftest(const void* A, const void* B, float* Cout, uint32_t N, uint32_t K, void* stream) {
  if (!A || !B || !Cout) return l4d_fail(L4D_EINVAL, "null pointer");
  if (N < 16 || N > 256 || N % 16 || K < 16 || K % 16 || K > 512) return l4d_fail(L4D_EINVAL, "need N%16==0 in [16,256], K%16==0 in [16,512]");
  const size_t smem = (size_t)(K / 8) * (128 + N) * 16 + 1024;
  L4D_CUDA(cudaFuncSetAttribute(k_tc_selftest, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ++g_launches; k_tc_selftest<<<1, 128, smem, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(A), reinterpret_cast<const __half*>(B),
                                                        Cout, (int)N, (int)K);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// wgmma self-test 2: operands pre-arranged in tile format; M in {64,128}; either operand may be MN-major
extern "C" int l4d_tc_selftest2(const void* A, const void* B, float* Cout, uint32_t M, uint32_t N, uint32_t K,
                                uint32_t a_mn, uint32_t b_mn, void* stream) {
  if (!A || !B || !Cout) return l4d_fail(L4D_EINVAL, "null pointer");
  if ((M != 64 && M != 128) || N < 8 || N > 256 || N % 8 || (M == 128 && N % 16) || K < 16 || K % 16 || K > 256)
    return l4d_fail(L4D_EINVAL, "need M in {64,128}, N%8==0 (N%16 for M=128) <= 256, K%16==0 <= 256");
  const size_t smem = (size_t)(((M * K * 2 + 1023) & ~1023u) + N * K * 2 + 2048);
  L4D_CUDA(cudaFuncSetAttribute(k_tc_selftest2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ++g_launches; k_tc_selftest2<<<1, 128, smem, (cudaStream_t)stream>>>(reinterpret_cast<const unsigned char*>(A),
                                                         reinterpret_cast<const unsigned char*>(B), Cout, (int)M, (int)N, (int)K,
                                                         (int)a_mn, (int)b_mn);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

#include "l4d_chamfer.cuh"
#include "l4d_rays.cuh"
#include "l4d_convert.cuh"
#include "l4d_ground.cuh"

#ifdef L4D_PHASE_CLOCKS
// debug build only: per-phase clock sums of k_bwd_dense_tc (thread 0 of every CTA), cleared on read
extern "C" int l4d_debug_phase_clocks(unsigned long long* out32) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out32, g_phase_clk, sizeof(unsigned long long) * 32);
  unsigned long long z[32] = {0};
  cudaMemcpyToSymbol(g_phase_clk, z, sizeof(z));
  return 0;
}
#endif


// =============================================================================
// SURVEY 8(f) #2: ray generation + ground-truth gather, and the main-loss epilogue (l4d_rays.cuh)
// =============================================================================
extern "C" int l4d_lidar_rays(const float* pose, float fov_up, float fov, uint32_t H, uint32_t W, const long long* inds, uint32_t n,
                              const float* image, uint32_t C, float* rays_o, float* rays_d, float* gt, void* stream) {
  if (!pose || !rays_o || !rays_d || H == 0 || W == 0) return l4d_fail(L4D_EINVAL, "l4d_lidar_rays: null pointer or empty image");
  if (gt && (!image || C == 0 || C > 8)) return l4d_fail(L4D_EINVAL, "l4d_lidar_rays: gt gather needs image and 1 <= C <= 8");
  if (n == 0) return L4D_OK;
  ++g_launches; k_lidar_rays<<<nblk(n), 256, 0, (cudaStream_t)stream>>>(pose, fov_up, fov, H, W, inds, n, image, C, rays_o, rays_d, gt);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// the main LiDAR loss (l4d_losses.cuh): one CTA for the criteria, then, with the chamfer term, l4d_chamfer_forward /
// _backward on the two clouds and one CTA that adds the chamfer mean and folds its gradient into d loss / d depth
static int main_loss_run(const float* depth, const float* image, const float* gt, const float* rays_d, uint32_t n,
                         const uint32_t* crit, const float* alpha, double smooth, float scale, float delta, uint32_t accumulate,
                         float* loss, float* g_depth, float* g_image, void* work, size_t work_bytes, void* stream,
                         const char* who) {
  if (!depth || !image || !gt || !loss || !g_depth || !g_image) return l4d_fail(L4D_EINVAL, "%s: null pointer", who);
  if (n == 0 || n > 0x7fffffffu) return l4d_fail(L4D_EINVAL, "%s: n must be in [1, 2^31)", who);
  for (int k = 0; k < L4D_MT_N; ++k)
    if (crit[k] > L4D_GRAD_COS) return l4d_fail(L4D_EINVAL, "%s: unknown criterion", who);
  if (rays_d && !(scale > 0.f && isfinite(scale))) return l4d_fail(L4D_EINVAL, "%s: the chamfer term needs scale > 0", who);
  const L4DMainLayout L = l4d_main_layout(n);
  if (rays_d && !work) return l4d_fail(L4D_EINVAL, "%s: null work buffer", who);
  if (rays_d && work_bytes < L.total) return l4d_fail(L4D_ESIZE, "%s: work buffer too small", who);
  const L4DMainArgs a = l4d_main_args(n, crit, alpha, smooth, scale, delta);
  cudaStream_t st = (cudaStream_t)stream;
  L4DMainPtrs P = {};
  char* w = static_cast<char*>(work);
  if (rays_d) {
    P.pred = (float*)(w + L.pred); P.gtc = (float*)(w + L.gtc); P.d1 = (float*)(w + L.d1); P.d2 = (float*)(w + L.d2);
    P.gdist = (float*)(w + L.gdist); P.gx1 = (float*)(w + L.gx1); P.gx2 = (float*)(w + L.gx2); P.crit_sum = (double*)(w + L.hdr);
  }
  ++g_launches;
  k_main_loss<<<1, L4D_MAIN_THREADS, 0, st>>>(depth, image, gt, rays_d, n, a, P, accumulate, loss, g_depth, g_image);
  L4D_CUDA(cudaGetLastError());
  if (!rays_d) return L4D_OK;
  int32_t* i1 = (int32_t*)(w + L.i1);
  int32_t* i2 = (int32_t*)(w + L.i2);
  if (int rc = l4d_chamfer_forward(P.pred, P.gtc, 1, n, n, P.d1, P.d2, i1, i2, w + L.keys, 2 * (size_t)n * 8, stream)) return rc;
  if (int rc = l4d_chamfer_backward(P.pred, P.gtc, 1, n, n, P.gdist, P.gdist + n, i1, i2, P.gx1, P.gx2, stream)) return rc;
  ++g_launches;
  k_main_finish<<<1, L4D_MAIN_THREADS, 0, st>>>(gt, rays_d, n, a, P, accumulate, loss, g_depth);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_lidar_loss(const float* depth, const float* image, const float* gt, uint32_t n, float alpha_d, float alpha_r,
                              float alpha_i, float smooth, float* loss, float* g_depth, float* g_image, void* stream) {
  if (n == 0 && depth && image && gt && loss && g_depth && g_image) return L4D_OK;
  const uint32_t crit[L4D_MT_N] = {L4D_GRAD_L1, L4D_GRAD_MSE, L4D_GRAD_MSE};
  const float alpha[L4D_MT_N] = {alpha_d, alpha_r, alpha_i};
  return main_loss_run(depth, image, gt, nullptr, n, crit, alpha, smooth, 0.f, 0.f, 1, loss, g_depth, g_image, nullptr, 0,
                       stream, "l4d_lidar_loss");
}

extern "C" size_t l4d_main_loss_work_bytes(uint32_t n) { return l4d_main_layout(n).total; }

extern "C" int l4d_main_loss(const float* depth, const float* image, const float* gt, const float* rays_d, uint32_t n,
                             uint32_t crit_d, uint32_t crit_r, uint32_t crit_i, float alpha_d, float alpha_r, float alpha_i,
                             double smooth, float scale, float delta, float* loss, float* g_depth, float* g_image, void* work,
                             size_t work_bytes, void* stream) {
  const uint32_t crit[L4D_MT_N] = {crit_d, crit_r, crit_i};
  const float alpha[L4D_MT_N] = {alpha_d, alpha_r, alpha_i};
  return main_loss_run(depth, image, gt, rays_d, n, crit, alpha, smooth, scale, delta, 0, loss, g_depth, g_image, work,
                       work_bytes, stream, "l4d_main_loss");
}

extern "C" int l4d_main_loss_backward(const float* g_saved_depth, const float* g_saved_image, uint32_t n, const float* g_loss,
                                      float* g_depth, float* g_image, void* stream) {
  if (!g_saved_depth || !g_saved_image || !g_loss || !g_depth || !g_image)
    return l4d_fail(L4D_EINVAL, "l4d_main_loss_backward: null pointer");
  if (n == 0 || n > 0x7fffffffu) return l4d_fail(L4D_EINVAL, "l4d_main_loss_backward: n must be in [1, 2^31)");
  int grid = nblk(3 * (size_t)n);
  if (grid > 4 * sm_count()) grid = 4 * sm_count();
  ++g_launches; k_main_scale<<<grid, 256, 0, (cudaStream_t)stream>>>(g_saved_depth, g_saved_image, g_loss, n, g_depth, g_image);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_main_eval_loss(const float* depth, const float* image, const float* gt, const void* raydrop, uint32_t raydrop_dtype,
                                  uint32_t B, uint32_t H, uint32_t W, uint32_t crit_d, uint32_t crit_r, uint32_t crit_i,
                                  float alpha_d, float alpha_r, float alpha_i, float delta, float* loss, void* stream) {
  if (!depth || !image || !gt || !loss) return l4d_fail(L4D_EINVAL, "l4d_main_eval_loss: null pointer");
  const unsigned long long n = (unsigned long long)B * H * W;
  if (n == 0 || n > 0x7fffffffull) return l4d_fail(L4D_EINVAL, "l4d_main_eval_loss: B*H*W must be in [1, 2^31)");
  if (crit_d > L4D_GRAD_COS || crit_r > L4D_GRAD_COS || crit_i > L4D_GRAD_COS)
    return l4d_fail(L4D_EINVAL, "l4d_main_eval_loss: unknown criterion");
  if (raydrop && raydrop_dtype > L4D_DTYPE_BF16) return l4d_fail(L4D_EINVAL, "l4d_main_eval_loss: unknown ray-drop dtype");
  const uint32_t crit[L4D_MT_N] = {crit_d, crit_r, crit_i};
  const float alpha[L4D_MT_N] = {alpha_d, alpha_r, alpha_i};
  const L4DMainArgs a = l4d_main_args((uint32_t)n, crit, alpha, 0.0, 0.f, delta);
  ++g_launches;
  k_main_eval<<<1, L4D_MAIN_THREADS, 0, (cudaStream_t)stream>>>(depth, image, gt, raydrop, raydrop_dtype, B, H, W, a, loss);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// the patch losses and the line-of-sight loss of train_step (l4d_losses.cuh)
// =============================================================================
extern "C" int l4d_patch_loss(const float* depth, const float* gt, uint32_t n, uint32_t px, uint32_t py, float scale, uint32_t crit,
                              uint32_t flags, float alpha_grad, float alpha_gn, float alpha_sp, float alpha_tv, float* loss,
                              float* g_depth, void* stream) {
  if (!depth || !gt || !loss || !g_depth) return l4d_fail(L4D_EINVAL, "l4d_patch_loss: null pointer");
  if (px == 0 || py == 0 || n % (px * py) != 0) return l4d_fail(L4D_EINVAL, "l4d_patch_loss: n is not a multiple of px*py");
  if (crit > L4D_GRAD_COS || (flags & ~31u)) return l4d_fail(L4D_EINVAL, "l4d_patch_loss: unknown criterion or flag");
  const L4DPatchArgs a = l4d_patch_args(n, px, py, scale, crit, flags, alpha_grad, alpha_gn, alpha_sp, alpha_tv);
  ++g_launches; k_patch_loss<<<1, L4D_PATCH_THREADS, 0, (cudaStream_t)stream>>>(depth, gt, n, a, loss, g_depth);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_patch_loss_backward(const float* g_saved, const float* g_loss, uint32_t n, float* g_depth, void* stream) {
  if (!g_saved || !g_loss || !g_depth) return l4d_fail(L4D_EINVAL, "l4d_patch_loss_backward: null pointer");
  if (n == 0) return L4D_OK;
  int grid = nblk(n);
  if (grid > 4 * sm_count()) grid = 4 * sm_count();
  ++g_launches; k_loss_scale<<<grid, 256, 0, (cudaStream_t)stream>>>(g_saved, g_loss, n, g_depth);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_los_work_bytes(void) { return sizeof(L4DLosWork); }

static int los_check(const float* w, const float* z, const float* gt, uint32_t n, uint32_t S, double eps, const char* who) {
  if (!w || !z || !gt) return l4d_fail(L4D_EINVAL, "%s: null pointer", who);
  if (n == 0 || S == 0 || (uint64_t)n * S >= (1ull << 32)) return l4d_fail(L4D_EINVAL, "%s: need 1 <= n, S and n*S < 2^32", who);
  if (!(eps > 0.0)) return l4d_fail(L4D_EINVAL, "%s: eps must be positive", who);
  return L4D_OK;
}

static int los_grid(uint32_t n, uint32_t S) {
  const size_t b = ((size_t)n * S + L4D_LOS_THREADS - 1) / L4D_LOS_THREADS;
  return (int)(b < L4D_LOS_BLOCKS ? b : L4D_LOS_BLOCKS);
}

extern "C" int l4d_los_loss(const float* w, const float* z, const float* gt, uint32_t n, uint32_t S, double eps, float* loss,
                            void* work, size_t work_bytes, void* stream) {
  if (int rc = los_check(w, z, gt, n, S, eps, "l4d_los_loss")) return rc;
  if (!loss || !work) return l4d_fail(L4D_EINVAL, "l4d_los_loss: null pointer");
  if (work_bytes < sizeof(L4DLosWork)) return l4d_fail(L4D_ESIZE, "l4d_los_loss: work buffer too small");
  const L4DLosArgs a = l4d_los_args(eps);
  const int grid = los_grid(n, S);
  cudaStream_t st = (cudaStream_t)stream;
  L4DLosWork* wk = (L4DLosWork*)work;
  ++g_launches; k_los_partial<<<grid, L4D_LOS_THREADS, 0, st>>>(w, z, gt, n, S, a, wk);
  L4D_CUDA(cudaGetLastError());
  ++g_launches; k_los_finalize<<<1, 1024, 0, st>>>(w, z, gt, n, S, (uint32_t)grid, a, wk, loss);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_los_loss_backward(const float* w, const float* z, const float* gt, uint32_t n, uint32_t S, double eps,
                                     const void* work, const float* g_loss, float* g_w, void* stream) {
  if (int rc = los_check(w, z, gt, n, S, eps, "l4d_los_loss_backward")) return rc;
  if (!work || !g_loss || !g_w) return l4d_fail(L4D_EINVAL, "l4d_los_loss_backward: null pointer");
  const L4DLosArgs a = l4d_los_args(eps);
  int grid = nblk((size_t)n * S);
  if (grid > 8 * sm_count()) grid = 8 * sm_count();
  ++g_launches; k_los_backward<<<grid, 256, 0, (cudaStream_t)stream>>>(w, z, gt, n, S, a, (const L4DLosWork*)work, g_loss, g_w);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// the depth / intensity / ray-drop evaluation meters (l4d_imgmetrics.cuh)
// =============================================================================
extern "C" size_t l4d_image_metrics_work_bytes(uint32_t H, uint32_t W) { return l4d_im_layout(H, W).total; }

extern "C" int l4d_image_metrics(const float* pred, const float* gt, uint32_t H, uint32_t W, float lo, float hi, float peak,
                                 double* out, void* work, size_t work_bytes, void* stream) {
  if (!pred || !gt || !out || !work) return l4d_fail(L4D_EINVAL, "l4d_image_metrics: null pointer");
  if (H < L4D_IM_WIN || W < L4D_IM_WIN || (uint64_t)H * W >= (1ull << 31))
    return l4d_fail(L4D_EINVAL, "l4d_image_metrics: need 7 <= H, W and H*W < 2^31");
  if ((uintptr_t)work & 15) return l4d_fail(L4D_EINVAL, "l4d_image_metrics: work must be 16-byte aligned");
  if (work_bytes < l4d_im_layout(H, W).total) return l4d_fail(L4D_ESIZE, "l4d_image_metrics: work buffer too small");
  cudaStream_t st = (cudaStream_t)stream;
  char* wk = (char*)work;
  ++g_launches; k_im_columns<<<nblk(W, L4D_IM_COL_NT), L4D_IM_COL_NT, 0, st>>>(pred, gt, H, W, lo, hi, wk);
  L4D_CUDA(cudaGetLastError());
  ++g_launches; k_im_rows<<<nblk(5 * (size_t)H, L4D_IM_ROW_NT), L4D_IM_ROW_NT, 0, st>>>(H, W, wk);
  L4D_CUDA(cudaGetLastError());
  const size_t crop = (size_t)(H - 2 * L4D_IM_R) * (W - 2 * L4D_IM_R);
  const int parts = nblk(crop, L4D_IM_SSIM_NT) < L4D_IM_PARTS ? nblk(crop, L4D_IM_SSIM_NT) : L4D_IM_PARTS;
  ++g_launches; k_im_ssim<<<parts, L4D_IM_SSIM_NT, 0, st>>>(H, W, wk);
  L4D_CUDA(cudaGetLastError());
  ++g_launches; k_im_finish<<<1, L4D_IM_FIN_NT, 0, st>>>(H, W, (uint32_t)parts, peak, wk, out);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_raydrop_metrics(const float* pred, const float* gt, uint32_t n, float ratio, double* out, void* stream) {
  if (!pred || !gt || !out) return l4d_fail(L4D_EINVAL, "l4d_raydrop_metrics: null pointer");
  if (n == 0 || n >= (1u << 31)) return l4d_fail(L4D_EINVAL, "l4d_raydrop_metrics: need 1 <= n < 2^31");
  ++g_launches; k_raydrop<<<1, L4D_IM_FIN_NT, 0, (cudaStream_t)stream>>>(pred, gt, n, ratio, out);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// LiDAR sweep images of the simulator, Trainer.test and the validation panel (l4d_sweep.cuh)
// =============================================================================
extern "C" int l4d_sweep_images(const float* depth, const float* image, const void* raydrop, uint32_t raydrop_dtype,
                                uint32_t H, uint32_t W, uint32_t layout, float scale, uint32_t test_mask,
                                const uint8_t* lut_intensity, const uint8_t* lut_depth, uint8_t* panel, float* pano,
                                float* intensities, void* stream) {
  if (layout > L4D_SWEEP_EVAL) return l4d_fail(L4D_EINVAL, "l4d_sweep_images: unknown layout");
  if (raydrop_dtype > L4D_SWEEP_F16 || (!raydrop && raydrop_dtype != L4D_SWEEP_F32))
    return l4d_fail(L4D_EINVAL, "l4d_sweep_images: unknown ray-drop dtype (or float16 without a ray-drop map)");
  if (!depth || !image || !panel) return l4d_fail(L4D_EINVAL, "l4d_sweep_images: null pointer");
  if (!lut_intensity || !lut_depth) return l4d_fail(L4D_EINVAL, "l4d_sweep_images: null colour table");
  if (layout != L4D_SWEEP_EVAL && !pano) return l4d_fail(L4D_EINVAL, "l4d_sweep_images: null pano");
  if (layout == L4D_SWEEP_SIM && !intensities) return l4d_fail(L4D_EINVAL, "l4d_sweep_images: null intensities");
  if (H == 0 || W == 0 || (uint64_t)H * W >= (1ull << 31))
    return l4d_fail(L4D_EINVAL, "l4d_sweep_images: need 1 <= H, W and H*W < 2^31");
  L4DSweepArgs A;
  A.depth = depth;
  A.image = image;
  A.raydrop = raydrop;
  A.lut[0] = lut_intensity;
  A.lut[1] = lut_depth;
  A.panel = panel;
  A.pano = pano;
  A.inten = intensities;
  A.hw = H * W;
  A.layout = layout;
  A.is_f16 = raydrop && raydrop_dtype == L4D_SWEEP_F16;
  A.test_mask = test_mask != 0;
  A.scale = scale;
  ++g_launches; k_sweep_images<<<nblk(A.hw, L4D_SWEEP_NT), L4D_SWEEP_NT, 0, (cudaStream_t)stream>>>(A);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// box masking and the BCE loss of the ray-drop refinement loop (l4d_refine.cuh)
// =============================================================================
extern "C" int l4d_box_mask(const float* x, float* out, uint32_t B, uint32_t C, uint32_t H, uint32_t W, const int32_t* boxes,
                            uint32_t n_boxes, void* stream) {
  if (!x || !out) return l4d_fail(L4D_EINVAL, "l4d_box_mask: null pointer");
  if (B == 0 || C == 0 || H == 0 || W == 0 || (uint64_t)B * C * H * W >= (1ull << 31))
    return l4d_fail(L4D_EINVAL, "l4d_box_mask: need 1 <= B, C, H, W and B*C*H*W < 2^31");
  if (n_boxes > L4D_MAX_BOXES) return l4d_fail(L4D_EINVAL, "l4d_box_mask: more than 32 boxes");
  if (n_boxes && !boxes) return l4d_fail(L4D_EINVAL, "l4d_box_mask: null boxes");
  L4DBoxes b;
  b.n = n_boxes;
  for (uint32_t k = 0; k < n_boxes; ++k) {
    const int32_t y0 = boxes[4 * k], x0 = boxes[4 * k + 1], h = boxes[4 * k + 2], w = boxes[4 * k + 3];
    if (y0 < 0 || x0 < 0 || h < 1 || w < 1 || (int64_t)y0 + h > (int64_t)H || (int64_t)x0 + w > (int64_t)W)
      return l4d_fail(L4D_EINVAL, "l4d_box_mask: box outside the image or empty (need y0, x0 >= 0, h, w >= 1, y0+h <= H, x0+w <= W)");
    b.y0[k] = y0; b.x0[k] = x0; b.h[k] = h; b.w[k] = w;
  }
  const uint32_t planes = B * C;
  const dim3 grid((H * W + L4D_BOX_NT - 1) / L4D_BOX_NT, (planes + L4D_BOX_PLANES - 1) / L4D_BOX_PLANES);
  if (grid.y > 65535) return l4d_fail(L4D_EINVAL, "l4d_box_mask: B*C too large");
  ++g_launches; k_box_mask<<<grid, L4D_BOX_NT, 0, (cudaStream_t)stream>>>(x, out, planes, H, W, b);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" size_t l4d_bce_loss_work_bytes(void) { return sizeof(L4DBceWork); }

static int bce_check(const void* pred, uint32_t dtype, const float* target, uint32_t n, const char* who) {
  if (!pred || !target) return l4d_fail(L4D_EINVAL, "%s: null pointer", who);
  if (dtype > L4D_DTYPE_BF16) return l4d_fail(L4D_EINVAL, "%s: unknown pred dtype", who);
  if (n == 0 || n >= (1u << 31)) return l4d_fail(L4D_EINVAL, "%s: need 1 <= n < 2^31", who);
  return L4D_OK;
}

extern "C" int l4d_bce_loss(const void* pred, uint32_t dtype, const float* target, uint32_t n, float* loss, void* work,
                            size_t work_bytes, void* stream) {
  if (int rc = bce_check(pred, dtype, target, n, "l4d_bce_loss")) return rc;
  if (!loss || !work) return l4d_fail(L4D_EINVAL, "l4d_bce_loss: null pointer");
  if (work_bytes < sizeof(L4DBceWork)) return l4d_fail(L4D_ESIZE, "l4d_bce_loss: work buffer too small");
  const size_t per = (size_t)L4D_BCE_NT * L4D_BCE_PER_THREAD;
  const uint32_t parts = (uint32_t)((n + per - 1) / per < L4D_BCE_BLOCKS ? (n + per - 1) / per : L4D_BCE_BLOCKS);
  cudaStream_t st = (cudaStream_t)stream;
  L4DBceWork* wk = (L4DBceWork*)work;
  ++g_launches;
  if (dtype == L4D_DTYPE_F16) k_bce<__half><<<parts, L4D_BCE_NT, 0, st>>>((const __half*)pred, target, n, wk);
  else if (dtype == L4D_DTYPE_BF16) k_bce<__nv_bfloat16><<<parts, L4D_BCE_NT, 0, st>>>((const __nv_bfloat16*)pred, target, n, wk);
  else k_bce<float><<<parts, L4D_BCE_NT, 0, st>>>((const float*)pred, target, n, wk);
  L4D_CUDA(cudaGetLastError());
  ++g_launches; k_bce_finish<<<1, 1024, 0, st>>>(wk, parts, n, loss);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_bce_loss_backward(const void* pred, uint32_t dtype, const float* target, uint32_t n, const float* g_loss,
                                     void* g_pred, void* stream) {
  if (int rc = bce_check(pred, dtype, target, n, "l4d_bce_loss_backward")) return rc;
  if (!g_loss || !g_pred) return l4d_fail(L4D_EINVAL, "l4d_bce_loss_backward: null pointer");
  int grid = nblk(n);
  if (grid > 8 * sm_count()) grid = 8 * sm_count();
  cudaStream_t st = (cudaStream_t)stream;
  ++g_launches;
  if (dtype == L4D_DTYPE_F16)
    k_bce_bwd<__half><<<grid, 256, 0, st>>>((const __half*)pred, target, n, g_loss, (__half*)g_pred);
  else if (dtype == L4D_DTYPE_BF16)
    k_bce_bwd<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)pred, target, n, g_loss, (__nv_bfloat16*)g_pred);
  else
    k_bce_bwd<float><<<grid, 256, 0, st>>>((const float*)pred, target, n, g_loss, (float*)g_pred);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

// =============================================================================
// exact grid nearest-neighbour search and the flow loss of train_step (l4d_nngrid.cuh)
// =============================================================================
extern "C" size_t l4d_nn_grid_bytes(uint32_t n) { return l4d_nng_layout(n).total; }
extern "C" size_t l4d_nn_grid_work_bytes(uint32_t n) { return l4d_nng_work(n).total; }

static int nng_grid(size_t n, int threads, int cap) {
  const int b = nblk(n, threads);
  return b < cap ? (b < 1 ? 1 : b) : cap;
}

extern "C" int l4d_nn_grid_build(const float* xyz, uint32_t n, void* grid, size_t grid_bytes, void* work, size_t work_bytes,
                                 void* stream) {
  if (!xyz || !grid || !work) return l4d_fail(L4D_EINVAL, "l4d_nn_grid_build: null pointer");
  if (n == 0 || n >= (1u << 31)) return l4d_fail(L4D_EINVAL, "l4d_nn_grid_build: need 1 <= n < 2^31");
  const L4DNNGLayout L = l4d_nng_layout(n);
  const L4DNNGWork W = l4d_nng_work(n);
  if (grid_bytes < L.total) return l4d_fail(L4D_ESIZE, "l4d_nn_grid_build: grid buffer too small");
  if (work_bytes < W.total) return l4d_fail(L4D_ESIZE, "l4d_nn_grid_build: work buffer too small");
  if (((uintptr_t)grid | (uintptr_t)work) & 15) return l4d_fail(L4D_EINVAL, "l4d_nn_grid_build: buffers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* g = reinterpret_cast<unsigned char*>(grid);
  unsigned char* w = reinterpret_cast<unsigned char*>(work);
  L4DNNGHeader* H = reinterpret_cast<L4DNNGHeader*>(g);
  uint32_t* start = reinterpret_cast<uint32_t*>(g + L.start);
  float* part = reinterpret_cast<float*>(w + W.bbox);
  uint32_t* cell_of = reinterpret_cast<uint32_t*>(w + W.cell_of);
  uint32_t* cursor = reinterpret_cast<uint32_t*>(w + W.cursor);
  const int bb = nng_grid((size_t)L.budget + 1 > n ? (size_t)L.budget + 1 : n, 256, L4D_NNG_BBOX_BLOCKS);
  const int pb = nng_grid(n, 256, 8 * sm_count());
  ++g_launches; k_nng_bbox<<<bb, 256, 0, st>>>(xyz, n, part, start, L.budget + 1);
  ++g_launches; k_nng_geometry<<<1, 32, 0, st>>>(part, (uint32_t)bb, L.budget, H);
  ++g_launches; k_nng_count<<<pb, 256, 0, st>>>(xyz, n, H, cell_of, start);
  ++g_launches; k_nng_scan<<<1, 1024, 0, st>>>(H, start, cursor);
  ++g_launches; k_nng_scatter<<<pb, 256, 0, st>>>(xyz, n, cell_of, cursor, reinterpret_cast<float4*>(g + L.pts));
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

static int nng_query_check(const void* grid, size_t grid_bytes, uint32_t n, const float* q, uint32_t nq, const int32_t* idx,
                           const char* who) {
  if (!grid || !q || !idx) return l4d_fail(L4D_EINVAL, "%s: null pointer", who);
  if (n == 0 || n >= (1u << 31) || nq == 0 || nq >= (1u << 31)) return l4d_fail(L4D_EINVAL, "%s: need 1 <= n, nq < 2^31", who);
  if (grid_bytes < l4d_nng_layout(n).total) return l4d_fail(L4D_ESIZE, "%s: grid buffer too small for n", who);
  return L4D_OK;
}

extern "C" int l4d_nn_grid_query(const void* grid, size_t grid_bytes, uint32_t n, const float* q, uint32_t nq, float* dist,
                                 int32_t* idx, double* sum_parts, void* stream) {
  if (int rc = nng_query_check(grid, grid_bytes, n, q, nq, idx, "l4d_nn_grid_query")) return rc;
  if (!dist && !sum_parts) return l4d_fail(L4D_EINVAL, "l4d_nn_grid_query: neither dist nor sum_parts given");
  ++g_launches;
  k_nng_query<false><<<nng_grid(nq, L4D_NNG_QT, L4D_FLOW_PARTS), L4D_NNG_QT, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned char*>(grid), l4d_nng_layout(n), q, nullptr, 0, 0.f, nullptr, nq, dist, idx, sum_parts);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_warp_query(const float* pc, const float* flow6, uint32_t n, uint32_t dir, float step, const void* grid,
                                   size_t grid_bytes, uint32_t m, float* warped, int32_t* idx1, double* sum_parts, void* stream) {
  if (int rc = nng_query_check(grid, grid_bytes, m, pc, n, idx1, "l4d_flow_warp_query")) return rc;
  if (!flow6 || !warped || !sum_parts || dir > 1) return l4d_fail(L4D_EINVAL, "l4d_flow_warp_query: null pointer or dir > 1");
  ++g_launches;
  k_nng_query<true><<<nng_grid(n, L4D_NNG_QT, L4D_FLOW_PARTS), L4D_NNG_QT, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned char*>(grid), l4d_nng_layout(m), pc, flow6, 3 * dir, step, warped, n, nullptr, idx1, sum_parts);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_term_backward(const float* warped, uint32_t n, const float* target, uint32_t m, const int32_t* idx1,
                                      const int32_t* idx2, uint32_t dir, float step, const float* g_loss, float* g_flow6,
                                      void* stream) {
  if (!warped || !target || !idx1 || !idx2 || !g_loss || !g_flow6 || dir > 1) return l4d_fail(L4D_EINVAL, "l4d_flow_term_backward: null pointer or dir > 1");
  if (n == 0 || m == 0) return l4d_fail(L4D_EINVAL, "l4d_flow_term_backward: empty point cloud");
  ++g_launches;
  k_flow_term_bwd<<<nng_grid(n > m ? n : m, 256, 8 * sm_count()), 256, 0, (cudaStream_t)stream>>>(warped, n, target, m, idx1, idx2,
                                                                                                3 * dir, step, g_loss, g_flow6);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_ground(const float* flow6, uint32_t n, double* sum_parts, void* stream) {
  if (!flow6 || !sum_parts) return l4d_fail(L4D_EINVAL, "l4d_flow_ground: null pointer");
  if (n >= (1u << 29)) return l4d_fail(L4D_EINVAL, "l4d_flow_ground: n too large");
  ++g_launches; k_flow_ground<<<nng_grid((size_t)n * 6, 256, L4D_FLOW_PARTS), 256, 0, (cudaStream_t)stream>>>(flow6, n * 6, sum_parts);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_ground_backward(const float* flow6, uint32_t n, const float* g_loss, float* g_flow6, void* stream) {
  if (!flow6 || !g_loss || !g_flow6) return l4d_fail(L4D_EINVAL, "l4d_flow_ground_backward: null pointer");
  if (n >= (1u << 29)) return l4d_fail(L4D_EINVAL, "l4d_flow_ground_backward: n too large");
  if (n == 0) return L4D_OK;
  ++g_launches; k_flow_ground_bwd<<<nng_grid((size_t)n * 6, 256, 8 * sm_count()), 256, 0, (cudaStream_t)stream>>>(flow6, n * 6, g_loss, g_flow6);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}

extern "C" int l4d_flow_loss_finish(const double* sum_parts, uint32_t n_chamfer, uint32_t n_ground, float* loss, void* stream) {
  if (!sum_parts || !loss) return l4d_fail(L4D_EINVAL, "l4d_flow_loss_finish: null pointer");
  ++g_launches; k_flow_finish<<<1, 1024, 0, (cudaStream_t)stream>>>(sum_parts, n_chamfer, n_ground, loss);
  L4D_CUDA(cudaGetLastError());
  return L4D_OK;
}
