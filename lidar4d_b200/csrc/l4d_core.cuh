// l4d_core.cuh - per-sample arithmetic of the LiDAR4D hot path, written once as
// __host__ __device__ code.  The sm_90a kernels (l4d_kernels.cu) call these per
// thread (thread == sample); tests/hostsim compiles the same functions for the
// host so the math can be checked against the oracle without a GPU.  The host
// build is TEST infrastructure only - the product has no CPU path.
//
// Reference semantics (paths relative to the reference checkout, see also
// SURVEY.md Appendix A):
//   sampling / compositing   model/renderer.py:69-129
//   density / attribute      model/lidar4d.py:139-223
//   hash grids (tcnn spec)   model/hash_field.py:65-88,141-172  [tcnn-ext]
//   hex-planes               model/planes_field.py:56-141
//   flow field               model/flow_field.py:102-130
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include "../../include/lidar4d_b200.h"

#define L4D_HD __host__ __device__ __forceinline__
#define L4D_H 64            // hidden width of every MLP (asserted on the host)
#define L4D_GEO 15
#define L4D_ENC 72          // 3 * 2 * view_degree(12)
#define L4D_FLOW_IN 16
#define L4D_PI_F 3.14159274101257324219f
#define L4D_HALF_PI_F 1.57079637050628662109f

// ---------------------------------------------------------------------------
// exact-rounding helpers: the reference is a graph of separate fp32 ops; where
// a fused multiply-add would change a result that is later amplified (hash cell
// selection, large-argument sin) the op order is pinned.
// ---------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define L4D_MUL(a, b) __fmul_rn((a), (b))
#define L4D_ADD(a, b) __fadd_rn((a), (b))
#define L4D_SUB(a, b) __fsub_rn((a), (b))
#define L4D_DIV(a, b) __fdiv_rn((a), (b))
#else
static inline float l4d_opaque(float v) { volatile float t = v; return t; }
#define L4D_MUL(a, b) l4d_opaque((a) * (b))
#define L4D_ADD(a, b) l4d_opaque((a) + (b))
#define L4D_SUB(a, b) l4d_opaque((a) - (b))
#define L4D_DIV(a, b) l4d_opaque((a) / (b))
#endif

// ---------------------------------------------------------------------------
// device-side model description (passed by value as a __grid_constant__ kernel
// parameter, < 4 KB together with the frame constants)
// ---------------------------------------------------------------------------
struct DevGrid {
  float    scale[L4D_MAX_LEVELS];
  uint32_t res[L4D_MAX_LEVELS];
  uint32_t entries[L4D_MAX_LEVELS];
  uint32_t offset[L4D_MAX_LEVELS + 1];
  uint32_t n_levels;
};

struct DevModel {
  DevGrid gs, gd[3], gf;
  const __half* hs;             // static table   [entries][4]
  const __half* hd[3];          // dynamic tables [pair k = slices k,k+1][entries][lo 4 | hi 4]
  const __half* hf;             // flow table     [entries][8]
  uint32_t hd_slice_entries[3]; // entries per time slice
  // optional, per launch (split pipeline): the dynamic tables contracted with the frame's time constants, ONE fp32 per
  // entry and time query (cur, fwd, bwd): con[e] = sum_k basis[k] * (w_lo * T_lo[e][k] + w_hi * T_hi[e][k]).  Every sample
  // of a launch shares the frame, and the feature is linear in the table, so k_contract_dynamic does this once per entry
  // instead of once per corner of every sample, and the gather reads 4 bytes per corner instead of a 16-byte pair record.
  const float* hd_con[3][3];    // [plane][query][entries]; nullptr = gather from the pair records
  // same idea for the three time planes (x,t) (y,t) (z,t) of every scale: the time coordinate of a query is a launch
  // constant, so its two plane rows are blended once (k_contract_planes) into ONE row [R][8] per (scale, plane, query) and a
  // sample reads 2 texels instead of 4.  Indexed [scale][0..2 = planes 2,4,5][query cur|fwd|bwd].
  const float* pl_con[L4D_MAX_PLANE_SCALES][3][3];
  const float* planes[L4D_MAX_PLANE_SCALES][6];   // channels-last [H][W][8]
  uint32_t plane_res[L4D_MAX_PLANE_SCALES];
  uint32_t n_scales, time_res;
  // MLP weights, fp32.  "t" = in-major [in][out]; plain = native [out][in].
  const float *sig_w1t, *sig_w2t, *sig_w2;
  const float *att_w1t[2], *att_w2t[2], *att_w2[2], *att_w3[2];   // net 0 = raydrop, 1 = intensity
  const float *flo_w0t, *flo_w1t, *flo_w1, *flo_w2t, *flo_w2;
  // fp16 copies in the wgmma K-major interleaved layout [k/8][row n][8 halves] (element (n,k) = W[n][k])
  const __half *tc_sig_w1, *tc_sig_w2, *tc_att_w1g, *tc_att_w2[2], *tc_att_w1g_net[2];
  const __half *tc_flo_w0, *tc_flo_w1, *tc_flo_w2;     // [2][64][8], [8][64][8], [8][16][8] (rows 6..15 zero)
  uint32_t mlp_fp16;
  uint32_t sigma_in_dim, sigma_in_pad, attr_in_dim, attr_in_pad, view_degree, active_sensor;
  float bound, near_lidar, far_lidar, density_scale;
};

// gradient sinks used by the backward pass
struct DevGrads {
  float* hs;                                   // [entries][4] fp32
  float* hd[3][L4D_MAX_TIME_SLICES];           // per slice [entries][4]
  float* hf;                                   // [entries][8]
  // optional work accumulators (split pipeline): every sample of a launch shares the frame, hence the time-slice
  // weights and the Lagrange basis, so the scatter kernels reduce the slice- / basis-independent part once per corner
  // and k_fold_* distributes it afterwards: half the reductions.
  float* hd_comb[3];                           // [entries]  sum of w_corner * d (before the time basis and the slice weights)
  float* hf_comb;                              // [entries][2]  sum of w_corner * dFin[2l + c]   (before the basis)
  // time-plane gradient rows [R][8] per (scale, plane 2|4|5, query): sum of w_x * g before the two time-row weights of the
  // query, which k_fold_planes applies (half the reductions of the time-plane sinks)
  float* pl_rows[L4D_MAX_PLANE_SCALES][3][3];
  float* planes_cl[L4D_MAX_PLANE_SCALES][6];   // channels-last work grads
  float *sig_w1t, *sig_w2;                     // [in_pad][64], [16][64]
  float *att_w1t[2], *att_w2t[2], *att_w3[2];  // [96][64], [64][64], [64]
  float *flo_w0t, *flo_w1t, *flo_w2;           // [16][64], [64][64], [8][64]
};

// where the training-mode forward saves what the backward needs, and what the kernels of the split pipeline hand
// to each other.  SoA planes hold P = n_rays*n_steps floats each -> every warp store / load is one 128 B line
struct SavedView {
  float* feat;      // [sigma_in_dim][P]   (fp32-FMA dense kernels)
  unsigned char* feat_tc;   // same region in the tensor-core path: per 128-sample tile of a ray, the fp16 operand tile
                            // itself: [ray][tile][hi|lo][k/8][128 rows][8 halves]  -> one bulk copy into shared memory
  float* flow_in;   // [16][P]
  float* sigma;     // [P]
  float* attr;      // [2][P]
  float* hidden;    // [ctas][64][NT] per-CTA scratch of the dense backward kernel
  float* flow;      // [6][P]   flow-field output (split pipeline: the scatter kernel needs the warped positions)
  float* dfeat;     // dL/dfeature, dense backward -> scatter kernels: [ray][tile][k/4][128 rows][4] (float4 per row)
  float* dflow;     // [6][P]   dL/dflow, scatter kernel -> flow backward kernel
  float* tstart;    // [ray][tile] transmittance at the start of every 128-sample tile (tensor-core dense kernels)
  size_t P;
  uint32_t n_tiles;   // 128-sample tiles per ray
  uint32_t x_chunks;  // stored 16-byte chunks per row of a feature tile = ceil(sigma_in_dim / 8)
  uint32_t d_quads;   // float4 per row of a dfeat tile = ceil(sigma_in_dim / 4)
};

// float offset of (sample j of ray, feature 0) in the dfeat tiles; feature k lives at + (k >> 2) * 512 + (k & 3)
L4D_HD size_t l4d_dfeat_off(const SavedView& sv, uint32_t ray, uint32_t j) {
  return (((size_t)ray * sv.n_tiles + (j >> 7)) * sv.d_quads * 128 + (j & 127)) * 4;
}
L4D_HD size_t l4d_dfeat_k(int k) { return (size_t)(k >> 2) * 512 + (size_t)(k & 3); }
// byte offset of the hi half of the feature tile holding sample j of ray, at the sample's row (chunk 0)
L4D_HD size_t l4d_feat_tc_off(const SavedView& sv, uint32_t ray, uint32_t j) {
  return ((size_t)ray * sv.n_tiles + (j >> 7)) * ((size_t)sv.x_chunks * 4096) + (size_t)(j & 127) * 16;
}

// ---------------------------------------------------------------------------
// small load / reduce wrappers (device: read-only path + vector RED; host: plain)
// ---------------------------------------------------------------------------
L4D_HD float4 l4d_ld4(const float* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(reinterpret_cast<const float4*>(p));
#else
  return *reinterpret_cast<const float4*>(p);
#endif
}
L4D_HD float l4d_ld1(const float* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}
L4D_HD uint2 l4d_ld_u2(const void* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(reinterpret_cast<const uint2*>(p));
#else
  return *reinterpret_cast<const uint2*>(p);
#endif
}
L4D_HD uint4 l4d_ld_u4(const void* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(reinterpret_cast<const uint4*>(p));
#else
  return *reinterpret_cast<const uint4*>(p);
#endif
}
L4D_HD float2 l4d_h2f(uint32_t packed) {
  __half2 h = *reinterpret_cast<__half2*>(&packed);
  return __half22float2(h);
}
// 16-byte vector reduction (RED.E.ADD.F32x4 on sm_90+): one L2 atomic op per table entry
L4D_HD void l4d_red4(float* p, float a, float b, float c, float d) {
#if defined(__CUDA_ARCH__)
  atomicAdd(reinterpret_cast<float4*>(p), make_float4(a, b, c, d));
#else
  p[0] += a; p[1] += b; p[2] += c; p[3] += d;
#endif
}
L4D_HD void l4d_red1(float* p, float a) {
#if defined(__CUDA_ARCH__)
  atomicAdd(p, a);
#else
  *p += a;
#endif
}

// ---------------------------------------------------------------------------
// hash-grid level addressing [tcnn-ext grid_index / grid_hash]
// ---------------------------------------------------------------------------
struct LevelAddr {
  uint32_t res, entries, mask;  // mask = entries-1 if power of two else 0
  bool hashed;
};

template <int D>
L4D_HD LevelAddr l4d_level_addr(const DevGrid& g, int l) {
  LevelAddr a;
  a.res = g.res[l];
  a.entries = g.entries[l];
  a.mask = ((a.entries & (a.entries - 1u)) == 0u) ? (a.entries - 1u) : 0u;
  uint32_t stride = 1;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (stride <= a.entries) stride *= a.res; else break;
  }
  a.hashed = a.entries < stride;
  return a;
}

template <int D>
L4D_HD uint32_t l4d_grid_index(const LevelAddr& a, uint32_t c0, uint32_t c1, uint32_t c2) {
  uint32_t index;
  if (a.hashed) {
    index = c0;
    if (D > 1) index ^= c1 * 2654435761u;
    if (D > 2) index ^= c2 * 805459861u;
  } else {
    index = c0;
    if (D > 1) index += c1 * a.res;
    if (D > 2) index += c2 * a.res * a.res;
  }
  return a.mask ? (index & a.mask) : (index % a.entries);
}

// pos = fmaf(scale, x, 0.5); cell = (uint32)(int)floor(pos); frac = pos - floor(pos)
L4D_HD void l4d_pos_fract(float scale, float x, uint32_t& cell, float& frac) {
  float pos = fmaf(scale, x, 0.5f);
  float fl = floorf(pos);
  cell = (uint32_t)(int)fl;
  frac = pos - fl;
}

// 3D level: 8 corner indices + weights (weight = ((1*f0)*f1)*f2)
L4D_HD void l4d_corners3(const DevGrid& g, int l, float x, float y, float z, uint32_t idx[8], float w[8]) {
  LevelAddr a = l4d_level_addr<3>(g, l);
  uint32_t cx, cy, cz; float fx, fy, fz;
  float s = g.scale[l];
  l4d_pos_fract(s, x, cx, fx);
  l4d_pos_fract(s, y, cy, fy);
  l4d_pos_fract(s, z, cz, fz);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float wx = (c & 1) ? fx : 1.0f - fx;
    float wy = (c & 2) ? fy : 1.0f - fy;
    float wz = (c & 4) ? fz : 1.0f - fz;
    w[c] = (wx * wy) * wz;
    idx[c] = l4d_grid_index<3>(a, cx + (c & 1), cy + ((c >> 1) & 1), cz + ((c >> 2) & 1));
  }
}

L4D_HD void l4d_corners2(const DevGrid& g, int l, float x, float y, uint32_t idx[4], float w[4]) {
  LevelAddr a = l4d_level_addr<2>(g, l);
  uint32_t cx, cy; float fx, fy;
  float s = g.scale[l];
  l4d_pos_fract(s, x, cx, fx);
  l4d_pos_fract(s, y, cy, fy);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float wx = (c & 1) ? fx : 1.0f - fx;
    float wy = (c & 2) ? fy : 1.0f - fy;
    w[c] = wx * wy;
    idx[c] = l4d_grid_index<2>(a, cx + (c & 1), cy + ((c >> 1) & 1), 0u);
  }
}

// static 3D grid, F=4 fp16: one 8-byte gather per corner, fp32 blend
L4D_HD void l4d_encode3_f4(const DevGrid& g, const __half* table, int l, float x, float y, float z, float out[4]) {
  uint32_t idx[8]; float w[8];
  l4d_corners3(g, l, x, y, z, idx, w);
  const uint2* base = reinterpret_cast<const uint2*>(table) + g.offset[l];
  uint2 v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = l4d_ld_u2(base + idx[c]);
  out[0] = out[1] = out[2] = out[3] = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float2 a = l4d_h2f(v[c].x), b = l4d_h2f(v[c].y);
    out[0] = fmaf(w[c], a.x, out[0]); out[1] = fmaf(w[c], a.y, out[1]);
    out[2] = fmaf(w[c], b.x, out[2]); out[3] = fmaf(w[c], b.y, out[3]);
  }
}

// flow 3D grid, F=8 fp16: one 16-byte gather per corner
L4D_HD void l4d_encode3_f8(const DevGrid& g, const __half* table, int l, float x, float y, float z, float out[8]) {
  uint32_t idx[8]; float w[8];
  l4d_corners3(g, l, x, y, z, idx, w);
  const uint4* base = reinterpret_cast<const uint4*>(table) + g.offset[l];
  uint4 v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = l4d_ld_u4(base + idx[c]);
#pragma unroll
  for (int i = 0; i < 8; ++i) out[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float2 a = l4d_h2f(v[c].x), b = l4d_h2f(v[c].y), cc = l4d_h2f(v[c].z), d = l4d_h2f(v[c].w);
    out[0] = fmaf(w[c], a.x, out[0]); out[1] = fmaf(w[c], a.y, out[1]);
    out[2] = fmaf(w[c], b.x, out[2]); out[3] = fmaf(w[c], b.y, out[3]);
    out[4] = fmaf(w[c], cc.x, out[4]); out[5] = fmaf(w[c], cc.y, out[5]);
    out[6] = fmaf(w[c], d.x, out[6]); out[7] = fmaf(w[c], d.y, out[7]);
  }
}

// one level of one time-sliced 2D grid at (x,y): blend of slices lo/hi, then the
// cubic Lagrange contraction over the 4 features -> 1 value (hash_field.py:65-88).
// Working layout: "pair" k holds slices k and k+1 of every entry in ONE 16-byte record
// {lo.f0..f3, hi.f0..f3} (fp16), so a corner costs one LDG.128 instead of two LDG.64 - the dynamic
// hash is 2/3 of the forward's divergent gathers.  table = [pair][entries][8 halves].
L4D_HD float l4d_encode2_time(const DevGrid& g, const __half* table, uint32_t slice_entries, uint32_t n_slices,
                              const L4DTimeQuery& q, int l, float x, float y) {
  uint32_t idx[4]; float w[4];
  l4d_corners2(g, l, x, y, idx, w);
  const uint32_t pair = q.slice_lo < n_slices - 1u ? q.slice_lo : n_slices - 2u;
  // idx1 == idx2 (hash_field.py:82): the feature is G_lo alone; expressed as exact 1/0 weights on the pair
  const float wl = q.single ? (q.slice_lo == pair ? 1.0f : 0.0f) : q.w_lo;
  const float wh = q.single ? 1.0f - wl : q.w_hi;
  const uint4* base = reinterpret_cast<const uint4*>(table) + (size_t)pair * slice_entries + g.offset[l];
  uint4 v[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) v[c] = l4d_ld_u4(base + idx[c]);
  float fl[4] = {0.f, 0.f, 0.f, 0.f}, fh[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float2 a = l4d_h2f(v[c].x), b = l4d_h2f(v[c].y), cc = l4d_h2f(v[c].z), d = l4d_h2f(v[c].w);
    fl[0] = fmaf(w[c], a.x, fl[0]); fl[1] = fmaf(w[c], a.y, fl[1]);
    fl[2] = fmaf(w[c], b.x, fl[2]); fl[3] = fmaf(w[c], b.y, fl[3]);
    fh[0] = fmaf(w[c], cc.x, fh[0]); fh[1] = fmaf(w[c], cc.y, fh[1]);
    fh[2] = fmaf(w[c], d.x, fh[2]); fh[3] = fmaf(w[c], d.y, fh[3]);
  }
  if (q.single) {
#pragma unroll
    for (int i = 0; i < 4; ++i) fl[i] = wl != 0.f ? fl[i] : fh[i];
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) fl[i] = wl * fl[i] + wh * fh[i];
  }
  return ((q.basis[0] * fl[0] + q.basis[1] * fl[1]) + q.basis[2] * fl[2]) + q.basis[3] * fl[3];
}

// the time-dependent part of l4d_encode2_time for ONE table entry: rec = pair record {lo f0..f3, hi f0..f3} (fp16) of the
// query's pair; same arithmetic as there with the corner blend factored out (the blend is linear)
L4D_HD uint32_t l4d_time_pair(const L4DTimeQuery& q, uint32_t n_slices) { return q.slice_lo < n_slices - 1u ? q.slice_lo : n_slices - 2u; }
L4D_HD float l4d_contract_entry(uint4 rec, const L4DTimeQuery& q, uint32_t n_slices) {
  const uint32_t pair = l4d_time_pair(q, n_slices);
  const float wl = q.single ? (q.slice_lo == pair ? 1.0f : 0.0f) : q.w_lo;
  const float wh = q.single ? 1.0f - wl : q.w_hi;
  const float2 a = l4d_h2f(rec.x), b = l4d_h2f(rec.y), cc = l4d_h2f(rec.z), d = l4d_h2f(rec.w);
  float fl[4] = {a.x, a.y, b.x, b.y};
  const float fh[4] = {cc.x, cc.y, d.x, d.y};
  if (q.single) {
#pragma unroll
    for (int i = 0; i < 4; ++i) fl[i] = wl != 0.f ? fl[i] : fh[i];
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) fl[i] = wl * fl[i] + wh * fh[i];
  }
  return ((q.basis[0] * fl[0] + q.basis[1] * fl[1]) + q.basis[2] * fl[2]) + q.basis[3] * fl[3];
}
// one level of one contracted dynamic table at (x,y): bilinear blend of four fp32 entries, as four independent 4-byte
// loads (what the gather is short of is requests in flight, not sectors: DESIGN.md 9)
L4D_HD float l4d_encode2_con(const DevGrid& g, const float* con, int l, float x, float y) {
  uint32_t idx[4]; float w[4];
  l4d_corners2(g, l, x, y, idx, w);
  const float* base = con + g.offset[l];
  const float v0 = l4d_ld1(base + idx[0]), v1 = l4d_ld1(base + idx[1]), v2 = l4d_ld1(base + idx[2]), v3 = l4d_ld1(base + idx[3]);
  return fmaf(w[3], v3, fmaf(w[2], v2, fmaf(w[1], v1, w[0] * v0)));
}

// ---------------------------------------------------------------------------
// hex-planes: F.grid_sample(bilinear, align_corners=True, border) on a
// channels-last [H][W][8] fp32 plane (planes_field.py:56-84)
// ---------------------------------------------------------------------------
struct Bilerp {
  int x0, x1, y0, y1;
  float wx0, wx1, wy0, wy1;
  float gx_mult, gy_mult;   // d(pixel coord)/d(input coord) incl. the border clamp (0 when clipped)
};

// coordinate in [0,1] -> pixel position, ATen grid_sampler_compute_source_index
L4D_HD void l4d_axis(float c, int size, int& i0, int& i1, float& w0, float& w1, float& gmult) {
  float g = L4D_SUB(L4D_MUL(c, 2.0f), 1.0f);                     // coords * 2 - 1
  float ix = L4D_MUL(L4D_DIV(L4D_ADD(g, 1.0f), 2.0f), (float)(size - 1));
  float mx = (float)(size - 1);
  gmult = mx;                                                      // (size-1)/2 * 2
  if (ix <= 0.f) { ix = 0.f; gmult = 0.f; }
  else if (ix >= mx) { ix = mx; gmult = 0.f; }
  float f = floorf(ix);
  i0 = (int)f;
  i1 = i0 + 1;
  w1 = ix - f;
  w0 = (f + 1.0f) - ix;
  if (i1 > size - 1) { i1 = size - 1; w1 = 0.f; }                  // out-of-bounds corner contributes 0
}

L4D_HD Bilerp l4d_bilerp(float cx, int W, float cy, int H) {
  Bilerp b;
  l4d_axis(cx, W, b.x0, b.x1, b.wx0, b.wx1, b.gx_mult);
  l4d_axis(cy, H, b.y0, b.y1, b.wy0, b.wy1, b.gy_mult);
  return b;
}

// 8-channel bilinear sample; optionally d(out)/d(cx) (per channel)
template <bool WITH_DX>
L4D_HD void l4d_plane_sample(const float* P, int W, const Bilerp& b, float out[8], float dx[8]) {
  const float* p00 = P + ((size_t)b.y0 * W + b.x0) * 8;
  const float* p01 = P + ((size_t)b.y0 * W + b.x1) * 8;
  const float* p10 = P + ((size_t)b.y1 * W + b.x0) * 8;
  const float* p11 = P + ((size_t)b.y1 * W + b.x1) * 8;
  float4 t00a = l4d_ld4(p00), t00b = l4d_ld4(p00 + 4);
  float4 t01a = l4d_ld4(p01), t01b = l4d_ld4(p01 + 4);
  float4 t10a = l4d_ld4(p10), t10b = l4d_ld4(p10 + 4);
  float4 t11a = l4d_ld4(p11), t11b = l4d_ld4(p11 + 4);
  float nw = b.wx0 * b.wy0, ne = b.wx1 * b.wy0, sw = b.wx0 * b.wy1, se = b.wx1 * b.wy1;
  float a00[8] = {t00a.x, t00a.y, t00a.z, t00a.w, t00b.x, t00b.y, t00b.z, t00b.w};
  float a01[8] = {t01a.x, t01a.y, t01a.z, t01a.w, t01b.x, t01b.y, t01b.z, t01b.w};
  float a10[8] = {t10a.x, t10a.y, t10a.z, t10a.w, t10b.x, t10b.y, t10b.z, t10b.w};
  float a11[8] = {t11a.x, t11a.y, t11a.z, t11a.w, t11b.x, t11b.y, t11b.z, t11b.w};
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    out[c] = ((a00[c] * nw + a01[c] * ne) + a10[c] * sw) + a11[c] * se;
    if (WITH_DX) dx[c] = b.gx_mult * ((a01[c] - a00[c]) * b.wy0 + (a11[c] - a10[c]) * b.wy1);
  }
}

// one texel of a contracted time-plane row (DevModel::pl_con): the y (time) half of the bilinear blend of
// l4d_plane_sample, b = l4d_bilerp(any x, W, tau, T)
L4D_HD float l4d_contract_texel(const float* P, int W, const Bilerp& b, int x, int c) {
  return P[((size_t)b.y0 * W + x) * 8 + c] * b.wy0 + P[((size_t)b.y1 * W + x) * 8 + c] * b.wy1;
}
// 8-channel sample of a contracted row: the x half of the blend; optionally d(out)/d(cx)
template <bool WITH_DX>
L4D_HD void l4d_row_sample(const float* row, const Bilerp& b, float out[8], float dx[8]) {
  const float* p0 = row + (size_t)b.x0 * 8;
  const float* p1 = row + (size_t)b.x1 * 8;
  const float4 t0a = l4d_ld4(p0), t0b = l4d_ld4(p0 + 4), t1a = l4d_ld4(p1), t1b = l4d_ld4(p1 + 4);
  const float a0[8] = {t0a.x, t0a.y, t0a.z, t0a.w, t0b.x, t0b.y, t0b.z, t0b.w};
  const float a1[8] = {t1a.x, t1a.y, t1a.z, t1a.w, t1b.x, t1b.y, t1b.z, t1b.w};
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    out[c] = a0[c] * b.wx0 + a1[c] * b.wx1;
    if (WITH_DX) dx[c] = b.gx_mult * (a1[c] - a0[c]);
  }
}
// scatter g[8] * the x weights into a gradient row (DevGrads::pl_rows)
L4D_HD void l4d_row_scatter(float* Grow, const Bilerp& b, const float g[8]) {
  float* p0 = Grow + (size_t)b.x0 * 8;
  float* p1 = Grow + (size_t)b.x1 * 8;
  l4d_red4(p0, g[0] * b.wx0, g[1] * b.wx0, g[2] * b.wx0, g[3] * b.wx0);
  l4d_red4(p0 + 4, g[4] * b.wx0, g[5] * b.wx0, g[6] * b.wx0, g[7] * b.wx0);
  if (b.wx1 != 0.f) {
    l4d_red4(p1, g[0] * b.wx1, g[1] * b.wx1, g[2] * b.wx1, g[3] * b.wx1);
    l4d_red4(p1 + 4, g[4] * b.wx1, g[5] * b.wx1, g[6] * b.wx1, g[7] * b.wx1);
  }
}

// scatter g[8] * bilinear weights into a channels-last grad plane (2 x 16 B RED per texel)
L4D_HD void l4d_plane_scatter(float* G, int W, const Bilerp& b, const float g[8]) {
  float wgt[4] = {b.wx0 * b.wy0, b.wx1 * b.wy0, b.wx0 * b.wy1, b.wx1 * b.wy1};
  int xs[4] = {b.x0, b.x1, b.x0, b.x1};
  int ys[4] = {b.y0, b.y0, b.y1, b.y1};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (wgt[k] == 0.f) continue;
    float* p = G + ((size_t)ys[k] * W + xs[k]) * 8;
    l4d_red4(p, g[0] * wgt[k], g[1] * wgt[k], g[2] * wgt[k], g[3] * wgt[k]);
    l4d_red4(p + 4, g[4] * wgt[k], g[5] * wgt[k], g[6] * wgt[k], g[7] * wgt[k]);
  }
}

// ---------------------------------------------------------------------------
// MLP building blocks.  Activations travel through a per-thread exchange column
// xb[k*xs] (shared memory on the device, stride = block size: bank-conflict
// free; a plain array with stride 1 on the host).  Weights are read with
// warp-uniform addresses (one broadcast transaction, L1-resident).
// ---------------------------------------------------------------------------
// y[0..64) += sum_{k<n} xb[k] * Wt[k][0..64)       (Wt in-major, 64 floats per row)
L4D_HD void l4d_layer64(float (&y)[L4D_H], const float* xb, int xs, int n, const float* Wt) {
  for (int k = 0; k < n; ++k) {
    float a = xb[k * xs];
    const float* w = Wt + (size_t)k * L4D_H;
#pragma unroll
    for (int q = 0; q < L4D_H / 4; ++q) {
      float4 v = l4d_ld4(w + 4 * q);
      y[4 * q + 0] = fmaf(a, v.x, y[4 * q + 0]);
      y[4 * q + 1] = fmaf(a, v.y, y[4 * q + 1]);
      y[4 * q + 2] = fmaf(a, v.z, y[4 * q + 2]);
      y[4 * q + 3] = fmaf(a, v.w, y[4 * q + 3]);
    }
  }
}
// y[0..64) += a * row[0..64)
L4D_HD void l4d_axpy64(float (&y)[L4D_H], float a, const float* row) {
#pragma unroll
  for (int q = 0; q < L4D_H / 4; ++q) {
    float4 v = l4d_ld4(row + 4 * q);
    y[4 * q + 0] = fmaf(a, v.x, y[4 * q + 0]);
    y[4 * q + 1] = fmaf(a, v.y, y[4 * q + 1]);
    y[4 * q + 2] = fmaf(a, v.z, y[4 * q + 2]);
    y[4 * q + 3] = fmaf(a, v.w, y[4 * q + 3]);
  }
}
// dot(y[0..64), row[0..64))
L4D_HD float l4d_dot64(const float (&y)[L4D_H], const float* row) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
  for (int q = 0; q < L4D_H / 4; ++q) {
    float4 v = l4d_ld4(row + 4 * q);
    s0 = fmaf(y[4 * q + 0], v.x, s0);
    s1 = fmaf(y[4 * q + 1], v.y, s1);
    s2 = fmaf(y[4 * q + 2], v.z, s2);
    s3 = fmaf(y[4 * q + 3], v.w, s3);
  }
  return (s0 + s1) + (s2 + s3);
}
// y[0..NOUT) += sum_{k<n} xb[k] * Wt[k][0..NOUT)   (NOUT = 16 or 8)
template <int NOUT>
L4D_HD void l4d_layer_small(float (&y)[NOUT], const float* xb, int xs, int n, const float* Wt) {
  for (int k = 0; k < n; ++k) {
    float a = xb[k * xs];
    const float* w = Wt + (size_t)k * NOUT;
#pragma unroll
    for (int q = 0; q < NOUT / 4; ++q) {
      float4 v = l4d_ld4(w + 4 * q);
      y[4 * q + 0] = fmaf(a, v.x, y[4 * q + 0]);
      y[4 * q + 1] = fmaf(a, v.y, y[4 * q + 1]);
      y[4 * q + 2] = fmaf(a, v.z, y[4 * q + 2]);
      y[4 * q + 3] = fmaf(a, v.w, y[4 * q + 3]);
    }
  }
}
// relu(y) -> xb, returns nothing; `bits` gets the y>0 pattern (2 x 32)
L4D_HD void l4d_relu_store(const float (&y)[L4D_H], float* xb, int xs, uint32_t& b0, uint32_t& b1) {
  b0 = 0u; b1 = 0u;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    bool on = y[k] > 0.f;
    xb[k * xs] = on ? y[k] : 0.f;
    if (k < 32) b0 |= on ? (1u << k) : 0u; else b1 |= on ? (1u << (k - 32)) : 0u;
  }
}
L4D_HD bool l4d_bit(uint32_t b0, uint32_t b1, int k) { return k < 32 ? ((b0 >> k) & 1u) : ((b1 >> (k - 32)) & 1u); }

// ---------------------------------------------------------------------------
// sampling along the ray (renderer.py:69-89) and the jitter stream
// ---------------------------------------------------------------------------
L4D_HD float l4d_jitter_u(uint64_t seed, uint64_t ray, uint32_t j) {
  uint64_t z = (ray << 32) | (uint64_t)j;
  z = z + seed * 0x9E3779B97F4A7C15ull + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (float)(uint32_t)(z >> 40) * 5.9604644775390625e-08f;   // 2^-24
}

struct RaySampling {
  float near_, far_, span, sample_dist, lin_step;
  uint32_t S, perturb;
  uint64_t seed;
};

L4D_HD RaySampling l4d_make_sampling(float near_, float far_, uint32_t S, uint32_t perturb, uint64_t seed) {
  RaySampling r;
  r.near_ = near_; r.far_ = far_; r.S = S; r.perturb = perturb; r.seed = seed;
  r.span = L4D_SUB(far_, near_);
  r.sample_dist = L4D_DIV(r.span, (float)S);
  r.lin_step = S > 1 ? L4D_DIV(1.0f, (float)(S - 1)) : 0.f;
  return r;
}

// torch.linspace(0,1,S) as the CUDA kernel computes it, then near + span*lin (+ jitter)
L4D_HD float l4d_z(const RaySampling& r, uint64_t ray_global, uint32_t j) {
  // ATen's linspace kernel (RangeFactories.cu): `start + step*i` below the midpoint, `end - step*(S-1-i)` above it; nvcc
  // contracts the latter into ONE fma (tests/golden/cuda_linspace.npz), the former is exact either way
  float lin = (j < r.S / 2) ? L4D_MUL(r.lin_step, (float)j)
                            : fmaf(-r.lin_step, (float)(r.S - 1 - j), 1.0f);
  float z = L4D_ADD(r.near_, L4D_MUL(r.span, lin));
  if (r.perturb) {
    float u = l4d_jitter_u(r.seed, ray_global, j);
    z = L4D_ADD(z, L4D_MUL(L4D_SUB(u, 0.5f), r.sample_dist));
  }
  return z;
}

// clamp(o + d*z, -bound, bound) then (p + bound) / (2 bound)    (renderer.py:88-89, lidar4d.py:141)
L4D_HD float l4d_x01(float o, float d, float z, float bound) {
  float p = L4D_ADD(o, L4D_MUL(d, z));
  p = fminf(fmaxf(p, -bound), bound);
  return L4D_DIV(L4D_ADD(p, bound), L4D_MUL(2.0f, bound));
}

// Frequency encoding of the view direction (per ray): enc[dim*24 + 2k + {0 sin,1 cos}]
L4D_HD float l4d_freq(float d, int k, int phase) {
  float v = L4D_DIV(L4D_ADD(d, 1.0f), 2.0f);
  float xs = L4D_MUL(v, (float)(1u << k));
  float arg = L4D_ADD(L4D_MUL(xs, L4D_PI_F), phase ? L4D_HALF_PI_F : 0.0f);
  return sinf(arg);
}

// ---------------------------------------------------------------------------
// flow field forward (flow_field.py:113-130): grid -> Lagrange -> 16 -> 64 -> 64 -> 6
// ---------------------------------------------------------------------------
// Lagrange-contracted flow-grid features of one sample -> xb[0..16) (and the save plane)
L4D_HD void l4d_flow_inputs(const DevModel& M, const float basis[4], float x, float y, float z,
                            float* xb, int xs, float* save, size_t save_stride) {
#pragma unroll 1
  for (int l = 0; l < 8; ++l) {
    float e[8];
    l4d_encode3_f8(M.gf, M.hf, l, x, y, z, e);
    float v0 = ((basis[0] * e[0] + basis[1] * e[2]) + basis[2] * e[4]) + basis[3] * e[6];
    float v1 = ((basis[0] * e[1] + basis[1] * e[3]) + basis[2] * e[5]) + basis[3] * e[7];
    xb[(2 * l) * xs] = v0;
    xb[(2 * l + 1) * xs] = v1;
    if (save) {
      save[(size_t)(2 * l) * save_stride] = v0;
      save[(size_t)(2 * l + 1) * save_stride] = v1;
    }
  }
}

// fin (already in xb[0..16)) -> flow[6]; returns the relu patterns for the backward
L4D_HD void l4d_flow_mlp(const DevModel& M, float* xb, int xs, float (&flow)[8],
                         uint32_t& m1a, uint32_t& m1b, uint32_t& m2a, uint32_t& m2b) {
  float y[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
  l4d_layer64(y, xb, xs, L4D_FLOW_IN, M.flo_w0t);
  l4d_relu_store(y, xb, xs, m1a, m1b);
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
  l4d_layer64(y, xb, xs, L4D_H, M.flo_w1t);
  l4d_relu_store(y, xb, xs, m2a, m2b);
#pragma unroll
  for (int k = 0; k < 8; ++k) flow[k] = 0.f;
  l4d_layer_small<8>(flow, xb, xs, L4D_H, M.flo_w2t);
}

// ---------------------------------------------------------------------------
// density forward for one sample (lidar4d.py:139-188).  Features are produced
// group by group, pushed through the exchange column into the first sigma layer
// and (training) saved.  Feature order = torch.cat([plane_s, plane_d, hash_s, hash_d]).
// ---------------------------------------------------------------------------
struct FeatSink {
  float* feat;      // SoA base or nullptr
  size_t P;         // plane stride
  size_t p;         // this sample
  float* dense;     // optional dense [sigma_in_dim] row (debug entry point) or nullptr
  unsigned char* tile = nullptr;   // tensor-core path: this sample's row in the hi half of its fp16 feature tile
  uint32_t tile_lo = 0;            // byte distance from the hi half to the lo half
};

#if defined(__CUDA_ARCH__)
// features [row0, row0+n) of one sample as fp16 hi + lo into its operand tile: hi = fp16(x), lo = fp16(x - hi), so
// |hi + lo - x| <= 2^-22 |x| + 2^-25.  Below |x| ~ 2^-3 the residual x - hi is an fp16 subnormal and the absolute 2^-25
// dominates (relative error 6e-5 at |x| = 1e-3, 6e-3 at 1e-5; DESIGN.md 4.2).
// 8-aligned groups are one 16-byte store per half (a warp writes 512 contiguous bytes), 4-aligned groups 8 bytes.
__device__ __forceinline__ void l4d_tile_emit(unsigned char* hi, uint32_t lo_off, int row0, int n, const float* xb, int xs) {
  int i = 0;
  while (i < n) {
    const int k = row0 + i;
    unsigned char* q = hi + (size_t)(k >> 3) * 2048 + (size_t)(k & 7) * 2;
    if ((k & 3) == 0 && i + 4 <= n) {
      const bool full = (k & 7) == 0 && i + 8 <= n;
      uint32_t h[4], l[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (u < 2 || full) {
          const float a = xb[(i + 2 * u) * xs], b = xb[(i + 2 * u + 1) * xs];
          const __half2 hh = __floats2half2_rn(a, b);
          const float2 f = __half22float2(hh);
          const __half2 ll = __floats2half2_rn(a - f.x, b - f.y);
          h[u] = *reinterpret_cast<const uint32_t*>(&hh);
          l[u] = *reinterpret_cast<const uint32_t*>(&ll);
        }
      }
      if (full) {
        *reinterpret_cast<uint4*>(q) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(q + lo_off) = make_uint4(l[0], l[1], l[2], l[3]);
        i += 8;
      } else {
        *reinterpret_cast<uint2*>(q) = make_uint2(h[0], h[1]);
        *reinterpret_cast<uint2*>(q + lo_off) = make_uint2(l[0], l[1]);
        i += 4;
      }
    } else {
      const float a = xb[i * xs];
      const __half hh = __float2half_rn(a);
      *reinterpret_cast<__half*>(q) = hh;
      *reinterpret_cast<__half*>(q + lo_off) = __float2half_rn(a - __half2float(hh));
      i += 1;
    }
  }
}
#endif

// push n feature values (held in the exchange column xb[0..n)) to the sinks and, when ACC, into the
// first sigma layer.  The split pipeline (k_fwd_gather) runs with ACC=false: no MLP registers live
// across the gathers.
template <bool ACC>
L4D_HD void l4d_emit(float (&acc)[L4D_H], const DevModel& M, float* xb, int xs, int row0, int n,
                     const FeatSink& sink) {
  if (sink.feat) {
    for (int i = 0; i < n; ++i) sink.feat[(size_t)(row0 + i) * sink.P + sink.p] = xb[i * xs];
  }
#if defined(__CUDA_ARCH__)
  if (sink.tile) l4d_tile_emit(sink.tile, sink.tile_lo, row0, n, xb, xs);
#endif
  if (sink.dense) {
    for (int i = 0; i < n; ++i) sink.dense[row0 + i] = xb[i * xs];
  }
  if (ACC) l4d_layer64(acc, xb, xs, n, M.sig_w1t + (size_t)row0 * L4D_H);
}

// weights of the neighbour aggregation 0.5*cur + 0.25*(fwd+bwd) with the
// missing neighbour replaced by cur (lidar4d.py:155-176)
L4D_HD void l4d_agg_weights(const L4DFrame& F, float& wc, float& wf, float& wb) {
  wf = F.has_fwd ? 0.25f : 0.f;
  wb = F.has_bwd ? 0.25f : 0.f;
  wc = 0.5f + (F.has_fwd ? 0.f : 0.25f) + (F.has_bwd ? 0.f : 0.25f);
}

// all encoder features of one sample given its flow; order = cat([plane_s, plane_d, hash_s, hash_d]).
// STATIC_HASH = false leaves out the static-hash rows: the split pipeline gathers them level-major (l4d_static_sweep, l4d_split.cuh).
template <bool ACC, bool STATIC_HASH = true>
L4D_HD void l4d_gather_features(const DevModel& M, const L4DFrame& F, float x, float y, float z, const float (&flow)[8],
                                float* xb, int xs, const FeatSink& sink, float (&acc)[L4D_H]) {
  const int nS = (int)M.n_scales;
  const int L = (int)M.gs.n_levels;
  const int row_plane_d = nS * 8;
  const int row_hash_s = 2 * nS * 8;
  const int row_hash_d = row_hash_s + L * 4;
  float wc, wf, wb;
  l4d_agg_weights(F, wc, wf, wb);
  const float xf0 = x + flow[0], xf1 = y + flow[1], xf2 = z + flow[2];     // lidar4d.py:158
  const float xw0 = x + flow[3], xw1 = y + flow[4], xw2 = z + flow[5];     // lidar4d.py:167

  // ---- hex-planes (planes_field.py:87-141) ----
#pragma unroll 1
  for (int s = 0; s < nS; ++s) {
    const int R = (int)M.plane_res[s];
    const int T = (int)M.time_res;
    // static: planes 0 (x,y), 1 (x,z), 3 (y,z) of itertools.combinations(range(4),2)
    {
      float v0[8], v1[8], v2[8], dummy[8];
      Bilerp b0 = l4d_bilerp(x, R, y, R), b1 = l4d_bilerp(x, R, z, R), b2 = l4d_bilerp(y, R, z, R);
      l4d_plane_sample<false>(M.planes[s][0], R, b0, v0, dummy);
      l4d_plane_sample<false>(M.planes[s][1], R, b1, v1, dummy);
      l4d_plane_sample<false>(M.planes[s][3], R, b2, v2, dummy);
#pragma unroll
      for (int c = 0; c < 8; ++c) xb[c * xs] = (v0[c] * v1[c]) * v2[c];
      l4d_emit<ACC>(acc, M, xb, xs, s * 8, 8, sink);
    }
    // dynamic: planes 2 (x,t), 4 (y,t), 5 (z,t); three queries
    {
      float comb[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) comb[c] = 0.f;
#pragma unroll 1
      for (int qi = 0; qi < 3; ++qi) {
        const float wq = qi == 0 ? wc : (qi == 1 ? wf : wb);
        if (wq == 0.f) continue;
        const float q0 = qi == 0 ? x : (qi == 1 ? xf0 : xw0);
        const float q1 = qi == 0 ? y : (qi == 1 ? xf1 : xw1);
        const float q2 = qi == 0 ? z : (qi == 1 ? xf2 : xw2);
        const float tau = qi == 0 ? F.cur.tau : (qi == 1 ? F.fwd.tau : F.bwd.tau);
        float v0[8], v1[8], v2[8], dummy[8];
        Bilerp b0 = l4d_bilerp(q0, R, tau, T), b1 = l4d_bilerp(q1, R, tau, T), b2 = l4d_bilerp(q2, R, tau, T);
        if (M.pl_con[s][0][0]) {        // contracted rows of this launch (k_contract_planes)
          l4d_row_sample<false>(M.pl_con[s][0][qi], b0, v0, dummy);
          l4d_row_sample<false>(M.pl_con[s][1][qi], b1, v1, dummy);
          l4d_row_sample<false>(M.pl_con[s][2][qi], b2, v2, dummy);
        } else {
          l4d_plane_sample<false>(M.planes[s][2], R, b0, v0, dummy);
          l4d_plane_sample<false>(M.planes[s][4], R, b1, v1, dummy);
          l4d_plane_sample<false>(M.planes[s][5], R, b2, v2, dummy);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) comb[c] = fmaf(wq, (v0[c] * v1[c]) * v2[c], comb[c]);
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) xb[c * xs] = comb[c];
      l4d_emit<ACC>(acc, M, xb, xs, row_plane_d + s * 8, 8, sink);
    }
  }

  // ---- static hash (hash_field.py:141-144) ----
#pragma unroll 1
  for (int l = 0; STATIC_HASH && l < L; ++l) {
    float f[4];
    l4d_encode3_f4(M.gs, M.hs, l, x, y, z, f);
#pragma unroll
    for (int i = 0; i < 4; ++i) xb[i * xs] = f[i];
    l4d_emit<ACC>(acc, M, xb, xs, row_hash_s + l * 4, 4, sink);
  }

  // ---- dynamic hash: planes xy, xz, yz at (x,t), (x+f+,t+), (x+f-,t-) (hash_field.py:146-158) ----
#pragma unroll 1
  for (int p = 0; p < 3; ++p) {
    const float ca = p == 2 ? y : x, cb = p == 0 ? y : z;           // (x,y) (x,z) (y,z)
    const float fa = p == 2 ? xf1 : xf0, fb = p == 0 ? xf1 : xf2;
    const float ba = p == 2 ? xw1 : xw0, bb = p == 0 ? xw1 : xw2;
    const float* const* con = M.hd_con[p];
    if (con[0]) {        // contracted tables of this launch (k_contract_dynamic)
#pragma unroll 1
      for (int l = 0; l < L; ++l) {
        float v = wc * l4d_encode2_con(M.gd[p], con[0], l, ca, cb);
        if (wf != 0.f) v = fmaf(wf, l4d_encode2_con(M.gd[p], con[1], l, fa, fb), v);
        if (wb != 0.f) v = fmaf(wb, l4d_encode2_con(M.gd[p], con[2], l, ba, bb), v);
        xb[l * xs] = v;
      }
    } else {
#pragma unroll 1
      for (int l = 0; l < L; ++l) {
        float v = wc * l4d_encode2_time(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, F.cur, l, ca, cb);
        if (wf != 0.f) v = fmaf(wf, l4d_encode2_time(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, F.fwd, l, fa, fb), v);
        if (wb != 0.f) v = fmaf(wb, l4d_encode2_time(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, F.bwd, l, ba, bb), v);
        xb[l * xs] = v;
      }
    }
    l4d_emit<ACC>(acc, M, xb, xs, row_hash_d + p * L, L, sink);
  }
}

// second sigma layer + trunc_exp from the hidden pre-activations (lidar4d.py:181-183)
L4D_HD void l4d_sigma_head(const DevModel& M, float (&acc)[L4D_H], float* xb, int xs, uint32_t& m0, uint32_t& m1,
                           float& sigma, float& h0_raw, float geo[L4D_GEO]) {
  l4d_relu_store(acc, xb, xs, m0, m1);
  float out[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) out[k] = 0.f;
  l4d_layer_small<16>(out, xb, xs, L4D_H, M.sig_w2t);
  h0_raw = out[0];
  sigma = expf(out[0]);
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) geo[k] = out[1 + k];
}

// fused density of one sample (used by the single-kernel path and the debug entry point)
L4D_HD void l4d_density_sample(const DevModel& M, const L4DFrame& F, float x, float y, float z,
                               float* xb, int xs, const FeatSink& sink, float* flow_in_save, size_t fi_stride,
                               float& sigma, float& h0_raw, float geo[L4D_GEO], float flow_out[6]) {
  // ---- flow (needed first: the warped queries depend on it) ----
  float flow[8];
  {
    l4d_flow_inputs(M, F.flow_basis, x, y, z, xb, xs, flow_in_save, fi_stride);
    uint32_t a, b, c, d;
    l4d_flow_mlp(M, xb, xs, flow, a, b, c, d);
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) flow_out[k] = flow[k];
  float acc[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) acc[k] = 0.f;
  l4d_gather_features<true>(M, F, x, y, z, flow, xb, xs, sink, acc);
  // ---- tcnn pads the MLP input to a multiple of 16 with ones [tcnn-ext] ----
  for (int k = (int)M.sigma_in_dim; k < (int)M.sigma_in_pad; ++k) l4d_axpy64(acc, 1.0f, M.sig_w1t + (size_t)k * L4D_H);
  uint32_t m0, m1;
  l4d_sigma_head(M, acc, xb, xs, m0, m1, sigma, h0_raw, geo);
}

// first sigma layer from features stored as SoA planes (split pipeline / backward recompute)
L4D_HD void l4d_sigma_hidden_from_feats(const DevModel& M, const float* feat, size_t stride, bool active,
                                        float (&acc)[L4D_H]) {
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) acc[k] = 0.f;
  if (active) {
    for (int k = 0; k < (int)M.sigma_in_dim; ++k) l4d_axpy64(acc, feat[(size_t)k * stride], M.sig_w1t + (size_t)k * L4D_H);
    for (int k = (int)M.sigma_in_dim; k < (int)M.sigma_in_pad; ++k) l4d_axpy64(acc, 1.0f, M.sig_w1t + (size_t)k * L4D_H);
  }
}

// ---------------------------------------------------------------------------
// attribute heads for one masked sample (lidar4d.py:207-214).  cdir[net][64] is
// the per-ray part of the first layer: W1[:, :72] @ enc(d) + W1[:, 87:96] @ 1.
// ---------------------------------------------------------------------------
L4D_HD float l4d_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

L4D_HD float l4d_attr_net(const DevModel& M, int net, const float* cdir, const float geo[L4D_GEO],
                          float* xb, int xs) {
  float y[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = cdir[net * L4D_H + k];
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) xb[k * xs] = geo[k];
  l4d_layer64(y, xb, xs, L4D_GEO, M.att_w1t[net] + (size_t)L4D_ENC * L4D_H);
  uint32_t a, b;
  l4d_relu_store(y, xb, xs, a, b);
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
  l4d_layer64(y, xb, xs, L4D_H, M.att_w2t[net]);
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = fmaxf(y[k], 0.f);
  return l4d_sigmoid(l4d_dot64(y, M.att_w3[net]));
}

// per-ray direction term of the first attribute layer, one output unit
L4D_HD float l4d_attr_cdir(const DevModel& M, int net, int o, const float* enc) {
  const float* Wt = M.att_w1t[net];
  float s = 0.f;
  for (int k = 0; k < L4D_ENC; ++k) s = fmaf(enc[k], l4d_ld1(Wt + (size_t)k * L4D_H + o), s);
  for (int k = (int)M.attr_in_dim; k < (int)M.attr_in_pad; ++k) s += l4d_ld1(Wt + (size_t)k * L4D_H + o);
  return s;
}

// alpha of one sample (renderer.py:98-102): 1 - exp(e), formed as -expm1(e).  On long rays alpha is ~1e-5, and
// 1 - expf(e) would keep only the few bits of it above expf's rounding near 1; that error enters every factor of the
// transmittance product behind the sample.
L4D_HD float l4d_alpha(const DevModel& M, float delta, float sigma) {
  float e = M.active_sensor ? (((-2.0f * delta) * M.density_scale) * sigma)
                            : (((-delta) * M.density_scale) * sigma);
  return -expm1f(e);
}
