// l4d_modules.cuh - LiDAR4D's encoder and MLP submodules as standalone ops (included by l4d_kernels.cu after
// l4d_points.cuh).  The reference builds LiDAR4D from nn.Modules that user code calls directly (hash_field.py:76-172,
// planes_field.py:198-239, flow_field.py:113-130 and the tiny-cuda-nn encodings / networks); these kernels evaluate one
// such module on [n, D] inputs that are already in [0, 1] (no bound normalisation), and accumulate its gradients.
//
// Thread == point, NT-point tiles, grid-stride loops.  The arithmetic is the render path's: the same corner / bilerp /
// time-blend / MLP device functions of l4d_core.cuh, and the backward phases and gradient sinks of l4d_bwd.cuh.  Both MLP
// modes run on the fp32 FMA code: with mlp_fp16 the fp32 working copies are already fp16-rounded (l4d_stage_params_ex),
// which is the function tiny-cuda-nn and the tensor-core path evaluate (as l4d_points.cuh does).
#pragma once

// cubic Lagrange basis at t with the reference's float32 op order (geometry.lagrange_basis, hash_field.py:70-72):
// nodes i/3 and node differences are python doubles rounded to float32; factors multiplied left to right
__device__ __forceinline__ void l4d_lagrange4(float t, float b[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float p = 1.0f;
    bool first = true;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      if (m == j) continue;
      const float fac = L4D_DIV(L4D_SUB(t, (float)(m / 3.0)), (float)(j / 3.0 - m / 3.0));
      p = first ? fac : L4D_MUL(p, fac);
      first = false;
    }
    b[j] = p;
  }
}

// one level of one raw time slice k of a dynamic table (HashGridT.hash_t[k]): the slice is a half of a pair record
__device__ __forceinline__ void l4d_encode2_slice(const DevGrid& g, const __half* table, uint32_t slice_entries,
                                                  uint32_t n_slices, uint32_t k, int l, float x, float y, float out[4]) {
  uint32_t idx[4]; float w[4];
  l4d_corners2(g, l, x, y, idx, w);
  const uint32_t pair = k < n_slices - 1u ? k : n_slices - 2u;
  const bool hi = k != pair;
  const uint4* base = reinterpret_cast<const uint4*>(table) + (size_t)pair * slice_entries + g.offset[l];
  out[0] = out[1] = out[2] = out[3] = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const uint4 v = l4d_ld_u4(base + idx[c]);
    const float2 a = l4d_h2f(hi ? v.z : v.x), b = l4d_h2f(hi ? v.w : v.y);
    out[0] = fmaf(w[c], a.x, out[0]); out[1] = fmaf(w[c], a.y, out[1]);
    out[2] = fmaf(w[c], b.x, out[2]); out[3] = fmaf(w[c], b.y, out[3]);
  }
}

// d(bilinear sample)/d(cy) per channel, the y counterpart of l4d_plane_sample's WITH_DX term
__device__ __forceinline__ void l4d_plane_dy(const float* P, int W, const Bilerp& b, float dy[8]) {
  const float* p00 = P + ((size_t)b.y0 * W + b.x0) * 8;
  const float* p01 = P + ((size_t)b.y0 * W + b.x1) * 8;
  const float* p10 = P + ((size_t)b.y1 * W + b.x0) * 8;
  const float* p11 = P + ((size_t)b.y1 * W + b.x1) * 8;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    dy[c] = b.gy_mult * ((l4d_ld1(p10 + c) - l4d_ld1(p00 + c)) * b.wx0 + (l4d_ld1(p11 + c) - l4d_ld1(p01 + c)) * b.wx1);
}

// dL/dfeature provider over one row of the caller's upstream gradient, for l4d_bw_dynhash_slice: row r of the module's
// output is g[r - row0]
struct DfeatFromRow {
  const float* g;
  int row0;
  __device__ float operator()(int row) const { return __ldg(g + (row - row0)); }
  __device__ void ld4(int row, float (&o)[4]) const { for (int i = 0; i < 4; ++i) o[i] = (*this)(row + i); }
};

struct ModuleArgs {
  DevModel M;
  DevGrads G;
  L4DTimeQuery q;
  uint32_t module, slice;
  const float* x;       // [n][in_dim]
  uint32_t n, in_dim, out_dim;
  float* out;           // [n][out_dim]           (forward)
  const float* g_out;   // [n][out_dim]           (backward)
  float* g_x;           // [n][in_dim] or null    (backward: planes, MLPs)
};

// planes_field.py:87-141 at one point for one scale: static (x,y)(x,z)(y,z) or dynamic (x,t)(y,t)(z,t)
__device__ __forceinline__ void l4d_mod_planes_scale(const DevModel& M, int s, bool dyn, const float* xt, float f[8]) {
  const int R = (int)M.plane_res[s], T = (int)M.time_res;
  const int ci[3] = {dyn ? 2 : 0, dyn ? 4 : 1, dyn ? 5 : 3};
  float v[3][8], dummy[8];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float ca = dyn ? xt[k] : xt[k == 2 ? 1 : 0], cb = dyn ? xt[3] : xt[k == 0 ? 1 : 2];
    const Bilerp b = l4d_bilerp(ca, R, cb, dyn ? T : R);
    l4d_plane_sample<false>(M.planes[s][ci[k]], R, b, v[k], dummy);
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) f[c] = (v[0][c] * v[1][c]) * v[2][c];
}

// =============================================================================
// forward: one point per thread, every module but the MLPs
// =============================================================================
template <int NT>
__global__ void __launch_bounds__(NT) k_module_fwd(const __grid_constant__ ModuleArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;
  const DevModel& M = A.M;
  const int L = (int)M.gs.n_levels;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < A.n; i += gridDim.x * NT) {
    const float* xi = A.x + (size_t)i * A.in_dim;
    float* o = A.out + (size_t)i * A.out_dim;
    switch (A.module) {
      case L4D_MOD_HASH_STATIC: {
        const float x = __ldg(xi), y = __ldg(xi + 1), z = __ldg(xi + 2);
#pragma unroll 1
        for (int l = 0; l < L; ++l) {
          float f[4];
          l4d_encode3_f4(M.gs, M.hs, l, x, y, z, f);
          for (int k = 0; k < 4; ++k) o[4 * l + k] = f[k];
        }
        break;
      }
      case L4D_MOD_HASH_T0: case L4D_MOD_HASH_T0 + 1: case L4D_MOD_HASH_T0 + 2: {
        const int p = (int)A.module - L4D_MOD_HASH_T0;
        const float a = __ldg(xi), b = __ldg(xi + 1);
#pragma unroll 1
        for (int l = 0; l < L; ++l) o[l] = l4d_encode2_time(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, A.q, l, a, b);
        break;
      }
      case L4D_MOD_HASH_DYNAMIC: {
        const float x = __ldg(xi), y = __ldg(xi + 1), z = __ldg(xi + 2);
#pragma unroll 1
        for (int p = 0; p < 3; ++p) {
          const float a = p == 2 ? y : x, b = p == 0 ? y : z;        // (x,y) (x,z) (y,z)
#pragma unroll 1
          for (int l = 0; l < L; ++l)
            o[p * L + l] = l4d_encode2_time(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, A.q, l, a, b);
        }
        break;
      }
      case L4D_MOD_HASH_SLICE0: case L4D_MOD_HASH_SLICE0 + 1: case L4D_MOD_HASH_SLICE0 + 2: {
        const int p = (int)A.module - L4D_MOD_HASH_SLICE0;
        const float a = __ldg(xi), b = __ldg(xi + 1);
#pragma unroll 1
        for (int l = 0; l < L; ++l) {
          float f[4];
          l4d_encode2_slice(M.gd[p], M.hd[p], M.hd_slice_entries[p], M.time_res, A.slice, l, a, b, f);
          for (int k = 0; k < 4; ++k) o[4 * l + k] = f[k];
        }
        break;
      }
      case L4D_MOD_PLANES_STATIC: case L4D_MOD_PLANES_DYNAMIC: {
        const float xt[4] = {__ldg(xi), __ldg(xi + 1), __ldg(xi + 2), __ldg(xi + 3)};
#pragma unroll 1
        for (int s = 0; s < (int)M.n_scales; ++s) {
          float f[8];
          l4d_mod_planes_scale(M, s, A.module == L4D_MOD_PLANES_DYNAMIC, xt, f);
          for (int c = 0; c < 8; ++c) o[8 * s + c] = f[c];
        }
        break;
      }
      case L4D_MOD_FLOW_GRID: {
        const float x = __ldg(xi), y = __ldg(xi + 1), z = __ldg(xi + 2);
#pragma unroll 1
        for (int l = 0; l < (int)M.gf.n_levels; ++l) {
          float f[8];
          l4d_encode3_f8(M.gf, M.hf, l, x, y, z, f);
          for (int k = 0; k < 8; ++k) o[8 * l + k] = f[k];
        }
        break;
      }
      case L4D_MOD_FLOW: {
        float basis[4];
        l4d_lagrange4(__ldg(A.x + 3), basis);                        // t = xt[0, 3] for every row (flow_field.py:122)
        l4d_flow_inputs(M, basis, __ldg(xi), __ldg(xi + 1), __ldg(xi + 2), xb, NT, nullptr, 0);
        float fl[8];
        uint32_t a, b, c, d;
        l4d_flow_mlp(M, xb, NT, fl, a, b, c, d);
        for (int k = 0; k < 6; ++k) o[k] = fl[k];
        break;
      }
      case L4D_MOD_FREQ: {
#pragma unroll 1
        for (int k = 0; k < L4D_ENC; ++k) {
          const int dim = k / 24, f = (k % 24) >> 1, ph = k & 1;
          o[k] = l4d_freq01(__ldg(xi + dim), f, ph);
        }
        break;
      }
    }
  }
}

// =============================================================================
// backward of the encoders.  Parameter gradients: hash tables straight into the master sinks (DevGrads::hs / hd / hf),
// planes into the channels-last work planes (folded by l4d_unstage_grads).  dL/dxt of the planes into g_x.
// The flow field recomputes its inputs into shared memory and runs k_flow_bwd's phases on them.
// =============================================================================
template <int NT>
__global__ void __launch_bounds__(NT) k_module_bwd(const __grid_constant__ ModuleArgs A) {
  extern __shared__ __align__(16) float smem[];
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int L = (int)M.gs.n_levels;
  if (A.module == L4D_MOD_FLOW) {        // block-uniform: every thread runs the tile loop and its barriers
    float* xbuf = smem;                                  // [64][NT]
    float* TA = xbuf + 64 * NT;                          // [NT][LD]
    float* TB = TA + NT * L4D_TILE_LD;                   // [NT][LD]
    float* fin = TB + NT * L4D_TILE_LD;                  // [16][NT] flow-MLP inputs
    float* xb = xbuf + threadIdx.x;
    float* fi = fin + threadIdx.x;
    float* ta_row = TA + (size_t)threadIdx.x * L4D_TILE_LD;
    float* tb_row = TB + (size_t)threadIdx.x * L4D_TILE_LD;
    L4DFrame F;
    memset(&F, 0, sizeof(F));
    l4d_lagrange4(__ldg(A.x + 3), F.flow_basis);
    for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
      const uint32_t i = base + threadIdx.x;
      BwSample s;
      s.active = i < A.n;
      s.masked = false;
      s.x = s.y = s.z = 0.f;
      float g[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      __syncthreads();                                   // the previous tile's last product has read TA / TB
      if (s.active) {
        s.x = __ldg(A.x + 4 * (size_t)i); s.y = __ldg(A.x + 4 * (size_t)i + 1); s.z = __ldg(A.x + 4 * (size_t)i + 2);
        for (int k = 0; k < 6; ++k) g[k] = __ldg(A.g_out + (size_t)i * 6 + k);
        l4d_flow_inputs(M, F.flow_basis, s.x, s.y, s.z, xb, NT, fi, NT);
      }
      l4d_bw_flow_fwd(M, s, fi, NT, xb, NT);
      l4d_bw_flow_a(M, s, fi, NT, g, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 8, G.flo_w2);
      __syncthreads();
      l4d_bw_flow_b(M, s, g, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 64, G.flo_w1t);
      __syncthreads();
      l4d_bw_flow_c(M, F, G, s, fi, NT, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 16, G.flo_w0t);
    }
    return;
  }
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < A.n; i += gridDim.x * NT) {
    const float* xi = A.x + (size_t)i * A.in_dim;
    const float* go = A.g_out + (size_t)i * A.out_dim;
    switch (A.module) {
      case L4D_MOD_HASH_STATIC: {
        const float x = __ldg(xi), y = __ldg(xi + 1), z = __ldg(xi + 2);
#pragma unroll 1
        for (int l = 0; l < L; ++l) {
          uint32_t idx[8]; float w[8];
          l4d_corners3(M.gs, l, x, y, z, idx, w);
          const float d0 = __ldg(go + 4 * l), d1 = __ldg(go + 4 * l + 1), d2 = __ldg(go + 4 * l + 2), d3 = __ldg(go + 4 * l + 3);
          float* gb = G.hs + (size_t)M.gs.offset[l] * 4;
#pragma unroll
          for (int c = 0; c < 8; ++c) l4d_red4(gb + (size_t)idx[c] * 4, w[c] * d0, w[c] * d1, w[c] * d2, w[c] * d3);
        }
        break;
      }
      case L4D_MOD_HASH_T0: case L4D_MOD_HASH_T0 + 1: case L4D_MOD_HASH_T0 + 2: case L4D_MOD_HASH_DYNAMIC: {
        // the dynamic-hash sink of the point / fused backwards with this call's query as the frame's current one
        L4DFrame F;
        memset(&F, 0, sizeof(F));
        F.cur = A.q;
        const bool all = A.module == L4D_MOD_HASH_DYNAMIC;
        const int p0 = all ? 0 : (int)A.module - L4D_MOD_HASH_T0;
        float x = 0.f, y = 0.f, z = 0.f;
        if (all) { x = __ldg(xi); y = __ldg(xi + 1); z = __ldg(xi + 2); }
        else if (p0 == 0) { x = __ldg(xi); y = __ldg(xi + 1); }    // (x,y)
        else if (p0 == 1) { x = __ldg(xi); z = __ldg(xi + 1); }    // (x,z)
        else { y = __ldg(xi); z = __ldg(xi + 1); }                 // (y,z)
        DynHashCursor cur;
        cur.p = p0; cur.l = 0;
        cur.dq[0] = cur.dq[1] = cur.dq[2] = cur.dq[3] = 0.f;
        const DfeatFromRow df{go, all ? 0 : p0 * L};
        l4d_bw_dynhash_slice<false>(M, F, G, x, y, z, 1.0f, df, 0, cur, all ? 3 * L : L, 0, true);
        break;
      }
      case L4D_MOD_HASH_SLICE0: case L4D_MOD_HASH_SLICE0 + 1: case L4D_MOD_HASH_SLICE0 + 2: {
        const int p = (int)A.module - L4D_MOD_HASH_SLICE0;
        const float a = __ldg(xi), b = __ldg(xi + 1);
        float* gs = G.hd[p][A.slice];
#pragma unroll 1
        for (int l = 0; l < L; ++l) {
          uint32_t idx[4]; float w[4];
          l4d_corners2(M.gd[p], l, a, b, idx, w);
          const float d0 = __ldg(go + 4 * l), d1 = __ldg(go + 4 * l + 1), d2 = __ldg(go + 4 * l + 2), d3 = __ldg(go + 4 * l + 3);
          float* gb = gs + (size_t)M.gd[p].offset[l] * 4;
#pragma unroll
          for (int c = 0; c < 4; ++c) l4d_red4(gb + (size_t)idx[c] * 4, w[c] * d0, w[c] * d1, w[c] * d2, w[c] * d3);
        }
        break;
      }
      case L4D_MOD_PLANES_STATIC: case L4D_MOD_PLANES_DYNAMIC: {
        const bool dyn = A.module == L4D_MOD_PLANES_DYNAMIC;
        const float xt[4] = {__ldg(xi), __ldg(xi + 1), __ldg(xi + 2), __ldg(xi + 3)};
        const int ci[3] = {dyn ? 2 : 0, dyn ? 4 : 1, dyn ? 5 : 3};
        // coordinate of plane k along W (a) and H (b): static (x,y)(x,z)(y,z), dynamic (x,t)(y,t)(z,t)
        const int ca[3] = {0, dyn ? 1 : 0, dyn ? 2 : 1};
        const int cb[3] = {dyn ? 3 : 1, dyn ? 3 : 2, dyn ? 3 : 2};
        float gx[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int s = 0; s < (int)M.n_scales; ++s) {
          const int R = (int)M.plane_res[s], T = (int)M.time_res;
          float v[3][8], dx[3][8], d[8];
          Bilerp bl[3];
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            bl[k] = l4d_bilerp(xt[ca[k]], R, xt[cb[k]], dyn ? T : R);
            l4d_plane_sample<true>(M.planes[s][ci[k]], R, bl[k], v[k], dx[k]);
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) d[c] = __ldg(go + 8 * s + c);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int k1 = k == 0 ? 1 : 0, k2 = k == 2 ? 1 : 2;
            float g[8], dy[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) g[c] = d[c] * v[k1][c] * v[k2][c];
            l4d_plane_scatter(G.planes_cl[s][ci[k]], R, bl[k], g);
            if (A.g_x) {
              l4d_plane_dy(M.planes[s][ci[k]], R, bl[k], dy);
              float sa = 0.f, sb = 0.f;
#pragma unroll
              for (int c = 0; c < 8; ++c) { sa = fmaf(g[c], dx[k][c], sa); sb = fmaf(g[c], dy[c], sb); }
              gx[ca[k]] += sa;
              gx[cb[k]] += sb;
            }
          }
        }
        if (A.g_x)
          for (int k = 0; k < 4; ++k) A.g_x[(size_t)i * 4 + k] = gx[k];
        break;
      }
      case L4D_MOD_FLOW_GRID: {
        const float x = __ldg(xi), y = __ldg(xi + 1), z = __ldg(xi + 2);
#pragma unroll 1
        for (int l = 0; l < (int)M.gf.n_levels; ++l) {
          uint32_t idx[8]; float w[8];
          l4d_corners3(M.gf, l, x, y, z, idx, w);
          float d[8];
          for (int k = 0; k < 8; ++k) d[k] = __ldg(go + 8 * l + k);
          float* gb = G.hf + (size_t)M.gf.offset[l] * 8;
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            float* p = gb + (size_t)idx[c] * 8;
            l4d_red4(p, w[c] * d[0], w[c] * d[1], w[c] * d[2], w[c] * d[3]);
            l4d_red4(p + 4, w[c] * d[4], w[c] * d[5], w[c] * d[6], w[c] * d[7]);
          }
        }
        break;
      }
    }
  }
}

// =============================================================================
// the three tcnn networks (lidar4d.py:84,96,108): input [n, n_in] padded with ones to the network width, ReLU hidden
// layers, linear output.  sigma_net -> 16 outputs, the attribute heads -> 1 (the sigmoid is LiDAR4D.attribute's).
// net: 0 sigma, 1 raydrop, 2 intensity (DevModel::att_* index net - 1).
// =============================================================================
struct MlpArgs {
  DevModel M;
  DevGrads G;
  uint32_t net;
  const float* in;      // [n][n_in]
  uint32_t n, n_in, n_out;
  float* out;           // [n][n_out]             (forward)
  const float* g_out;   // [n][n_out]             (backward)
  float* g_in;          // [n][n_in] or null      (backward)
};

// first layer: y = W1 [in | 1] (pre-activation)
__device__ __forceinline__ void l4d_mlp_layer1(const MlpArgs& A, const float* row, float (&y)[L4D_H]) {
  const float* W1t = A.net == 0 ? A.M.sig_w1t : A.M.att_w1t[A.net - 1];
  const int pad = A.net == 0 ? (int)A.M.sigma_in_pad : (int)A.M.attr_in_pad;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
  l4d_layer64(y, row, 1, (int)A.n_in, W1t);
  for (int k = (int)A.n_in; k < pad; ++k) l4d_axpy64(y, 1.0f, W1t + (size_t)k * L4D_H);
}

template <int NT>
__global__ void __launch_bounds__(NT) k_mlp_fwd(const __grid_constant__ MlpArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;
  const DevModel& M = A.M;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < A.n; i += gridDim.x * NT) {
    float y[L4D_H];
    l4d_mlp_layer1(A, A.in + (size_t)i * A.n_in, y);
    uint32_t m0, m1;
    l4d_relu_store(y, xb, NT, m0, m1);
    float* o = A.out + (size_t)i * A.n_out;
    if (A.net == 0) {
      float out[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) out[k] = 0.f;
      l4d_layer_small<16>(out, xb, NT, L4D_H, M.sig_w2t);
      for (int k = 0; k < 16; ++k) o[k] = out[k];
    } else {
      const int h = (int)A.net - 1;
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
      l4d_layer64(y, xb, NT, L4D_H, M.att_w2t[h]);
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) y[k] = fmaxf(y[k], 0.f);
      o[0] = l4d_dot64(y, M.att_w3[h]);
    }
  }
}

// Per tile: recompute the forward, backprop the upstream gradient per thread, weight gradients through the cooperative
// tile products into grad_work (sigma: [in_pad][64] + [16][64]; heads: [96][64] + [64][64] + [64]), dL/din = W1^T dh1.
template <int NT>
__global__ void __launch_bounds__(NT) k_mlp_bwd(const __grid_constant__ MlpArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;                                  // [64][NT]
  float* TA = xbuf + 64 * NT;                          // [NT][LD]
  float* TB = TA + NT * L4D_TILE_LD;                   // [NT][LD]
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  float* ta_row = TA + (size_t)tid * L4D_TILE_LD;
  float* tb_row = TB + (size_t)tid * L4D_TILE_LD;
  const bool sig = A.net == 0;
  const int h = sig ? 0 : (int)A.net - 1;
  const float* W1t = sig ? M.sig_w1t : M.att_w1t[h];
  float* gW1t = sig ? G.sig_w1t : G.att_w1t[h];
  const int pad = sig ? (int)M.sigma_in_pad : (int)M.attr_in_pad;
  const int n_chunks = (pad + 63) / 64;
  for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
    const uint32_t i = base + tid;
    const bool active = i < A.n;
    const float* row = A.in + (size_t)(active ? i : 0) * A.n_in;
    __syncthreads();                                   // the previous tile's last product has read TA / TB
    float y[L4D_H];
    l4d_mlp_layer1(A, row, y);
    uint32_t m1a, m1b;
    l4d_relu_store(y, xb, NT, m1a, m1b);               // h1 -> xb
    float dh[L4D_H];
    if (sig) {
      // dW2[o][k] += dout[o] h1[k]: TA <- dout (16), TB <- h1
#pragma unroll
      for (int k = 0; k < 16; ++k) ta_row[k] = active ? __ldg(A.g_out + (size_t)i * 16 + k) : 0.f;
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) tb_row[k] = active ? xb[k * NT] : 0.f;
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 16, G.sig_w2);
      __syncthreads();
      // dh1 = (W2^T dout) * relu1, W2 native [16][64]
#pragma unroll
      for (int k = 0; k < 16; ++k) xb[k * NT] = ta_row[k];
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) dh[k] = 0.f;
      l4d_layer64(dh, xb, NT, 16, M.sig_w2);
    } else {
      // h2 = relu(W2 h1); out = w3 . h2
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) ta_row[k] = active ? xb[k * NT] : 0.f;        // h1 for dW2t
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
      l4d_layer64(y, xb, NT, L4D_H, M.att_w2t[h]);
      const float d_o = active ? __ldg(A.g_out + i) : 0.f;
      uint32_t m2a = 0u, m2b = 0u;
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) {
        const bool on = y[k] > 0.f;
        if (k < 32) m2a |= on ? (1u << k) : 0u; else m2b |= on ? (1u << (k - 32)) : 0u;
        tb_row[k] = on ? d_o * y[k] : 0.f;                                          // dw3 = colsum
      }
      __syncthreads();
      {
        const float cs = tile_colsum<NT>(TB);
        if (tid < 64) atomicAdd(G.att_w3[h] + tid, cs);
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < L4D_H / 4; ++q) {
        const float4 w3 = l4d_ld4(M.att_w3[h] + 4 * q);
        const float wv[4] = {w3.x, w3.y, w3.z, w3.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int k = 4 * q + u;
          const float v = l4d_bit(m2a, m2b, k) ? wv[u] * d_o : 0.f;                 // dh2
          tb_row[k] = v;
          xb[k * NT] = v;
        }
      }
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 64, G.att_w2t[h]);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < L4D_H; ++k) dh[k] = 0.f;
      l4d_layer64(dh, xb, NT, L4D_H, M.att_w2[h]);                                 // native [o][k]
    }
#pragma unroll
    for (int k = 0; k < L4D_H; ++k) {
      dh[k] = (active && l4d_bit(m1a, m1b, k)) ? dh[k] : 0.f;
      tb_row[k] = dh[k];
    }
    // dW1t[r][k] += [in | 1][r] dh1[k], 64 input rows per product
#pragma unroll 1
    for (int c = 0; c < n_chunks; ++c) {
      for (int k = 0; k < 64; ++k) {
        const int r = c * 64 + k;
        ta_row[k] = (!active || r >= pad) ? 0.f : (r < (int)A.n_in ? __ldg(row + r) : 1.0f);
      }
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, min(64, pad - c * 64), gW1t + (size_t)c * 64 * 64);
      __syncthreads();
    }
    if (active && A.g_in)
      for (int r = 0; r < (int)A.n_in; ++r) A.g_in[(size_t)i * A.n_in + r] = l4d_dot64(dh, W1t + (size_t)r * L4D_H);
  }
}
