// l4d_split.cuh - the split pipeline (default path).
//
// Why: the single-kernel path (k_render_fwd / k_render_bwd in l4d_kernels.cu) keeps 64-wide MLP
// accumulators live across the irregular gathers / scatters -> 255 registers, 8 warps/SM, and ncu
// shows both kernels latency-bound on long_scoreboard with DRAM at 2% (profiles/r01_v1_*).  Here
// the memory-irregular work runs in lean, high-occupancy kernels (thread == sample, grid-stride,
// no shared memory) and the dense work (MLPs, compositing) in per-ray kernels; they exchange
// ~1.6 KB/sample through the buffers of SavedView (l4d_core.cuh): features as the tensor-core operand tiles
// themselves, dL/dfeature as float4 tiles, the rest as SoA planes [k][P] (every warp access = one 128 B line),
// which the otherwise idle HBM absorbs.  Same per-sample functions (l4d_core.cuh / l4d_bwd.cuh), same numerics.
//
//   forward :  [k_fwd_flow_tc ->] k_fwd_gather -> k_fwd_dense{,_tc}
//   backward:  k_bwd_dense{,_tc} -> k_bwd_scatter + k_bwd_scatter_static -> k_fold_dynamic
//              -> k_bwd_flow  |  k_bwd_flow_tc -> k_bwd_flowgrid -> k_fold_flow
// (the *_tc kernels live in l4d_dense_tc.cuh; DESIGN.md 4.2 has the measured time and limiter of each)
#pragma once
#include "l4d_bwd.cuh"
#include "l4d_core.cuh"

struct SplitArgs {
  DevModel M;
  L4DFrameTable FT;     // frame of every ray (l4d_frame_of); the per-frame tables below sit con_fstride / comb_fstride apart
  size_t con_fstride;   // floats between two frames' contracted tables (DevModel::hd_con, pl_con)
  size_t comb_fstride;  // floats between two frames' accumulators (DevGrads::hd_comb, hf_comb, pl_rows)
  DevGrads G;
  const float* rays_o;
  const float* rays_d;
  uint32_t n_rays, S, perturb, train;
  uint64_t seed, ray_offset;
  float *depth, *image, *wsum, *weights, *zvals;
  const float *g_depth, *g_image, *g_wsum, *g_weights;
  SavedView sv;
};

// static-hash rows of k_fwd_gather, LEVEL-MAJOR (the forward twin of k_bwd_scatter_static).  The fp16 static table is 4 MB per
// hashed level (64 MB at L = 16, more than the H100's 50 MB L2): gathered sample-major, all levels are live at once.  Here every
// CTA sweeps its samples once per level PAIR, so the chip reads 8 MB of the table at a time.  row_hash_s is a multiple of 16,
// so a pair fills one 16-byte chunk of an operand-tile row and a warp stores 512 contiguous bytes per half.  Same per-sample
// function (l4d_encode3_f4) and sink as the sample-major loop of l4d_gather_features: the same bits.
template <int NT, bool TILE, int NL>
__device__ __forceinline__ void l4d_static_sweep(const SplitArgs& A, const RaySampling& rs, int l0, float* xb) {
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const int row0 = 2 * (int)M.n_scales * 8 + 4 * l0;
  for (size_t base = (size_t)blockIdx.x * NT; base < P; base += (size_t)gridDim.x * NT) {
    const size_t p = base + threadIdx.x;
    if (p >= P) continue;
    const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
    const float zj = l4d_z(rs, A.ray_offset + ray, j);
    const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
    const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
    const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
#pragma unroll
    for (int i = 0; i < NL; ++i) {
      float f[4];
      l4d_encode3_f4(M.gs, M.hs, l0 + i, x, y, z, f);
#pragma unroll
      for (int c = 0; c < 4; ++c) xb[(4 * i + c) * NT] = f[c];
    }
    FeatSink sink;
    sink.feat = TILE ? nullptr : A.sv.feat; sink.P = P; sink.p = p; sink.dense = nullptr;
    sink.tile = TILE ? A.sv.feat_tc + l4d_feat_tc_off(A.sv, ray, j) : nullptr; sink.tile_lo = A.sv.x_chunks * 2048u;
    float dummy[L4D_H];
    l4d_emit<false>(dummy, M, xb, NT, row0, 4 * NL, sink);
  }
}

// -------------------------------------------------------------------------------------------
// forward 1/2: encoders.  thread == sample; writes features, flow-MLP inputs and flow.
// -------------------------------------------------------------------------------------------
// FLOW_GIVEN: the flow was already written by k_fwd_flow_tc; then this kernel has no MLP at all.
// TILE: features go out as the fp16 hi|lo operand tiles of the tensor-core dense kernels (SavedView::feat_tc);
// the sample space is then walked in whole 128-row tiles so the rows past the end of a ray get zeros.
// Two phases, no barrier between them: planes, dynamic hash, padding rows and ones-padding sample-major, then the static hash
// level-major (l4d_static_sweep).  The phases write disjoint bytes of the tiles, so CTAs that finish the first phase early
// start the sweep at once; the grid is persistent and its CTAs get equal shares, so they move through the levels together.
// Occupancy of the MLP-free variant, measured at L = 16 on an H100 80GB HBM3 at a 400 W power limit (ms per launch of 16,384
// rays, first phase alone): 6 CTAs/SM 18.3 (80 registers, 60 B of spill stores), 7: 18.9 (72, 112 B), 8: 19.9 (64, 160 B),
// 10: 22.7 (48, 356 B); the level-major static hash alone, as a kernel of its own: 6.7-6.9 at 53 registers (9 CTAs/SM),
// 8.2 at 12 CTAs/SM (40 registers), 10.3 at 16 (32); both phases in this kernel: 6: 25.3 (80 registers, 20 B of spill
// stores), 8: 34.8 (64, 172 B) -> 6.  The variant that also runs the flow MLP keeps 64 accumulators live and stays at 4.
#ifndef L4D_GATHER_MIN_CTAS
#define L4D_GATHER_MIN_CTAS 6
#endif
// MF: several frames in the launch (l4d_frame_of)
template <int NT, bool FLOW_GIVEN, bool TILE, bool MF>
__global__ void __launch_bounds__(NT, FLOW_GIVEN ? L4D_GATHER_MIN_CTAS : 4) k_fwd_gather(const __grid_constant__ SplitArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xb = smem + threadIdx.x;          // exchange column for the flow MLP, stride NT
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t span = TILE ? A.sv.n_tiles * 128u : A.S;      // index space per ray
  const size_t PP = (size_t)A.n_rays * span;
  const uint32_t lo_off = A.sv.x_chunks * 2048u;
  for (size_t base = (size_t)blockIdx.x * NT; base < PP; base += (size_t)gridDim.x * NT) {
    const size_t pp = base + threadIdx.x;
    if (pp >= PP) continue;
    const uint32_t ray = (uint32_t)(pp / span), j = (uint32_t)(pp % span);
    unsigned char* tile = TILE ? A.sv.feat_tc + l4d_feat_tc_off(A.sv, ray, j) : nullptr;
    if (TILE && j >= A.S) {                 // padding row of the last tile of the ray
      for (uint32_t c = 0; c < 2 * A.sv.x_chunks; ++c) *reinterpret_cast<uint4*>(tile + (size_t)c * 2048) = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const size_t p = (size_t)ray * A.S + j;
    const uint32_t fi = l4d_frame_of<MF>(A.FT, ray);
    const L4DFrame& F = A.FT.frames[fi];
    const float zj = l4d_z(rs, A.ray_offset + ray, j);
    const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
    const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
    const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
    float flow[8];
    if (FLOW_GIVEN) {
#pragma unroll
      for (int k = 0; k < 6; ++k) flow[k] = __ldg(A.sv.flow + (size_t)k * P + p);
      flow[6] = flow[7] = 0.f;
    } else {
      l4d_flow_inputs(M, F.flow_basis, x, y, z, xb, NT, A.sv.flow_in + p, P);
      uint32_t a, b, c, d;
      l4d_flow_mlp(M, xb, NT, flow, a, b, c, d);
#pragma unroll
      for (int k = 0; k < 6; ++k) A.sv.flow[(size_t)k * P + p] = flow[k];
    }
    FeatSink sink;
    sink.feat = TILE ? nullptr : A.sv.feat; sink.P = P; sink.p = p; sink.dense = nullptr;
    sink.tile = tile; sink.tile_lo = lo_off;
    float dummy[L4D_H];
    l4d_gather_features<false, false>(M, F, x, y, z, flow, xb, NT, sink, dummy, fi * A.con_fstride);   // static hash: below
    if (TILE) {                             // tcnn's ones-padding inside the last stored chunk
      for (uint32_t k = M.sigma_in_dim; k < A.sv.x_chunks * 8u; ++k) {
        unsigned char* q = tile + (size_t)(k >> 3) * 2048 + (size_t)(k & 7u) * 2;
        *reinterpret_cast<__half*>(q) = __float2half_rn(k < M.sigma_in_pad ? 1.0f : 0.f);
        *reinterpret_cast<__half*>(q + lo_off) = __float2half_rn(0.f);
      }
    }
  }
  const int L = (int)M.gs.n_levels;
#pragma unroll 1
  for (int l = 0; l + 1 < L; l += 2) l4d_static_sweep<NT, TILE, 2>(A, rs, l, xb);
  if (L & 1) l4d_static_sweep<NT, TILE, 1>(A, rs, L - 1, xb);
}

// -------------------------------------------------------------------------------------------
// forward 2/2: sigma MLP, compositing, attribute heads.  One CTA per ray, tiles of NT samples.
// -------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(NT) k_fwd_dense(const __grid_constant__ SplitArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;
  float* s_enc = xbuf + 64 * NT;
  float* s_cdir = s_enc + 80;
  float* s_w = s_cdir + 128;
  const DevModel& M = A.M;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t S = A.S;
  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
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
      const size_t p = (size_t)ray * S + (valid ? j : 0);
      float zj = 0.f, alpha = 0.f, sigma = 0.f, h0, geo[L4D_GEO];
      {
        float acc[L4D_H];
        l4d_sigma_hidden_from_feats(M, A.sv.feat + p, A.sv.P, valid, acc);
        uint32_t m0, m1;
        l4d_sigma_head(M, acc, xb, NT, m0, m1, sigma, h0, geo);
      }
      if (valid) {
        zj = l4d_z(rs, rg, j);
        const float delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
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
    if (tid == 0) { A.depth[ray] = pd; A.image[2 * ray] = p0; A.image[2 * ray + 1] = p1; A.wsum[ray] = pw; }
  }
}

// -------------------------------------------------------------------------------------------
// backward 1/3: compositing + attribute heads + sigma MLP, weight gradients; writes dL/dfeature.
// -------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(NT) k_bwd_dense(const __grid_constant__ SplitArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;
  float* TA = xbuf + 64 * NT;
  float* TB = TA + NT * L4D_TILE_LD;
  float* s_enc = TB + NT * L4D_TILE_LD;
  float* s_cdir = s_enc + 80;
  float* s_csum = s_cdir + 128;
  float* s_w = s_csum + 128;
  float* s_tstart = s_w + 32;
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  float* ta_row = TA + (size_t)tid * L4D_TILE_LD;
  float* tb_row = TB + (size_t)tid * L4D_TILE_LD;
  float* hid = A.sv.hidden + (size_t)blockIdx.x * 64 * NT + tid;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const uint32_t S = A.S;
  const int n_tiles = (int)((S + NT - 1) / NT);
  const float kk = M.active_sensor ? 2.0f : 1.0f;
  const int n_chunks = (int)(M.sigma_in_pad + 63) / 64;

  for (uint32_t ray = blockIdx.x; ray < A.n_rays; ray += gridDim.x) {
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
    {   // pass 1: transmittance at the start of every tile
      float carry = 1.f;
      for (int t = 0; t < n_tiles; ++t) {
        const uint32_t j = (uint32_t)t * NT + tid;
        float v = 1.f;
        if (j < S) {
          const float zj = l4d_z(rs, rg, j);
          const float delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
          v = (1.0f - l4d_alpha(M, delta, A.sv.sigma[(size_t)ray * S + j])) + 1e-15f;
        }
        if (tid == 0) s_tstart[t] = carry;
        float total;
        block_excl_prod<NT>(v, s_w, total);
        carry *= total;
      }
    }
    __syncthreads();
    float suffix = 0.f;
    for (int t = n_tiles - 1; t >= 0; --t) {
      const uint32_t j = (uint32_t)t * NT + tid;
      BwSample s;
      s.active = j < S;
      const size_t p = (size_t)ray * S + (s.active ? j : 0);
      s.masked = false;
      s.dsigma = 0.f; s.da[0] = 0.f; s.da[1] = 0.f;
      float v = 1.f, alpha = 0.f, gw = 0.f, delta = 0.f;
      if (s.active) {
        const float zj = l4d_z(rs, rg, j);
        delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
        alpha = l4d_alpha(M, delta, A.sv.sigma[p]);
        v = (1.0f - alpha) + 1e-15f;
        gw = gd * zj + gi0 * A.sv.attr[p] + gi1 * A.sv.attr[A.sv.P + p] + gws;
        if (A.g_weights) gw += __ldg(A.g_weights + p);
      }
      float total, qtot;
      const float T = s_tstart[t] * block_excl_prod<NT>(v, s_w, total);
      const float w = alpha * T;
      const float suf = suffix + block_excl_suffix_sum<NT>(gw * w, s_w, qtot);
      suffix += qtot;
      if (s.active) {
        s.dsigma = (gw * T - suf / v) * (kk * delta * M.density_scale) * (1.0f - alpha);
        s.masked = w > 1e-4f;
        if (s.masked) { s.da[0] = w * gi0; s.da[1] = w * gi1; }
      }
      l4d_bw_sigma_fwd(M, s, A.sv.feat + p, A.sv.P, xb, NT, hid, NT);
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
      // dL/dfeature for the scatter kernel
      if (s.active) {
        float* dq = A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j);
        for (int k = 0; k < (int)M.sigma_in_dim; ++k) dq[l4d_dfeat_k(k)] = l4d_dot64(s.dh, M.sig_w1t + (size_t)k * L4D_H);
      }
    }
    for (int i = tid; i < 2 * (L4D_ENC + 9) * 64; i += NT) {
      const int net = i / ((L4D_ENC + 9) * 64);
      const int r = (i / 64) % (L4D_ENC + 9), jx = i & 63;
      const float cs = s_csum[net * 64 + jx];
      if (r < L4D_ENC) atomicAdd(G.att_w1t[net] + (size_t)r * 64 + jx, s_enc[r] * cs);
      else atomicAdd(G.att_w1t[net] + (size_t)(M.attr_in_dim + (r - L4D_ENC)) * 64 + jx, cs);
    }
  }
}

// -------------------------------------------------------------------------------------------
// backward 2/3: scatter dL/dfeature through the encoders (vector REDs), thread == sample.
// -------------------------------------------------------------------------------------------
// H100 80GB HBM3 at a 400 W power limit, L = 16, ms per launch of 16,384 rays: 3 CTAs/SM 27.1 (168 registers, 16 B of spill
// stores), 4: 26.3-26.9 (128, 36 B), 5: 29.4 (96, 224 B) -> 4 (short runs, before the dynamic hash's vertex runs).  With the
// contracted time rows (the benchmark's kernel) at 4: 36.1-36.2 ms (128 registers, 36 B of spill stores) before the vertex
// runs, 31.8-31.9 (128, 48 B) with them; 18.7 with the dynamic hash left out (a scratch build), so the dynamic hash went from
// 17.5 to about 13.2 ms of it.
#ifndef L4D_SCATTER_MIN_CTAS
#define L4D_SCATTER_MIN_CTAS 4
#endif
struct DfeatFromTile {
  const float* base;     // this sample's row in its dfeat tile
  bool on;
  __device__ __forceinline__ float operator()(int k) const { return on ? __ldg(base + l4d_dfeat_k(k)) : 0.f; }
  __device__ __forceinline__ void ld4(int k, float (&o)[4]) const {        // k % 4 == 0: the float4 of the tile row
    const float4 v = on ? __ldg(reinterpret_cast<const float4*>(base + l4d_dfeat_k(k))) : make_float4(0.f, 0.f, 0.f, 0.f);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
};

// the time planes come from the forward's contracted rows (DevModel::pl_con) and reduce into DevGrads::pl_rows, both those of
// the sample's frame
template <int NT, int MIN_CTAS, bool MF>
__global__ void __launch_bounds__(NT, MIN_CTAS) k_bwd_scatter(const __grid_constant__ SplitArgs A) {
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  for (size_t base = (size_t)blockIdx.x * NT; base < P; base += (size_t)gridDim.x * NT) {
    // whole warps stay together (plane gradients are aggregated across lanes); lanes past the end
    // shadow the last sample with zero gradient
    const size_t pp = base + threadIdx.x;
    const bool active = pp < P;
    const size_t p = active ? pp : P - 1;
    const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
    const float zj = l4d_z(rs, A.ray_offset + ray, j);
    const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
    const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
    const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
    float flow[6], dflow[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) flow[k] = A.sv.flow[(size_t)k * P + p];
    DfeatFromTile df{A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j), active};
    const uint32_t fi = l4d_frame_of<MF>(A.FT, ray);
    l4d_bw_scatter_t<true, DfeatFromTile, false, true>(M, A.FT.frames[fi], A.G, x, y, z, flow, df, dflow, active, (int)ray, fi,
                                                       fi * A.con_fstride, fi * A.comb_fstride);
    if (active) {
#pragma unroll
      for (int k = 0; k < 6; ++k) A.sv.dflow[(size_t)k * P + p] = dflow[k];
    }
  }
}

// -------------------------------------------------------------------------------------------
// backward 3/3: flow MLP backprop + flow-grid scatter; tiles of NT consecutive samples.
// -------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(NT) k_bwd_flow(const __grid_constant__ SplitArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;
  float* TA = xbuf + 64 * NT;
  float* TB = TA + NT * L4D_TILE_LD;
  float* xb = xbuf + threadIdx.x;
  float* ta_row = TA + (size_t)threadIdx.x * L4D_TILE_LD;
  float* tb_row = TB + (size_t)threadIdx.x * L4D_TILE_LD;
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  for (size_t base = (size_t)blockIdx.x * NT; base < P; base += (size_t)gridDim.x * NT) {
    const size_t pp = base + threadIdx.x;
    BwSample s;
    s.active = pp < P;
    s.masked = false;
    s.x = s.y = s.z = 0.f;
    const size_t p = s.active ? pp : 0;
    const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
    const L4DFrame& F = A.FT.frames[l4d_frame_of(A.FT, ray)];
    float g[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (s.active) {
      const float zj = l4d_z(rs, A.ray_offset + ray, j);
      s.x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
      s.y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
      s.z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
#pragma unroll
      for (int k = 0; k < 6; ++k) g[k] = A.sv.dflow[(size_t)k * P + p];
    }
    __syncthreads();
    l4d_bw_flow_a_t<true>(M, s, A.sv.flow_in + p, P, g, xb, NT, ta_row, tb_row);   // also records the relu patterns
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 8, A.G.flo_w2);
    __syncthreads();
    l4d_bw_flow_b(M, s, g, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 64, A.G.flo_w1t);
    __syncthreads();
    l4d_bw_flow_c(M, F, A.G, s, A.sv.flow_in + p, P, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 16, A.G.flo_w0t);
  }
}

// -------------------------------------------------------------------------------------------
// backward 4/4 (tensor-core path): flow-grid reductions from dL/d(flow-MLP input), thread == sample.
// Feature (l, 2i+c) of a corner gets basis[i] * w_corner * dFin[2l+c].  The coarse levels (cells wider than
// the span of a warp of consecutive samples) are summed per run of equal cells with segmented warp scans first.
// -------------------------------------------------------------------------------------------
// H100 80GB HBM3 at a 400 W power limit, L = 16, ms per launch of 16,384 rays: bound 4 (64 registers, 8 CTAs/SM resident)
// 5.03, 8 (62) 5.03, 12 (40, 56 B of spills) 5.09, 16 (32, 88 B) 5.18 -> 4.
#ifndef L4D_FLOWGRID_MIN_CTAS
#define L4D_FLOWGRID_MIN_CTAS 4
#endif
template <int NT, bool MF>
__global__ void __launch_bounds__(NT, L4D_FLOWGRID_MIN_CTAS) k_bwd_flowgrid(const __grid_constant__ SplitArgs A) {
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  for (size_t base = (size_t)blockIdx.x * NT; base < P; base += (size_t)gridDim.x * NT) {
    const size_t pp = base + threadIdx.x;
    const bool active = pp < P;
    const size_t p = active ? pp : P - 1;
    const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
    const uint32_t fi = l4d_frame_of<MF>(A.FT, ray);
    const float* b = A.FT.frames[fi].flow_basis;
    const float zj = l4d_z(rs, A.ray_offset + ray, j);
    const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
    const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
    const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
#pragma unroll 1
    for (int l = 0; l < 8; ++l) {
      const float d0 = active ? __ldg(A.sv.flow_in + (size_t)(2 * l) * P + p) : 0.f;
      const float d1 = active ? __ldg(A.sv.flow_in + (size_t)(2 * l + 1) * P + p) : 0.f;
      uint32_t idx[8]; float w[8];
      l4d_corners3(M.gf, l, x, y, z, idx, w);
      float* gb = A.G.hf + (size_t)M.gf.offset[l] * 8;
      float* gc = A.G.hf_comb ? A.G.hf_comb + fi * A.comb_fstride + (size_t)M.gf.offset[l] * 2 : nullptr;   // basis: k_fold_flow
      if (M.gf.res[l] <= 400u) {            // warp-uniform: aggregate runs of equal cells
        uint32_t cx, cy, cz; float fx, fy, fz;
        const float sc = M.gf.scale[l];
        l4d_pos_fract(sc, x, cx, fx); l4d_pos_fract(sc, y, cy, fy); l4d_pos_fract(sc, z, cz, fz);
        // runs never join two frames: their sums go to different accumulators (cell indices stay below 400^3 < 2^26)
        const WarpRuns r = l4d_warp_runs((int)(cx + M.gf.res[l] * (cy + M.gf.res[l] * cz) + (fi << 26)));
        float s0[8], s1[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) { s0[c] = w[c] * d0; s1[c] = w[c] * d1; }
        l4d_seg_sum8(s0, r);
        l4d_seg_sum8(s1, r);
        if (r.tail) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            if (gc) {
              atomicAdd(reinterpret_cast<float2*>(gc + (size_t)idx[c] * 2), make_float2(s0[c], s1[c]));
            } else {
              float* q = gb + (size_t)idx[c] * 8;
              l4d_red4(q, b[0] * s0[c], b[0] * s1[c], b[1] * s0[c], b[1] * s1[c]);
              l4d_red4(q + 4, b[2] * s0[c], b[2] * s1[c], b[3] * s0[c], b[3] * s1[c]);
            }
          }
        }
      } else if (active && gc) {
#pragma unroll
        for (int c = 0; c < 8; ++c) atomicAdd(reinterpret_cast<float2*>(gc + (size_t)idx[c] * 2), make_float2(w[c] * d0, w[c] * d1));
      } else if (active) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          float* q = gb + (size_t)idx[c] * 8;
          l4d_red4(q, w[c] * b[0] * d0, w[c] * b[0] * d1, w[c] * b[1] * d0, w[c] * b[1] * d1);
          l4d_red4(q + 4, w[c] * b[2] * d0, w[c] * b[2] * d1, w[c] * b[3] * d0, w[c] * b[3] * d1);
        }
      }
    }
  }
}

// -------------------------------------------------------------------------------------------
// backward 2b: static-hash reductions, LEVEL-MAJOR.  The fp32 gradient of the static table is 8 MB per level
// (134 MB at L=16, far more than the 50 MB L2): walking all levels per sample makes the reductions miss in L2.
// Here every CTA sweeps the samples once per level, so the whole
// chip works on one level at a time and its gradient slab stays L2-resident.
// -------------------------------------------------------------------------------------------
// The kernel's time follows the reductions it issues (H100: 31.1 ms at 112.6 RED.128 per sample, 35.2 ms at 128).
// L4D_STATIC_VERTEX_RUNS (default 1): every level goes through l4d_static_vertex_scatter_warp: at the coarse levels (0-7 at
// L = 16) consecutive samples share cells or corners, and each distinct vertex of a warp gets one RED (97.4 per sample on the
// benchmark's rays, scripts/red_count.py); at the fine levels one ballot finds no shared vertex and the lanes issue their 8
// corners.  0 selects the former path, kept as the A/B reference while the step-time effect under a power cap is open (DESIGN.md
// 9, item 4): runs of equal cells (l4d_static_scatter_warp) at the levels up to res L4D_STATIC_AGG_RES (113.4 REDs per sample;
// bench.py::red_counts models this path), per-lane REDs above.
// H100 80GB HBM3 at a 400 W power limit, L = 16, ms per launch of 16,384 rays: former path at res 1200 and bound 5 (54
// registers, 9 CTAs/SM resident, no spills) 31.1-31.7, at bound 12 (40 registers, 16 B of spills) 33.4, at 16 (32, 56 B) 40.7,
// aggregation off at bound 12 (40, no spills) 35.2; vertex runs at bound 4 (96 registers, no spills) 27.4, 5 (94, no spills)
// 27.1-27.5, 6 (80, 60 B of spill stores) 31.2, 8 (64, 136 B) not run -> 5 either way.
#ifndef L4D_STATIC_VERTEX_RUNS
#define L4D_STATIC_VERTEX_RUNS 1
#endif
#ifndef L4D_STATIC_AGG_RES
#define L4D_STATIC_AGG_RES 1200
#endif
#ifndef L4D_STATIC_SCATTER_MIN_CTAS
#define L4D_STATIC_SCATTER_MIN_CTAS (L4D_STATIC_VERTEX_RUNS || L4D_STATIC_AGG_RES ? 5 : 8)
#endif
template <int NT>
__global__ void __launch_bounds__(NT, L4D_STATIC_SCATTER_MIN_CTAS) k_bwd_scatter_static(const __grid_constant__ SplitArgs A) {
  const DevModel& M = A.M;
  const size_t P = A.sv.P;
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, A.S, A.perturb, A.seed);
  const int L = (int)M.gs.n_levels;
  const int row_hash_s = 2 * (int)M.n_scales * 8;
#pragma unroll 1
  for (int l = 0; l < L; ++l) {
    float* gbase = A.G.hs + (size_t)M.gs.offset[l] * 4;
    const size_t dk = l4d_dfeat_k(row_hash_s + 4 * l);     // row_hash_s is a multiple of 16: one float4 per level
    for (size_t base = (size_t)blockIdx.x * NT; base < P; base += (size_t)gridDim.x * NT) {
      // whole warps stay together (the warp sinks shuffle); lanes past the end shadow the last sample with zero gradient
      const size_t pp = base + threadIdx.x;
      const bool active = pp < P;
      const size_t p = active ? pp : P - 1;
      const uint32_t ray = (uint32_t)(p / A.S), j = (uint32_t)(p % A.S);
      float4 dd = __ldg(reinterpret_cast<const float4*>(A.sv.dfeat + l4d_dfeat_off(A.sv, ray, j) + dk));
      if (!active) dd = make_float4(0.f, 0.f, 0.f, 0.f);
      const float zj = l4d_z(rs, A.ray_offset + ray, j);
      const float x = l4d_x01(__ldg(A.rays_o + 3 * ray), __ldg(A.rays_d + 3 * ray), zj, M.bound);
      const float y = l4d_x01(__ldg(A.rays_o + 3 * ray + 1), __ldg(A.rays_d + 3 * ray + 1), zj, M.bound);
      const float z = l4d_x01(__ldg(A.rays_o + 3 * ray + 2), __ldg(A.rays_d + 3 * ray + 2), zj, M.bound);
      uint32_t idx[8]; float w[8];
      l4d_corners3(M.gs, l, x, y, z, idx, w);
      uint32_t cx, cy, cz; float fx, fy, fz;
      const float sc = M.gs.scale[l];
      l4d_pos_fract(sc, x, cx, fx); l4d_pos_fract(sc, y, cy, fy); l4d_pos_fract(sc, z, cz, fz);
#if L4D_STATIC_VERTEX_RUNS
      const int cell[3] = {(int)cx, (int)cy, (int)cz};
      l4d_static_vertex_scatter_warp(gbase, idx, w, dd, cell, (int)ray, active);
#else
      if (L4D_STATIC_AGG_RES && M.gs.res[l] <= (uint32_t)L4D_STATIC_AGG_RES) {       // warp-uniform
        // equal keys <=> equal cells for neighbouring lanes (their linear cell indices differ by far less than 2^32)
        l4d_static_scatter_warp(gbase, idx, w, dd, (int)(cx + M.gs.res[l] * (cy + M.gs.res[l] * cz)));
      } else if (active) {
#pragma unroll
        for (int c = 0; c < 8; ++c) l4d_red4(gbase + (size_t)idx[c] * 4, w[c] * dd.x, w[c] * dd.y, w[c] * dd.z, w[c] * dd.w);
      }
#endif
    }
  }
}
