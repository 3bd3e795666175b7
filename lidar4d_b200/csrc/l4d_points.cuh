// l4d_points.cuh - LiDAR4D.density / .attribute on explicit points with a backward (included by l4d_kernels.cu after
// the block primitives and k_density / k_attribute).  Thread == point, 128-point tiles, grid-stride loops.  The kernels
// compose the per-sample phases of l4d_bwd.cuh the way k_render_bwd does for ray samples; what differs is where the
// upstream gradient comes from (dL/dsigma, dL/dgeo, dL/d(raydrop, intensity) per point instead of the compositing
// backward) and that every point carries its own view direction.
//
// Both MLP modes run here: with mlp_fp16 the fp32 working copies the FMA code reads are already fp16-rounded
// (l4d_stage_params_ex), which is the function the tensor-core path and tiny-cuda-nn evaluate.
#pragma once

// x in [-bound, bound] -> [0,1] (lidar4d.py:141), as k_density does it
__device__ __forceinline__ void l4d_point_x01(const DevModel& M, const float* x, uint32_t i, float& px, float& py, float& pz) {
  const float b2 = L4D_MUL(2.0f, M.bound);
  px = L4D_DIV(L4D_ADD(__ldg(x + 3 * i), M.bound), b2);
  py = L4D_DIV(L4D_ADD(__ldg(x + 3 * i + 1), M.bound), b2);
  pz = L4D_DIV(L4D_ADD(__ldg(x + 3 * i + 2), M.bound), b2);
}

// =============================================================================
// density forward, training variant: k_density's per-point code with the flow-MLP inputs and the sigma-MLP input
// features also written to the saved SoA planes (DensitySavedLayout).  sigma / geo / features / flow are those of
// k_density bit for bit: same l4d_density_sample, the sinks only add stores.
// =============================================================================
struct DensityTrainArgs {
  DevModel M;
  L4DFrame F;
  const float* x;
  uint32_t n;
  float *sigma, *geo, *features, *flow;
  float* flow_in;     // [16][n]
  float* feat;        // [sigma_in_dim][n]
};
template <int NT>
__global__ void __launch_bounds__(NT) k_density_train(const __grid_constant__ DensityTrainArgs A) {
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
  sink.feat = A.feat; sink.P = A.n; sink.p = i;
  sink.dense = A.features ? A.features + (size_t)i * M.sigma_in_dim : nullptr;
  float sigma, h0, geo[L4D_GEO], fl[6];
  l4d_density_sample(M, A.F, x, y, z, xb, NT, sink, A.flow_in + i, A.n, sigma, h0, geo, fl);
  A.sigma[i] = sigma;
  for (int k = 0; k < L4D_GEO; ++k) A.geo[(size_t)i * L4D_GEO + k] = geo[k];
  if (A.flow) for (int k = 0; k < 6; ++k) A.flow[(size_t)i * 6 + k] = fl[k];
}

// =============================================================================
// density backward.  Per tile of NT points:
//   B0  flow MLP recompute from the saved inputs
//   B1  sigma MLP recompute from the saved features, relu(hidden) into this CTA's scratch column block
//   B3  sigma MLP backprop with dsigma = g_sigma[i], dgeo = g_geo[i]      -> dW tiles, dh[64]
//   B4  l4d_bw_scatter<false>: planes (work layout), static hash and the (x,t) slices of the dynamic hash (masters)
//   B5  flow MLP backprop + flow-grid scatter (skipped when the frame has no neighbour: nothing reaches the flow field)
// Weight gradients go through the cooperative tile products into grad_work.  grid <= DensitySavedLayout::ctas.
// =============================================================================
struct DensityBwdArgs {
  DevModel M;
  L4DFrame F;
  DevGrads G;
  const float* x;
  uint32_t n;
  const float* flow_in;   // [16][n]
  const float* feat;      // [sigma_in_dim][n]
  float* hidden;          // [ctas][64][NT]
  const float* g_sigma;   // [n] or null
  const float* g_geo;     // [n][15] or null
};
template <int NT>
__global__ void __launch_bounds__(NT) k_density_bwd(const __grid_constant__ DensityBwdArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;                             // [64][NT]
  float* TA = xbuf + 64 * NT;                     // [NT][LD]
  float* TB = TA + NT * L4D_TILE_LD;              // [NT][LD]
  const DevModel& M = A.M;
  const L4DFrame& F = A.F;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  float* ta_row = TA + (size_t)tid * L4D_TILE_LD;
  float* tb_row = TB + (size_t)tid * L4D_TILE_LD;
  float* hid = A.hidden + (size_t)blockIdx.x * 64 * NT + tid;   // per-CTA scratch column, stride NT
  const int n_chunks = (int)(M.sigma_in_pad + 63) / 64;
  const bool flow_live = F.has_fwd || F.has_bwd;

  for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
    const uint32_t i = base + tid;
    BwSample s;
    s.active = i < A.n;
    s.masked = false;
    s.x = s.y = s.z = 0.f;
    s.dsigma = 0.f; s.da[0] = 0.f; s.da[1] = 0.f;
    const size_t ii = s.active ? i : 0;
    if (s.active) l4d_point_x01(M, A.x, i, s.x, s.y, s.z);
    __syncthreads();                    // the previous tile's last product has read TA / TB

    // B0 / B1
    l4d_bw_flow_fwd(M, s, A.flow_in + ii, A.n, xb, NT);
    l4d_bw_sigma_fwd(M, s, A.feat + ii, A.n, xb, NT, hid, NT);
    if (s.active) {
      s.dsigma = A.g_sigma ? __ldg(A.g_sigma + i) : 0.f;
#pragma unroll
      for (int k = 0; k < L4D_GEO; ++k) s.dgeo[k] = A.g_geo ? __ldg(A.g_geo + (size_t)i * L4D_GEO + k) : 0.f;
    }

    // B3
    l4d_bw_sigma_a(M, s, hid, NT, xb, NT, ta_row, tb_row);
    __syncthreads();
    tile_outer_accum<NT>(TA, TB, 16, G.sig_w2);
    __syncthreads();
    l4d_bw_sigma_b(M, s, xb, NT, tb_row);
#pragma unroll 1
    for (int c = 0; c < n_chunks; ++c) {
      l4d_bw_sigma_c(M, s, A.feat + ii, A.n, c, ta_row);
      __syncthreads();
      const int rows = min(64, (int)M.sigma_in_pad - c * 64);
      tile_outer_accum<NT>(TA, TB, rows, G.sig_w1t + (size_t)c * 64 * 64);
      __syncthreads();
    }

    // B4
    l4d_bw_scatter<false>(M, F, G, s);

    // B5 (block-uniform branch)
    if (flow_live) {
      l4d_bw_flow_a(M, s, A.flow_in + ii, A.n, s.dflow, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 8, G.flo_w2);
      __syncthreads();
      l4d_bw_flow_b(M, s, s.dflow, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 64, G.flo_w1t);
      __syncthreads();
      l4d_bw_flow_c(M, F, G, s, A.flow_in + ii, A.n, xb, NT, ta_row, tb_row);
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 16, G.flo_w0t);
    }
  }
}

// =============================================================================
// attribute backward.  Nothing is saved: the forward is recomputed from d, geo, mask.  Per tile and head (B2):
//   the point's direction part of the first layer, W1[:, :72] enc(d) + W1[:, 87:96] 1, goes into its TB row, where
//   l4d_bw_attr_a reads it before it overwrites the row; steps a / b / c as in k_render_bwd with masked = mask[i] and
//   da = g_out[i].  The direction differs per point, so the 72 encoding rows of dW1 are a per-point outer product
//   enc (x) dh1 (two tile products: rows 64..71 together with the 15 geo rows, then rows 0..63); the 9 ones rows get
//   sum_points dh1, kept per thread (< 64) over the whole grid-stride loop and added once at the end.
// g_geo[i] = sum over both heads of W1g^T dh1 (zero outside the mask).
// =============================================================================
struct AttributeBwdArgs {
  DevModel M;
  DevGrads G;
  const float* d;
  const float* geo;
  const unsigned char* mask;
  uint32_t n;
  const float* g_out;     // [n][2]
  float* g_geo;           // [n][15] or null
};
template <int NT>
__global__ void __launch_bounds__(NT) k_attribute_bwd(const __grid_constant__ AttributeBwdArgs A) {
  extern __shared__ __align__(16) float smem[];
  float* xbuf = smem;                             // [64][NT]
  float* TA = xbuf + 64 * NT;                     // [NT][LD]
  float* TB = TA + NT * L4D_TILE_LD;              // [NT][LD]
  float* encbuf = TB + NT * L4D_TILE_LD;          // [72][NT]
  const DevModel& M = A.M;
  const DevGrads& G = A.G;
  const int tid = threadIdx.x;
  float* xb = xbuf + tid;
  float* ec = encbuf + tid;                       // this point's encoding, stride NT
  float* ta_row = TA + (size_t)tid * L4D_TILE_LD;
  float* tb_row = TB + (size_t)tid * L4D_TILE_LD;
  float csum[2] = {0.f, 0.f};                     // threads < 64: column tid of sum_points dh1, per head

  for (uint32_t base = blockIdx.x * NT; base < A.n; base += gridDim.x * NT) {
    const uint32_t i = base + tid;
    BwSample s;
    s.active = i < A.n;
    s.masked = s.active && (!A.mask || A.mask[i]);
    s.x = s.y = s.z = 0.f;
    s.dsigma = 0.f;
#pragma unroll
    for (int net = 0; net < 2; ++net) s.da[net] = s.masked ? __ldg(A.g_out + 2 * (size_t)i + net) : 0.f;
#pragma unroll
    for (int k = 0; k < L4D_GEO; ++k) {
      s.geo[k] = s.masked ? __ldg(A.geo + (size_t)i * L4D_GEO + k) : 0.f;
      s.dgeo[k] = 0.f;
    }
    {
      const float dx = s.masked ? __ldg(A.d + 3 * (size_t)i) : 0.f;
      const float dy = s.masked ? __ldg(A.d + 3 * (size_t)i + 1) : 0.f;
      const float dz = s.masked ? __ldg(A.d + 3 * (size_t)i + 2) : 0.f;
      for (int k = 0; k < L4D_ENC; ++k) {
        const int dim = k / 24, f = (k % 24) >> 1, ph = k & 1;
        ec[k * NT] = s.masked ? l4d_freq(dim == 0 ? dx : (dim == 1 ? dy : dz), f, ph) : 0.f;
      }
    }
    __syncthreads();                    // the previous tile's last product has read TA / TB

#pragma unroll 1
    for (int net = 0; net < 2; ++net) {
      {
        // direction part of the first layer, summed in l4d_attr_cdir's order
        float y[L4D_H];
#pragma unroll
        for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
        if (s.masked) {
          l4d_layer64(y, ec, NT, L4D_ENC, M.att_w1t[net]);
          for (int k = (int)M.attr_in_dim; k < (int)M.attr_in_pad; ++k) l4d_axpy64(y, 1.0f, M.att_w1t[net] + (size_t)k * L4D_H);
        }
#pragma unroll
        for (int k = 0; k < L4D_H; ++k) tb_row[k] = y[k];
      }
      uint32_t m1a, m1b;
      l4d_bw_attr_a(M, net, s, tb_row - net * L4D_H, xb, NT, ta_row, tb_row, m1a, m1b);
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
      // rows 64..87 of dW1 in one product: enc[64..72) | geo[0..15) | 0
#pragma unroll
      for (int k = 0; k < 8; ++k) ta_row[k] = ec[(64 + k) * NT];
#pragma unroll
      for (int k = 0; k < L4D_GEO; ++k) ta_row[8 + k] = s.geo[k];
      ta_row[8 + L4D_GEO] = 0.f;
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 24, G.att_w1t[net] + (size_t)64 * 64);
      {
        const float cs = tile_colsum<NT>(TB);
        if (tid < 64) csum[net] += cs;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 64; ++k) ta_row[k] = ec[k * NT];
      __syncthreads();
      tile_outer_accum<NT>(TA, TB, 64, G.att_w1t[net]);
      __syncthreads();
    }
    if (s.active && A.g_geo) {
#pragma unroll
      for (int k = 0; k < L4D_GEO; ++k) A.g_geo[(size_t)i * L4D_GEO + k] = s.masked ? s.dgeo[k] : 0.f;
    }
  }
  if (tid < 64) {
#pragma unroll 1
    for (int net = 0; net < 2; ++net)
      for (int k = (int)M.attr_in_dim; k < (int)M.attr_in_pad; ++k) atomicAdd(G.att_w1t[net] + (size_t)k * 64 + tid, csum[net]);
  }
}
